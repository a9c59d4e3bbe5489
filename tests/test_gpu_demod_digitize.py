"""GPU parity tests (run with -m gpu on the H100): CUDA afp_demod / grab_pulse_lens / fused path vs the
oracle and the committed golden vectors.  Bit-exact is the bar for ASK/FSK/PSK demodulated samples and for all
pulse tables."""
import numpy as np
import pytest

from conftest import CAPTURES, bits_equal, load_golden, synth_fsk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sf():
    from urh_b200.cythonext import signal_functions

    return signal_functions


@pytest.mark.parametrize("name", CAPTURES)
def test_afp_demod_golden_bit_exact(sf, name):
    g = load_golden("capture_" + name)
    noise = float(g["noise"])
    for mod in ("ASK", "FSK"):
        q = sf.afp_demod(g["iq"], noise, mod, 2)
        assert q.dtype == np.float32 and q.shape == (len(g["iq"]),)
        assert bits_equal(q, g["qad_" + mod]) == 0, (name, mod)


@pytest.mark.parametrize("name", CAPTURES)
def test_afp_demod_psk_golden(sf, name):
    g = load_golden("capture_" + name)
    noise = float(g["noise"])
    for order, key in ((2, "qad_PSK"), (4, "qad_PSK4")):
        q = sf.afp_demod(g["iq"], noise, "PSK", order)
        ref = g[key]
        # Costas loop with glibc's sinf/cosf restated bit-for-bit (glibc_sincosf.h): bit-exact, index 0 is
        # uninitialised memory in the reference (np.empty) and pinned to 0 on both sides
        assert bits_equal(q[1:], ref[1:]) == 0, (name, order)


@pytest.mark.parametrize("dtype", [np.int8, np.uint8, np.int16, np.uint16, np.float32])
@pytest.mark.parametrize("n", [3, 63, 64, 65, 2047, 2048, 2049, 100001])
def test_afp_demod_vs_oracle_sizes_dtypes(sf, oracle, dtype, n):
    iq = synth_fsk(n, sps=20, seed=n, gap_every=500, dtype=dtype)
    iq[n // 3: n // 3 + 5] = 0  # exact zeros exercise the signed-zero bookkeeping of the conj product
    noise = {np.float32: 0.05}.get(dtype, 5.0 if dtype in (np.int8, np.uint8) else 1000.0)
    if dtype in (np.uint8, np.uint16):
        noise = 0.0
    for mod in ("ASK", "FSK"):
        assert bits_equal(sf.afp_demod(iq, noise, mod, 2), oracle.afp_demod(iq, noise, mod, 2)) == 0, (dtype, n, mod)


def test_afp_demod_edge_cases(sf, oracle):
    for n in (0, 1, 2):
        iq = np.ones((n, 2), dtype=np.float32)
        assert np.array_equal(sf.afp_demod(iq, 0.0, "FSK", 2), np.zeros(n, np.float32))
    iq = synth_fsk(1000, seed=5)
    assert bits_equal(sf.afp_demod(iq, 0.0, "QAM", 2), oracle.afp_demod(iq, 0.0, "QAM", 2)) == 0
    with pytest.raises(TypeError):
        sf.afp_demod(iq.astype(np.float64), 0.0, "FSK", 2)
    with pytest.raises(ValueError):
        sf.afp_demod(iq[::2], 0.0, "FSK", 2)  # not C-contiguous
    # misaligned views (odd sample offset) take the scalar load path
    assert bits_equal(sf.afp_demod(iq[1:], 0.02, "FSK", 2), oracle.afp_demod(iq[1:], 0.02, "FSK", 2)) == 0


@pytest.mark.parametrize("name", CAPTURES)
def test_grab_pulse_lens_golden(sf, name):
    g = load_golden("capture_" + name)
    m = g["meta"]
    qad = g["qad_" + m["mod"]]
    for key in [k for k in g if k.startswith("pulses_tol")]:
        tol = int(key[len("pulses_tol"):])
        r = sf.grab_pulse_lens(qad, m["center"], tol, m["mod"], m["sps"], m["bps"], m["spacing"])
        assert r.dtype == np.int64 and np.array_equal(r, g[key]), (name, key)
    r = sf.grab_pulse_lens(qad, m["center"], m["tol"], m["mod"], m["sps"], 2, 0.1)
    assert np.array_equal(r, g["pulses_bps2"])


def test_grab_pulse_lens_randomised_vs_oracle(sf, oracle):
    rng = np.random.default_rng(11)
    for trial in range(150):
        n = int(rng.choice([1, 2, 5, 63, 64, 65, 500, 2047, 2048, 2049, 4097, 20000]))
        mod = ["ASK", "FSK", "PSK"][trial % 3]
        noise_v = 0.0 if mod == "ASK" else -4.0
        period = int(rng.integers(2, 60))
        base = np.repeat(rng.standard_normal(n // period + 1), period)[:n] * 0.5
        x = (base + 0.15 * rng.standard_normal(n)).astype(np.float32)
        x[rng.random(n) < rng.choice([0.0, 0.02, 0.3])] = noise_v
        if n > 10:
            s = int(rng.integers(0, n))
            x[s: s + int(rng.integers(0, 3000))] = noise_v
        tol = int(rng.choice([0, 1, 2, 5, 9, 31, 32, 63, 64, 100, 2500]))
        bps = int(rng.choice([1, 1, 2, 3]))
        sps = int(rng.choice([1, 8, 100]))
        a = sf.grab_pulse_lens(x, 0.05, tol, mod, sps, bps, 0.3)
        b = oracle.grab_pulse_lens(x, 0.05, tol, mod, sps, bps, 0.3)
        assert np.array_equal(a, b), (trial, n, mod, tol, bps, sps, a[:5], b[:5])
        assert a[:, 1].sum() == n - tol or len(a) == 0


def test_grab_pulse_lens_long_runs_cross_tiles(sf, oracle):
    """runs much longer than a tile, tolerance larger than a tile, and constant inputs"""
    n = 50000
    x = np.full(n, -4.0, np.float32)
    x[7000:23000] = 0.5
    x[23000:23003] = -0.5
    x[23003:41000] = 0.5
    for tol in (0, 5, 2047, 2048, 5000, 20000, 60000):
        a = sf.grab_pulse_lens(x, 0.0, tol, "FSK", 100)
        b = oracle.grab_pulse_lens(x, 0.0, tol, "FSK", 100)
        assert np.array_equal(a, b), (tol, a, b)
    c = np.zeros(10000, np.float32)
    assert np.array_equal(sf.grab_pulse_lens(c, 0.0, 5, "ASK", 100), oracle.grab_pulse_lens(c, 0.0, 5, "ASK", 100))
    assert sf.grab_pulse_lens(np.zeros(0, np.float32), 0.0, 5, "FSK", 100).shape == (0, 2)


@pytest.mark.parametrize("dtype", [np.float32, np.int8, np.int16])
@pytest.mark.parametrize("mod", ["FSK", "ASK"])
def test_fused_demod_digitize_equals_two_step(sf, oracle, dtype, mod):
    n = 300000
    iq = synth_fsk(n, sps=50, seed=42, gap_every=20000, dtype=dtype)
    if mod == "ASK":
        env = (np.repeat(np.random.default_rng(1).integers(0, 2, n // 50 + 1), 50)[:n] * 0.9 + 0.1)
        iq = (iq.astype(np.float32) * env[:, None]).astype(dtype)
    noise = {np.float32: 0.05, np.int8: 5.0, np.int16: 1000.0}[dtype]
    center = 0.0 if mod == "FSK" else 0.3
    qad_ref = oracle.afp_demod(iq, noise, mod, 2)
    for tol in (0, 5):
        rows_ref = oracle.grab_pulse_lens(qad_ref, center, tol, mod, 50)
        qad, rows = sf.demod_digitize(iq, noise, mod, center, tol, 50)
        assert bits_equal(qad, qad_ref) == 0
        assert np.array_equal(rows, rows_ref)
        _, rows2 = sf.demod_digitize(iq, noise, mod, center, tol, 50, return_qad=False)
        assert np.array_equal(rows2, rows_ref)


def test_device_resident_roundtrip(sf, oracle, ctx):
    from urh_b200.device import to_device, DeviceArray

    iq = synth_fsk(123457, seed=9, gap_every=10000)
    d = to_device(iq, ctx)
    q = sf.afp_demod(d, 0.05, "FSK", 2)
    assert isinstance(q, DeviceArray)
    rows = sf.grab_pulse_lens(q, 0.0, 5, "FSK", 100)
    qr = oracle.afp_demod(iq, 0.05, "FSK", 2)
    assert bits_equal(q.get(), qr) == 0
    assert np.array_equal(rows, oracle.grab_pulse_lens(qr, 0.0, 5, "FSK", 100))
    assert ctx.launch_count() > 0
