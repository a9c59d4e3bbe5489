"""CPU suite: pin the C/numpy oracle against the golden vectors generated from the unmodified reference
(tests/golden/make_golden.py) and, when oracle/_ref is present, against the reference's compiled kernels."""
import numpy as np
import pytest

from conftest import CAPTURES, bits_equal, load_golden


@pytest.mark.parametrize("name", CAPTURES)
def test_afp_demod_matches_golden(oracle, name):
    g = load_golden("capture_" + name)
    noise = float(g["noise"])
    for mod in ("ASK", "FSK", "PSK"):
        q = oracle.afp_demod(g["iq"], noise, mod, 2)
        assert bits_equal(q, g["qad_" + mod]) == 0, (name, mod)
    assert bits_equal(oracle.afp_demod(g["iq"], noise, "PSK", 4), g["qad_PSK4"]) == 0


@pytest.mark.parametrize("name", CAPTURES)
def test_grab_pulse_lens_matches_golden(oracle, name):
    g = load_golden("capture_" + name)
    m = g["meta"]
    qad = g["qad_" + m["mod"]]
    for key in [k for k in g if k.startswith("pulses_tol")]:
        tol = int(key[len("pulses_tol"):])
        r = oracle.grab_pulse_lens(qad, m["center"], tol, m["mod"], m["sps"], m["bps"], m["spacing"])
        assert np.array_equal(r, g[key]), (name, key)
    r = oracle.grab_pulse_lens(qad, m["center"], m["tol"], m["mod"], m["sps"], 2, 0.1)
    assert np.array_equal(r, g["pulses_bps2"])


@pytest.mark.parametrize("name", CAPTURES)
def test_magnitudes_noise_segments_center(oracle, name):
    g = load_golden("capture_" + name)
    m = g["meta"]
    mags = oracle.get_magnitudes(g["iq"])
    assert np.array_equal(mags[:64], g["mag_head"])
    assert mags.sum() == float(g["mag_sum"])
    assert oracle.detect_noise_level(mags) == float(g["auto_noise"])
    seg = oracle.segment_messages_from_magnitudes(mags, float(g["noise"]))
    assert np.array_equal(np.array(seg, dtype=np.int64).reshape(-1, 2), g["segments"])
    c = oracle.detect_center(g["qad_" + m["mod"]])
    gc = float(g["detect_center"])
    assert (c is None and np.isnan(gc)) or c == gc


def test_modulator_matches_golden(oracle):
    g = load_golden("modulator")
    bits = g["bits"]
    cases = {
        "ask": ("ASK", [0, 100], 1, np.float32), "ask_i8": ("ASK", [0, 100], 1, np.int8),
        "fsk": ("FSK", [-10e3, 10e3], 1, np.float32), "fsk4": ("FSK", [-20e3, -10e3, 10e3, 20e3], 2, np.float32),
        "fsk_i16": ("FSK", [-10e3, 10e3], 1, np.int16),
        "psk": ("PSK", [-90, 90], 1, np.float32), "psk4": ("PSK", [-135, -45, 45, 135], 2, np.float32),
        "oqpsk": ("OQPSK", [-135, -45, 45, 135], 2, np.float32),
        "gfsk": ("GFSK", [-10e3, 10e3], 1, np.float32), "gfsk_i8": ("GFSK", [-10e3, 10e3], 1, np.int8),
    }
    import math
    for name, (mt, params, bps, dt) in cases.items():
        a = 1 * (1 if dt == np.float32 else np.iinfo(dt).max)
        p = params
        if mt == "ASK":
            p = [a * x / 100 for x in params]
        elif mt in ("PSK", "OQPSK") and mt == "PSK":
            p = [x * (math.pi / 180) for x in params]
        for suffix, b, pause, start in (("", bits, 77, 0), ("_start5", bits[:32], 3, 5)):
            r = oracle.modulate_c(b, 50, mt, np.array(p, dtype=np.float32), bps, a, 40e3, 30 * (np.pi / 180), 1e6, pause, start, dt)
            ref = g["mod_" + name + suffix]
            assert r.dtype == ref.dtype and r.shape == ref.shape
            if np.issubdtype(ref.dtype, np.integer):
                assert np.array_equal(r, ref), name + suffix
            else:
                assert bits_equal(r, ref) == 0, name + suffix


def test_filters_match_golden(oracle):
    g = load_golden("filters")
    assert bits_equal(oracle.fir_filter(g["x"], g["taps"]).view(np.float32), g["fir"].view(np.float32)) == 0
    assert bits_equal(oracle.fir_filter(g["x"], np.array([0.1] * 10, np.complex64)).view(np.float32), g["fir_ma10"].view(np.float32)) == 0
    assert np.array_equal(oracle.fir_filter(g["kat_in"], np.array([0.25] * 4, np.complex64)), g["kat_out"])
    assert np.array_equal(g["kat_out"], np.array([0.25, 0.75, 1.5, 2.5, 3.5, 4.5, 5.5, 6.5, 7.5, 16.5], dtype=np.complex64))
    assert np.array_equal(oracle.design_windowed_sinc_bandpass(0.03, 0.07, 0.04), g["bandpass_taps"])
    assert np.array_equal(oracle.apply_bandpass_filter(g["x"][:300], 0.03, 0.07, 0.2), g["bandpass_direct"])
    assert np.array_equal(oracle.apply_bandpass_filter(g["x"], 0.03, 0.07, 0.04), g["bandpass_fft"])
    assert bits_equal(oracle.spectrogram_db(g["x"]), g["spec_db"]) == 0
    assert bits_equal(oracle.spectrogram_db(g["x"][:300]), g["short_db"]) == 0


def test_spectrogram_db_parameters(oracle):
    """spectrogram_db's window_function / overlap_factor: the defaults spelled out give the golden bits; both reach the STFT"""
    g = load_golden("filters")
    x = g["x"]
    assert bits_equal(oracle.spectrogram_db(x, 1024, 0.5, window_function=np.hanning), g["spec_db"]) == 0
    assert bits_equal(oracle.spectrogram_db(x[:300], 1024, 0.5, window_function=np.hanning), g["short_db"]) == 0
    ramp = lambda w: np.linspace(0.5, 1.0, w)   # noqa: E731  asymmetric: a reversed window would change the result
    for W, ov in ((1024, 0.5), (1001, 0.3), (256, 0.75)):
        want = np.fliplr(oracle.arr2decibel(np.fft.fftshift(oracle.stft(x, W, ov, ramp), axes=(1,)).astype(np.complex64)))
        got = oracle.spectrogram_db(x, W, ov, window_function=ramp)
        assert got.shape == (max(1, (len(x) - W) // (W - int(ov * W)) + 1), W)
        assert bits_equal(got, want) == 0, (W, ov)
        assert bits_equal(got, oracle.spectrogram_db(x, W, ov)) > 0


def test_oracle_vs_compiled_reference_random(oracle):
    """Randomised digitizer / demod cases against the reference's own compiled kernels (if built)."""
    from oracle import ref_loader

    if not ref_loader.kernels_available():
        pytest.skip("oracle/_ref not built")
    sf, ut, ai = ref_loader.load_kernels()
    rng = np.random.default_rng(7)
    for trial in range(60):
        n = int(rng.integers(1, 3000))
        mod = ["ASK", "FSK", "PSK"][trial % 3]
        noise_v = 0.0 if mod == "ASK" else -4.0
        base = np.repeat(rng.standard_normal(n // 7 + 1), 7)[:n] * 0.5
        x = (base + 0.2 * rng.standard_normal(n)).astype(np.float32)
        x[rng.random(n) < 0.1] = noise_v
        s = int(rng.integers(0, n))
        x[s: s + int(rng.integers(0, 40))] = noise_v
        tol = int(rng.integers(0, 8))
        bps = int(rng.integers(1, 3))
        a = np.array(sf.grab_pulse_lens(x, 0.05, tol, mod, 20, bps, 0.3))
        b = oracle.grab_pulse_lens(x, 0.05, tol, mod, 20, bps, 0.3)
        assert np.array_equal(a, b), (trial, n, mod, tol, bps)
    for dt in (np.int8, np.uint8, np.int16, np.uint16, np.float32):
        iq = (rng.standard_normal((777, 2)) * (0.5 if dt == np.float32 else 60)).astype(dt)
        iq[100:120] = 0
        for mod in ("ASK", "FSK", "PSK"):
            a = np.array(sf.afp_demod(iq, 0.1 if dt == np.float32 else 12.0, mod, 2))
            b = oracle.afp_demod(iq, 0.1 if dt == np.float32 else 12.0, mod, 2)
            a[0] = b[0] if mod == "PSK" else a[0]
            assert bits_equal(a, b) == 0, (dt, mod)
        assert np.array_equal(ut.get_magnitudes(iq), oracle.get_magnitudes(iq), equal_nan=True)


def _costas_cases():
    """seeded 40 000-sample PSK captures with bursts and gaps in every dtype, loop orders 2 / 4 / 8, eight loop bandwidths; then
    float32 captures with huge, infinite and NaN samples"""
    rng = np.random.default_rng(11)
    n = 40_000
    on = (np.arange(n) % 15000) < 11000
    for dt, (scale, zero, noise) in ((np.int8, (100, 0, 20.0)), (np.uint8, (100, 128, 0.0)), (np.int16, (20000, 0, 4000.0)),
                                     (np.uint16, (20000, 32768, 0.0)), (np.float32, (1, 0, 0.2))):
        for order in (2, 4, 8):
            sym = rng.integers(0, order, n // 300 + 1)
            x = on * np.exp(1j * (2 * np.pi * 0.025 * np.arange(n) + np.repeat(2 * np.pi * sym / order, 300)[:n]))
            x = x + 0.05 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
            iq = np.stack([x.real, x.imag], axis=1) * scale + zero
            iq = iq.astype(np.float32) if dt == np.float32 else np.clip(np.round(iq), np.iinfo(dt).min, np.iinfo(dt).max).astype(dt)
            for bw in (0.001, 0.01, 0.05, 0.1, 0.2, 0.5, 1.0, 2.0):
                yield iq, noise, order, bw
    x = np.exp(1j * (2 * np.pi * 0.025 * np.arange(n) + np.pi * np.repeat(rng.integers(0, 2, n // 300 + 1), 300)[:n]))
    base = np.stack([x.real, x.imag], axis=1).astype(np.float32)
    for val in ((1e30, -1e30), (-1e30, 1e30), (np.inf, 0.0), (-np.inf, 0.0), (0.3, np.inf), (-0.3, -np.inf), (np.inf, np.inf),
                (np.nan, 0.5), (0.5, np.nan)):
        iq = base.copy()
        iq[[5000, 5007, 30000]] = val
        for order in (2, 4):
            yield iq, 0.2, order, 0.1


def _costas_words(q):
    """the result words after index 0 (np.empty in the reference), NaN folded to one word: its payload is not pinned"""
    w = np.asarray(q, dtype=np.float32)[1:].view(np.uint32).copy()
    w[np.isnan(np.asarray(q, dtype=np.float32)[1:])] = 0x7FC00000
    return w


def test_oracle_costas_pinned_to_reference(oracle, request):
    """The oracle's Costas loop (PSK afp_demod) against the reference's compiled costa_demod: every dtype, loop order and
    bandwidth, and non-finite samples (an infinite imaginary part takes the Annex G recovery of the complex product).  The
    reference's answers are recorded in tests/golden/ref_costas.json, so the pin also runs without the reference; with
    oracle/_ref built it also runs live."""
    from oracle import ref_loader
    from oracle.cassette import RECORD, Cassette, same

    c = Cassette("costas", request.node.name)
    sf = ref_loader.load_kernels()[0] if (RECORD or ref_loader.kernels_available()) else None
    cases = 0
    for iq, noise, order, bw in _costas_cases():
        mine = _costas_words(oracle.afp_demod(iq, noise, "PSK", order, bw))
        want = c.want(lambda: _costas_words(sf.afp_demod(iq, noise, "PSK", order, bw)))
        assert same(mine, want), (iq.dtype, order, bw, cases)
        if sf is not None:
            assert np.array_equal(mine, _costas_words(sf.afp_demod(iq, noise, "PSK", order, bw))), (iq.dtype, order, bw, cases)
        cases += 1
    c.close()
    assert cases == 5 * 3 * 8 + 9 * 2
