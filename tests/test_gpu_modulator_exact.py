"""GPU: the modulator (modulate.cu) word for word against the oracle's modulate_c, which tests/test_modulator_pin.py pins to the
reference: the random ASK / FSK / PSK / OQPSK matrix, the batch kernel's own cases (ragged, empty and misaligned messages,
70 000 messages, long FSK runs, every fmod branch, a 2^25-sample message, overflowing arguments), the device sinf / cosf /
fmod(., 2 pi) against libm, and GFSK in its three stages (frequencies, phases, samples)."""
import array
import ctypes as C
import math
import tempfile

import numpy as np
import pytest

from conftest import bits_equal
from test_modulator_pin import Libm, arange_f32, mod_words, modulator_cases, near_half_pi_multiples

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sf():
    from urh_b200.cythonext import signal_functions

    return signal_functions


@pytest.fixture(scope="module")
def libm():
    with tempfile.TemporaryDirectory() as td:
        yield Libm(td)


def _same(got, want, where):
    assert got.dtype == want.dtype and got.shape == want.shape, (where, got.dtype, got.shape, want.shape)
    assert np.array_equal(mod_words(got), mod_words(want)), (where, int((mod_words(got) != mod_words(want)).sum()))


# ---- device math: urh_glibc_sincosf over the whole float range, urh_fmod_2pi -----------------------------------------------------
def _device_modmath(ctx, x, v):
    from urh_b200.device import DeviceArray, to_device

    x = np.ascontiguousarray(x, np.float32)
    v = np.ascontiguousarray(v, np.float64)
    dx, dv = to_device(x, ctx), to_device(v, ctx)
    sn, cs, ok = DeviceArray(ctx, x.shape, np.float32), DeviceArray(ctx, x.shape, np.float32), DeviceArray(ctx, x.shape, np.int32)
    r = DeviceArray(ctx, v.shape, np.float64)
    ctx.check(ctx.lib.urh_selftest_modmath(ctx.handle, C.c_void_p(dx.ptr), len(x), C.c_void_p(sn.ptr), C.c_void_p(cs.ptr),
                                           C.c_void_p(ok.ptr), C.c_void_p(dv.ptr), len(v), C.c_void_p(r.ptr)))
    return sn.get(), cs.get(), ok.get(), r.get()


def test_device_sincosf_matches_libm_over_the_float_range(ctx, libm):
    """urh_glibc_sincosf on the device equals libm's sinf / cosf bit for bit on a stratified sample of every binade (2^-149 to
    2^127, both signs), denormals, +-0, FLT_MAX, both sides of the 2^-12 / 0.75 (pi/4 polynomial) / 120 range cuts and floats
    next to k pi/2 at every magnitude; ok = 0 exactly for inf and NaN (their NaN payload is not pinned)"""
    rng = np.random.default_rng(31)
    per = 4000
    expo = np.repeat(np.arange(0, 255, dtype=np.uint32), per)
    mant = rng.integers(0, 1 << 23, len(expo), dtype=np.uint32)
    strat = ((expo << 23) | mant).view(np.float32)
    edges = np.array([0x00000001, 0x00000002, 0x007FFFFF, 0x00800000, 0x39800000, 0x3F400000, 0x3F490FDB, 0x42F00000, 0x7F7FFFFF],
                     np.int64)
    near = (edges[:, None] + np.arange(-8, 9)[None, :]).reshape(-1)
    near = near[(near >= 0) & (near <= 0x7F7FFFFF)].astype(np.uint32).view(np.float32)
    x = np.concatenate([strat, near, near_half_pi_multiples(), np.float32([0.0, 2.0 ** -12, np.pi / 4, 120.0, 3.4028235e38])])
    x = np.concatenate([x, -x]).astype(np.float32)
    nonfinite = np.float32([np.inf, -np.inf, np.nan, -np.nan])
    nonfinite = np.concatenate([nonfinite, np.uint32([0x7F800001, 0x7FC12345, 0xFFFFFFFF]).view(np.float32)])
    sn, cs, ok, _ = _device_modmath(ctx, np.concatenate([x, nonfinite]), np.zeros(0))
    rs, rc = libm.sincosf(x)
    n = len(x)
    assert ok[:n].all() and not ok[n:].any()
    bad = (sn[:n].view(np.uint32) != rs.view(np.uint32)) | (cs[:n].view(np.uint32) != rc.view(np.uint32))
    assert not bad.any(), (int(bad.sum()), x[bad][:8])


def test_device_fmod_2pi_matches_c_fmod(ctx, libm):
    """urh_fmod_2pi (quotient estimate + FMA below 1e15, library fmod above) equals C fmod(v, 2 pi) bit for bit: |v| < 2 pi, values
    within a few ulps of multiples of 2 pi at every magnitude, random values up to 1e20, the 1e15 switch, +-0, +-inf and NaN"""
    rng = np.random.default_rng(37)
    two_pi = 2 * math.pi
    small = rng.uniform(-two_pi, two_pi, 100_000)
    ks = np.unique(np.round(10.0 ** rng.uniform(0, 16, 20_000)))
    mult = ks * two_pi
    steps = np.arange(-4, 5)
    near = (mult.view(np.int64)[:, None] + steps[None, :]).reshape(-1).view(np.float64)
    big = 10.0 ** rng.uniform(0, 20, 200_000) * rng.choice([-1.0, 1.0], 200_000)
    switch = (np.float64(1e15).view(np.int64) + np.arange(-50, 51)).view(np.float64)
    v = np.concatenate([small, near, -near, big, switch, -switch, [two_pi, -two_pi, np.nextafter(two_pi, 0), 0.0, -0.0, 5e-324]])
    special = np.array([np.inf, -np.inf, np.nan])
    _, _, _, r = _device_modmath(ctx, np.zeros(0, np.float32), np.concatenate([v, special]))
    want = libm.fmod_2pi(v)
    assert np.array_equal(r[: len(v)].view(np.int64), want.view(np.int64)), int((r[: len(v)].view(np.int64) != want.view(np.int64)).sum())
    assert np.isnan(r[len(v):]).all()


# ---- ASK / FSK / PSK / OQPSK against the oracle -----------------------------------------------------------------------------------
def test_modulator_matrix_matches_oracle(sf, oracle):
    """every case of the pinned matrix (tests/test_modulator_pin.py: modulator_cases) through modulate_c (one message, what
    Modulator.modulate calls), word for word"""
    for k, (bits, sps, mod, p, bps, a, fc, phi, fs, pause, start, dt) in enumerate(modulator_cases()):
        got = sf.modulate_c(bits, sps, mod, p, bps, a, fc, phi, fs, pause, start, dt)
        want = oracle.modulate_c(bits, sps, mod, p, bps, a, fc, phi, fs, pause, start, dt)
        _same(got, want, (k, mod, np.dtype(dt).name, sps, bps, len(bits), start, fs))


def test_modulator_object_matches_oracle(oracle):
    """Modulator.modulate with its own units (ASK parameters in %, PSK in degrees, carrier phase in degrees, amplitude relative to the
    dtype's full scale) against the oracle given the arguments the reference's Modulator.modulate derives (Modulator.py:215-255)"""
    from urh_b200.signalprocessing.Modulator import Modulator

    rng = np.random.default_rng(41)
    for k in range(48):
        mt = ("ASK", "FSK", "PSK", "OQPSK")[k % 4]
        dt = (np.int8, np.int16, np.float32)[(k // 4) % 3]
        bps = 2 if mt == "OQPSK" else 1 + k % 4
        m = Modulator("m%d" % k)
        m.modulation_type = mt
        m.bits_per_symbol = bps
        m.samples_per_symbol = (1, 3, 7, 100)[k % 4]
        m.sample_rate = (44100.0, 1e6, 2e6)[k % 3]
        m.carrier_freq_hz = float(rng.uniform(-1.5, 1.5) * m.sample_rate)
        m.carrier_phase_deg = float(rng.uniform(-180, 180))
        m.carrier_amplitude = float(rng.uniform(0.1, 1.0))
        if mt == "ASK":
            params = np.round(rng.uniform(0, 100, 2 ** bps))
            params[0] = 0
        elif mt == "FSK":
            params = rng.uniform(-1.5, 1.5, 2 ** bps) * m.sample_rate
        else:
            params = rng.uniform(-180, 180, 2 ** bps)
        m.parameters = array.array("f", params)
        bits = list(map(int, rng.integers(0, 2, int(rng.integers(2, 400)))))
        start, pause = int((0, 5, 2 ** 24 + 1)[k % 3]), int(rng.integers(0, 30))
        got = m.modulate(bits, pause=pause, start=start, dtype=dt).data
        a = m.carrier_amplitude * (1 if dt == np.float32 else np.iinfo(dt).max)
        p = np.asarray(m.parameters, np.float32)
        if mt == "ASK":
            p = [a * x / 100 for x in m.parameters]
        elif mt == "PSK":
            p = [x * (math.pi / 180) for x in m.parameters]
        want = oracle.modulate_c(np.uint8(bits), m.samples_per_symbol, mt, np.float32(p), bps, a, m.carrier_freq_hz,
                                 m.carrier_phase_deg * (np.pi / 180), m.sample_rate, pause, start, dt)
        _same(got, want, (k, mt, np.dtype(dt).name))


def _ragged(rng, mod, bps, n):
    """n messages: empty (not for OQPSK: the reference's zeroing loop writes outside its array below 2 bits), one symbol, bit
    counts that are not a multiple of bps, a few hundred symbols"""
    out = []
    for j in range(n):
        kind = j % 5
        if kind == 0:
            nb = 2 if mod == "OQPSK" else 0
        elif kind == 1:
            nb = bps
        elif kind == 2:
            nb = bps * int(rng.integers(1, 40)) + int(rng.integers(0, bps))
        elif kind == 3:   # fewer bits than one symbol (OQPSK: one symbol)
            nb = 2 if mod == "OQPSK" else max(1, bps - 1)
        else:
            nb = bps * int(rng.integers(100, 400))
        out.append(rng.integers(0, 2, nb).astype(np.uint8))
    return out


@pytest.mark.parametrize("mod", ["ASK", "FSK", "PSK", "OQPSK"])
def test_ragged_batches_match_per_message_oracle(sf, oracle, mod):
    """ragged batches with empty and one-symbol messages, odd and zero pauses (later messages start misaligned for the vector
    store): every message equals the oracle; device_result=True gives the same offsets and samples; a rectangular [nmsg, nbits]
    batch equals the ragged path and per-message calls"""
    rng = np.random.default_rng(["ASK", "FSK", "PSK", "OQPSK"].index(mod))
    for dt in (np.int8, np.int16, np.float32):
        for bps in ((2,) if mod == "OQPSK" else (1, 3, 8)):
            msgs = _ragged(rng, mod, bps, 25)
            pauses = [int(x) for x in rng.choice([0, 1, 3, 7, 64], len(msgs))]
            if mod == "ASK":
                p = rng.uniform(0, 1 if dt == np.float32 else 3 * np.iinfo(dt).max, 1 << bps).astype(np.float32)
                p[0] = 0
            elif mod == "FSK":
                p = rng.uniform(-3e6, 3e6, 1 << bps).astype(np.float32)
            else:
                p = rng.uniform(-np.pi, np.pi, 1 << bps).astype(np.float32)
            a = 0.8 if dt == np.float32 else 0.8 * np.iinfo(dt).max
            args = (7, mod, p, bps, a, 123e3, 0.3, 2e6)
            got = sf.modulate_batch(msgs, *args, pauses, 5, dt)
            for j, (b, ps) in enumerate(zip(msgs, pauses)):
                _same(got[j], oracle.modulate_c(b, *args, ps, 5, dt), (mod, np.dtype(dt).name, bps, j, len(b), ps))
            d, off = sf.modulate_batch(msgs, *args, pauses, 5, dt, device_result=True)
            lens = [len(b) // bps * 7 + ps for b, ps in zip(msgs, pauses)]
            assert np.array_equal(off, np.concatenate([[0], np.cumsum(lens)]))
            _same(d.get(), np.concatenate(got), (mod, "device_result"))
            rect = rng.integers(0, 2, (9, bps * 13 + 1)).astype(np.uint8)
            rp = [1, 0, 3, 2, 5, 0, 0, 7, 1]
            by_rect = sf.modulate_batch(rect, *args, rp, 5, dt)
            by_list = sf.modulate_batch(list(rect), *args, rp, 5, dt)
            for j in range(len(rect)):
                _same(by_rect[j], by_list[j], (mod, "rect", j))
                _same(by_rect[j], sf.modulate_c(rect[j], *args, rp[j], 5, dt), (mod, "rect/single", j))
                _same(by_rect[j], oracle.modulate_c(rect[j], *args, rp[j], 5, dt), (mod, "rect/oracle", j))


def test_seventy_thousand_messages(sf, oracle):
    """70 000 messages in one call: grid.y is capped at 65 535, the kernels loop over the rest (FSK: the correction warps too)"""
    rng = np.random.default_rng(43)
    n = 70_000
    msgs = [rng.integers(0, 2, int(rng.integers(1, 12))).astype(np.uint8) for _ in range(n)]
    pauses = [int(x) for x in rng.integers(0, 3, n)]
    p = np.float32([-250e3, 310e3])
    got = sf.modulate_batch(msgs, 3, "FSK", p, 1, 1.0, 0.0, 0.1, 1e6, pauses, 7, np.float32)
    for j in list(range(0, 200)) + list(range(65_000, n)):
        _same(got[j], oracle.modulate_c(msgs[j], 3, "FSK", p, 1, 1.0, 0.0, 0.1, 1e6, pauses[j], 7, np.float32), ("70k", j))


def test_fsk_correction_warp_blocks(sf, oracle):
    """k_fsk_corrections: 31 / 32 / 33 / 65 / 5000-symbol messages, in long runs of equal symbols and alternating (the carry from
    one 32-symbol block to the next and the `changed` mask), bps 1 and 3, two symbols sharing a frequency"""
    rng = np.random.default_rng(47)
    for bps in (1, 3):
        m = 1 << bps
        p = rng.uniform(-400e3, 400e3, m).astype(np.float32)
        p[-1] = p[0]
        msgs = []
        for nsym in (31, 32, 33, 65, 5000):
            runs = np.repeat(rng.integers(0, m, nsym // 20 + 2), rng.integers(1, 90, nsym // 20 + 2))
            runs = np.resize(runs, nsym)
            alt = np.where(np.arange(nsym) % 2 == 0, 0, m - 1)
            alt2 = np.where(np.arange(nsym) % 2 == 0, 0, m - 1) if m == 2 else np.where(np.arange(nsym) % 2 == 0, m - 1, 0)
            for sym in (runs, alt, alt2, rng.integers(0, m, nsym)):
                msgs.append(((sym[:, None] >> np.arange(bps - 1, -1, -1)) & 1).reshape(-1).astype(np.uint8))
        for dt, start in ((np.float32, 0), (np.int16, 2 ** 24 + 1), (np.float32, 2 ** 32 - 1)):
            got = sf.modulate_batch(msgs, 5, "FSK", p, bps, 0.9 if dt == np.float32 else 30000, 0.0, 0.0, 2e6, 3, start, dt)
            for j, b in enumerate(msgs):
                want = oracle.modulate_c(b, 5, "FSK", p, bps, 0.9 if dt == np.float32 else 30000, 0.0, 0.0, 2e6, 3, start, dt)
                _same(got[j], want, ("fsk blocks", bps, j, len(b), start))


def test_fsk_correction_takes_every_fmod_branch(sf, oracle):
    """the FSK correction term through all three branches of urh_fmod_2pi: |v| < 2 pi, the quotient estimate, and the library
    fmod at |v| >= 1e15 (fs = 1 Hz, start = 2^32 - 1, 1 MHz steps: 2 pi * 1e6 * 4.3e9 = 2.7e16); carrier arguments in sincosf's
    large range from a large start or a small sample rate"""
    rng = np.random.default_rng(53)
    bits = rng.integers(0, 2, 600).astype(np.uint8)
    cases = [  # (params, fs, start, largest |term| class)
        (np.float32([1e-3, 2e-3]), 1e6, 0, "small"),
        (np.float32([-1e3, 1e3]), 1e6, 0, "estimate"),
        (np.float32([0, 1e6, 2e6, 3e6]), 1.0, 2 ** 32 - 1, "library"),
        (np.float32([-7e5, 2e5]), 1.0, 2 ** 31 + 1, "library"),
        (np.float32([0.11, 0.37]), 1.0, 2 ** 32 - 1, "estimate"),
    ]
    for p, fs, start, kind in cases:
        bps = 2 if len(p) == 4 else 1
        nsym = len(bits) // bps
        t = np.float32(nsym * 4 + start) / np.float32(fs)
        term = 2 * math.pi * float(np.ptp(p)) * float(t)
        assert {"small": term < 2 * math.pi, "estimate": 2 * math.pi <= term < 1e15, "library": term >= 1e15}[kind], (kind, term)
        for dt in (np.float32, np.int8):
            a = 1.0 if dt == np.float32 else 127.0
            got = sf.modulate_c(bits, 4, "FSK", p, bps, a, 0.0, 0.2, fs, 5, start, dt)
            _same(got, oracle.modulate_c(bits, 4, "FSK", p, bps, a, 0.0, 0.2, fs, 5, start, dt), (kind, float(p[1]), start))
    for mod, p in (("PSK", np.float32([0.5, -2.0])), ("ASK", np.float32([0.0, 0.7]))):
        for fs, start, fc in ((1.0, 2 ** 31 + 1, 0.37), (44100.0, 2 ** 32 - 1, 1.9e4), (3.0, 5, 1e7)):
            got = sf.modulate_c(bits, 3, mod, p, 1, 1.0, fc, 0.4, fs, 0, start, np.float32)
            _same(got, oracle.modulate_c(bits, 3, mod, p, 1, 1.0, fc, 0.4, fs, 0, start, np.float32), (mod, fs, start))


def test_fsk_message_longer_than_2_24_samples(sf, oracle):
    """one float32 FSK message of 2^25 + 700 samples, checked in full: past 2^24 the float32 time base (i + start) / fs rounds"""
    rng = np.random.default_rng(59)
    nsym = (2 ** 25) // 100 + 7
    bits = np.repeat(rng.integers(0, 2, nsym // 5 + 1), 5)[:nsym].astype(np.uint8)
    p = np.float32([-20e3, 20e3])
    got = sf.modulate_c(bits, 100, "FSK", p, 1, 1.0, 0.0, 0.0, 2e6, 11, 1, np.float32)
    want = oracle.modulate_c(bits, 100, "FSK", p, 1, 1.0, 0.0, 0.0, 2e6, 11, 1, np.float32)
    assert got.shape == want.shape == (nsym * 100 + 11, 2)
    assert bits_equal(got, want) == 0


def test_overflowing_arguments(sf, oracle):
    """carrier arguments that overflow float32 to +-inf (and time bases that do): sinf / cosf give NaN on both sides.  NaN
    positions and integer outputs match; NaN payloads are not compared"""
    rng = np.random.default_rng(61)
    bits = rng.integers(0, 2, 200).astype(np.uint8)
    for mod, p in (("PSK", np.float32([0.0, 1.0])), ("FSK", np.float32([-1e9, 1e9])), ("ASK", np.float32([0.0, 50.0]))):
        for fs, fc in ((1e-30, 1e9), (1e-38, 1e3), (2e-45, 0.0)):
            for dt in (np.float32, np.int16, np.int8):
                got = sf.modulate_c(bits, 3, mod, p, 1, 60.0, fc, 0.1, fs, 2, 5, dt)
                want = oracle.modulate_c(bits, 3, mod, p, 1, 60.0, fc, 0.1, fs, 2, 5, dt)
                if dt == np.float32 and mod != "ASK":
                    assert np.isnan(want).any(), (mod, fs)
                _same(got, want, (mod, fs, fc, np.dtype(dt).name))


# ---- GFSK in three stages ---------------------------------------------------------------------------------------------------
def _gfsk_table(ctx, sf, msgs, sps, p, bps, phi, fs, start, bt, width):
    from urh_b200.device import DeviceArray, to_device

    lens = np.array([len(b) for b in msgs], np.int64)
    bit_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    nval = lens // bps * sps
    tab = DeviceArray(ctx, (int(nval.sum()), 2), np.float32)
    taps = sf.gauss_fir(fs, sps, bt=bt, filter_width=width)
    d_bits = to_device(np.concatenate(msgs).astype(np.uint8), ctx)
    p = np.ascontiguousarray(p, np.float32)
    ctx.check(ctx.lib.urh_modulate_gfsk_table(ctx.handle, C.c_void_p(d_bits.ptr), bit_off.ctypes.data_as(C.c_void_p), len(msgs), sps,
                                              p.ctypes.data_as(C.c_void_p), len(p), bps, float(phi), float(fs), start,
                                              taps.ctypes.data_as(C.c_void_p), len(taps), C.c_void_p(tab.ptr)))
    host = tab.get()
    off = np.concatenate([[0], np.cumsum(nval)])
    return [host[off[j]: off[j + 1]] for j in range(len(msgs))], taps


def _freqs64(bits, p, bps, sps, taps):
    """the reference's filtered frequencies (signal_functions.pyx:200-216) in float64 from the same float32 symbol frequencies
    and taps, the shorter-than-filter branch included"""
    nsym = len(bits) // bps
    idx = (bits[: nsym * bps].reshape(nsym, bps).astype(np.int64) << np.arange(bps - 1, -1, -1)).sum(axis=1)
    f = np.repeat(np.asarray(p, np.float32)[idx].astype(np.float64), sps)
    g = taps.astype(np.float64)
    return np.convolve(f, g, mode="same") if len(f) >= len(g) else np.convolve(g, f, mode="same")[: len(f)]


def _gfsk_cases():
    """(messages, sps, params, bps, phi, fs, start, bt, width): several sps / BT / bps / batch sizes / starts; messages shorter
    than the filter; +-20 kHz at 100 sps; carrier phases just below a binade edge and phase sign changes"""
    rng = np.random.default_rng(67)
    below = lambda x: float(np.nextafter(np.float32(x), np.float32(0)))   # noqa: E731
    specs = [
        (100, [-20e3, 20e3], 1, 0.0, 2e6, 0, 0.5, 1.0),
        (100, [-20e3, 20e3], 1, below(4.0), 2e6, 1, 0.5, 1.0),
        (50, [-10e3, 10e3], 1, below(-8.0), 1e6, 5, 0.3, 1.0),
        (8, [-50e3, -10e3, 10e3, 50e3], 2, 1e-3, 1e6, 2 ** 24 - 1, 0.5, 2.0),
        (7, list(np.linspace(-90e3, 90e3, 8)), 3, below(2.0 ** 10), 1e6, 2 ** 24 + 1, 1.0, 1.0),
        (3, [-3e5, 3e5], 1, -1e-3, 2e6, 2 ** 31 + 1, 0.5, 1.0),
        (1, [-1e5, 1e5], 1, 0.5, 1e6, 2 ** 32 - 1, 0.5, 1.0),
        (100, [0.0, 40e3], 1, 0.0, 2e6, 2 ** 31 + 1, 0.5, 1.0),
    ]
    for sps, p, bps, phi, fs, start, bt, width in specs:
        # bits left over after the last symbol only where they are fewer than the symbols: the reference's GFSK branch takes
        # bps = len(bits) // symbols (signal_functions.pyx:202), which differs from bps otherwise and indexes past the parameters
        msgs = [rng.integers(0, 2, bps * n + (int(rng.integers(0, bps)) if n >= bps else 0)).astype(np.uint8)
                for n in (1, 2, 37, 700, 3000)]
        yield msgs, sps, np.float32(p), bps, phi, fs, start, bt, width


def test_gfsk_three_stages(ctx, sf, oracle, libm):
    """frequencies within one float32 ulp of the float64 convolution; phases bit-identical to the serial float32 recurrence on the
    device's own frequencies with numpy's arange time base; samples bit-identical to the oracle fed the device's table; a batch
    equals per-message calls; both phase paths (integer prefix sums, one by one) ran"""
    stats = np.zeros(2, np.int64)
    ctx.check(ctx.lib.urh_modulate_stats(ctx.handle, stats.ctypes.data_as(C.c_void_p)))   # reset
    for msgs, sps, p, bps, phi, fs, start, bt, width in _gfsk_cases():
        tabs, taps = _gfsk_table(ctx, sf, msgs, sps, p, bps, phi, fs, start, bt, width)
        for j, (b, tab) in enumerate(zip(msgs, tabs)):
            where = (sps, bps, phi, fs, start, j, len(b))
            ref = _freqs64(b, p, bps, sps, taps)
            ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
            # + the float64 convolution's own rounding where the sum cancels near zero
            assert np.all(np.abs(tab[:, 0] - ref) <= ulp + 2.0 ** -44 * float(np.abs(p).max())), where
            t = (arange_f32(start, len(tab)) / np.float32(fs)).astype(np.float32)
            ph = libm.serial_phases(tab[:, 0], t, np.float32(phi))
            assert bits_equal(tab[:, 1], ph) == 0, where
        pauses = [3, 0, 1, 5, 2]
        for dt in (np.float32, np.int8):
            a = 1.0 if dt == np.float32 else 127.0
            got = sf.modulate_batch(msgs, sps, "GFSK", p, bps, a, 0.0, phi, fs, pauses, start, dt, bt, width)
            for j, (b, tab) in enumerate(zip(msgs, tabs)):
                want = oracle.modulate_c(b, sps, "GFSK", p, bps, a, 0.0, phi, fs, pauses[j], start, dt, gfsk_table=tab)
                _same(got[j], want, ("gfsk samples", sps, start, j))
                single = sf.modulate_c(b, sps, "GFSK", p, bps, a, 0.0, phi, fs, pauses[j], start, dt, bt, width)
                _same(got[j], single, ("gfsk batch vs single", sps, start, j))
    ctx.check(ctx.lib.urh_modulate_stats(ctx.handle, stats.ctypes.data_as(C.c_void_p)))
    assert stats[0] > 0 and stats[1] > 0, stats


@pytest.mark.parametrize("start", [1, 2 ** 31 + 1])
def test_gfsk_phases_of_a_message_longer_than_2_24_samples(ctx, sf, libm, start):
    """the GFSK time base is numpy's float32 arange (t_i = fl(t0 + fl(i) * d)), not fl(start + i): from start = 1 they part at
    i = 2^24 + 1, and at start = 2^31 + 1 numpy's t is constant.  Phases of a 17-million-sample message, checked in full"""
    rng = np.random.default_rng(71)
    sps, nsym = 10, 1_700_000
    bits = np.repeat(rng.integers(0, 2, nsym // 3 + 1), 3)[:nsym].astype(np.uint8)
    p, fs = np.float32([-20e3, 20e3]), 1e6
    (tab,), _ = _gfsk_table(ctx, sf, [bits], sps, p, 1, 0.25, fs, start, 0.5, 1.0)
    assert len(tab) > 2 ** 24 + 1000
    t = (arange_f32(start, len(tab)) / np.float32(fs)).astype(np.float32)
    ph = libm.serial_phases(tab[:, 0], t, np.float32(0.25))
    bad = np.flatnonzero(tab[:, 1].view(np.uint32) != ph.view(np.uint32))
    assert len(bad) == 0, (len(bad), bad[:3])
