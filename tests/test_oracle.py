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


def test_oracle_dense_edges_pinned_to_reference(oracle, request):
    """The oracle's ASK/FSK afp_demod against the reference's compiled afp_demod on float32 captures with infinite, NaN, huge,
    subnormal and zero samples of every sign, each after and before neighbours with zero and nonzero parts (tests/dense_edge_cases.py),
    at noise 0 and 0.05.  An infinite part takes the reference's Annex G recovery of the float complex FSK product.  Words are
    compared with NaN folded (the payload is not pinned).  The reference's answers are recorded in tests/golden/ref_dense_edges.json;
    with oracle/_ref built the pin also runs live."""
    from dense_edge_cases import REFERENCE_TABLE, folded, pinned_captures
    from oracle import ref_loader
    from oracle.cassette import RECORD, Cassette, same

    c = Cassette("dense_edges", request.node.name)
    sf = ref_loader.load_kernels()[0] if (RECORD or ref_loader.kernels_available()) else None
    cases = 0
    for name, iq in pinned_captures():
        for mod in ("ASK", "FSK"):
            for noise in (0.0, 0.05):
                mine = folded(oracle.afp_demod(iq, noise, mod, 2))
                want = c.want(lambda: folded(sf.afp_demod(iq, noise, mod, 2)))
                assert same(mine, want), (name, mod, noise)
                if sf is not None:
                    assert np.array_equal(mine, folded(sf.afp_demod(iq, noise, mod, 2))), (name, mod, noise)
                cases += 1
    c.close()
    assert cases == 2 * 2 * 2
    # the recovery by value: (predecessor, sample) -> the reference's angle
    for prev, cur, word in REFERENCE_TABLE:
        q = oracle.afp_demod(np.array([(1.0, 1.0), prev, cur], np.float32), 0.05, "FSK", 2)
        assert q[2].view(np.uint32) == word, (prev, cur, hex(q[2].view(np.uint32)))


def _center_bits(c):
    """a center as comparable bits: None stays None, a value becomes its float64 word"""
    return None if c is None else int(np.float64(c).view(np.uint64))


def test_oracle_center_edges_pinned_to_reference(oracle, request):
    """The oracle's detect_center against the reference's own AutoInterpretation.detect_center on the named arrays of
    tests/center_edge_cases.py: the keep rule at -4 and at non-finite samples, huge / subnormal / all-equal windows, windows of
    0..3 kept samples, samples on bin edges, rank windows at tile boundaries and cut by max_size, levels far from zero.  Centers
    are compared as float64 words, None as None.  The reference's answers are recorded in tests/golden/ref_center_edges.json;
    with oracle/_ref built the pin also runs live."""
    import warnings

    from center_edge_cases import cases
    from oracle import ref_loader
    from oracle.cassette import RECORD, Cassette

    c = Cassette("center_edges", request.node.name)
    live = RECORD or ref_loader.python_layer_available()
    AIref = ref_loader.load_python_layer().AutoInterpretation if live else None
    got = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)   # np.var / np.mean of empty and overflowing windows
        for name, x, max_size in cases():
            mine = _center_bits(oracle.detect_center(x, max_size))
            want = c.want(lambda: [name, _center_bits(AIref.detect_center(x, max_size))])
            assert want == [name, mine], (name, want, mine)
            if AIref is not None:
                assert _center_bits(AIref.detect_center(x, max_size)) == mine, name
            assert name not in got
            got[name] = mine
    c.close()
    assert len(got) >= 50
    # the cases reach both outcomes and the keep rule's corners
    assert got["posinf_in_window"] is None and got["posinf_trimmed"] is not None
    assert got["posinf_first_window_rank"] is None and got["posinf_last_trimmed_rank"] is not None
    assert got["kept_2"] is None and got["kept_3"] is not None


def test_oracle_pulse_edges_pinned_to_reference(oracle, request):
    """The oracle's grab_pulse_lens against the reference's compiled grab_pulse_lens on the named cases of tests/pulse_edge_cases.py:
    orders 1 .. 256, coinciding / descending / NaN / infinite thresholds, samples on and next to each threshold, the sentinels of
    every modulation string (-0.0 for QAM), NaN and +-inf samples, runs at tile edges, tolerances up to 65535 and >= n, the ASK
    relabel at sps - 1 / sps / sps + 1 and the tail row dropped at n rows.  The reference's tables are recorded in
    tests/golden/ref_pulse_edges.json (large ones as digests); with oracle/_ref built the pin also runs live."""
    from oracle import ref_loader
    from oracle.cassette import RECORD, Cassette, same
    from pulse_edge_cases import cases, thresholds

    c = Cassette("pulse_edges", request.node.name)
    sf = ref_loader.load_kernels()[0] if (RECORD or ref_loader.kernels_available()) else None
    got = {}
    for case in cases():
        mine = oracle.grab_pulse_lens(case.x, *case.args())
        want = c.want(lambda: [case.name, np.array(sf.grab_pulse_lens(case.x, *case.args()), dtype=np.int64)])
        assert want[0] == case.name, (want[0], case.name)
        assert same(mine, want[1]), case.name
        if sf is not None:
            assert np.array_equal(mine, np.array(sf.grab_pulse_lens(case.x, *case.args()))), case.name
        got[case.name] = (case, mine)
    c.close()
    assert len(got) == 346
    # the corners the cases must reach
    for n in (2047, 2048, 2049, 4097, 2 ** 20 + 1):
        for name in ("tail_drop_fsk_%d", "tail_drop_ask_%d"):
            assert len(got[name % n][1]) == n, name % n                           # n firings: the tail row is dropped
        assert len(got["tail_merge_one_ask_%d" % n][1]) == n - 1                  # merges leave room: the tail row stays
    assert got["tol_ge_n_1_tol65535_FSK_data"][1].tolist() == [[0, 1 - 65535]]   # one row, negative length
    assert got["tol_ge_n_5_tol5_FSK_data"][1].tolist() == [[0, 0]]
    nan_thr = [k for k, (cs, _) in got.items() if cs.bps > 0 and np.isnan(thresholds(cs.center, cs.spacing, 1 << cs.bps)).any()]
    assert len(nan_thr) == 64
    assert sum(cs.bps == 8 for cs, _ in got.values()) == 42
    qam = got["signed_zero_QAM"][0]
    assert (np.signbit(qam.x) & (qam.x == 0)).any() and (~np.signbit(qam.x) & (qam.x == 0)).any()
    assert not np.array_equal(got["signed_zero_QAM"][1], got["signed_zero_FSK"][1])


def test_oracle_fir_edges_pinned_to_reference(oracle, request):
    """The oracle's fir_filter against the reference's compiled fir_filter on the named cases of tests/fir_edge_cases.py: tap and sample
    counts around the 1024-output block, non-finite samples at block, halo and head positions, non-finite taps at q = 0, m // 2 and
    m - 1, the three branches of __mulsc3's Annex G recovery, sums that overflow and meet -inf, subnormals, signed zeros, tap counts
    past the shared-memory tile and empty inputs.  Words are compared with NaN folded and -0 apart from +0.  The reference's outputs
    are recorded in tests/golden/ref_fir_edges.json (large ones as digests); with oracle/_ref built the pin also runs live."""
    import warnings

    from fir_edge_cases import cases, fast_loop, folded
    from oracle import ref_loader
    from oracle.cassette import RECORD, Cassette, same

    def answer(fir, case):
        try:
            return folded(np.asarray(fir(case.x, case.taps)))
        except ValueError:
            return "ValueError"

    c = Cassette("fir_edges", request.node.name)
    sf = ref_loader.load_kernels()[0] if (RECORD or ref_loader.kernels_available()) else None
    got = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        for case in cases():
            mine = answer(oracle.fir_filter, case)
            want = c.want(lambda: [case.name, answer(sf.fir_filter, case)])
            assert want[0] == case.name, (want[0], case.name)
            assert (mine == want[1]) if isinstance(mine, str) or isinstance(want[1], str) else same(mine, want[1]), case.name
            if sf is not None:
                live = answer(sf.fir_filter, case)
                assert (mine == live) if isinstance(mine, str) or isinstance(live, str) else np.array_equal(mine, live), case.name
            got[case.name] = (case, mine)
    c.close()
    assert len(got) == 685
    # the corners the cases must reach: outputs where the naive product or a padded product gives what the reference does not
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        differs = {name for name, (cs, y) in got.items()
                   if cs.group not in ("large_m", "empty") and not np.array_equal(folded(fast_loop(cs.x, cs.taps)), y)}
    assert {name for name, (cs, _) in got.items() if cs.group == "annexg"} <= differs
    assert sum(got[k][0].group == "nonfinite_samples" for k in differs) >= 80
    assert sum(got[k][0].group == "nonfinite_taps" for k in differs) >= 100
    assert not differs & {name for name, (cs, _) in got.items() if cs.group in ("shapes", "subnormal", "signed_zero")}
    # a non-finite tap at q = m - 1 only meets the zero initial state in the first m - 1 outputs
    y = got["annexg_padded_inf_tap3_example"][1].view(np.float32)
    assert np.array_equal(y[:4], np.array([0.5, 0.5, 1.25, 0.25], np.float32)) and np.isinf(y[4])
    # recovered products: infinite, not NaN
    assert np.isinf(got["annexg_inf_sample_example"][1].view(np.float32)[2:]).all()
    y = got["annexg_overflow_nan_example"][1].view(np.float32)
    assert y[0] == -np.inf and y[1] == np.inf
    # an overflowed sum meets -inf: NaN in the real part without a NaN product
    assert np.isnan(got["overflow_then_neginf_real"][1].view(np.float32)[0::2]).any()
    # subnormal words survive (no flush to zero), and the outputs of all -0 terms are +0
    tiny = np.float32(np.finfo(np.float32).tiny)
    for name in ("subnormal_products", "subnormal_samples", "subnormal_taps", "subnormal_near_flt_min", "subnormal_tiny_sums"):
        v = got[name][1].view(np.float32)
        assert ((v != 0) & (np.abs(v) < tiny)).sum() > 10, name
    assert (got["neg_zero_samples"][1] == 0).all() and (got["neg_zero_all_terms"][1] == 0).all()
    assert (np.signbit(got["neg_zero_all_terms"][0].x.view(np.float32))).any()
    # the reference's shapes for empty inputs
    assert got["empty_taps_n0"][1] == "ValueError"
    assert len(got["empty_taps_n1"][1]) == 0 and len(got["empty_taps_n3"][1]) == 4 and len(got["empty_samples_m2"][1]) == 0
    assert {len(cs.taps) for cs, _ in got.values() if cs.group == "large_m"} == {12287, 12288, 20000}


def test_oracle_spectral_edges_pinned_to_reference(oracle, request, tmp_path):
    """The oracle's STFT, dB map, FTA amplitudes, band-pass, fft_convolve_1d and DC correction against the reference's own Filter and
    Spectrogram (Spectrogram.stft, its __calculate_spectrogram, export_to_fta, Filter.apply_bandpass_filter, Filter.fft_convolve_1d and
    Filter.work with FilterType.dc_correction) on the named cases of tests/spectral_edge_cases.py.  Per result: dtype, shape, the words
    with NaN folded and -0 apart from +0, and the per-component classes (finite, NaN, +inf, -inf), recorded as digests in
    tests/golden/ref_spectral_edges.json and replayed where the reference is absent; with the reference present the pin also runs live."""
    import warnings

    from oracle import ref_loader
    from oracle.cassette import RECORD, Cassette, digest
    from spectral_edge_cases import answers, bad_frames, cases, classes, folded, frames_of, hop_of

    def pack(results):
        return [[k, np.asarray(a).dtype.str, list(np.shape(a)), digest(folded(a)), digest(classes(a))] for k, a in results]

    def o_fta(x, W, ov):
        return np.flipud(oracle.spectrogram_db(x, W, ov).T)

    def functions(ns):
        if ns is None:
            return dict(stft=oracle.stft, spectrogram_db=lambda x, W, ov: oracle.spectrogram_db(x, W, ov), fta=o_fta,
                        apply_bandpass_filter=oracle.apply_bandpass_filter, fft_convolve_1d=oracle.fft_convolve_1d,
                        dc_correction=oracle.dc_correction)

        def r_fta(x, W, ov):
            path = str(tmp_path / "spectrogram.fta")
            ns.Spectrogram(x, W, ov).export_to_fta(1e6, path, include_amplitude=True)
            rec = np.fromfile(path, dtype=[("f", np.float64), ("t", np.uint32), ("a", np.float32)])
            return rec["a"].reshape(W, -1, 3)[:, :, 0]
        return dict(stft=lambda x, W, ov: ns.Spectrogram(x, W, ov).stft(x),
                    spectrogram_db=lambda x, W, ov: ns.Spectrogram(x, W, ov)._Spectrogram__calculate_spectrogram(x), fta=r_fta,
                    apply_bandpass_filter=ns.Filter.apply_bandpass_filter, fft_convolve_1d=ns.Filter.fft_convolve_1d,
                    dc_correction=lambda x: ns.Filter([], ns.FilterType.dc_correction).work(x))

    c = Cassette("spectral_edges", request.node.name)
    ns = ref_loader.load_python_layer() if (RECORD or ref_loader.python_layer_available()) else None
    mine_f, ref_f = functions(None), (functions(ns) if ns is not None else None)
    got = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        for case in cases():
            mine = answers(case, **mine_f)
            live = answers(case, **ref_f) if ref_f is not None else None
            want = c.want(lambda: [case.name, pack(live)])
            assert want[0] == case.name, (want[0], case.name)
            assert pack(mine) == want[1], case.name
            got[case.name] = (case, dict(mine))
        # the hop-0 overlap: the reference divides by zero, and so does the oracle
        kinds = []
        for f in (mine_f, ref_f):
            try:
                f["stft"](np.ones(100, np.complex64), 64, 1.0)
                kinds.append("returned")
            except Exception as e:   # noqa: BLE001 - the exception's type is what is compared
                kinds.append(type(e).__name__)
        assert kinds[0] == c.want(lambda: kinds[1]) == "ZeroDivisionError"
    c.close()
    assert len(got) == 464, len(got)

    # the corners the cases must reach
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore", RuntimeWarning)
        # band-pass, FFT branch: one non-finite sample makes every output NaN in both parts; a direct convolution would not
        all_nan = []
        for name, (cs, r) in got.items():
            if cs.group != "bandpass":
                continue
            y = r["out"]
            m = len(oracle.design_windowed_sinc_bandpass(0.0, 0.1, cs.bw))
            fft_branch = not m < 8 * np.log(np.sqrt(len(cs.x)))
            bad = not np.isfinite(cs.x.view(np.float32)).all()
            if fft_branch and bad:
                assert np.isnan(y.real).all() and np.isnan(y.imag).all(), name
                h = oracle.design_windowed_sinc_bandpass(*sorted((cs.f_low, cs.f_high)), cs.bw)
                direct = np.convolve(cs.x.astype(np.complex128), h, "full")[(m - 1) // 2: (m - 1) // 2 + len(cs.x)]
                if np.isfinite(direct).sum() > len(cs.x) // 2:
                    all_nan.append(name)
            elif not bad and not (fft_branch and ("fft_overflow" in name or "huge_3e38" in name)):
                assert np.isfinite(y).all(), name
        assert len(all_nan) >= 6 and "bandpass_m51_fft_n5000_inf" in all_nan, all_nan
        # ... and the single-precision transform of a complex64 capture overflows on samples near FLT_MAX: all NaN, where the float64
        # result of the same operation is finite (the device's double convolution gives the latter, DESIGN.md §4.5)
        for name in ("bandpass_m41_fft_fft_overflow", "bandpass_m51_fft_fft_overflow", "bandpass_m41_fft_huge_3e38", "bandpass_m51_fft_huge_3e38"):
            cs, r = got[name]
            assert np.isnan(r["out"]).all(), name
            assert np.isfinite(oracle.apply_bandpass_filter(cs.x.astype(np.complex128), cs.f_low, cs.f_high, cs.bw)).all(), name
        assert np.isfinite(got["bandpass_m51_direct_fft_overflow"][1]["out"]).all()
        # fft_convolve_1d of real x and real h: the rfft branch's real result
        assert got["convolve_real_real"][1]["out"].dtype == np.float64 and got["convolve_real_f32"][1]["out"].dtype == np.float32
        assert np.isnan(got["convolve_inf_tap"][1]["out"]).all() and np.isnan(got["convolve_real_nonfinite"][1]["out"]).all()
        # STFT: every bin of a frame that reads a non-finite sample is NaN + NaN j (numpy's complex product forms (inf, NaN) or NaN, and
        # the transform spreads it), so its dB value is NaN; a real-window product would leave whole frames with finite or infinite parts
        whole_nan = []
        for name, (cs, r) in got.items():
            if cs.group not in ("stft", "segments"):
                continue
            hop = hop_of(cs.W, cs.ov)
            bad = bad_frames(cs.x, cs.W, hop)
            X, db = r["stft"], r["db"]
            assert X.shape == db.shape == (frames_of(len(cs.x), cs.W, hop), cs.W)
            assert (np.isnan(X.real) & np.isnan(X.imag))[bad].all() and np.isnan(db[bad]).all(), name
            assert np.isfinite(X[~bad]).all(), name
            if cs.group == "stft" and bad.any():
                x = np.concatenate([cs.x, np.zeros(max(0, cs.W - len(cs.x)), np.complex64)])
                w = np.hanning(cs.W)
                for f in np.nonzero(bad)[0]:
                    fr = x[f * hop: f * hop + cs.W]
                    prod = np.empty(cs.W, np.complex128)
                    prod.real, prod.imag = fr.real * w, fr.imag * w
                    real_win = np.fft.fft(prod)
                    if np.isnan(X[f]).all() and not (np.isnan(real_win.real) & np.isnan(real_win.imag)).all():
                        whole_nan.append(name)
                        break
        assert len(whole_nan) >= 100, len(whole_nan)
        # huge and squared-overflow captures: a +inf dB value from float32 |X|^2, with finite STFT bins
        assert np.isposinf(got["stft_W1024_ov0.5_sq_overflow"][1]["db"]).any()
        assert np.isposinf(got["stft_W128_ov0.5_huge_1e30"][1]["db"]).all()
        # DC: float32 column sums that overflow give non-finite columns up to 2^22 rows; a NaN or +-inf column is NaN
        for n in (2, 1025, 1 << 22):
            y = got["dc_n%d_overflow_col0" % n][1]["out"]
            assert not np.isfinite(y[:, 0]).any() and np.isfinite(y[:, 1]).all(), n
            assert np.isnan(got["dc_n%d_nan_col0" % n][1]["out"][:, 0]).all()
            assert np.isnan(got["dc_n%d_pm_inf_col1" % n][1]["out"][:, 1]).all()
        y = got["dc_n1025_subnormal_negzero"][1]["out"]
        assert (y[:, 1] == 0).all() and np.signbit(y[:, 1]).all()   # the column sum starts from +0: -0 - (+0) = -0
        assert got["dc_int16_n1025_extremes"][1]["out"].dtype == np.float64
