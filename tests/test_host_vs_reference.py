"""CPU: the host-side logic of the drop-in layer against the REFERENCE's own functions on randomized inputs.  These functions never
touch the GPU: pulses -> bits, plateau / bit-length bookkeeping of estimate(), modulator parameter preparation, filter design,
bit utilities.  The reference's answers (imported through oracle/ref_loader.py while recording) are stored in
tests/golden/ref_host_vs_reference.json (oracle/cassette.py); a randomized trial's answers are stored as one fingerprint."""
import array

import numpy as np
import pytest

from oracle.cassette import RECORD, Cassette, fingerprint, same


def _oracle_ppseq_to_bits(*a, **k):
    """the sequential CPU restatement of ProtocolAnalyzer._ppseq_to_bits lives in the test oracle, not in the product"""
    from oracle import oracle
    return oracle.ppseq_to_bits(*a, **k)


@pytest.fixture
def cassette(request):
    c = Cassette("host_vs_reference", request.node.name)
    yield c
    c.close()


@pytest.fixture(scope="module")
def ref():
    if not RECORD:
        return None
    from oracle import ref_loader
    ns = ref_loader.load_python_layer()
    sf, ut, ai = ref_loader.load_kernels()
    ns.sf, ns.ut, ns.ai = sf, ut, ai
    return ns


def test_ppseq_to_bits_port(cassette, ref):
    rfun = cassette.make(lambda: ref.ProtocolAnalyzer(None)._ppseq_to_bits)   # an instance method in the reference (ProtocolAnalyzer.py:323)
    rng = np.random.default_rng(5)
    for trial in range(300):
        bps = int(rng.choice([1, 2]))
        pt = int(rng.choice([8, 0, 2]))
        sps = int(rng.choice([1, 3, 10, 100]))
        k = int(rng.integers(1, 80))
        kinds = rng.integers(-1, 1 << bps, k)
        ns = np.where(rng.random(k) < 0.15, rng.integers(9, 30, k) * sps, rng.integers(0, 5 * sps + 1, k))
        rows = np.stack([kinds, ns], axis=1).astype(np.int64)
        wp = bool(trial % 2)

        def answers(r):
            return [[list(x) for x in r[0]], list(r[1]), [list(x) for x in r[2]]]
        mine = answers(_oracle_ppseq_to_bits(rows, sps, bps, write_bit_sample_pos=wp, pause_threshold=pt))
        assert fingerprint(mine) == cassette.want(lambda: fingerprint(answers(rfun(rows, sps, bps, write_bit_sample_pos=wp, pause_threshold=pt)))), trial



def pulse_edge_tables(oracle):
    """(name, rows, sps, bps) for the tables of tests/pulse_edge_cases.py that ppseq_to_bits takes (bps >= 1, sps >= 1) and that stay
    small: orders up to 256, negative lengths, tables of n rows"""
    from pulse_edge_cases import cases

    for c in cases():
        if c.bps >= 1 and c.sps >= 1 and len(c.x) <= 8192:
            yield c.name, oracle.grab_pulse_lens(c.x, *c.args()), c.sps, c.bps


def test_ppseq_to_bits_on_pulse_edge_tables(cassette, ref, oracle):
    """_ppseq_to_bits on the pulse tables of the digitizer's edge cases, at each table's own bits per symbol"""
    rfun = cassette.make(lambda: ref.ProtocolAnalyzer(None)._ppseq_to_bits)
    tables = 0
    for name, rows, sps, bps in pulse_edge_tables(oracle):
        for pt, wp in ((8, True), (0, False)):
            def answers(r):
                return [[list(x) for x in r[0]], list(r[1]), [list(x) for x in r[2]]]
            mine = answers(_oracle_ppseq_to_bits(rows, sps, bps, write_bit_sample_pos=wp, pause_threshold=pt))
            assert fingerprint(mine) == cassette.want(lambda: fingerprint(answers(rfun(rows, sps, bps, write_bit_sample_pos=wp,
                                                                                         pause_threshold=pt)))), (name, pt)
        tables += 1
    assert tables == 250

def test_plateau_bookkeeping(cassette, ref):
    from urh_b200.ainterpretation import AutoInterpretation as AI
    rng = np.random.default_rng(9)
    for trial in range(300):
        n = int(rng.integers(2, 60))
        base = int(rng.choice([8, 40, 100, 300]))
        pl = (rng.integers(1, 6, n) * base + rng.integers(-base // 8 - 1, base // 8 + 2, n)).clip(1)
        if trial % 3 == 0:
            pl[rng.integers(0, n, max(1, n // 6))] = rng.integers(1, 4, max(1, n // 6))   # tiny glitches
        pl = pl.astype(np.uint64)
        vals = [int(v) for v in rng.integers(0, 6, n)]
        data = rng.standard_normal(n + 3) * 10 + 50

        def answers(M, pl):   # each side on its own copy: get_bit_length_from_plateau_lengths rounds `merged` (maybe pl) in place
            out = [M.estimate_tolerance_from_plateau_lengths(pl)]
            out += [list(M.merge_plateau_lengths(pl, tolerance=tol)) for tol in (None, 0, 1, 3)]
            merged = M.merge_plateau_lengths(pl)
            if len(merged) >= 2:
                out.append(M.get_bit_length_from_plateau_lengths(merged))
            b = [int(v) for v in pl]
            M.round_plateau_lengths(b)       # in place
            out += [b, M.get_tolerant_greatest_common_divisor(list(pl)), M.get_most_frequent_value(vals),
                    M.max_without_outliers(data), M.min_without_outliers(data)]
            return out
        assert fingerprint(answers(AI, pl.copy())) == cassette.want(lambda: fingerprint(answers(ref.AutoInterpretation, pl.copy()))), trial


def test_cython_host_helpers(cassette, ref):
    from urh_b200.cythonext import auto_interpretation as cai, signal_functions as sf, util
    rng = np.random.default_rng(2)
    for trial in range(200):
        n = int(rng.integers(1, 80))
        pl = rng.integers(1, 400, n).astype(np.uint64)
        tol, mc = int(rng.integers(0, 12)), int(rng.integers(1, 40))
        big = None
        if trial % 10 == 0:   # long tables with repeated values and zeros (a message of thousands of rounded plateaus)
            big = (rng.integers(0, 7, 3000) * int(rng.choice([10, 100, 300])) + (rng.integers(0, 3, 3000) if trial % 20 else 0)).astype(np.uint64)
            if big.max() == 0:
                big[0] = 5
        bits = rng.integers(0, 2, int(rng.integers(0, 40))).astype(np.uint8)
        a, b = sorted(rng.integers(0, len(bits) + 1, 2)) if len(bits) else (0, 0)

        def answers(ai, sfm, ut):
            out = [list(np.asarray(ai.merge_plateaus(pl, tol, mc))), list(np.asarray(ai.get_threshold_divisor_histogram(pl)))]
            if big is not None:
                out.append(np.asarray(ai.get_threshold_divisor_histogram(big)))
            out.append(list(np.asarray(sfm.get_oqpsk_bits(bits))))
            if len(bits):
                out.append(ut.bit_array_to_number(bits, int(b), int(a)))
            return out
        assert fingerprint(answers(cai, sf, util)) == cassette.want(lambda: fingerprint(answers(ref.ai, ref.sf, ref.ut))), trial
    for sr, sps, bt, fw in ((2e6, 100, 0.5, 1.0), (1e6, 8, 0.3, 1.5), (250e3, 33, 1.0, 0.7)):
        mine = sf.gauss_fir(sr, sps, bt, fw)
        theirs = cassette.want(lambda: np.asarray(ref.sf.get_gauss_fir(sr, sps, bt, fw)) if hasattr(ref.sf, "get_gauss_fir") else None)
        if theirs is not None:
            assert same(mine, theirs)


def test_modulator_and_filter_host_logic(cassette, ref):
    from urh_b200.signalprocessing.Filter import Filter
    from urh_b200.signalprocessing.Modulator import Modulator
    for bw in (0.001, 0.04, 0.08, 0.42):
        def answers(F):
            N = F.get_filter_length_from_bandwidth(bw)
            out = [N, F.get_bandwidth_from_filter_length(N)]
            if N < 2000:
                out += [F.design_windowed_sinc_lpf(0.1, bw), F.design_windowed_sinc_bandpass(-0.1, 0.2, bw)]
            return out
        assert fingerprint(answers(Filter)) == cassette.want(lambda: fingerprint(answers(ref.Filter))), bw
    for mod in ("ASK", "FSK", "PSK", "GFSK", "OQPSK"):
        for bps in ((1, 2, 3) if mod != "OQPSK" else (2,)):
            def answers(M):
                o = M("m")
                o.modulation_type = mod
                o.bits_per_symbol = bps
                o.sample_rate = 2e6
                return [list(o.get_default_parameters()), o.modulation_order, o.is_binary_modulation,
                        o.is_amplitude_based, o.is_frequency_based, o.is_phase_based]
            assert fingerprint(answers(Modulator)) == cassette.want(lambda: fingerprint(answers(ref.Modulator))), (mod, bps)


def test_iq_array_host_logic(cassette, ref):
    from urh_b200.signalprocessing.IQArray import IQArray
    rng = np.random.default_rng(4)
    for dt in (np.int8, np.uint8, np.int16, np.uint16, np.float32):
        assert IQArray.min_max_for_dtype(dt) == cassette.want(lambda: ref.IQArray.min_max_for_dtype(dt))
    c = (rng.standard_normal(10) + 1j * rng.standard_normal(10)).astype(np.complex64)
    for arr in (c, c.astype(np.complex128), rng.standard_normal(20).astype(np.float32), rng.integers(-100, 100, (10, 2)).astype(np.int16),
                rng.integers(0, 255, 20).astype(np.uint8)):
        def answers(Q):
            a = Q(arr)
            return [Q.convert_array_to_iq(arr), a.num_samples, a.dtype, a.minimum, a.maximum, a.real, a.imag]
        assert fingerprint(answers(IQArray)) == cassette.want(lambda: fingerprint(answers(ref.IQArray)))
    for name in ("x.complex", "x.cs8", "x.complex16u", "x.cu16", "x.complex32s", "x.wav"):
        exp = {"x.complex": np.float32, "x.cs8": np.int8, "x.complex16u": np.uint8, "x.cu16": np.uint16, "x.complex32s": np.int16, "x.wav": np.float32}[name]
        assert IQArray._dtype_for_filename(name) == exp


def test_ring_buffer(cassette, ref):
    """util/RingBuffer.py:7-140: push / pop / wrap-around / clear on randomized traffic"""
    import importlib
    from urh_b200.util.RingBuffer import RingBuffer
    from urh_b200.signalprocessing.IQArray import IQArray
    RRing = cassette.make(lambda: importlib.import_module("urh.util.RingBuffer").RingBuffer)
    rng = np.random.default_rng(6)
    for dtype in (np.float32, np.int8):
        mine, theirs = RingBuffer(size=64, dtype=dtype), cassette.make(lambda: RRing(size=64, dtype=dtype))
        got, expected = [], []   # one fingerprint per run; the step that differs shows when recording
        for step in range(300):
            if rng.random() < 0.55:
                k = int(rng.integers(1, 40))
                vals = (rng.standard_normal((k, 2)) * 50).astype(dtype)

                def op(rb, Q):
                    fit = rb.will_fit(k)
                    if fit:
                        rb.push(Q(vals.copy()))
                    return [fit]
            else:
                k = int(rng.integers(1, 50))
                even = bool(step % 2)

                def op(rb, Q):
                    return [np.asarray(rb.pop(k, ensure_even_length=even))]

            def run(rb, Q):
                out = op(rb, Q) + [rb.left_index, rb.right_index, rb.space_left, rb.is_empty, len(rb), np.asarray(rb.view_data)]
                if step % 97 == 0:
                    rb.clear()
                return out
            got.append(fingerprint(run(mine, IQArray)))
            if theirs is not None:
                expected.append(fingerprint(run(theirs, ref.IQArray)))
                assert got[-1] == expected[-1], (dtype, step)
        assert fingerprint(got) == cassette.want(lambda: fingerprint(expected)), dtype


def test_modulator_prepares_the_same_kernel_call(cassette, ref, monkeypatch):
    """Modulator.modulate (Modulator.py:215-255): the arguments handed to modulate_c are the reference's (both kernels are
    replaced by recorders here, so no GPU and no Cython code runs)"""
    import importlib
    import urh_b200.signalprocessing.Modulator as mine_mod
    ref_mod = cassette.make(lambda: importlib.import_module("urh.signalprocessing.Modulator"))
    calls = {"mine": [], "ref": []}

    def recorder(key):
        def fake(bits, sps, mod_type, parameters, bps, a, f, phi, sr, pause, start, dtype=np.float32, gauss_bt=0.5, filter_width=1.0):
            calls[key].append((list(bits), sps, mod_type, [float(p) for p in parameters], bps, float(a), float(f), float(phi), float(sr),
                               pause, start, np.dtype(dtype), float(gauss_bt), float(filter_width)))
            total = (len(bits) // bps) * sps + pause
            return np.zeros((total, 2), dtype=dtype)
        return fake

    monkeypatch.setattr(mine_mod.signal_functions, "modulate_c", recorder("mine"))
    if ref_mod is not None:
        monkeypatch.setattr(ref_mod.signal_functions, "modulate_c", recorder("ref"))
    rng = np.random.default_rng(12)
    for mod in ("ASK", "FSK", "PSK", "GFSK"):
        for trial in range(6):
            bps = int(rng.choice([1, 2]))
            cfg = dict(modulation_type=mod, bits_per_symbol=bps, samples_per_symbol=int(rng.choice([8, 100])), sample_rate=float(rng.choice([1e6, 2e6])),
                       carrier_freq_hz=float(rng.choice([0.0, 20e3])), carrier_amplitude=float(rng.choice([1.0, 0.5])),
                       carrier_phase_deg=float(rng.choice([0.0, 45.0])), gauss_bt=0.5, gauss_filter_width=1.0)
            nbits = int(rng.integers(0, 12)) * bps
            data = [int(b) for b in rng.integers(0, 2, nbits)]
            payload = "".join(map(str, data)) if trial % 2 else list(data)
            pause, start = int(rng.integers(0, 50)), int(rng.integers(0, 1000))
            dtype = [None, np.int8, np.int16, np.float32][trial % 4]

            def modulate(M):
                o = M.Modulator("t")
                for k_, v in cfg.items():
                    setattr(o, k_, v)
                o.parameters = o.get_default_parameters()
                r = o.modulate(payload, pause=pause, start=start, dtype=dtype)
                return [r.data.shape, r.dtype]
            a = modulate(mine_mod)
            assert a == cassette.want(lambda: modulate(ref_mod))
    ref_calls = cassette.want(lambda: calls["ref"])
    assert len(calls["mine"]) == len(ref_calls) > 0
    assert calls["mine"] == ref_calls


def test_spectrogram_geometry(cassette, ref):
    """Spectrogram.py:84-103: hop size, bin counts and the number of STFT frames (the reference's frame count is the
    shape of its strided view; ours is computed up front to size the device buffers)"""
    from urh_b200.signalprocessing.Spectrogram import Spectrogram
    rng = np.random.default_rng(1)
    for trial in range(40):
        n = int(rng.integers(1, 5000))
        w = int(rng.choice([16, 64, 256, 1024]))
        ov = float(rng.choice([0.5, 0.0, 0.75, 0.3]))
        x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
        a = Spectrogram(x, window_size=w, overlap_factor=ov)

        def geometry():
            b = ref.Spectrogram(x, window_size=w, overlap_factor=ov)
            return (b.hop_size, b.time_bins, b.freq_bins, b.stft(x).shape[0])
        assert (a.hop_size, a.time_bins, a.freq_bins, a._num_frames(n)) == cassette.want(geometry), (n, w, ov)


def test_merge_message_segments_for_ook(cassette, ref):
    from urh_b200.ainterpretation import AutoInterpretation as AI
    rng = np.random.default_rng(21)
    assert AI.merge_message_segments_for_ook([]) == cassette.want(lambda: ref.AutoInterpretation.merge_message_segments_for_ook([]))
    for trial in range(300):
        k = int(rng.integers(1, 25))
        pos = 0
        segs = []
        pulse = int(rng.choice([20, 100, 400]))
        for _ in range(k):
            pos += int(rng.choice([pulse // 2, pulse, 3 * pulse, 9 * pulse, 40 * pulse])) + int(rng.integers(0, 5))
            length = int(rng.integers(1, 4)) * pulse + int(rng.integers(0, 7))
            segs.append((pos, pos + length))
            pos += length
        mine = AI.merge_message_segments_for_ook(list(segs))
        assert fingerprint(mine) == cassette.want(lambda: fingerprint(ref.AutoInterpretation.merge_message_segments_for_ook(list(segs)))), trial


def test_noise_level_decision_from_chunk_statistics(cassette, ref):
    """detect_noise_level (AutoInterpretation.py:60-91): the device only delivers (sum, max) of the 100 end-aligned
    chunks; here they come from numpy, the decision logic is ours, the expected value is the reference's."""
    from urh_b200.ainterpretation import AutoInterpretation as AI
    rng = np.random.default_rng(14)
    for trial in range(200):
        n = int(rng.integers(4, 40000))
        dtype = np.float64 if trial % 2 else np.float32
        mags = np.abs(rng.standard_normal(n) * 0.01)
        kind = trial % 5
        if kind < 3:
            a = int(rng.integers(0, n))
            mags[a: a + n // 3] += rng.uniform(0.3, 1.0)          # a burst
        elif kind == 3:
            mags += 0.5                                            # signal everywhere: chunk means nearly equal -> 0
        else:
            mags[:] = 0.0
        mags = mags.astype(dtype)
        chunksize, nchunks = AI._chunking(n)
        tail = mags[n - nchunks * chunksize:].reshape(nchunks, chunksize)   # chunks are taken from the end backwards
        sums = tail.astype(np.float64).sum(axis=1)
        maxs = tail.max(axis=1).astype(np.float64)
        got = AI._noise_from_chunk_stats(n, chunksize, sums, maxs, dtype)
        assert got == cassette.want(lambda: ref.AutoInterpretation.detect_noise_level(mags)), (trial, n)


def test_oracle_convert_iq_is_the_references_convert_to(cassette, ref, oracle):
    """closes the chain for the format conversions: reference IQArray.convert_to == oracle.convert_iq (here) == convert.cu
    (tests/test_gpu_objects.py::test_convert_to_all_pairs)"""
    rng = np.random.default_rng(5)
    types = [np.int8, np.uint8, np.int16, np.uint16, np.float32]
    for src in types:
        if src == np.float32:
            x = np.concatenate([rng.uniform(-1, 1, 4000), [-1.0, 1.0, 0.0, -0.0, 0.999999, -0.999999]]).astype(np.float32)
        else:
            info = np.iinfo(src)
            x = np.concatenate([rng.integers(info.min, info.max + 1, 4000), [info.min, info.max, 0, 1]]).astype(src)
        x = np.ascontiguousarray(x.reshape(-1, 2))
        for dst in types:
            a = oracle.convert_iq(x, dst)
            assert a.dtype == cassette.want(lambda: ref.IQArray(x).convert_to(dst).dtype), (src, dst)
            assert same(a.view(np.uint8), cassette.want(lambda: ref.IQArray(x).convert_to(dst).view(np.uint8))), (src, dst)
