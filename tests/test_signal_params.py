"""CPU: the parameter setters of urh_b200.signalprocessing.Signal (one descriptor table) behave like the reference's
hand-written properties (Signal.py:215-400): same values, same events in the same order with the same arguments, same
invalidation of the cached demodulation.  The reference's answers are recorded in tests/golden/ref_signal_params.json
(oracle/cassette.py)."""
import numpy as np
import pytest

from oracle.cassette import RECORD, Cassette, fingerprint, same


@pytest.fixture
def cassette(request):
    c = Cassette("signal_params", request.node.name)
    yield c
    c.close()


@pytest.fixture(scope="module")
def ref():
    if not RECORD:
        return None
    from oracle import ref_loader
    return ref_loader.load_python_layer()


EVENTS = ("samples_per_symbol_changed", "tolerance_changed", "noise_threshold_changed", "center_changed",
          "center_spacing_changed", "name_changed", "sample_rate_changed", "modulation_type_changed",
          "bits_per_symbol_changed", "protocol_needs_update")


class Recorder(object):
    def __init__(self, log, name):
        self.log, self.name = log, name

    def emit(self, *args):
        self.log.append((self.name, tuple(args)))

    def connect(self, *a, **k):
        pass


def instrument(sig):
    log = []
    for e in EVENTS:
        setattr(sig, e, Recorder(log, e))
    return log


SCRIPT = [
    ("tolerance", 5), ("tolerance", 7), ("tolerance", 7.9), ("tolerance", "9"),
    ("samples_per_symbol", 100), ("samples_per_symbol", 250), ("samples_per_symbol", 250),
    ("modulation_type", "FSK"), ("modulation_type", "ASK"), ("modulation_type", "PSK"), ("modulation_type", "PSK"),
    ("bits_per_symbol", 1), ("bits_per_symbol", 2), ("bits_per_symbol", 2.0), ("bits_per_symbol", 3),
    ("center", 0), ("center", 0.25), ("center", 0.25), ("center", -1e-3),
    ("center_spacing", 1), ("center_spacing", 0.5),
    ("pause_threshold", 8), ("pause_threshold", 0), ("pause_threshold", 0),
    ("message_length_divisor", 1), ("message_length_divisor", 4),
    ("costas_loop_bandwidth", 0.1), ("costas_loop_bandwidth", 0.05),
    ("name", "x"), ("name", "renamed"), ("name", "renamed"),
    ("sample_rate", 1e6), ("sample_rate", 2e6),
    ("block_protocol_update", True), ("tolerance", 3), ("modulation_type", "FSK"), ("center", 0.5), ("block_protocol_update", False),
    ("samples_per_symbol", 40), ("timestamp", 12.5),
]


def test_parameter_setters_match_reference(cassette, ref):
    from urh_b200.signalprocessing.Signal import Signal

    mine = Signal("", "x", sample_rate=1e6)
    theirs = cassette.make(lambda: ref.Signal("", "x", sample_rate=1e6))
    log_mine, log_ref = instrument(mine), cassette.make(lambda: instrument(theirs))
    for attr, value in SCRIPT:
        mine._qad = np.zeros(3, np.float32)   # a cached demodulation that the setter may have to drop
        setattr(mine, attr, value)
        cassette.make(lambda: setattr(theirs, "_qad", np.zeros(3, np.float32)))
        cassette.make(lambda: setattr(theirs, attr, value))
        assert (mine._qad is None) == cassette.want(lambda: theirs._qad is None), (attr, value)
        if attr != "block_protocol_update":
            got = getattr(mine, attr)
            assert got == cassette.want(lambda: getattr(theirs, attr)), (attr, value)
            assert type(got).__name__ == cassette.want(lambda: type(getattr(theirs, attr)).__name__), (attr, value)
    assert log_mine == cassette.want(lambda: log_ref)
    assert mine.modulation_order == cassette.want(lambda: theirs.modulation_order) == 8


def test_construction_defaults_match_reference(cassette, ref):
    from urh_b200.signalprocessing.Signal import Signal

    for kw in (dict(), dict(modulation="ASK", sample_rate=250e3, timestamp=3.0)):
        mine, theirs = Signal("", "n", **kw), cassette.make(lambda: ref.Signal("", "n", **kw))
        for attr in ("name", "tolerance", "samples_per_symbol", "pause_threshold", "message_length_divisor", "costas_loop_bandwidth",
                     "center", "sample_rate", "bits_per_symbol", "center_spacing", "modulation_type", "timestamp", "noise_threshold",
                     "already_demodulated", "modulation_order"):
            assert getattr(mine, attr) == cassette.want(lambda: getattr(theirs, attr)), attr
        assert mine.parameter_cache == cassette.want(lambda: theirs.parameter_cache)


def test_edit_operations_match_reference(cassette, ref):
    """insert / delete / mute / crop (Signal.py:613-651) on host data: same samples, same cached demodulation, same flags"""
    from urh_b200.signalprocessing.Signal import Signal

    rng = np.random.default_rng(8)
    for trial in range(20):
        n = int(rng.integers(20, 200))
        iq = rng.integers(-100, 100, (n, 2)).astype(np.int16) if trial % 2 else rng.standard_normal((n, 2)).astype(np.float32)
        mine, theirs = Signal.from_samples(iq.copy(), "e", 1e6), cassette.make(lambda: ref.Signal.from_samples(iq.copy(), "e", 1e6))
        qad = rng.standard_normal(n).astype(np.float32)
        a, b = sorted(int(v) for v in rng.integers(0, n, 2))
        op = trial % 4

        def edit(s):
            s._qad = qad.copy()
            s.parameter_cache["FSK"]["center"] = 0.5
            if op == 0:
                s.mute_range(a, b)
            elif op == 1:
                s.delete_range(a, b)
            elif op == 2:
                s.crop_to_range(a, max(b, a + 1))
            else:
                s.insert_data(a, iq[:5].copy())
        edit(mine)
        cassette.make(lambda: edit(theirs))
        assert same(mine.iq_array.data, cassette.want(lambda: np.asarray(theirs.iq_array.data))), (trial, op)
        assert mine.iq_array.data.dtype == cassette.want(lambda: theirs.iq_array.data.dtype)
        ref_qad = cassette.want(lambda: None if theirs._qad is None else np.asarray(theirs._qad))
        assert (mine._qad is None) == (ref_qad is None), (trial, op)
        if mine._qad is not None:
            assert same(mine._qad, ref_qad), (trial, op)
        assert mine.changed == cassette.want(lambda: theirs.changed) and mine.num_samples == cassette.want(lambda: theirs.num_samples)
        assert fingerprint(mine.parameter_cache) == cassette.want(lambda: fingerprint(theirs.parameter_cache))
