"""The reference's answers for the CPU tests that compare host logic with the reference's own Python, stored under tests/golden/.

A test asks for every reference result through ``Cassette.want(thunk)``.  With URH_RECORD_GOLDEN=1 (only where the reference tree
exists) the thunk runs against the reference and its result is recorded; ``close()`` writes tests/golden/ref_<module>.json.
Everywhere else the recorded results are replayed in order and the thunk never runs, so the tests need nothing outside the
repository.  Regenerate after changing such a test:

    URH_RECORD_GOLDEN=1 python -m pytest tests/test_host_vs_reference.py tests/test_signal_files.py tests/test_signal_params.py

A randomized trial's answers are usually recorded as one ``fingerprint`` (10 hex digits of a hash of the values in plain Python
form).  Arrays of more than INLINE elements are stored as a digest of their values (shape, value kind, float64 / complex128 / int64
bytes with -0 folded into +0, i.e. what np.array_equal compares); compare them with ``same``.
"""
import base64
import hashlib
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
RECORD = os.environ.get("URH_RECORD_GOLDEN") == "1"
INLINE = 64


def digest(a) -> str:
    a = np.asarray(a)
    kind = a.dtype.kind
    if kind == "f":
        a = a.astype(np.float64) + 0.0
    elif kind == "c":
        a = a.astype(np.complex128) + 0.0
    elif kind in "iub":
        kind = "i"
        a = a.astype(np.int64)
    else:
        raise TypeError("no digest for dtype %s" % a.dtype)
    h = hashlib.sha256(("%s%s" % (kind, a.shape)).encode())
    h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


class Digest:
    """a large recorded array, known by its digest"""

    def __init__(self, d):
        self.d = d

    def __eq__(self, other):
        return other.d == self.d if isinstance(other, Digest) else digest(other) == self.d

    __hash__ = None


def same(mine, expected) -> bool:
    """np.array_equal(mine, expected) for a recorded array (stored inline or as a digest)"""
    if isinstance(expected, Digest):
        return expected == mine
    return bool(np.array_equal(mine, expected))


def _plain(v):
    if isinstance(v, np.ndarray):
        return _plain(v.tolist())
    if isinstance(v, np.generic):
        return _plain(v.item())
    if isinstance(v, (list, tuple)):
        return [_plain(x) for x in v]
    if isinstance(v, bool):
        return int(v)
    if isinstance(v, complex):
        return [_plain(v.real), _plain(v.imag)]
    if isinstance(v, float) and v.is_integer():
        return int(v) if v != 0 else 0   # 3.0 == 3 and -0.0 == 0, as == sees them
    if isinstance(v, np.dtype):
        return str(v)
    if isinstance(v, dict):
        return sorted([json.dumps(_plain(k)), _plain(x)] for k, x in v.items())
    return v


def fingerprint(v) -> str:
    """40-bit digest of a nest of lists / tuples / dicts / arrays / numbers in plain Python form (equal as == compares them)"""
    return hashlib.sha256(json.dumps(_plain(v)).encode()).hexdigest()[:10]


def _b64(b):
    return base64.b64encode(b).decode()


def encode(v):
    if v is None or isinstance(v, (bool, int, float, str)):
        return v
    if isinstance(v, np.ndarray):
        if v.dtype.kind not in "biufc":
            raise TypeError("cannot record an array of dtype %s" % v.dtype)
        if v.size > INLINE:
            return {"digest": digest(v)}
        return {"nd": v.dtype.str, "shape": list(v.shape), "b64": _b64(np.ascontiguousarray(v).tobytes())}
    if isinstance(v, np.generic):
        return {"np": v.dtype.str, "b64": _b64(np.asarray(v).tobytes())}
    if isinstance(v, np.dtype):
        return {"dtype": v.str}
    if isinstance(v, tuple):
        return {"tuple": [encode(x) for x in v]}
    if isinstance(v, list):
        return [encode(x) for x in v]
    if isinstance(v, dict):
        return {"dict": [[encode(k), encode(x)] for k, x in v.items()]}
    raise TypeError("cannot record %r" % type(v))


def decode(v):
    if isinstance(v, list):
        return [decode(x) for x in v]
    if not isinstance(v, dict):
        return v
    if "digest" in v:
        return Digest(v["digest"])
    if "nd" in v:
        return np.frombuffer(base64.b64decode(v["b64"]), dtype=np.dtype(v["nd"])).reshape(v["shape"]).copy()
    if "np" in v:
        return np.frombuffer(base64.b64decode(v["b64"]), dtype=np.dtype(v["np"]))[0]
    if "dtype" in v:
        return np.dtype(v["dtype"])
    if "tuple" in v:
        return tuple(decode(x) for x in v["tuple"])
    if "dict" in v:
        return {_key(decode(k)): decode(x) for k, x in v["dict"]}
    raise ValueError("unknown record %r" % v)


def _key(k):
    return tuple(k) if isinstance(k, list) else k


class Cassette:
    def __init__(self, module: str, test: str):
        self.path = os.path.join(GOLDEN, "ref_%s.json" % module)
        self.test = test
        self.recording = RECORD
        self.i = 0
        if self.recording:
            self.values = []
        else:
            with open(self.path) as fh:
                data = json.load(fh)
            assert test in data, "no recorded reference answers for %s in %s" % (test, self.path)
            self.values = [decode(v) for v in data[test]]

    def want(self, thunk):
        """the reference's answer: thunk() while recording, else the next recorded value"""
        if self.recording:
            enc = encode(thunk())
            self.values.append(enc)
            return decode(enc)   # compared exactly as it will be when replayed
        assert self.i < len(self.values), "%s asks for more reference answers than were recorded" % self.test
        self.i += 1
        return self.values[self.i - 1]

    def make(self, thunk):
        """a reference object: only exists while recording"""
        return thunk() if self.recording else None

    def close(self):
        if not self.recording:
            assert self.i == len(self.values), "%s used %d of %d recorded reference answers" % (self.test, self.i, len(self.values))
            return
        data = {}
        if os.path.isfile(self.path):
            with open(self.path) as fh:
                data = json.load(fh)
        data[self.test] = self.values
        with open(self.path, "w") as fh:   # one test per line
            fh.write("{\n" + ",\n".join("%s:%s" % (json.dumps(k), json.dumps(data[k], separators=(",", ":"))) for k in sorted(data)) + "\n}\n")
