"""CPU check of the host references behind tests/test_gpu_scan.py: loop-free numpy prefixes of the look-back scan's three test
operators (urh_selftest_scan: int64 sums, RunCarry under RunCarryOp, 2x2 uint64 matrix products mod 2^64), each equal to a
plain Python left fold of the operator's definition."""
import numpy as np

RC_DTYPE = np.dtype([("len", "<i8"), ("cls", "<i4"), ("flags", "<i4")])   # RunCarry (sparse.cuh), 16 bytes
RC_IDENTITY = (0, 0, 3)                                                      # the identity the library's scans start from
MAT_IDENTITY = np.array([1, 0, 0, 1], np.uint64)


def i64_prefixes(x):
    """exclusive prefix sums and the total of int64 x"""
    x = np.asarray(x, np.int64)
    incl = np.cumsum(x, dtype=np.int64)
    excl = np.zeros(len(x), np.int64)
    excl[1:] = incl[:-1]
    return excl, (int(incl[-1]) if len(x) else 0)


def rc_prefixes(x):
    """exclusive RunCarryOp prefixes of a RC_DTYPE table and its total (a RC_DTYPE array of one element).

    Elements with flags & 2 are identities and drop out.  Over the others, a run breaks at every element that is not whole
    (flags & 1) or has another class than the element before it; the prefix ending at element j is the run j is in: the
    lengths of that run up to j, j's class, and flags 1 only if the run started at the first element and that one was whole."""
    x = np.asarray(x, RC_DTYPE)
    live = (x["flags"] & 2) == 0
    e = x[live]
    m = len(e)
    p = np.zeros(m + 1, RC_DTYPE)
    p[0] = RC_IDENTITY
    if m:
        whole = (e["flags"] & 1) != 0
        brk = np.ones(m, bool)
        brk[1:] = ~(whole[1:] & (e["cls"][1:] == e["cls"][:-1]))
        run = np.cumsum(brk) - 1
        csum = np.cumsum(e["len"], dtype=np.int64)
        before = (csum - e["len"])[np.nonzero(brk)[0]]
        p["len"][1:] = csum - before[run]
        p["cls"][1:] = e["cls"]
        p["flags"][1:] = np.where(run == 0, e["flags"][0] & 1, 0)
    ahead = np.cumsum(live) - live   # live elements before each element
    return p[ahead], p[m:m + 1].copy()


def mat_mul(a, b):
    """row-major 2x2 uint64 products a @ b mod 2^64, element-wise over the leading axis"""
    r = np.empty(np.broadcast_shapes(a.shape, b.shape), np.uint64)
    with np.errstate(over="ignore"):   # wrapping is the operator
        r[..., 0] = a[..., 0] * b[..., 0] + a[..., 1] * b[..., 2]
        r[..., 1] = a[..., 0] * b[..., 1] + a[..., 1] * b[..., 3]
        r[..., 2] = a[..., 2] * b[..., 0] + a[..., 3] * b[..., 2]
        r[..., 3] = a[..., 2] * b[..., 1] + a[..., 3] * b[..., 3]
    return r


def mat_prefixes(x):
    """exclusive matrix-product prefixes of uint64[n, 4] and the total (uint64[4]): Hillis-Steele doubling, P_i <- P_(i-d) P_i"""
    p = np.array(x, np.uint64).reshape(-1, 4)
    n = len(p)
    d = 1
    while d < n:
        p[d:] = mat_mul(p[:-d], p[d:])
        d *= 2
    excl = np.empty_like(p)
    if n:
        excl[0] = MAT_IDENTITY
        excl[1:] = p[:-1]
    return excl, (p[-1].copy() if n else MAT_IDENTITY.copy())


def random_mats(rng, n):
    """[[1 + ab, a], [b, 1]] = [[1, a], [0, 1]] [[1, 0], [b, 1]]: determinant 1, so long products never collapse to 0 mod 2^64"""
    a = rng.integers(0, 1 << 64, n, dtype=np.uint64, endpoint=False)
    b = rng.integers(0, 1 << 64, n, dtype=np.uint64, endpoint=False)
    with np.errstate(over="ignore"):
        return np.stack([np.uint64(1) + a * b, a, b, np.ones(n, np.uint64)], axis=1)


# ---- the operators' definitions, folded left one element at a time --------------------------------------------------
def _rc_op(a, b):   # RunCarryOp, sparse.cuh
    if b[2] & 2:
        return a
    if a[2] & 2:
        return b
    if (b[2] & 1) and b[1] == a[1]:
        return (a[0] + b[0], a[1], a[2] & 1)
    return (b[0], b[1], 0)


def _mat_op(a, b):
    M = (1 << 64) - 1
    return ((a[0] * b[0] + a[1] * b[2]) & M, (a[0] * b[1] + a[1] * b[3]) & M,
            (a[2] * b[0] + a[3] * b[2]) & M, (a[2] * b[1] + a[3] * b[3]) & M)


def _fold(op, ident, elems):
    out, acc = [], ident
    for e in elems:
        out.append(acc)
        acc = op(acc, e)
    return out, acc


def random_rc(rng, n, classes=3):
    x = np.zeros(n, RC_DTYPE)
    x["len"] = rng.integers(0, 1 << 40, n)
    x["cls"] = rng.integers(0, classes, n)
    x["flags"] = rng.choice([0, 1, 1, 1, 2, 3], n)
    return x


def test_i64_prefixes_equal_left_fold():
    rng = np.random.default_rng(1)
    for n in (0, 1, 2, 3, 17, 200):
        x = rng.integers(-(1 << 40), 1 << 40, n)
        excl, total = i64_prefixes(x)
        ref, acc = _fold(lambda a, b: a + b, 0, [int(v) for v in x])
        assert excl.tolist() == ref and total == acc


def test_rc_prefixes_equal_left_fold():
    rng = np.random.default_rng(2)
    for trial in range(300):
        n = int(rng.integers(0, 60))
        x = random_rc(rng, n, classes=int(rng.integers(1, 4)))
        excl, total = rc_prefixes(x)
        ref, acc = _fold(_rc_op, RC_IDENTITY, [(int(e["len"]), int(e["cls"]), int(e["flags"])) for e in x])
        assert [tuple(int(v) for v in e) for e in excl] == ref, trial
        assert tuple(int(v) for v in total[0]) == acc, trial


def test_mat_prefixes_equal_left_fold():
    rng = np.random.default_rng(3)
    for n in (0, 1, 2, 3, 5, 31, 64, 100):
        x = random_mats(rng, n)
        excl, total = mat_prefixes(x)
        ref, acc = _fold(_mat_op, (1, 0, 0, 1), [tuple(int(v) for v in e) for e in x])
        assert [tuple(int(v) for v in e) for e in excl] == ref
        assert tuple(int(v) for v in total) == acc


def test_mat_operator_is_not_commutative():
    """a dropped, repeated or swapped factor must change the product"""
    x = random_mats(np.random.default_rng(4), 3)
    ab, ba = mat_mul(x[0], x[1]), mat_mul(x[1], x[0])
    assert not np.array_equal(ab, ba)
    assert not np.array_equal(mat_mul(ab, x[2]), mat_mul(ba, x[2]))
