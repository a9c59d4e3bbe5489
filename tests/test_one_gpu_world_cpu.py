"""CPU suite: the in-process world of tests/one_gpu_world.py with plain-Python ranks (no device).  Collectives return every
rank's contribution in rank order, reductions fold in rank order, sends pair with receives, and a failure or an unmatched
collective surfaces as an error naming the rank and the collective instead of a hang."""
import os
import sys
import threading
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from one_gpu_world import OneGpuWorld, WorldError  # noqa: E402

WORLDS = (1, 2, 3, 5, 8)


@pytest.mark.parametrize("W", WORLDS)
def test_allgather_and_broadcast_order(W):
    w = OneGpuWorld(W, timeout=10)
    order = []

    def rank(r):
        hx = w.hx[r]
        order.append(r)
        got = hx.allgather(("r", r, [r] * r))
        b = hx.broadcast("from %d" % r, src=W - 1)
        hx.barrier()
        return got, b

    res = w.run(rank)
    assert order == list(range(W))   # the baton starts the ranks in rank order
    for got, b in res:
        assert got == [("r", q, [q] * q) for q in range(W)]
        assert b == "from %d" % (W - 1)
    assert w.calls == {"allgather": 1, "broadcast": 1, "barrier": 1}


def test_exactly_one_rank_runs():
    w = OneGpuWorld(5, timeout=10)
    running = []
    overlap = []

    def rank(r):
        for step in range(4):
            running.append(r)
            if len(running) > 1:
                overlap.append(list(running))
            time.sleep(0.002)
            running.remove(r)
            w.hx[r].allgather(step)

    w.run(rank)
    assert not overlap


class _FakeCtx(object):
    """a context handle without a device: "device" pointers are host pointers"""

    def __init__(self, h):
        import ctypes as C
        self.handle = C.c_void_p(h)

    def sync(self):
        pass

    def check(self, rc):
        assert rc == 0


def _fake_lib():
    import ctypes as C

    class FakeLib(object):
        pass

    lib = FakeLib()
    for name in ("urh_nccl_allgather_host", "urh_nccl_allreduce_host_i64", "urh_nccl_allreduce_f64", "urh_nccl_allgather",
                 "urh_nccl_sendrecv"):
        setattr(lib, name, None)
    lib.urh_memcpy_d2h = lib.urh_memcpy_h2d = lambda h, dst, src, n: C.memmove(dst.value, src.value, n) and 0
    return lib


def test_sum_and_max_fold_in_rank_order(monkeypatch):
    """the NCCL stand-ins reduce in rank order: 1e16 + 1 - 1e16 + 1 is 1.0 that way round, 0.0 the other"""
    import ctypes as C

    vals = [1e16, 1.0, -1e16, 1.0]
    ctxs = [_FakeCtx(0x1000 + 16 * r) for r in range(4)]
    w = OneGpuWorld(4, contexts=ctxs, timeout=10)
    lib = _fake_lib()
    w.install(monkeypatch, lib)
    monkeypatch.setattr("urh_b200._lib._default_ctx", {})

    def rank(r):
        h = ctxs[r].handle
        out = {}
        for op in (0, 1, 2):
            buf = np.array([r * 10, -r, 7], dtype=np.int64)
            assert lib.urh_nccl_allreduce_host_i64(h, buf.ctypes.data_as(C.c_void_p), 3, op) == 0
            out["i64", op] = buf.tolist()
            f = np.array([vals[r], -vals[r], float(r)], dtype=np.float64)
            assert lib.urh_nccl_allreduce_f64(h, C.c_void_p(f.ctypes.data), 3, op) == 0
            out["f64", op] = f.tolist()
        send = np.array([vals[r]], dtype=np.float64)
        recv = np.zeros(4, dtype=np.float64)
        lib.urh_nccl_allgather_host(h, send.ctypes.data_as(C.c_void_p), recv.ctypes.data_as(C.c_void_p), 8)
        out["gather_host"] = recv.tolist()
        d_recv = np.zeros(4, dtype=np.float64)
        lib.urh_nccl_allgather(h, C.c_void_p(send.ctypes.data), C.c_void_p(d_recv.ctypes.data), 8)
        out["gather"] = d_recv.tolist()
        return out

    for out in w.run(rank):
        assert out["i64", 0] == [60, -6, 28] and out["i64", 1] == [30, 0, 7] and out["i64", 2] == [0, -3, 7]
        assert out["f64", 0] == [1.0, -1.0, 6.0]
        assert out["f64", 1] == [1e16, 1e16, 3.0] and out["f64", 2] == [-1e16, -1e16, 0.0]
        assert out["gather_host"] == vals and out["gather"] == vals
    assert (vals[3] + vals[2]) + vals[1] + vals[0] == 0.0   # what the rank order decides
    assert w.calls["nccl_allreduce_f64"] == 3 and w.calls["nccl_allgather_host"] == 1


def test_a_call_from_outside_the_world_fails(monkeypatch):
    import ctypes as C

    lib = _fake_lib()
    w = OneGpuWorld(2, contexts=[_FakeCtx(0x2000), _FakeCtx(0x2010)], timeout=10)
    w.install(monkeypatch, lib)
    monkeypatch.setattr("urh_b200._lib._default_ctx", {})
    buf = np.zeros(1, np.int64)
    with pytest.raises(WorldError, match="outside the 2-rank world"):
        w.run(lambda r: lib.urh_nccl_allreduce_host_i64(C.c_void_p(0x9999), buf.ctypes.data_as(C.c_void_p), 1, 0))


@pytest.mark.parametrize("W", (2, 3, 5))
def test_sendrecv_pairing(W):
    """a ring exchange both ways (exchange_halos' shape), then fetch_range's one-sided sends to an owner"""
    w = OneGpuWorld(W, timeout=10)

    def rank(r):
        got = {}
        if r + 1 < W:
            w.send(r, r + 1, ("tail", r))
        if r > 0:
            got["left"] = w.recv(r, r - 1)
        if r > 0:
            w.send(r, r - 1, ("head", r))
        if r + 1 < W:
            got["right"] = w.recv(r, r + 1)
        owner = W // 2
        if r == owner:
            got["fetched"] = [w.recv(r, q) for q in range(W) if q != owner]
        else:
            w.send(r, owner, ("part", r))    # one-sided: this rank receives nothing
        # two messages between the same pair arrive in order
        if r == 0 and W > 1:
            w.send(0, 1, "first")
            w.send(0, 1, "second")
        if r == 1:
            got["pair"] = [w.recv(1, 0), w.recv(1, 0)]
        return got

    res = w.run(rank)
    for r, got in enumerate(res):
        if r > 0:
            assert got["left"] == ("tail", r - 1)
        if r + 1 < W:
            assert got["right"] == ("head", r + 1)
    assert res[W // 2]["fetched"] == [("part", q) for q in range(W) if q != W // 2]
    assert res[1]["pair"] == ["first", "second"]
    assert w.undelivered() == []


@pytest.mark.parametrize("W", (2, 3, 8))
@pytest.mark.parametrize("who", ("first", "last"))
def test_an_exception_on_one_rank_surfaces(W, who):
    w = OneGpuWorld(W, timeout=10)
    bad = 0 if who == "first" else W - 1

    def rank(r):
        w.hx[r].allgather(r)
        if r == bad:
            raise KeyError("rank %d broke" % r)
        w.hx[r].allgather(r)
        return r

    with pytest.raises(KeyError, match="rank %d broke" % bad):
        w.run(rank)
    assert isinstance(w.errors[bad], KeyError)
    for r in range(W):
        if r != bad:
            assert isinstance(w.errors[r], WorldError)
            assert "rank %d left waiting in allgather #1" % r in str(w.errors[r])
    assert not [t for t in threading.enumerate() if t.name.startswith("urh-rank-")]


def test_every_rank_raising_before_its_first_collective_is_seen_on_every_rank():
    w = OneGpuWorld(3, timeout=10)

    def rank(r):
        raise ValueError("rank %d: shard too short" % r)

    with pytest.raises(ValueError, match="rank 0"):
        w.run(rank)
    assert [type(e) for e in w.errors] == [ValueError] * 3


def test_an_unmatched_collective_is_reported():
    """rank 1 returns without the second all-gather: rank 0 waits in it and nobody can proceed"""
    w = OneGpuWorld(3, timeout=10)

    def rank(r):
        w.hx[r].allgather(r)
        if r != 1:
            w.hx[r].allgather("again")

    t0 = time.time()
    with pytest.raises(WorldError, match="no rank can proceed: rank 0 waits in allgather #1; rank 2 waits in allgather #1"):
        w.run(rank)
    assert time.time() - t0 < 5


def test_mismatched_collectives_are_reported():
    w = OneGpuWorld(2, timeout=10)

    def rank(r):
        w.hx[r].allgather(r)
        if r == 0:
            w.hx[r].allgather("again")
        else:
            w.hx[r].barrier()

    with pytest.raises(WorldError, match="collective #1: rank 0 calls allgather, another rank called barrier"):
        w.run(rank)
    assert "rank 1 left waiting in barrier #1" in str(w.errors[1])


def test_a_rank_left_waiting_times_out():
    """a lone rank waiting for a message nobody sends: the world ends with an error naming the rank and the wait"""
    w = OneGpuWorld(2, timeout=10)

    def rank(r):
        if r == 1:
            w.recv(1, 0)

    with pytest.raises(WorldError, match="rank 1 waits in recv from rank 0"):
        w.run(rank)


def test_a_wait_past_the_timeout_is_reported():
    """rank 0 holds the baton too long: rank 1, waiting in the second all-gather, gives up after the timeout"""
    w = OneGpuWorld(2, timeout=0.5)

    def rank(r):
        w.hx[r].allgather(r)
        if r == 0:
            time.sleep(1.0)
            return None
        w.hx[r].allgather(r)

    with pytest.raises(WorldError, match="rank 1 timed out after 0 s waiting in allgather #1"):
        w.run(rank)


@pytest.mark.parametrize("W", (3, 5))
def test_center_protocol_folds_the_window_partials_in_rank_order(W):
    """Σ partials of 1, 1e16, -1e16 (then zeros) sum to 0 in rank order and to 1 in reverse: the bin edges the histogram receives
    must be the rank-order ones on every rank"""
    from urh_b200 import dist as udist
    from urh_b200.ainterpretation import AutoInterpretation as AI

    sums = [1.0, 1e16, -1e16] + [0.0] * (W - 3)
    parts = [np.array([100.0, -5.0 - q, 5.0 + q, sums[q], 1000.0]) for q in range(W)]
    w = OneGpuWorld(W, timeout=10)
    seen = [None] * W

    def rank(r):
        hx = w.hx[r]

        def histogram(lr0, lr1, edges):
            seen[r] = np.array(edges)
            return np.arange(len(edges) - 1) % 7

        def allreduce(y):
            return np.sum(hx.allgather(np.asarray(y)), axis=0)
        return udist.center_protocol(r, W, 1000, lambda lr0, lr1: parts[r], histogram,
                                     lambda v: np.array(hx.allgather(list(np.asarray(v)))), allreduce)

    w.run(rank)
    total = W * 1000
    r0, r1 = AI.center_rank_window(total)

    def edges(order):
        g = np.array([sum(p[0] for p in parts), min(p[1] for p in parts), max(p[2] for p in parts), 0.0, 0.0])
        for q in order:
            g[3] += parts[q][3]
            g[4] += parts[q][4]
        return AI.center_bin_edges(AI.center_stats_from_window(total, r0, r1, g))

    want, reverse = edges(range(W)), edges(reversed(range(W)))
    assert len(want) != len(reverse) or not np.array_equal(want, reverse)   # the case tells the two orders apart
    for r in range(W):
        assert np.array_equal(seen[r], want), r
