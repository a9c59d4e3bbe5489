"""W ranks of urh_b200.dist as threads of one process, all on device 0 (a test helper, like tests/*_cases.py).

Each rank has its own ``_lib.Context`` (its own stream and arena), as each torchrun process has.  The ranks take turns: exactly one
holds the baton, and it gives the baton up only while it waits inside a collective.  At every hand-over the outgoing rank's context
is synchronised and ``_lib._default_ctx[0]`` is pointed at the incoming rank's context, so code that calls ``default_context()``
mid-call (``AI.detect_center``, ``util.get_magnitudes``, ``IQArray``) runs on the running rank's stream, as it does under torchrun.

The five NCCL entry points dist.py calls from Python are replaced on the loaded library by host stand-ins that find the calling rank
from the context handle.  They reduce in rank order.  No NCCL communicator is created and no process or daemon is started.

Failures propagate: when a rank raises, every rank waiting in a collective raises ``WorldError`` naming itself and the collective, and
``run`` re-raises the first error.  A collective no other rank can match (every live rank waits), or a wait longer than ``timeout``,
is reported the same way instead of hanging.  Ranks that have not started yet still run, so a test can check that every rank raises
the same error before its first collective (``errors``).
"""
import collections
import copy
import ctypes as C
import threading

import numpy as np

NCCL_ENTRIES = ("urh_nccl_allgather_host", "urh_nccl_allreduce_host_i64", "urh_nccl_allreduce_f64", "urh_nccl_allgather",
                "urh_nccl_sendrecv")
HOST_STAGE = 65536   # urh_nccl_allgather_host's staging buffer (nccl.cu)


class WorldError(AssertionError):
    """a rank left waiting: an unmatched collective, a timeout, another rank's failure, or a call from outside the world"""


def _addr(p):
    if p is None:
        return 0
    return int(p.value or 0) if hasattr(p, "value") else int(p)


class HostExchange(object):
    """dist.HostExchange for one rank of a OneGpuWorld: the same four members, over the world's collectives"""

    def __init__(self, world, rank):
        self._w = world
        self.rank = rank
        self.world = world.world

    def allgather(self, obj):
        return self._w.collective(self.rank, "allgather", obj)

    def broadcast(self, obj, src=0):
        return self._w.collective(self.rank, "broadcast(src=%d)" % src, obj)[src]

    def barrier(self):
        self._w.collective(self.rank, "barrier", None)


class OneGpuWorld(object):
    def __init__(self, world, contexts=None, timeout=120.0):
        """contexts: one ``_lib.Context`` per rank (None: plain-Python ranks, no device)"""
        if not 1 <= int(world) <= 8:
            raise ValueError("world size %d: 1 ... 8 ranks" % world)
        self.world = int(world)
        self.contexts = list(contexts) if contexts is not None else None
        assert self.contexts is None or len(self.contexts) == self.world
        self.timeout = float(timeout)
        self.hx = [HostExchange(self, r) for r in range(self.world)]
        self.calls = collections.Counter()    # collectives by name, counted once per collective (not per rank)
        self._cv = threading.Condition()
        self._reset()

    def _reset(self):
        W = self.world
        self._turn = None
        self._state = ["ready"] * W    # ready (not started) / run / wait / done
        self._pred = [None] * W
        self._what = [None] * W
        self._seq = [0] * W            # collectives entered per rank
        self._slots = {}               # collective number -> [name, values, entered, read]
        self._mail = collections.defaultdict(collections.deque)   # (src, dst) -> deposited sends
        self._first = None             # (rank, exception) of the first failure
        self.errors = [None] * W
        self.results = [None] * W

    # ---- running the ranks --------------------------------------------------------------------------------------------------
    def run(self, fn, reraise=True):
        """fn(rank) on every rank, taking turns -> [result per rank].  Re-raises the first failure unless ``reraise`` is False
        (then ``errors`` holds every rank's exception or None)."""
        from urh_b200 import _lib

        self._reset()
        saved = _lib._default_ctx.get(0, None) if self.contexts else None
        threads = [threading.Thread(target=self._main, args=(r, fn), name="urh-rank-%d" % r, daemon=True) for r in range(self.world)]
        with self._cv:
            self._give(0)
        try:
            for t in threads:
                t.start()
            for t in threads:
                t.join(self.timeout * 4)
            alive = [t.name for t in threads if t.is_alive()]
            if alive:
                raise WorldError("ranks still running after %.0f s: %s" % (self.timeout * 4, alive))
        finally:
            if self.contexts:
                if saved is None:
                    _lib._default_ctx.pop(0, None)
                else:
                    _lib._default_ctx[0] = saved
        if reraise and self._first is not None:
            raise self._first[1]
        return list(self.results)

    def _main(self, r, fn):
        with self._cv:
            if not self._cv.wait_for(lambda: self._turn == r, self.timeout):
                self._fail(r, WorldError("rank %d never got the baton to start" % r))
                self._state[r] = "done"
                return
            self._state[r] = "run"
        try:
            self.results[r] = fn(r)
        except BaseException as e:   # noqa: B902 - every failure of a rank is reported
            with self._cv:
                self._fail(r, e)
        finally:
            with self._cv:
                self._state[r] = "done"
                self._hand_over(r)

    def _fail(self, r, e):
        self.errors[r] = e
        if self._first is None:
            self._first = (r, e)

    def _runnable(self, q):
        return self._state[q] == "ready" or (self._state[q] == "wait" and (self._first is not None or self._pred[q]()))

    def _give(self, q):
        self._turn = q
        if self.contexts:
            from urh_b200 import _lib
            _lib._default_ctx[0] = self.contexts[q]
        self._cv.notify_all()

    def _hand_over(self, r):
        """rank r gives up the baton (it waits in a collective or is done); lock held"""
        if self.contexts:
            try:
                self.contexts[r].sync()
            except Exception as e:
                self._fail(r, e)
        for k in range(1, self.world + 1):
            q = (r + k) % self.world
            if self._runnable(q):
                self._give(q)
                return
        waiting = [q for q in range(self.world) if self._state[q] == "wait"]
        if waiting:
            self._fail(waiting[0], WorldError("no rank can proceed: " + "; ".join("rank %d waits in %s" % (q, self._what[q]) for q in waiting)))
            self._give(waiting[0])
        else:
            self._turn = None
            self._cv.notify_all()

    def _block(self, r, pred, what):
        """rank r (holding the baton, lock held) waits until pred() holds"""
        if pred():
            return
        self._state[r], self._pred[r], self._what[r] = "wait", pred, what
        self._hand_over(r)
        if not self._cv.wait_for(lambda: self._turn == r, self.timeout):
            err = WorldError("rank %d timed out after %.0f s waiting in %s" % (r, self.timeout, what))
            self._fail(r, err)
            self._state[r] = "done"
            raise err
        self._state[r] = "run"
        if not pred():
            fr, fe = self._first
            raise WorldError("rank %d left waiting in %s: rank %d failed first (%s: %s)" % (r, what, fr, type(fe).__name__, fe))

    def _check_turn(self, r, what):
        if not 0 <= r < self.world or self._turn != r:
            err = WorldError("%s called by rank %s while rank %s holds the baton" % (what, r, self._turn))
            self._fail(r if 0 <= r < self.world else 0, err)
            raise err

    # ---- collectives --------------------------------------------------------------------------------------------------------
    def collective(self, r, name, value):
        """the k-th collective of every rank meets the k-th of every other: -> [value of rank q for q in range(world)]"""
        with self._cv:
            self._check_turn(r, name)
            k = self._seq[r]
            self._seq[r] += 1
            slot = self._slots.get(k)
            if slot is None:
                slot = self._slots[k] = [name, [None] * self.world, [False] * self.world, 0]
                self.calls[name.split("(")[0]] += 1
            if slot[0] != name:
                err = WorldError("collective #%d: rank %d calls %s, another rank called %s" % (k, r, name, slot[0]))
                self._fail(r, err)
                raise err
            slot[1][r] = copy.deepcopy(value)
            slot[2][r] = True
            self._block(r, lambda: all(slot[2]), "%s #%d" % (name, k))
            out = copy.deepcopy(slot[1])
            slot[3] += 1
            if slot[3] == self.world:
                del self._slots[k]
            return out

    def send(self, r, peer, payload):
        """deposit a point-to-point message for `peer` (never blocks)"""
        with self._cv:
            self._check_turn(r, "send")
            if not 0 <= peer < self.world or peer == r:
                err = WorldError("rank %d sends to rank %d of a %d-rank world" % (r, peer, self.world))
                self._fail(r, err)
                raise err
            self._mail[(r, peer)].append(payload)

    def recv(self, r, peer):
        """the oldest message `peer` deposited for rank r, waiting until there is one"""
        with self._cv:
            self._check_turn(r, "recv")
            if not 0 <= peer < self.world or peer == r:
                err = WorldError("rank %d receives from rank %d of a %d-rank world" % (r, peer, self.world))
                self._fail(r, err)
                raise err
            box = self._mail[(peer, r)]
            self._block(r, lambda: len(box) > 0, "recv from rank %d" % peer)
            return box.popleft()

    def undelivered(self):
        """(src, dst, count) of sends nobody received"""
        return [(s, d, len(b)) for (s, d), b in self._mail.items() if b]

    # ---- the NCCL stand-ins -------------------------------------------------------------------------------------------------
    def install(self, monkeypatch, lib):
        """replace dist.py's five NCCL entry points on the loaded library `lib` (restored by pytest's monkeypatch)"""
        assert self.contexts is not None, "the NCCL stand-ins need one context per rank"
        ranks = {_addr(ctx.handle): r for r, ctx in enumerate(self.contexts)}
        memcpy_d2h, memcpy_h2d = lib.urh_memcpy_d2h, lib.urh_memcpy_h2d

        def rank_of(handle, entry):
            r = ranks.get(_addr(handle))
            if r is None:
                err = WorldError("%s called from a context outside the %d-rank world" % (entry, self.world))
                with self._cv:
                    self._fail(0, err)
                raise err
            return r

        def d2h(r, ptr, nbytes):
            host = np.empty(nbytes, np.uint8)
            if nbytes:
                self.contexts[r].check(memcpy_d2h(self.contexts[r].handle, C.c_void_p(host.ctypes.data), C.c_void_p(ptr), nbytes))
            return host

        def h2d(r, ptr, host):
            if host.nbytes:
                ctx = self.contexts[r]
                ctx.check(memcpy_h2d(ctx.handle, C.c_void_p(ptr), C.c_void_p(host.ctypes.data), host.nbytes))
                ctx.sync()

        def reduce(parts, op):
            acc = parts[0].copy()
            for p in parts[1:]:   # rank order
                acc = acc + p if op == 0 else (np.maximum(acc, p) if op == 1 else np.minimum(acc, p))
            return acc

        def allgather_host(handle, h_send, h_recv, nbytes):
            r = rank_of(handle, "urh_nccl_allgather_host")
            if ((nbytes + 255) & ~255) + nbytes * self.world > HOST_STAGE:
                raise WorldError("urh_nccl_allgather_host: %d bytes per rank exceed the staging buffer" % nbytes)
            parts = self.collective(r, "nccl_allgather_host(%d B)" % nbytes, C.string_at(_addr(h_send), nbytes))
            C.memmove(_addr(h_recv), b"".join(parts), nbytes * self.world)
            return 0

        def allreduce_host_i64(handle, h_buf, count, op):
            r = rank_of(handle, "urh_nccl_allreduce_host_i64")
            if count <= 0:
                return 0
            mine = np.frombuffer(C.string_at(_addr(h_buf), count * 8), dtype=np.int64).copy()
            out = reduce(self.collective(r, "nccl_allreduce_host_i64(%d, op %d)" % (count, op), mine), op)
            C.memmove(_addr(h_buf), out.ctypes.data, out.nbytes)
            return 0

        def allreduce_f64(handle, d_buf, count, op):
            r = rank_of(handle, "urh_nccl_allreduce_f64")
            mine = d2h(r, _addr(d_buf), count * 8).view(np.float64)
            out = reduce(self.collective(r, "nccl_allreduce_f64(%d, op %d)" % (count, op), mine), op)
            h2d(r, _addr(d_buf), np.ascontiguousarray(out))
            return 0

        def allgather(handle, d_send, d_recv, nbytes):
            r = rank_of(handle, "urh_nccl_allgather")
            parts = self.collective(r, "nccl_allgather(%d B)" % nbytes, d2h(r, _addr(d_send), nbytes))
            h2d(r, _addr(d_recv), np.concatenate(parts))
            return 0

        def sendrecv(handle, d_send, send_bytes, send_peer, d_recv, recv_bytes, recv_peer):
            r = rank_of(handle, "urh_nccl_sendrecv")
            if send_peer >= 0 and send_bytes > 0:
                self.send(r, send_peer, d2h(r, _addr(d_send), send_bytes))
            if recv_peer >= 0 and recv_bytes > 0:
                got = self.recv(r, recv_peer)
                if got.nbytes != recv_bytes:
                    raise WorldError("rank %d expects %d bytes from rank %d, which sent %d" % (r, recv_bytes, recv_peer, got.nbytes))
                h2d(r, _addr(d_recv), got)
            return 0

        fakes = {"urh_nccl_allgather_host": allgather_host, "urh_nccl_allreduce_host_i64": allreduce_host_i64,
                 "urh_nccl_allreduce_f64": allreduce_f64, "urh_nccl_allgather": allgather, "urh_nccl_sendrecv": sendrecv}
        for name in NCCL_ENTRIES:
            monkeypatch.setattr(lib, name, fakes[name])
