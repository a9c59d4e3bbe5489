"""GPU: the sharded PSK demodulator (urh_costas_shard_*) on one device.  2, 3, 4 and 8 shards of one capture are emulated one
after another in one process: each shard is speculated, its hypotheses ("the shard starts in candidate h's start state") are
hopped over, and the hypothesis whose start state equals the preceding shard's end state bit for bit is adopted
(dist.resolve_psk_chain); without one, the serial hand-over (urh_costas_shard_resolve) continues from that end state.  Shards
run strictly one after another: one sharded run is in flight per process.

The concatenated output must equal the serial loop (oracle.afp_demod) bit for bit, and every shard's end state the oracle's
loop state at the same sample (oracle.costas_from)."""
import ctypes as C

import numpy as np
import pytest

from conftest import bits_equal
from test_gpu_costas import SENTINEL, psk_burst, spikes, to_dtype

pytestmark = pytest.mark.gpu

N = 1_600_000
SPIKE = 700_000   # a shard boundary on an isolated spike inside a gap: the shard's sample 0 is live and stepped
# boundaries: 200k / 350k / 1.2M / 1.25M inside locked bursts, 500k in a gap of zeros, 700k / 800k in a gap with spikes;
# 1.2M .. 1.25M is a shard shorter than a super-chunk
SPLITS = {2: [200_000], 3: [500_000, 1_200_000], 4: [350_000, SPIKE, 1_250_000],
          8: [200_000, 350_000, 500_000, SPIKE, 800_000, 1_200_000, 1_250_000]}
LOCKED = {200_000, 350_000, 1_200_000, 1_250_000}
NOISE = {np.float32: 0.2, np.int8: 20.0}


def capture(order, dtype):
    rng = np.random.default_rng(order)
    x = psk_burst(N, order, rng)
    x[400_000:900_000] = 0
    spikes(x, 600_000, 900_000, rng)
    x[SPIKE] = np.exp(0.7j)
    x[900_000:] = psk_burst(N - 900_000, order, rng)   # a second burst, in its own lock branch
    return to_dtype(x, np.abs(x) > 0, dtype)


def run_shard(ctx, iq, lo, hi, first, noise, order, prev_end):
    """one shard: speculate, hop over the hypotheses, adopt or hand over -> (output, end state, how it was resolved)"""
    from urh_b200 import _lib, dist
    from urh_b200.device import DeviceArray

    lib = ctx.lib
    halo = dist.costas_halo(ctx)
    sb = dist.ShardBuffer(ctx, hi - lo, iq.dtype, halo=halo)
    sb.shard.set(iq[lo:hi])
    if not first:
        sb.halo.set(iq[lo - halo: lo])
    out = DeviceArray(ctx, (hi - lo,), np.float32)
    out.set(np.full(hi - lo, SENTINEL, np.uint32).view(np.float32))
    ctx.check(lib.urh_costas_shard_speculate(ctx.handle, C.c_void_p(sb.shard.ptr), _lib.dtype_code(iq.dtype), hi - lo, int(first),
                                             float(noise), int(order), 0.1, C.c_void_p(out.ptr)))
    h4 = np.zeros((4, 4), np.float32)
    count = C.c_int(0)
    ctx.check(lib.urh_costas_shard_hypotheses(ctx.handle, h4.ctypes.data_as(C.c_void_p), C.byref(count)))
    state = np.zeros(2, np.float32)
    if first:
        assert count.value == 1
        ctx.check(lib.urh_costas_shard_adopt(ctx.handle, 0, state.ctypes.data_as(C.c_void_p)))
        how = 0
    else:
        assert count.value == min(order, 4)
        hyps = [(h4[h, 0:2].tobytes(), h4[h, 2:4].tobytes()) for h in range(count.value)]
        picks, unresolved = dist.resolve_psk_chain([[(b"", prev_end.tobytes())], hyps])
        if unresolved == 2:
            how = picks[1]
            ctx.check(lib.urh_costas_shard_adopt(ctx.handle, how, state.ctypes.data_as(C.c_void_p)))
            assert state.tobytes() == hyps[how][1]   # the adopted run ends where its hypothesis said
        else:
            how = "resolve"
            ctx.check(lib.urh_costas_shard_resolve(ctx.handle, prev_end.ctypes.data_as(C.c_void_p), state.ctypes.data_as(C.c_void_p)))
    q = out.get()
    assert not (q.view(np.uint32) == SENTINEL).any(), "samples left unwritten"
    return q, state, how


@pytest.mark.parametrize("segs", (2, 4, 8, 16))
@pytest.mark.parametrize("shards", sorted(SPLITS))
@pytest.mark.parametrize("dtype", (np.float32, np.int8), ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("order", (2, 4))
def test_sharded_costas_on_one_gpu(oracle, ctx, monkeypatch, order, dtype, shards, segs):
    monkeypatch.setenv("URH_B200_COSTAS_SEGS", str(segs))
    iq = capture(order, dtype)
    noise = NOISE[dtype]
    bounds = [0] + SPLITS[shards] + [N]
    parts, hows = [], {}
    prev_end = None
    true_end = np.array([0.0, 1.5], np.float32)
    for r in range(shards):
        lo, hi = bounds[r], bounds[r + 1]
        q, state, how = run_shard(ctx, iq, lo, hi, r == 0, noise, order, prev_end)
        # the oracle's loop over the same range, continued from the true state (the capture's loop starts at sample 1)
        _, true_end = oracle.costas_from(iq[max(lo, 1):hi], noise, order, true_end)
        assert state.tobytes() == true_end.tobytes(), (r, lo, how, state, true_end)
        st4 = (C.c_int64 * 4)()
        ctx.check(ctx.lib.urh_costas_stitch_stats(ctx.handle, st4))
        assert st4[3] == segs
        parts.append(q)
        hows[lo] = how
        prev_end = state
    got = np.concatenate(parts)
    want = oracle.afp_demod(iq, noise, "PSK", order)
    assert bits_equal(got[1:], want[1:]) == 0
    for lo, how in hows.items():
        if lo in LOCKED:
            assert how != "resolve", hows    # a boundary inside a locked burst is resolved by adoption
    if SPIKE in hows:
        assert hows[SPIKE] == "resolve", hows
    print(order, np.dtype(dtype).name, shards, segs, hows)


def test_some_shard_adopts_another_lock_branch(oracle, ctx, monkeypatch):
    """the loop locks in a branch other than candidate 0's at some boundary: hypothesis h != 0 is adopted there"""
    monkeypatch.delenv("URH_B200_COSTAS_SEGS", raising=False)
    adopted = set()
    for order in (2, 4):
        iq = capture(order, np.float32)
        bounds = [0] + SPLITS[8] + [N]
        prev_end = None
        for r in range(8):
            q, prev_end, how = run_shard(ctx, iq, bounds[r], bounds[r + 1], r == 0, 0.2, order, prev_end)
            if bounds[r] in LOCKED:
                adopted.add((order, how))
    assert any(h != 0 for _, h in adopted), adopted
