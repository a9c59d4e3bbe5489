"""GPU: urh_segment_messages keeps a resident capture's segments in the context for urh_fetch_segments, so a capture with more
messages than any first guess at a host buffer is segmented by one dense pass, one candidate collection and one state machine."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def messages(nmsg):
    """nmsg messages of 10 magnitudes above a threshold of 0.5, each followed by 10 below"""
    return np.tile(np.repeat([0.9, 0.05], 10), nmsg)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_many_segments_from_one_pass(ctx, oracle, dtype):
    from urh_b200.ainterpretation import AutoInterpretation as AI
    from urh_b200.device import to_device

    def segment(mags):
        d = to_device(mags, ctx)
        before = ctx.launch_count()
        got = AI.segment_messages_from_magnitudes(d, 0.5)
        return got, ctx.launch_count() - before

    few = messages(3).astype(dtype)
    many = messages((1 << 16) + 5).astype(dtype)
    got_few, launches_few = segment(few)
    got, launches = segment(many)
    assert got_few == oracle.segment_messages_from_magnitudes(few, 0.5)
    assert len(got) == (1 << 16) + 5
    assert got == oracle.segment_messages_from_magnitudes(many, 0.5)
    # the dense pass, the collector's two scans and its gather, whether the call returns 3 segments or 65541
    assert launches == launches_few == 4, (launches_few, launches)
