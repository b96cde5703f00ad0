"""Kernel launches of one KLT call of each kind (needs a GPU).

The KLT entry points fold launches together: the gain tracker writes the feature table and the
suppression marks itself, the detector's prefilter runs on a side stream next to the tracker, and
klt_select_refill writes the provided set to both feature buffers so that the advance that follows
needs no copy.  A lost fold leaves every output bit-identical and only adds a launch, so these counts
are the one place it shows.  At 640x480 with 6 levels the pyramid tail is 4 launches; a group of 3
cameras uploaded from the host runs the front pass as 2 launches (two half-groups)."""
import numpy as np
import pytest

from helpers import live_cfg, seq

pytestmark = pytest.mark.gpu

W, H, L, FW, FH, NCAM = 640, 480, 6, 32, 32, 3


def _count(api, fn):
    n0 = api.kernel_launch_count()
    fn()
    return api.kernel_launch_count() - n0


@pytest.mark.parametrize("gain", [True, False])
def test_single_tracker_launches(api, gain):
    # gain: front + prefilter + 4 pyramid + fused tracker (with status and marks) + verify + select;
    # 2x2: front + prefilter + 4 pyramid + tracker + status + suppress + verify + select
    want = {"detect": 8, "redetect": 9, "track": 7, "first": 9, "next": 10} if gain else \
           {"detect": 8, "redetect": 11, "track": 8, "first": 9, "next": 12}
    s = seq(H, W, 31, n=6)
    t = api.KltTracker(live_cfg(gain=gain, min_corner=1500.0), W, H, L, FW, FH)
    got = {"detect": _count(api, lambda: t.detect(s.frames[0]))}
    t.advance()
    got["redetect"] = _count(api, lambda: t.redetect(s.frames[1]))
    t.advance()
    got["track"] = _count(api, lambda: t.track(s.frames[2]))
    t.advance()
    got["first"] = _count(api, lambda: t.first(s.frames[3]))
    got["next"] = _count(api, lambda: t.next(s.frames[4]))
    t.close()
    assert got == want


def test_group_launches(api):
    import torch

    cfg = live_cfg(gain=True, min_corner=1500.0)
    seqs = [seq(H, W, 40 + c, n=6) for c in range(NCAM)]
    frames = lambda k: [s.frames[k] for s in seqs]  # noqa: E731
    dev = [torch.from_numpy(f).cuda() for f in frames(3)]
    torch.cuda.synchronize()
    g = api.KltGroup(cfg, NCAM, W, H, L, FW, FH)
    rng = np.random.default_rng(5)
    pts = lambda n: np.column_stack([rng.uniform(0.05, 0.95, (n, 2)), np.zeros(n)])  # noqa: E731
    got = {"first": _count(api, lambda: g.first(frames(0)))}
    got["next"] = _count(api, lambda: g.next(frames(1)))
    got["submit"] = _count(api, lambda: g.submit(frames(2)))
    g.collect()
    got["next_dev"] = _count(api, lambda: g.next_dev([t.data_ptr() for t in dev], W))
    g.fetch()
    got["feed"] = _count(api, lambda: g.feed([pts(20), None, pts(30)]))
    got["advance_subset"] = _count(api, lambda: g.advance([0, 2]))
    got["advance_all"] = _count(api, lambda: g.advance())
    got["first_present"] = _count(api, lambda: g.first(frames(4), present=[pts(40), pts(0), pts(90)]))
    g.close()
    # first: 2 front + 4 pyramid + prefilter + verify + select (advance folded into select);
    # next / submit: 2 front + prefilter + 4 pyramid + fused tracker + verify + select;
    # next_dev: as next with a one-launch front pass (device images are not split by camera);
    # first with present lists: first + suppress; feed: kill + place
    assert got == {"first": 9, "next": 10, "submit": 10, "next_dev": 9, "feed": 2, "advance_subset": 1,
                   "advance_all": 1, "first_present": 10}
