"""Look-ahead of back-to-back KLT frames over three pyramid buffers (DESIGN.md §3.2): the front pass of
frame n+1 writes the buffer frame n-1's tracker read, and may run while frame n's tracker and frame
n-1's detector still run.  Group b runs each segment of calls back to back with no synchronise, behind
a spin kernel on its stream: every frame of the segment is enqueued before its first tracker may
start, so the front stream runs ahead as far as its fences let it and every fence is put to work.
Group a then runs the same segment with the synchronous calls.  After each segment both must agree
bit for bit: feature tables, counts, both pyramids of every camera and level, and the cornerness map.
The segments cover runs of next_dev, track steps between them (the pyramid ring and the cornerness
ring fall out of step), first with present lists, feed + advance of a subset, mixed steps with SKIP,
submit_step / collect and set_margin, and they take both rings through every position many times
(needs a GPU)."""
import numpy as np
import pytest

from coslam_b200.ctypes_defs import COSL_KLT_OP_FIRST, COSL_KLT_OP_NEXT, COSL_KLT_OP_SKIP, COSL_KLT_OP_TRACK
from helpers import live_cfg, seq

pytestmark = pytest.mark.gpu

S, F, T, N = COSL_KLT_OP_SKIP, COSL_KLT_OP_FIRST, COSL_KLT_OP_TRACK, COSL_KLT_OP_NEXT
MIXED = [(640, 480), (320, 240), (752, 480), (333, 251)]
STALL_CYCLES = 20_000_000  # about 10 ms: far longer than the host takes to enqueue a segment


def _pts(rng, n):
    return np.column_stack([rng.uniform(0.05, 0.95, (n, 2)), np.zeros(n)]).astype(np.float32)


class _Pair:
    def __init__(self, api, cfg, sizes, L, fw, fh, seed, n_frames):
        import torch

        self.torch, self.api, self.L = torch, api, L
        C = len(sizes)
        mixed = len(set(sizes)) > 1
        make = (lambda: api.KltGroup(cfg, C, [w for w, _ in sizes], [h for _, h in sizes], L, fw, fh)) if mixed \
            else (lambda: api.KltGroup(cfg, C, sizes[0][0], sizes[0][1], L, fw, fh))
        self.a, self.b = make(), make()
        self.C = C
        self.pitch = 0 if mixed else sizes[0][0]
        seqs = [seq(h, w, seed + c, n=6) for c, (w, h) in enumerate(sizes)]
        self.host = [[np.ascontiguousarray(s.frame(k)) for s in seqs] for k in range(n_frames)]
        self.dev = [[torch.from_numpy(im).cuda() for im in row] for row in self.host]
        torch.cuda.synchronize()
        self.bstream = torch.cuda.ExternalStream(self.b.stream())
        self.k = 0
        self.corn = list(range(C))  # the cameras whose cornerness map the last detecting frame made
        self.rng = np.random.default_rng(seed)

    def _b(self, act, k, events):
        kind = act[0]
        if kind == "next":
            self.b.next_dev([t.data_ptr() for t in self.dev[k]], self.pitch)
        elif kind == "step":
            ops = act[1]
            self.b.step_dev(ops, [0 if o == S else t.data_ptr() for o, t in zip(ops, self.dev[k])], self.pitch)
        elif kind == "first":
            self.b.first(self.host[k], act[1])
        elif kind == "feed":
            self.fed_b = self.b.feed(act[1])
            self.b.advance(act[2])
        elif kind == "margin":
            assert self.api.LIB.cosl_klt_set_margin(self.b.h, act[1]) == 0
        if kind in ("next", "step"):
            ev = self.torch.cuda.Event()
            ev.record(self.bstream)
            events.append(ev)

    def _a(self, act, k):
        kind = act[0]
        if kind == "next":
            self.a.next(self.host[k])
        elif kind == "step":
            ops = act[1]
            self.a.step(ops, [None if o == S else im for o, im in zip(ops, self.host[k])])
        elif kind == "first":
            self.a.first(self.host[k], act[1])
        elif kind == "feed":
            fed = self.a.feed(act[1])
            self.a.advance(act[2])
            assert np.array_equal(fed[1], self.fed_b[1])
            for x, y in zip(fed[0], self.fed_b[0]):
                assert (x is None and y is None) or np.array_equal(x, y)
        elif kind == "margin":
            assert self.api.LIB.cosl_klt_set_margin(self.a.h, act[1]) == 0
        if kind in ("next", "first") or (kind == "step" and any(o in (F, N) for o in act[1])):
            self.corn = list(range(self.C)) if kind != "step" else [c for c, o in enumerate(act[1]) if o in (F, N)]

    def segment(self, acts, what):
        """b: the whole segment enqueued behind a spin on its stream; then a, synchronously; compare.
        Returns how many of b's frames were still queued when the host had enqueued them all."""
        ks = []
        for act in acts:
            ks.append(self.k if act[0] in ("next", "step", "first") else None)
            if ks[-1] is not None:
                self.k += 1
        events = []
        with self.torch.cuda.stream(self.bstream):
            self.torch.cuda._sleep(STALL_CYCLES)
        for act, k in zip(acts, ks):
            self._b(act, k, events)
        queued = sum(not e.query() for e in events)
        for act, k in zip(acts, ks):
            self._a(act, k)
        self.check(what)
        return queued, len(events)

    def submit_steps(self, sched, what):
        """b submits each step before it collects the one before (two in flight); a runs them
        synchronously afterwards; the collected tables must equal a's"""
        got, pending = [], []
        with self.torch.cuda.stream(self.bstream):
            self.torch.cuda._sleep(STALL_CYCLES)
        ks = list(range(self.k, self.k + len(sched)))
        self.k += len(sched)
        for ops, k in zip(sched, ks):
            self.b.submit_step(ops, [None if o == S else im for o, im in zip(ops, self.host[k])])
            pending.append(ops)
            if len(pending) == 2:
                pending.pop(0)
                t, n = self.b.collect()
                got.append(([None if x is None else x.copy() for x in t], n))
        t, n = self.b.collect()
        got.append(([None if x is None else x.copy() for x in t], n))
        for j, (ops, k) in enumerate(zip(sched, ks)):
            t, n = self.a.step(ops, [None if o == S else im for o, im in zip(ops, self.host[k])])
            gt, gn = got[j]
            assert list(n) == list(gn), (what, j)
            for x, y in zip(t, gt):
                assert (x is None) == (y is None), (what, j)
                if x is not None:
                    assert x.tobytes() == y.tobytes(), (what, j)
            if any(o in (F, N) for o in ops):
                self.corn = [c for c, o in enumerate(ops) if o in (F, N)]
        self.check(what)

    def check(self, what):
        fa, na = self.a.fetch()
        fa, na = fa.copy(), na.copy()
        fb, nb = self.b.fetch()
        assert np.array_equal(na, nb), what
        assert fa.tobytes() == fb.tobytes(), what
        for c in range(self.C):
            for which in (0, 1):
                for level in range(self.L):
                    got = []
                    for g in (self.a, self.b):
                        try:
                            got.append(g.pyramid(c, which, level).tobytes())
                        except self.api.CoslError:
                            got.append(None)
                    assert got[0] == got[1], (what, c, which, level)
        for c in self.corn:
            assert self.a.cornerness(c).tobytes() == self.b.cornerness(c).tobytes(), (what, c)

    def close(self):
        self.a.close()
        self.b.close()


def _script(p):
    C = p.C
    nx = ("next",)
    p.segment([("first", None)], "first")
    queued, n = p.segment([nx] * 8, "next_dev run")
    assert queued == n == 8  # every frame of the run was in flight at once
    # track frames between next frames: the cornerness ring stands still while the pyramid ring turns
    p.segment([("step", ops) for ops in ([T] * C, [N] * C, [T] * C, [T] * C, [N] * C, [N] * C, [T] * C,
                                         [N] * C, [T] * C)], "track / next")
    p.segment([nx, ("margin", 6.0), nx, nx, ("margin", 10.0), nx, nx], "set_margin between frames")
    present = [_pts(p.rng, 30 + 10 * c) if c % 2 == 0 else None for c in range(C)]
    p.segment([nx, nx, nx, ("first", present)], "first with present lists behind queued frames")
    p.segment([nx] * 5, "after first")
    pts = [(_pts(p.rng, 25) if c in (0, C - 1) else None) for c in range(C)]
    p.segment([nx, nx, ("feed", pts, [0, C - 1] if C > 2 else [0])], "feed + advance of a subset")
    p.segment([nx] * 5, "after feed")
    # mixed steps with SKIP (strict subsets both ways), then full steps
    p.segment([("step", ops) for ops in ([N] * (C - 1) + [S], [T, N] + [S] * (C - 2), [S] * C, [N] * C,
                                         [F] + [N] * (C - 1), [N] * C, [T] * C, [N, S] + [T] * (C - 2),
                                         [N] * C, [N] * C)], "mixed steps")
    p.submit_steps([[N] * C, [T] + [N] * (C - 1), [S] + [N] * (C - 1), [T] * C, [N] * C, [N] * C],
                   "submit_step / collect")
    p.segment([nx] * 4, "after submit_step")


@pytest.mark.parametrize("gain", [True, False], ids=["gain", "2x2"])
def test_lookahead_equals_synchronous(api, gain):
    p = _Pair(api, live_cfg(gain=gain, min_corner=1500.0), [(640, 480)] * 3, 6, 32, 32, 900, 70)
    _script(p)
    p.close()


def test_lookahead_mixed_sizes(api):
    p = _Pair(api, live_cfg(gain=True, min_corner=1500.0), MIXED, 5, 32, 32, 930, 70)
    _script(p)
    p.close()


def test_lookahead_slots_not_multiple_of_four(api):
    # F = 15 x 13 = 195 slots per camera
    p = _Pair(api, live_cfg(gain=True, min_corner=800.0), [(328, 250)] * 2, 4, 15, 13, 960, 70)
    _script(p)
    p.close()


def test_lookahead_more_slots_than_resident(api):
    # 4 x 64 x 48 slots: more lane groups than the persistent gain tracker keeps resident at once
    p = _Pair(api, live_cfg(gain=True, min_corner=500.0), [(640, 480)] * 4, 4, 64, 48, 990, 70)
    _script(p)
    p.close()
