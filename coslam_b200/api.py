"""Thin ctypes binding of coslam_b200/libcoslam_b200.so (the C-ABI of include/coslam_b200.h).

This is plumbing for tests/ and bench.py -- the product is the shared library.  There is NO CPU
fallback: if the library is missing, importing this module raises; if no CUDA device is present,
the first call that needs one returns COSL_E_CUDA and raises CoslError."""
import collections
import ctypes as C
import os

import numpy as np

from .ctypes_defs import (COSL_BA_INFOSZ, COSL_KLT_OP_SKIP, FEAT_DTYPE, BaOptions, BaProblem, KltConfig,
                          KltFeature, PoseOpt)

_HERE = os.path.dirname(os.path.abspath(__file__))
# COSLAM_B200_LIB selects another build of the same library (kernel tuning experiments)
LIB_PATH = os.environ.get("COSLAM_B200_LIB") or os.path.join(_HERE, "libcoslam_b200.so")


class CoslError(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `make` (or __graft_entry__.build()); "
            "coslam_b200 has no CPU fallback")
    L = C.CDLL(LIB_PATH)
    vp, ci, cf, cd = C.c_void_p, C.c_int, C.c_float, C.c_double
    pint = C.POINTER(C.c_int)
    L.cosl_last_error.restype = C.c_char_p
    L.cosl_version.restype = C.c_char_p
    L.cosl_kernel_launch_count.restype = C.c_uint64
    L.cosl_klt_config_default.argtypes = [C.POINTER(KltConfig)]
    L.cosl_klt_create.argtypes = [C.POINTER(KltConfig)] + [ci] * 8 + [C.POINTER(vp)]
    L.cosl_klt_group_create.argtypes = [C.POINTER(KltConfig)] + [ci] * 9 + [C.POINTER(vp)]
    L.cosl_klt_group_create_sizes.argtypes = [C.POINTER(KltConfig), ci, vp, vp] + [ci] * 6 + [C.POINTER(vp)]
    L.cosl_klt_destroy.argtypes = [vp]
    L.cosl_klt_detect.argtypes = [vp, vp, C.c_size_t, ci, vp, vp, pint]
    L.cosl_klt_redetect.argtypes = [vp, vp, C.c_size_t, vp, pint]
    L.cosl_klt_track.argtypes = [vp, vp, C.c_size_t, vp, pint]
    L.cosl_klt_feed.argtypes = [vp, ci, vp, vp, pint]
    L.cosl_klt_advance.argtypes = [vp]
    for f in (L.cosl_klt_set_margin, L.cosl_klt_set_conv, L.cosl_klt_set_ssd, L.cosl_klt_set_covariance):
        f.argtypes = [vp, cf]
    L.cosl_klt_group_download_covariance.argtypes = [vp, vp]
    L.cosl_klt_group_next.argtypes = [vp, vp, C.c_size_t, vp, vp]
    L.cosl_klt_group_first.argtypes = [vp, vp, C.c_size_t, vp, vp]
    L.cosl_klt_group_first_present.argtypes = [vp, vp, C.c_size_t, vp, vp, vp, vp]
    L.cosl_klt_group_feed.argtypes = [vp, vp, vp, vp, vp]
    L.cosl_klt_group_advance_cams.argtypes = [vp, vp]
    L.cosl_klt_group_next_dev.argtypes = [vp, vp, C.c_size_t]
    L.cosl_klt_group_step.argtypes = [vp, vp, vp, C.c_size_t, vp, vp]
    L.cosl_klt_group_step_dev.argtypes = [vp, vp, vp, C.c_size_t]
    L.cosl_klt_group_fetch.argtypes = [vp, vp, vp]
    L.cosl_klt_group_sync.argtypes = [vp]
    L.cosl_klt_group_submit.argtypes = [vp, vp, C.c_size_t]
    L.cosl_klt_group_submit_step.argtypes = [vp, vp, vp, C.c_size_t]
    L.cosl_klt_group_collect.argtypes = [vp, vp, vp]
    L.cosl_klt_group_prefetch.argtypes = [vp, vp, vp, C.c_size_t]
    L.cosl_klt_group_run_prefetched.argtypes = [vp, vp, vp]
    L.cosl_klt_group_submit_prefetched.argtypes = [vp]
    L.cosl_klt_group_discard_prefetch.argtypes = [vp]
    L.cosl_klt_stream.argtypes = [vp]
    L.cosl_klt_stream.restype = vp
    L.cosl_klt_debug_pyramid.argtypes = [vp, ci, ci, ci, vp, pint, pint]
    L.cosl_klt_debug_cornerness.argtypes = [vp, ci, vp]
    L.cosl_klt_debug_num_candidates.argtypes = [vp, ci]
    L.cosl_klt_algorithmic_bytes.argtypes = [vp]
    L.cosl_klt_algorithmic_bytes.restype = cd
    L.cosl_klt_profile_enable.argtypes = [vp, ci]
    L.cosl_klt_profile_get.argtypes = [vp, ci, C.POINTER(cd), pint]
    L.cosl_klt_profile_get.restype = C.c_char_p
    L.cosl_pose_opt_default.argtypes = [C.POINTER(PoseOpt)]
    L.cosl_pose_intracam.argtypes = [vp, vp, vp, ci, vp, vp, vp, cd, vp, vp, C.POINTER(PoseOpt),
                                     pint]
    L.cosl_pose_intracam_batch.argtypes = [ci, vp, vp, vp, vp, vp, vp, vp, cd, vp, vp, vp, vp, ci]
    L.cosl_pose_solver_create.argtypes = [ci, ci, ci, C.POINTER(vp)]
    L.cosl_pose_solver_destroy.argtypes = [vp]
    L.cosl_pose_solver_submit.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp, vp, cd, vp]
    L.cosl_pose_solver_query.argtypes = [vp, pint]
    L.cosl_pose_solver_collect.argtypes = [vp, vp, vp, vp, vp, vp]
    L.cosl_pose_solver_stream.argtypes = [vp]
    L.cosl_pose_solver_stream.restype = vp
    L.cosl_pose_solver_set_covariance.argtypes = [vp, cd]
    L.cosl_pose_solver_download_covariance.argtypes = [vp, vp, vp, vp]
    L.cosl_ba_options_default.argtypes = [C.POINTER(BaOptions)]
    L.cosl_ba_solve.argtypes = [C.POINTER(BaProblem), C.POINTER(BaOptions), vp]
    L.cosl_ba_solve_multi.argtypes = [C.POINTER(BaProblem), C.POINTER(BaOptions), ci, vp, vp]
    L.cosl_sba_motstr_levmar_x.argtypes = [ci] * 4 + [vp, vp, ci, ci, vp, ci, vp, ci, ci, vp, vp, ci]
    L.cosl_sba_motstr_levmar_x_cov.argtypes = [ci] * 4 + [vp, vp, ci, ci, vp, vp, ci, vp, ci, ci, vp, vp, ci]
    L.cosl_nccl_unique_id.argtypes = [vp]
    L.cosl_ba_comm_create.argtypes = [vp, ci, ci, ci, C.POINTER(vp)]
    L.cosl_ba_comm_destroy.argtypes = [vp]
    L.cosl_ba_solver_create.argtypes = [C.POINTER(BaProblem), C.POINTER(BaOptions), vp,
                                        C.POINTER(vp)]
    L.cosl_ba_solver_reset.argtypes = [vp, C.POINTER(BaProblem)]
    L.cosl_ba_solver_load.argtypes = [vp, C.POINTER(BaProblem)]
    L.cosl_ba_solver_run.argtypes = [vp, vp]
    L.cosl_ba_solver_run_fixed.argtypes = [vp, ci, vp]
    L.cosl_ba_solver_submit.argtypes = [vp]
    L.cosl_ba_solver_query.argtypes = [vp, pint]
    L.cosl_ba_solver_collect.argtypes = [vp, vp]
    L.cosl_ba_solver_stop.argtypes = [vp]
    L.cosl_ba_solver_progress.argtypes = [vp, C.POINTER(cd)]
    L.cosl_ba_solver_set_covariance.argtypes = [vp, cd]
    L.cosl_ba_solver_download_covariance.argtypes = [vp, vp, vp, C.POINTER(cd)]
    L.cosl_ba_solver_set_obs_cov.argtypes = [vp, vp]
    L.cosl_ba_solver_download.argtypes = [vp, C.POINTER(BaProblem)]
    L.cosl_ba_solver_destroy.argtypes = [vp]
    L.cosl_ba_solver_stream.argtypes = [vp]
    L.cosl_ba_solver_stream.restype = vp
    L.cosl_ba_solver_timer.argtypes = [vp, ci, C.POINTER(cd), pint]
    L.cosl_ba_solver_timer.restype = C.c_char_p
    L.cosl_ba_solver_profile_enable.argtypes = [vp, ci]
    L.cosl_ba_solver_stats.argtypes = [vp, C.POINTER(cd)]
    L.cosl_ba_solver_plan_info.argtypes = [vp, pint]
    L.cosl_ba_solver_trace.argtypes = [vp, ci, vp, vp, ci]
    L.cosl_ba_solver_tasks.argtypes = [vp, vp, ci, vp, ci]
    L.cosl_ba_debug_tile_solve.argtypes = [ci, vp, ci, vp, vp, vp, pint, pint]
    L.cosl_ba_debug_tile_selinv.argtypes = [ci, vp, ci, vp, vp, pint, pint]
    L.cosl_posegraph_spread_chains.argtypes = [ci, vp, vp, vp, vp, vp, vp, vp, vp, ci]
    L.cosl_posegraph_solve.argtypes = [ci, vp, vp, vp, ci, vp, vp, vp, vp, vp, ci, vp, vp, vp, ci]
    L.cosl_posegraph_last_host_ms.restype = cd
    L.cosl_posegraph_solver_create.argtypes = [ci, C.POINTER(vp)]
    L.cosl_posegraph_solver_destroy.argtypes = [vp]
    L.cosl_posegraph_solver_submit_chains.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp]
    L.cosl_posegraph_solver_submit.argtypes = [vp, ci, vp, vp, vp, ci, vp, vp, vp, vp, vp, ci]
    L.cosl_posegraph_solver_query.argtypes = [vp, pint]
    L.cosl_posegraph_solver_collect.argtypes = [vp, vp, vp, vp, vp]
    L.cosl_posegraph_solver_stream.argtypes = [vp]
    L.cosl_posegraph_solver_stream.restype = vp
    return L


LIB = _load()


def _ck(rc):
    if rc != 0:
        raise CoslError(f"coslam_b200 error {rc}: {LIB.cosl_last_error().decode()}")


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def kernel_launch_count():
    return int(LIB.cosl_kernel_launch_count())


class KltTracker:
    """One camera.  Mirrors V3D_GPU::KLT_SequenceTracker (tracking/CGKLT/v3d_gpuklt.h:202-262)."""

    def __init__(self, cfg, width, height, n_levels, feat_w, feat_h, pl_w=0, pl_h=0, device=0):
        self.cfg, self.W, self.H, self.nl = cfg, width, height, n_levels
        self.fw, self.fh, self.F = feat_w, feat_h, feat_w * feat_h
        h = C.c_void_p()
        _ck(LIB.cosl_klt_create(C.byref(cfg), width, height, n_levels, feat_w, feat_h, pl_w, pl_h,
                                device, C.byref(h)))
        self.h = h
        self.feats = (KltFeature * self.F)()

    def close(self):
        if getattr(self, "h", None):
            LIB.cosl_klt_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _out(self):
        return np.frombuffer(bytes(self.feats), dtype=FEAT_DTYPE).copy()

    def detect(self, img, present=None):
        img = np.ascontiguousarray(img, np.uint8)
        n = C.c_int(0)
        npres = 0 if present is None else len(present)
        pres = None if present is None else np.ascontiguousarray(present, np.float32)
        _ck(LIB.cosl_klt_detect(self.h, _ptr(img), img.strides[0], npres, _ptr(pres),
                                C.byref(self.feats), C.byref(n)))
        return self._out(), n.value

    def redetect(self, img):
        img = np.ascontiguousarray(img, np.uint8)
        n = C.c_int(0)
        _ck(LIB.cosl_klt_redetect(self.h, _ptr(img), img.strides[0], C.byref(self.feats),
                                  C.byref(n)))
        return self._out(), n.value

    def track(self, img):
        img = np.ascontiguousarray(img, np.uint8)
        n = C.c_int(0)
        _ck(LIB.cosl_klt_track(self.h, _ptr(img), img.strides[0], C.byref(self.feats), C.byref(n)))
        return self._out(), n.value

    def feed(self, pts3):
        pts3 = np.ascontiguousarray(pts3, np.float32).reshape(-1, 3)
        ids = np.full(len(pts3), -1, np.int32)
        n = C.c_int(0)
        _ck(LIB.cosl_klt_feed(self.h, len(pts3), _ptr(pts3), _ptr(ids), C.byref(n)))
        return ids, n.value

    def advance(self):
        _ck(LIB.cosl_klt_advance(self.h))

    def next(self, img):
        """GPUKLT::next (tracking/GPUKLT.cpp:144-161): redetect + advanceFrame."""
        out = self.redetect(img)
        self.advance()
        return out

    def first(self, img):
        """GPUKLT::first (tracking/GPUKLT.cpp:133-142): detect + advanceFrame."""
        out = self.detect(img)
        self.advance()
        return out

    def set_margin(self, m):
        _ck(LIB.cosl_klt_set_margin(self.h, m))

    def set_conv(self, t):
        _ck(LIB.cosl_klt_set_conv(self.h, t))

    def set_ssd(self, t):
        _ck(LIB.cosl_klt_set_ssd(self.h, t))

    def pyramid(self, which, level, cam=0):
        w, h = self.W >> level, self.H >> level
        out = np.empty((h, w, 3), np.float32)
        _ck(LIB.cosl_klt_debug_pyramid(self.h, cam, which, level, _ptr(out), None, None))
        return out

    def cornerness(self, cam=0):
        out = np.empty((self.H, self.W), np.float32)
        _ck(LIB.cosl_klt_debug_cornerness(self.h, cam, _ptr(out)))
        return out

    def num_candidates(self, cam=0):
        return LIB.cosl_klt_debug_num_candidates(self.h, cam)


class KltGroup:
    """C cameras, one launch per kernel for the whole group (batched GPUKLT::first / GPUKLT::next).

    width, height: one size for every camera (cosl_klt_group_create), or one per camera
    (sequences of n_cams entries: cosl_klt_group_create_sizes).  self.sizes lists each camera's
    (width, height); self.W, self.H are the largest width and height."""

    def __init__(self, cfg, n_cams, width, height, n_levels, feat_w, feat_h, device=0):
        self.mixed = not (np.isscalar(width) and np.isscalar(height))
        ws = [int(v) for v in np.broadcast_to(width, (n_cams,))]
        hs = [int(v) for v in np.broadcast_to(height, (n_cams,))]
        self.cfg, self.C, self.nl = cfg, n_cams, n_levels
        self.sizes = list(zip(ws, hs))
        self.W, self.H = max(ws), max(hs)
        self.fw, self.fh, self.F = feat_w, feat_h, feat_w * feat_h
        h = C.c_void_p()
        if self.mixed:
            wa, ha = np.asarray(ws, np.int32), np.asarray(hs, np.int32)
            _ck(LIB.cosl_klt_group_create_sizes(C.byref(cfg), n_cams, _ptr(wa), _ptr(ha), n_levels,
                                                feat_w, feat_h, 0, 0, device, C.byref(h)))
        else:
            _ck(LIB.cosl_klt_group_create(C.byref(cfg), n_cams, width, height, n_levels, feat_w,
                                          feat_h, 0, 0, device, C.byref(h)))
        self.h = h
        self.feats = np.zeros((n_cams, self.F), FEAT_DTYPE)
        self.counts = np.zeros(n_cams, np.int32)
        self._dest = (C.c_void_p * n_cams)(*[self.feats[c].ctypes.data for c in range(n_cams)])
        # ops of each submitted frame not yet collected, oldest first (None: a submit)
        self._in_flight = collections.deque()
        # ops of the pending prefetch (None: prefetched without ops, as next / submit)
        self._prefetched = None

    def close(self):
        if getattr(self, "h", None):
            LIB.cosl_klt_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _imgs(self, imgs):
        """(pointer array, pitch).  Camera c's frame is (H_c, W_c) uint8.  One row pitch shared by
        every frame is passed as is; on a group made with per-camera sizes, frames whose rows are
        each their own width apart (C-contiguous) pass pitch 0."""
        assert len(imgs) == self.C
        for im, (w, h) in zip(imgs, self.sizes):
            assert im.dtype == np.uint8 and im.shape == (h, w) and im.strides[1] == 1
        pitches = {im.strides[0] for im in imgs}
        if len(pitches) == 1:
            pitch = pitches.pop()
        else:
            assert self.mixed and all(im.strides[0] == w for im, (w, _) in zip(imgs, self.sizes)), \
                "frames of different pitches: give each camera's frame rows of its own width"
            pitch = 0
        return (C.c_void_p * self.C)(*[im.ctypes.data for im in imgs]), pitch

    def _per_cam(self, lists):
        """Per-camera (n, 3) float32 point lists (None: camera not addressed) -> (counts with -1
        for None, the arrays, a pointer array)."""
        assert len(lists) == self.C
        arrs = [None if p is None else np.ascontiguousarray(p, np.float32).reshape(-1, 3) for p in lists]
        n = np.array([-1 if a is None else len(a) for a in arrs], np.int32)
        ptrs = (C.c_void_p * self.C)(*[None if a is None or not len(a) else a.ctypes.data for a in arrs])
        return n, arrs, ptrs

    def first(self, imgs, present=None):
        """Batched GPUKLT::first.  present: per-camera (n, 3) point lists (None or empty: no present
        points for that camera), as in KltTracker.detect."""
        arr, pitch = self._imgs(imgs)
        if present is None:
            _ck(LIB.cosl_klt_group_first(self.h, arr, pitch, self._dest, _ptr(self.counts)))
        else:
            n, _arrs, ptrs = self._per_cam(present)
            n = np.maximum(n, 0)
            _ck(LIB.cosl_klt_group_first_present(self.h, arr, pitch, _ptr(n), ptrs, self._dest,
                                                 _ptr(self.counts)))
        return self.feats, self.counts

    def feed(self, pts):
        """cosl_klt_group_feed: pts[c] = (n, 3) points for camera c, or None to leave it alone.
        Returns (trackIds per camera, None where not addressed; nFed per camera, 0 where not
        addressed).  No advance: call advance(cams) after it, as GPUKLT::feedExternFeatPoints does."""
        n, arrs, ptrs = self._per_cam(pts)
        ids = [None if a is None else np.full(len(a), -1, np.int32) for a in arrs]
        idp = (C.c_void_p * self.C)(*[None if i is None or not len(i) else i.ctypes.data for i in ids])
        fed = np.zeros(self.C, np.int32)
        _ck(LIB.cosl_klt_group_feed(self.h, _ptr(n), ptrs, idp, _ptr(fed)))
        return ids, fed

    def advance(self, cams=None):
        """advanceFrame for the cameras in `cams` (indices; None: every camera, cosl_klt_advance)."""
        if cams is None:
            _ck(LIB.cosl_klt_advance(self.h))
            return
        mask = np.zeros(self.C, np.uint8)
        mask[list(cams)] = 1
        _ck(LIB.cosl_klt_group_advance_cams(self.h, _ptr(mask)))

    def next(self, imgs):
        arr, pitch = self._imgs(imgs)
        _ck(LIB.cosl_klt_group_next(self.h, arr, pitch, self._dest, _ptr(self.counts)))
        return self.feats, self.counts

    def host_ptrs(self, imgs):
        """Pre-built argument for next_raw(): the per-camera pointer array of a set of host frames
        (the caller keeps the frames alive)."""
        return self._imgs(imgs)

    def next_raw(self, ptrs_pitch):
        """cosl_klt_group_next with a pointer array from host_ptrs(): no per-call marshalling."""
        _ck(LIB.cosl_klt_group_next(self.h, ptrs_pitch[0], ptrs_pitch[1], self._dest,
                                    _ptr(self.counts)))
        return self.feats, self.counts

    def next_dev(self, dev_ptrs, pitch):
        arr = (C.c_void_p * self.C)(*dev_ptrs)
        _ck(LIB.cosl_klt_group_next_dev(self.h, arr, pitch))

    def _ops(self, ops):
        ops = np.ascontiguousarray(ops, np.uint8)
        assert ops.shape == (self.C,)
        return ops

    def _step_result(self, ops):
        """(tables, counts) of the addressed cameras, None for a skipped one"""
        tables = [None if o == COSL_KLT_OP_SKIP else self.feats[c] for c, o in enumerate(ops)]
        counts = [None if o == COSL_KLT_OP_SKIP else int(self.counts[c]) for c, o in enumerate(ops)]
        return tables, counts

    def _step_args(self, ops, imgs):
        """(ops, pointer array, pitch) of a step: imgs[c] is camera c's frame, None if skipped"""
        ops = self._ops(ops)
        addr = [im for im, o in zip(imgs, ops) if o != COSL_KLT_OP_SKIP]
        ptrs = (C.c_void_p * self.C)()
        pitch = self.W  # read by no camera when every camera is skipped
        if addr:
            for im, (w, h), o in zip(imgs, self.sizes, ops):
                if o != COSL_KLT_OP_SKIP:
                    assert im.dtype == np.uint8 and im.shape == (h, w) and im.strides[1] == 1
            # one pitch must hold the widest camera, which need not be addressed: frames whose rows
            # are each their own camera's width apart pass 0 instead (per-camera sizes only)
            pitches = {im.strides[0] for im in addr}
            if len(pitches) == 1 and min(pitches) >= self.W:
                pitch = pitches.pop()
            else:
                assert self.mixed and all(im.strides[0] == w for im, (w, _), o in zip(imgs, self.sizes, ops)
                                          if o != COSL_KLT_OP_SKIP), \
                    "give every frame one row pitch >= the widest camera, or rows of its camera's own width"
                pitch = 0
            for c, (im, o) in enumerate(zip(imgs, ops)):
                ptrs[c] = None if o == COSL_KLT_OP_SKIP else im.ctypes.data
        return ops, ptrs, pitch

    def step(self, ops, imgs):
        """cosl_klt_group_step: ops[c] in COSL_KLT_OP_* for camera c; imgs[c] its frame, or None
        for a skipped camera.  Returns (tables, counts), None for a skipped camera."""
        ops, ptrs, pitch = self._step_args(ops, imgs)
        _ck(LIB.cosl_klt_group_step(self.h, _ptr(ops), ptrs, pitch, self._dest, _ptr(self.counts)))
        return self._step_result(ops)

    def step_dev(self, ops, dev_ptrs, pitch):
        """cosl_klt_group_step_dev: device frames (None or 0 for a skipped camera); fetch() hands
        back the result."""
        ops = self._ops(ops)
        arr = (C.c_void_p * self.C)(*[p or None for p in dev_ptrs])
        _ck(LIB.cosl_klt_group_step_dev(self.h, _ptr(ops), arr, pitch))

    def fetch(self):
        _ck(LIB.cosl_klt_group_fetch(self.h, self._dest, _ptr(self.counts)))
        return self.feats, self.counts

    def sync(self):
        _ck(LIB.cosl_klt_group_sync(self.h))

    def submit_raw(self, ptrs_pitch):
        """cosl_klt_group_submit: enqueue one frame (pointer array from host_ptrs()) and return."""
        _ck(LIB.cosl_klt_group_submit(self.h, ptrs_pitch[0], ptrs_pitch[1]))
        self._in_flight.append(None)

    def submit(self, imgs):
        self.submit_raw(self._imgs(imgs))

    def submit_step(self, ops, imgs):
        """cosl_klt_group_submit_step: enqueue the step of step(ops, imgs) and return; collect()
        hands back its tables.  The addressed frames must stay untouched until then."""
        ops, ptrs, pitch = self._step_args(ops, imgs)
        _ck(LIB.cosl_klt_group_submit_step(self.h, _ptr(ops), ptrs, pitch))
        self._in_flight.append(ops)

    def collect(self):
        """cosl_klt_group_collect: wait for the oldest submitted frame and return its tables: (feats,
        counts) for a submit, (tables, counts) with None for a skipped camera for a submit_step."""
        _ck(LIB.cosl_klt_group_collect(self.h, self._dest, _ptr(self.counts)))
        ops = self._in_flight.popleft()
        if ops is None:
            return self.feats, self.counts
        return self._step_result(ops)

    def prefetch(self, imgs, ops=None):
        """cosl_klt_group_prefetch: enqueue the image half (upload, pyramid, cornerness map) of the
        frame next(imgs) (ops None) or step(ops, imgs) would run, and return.  Feeds and advances may
        follow; run_prefetched() or submit_prefetched() then runs the rest on the state they leave.
        The frames must stay untouched until then."""
        if ops is None:
            ptrs, pitch = self._imgs(imgs)
            _ck(LIB.cosl_klt_group_prefetch(self.h, None, ptrs, pitch))
        else:
            ops, ptrs, pitch = self._step_args(ops, imgs)
            _ck(LIB.cosl_klt_group_prefetch(self.h, _ptr(ops), ptrs, pitch))
        self._prefetched = ops

    def run_prefetched(self):
        """cosl_klt_group_run_prefetched: what next() (prefetched without ops) or step() returns."""
        _ck(LIB.cosl_klt_group_run_prefetched(self.h, self._dest, _ptr(self.counts)))
        ops, self._prefetched = self._prefetched, None
        if ops is None:
            return self.feats, self.counts
        return self._step_result(ops)

    def submit_prefetched(self):
        """cosl_klt_group_submit_prefetched: enqueue the rest of the prefetched frame as a submitted
        frame; collect() hands back its tables."""
        _ck(LIB.cosl_klt_group_submit_prefetched(self.h))
        self._in_flight.append(self._prefetched)
        self._prefetched = None

    def discard_prefetch(self):
        _ck(LIB.cosl_klt_group_discard_prefetch(self.h))
        self._prefetched = None

    def stream(self):
        return LIB.cosl_klt_stream(self.h)

    def algorithmic_bytes(self):
        return float(LIB.cosl_klt_algorithmic_bytes(self.h))

    def profile_enable(self, on=True):
        _ck(LIB.cosl_klt_profile_enable(self.h, 1 if on else 0))

    def profile(self):
        out, i = {}, 0
        while True:
            ms, calls = C.c_double(0), C.c_int(0)
            name = LIB.cosl_klt_profile_get(self.h, i, C.byref(ms), C.byref(calls))
            if not name:
                break
            out[name.decode()] = (ms.value, calls.value)
            i += 1
        return out

    def set_covariance(self, noise_var=0.0):
        """cosl_klt_set_covariance: arm the position covariance of every tracked slot for the frames
        enqueued from now on (noise_var > 0: that residual variance; 0: estimated per slot) or disarm
        it (noise_var < 0)."""
        _ck(LIB.cosl_klt_set_covariance(self.h, noise_var))

    def download_covariance(self):
        """cosl_klt_group_download_covariance: (C, F, 3) float32 (xx, xy, yy) in level-0 pixels^2 of
        the last frame handed out; NaN where no slot was tracked."""
        out = np.empty((self.C, self.F, 3), np.float32)
        ptrs = (C.c_void_p * self.C)(*[out[c].ctypes.data for c in range(self.C)])
        _ck(LIB.cosl_klt_group_download_covariance(self.h, ptrs))
        return out

    def pyramid(self, cam, which, level):
        w, h = self.sizes[cam][0] >> level, self.sizes[cam][1] >> level
        out = np.empty((h, w, 3), np.float32)
        _ck(LIB.cosl_klt_debug_pyramid(self.h, cam, which, level, _ptr(out), None, None))
        return out

    def cornerness(self, cam):
        w, h = self.sizes[cam]
        out = np.empty((h, w), np.float32)
        _ck(LIB.cosl_klt_debug_cornerness(self.h, cam, _ptr(out)))
        return out


def pose_intracam(K, R0, t0, Ms, ms, tau, prev_errs=None, opt=None):
    """intraCamEstimate (slam/SL_IntraCamPose.cpp:626-709) on the GPU."""
    K = np.ascontiguousarray(K, np.float64).ravel()
    R0 = np.ascontiguousarray(R0, np.float64).ravel()
    t0 = np.ascontiguousarray(t0, np.float64).ravel()
    Ms = np.ascontiguousarray(Ms, np.float64).reshape(-1, 3)
    ms = np.ascontiguousarray(ms, np.float64).reshape(-1, 2)
    pe = None if prev_errs is None else np.ascontiguousarray(prev_errs, np.float64)
    opt = opt if opt is not None else PoseOpt.defaults()
    R, t, ok = np.empty(9), np.empty(3), C.c_int(0)
    _ck(LIB.cosl_pose_intracam(_ptr(K), _ptr(R0), _ptr(t0), len(Ms), _ptr(pe), _ptr(Ms), _ptr(ms),
                               float(tau), _ptr(R), _ptr(t), C.byref(opt), C.byref(ok)))
    return bool(ok.value), R.reshape(3, 3), t, opt


def _pose_batch_args(Ks, R0s, t0s, Ms_list, ms_list, tau, prev_list, opts):
    """C-ABI arguments of a batched pose solve up to tau, then opts (C PoseOpts; defaults when None).
    The arrays behind the pointers live in the returned tuple."""
    Cn = len(Ms_list)
    Ks = np.ascontiguousarray(Ks, np.float64).reshape(Cn, 9)
    R0s = np.ascontiguousarray(R0s, np.float64).reshape(Cn, 9)
    t0s = np.ascontiguousarray(t0s, np.float64).reshape(Cn, 3)
    Ms_list = [np.ascontiguousarray(a, np.float64).reshape(-1, 3) for a in Ms_list]
    ms_list = [np.ascontiguousarray(a, np.float64).reshape(-1, 2) for a in ms_list]
    npts = np.array([len(a) for a in Ms_list], np.int32)
    Mp = (C.c_void_p * Cn)(*[a.ctypes.data for a in Ms_list])
    mp = (C.c_void_p * Cn)(*[a.ctypes.data for a in ms_list])
    pp = None
    if prev_list is not None:
        prev_list = [None if a is None else np.ascontiguousarray(a, np.float64) for a in prev_list]
        pp = (C.c_void_p * Cn)(*[None if a is None else a.ctypes.data for a in prev_list])
    opts = opts if opts is not None else (PoseOpt * Cn)(*[PoseOpt.defaults() for _ in range(Cn)])
    keep = (Ks, R0s, t0s, Ms_list, ms_list, prev_list)
    return (Cn, _ptr(Ks), _ptr(R0s), _ptr(t0s), _ptr(npts), Mp, mp, pp, float(tau)), opts, keep


def pose_intracam_batch(Ks, R0s, t0s, Ms_list, ms_list, tau, prev_list=None, opts=None, device=0):
    args, opts, _keep = _pose_batch_args(Ks, R0s, t0s, Ms_list, ms_list, tau, prev_list, opts)
    Cn = args[0]
    R, t, ok = np.empty((Cn, 9)), np.empty((Cn, 3)), np.zeros(Cn, np.int32)
    _ck(LIB.cosl_pose_intracam_batch(*args, _ptr(R), _ptr(t), opts, _ptr(ok), device))
    return ok.astype(bool), R.reshape(Cn, 3, 3), t, opts


class _SolverHandle:
    """A solver handle of the C-ABI with one request in flight at a time: close, done and stream call
    <_prefix>_destroy, _query and _stream on self.h."""

    _prefix = None

    def close(self):
        """destroy: waits for a request in flight."""
        if getattr(self, "h", None):
            getattr(LIB, self._prefix + "_destroy")(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def done(self):
        """query: True once the submitted request has finished (never waits)."""
        d = C.c_int(0)
        _ck(getattr(LIB, self._prefix + "_query")(self.h, C.byref(d)))
        return bool(d.value)

    def stream(self):
        return getattr(LIB, self._prefix + "_stream")(self.h)


class PoseSolver(_SolverHandle):
    """cosl_pose_solver: pose_intracam_batch without blocking, on a stream and buffers of its own for at
    most max_cams cameras and max_pts points (all cameras together) per submit."""

    _prefix = "cosl_pose_solver"

    def __init__(self, device, max_cams, max_pts):
        h = C.c_void_p()
        _ck(LIB.cosl_pose_solver_create(int(device), int(max_cams), int(max_pts), C.byref(h)))
        self.h, self.device, self.max_cams, self.max_pts = h, device, max_cams, max_pts
        self._opts = None
        self._npts = []  # points per camera of the last accepted submit: the shapes download_covariance returns

    def submit(self, Ks, R0s, t0s, Ms_list, ms_list, tau, prev_list=None, opts=None):
        """cosl_pose_solver_submit: enqueue pose_intracam_batch's solve and return at once; the input arrays
        may be reused when it returns.  opts (C PoseOpts, defaults when None) is what collect() fills."""
        args, opts, keep = _pose_batch_args(Ks, R0s, t0s, Ms_list, ms_list, tau, prev_list, opts)
        _ck(LIB.cosl_pose_solver_submit(self.h, *args, opts))
        self._opts = opts
        self._npts = [len(a) for a in keep[3]]

    def collect(self):
        """cosl_pose_solver_collect: wait for the submitted solve.  Returns (ok, R, t, opts) as
        pose_intracam_batch does, then the device time of its copies and kernel in ms."""
        opts = self._opts if self._opts is not None else (PoseOpt * 1)()
        Cn = len(opts)
        R, t, ok, ms = np.empty((Cn, 9)), np.empty((Cn, 3)), np.zeros(Cn, np.int32), C.c_double(0)
        _ck(LIB.cosl_pose_solver_collect(self.h, _ptr(R), _ptr(t), opts, _ptr(ok), C.byref(ms)))
        self._opts = None
        return ok.astype(bool), R.reshape(Cn, 3, 3), t, opts, ms.value

    def set_covariance(self, pixel_var):
        """cosl_pose_solver_set_covariance: pixel_var > 0 makes every later submit() end with the covariance
        stage; 0 turns it off."""
        _ck(LIB.cosl_pose_solver_set_covariance(self.h, float(pixel_var)))

    def download_covariance(self):
        """cosl_pose_solver_download_covariance after collect() of an armed solve: (cov [C, 6, 6] for (w, dt),
        err: per camera the residuals of its points in px, stats [C, 4] = sigma2_hat, dof, smallest relative
        pivot, valid)."""
        npts = self._npts
        cov, stats = np.empty((len(npts), 6, 6)), np.empty((len(npts), 4))
        err = np.empty(sum(npts))
        _ck(LIB.cosl_pose_solver_download_covariance(self.h, _ptr(cov), _ptr(err), _ptr(stats)))
        return cov, np.split(err, np.cumsum(npts)[:-1]), stats


def ba_solve(prob, opt):
    """bundleAdjustRobust drop-in: prob (coslam_b200.problem.BAProblem) is updated in place."""
    info = np.zeros(COSL_BA_INFOSZ)
    s = prob.struct()
    _ck(LIB.cosl_ba_solve(C.byref(s), C.byref(opt), _ptr(info)))
    return info


def ba_solve_multi(prob, opt, n_gpus, devices=None):
    """cosl_ba_solve_multi: the same drop-in on n_gpus devices of this process."""
    info = np.zeros(COSL_BA_INFOSZ)
    s = prob.struct()
    dev = None if devices is None else np.ascontiguousarray(devices, np.int32)
    _ck(LIB.cosl_ba_solve_multi(C.byref(s), C.byref(opt), int(n_gpus), _ptr(dev), _ptr(info)))
    return info


def _obs_cov(covx, nobs):
    """covx as the C-ABI's contiguous [nobs][4] float64 array (None stays None)"""
    if covx is None:
        return None
    c = np.ascontiguousarray(covx, np.float64).reshape(-1, 4)
    if len(c) != nobs:
        raise ValueError(f"covx has {len(c)} covariances for {nobs} observations")
    return c


def sba_motstr_levmar_x(p, rot0, vmask, x, itmax, opts, n_con=0, m_con=0, covx=None, verbose=0, device=0):
    """cosl_sba_motstr_levmar_x (cnp = 11, pnp = 3, mnp = 2), or cosl_sba_motstr_levmar_x_cov with covx [nobs, 2, 2]
    (px^2) in x's point-major order.  p [11 m + 3 n] is updated in place; returns (iterations, info [10])."""
    vmask = np.ascontiguousarray(vmask, np.int8)
    n, m = vmask.shape
    assert p.dtype == np.float64 and p.flags.c_contiguous and p.size == 11 * m + 3 * n
    x = np.ascontiguousarray(x, np.float64)
    rot0 = np.ascontiguousarray(rot0, np.float64)
    opts = np.ascontiguousarray(opts, np.float64)
    c = _obs_cov(covx, int(np.count_nonzero(vmask)))
    info = np.zeros(10)
    rc = LIB.cosl_sba_motstr_levmar_x_cov(n, int(n_con), m, int(m_con), _ptr(vmask), _ptr(p), 11, 3, _ptr(x), _ptr(c),
                                          2, _ptr(rot0), int(itmax), int(verbose), _ptr(opts), _ptr(info),
                                          int(device))
    if rc < 0:
        _ck(rc)
    return rc, info


PLAN_INFO_KEYS = ("blocks", "tiles_schur", "tiles", "tasks", "nd_depth", "critical_tasks", "grid",
                  "small_solve")


def ba_debug_tile_solve(S, b, adj, nd_depth=-1):
    """cosl_ba_debug_tile_solve: x = S^-1 b with the BA's reduced-system solve (S dense 6mf x 6mf, lower
    triangle read; adj the mf x mf block pattern).  Returns (x, fail flag, plan info dict)."""
    adj = np.ascontiguousarray(adj, np.uint8)
    mf = adj.shape[0]
    assert adj.shape == (mf, mf)
    S = np.ascontiguousarray(S, np.float64)
    b = np.ascontiguousarray(b, np.float64)
    assert S.shape == (6 * mf, 6 * mf) and b.shape == (6 * mf,)
    x = np.empty(6 * mf)
    fail = C.c_int(0)
    out = (C.c_int * 8)()
    _ck(LIB.cosl_ba_debug_tile_solve(mf, _ptr(adj), int(nd_depth), _ptr(S), _ptr(b), _ptr(x), C.byref(fail),
                                     out))
    return x, fail.value, dict(zip(PLAN_INFO_KEYS, [int(v) for v in out]))


SELINV_INFO_KEYS = ("blocks", "tiles_schur", "tiles", "selinv_tasks", "nd_depth", "steps", "grid", "small_solve")


def ba_debug_tile_selinv(S, adj, nd_depth=-1):
    """cosl_ba_debug_tile_selinv: Z = S^-1 on the tile pattern of the BA's reduced-system factorisation (S dense
    6mf x 6mf, lower triangle read; adj the mf x mf block pattern).  Returns (Z with the pattern's blocks (a, c),
    a >= c, zero elsewhere; fail flag; info dict)."""
    adj = np.ascontiguousarray(adj, np.uint8)
    mf = adj.shape[0]
    assert adj.shape == (mf, mf)
    S = np.ascontiguousarray(S, np.float64)
    assert S.shape == (6 * mf, 6 * mf)
    Z = np.empty((6 * mf, 6 * mf))
    fail = C.c_int(0)
    out = (C.c_int * 8)()
    _ck(LIB.cosl_ba_debug_tile_selinv(mf, _ptr(adj), int(nd_depth), _ptr(S), _ptr(Z), C.byref(fail), out))
    return Z, fail.value, dict(zip(SELINV_INFO_KEYS, [int(v) for v in out]))


def _chain_args(chain_off, fixed, R, t, eR, et):
    """C-ABI arguments of a chain spread from nChains on, and N.  The arrays behind the pointers live in the
    returned tuple."""
    off = np.ascontiguousarray(chain_off, np.int32)
    N = int(off[-1])
    fx = np.ascontiguousarray(fixed, np.uint8)
    R = np.ascontiguousarray(R, np.float64).reshape(N, 3, 3)
    t = np.ascontiguousarray(t, np.float64).reshape(N, 3)
    eR = np.ascontiguousarray(eR, np.float64).reshape(N, 3, 3)
    et = np.ascontiguousarray(et, np.float64).reshape(N, 3)
    assert fx.size == N
    keep = (off, fx, R, t, eR, et)
    return (len(off) - 1, _ptr(off), _ptr(fx), _ptr(R), _ptr(t), _ptr(eR), _ptr(et)), N, keep


def posegraph_spread_chains(chain_off, fixed, R, t, eR, et, device=0):
    """cosl_posegraph_spread_chains: post-BA spreading of the non-key-frame poses of all cameras
    (GlobalPoseGraph::computeNewCameraRotations + ::computeNewCameraTranslations on the chain
    graphs of RobustBundleRTS::constructCameraGraphs).  chain_off[nChains+1]; fixed[N]; R (N,3,3);
    t (N,3); eR (N,3,3), et (N,3): edge k = node k -> k+1.  Returns newR (N,3,3), newt (N,3)."""
    args, N, _keep = _chain_args(chain_off, fixed, R, t, eR, et)
    nR, nt = np.empty((N, 3, 3)), np.empty((N, 3))
    _ck(LIB.cosl_posegraph_spread_chains(*args, _ptr(nR), _ptr(nt), int(device)))
    return nR, nt


def _graph_args(fixed, R, t, id1, id2, eR, et, scale_col, n_scale):
    """C-ABI arguments of a general pose graph from nNodes to nScale, and nNodes.  The arrays behind the
    pointers live in the returned tuple."""
    fx = np.ascontiguousarray(fixed, np.uint8)
    n = fx.size
    R = np.ascontiguousarray(R, np.float64).reshape(n, 3, 3)
    t = np.ascontiguousarray(t, np.float64).reshape(n, 3)
    id1 = np.ascontiguousarray(id1, np.int32)
    id2 = np.ascontiguousarray(id2, np.int32)
    ne = id1.size
    assert id2.size == ne
    eR = np.ascontiguousarray(eR, np.float64).reshape(ne, 3, 3)
    et = np.ascontiguousarray(et, np.float64).reshape(ne, 3)
    sc = None if scale_col is None else np.ascontiguousarray(scale_col, np.int32)
    assert sc is None or sc.size == ne
    keep = (fx, R, t, id1, id2, eR, et, sc)
    return (n, _ptr(fx), _ptr(R), _ptr(t), ne, _ptr(id1), _ptr(id2), _ptr(eR), _ptr(et), _ptr(sc),
            int(n_scale)), n, keep


def posegraph_solve(fixed, R, t, id1, id2, eR, et, scale_col=None, n_scale=0, device=0):
    """cosl_posegraph_solve: GlobalPoseGraph::computeNewCameraRotations + ::computeNewCameraTranslations4
    on an arbitrary edge set (the camera-group merge).  fixed[n]; R (n,3,3); t (n,3); edges id1 -> id2 with
    eR (e,3,3), et (e,3); scale_col[e] = shared scale column of edge e (-1: known scale; None: all known).
    Returns newR (n,3,3), newt (n,3), scale (n_scale,)."""
    args, n, _keep = _graph_args(fixed, R, t, id1, id2, eR, et, scale_col, n_scale)
    nR, nt, s = np.empty((n, 3, 3)), np.empty((n, 3)), np.empty(max(1, int(n_scale)))
    _ck(LIB.cosl_posegraph_solve(*args, _ptr(nR), _ptr(nt), _ptr(s), int(device)))
    return nR, nt, s[:int(n_scale)]


class PoseGraphSolver(_SolverHandle):
    """cosl_posegraph_solver: posegraph_spread_chains and posegraph_solve without blocking, on a stream and
    buffers of its own that grow with the largest request."""

    _prefix = "cosl_posegraph_solver"

    def __init__(self, device):
        h = C.c_void_p()
        _ck(LIB.cosl_posegraph_solver_create(int(device), C.byref(h)))
        self.h, self.device = h, device
        self._shape = None  # (nodes, scale columns or None for a chain spread) of the request in flight

    def submit_chains(self, chain_off, fixed, R, t, eR, et):
        """cosl_posegraph_solver_submit_chains: enqueue posegraph_spread_chains' spread and return at once; the
        input arrays may be reused when it returns."""
        args, N, _keep = _chain_args(chain_off, fixed, R, t, eR, et)
        _ck(LIB.cosl_posegraph_solver_submit_chains(self.h, *args))
        self._shape = (N, None)

    def submit(self, fixed, R, t, id1, id2, eR, et, scale_col=None, n_scale=0):
        """cosl_posegraph_solver_submit: enqueue posegraph_solve's solve and return at once; the input arrays
        may be reused when it returns."""
        args, n, _keep = _graph_args(fixed, R, t, id1, id2, eR, et, scale_col, n_scale)
        _ck(LIB.cosl_posegraph_solver_submit(self.h, *args))
        self._shape = (n, int(n_scale))

    def collect(self):
        """cosl_posegraph_solver_collect: wait for the submitted request.  Returns (newR, newt, scale, device_ms):
        what posegraph_spread_chains (scale None) or posegraph_solve returns, then the device time of the
        copies and kernels in ms.  Raises CoslError as those calls do."""
        n, ns = self._shape if self._shape is not None else (0, 0)
        nR, nt, s = np.empty((n, 3, 3)), np.empty((n, 3)), np.empty(max(1, ns or 0))
        ms = C.c_double(0)
        self._shape = None  # a collect that reports an error consumes the request as well
        _ck(LIB.cosl_posegraph_solver_collect(self.h, _ptr(nR), _ptr(nt), _ptr(s), C.byref(ms)))
        return nR, nt, (None if ns is None else s[:ns]), ms.value


def posegraph_last_host_ms():
    """Host time (ms) of this thread's last posegraph_solve: validation, numbering, planning, lists."""
    return float(LIB.cosl_posegraph_last_host_ms())


def nccl_unique_id():
    buf = np.zeros(128, np.uint8)
    _ck(LIB.cosl_nccl_unique_id(_ptr(buf)))
    return buf


class BaComm:
    def __init__(self, uid, rank, nranks, device):
        uid = np.ascontiguousarray(uid, np.uint8)
        h = C.c_void_p()
        _ck(LIB.cosl_ba_comm_create(_ptr(uid), rank, nranks, device, C.byref(h)))
        self.h, self.rank, self.nranks = h, rank, nranks

    def close(self):
        if getattr(self, "h", None):
            LIB.cosl_ba_comm_destroy(self.h)
            self.h = None


class BaSolver(_SolverHandle):
    """Problem resident on the device (this rank's shard of points when `comm` is given)."""

    _prefix = "cosl_ba_solver"

    def __init__(self, prob, opt, comm=None):
        self.prob, self.opt = prob, opt
        self._s = prob.struct()
        h = C.c_void_p()
        _ck(LIB.cosl_ba_solver_create(C.byref(self._s), C.byref(opt), comm.h if comm else None,
                                      C.byref(h)))
        self.h = h

    def reset(self, prob=None):
        if prob is not None:
            self.prob = prob
            self._s = prob.struct()
        _ck(LIB.cosl_ba_solver_reset(self.h, C.byref(self._s)))

    def load(self, prob):
        """cosl_ba_solver_load: make `prob` (any shape) the solver's problem without waiting for the device;
        download() then writes into `prob`."""
        s = prob.struct()
        _ck(LIB.cosl_ba_solver_load(self.h, C.byref(s)))
        self.prob, self._s = prob, s

    def run(self):
        info = np.zeros(COSL_BA_INFOSZ)
        _ck(LIB.cosl_ba_solver_run(self.h, _ptr(info)))
        return info

    def run_fixed(self, trials):
        info = np.zeros(COSL_BA_INFOSZ)
        _ck(LIB.cosl_ba_solver_run_fixed(self.h, int(trials), _ptr(info)))
        return info

    def submit(self):
        """cosl_ba_solver_submit: enqueue run()'s robust loop on the solver's stream and return at once."""
        _ck(LIB.cosl_ba_solver_submit(self.h))

    def collect(self):
        """cosl_ba_solver_collect: wait for the submitted loop; the info vector of run()."""
        info = np.zeros(COSL_BA_INFOSZ)
        _ck(LIB.cosl_ba_solver_collect(self.h, _ptr(info)))
        return info

    def stop(self):
        """cosl_ba_solver_stop: ask the running or submitted BA to end at its next decision point (stop
        reason 8); returns at once.  May be called from another thread while one is inside run / collect."""
        _ck(LIB.cosl_ba_solver_stop(self.h))

    def progress(self):
        """cosl_ba_solver_progress: where the running or last BA is, without waiting for it."""
        out = (C.c_double * 8)()
        _ck(LIB.cosl_ba_solver_progress(self.h, out))
        return {"running": bool(out[0]), "round": int(out[1]), "iteration": int(out[2]), "trials": int(out[3]),
                "cost": out[4], "init_cost": out[5], "mu": out[6], "stop_requested": bool(out[7])}

    def set_covariance(self, pixel_var):
        """cosl_ba_solver_set_covariance: pixel_var > 0 makes every later run() and submit() end with the
        covariance stage; 0 turns it off."""
        _ck(LIB.cosl_ba_solver_set_covariance(self.h, float(pixel_var)))

    def set_obs_cov(self, covx):
        """cosl_ba_solver_set_obs_cov: covx [nobs, 2, 2] (px^2, in the order of the problem's xy) weights every
        observation by its inverse covariance in every later run / run_fixed / submit; None clears.  load() clears
        it, reset() keeps it."""
        c = _obs_cov(covx, int(self.prob.nobs))
        _ck(LIB.cosl_ba_solver_set_obs_cov(self.h, _ptr(c)))

    def download_covariance(self):
        """cosl_ba_solver_download_covariance: (camCov [m, 6, 6] for (w, t), ptCov [n, 3, 3], info dict) of the
        last armed run or collect."""
        cam = np.empty((self.prob.m, 6, 6))
        pt = np.empty((self.prob.n, 3, 3))
        out = (C.c_double * 8)()
        _ck(LIB.cosl_ba_solver_download_covariance(self.h, _ptr(cam), _ptr(pt), out))
        return cam, pt, {"pixel_var": out[0], "sigma2_hat": out[1], "dof": out[2], "unconstrained": int(out[3]),
                         "device_ms": out[4], "min_pivot": out[5]}

    def download(self, into=None):
        """Current cameras and points into the solver's problem, or into `into` (same shape)."""
        if into is None:
            _ck(LIB.cosl_ba_solver_download(self.h, C.byref(self._s)))
            return self.prob
        s = into.struct()
        _ck(LIB.cosl_ba_solver_download(self.h, C.byref(s)))
        return into

    def stats(self):
        out = (C.c_double * 8)()
        _ck(LIB.cosl_ba_solver_stats(self.h, out))
        return {"ns": int(out[0]), "reduce_doubles": out[1], "factor_flops": out[2],
                "pair_entries": out[3], "pair_items": out[4], "blocks": int(out[5]),
                "tiles": int(out[6]), "tasks": int(out[7])}

    def plan_info(self):
        out = (C.c_int * 8)()
        _ck(LIB.cosl_ba_solver_plan_info(self.h, out))
        return dict(zip(PLAN_INFO_KEYS, [int(v) for v in out]))

    def tasks(self):
        """Task list of the solve plan: (tasks [n,16] int32, wait lists [m,2] int32)."""
        n = self.plan_info()["tasks"]
        t = np.zeros((n, 16), np.int32)
        lst = np.zeros((64 * n + 16, 2), np.int32)
        LIB.cosl_ba_solver_tasks(self.h, _ptr(t), n, _ptr(lst), len(lst))
        return t, lst

    def trace_arm(self):
        return int(LIB.cosl_ba_solver_trace(self.h, 1, None, None, 0))

    def trace_get(self):
        """Timeline of the last persistent solve: (times [n,8] uint64, meta [n,3] int32)."""
        n = self.plan_info()["tasks"]
        tm = np.zeros((n, 8), np.uint64)
        meta = np.zeros((n, 3), np.int32)
        LIB.cosl_ba_solver_trace(self.h, 0, _ptr(tm), _ptr(meta), n)
        return tm, meta

    def profile_enable(self, on=True):
        _ck(LIB.cosl_ba_solver_profile_enable(self.h, 1 if on else 0))

    def timers(self):
        out, i = {}, 0
        while True:
            ms, calls = C.c_double(0), C.c_int(0)
            name = LIB.cosl_ba_solver_timer(self.h, i, C.byref(ms), C.byref(calls))
            if not name:
                break
            out[name.decode()] = (ms.value, calls.value)
            i += 1
        return out
