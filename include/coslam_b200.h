/*
 * coslam_b200.h -- C-ABI of the H100-native CoSLAM hot paths (KLT tracker, 6-DoF pose solver,
 * multi-camera bundle adjustment).  Plain pointers and sizes only; no C++/torch types.
 *
 * Every entry point returns an int status (COSL_OK == 0, negative == error) and never throws.
 * All reference citations are relative to the upstream tree (danping/CoSLAM, src/...).
 *
 * Seams replaced (SURVEY.md section 8b):
 *   KLT engine  : V3D_GPU::KLT_SequenceTracker            tracking/CGKLT/v3d_gpuklt.h:202-262
 *   Pose solver : intraCamEstimate                        slam/SL_IntraCamPose.h:92-95
 *   BA solver   : bundleAdjustRobust (LibVisualSLAM)      call site app/SL_CoSLAMRobustBA.cpp:174
 *                 sba_motstr_levmar_x  (sba-1.6)           call site app/SL_CoSLAMBA.cpp:360-363
 */
#ifndef COSLAM_B200_H_
#define COSLAM_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------- status codes */
enum {
  COSL_OK = 0,
  COSL_E_INVALID = -1,   /* bad argument                                          */
  COSL_E_CUDA = -2,      /* CUDA runtime error (see cosl_last_error())            */
  COSL_E_NOMEM = -3,     /* host or device allocation failed                      */
  COSL_E_NUMERIC = -4,   /* solver break-down (non-SPD reduced system, NaN, ...)  */
  COSL_E_NCCL = -5,      /* NCCL not loadable / collective failed                 */
  COSL_E_STATE = -6      /* call sequence error (e.g. track before detect)        */
};

/* Thread-local, human readable description of the last error on the calling thread. */
const char* cosl_last_error(void);
/* Library version string "coslam_b200 x.y (sm_90a)". */
const char* cosl_version(void);
/* Number of this library's kernel launches issued so far by the calling process (for bench.py). */
uint64_t cosl_kernel_launch_count(void);

/* ================================================================ KLT tracker */

/* Mirrors V3D_GPU::KLT_SequenceTrackerConfig (v3d_gpuklt.h:180-199), same field order and
 * defaults (use cosl_klt_config_default()).  `trackWithGain` is an int instead of bool.
 * `compat` is an extension: bit 0 (COSL_KLT_COMPAT_ITER5) reproduces the reference's macro-name
 * bug that makes the 2x2 tracker run 5 iterations per level whatever nIterations says
 * (klt_tracker.cg:16-18 vs v3d_gpuklt.cpp:108). */
typedef struct cosl_klt_config {
  int nIterations;            /* 12  */
  int nLevels;                /* 3   (CoSLAM live: 6, app/SL_GlobParam.cpp:30)   */
  int levelSkip;              /* 2   (<=0 means nLevels-1, v3d_gpuklt.h:14)      */
  int windowWidth;            /* 5   (CoSLAM live: 6 -> half width 3)            */
  float trackBorderMargin;    /* 4.0 px */
  float convergenceThreshold; /* 0.1 px  (live 1.0)   */
  float SSD_Threshold;        /* 5000    (live 20000) */
  int trackWithGain;          /* 0       (live 1)     */
  int minDistance;            /* 8  */
  float minCornerness;        /* 1000    (live 3000)  */
  float detectBorderMargin;   /* 4.0 -- dead in the reference: the detector always uses 10 px
                                 (v3d_gpuklt.h:113-114); honoured only via cosl_klt_set_margin */
  int compat;                 /* extension, see above; default COSL_KLT_COMPAT_ITER5 */
} cosl_klt_config;

/* bit 1 (COSL_KLT_PASS_KERNELS, diagnostic): run the gain tracker as one kernel launch per
 * (level, iteration) pass like the reference's draw calls, instead of the single persistent
 * kernel; results are bit-identical, only slower. */
enum { COSL_KLT_COMPAT_ITER5 = 1, COSL_KLT_PASS_KERNELS = 2, COSL_KLT_COMPAT_FEED_STRIDE2 = 4,
       COSL_KLT_COMPAT_HISTOPYR = 8 };
/* bit 2 (COSL_KLT_COMPAT_FEED_STRIDE2, parity runs): feedExternFeaturePoints' proximity test reads
 * the fed points as featPts[2k], featPts[2k+1] although the array holds 3 floats per point
 * (v3d_gpuklt.cpp:826-827 vs :841-842).  The default uses stride 3 in both loops (the evident
 * intent); with this bit the kill test reproduces the reference's stride-2 reads, so the same
 * tracks die and the same trackIds come back as from the reference for the same input.
 * bit 3 (COSL_KLT_COMPAT_HISTOPYR, parity runs): the reference's candidate list instead of "all
 * non-max survivors, strongest first": the corners are read back in HistoPyramid extraction order
 * (Morton order of the pixel, x in the even bits; klt_detector_traverse_histpyr.cg:33-50) and
 * TRUNCATED to pointListWidth*pointListHeight entries before anything is ranked
 * (v3d_gpuklt.cpp:660-661, 755-757), a last odd image row / column is never examined (:519-523),
 * and the list is ordered by cornerness only when it exceeds the free slots (:662-665, 761-768),
 * otherwise slots are filled in extraction order.  With the bit set the SET of new corners equals
 * the reference's; when the list was cut by cornerness their ORDER is strongest-first, whereas the
 * reference's std::nth_element leaves an implementation-defined order. */

/* Mirrors V3D_GPU::KLT_TrackedFeature (v3d_gpuklt.h:166-176): 20 bytes. */
typedef struct cosl_klt_feature {
  int status;   /* 0 tracked from previous frame, 1 newly created, -1 invalid */
  float pos[2]; /* normalised [0,1] image coordinates, texel centres at (i+0.5)/W */
  float gain;
  int fed;      /* >=0: index of the externally fed point */
} cosl_klt_feature;

typedef struct cosl_klt cosl_klt; /* opaque: one tracker group = C cameras */

void cosl_klt_config_default(cosl_klt_config* cfg);

/* KLT_SequenceTracker ctor + allocate(w,h,nLevels,featW,featH[,plW,plH]) (v3d_gpuklt.h:212-215,
 * v3d_gpuklt.cpp:592-624).  plW/plH <= 0 selects the reference default 2*featW x 2*featH
 * (capacity of the candidate list).  `device` is the CUDA ordinal.  One camera. */
int cosl_klt_create(const cosl_klt_config* cfg, int width, int height, int nLevels, int featW,
                    int featH, int plW, int plH, int device, cosl_klt** out);
/* Extension: C cameras of identical geometry that are always advanced together; every kernel is
 * launched once for the whole group (camera = grid.z).  Single-camera calls below address
 * camera 0 of a group.
 * Device memory: a tracker keeps three pyramids per camera, not the reference's two, and three
 * cornerness maps and corner lists, so that the next frame's pyramid is built while the current
 * frame is tracked.  The third set costs about 24 MB per 1280x720 camera (19.7 MB of it the
 * pyramid) and about 55 MB per 1920x1080 camera (44 MB). */
int cosl_klt_group_create(const cosl_klt_config* cfg, int nCams, int width, int height,
                          int nLevels, int featW, int featH, int plW, int plH, int device,
                          cosl_klt** out);
/* Extension: a group whose camera c is widths[c] x heights[c] (each SingleSLAM's tracker takes its
 * size from its own video, app/SL_SingleSLAM.cpp:267-300); the configuration, level count and
 * feature grid are shared.  Every camera must satisfy the per-camera checks of
 * cosl_klt_group_create, the smallest one included ((W >> (nLevels-1)) >= 2).  Every group call
 * works on such a group, and each camera behaves bit for bit like a single-camera tracker of its own
 * size.  Image-taking calls accept pitch == 0 on such a group: camera c's rows are then widths[c]
 * bytes apart; a pitch > 0 must be at least the largest width.  Buffers are laid out at the largest
 * width and the largest height for every camera.  cosl_klt_group_create is this call with equal
 * sizes, except that it keeps rejecting pitch == 0. */
int cosl_klt_group_create_sizes(const cosl_klt_config* cfg, int nCams, const int* widths,
                                const int* heights, int nLevels, int featW, int featH, int plW, int plH,
                                int device, cosl_klt** out);
/* KLT_SequenceTracker::deallocate (v3d_gpuklt.cpp:626-648). */
int cosl_klt_destroy(cosl_klt* h);

/* KLT_SequenceTracker::detect(image, n, dest) and detect(image, n, dest, nPresent, present)
 * (v3d_gpuklt.cpp:651-738).  `img` is a HOST pointer, rows `pitch` bytes apart.  present3 =
 * nPresent float triples (x, y, ignored), may be NULL when nPresent == 0.  dest has featW*featH
 * entries. */
int cosl_klt_detect(cosl_klt* h, const uint8_t* img, size_t pitch, int nPresent,
                    const float* present3, cosl_klt_feature* dest, int* nDetected);
/* KLT_SequenceTracker::redetect (v3d_gpuklt.cpp:740-805): track + detect around live tracks +
 * refill dead slots in slot order with the strongest new corners. */
int cosl_klt_redetect(cosl_klt* h, const uint8_t* img, size_t pitch, cosl_klt_feature* dest,
                      int* nNewFeatures);
/* KLT_SequenceTracker::track (v3d_gpuklt.cpp:857-889). */
int cosl_klt_track(cosl_klt* h, const uint8_t* img, size_t pitch, cosl_klt_feature* dest,
                   int* nPresent);
/* KLT_SequenceTracker::feedExternFeaturePoints (v3d_gpuklt.cpp:808-855).  pts3 = npts float
 * triples (stride 3 everywhere; the reference reads stride 2 in its distance test -- a bug the
 * survey documents).  trackIds receives the slot of each fed point (npts entries). */
int cosl_klt_feed(cosl_klt* h, int npts, const float* pts3, int* trackIds, int* nFed);
/* KLT_SequenceTracker::advanceFrame (v3d_gpuklt.h:252-259). */
int cosl_klt_advance(cosl_klt* h);
/* setBorderMargin / setConvergenceThreshold / setSSD_Threshold (v3d_gpuklt.h:217-239).  A new value
 * applies to every frame enqueued after the call, on every path: a frame already submitted with
 * cosl_klt_group_submit / _submit_step and not yet collected keeps the values it was enqueued with,
 * and the next submitted frame is the first to use the new one. */
int cosl_klt_set_margin(cosl_klt* h, float margin);
int cosl_klt_set_conv(cosl_klt* h, float thr);
int cosl_klt_set_ssd(cosl_klt* h, float thr);
/* Extension: the 2x2 position covariance of every tracked feature (DESIGN.md section 3.4), the
 * measurement covariance cosl_ba_solver_set_obs_cov / cosl_sba_motstr_levmar_x_cov take.  For each
 * slot with status 0 in a frame where its camera ran the tracker, at the tracker's last level L:
 *   M = J^T J of the tracker's window at the returned position and gain (the gain tracker's 3x3 system
 *       with its gain prior, the neighbour gains fixed; the 2x2 tracker's data matrix),
 *   sigma^2 = noise_var, or SSD / (npx - k) of the window residual when noise_var == 0 (k = 3 with
 *       gain, 2 without; npx = window pixels),
 *   cov = sigma^2 diag(W_c, H_c) [M^-1]_position diag(W_c, H_c), level-0 pixels^2 of camera c.
 * noise_var > 0: fixed residual variance, in the pyramid's intensity units; 0: estimated per slot;
 * < 0: disarmed (the default: nothing is computed and the group launches exactly what it launches
 * without this call).  NaN or inf gives COSL_E_INVALID.  Like cosl_klt_set_ssd it applies to the
 * frames enqueued after the call; a pending prefetch takes it when it is consumed.  An armed frame
 * adds one kernel after the tracker and one D2H copy of C * featW * featH * 3 floats. */
int cosl_klt_set_covariance(cosl_klt* h, float noise_var);
/* The covariances of the last frame handed out (by next, step, track, redetect, detect, first*,
 * run_prefetched, collect or fetch): cov[c] (may be NULL: not written) receives featW * featH
 * (xx, xy, yy) float triples, slot-major.  NaN for a slot that is not tracked (status != 0), whose
 * normal matrix is singular, and for every slot of a camera that frame addressed with FIRST / detect;
 * a camera the frame skipped keeps the entries it had, as its dest[c] does.  COSL_E_STATE when the
 * last frame handed out was not armed, or none was. */
int cosl_klt_group_download_covariance(cosl_klt* h, float* const* cov);
/* Extension: the undistorted pixel position of every slot and, where the frame has position
 * covariances, their covariance in the undistorted image (DESIGN.md section 3.5).  K: C row-major
 * 3x3 camera matrices (C * 9 doubles; K[3] = K[6] = K[7] = 0, K[8] = 1, fx = K[0] > 0, fy = K[4] > 0,
 * skew K[1]); kc: C Bouguet 5-vectors (k1, k2, p1, p2, k3), the forward model OpenCV's projectPoints
 * applies.  For slot i of camera c (W_c x H_c):
 *   u_d = pos[0] W_c, v_d = pos[1] H_c (texel centres at i + 0.5), x_d = K2^-1 (u_d - cx, v_d - cy),
 *       K2 = [[fx, s], [0, fy]];
 *   x* solves d(x*) = x_d by at most 20 Newton steps from x_d, stopping once |K2 (d(x) - x_d)|_inf
 *       <= 1e-9 px; (u, v) = K2 x* + (cx, cy), fp64;
 *   cov = A Sigma_d A^T, A = K2 J(x*)^-1 K2^-1 (J = dd/dx), from the slot's cosl_klt_set_covariance
 *       entry Sigma_d, computed in fp64 and stored as float (xx, xy, yy).
 * NaN for a slot with status < 0 and where the inverse fails (the tolerance is not met, det J <= 0 at an
 * iterate or at the answer, a non-finite value); cov also where Sigma_d is NaN.  With kc = 0 the stage
 * is the identity to roundoff.  K == NULL disarms (the default: nothing is computed, and the group
 * launches exactly what it launches without this call).  COSL_E_INVALID, naming the first bad camera,
 * for a non-finite K or kc, fx <= 0 or fy <= 0, or a malformed K; nothing changes then.  Like
 * cosl_klt_set_covariance it applies to the frames enqueued after the call; a pending prefetch takes
 * it when it is consumed.  An armed frame adds one kernel after the last writer of the feature table and
 * a D2H copy of C * featW * featH * 2 doubles (and * 3 floats with covariances). */
int cosl_klt_set_undistortion(cosl_klt* h, const double* K, const double* kc);
/* Of the last frame handed out (by next, step, track, redetect, detect, first*, run_prefetched, collect
 * or fetch): pos[c] receives featW * featH (u, v) doubles, cov[c] featW * featH (xx, xy, yy) floats,
 * slot-major.  Either array, or any entry of it, may be NULL: not written.  A camera the frame skipped
 * keeps the entries it had, as its dest[c] does.  COSL_E_STATE when the last frame handed out was not
 * armed (or none was), and when cov is given and that frame had no position covariances. */
int cosl_klt_group_download_undistorted(cosl_klt* h, double* const* pos, float* const* cov);

/* Extension (batched GPUKLT::next, tracking/GPUKLT.cpp:144-161): redetect + advanceFrame for all
 * cameras of the group.  imgs[c] are HOST pointers (pinned memory recommended); dest[c] has
 * featW*featH entries; nNew[c] as in redetect.  One H2D copy per camera, one D2H copy of the
 * whole feature table, one stream synchronise. */
int cosl_klt_group_next(cosl_klt* h, const uint8_t* const* imgs, size_t pitch,
                        cosl_klt_feature* const* dest, int* nNew);
/* Same, but images already resident in device memory (dimgs[c] = device pointers, tightly packed
 * rows of `pitch` bytes) and the feature table left on the device: no host transfer, no
 * synchronise; used for the kernel-only throughput number.  Results can be fetched later with
 * cosl_klt_group_fetch.
 * The device images must hold the frame when the call is made, as the host images of next() and
 * submit() do: the group copies them on a stream of its own that runs ahead of the group's stream
 * (cosl_klt_stream) and is NOT ordered after work the caller enqueued there since the previous call.
 * They must stay unchanged until work enqueued on the group's stream after this call has run. */
int cosl_klt_group_next_dev(cosl_klt* h, const uint8_t* const* dimgs, size_t pitch);
int cosl_klt_group_first(cosl_klt* h, const uint8_t* const* imgs, size_t pitch,
                         cosl_klt_feature* const* dest, int* nDetected);
int cosl_klt_group_fetch(cosl_klt* h, cosl_klt_feature* const* dest, int* nNew);
int cosl_klt_group_sync(cosl_klt* h);
/* Per-camera forms of the calls a multi-camera CoSLAM loop makes besides next().  Each camera of the
 * group behaves bit for bit like a single-camera tracker that receives the same calls; cameras a
 * call does not address keep their state.  All three return COSL_E_STATE while frames submitted
 * with cosl_klt_group_submit or _submit_step are not yet collected.
 *
 * KLT_SequenceTracker::feedExternFeaturePoints (v3d_gpuklt.cpp:808-855) for the cameras with
 * npts[c] >= 0; what NewMapPtsNCC::output -> SingleSLAM::feedExtraFeatPtsToTracker ->
 * GPUKLT::feedExternFeatPoints does for one CoSLAM camera group (app/SL_NewMapPointsInterCam.cpp:540-544,
 * app/SL_SingleSLAM.cpp:1168-1171, tracking/GPUKLT.cpp:163-190), without its advanceFrame.
 * npts[c] < 0: camera not addressed, pts3[c] / trackIds[c] not read, nFed[c] not written.
 * pts3[c] = npts[c] float triples as in cosl_klt_feed; trackIds[c] receives npts[c] slots (-1: no
 * dead slot left); nFed[c] = points placed.  One launch per kernel for all addressed cameras, one
 * H2D and one D2H copy, one synchronise. */
int cosl_klt_group_feed(cosl_klt* h, const int* npts, const float* const* pts3, int* const* trackIds,
                        int* nFed);
/* KLT_SequenceTracker::advanceFrame (v3d_gpuklt.h:252-259) for the cameras with cams[c] != 0 (C
 * entries).  All cameras marked is exactly cosl_klt_advance; a strict subset exchanges those
 * cameras' slices of the previous and the current pyramid on the device (a second call swaps them
 * back). */
int cosl_klt_group_advance_cams(cosl_klt* h, const uint8_t* cams);
/* GPUKLT::first(f, img, present, ips) (tracking/GPUKLT.cpp:111-135, called per camera by
 * CoSLAM::initMapMultiCam, app/SL_CoSLAM.cpp:258-262) for the whole group: detect with camera c's
 * nPresent[c] in [0, featW*featH] present points present3[c] (float triples as in cosl_klt_detect,
 * may be NULL when nPresent[c] == 0) + advanceFrame.  All nPresent[c] == 0 is exactly
 * cosl_klt_group_first. */
int cosl_klt_group_first_present(cosl_klt* h, const uint8_t* const* imgs, size_t pitch,
                                 const int* nPresent, const float* const* present3,
                                 cosl_klt_feature* const* dest, int* nDetected);
/* A frame with an op of its own for each camera: GPUKLT::next with a track / re-detect cadence
 * (tracking/GPUKLT.cpp:144-161 picks track() or redetect() from a frame counter), or a rig whose
 * cameras do not all have a frame at every step.  ops[c] is one of: */
enum { COSL_KLT_OP_SKIP = 0,   /* camera not addressed: image not read, state untouched          */
       COSL_KLT_OP_FIRST = 1,  /* detect + advanceFrame      (GPUKLT::first, GPUKLT.cpp:133-142)  */
       COSL_KLT_OP_TRACK = 2,  /* track + advanceFrame       (GPUKLT::next, track branch :153-158) */
       COSL_KLT_OP_NEXT = 3 }; /* redetect + advanceFrame    (GPUKLT::next, :149-152)             */
/* Camera c addressed with an op behaves bit for bit like a single-camera tracker that receives the
 * matching call followed by cosl_klt_advance: its table, its count and every later frame.  n[c] is
 * what that call returns (FIRST: nDetected, TRACK: nPresent, NEXT: nNewFeatures).  A skipped camera
 * keeps all of its state (both pyramids, feature table, gains, the level-0 record of
 * cosl_klt_debug_pyramid); imgs[c] may then be NULL and dest[c] / n[c] are not written.  Every op
 * equal is exactly cosl_klt_group_first / group_next (or track + advance for every camera); all
 * SKIP returns COSL_OK and launches nothing.  Otherwise one launch per kernel serves every
 * addressed camera, and a camera gets the work of its op's stages only.  An op outside the four
 * values or a NULL image of an addressed camera gives COSL_E_INVALID; frames submitted with
 * cosl_klt_group_submit or _submit_step and not yet collected give COSL_E_STATE.  imgs, pitch,
 * dest: as in cosl_klt_group_next. */
int cosl_klt_group_step(cosl_klt* h, const uint8_t* ops, const uint8_t* const* imgs, size_t pitch,
                        cosl_klt_feature* const* dest, int* n);
/* Same with device images, as cosl_klt_group_next_dev: no host transfer, no synchronise (a step
 * whose ops differ copies its small per-camera op table from one of two pinned buffers, and waits
 * for the copy made two such steps earlier only when the host runs that far ahead of the group's
 * streams).  cosl_klt_group_fetch then hands back the tables and counts of the addressed cameras. */
int cosl_klt_group_step_dev(cosl_klt* h, const uint8_t* ops, const uint8_t* const* dimgs, size_t pitch);
/* Frame-pipelined form of cosl_klt_group_next (ingest half of SURVEY.md 8f-4; what
 * SingleSLAM::grabReadFrame + GPUKLT::next become when the next frame is already decoded,
 * app/SL_SingleSLAM.cpp:317-327, tracking/GPUKLT.cpp:144-161): submit() enqueues upload, kernels and
 * the read-back of one frame and returns at once; collect() blocks for the OLDEST submitted frame
 * and hands out its feature tables.  At most two frames may be in flight; calling submit(n+1)
 * before collect(n) overlaps the upload of frame n+1 with the kernels of frame n.  The image
 * buffers of a submitted frame must stay untouched until that frame has been collected. */
int cosl_klt_group_submit(cosl_klt* h, const uint8_t* const* imgs, size_t pitch);
/* Frame-pipelined form of cosl_klt_group_step: enqueues what group_step does plus the read-back of
 * the step, and returns.  ops, imgs, pitch and their checks (COSL_E_INVALID) are group_step's.  It
 * shares the two frames in flight and their order with cosl_klt_group_submit, and the two may be
 * mixed; a third frame gives COSL_E_STATE.  An all-SKIP step launches nothing but still counts as a
 * submitted frame, whose collect writes nothing.  The image buffers of the addressed cameras must
 * stay untouched until the step has been collected.  Like submit it does not wait for the device,
 * with one exception: a step whose ops differ reuses the pinned op table of the step two such steps
 * earlier, and when that step was given to cosl_klt_group_step_dev and its front pass has not yet
 * started, this call waits for it (as step_dev itself does). */
int cosl_klt_group_submit_step(cosl_klt* h, const uint8_t* ops, const uint8_t* const* imgs, size_t pitch);
/* Waits for the oldest frame submitted by either call.  For a submit, every camera's dest[c] / nNew[c]
 * are written as by cosl_klt_group_next; for a submit_step only the addressed cameras' are, with n[c]
 * as cosl_klt_group_step documents it (FIRST: nDetected, TRACK: nPresent, NEXT: nNewFeatures); a
 * skipped camera's entries are left untouched.  COSL_E_STATE when nothing is in flight. */
int cosl_klt_group_collect(cosl_klt* h, cosl_klt_feature* const* dest, int* nNew);
/* A frame in two halves, for a loop that maps between frames (CoSLAM::genNewMapPoints feeds new
 * points to one camera group and advances those cameras, app/SL_CoSLAM.cpp:1368-1371): prefetch
 * enqueues the half that depends on the images alone -- upload, pyramid, cornerness map, the
 * detector's prefilter -- and returns without waiting for the device; feeds and advances may follow;
 * run_prefetched or submit_prefetched then runs the rest (tracker, detector, refill) on the state
 * they left.  The tables, counts and every later frame are bit for bit those of the synchronous call
 * made at consume time: cosl_klt_group_next (ops == NULL, NEXT for every camera, as submit) or
 * cosl_klt_group_step with the same ops.
 *
 * ops: FIRST, TRACK or NEXT for each camera, or NULL.  A SKIP op gives COSL_E_INVALID: a step with
 * skipped cameras builds into the current pyramid, which a feed's advance may still exchange, not
 * into the third buffer, so it cannot be prefetched.  An image for every camera; imgs and pitch as in
 * cosl_klt_group_next.  The upload may still read the image buffers after any call returns except
 * these three: they must stay untouched until run_prefetched returns, until the frame
 * submit_prefetched enqueued has been collected (as for submit), or until discard_prefetch returns.
 * Until the prefetch is consumed, group_fetch and the debug reads show the last consumed frame.  At
 * most one prefetch may be pending (COSL_E_STATE).  While one is, every call that
 * processes a frame of its own images (first*, next*, track, redetect, detect, step*, submit*) and
 * cosl_klt_set_margin (the margin enters the cornerness map) give COSL_E_STATE and change nothing;
 * set_conv / set_ssd act on the tracker, which runs at consume time.  Feeds and advances
 * (cosl_klt_feed, _advance, cosl_klt_group_feed, _advance_cams) are allowed and do not wait for the
 * prefetched work; they still refuse while submitted frames are uncollected.  A prefetch may be made
 * while frames are submitted: the steady state of a loop that maps is
 *   submit_prefetched(n), prefetch(n+1), collect(n), map + feed + advance, submit_prefetched(n+1). */
int cosl_klt_group_prefetch(cosl_klt* h, const uint8_t* ops, const uint8_t* const* imgs, size_t pitch);
/* The dependent half of the pending prefetch, then the read-back: dest / n as group_next (ops ==
 * NULL) or group_step (and, like group_step, COSL_E_STATE while submitted frames are uncollected)
 * would write them.  COSL_E_STATE when nothing is prefetched. */
int cosl_klt_group_run_prefetched(cosl_klt* h, cosl_klt_feature* const* dest, int* n);
/* The same, enqueued as a submitted frame: it shares the two frames in flight and their order with
 * submit / submit_step, and cosl_klt_group_collect returns it.  COSL_E_STATE when nothing is
 * prefetched or two frames are in flight (the prefetch then stays pending). */
int cosl_klt_group_submit_prefetched(cosl_klt* h);
/* Drops the pending prefetch (e.g. a camera must restart with FIRST): every later table, pyramid
 * (cosl_klt_debug_pyramid, its level-0 record), count (cosl_klt_group_fetch) and cornerness map is
 * as if it had never been made.  It waits on the host for the dropped work, the upload included, so
 * the image buffers may be reused when it returns; since that work waits for the submitted frames'
 * trackers that last read its pyramid buffer, a discard may wait for those too.  COSL_E_STATE when
 * nothing is prefetched.  destroy and cosl_klt_group_sync wait for a pending prefetch. */
int cosl_klt_group_discard_prefetch(cosl_klt* h);
/* CUDA stream (cudaStream_t as void*) the group launches on; lets callers time with events.  Parts of
 * a frame run on side streams, but every call joins them into this stream before it returns: work
 * enqueued here after a call sees the whole frame.  The one exception is a pending prefetch: its
 * image half joins this stream only when it is consumed, so work enqueued here in between (feeds and
 * advances included) neither waits for it nor is seen by it, and the consumed frame runs after it. */
void* cosl_klt_stream(cosl_klt* h);

/* Test/inspection hooks (not part of the reference surface). */
/* Copy pyramid level `level` of camera `cam` to host as interleaved (I, Ix, Iy) floats: the camera's
 * own (W_c >> level) x (H_c >> level) texels, returned in *w, *ht.
 * which: 0 = previous frame (pyr0), 1 = current frame (pyr1).  Level 0 of a frame built by
 * next()/redetect() is not stored when the tracker does not visit level 0 (levels L-1, L-1-levelSkip,
 * ...); reading it then returns COSL_E_INVALID.  detect()/first() and track() store every level.
 * The record of what was stored follows each camera through cosl_klt_group_advance_cams. */
int cosl_klt_debug_pyramid(cosl_klt* h, int cam, int which, int level, float* out3, int* w,
                           int* ht);
/* Copy the cornerness map after non-max suppression input stage (W_c*H_c floats) of camera cam. */
int cosl_klt_debug_cornerness(cosl_klt* h, int cam, float* out);
/* Raw number of detector candidates of the last detect/redetect fetched to the host. */
int cosl_klt_debug_num_candidates(cosl_klt* h, int cam);
/* Per-kernel-class device time (CUDA events on the group's stream).  enable(1) resets and starts
 * accumulating; get(idx) returns the class name ("klt_pyramid", "klt_track", "klt_detect",
 * "klt_select") or NULL past the end. */
int cosl_klt_profile_enable(cosl_klt* h, int on);
const char* cosl_klt_profile_get(cosl_klt* h, int idx, double* ms, int* calls);
/* Algorithmic HBM bytes of one group_next call (SURVEY.md 8d contract): C*(25*W*H + 4640*F). */
double cosl_klt_algorithmic_bytes(cosl_klt* h);

/* ================================================================ pose solver */

/* Mirrors IntraCamPoseOption (slam/SL_IntraCamPose.h:19-57). */
typedef struct cosl_pose_opt {
  int maxIterLM;           /* 100  */
  int maxIterRW;           /* 5    */
  double epsErrorChangeLM; /* 1e-7 */
  double epsParamChangeLM; /* 1e-6 */
  double epsErrorChangeRW; /* 1e-6 */
  int verboseLM, verboseRW;
  double lambda0;          /* 1e-3 */
  double lambda;
  double err0, err, errRW;
  int retTypeLM;
  int npts;
  int nIterLM, nIterRW;
} cosl_pose_opt;

void cosl_pose_opt_default(cosl_pose_opt* opt);

/* intraCamEstimate (slam/SL_IntraCamPose.cpp:626-709), exact reference argument list; returns
 * 1 (true) / 0 (false = LM failure) through *ok.  Arrays are HOST pointers. */
int cosl_pose_intracam(const double K[9], const double R0[9], const double t0[3], int npts,
                       const double* prevErrs /* nullable */, const double* Ms, const double* ms,
                       double tau, double R_opt[9], double t_opt[3], cosl_pose_opt* opt, int* ok);
/* Batched over C cameras in one launch (one 128-thread CTA per camera; the option
 * fields maxIterLM, maxIterRW, lambda0 and the three eps* must be equal for all cameras, else
 * COSL_E_INVALID).  K9/R0/t0/R_opt/t_opt are C
 * consecutive blocks; Ms[c]/ms[c]/prevErrs[c] per-camera HOST arrays (prevErrs or prevErrs[c]
 * may be NULL); opts has C entries; ok has C entries. */
int cosl_pose_intracam_batch(int C, const double* K9, const double* R0, const double* t0,
                             const int* npts, const double* const* Ms, const double* const* ms,
                             const double* const* prevErrs, double tau, double* R_opt,
                             double* t_opt, cosl_pose_opt* opts, int* ok, int device);

/* A pose solver handle: the batched solve above without blocking the calling thread, what
 * CoSLAM::parallelPoseUpdate (app/SL_CoSLAM.cpp:398-417) needs to keep tracking while the poses of
 * a frame are refined.  A handle owns a non-blocking stream, its device buffers, a pinned staging
 * buffer for the inputs, a pinned buffer for the results and its events, all allocated by create
 * for at most maxCams cameras and maxPts points (all cameras together) per submit; nothing is
 * allocated afterwards.  Without a usable device create gives COSL_E_CUDA; there is no CPU path.
 *
 * submit takes the arguments of cosl_pose_intracam_batch less the outputs and the device, runs its
 * checks on the calling thread with its codes (COSL_E_INVALID for a NULL argument, a bad camera or
 * options that differ between cameras), and COSL_E_INVALID when C > maxCams or the points exceed
 * maxPts (the handle stays usable).  It packs the inputs into the pinned buffer, so the caller may
 * reuse its arrays when it returns, enqueues one host-to-device copy, the batch call's kernel and
 * the read-back of the results on the handle's stream, and returns without waiting for the device.
 * query sets *done = 1 once the solve has finished, without waiting.  collect waits for it and
 * writes R_opt, t_opt, the opts fields and ok (nullable) exactly as cosl_pose_intracam_batch does
 * for the same inputs, bit for bit; *device_ms (nullable) is the device time of the copies and the
 * kernel, from CUDA events.
 *
 * One solve may be in flight per handle: a second submit gives COSL_E_STATE, and so do query and
 * collect with nothing in flight.  destroy waits for a solve in flight.  A handle is not
 * re-entrant; different handles, on any threads and devices, share no lock.  Every call makes the
 * handle's device current on the calling thread. */
typedef struct cosl_pose_solver cosl_pose_solver;
int cosl_pose_solver_create(int device, int maxCams, int maxPts, cosl_pose_solver** out);
int cosl_pose_solver_destroy(cosl_pose_solver* s);
int cosl_pose_solver_submit(cosl_pose_solver* s, int C, const double* K9, const double* R0,
                            const double* t0, const int* npts, const double* const* Ms,
                            const double* const* ms, const double* const* prevErrs, double tau,
                            const cosl_pose_opt* opts);
/* submit with 2x2 measurement covariances (an extension: the reference's covariance-weighted solve,
 * intraCamCovEstimate, builds them from the map points instead; DESIGN.md 5.2).  covx[c] holds npts[c]
 * row-major covariances [xx, xy, yx, yy] in px^2, in the order of ms[c]; covx == NULL or covx[c] == NULL
 * means identity covariances for that camera.  Per point, with Sigma = [a b; b c] and det = ac - b^2,
 * the upper-triangular whitening factor
 *   L = [sqrt(c/det), -b/sqrt(c det); 0, 1/sqrt(c)],  L^T L = Sigma^-1,
 * is computed on the calling thread (Sigma = I gives exactly L = I, Sigma = 4I exactly 0.5 I) and:
 *   the residual is r~ = L (m - pi(K, R, t, M)) and the rows of the forward-difference Jacobian are
 *   whitened by the same L; the cost is sum w |r~|^2; the LM step is that of cosl_pose_intracam_batch
 *   (rows scaled by w) on the whitened rows, lambda added to the whitened system's diagonal;
 *   the Tukey weights w (from prevErrs and from every re-weighting) stay on the Euclidean pixel
 *   distance |m - pi| against tau;
 *   opts[c].err0, err and errRW are whitened costs.
 * An armed handle's covariance stage uses the same L: H = sum w (L J)^T (L J) with the analytic J,
 * sigma2_hat = sum w |L e|^2 / dof, cov = pixel_var H^-1 (so covariances in px^2 arm with pixel_var
 * = 1); download_covariance's err stays the pixel distance |e|.
 * Every covariance must be finite with xy == yx exactly, xx > 0 and det > 0 (and a finite L), else
 * COSL_E_INVALID naming the first bad camera and point, before anything is staged; the handle stays
 * usable.  Everything else is cosl_pose_solver_submit's: its checks and codes, COSL_E_STATE while a
 * solve is in flight, and query, collect and download_covariance.  cosl_pose_solver_submit is this
 * call with covx = NULL, and runs the unweighted kernels. */
int cosl_pose_solver_submit_cov(cosl_pose_solver* s, int C, const double* K9, const double* R0,
                                const double* t0, const int* npts, const double* const* Ms,
                                const double* const* ms, const double* const* covx,
                                const double* const* prevErrs, double tau, const cosl_pose_opt* opts);
/* submit with Gaussian pose priors (an extension: intraCamEstimate solves every frame from the
 * observations alone; DESIGN.md 5.3).  prior == NULL is cosl_pose_solver_submit_cov exactly; otherwise
 * prior[c] is NULL (no prior on camera c) or 48 doubles: R_p[9] row-major, t_p[3], P[36] row-major, a
 * mean (R_p, t_p) and a 6x6 covariance P in the order (w, dt) of the solver's own chart, the chart of
 * download_covariance: R = R_p exp([w]x), t = t_p + dt.  So a download_covariance block is a valid P.
 * With the upper-triangular L, L^T L = P^-1, computed on the calling thread:
 *   the prior residual is r = [Log(R_p^T R); t - t_p] (Log exact to roundoff up to pi), and the
 *   objective sum_i w_i |L_i (m_i - pi(K, R, t, M_i))|^2 + r^T P^-1 r (L_i = I without covx);
 *   the observation rows are those of cosl_pose_solver_submit_cov; the prior adds the six rows L J_p,
 *   residual L r, with J_p = diag(Jr^-1(r_w), I) for the update R' = R exp([dw]x), t' = t + dt
 *   (Jr^-1 the inverse right Jacobian of SO(3)): (L J_p)^T (L J_p) joins the LM system and
 *   -(L J_p)^T (L r) its right-hand side before lambda is added, with no Tukey weight;
 *   every cost the loop evaluates gains |L r|^2, so opts[c].err0, err and errRW include it and
 *   the LM and re-weighting tests see it; the Tukey weights, prevErrs and download_covariance's err
 *   stay on the pixel distance.
 * An armed handle's covariance stage adds J_p^T P^-1 J_p to H at the answer, 6 to dof and r^T P^-1 r
 * to sigma2_hat's numerator: a camera with a prior and 0, 1 or 2 weighted points is regular, and an
 * unobserved camera (npts 0) with a prior converges to its mean with cov = pixel_var P.  With covx
 * in px^2 (or none and pixel_var = 1) a stored pose covariance is a valid P as it stands; with
 * unweighted observations of pixel variance s2, pass cov / s2.
 * Every prior is checked before anything is staged: |R_p^T R_p - I|_max <= 1e-9 and det R_p > 0,
 * every value finite, P symmetric to 1e-12 of its largest diagonal entry and positive definite;
 * else COSL_E_INVALID naming the first bad camera, and the handle stays usable.  Everything else is
 * cosl_pose_solver_submit_cov's: covx (nullable per camera), its checks and codes, COSL_E_STATE
 * while a solve is in flight, and query, collect and download_covariance. */
int cosl_pose_solver_submit_prior(cosl_pose_solver* s, int C, const double* K9, const double* R0,
                                  const double* t0, const int* npts, const double* const* Ms,
                                  const double* const* ms, const double* const* covx,
                                  const double* const* prior, const double* const* prevErrs, double tau,
                                  const cosl_pose_opt* opts);
int cosl_pose_solver_query(cosl_pose_solver* s, int* done);
int cosl_pose_solver_collect(cosl_pose_solver* s, double* R_opt, double* t_opt, cosl_pose_opt* opts,
                             int* ok, double* device_ms);
/* CUDA stream (cudaStream_t as void*) the handle's solves run on; work enqueued there after a
 * submit runs after that solve. */
void* cosl_pose_solver_stream(cosl_pose_solver* s);
/* Covariance of each refined pose and the residuals of its points (an extension: the reference
 * reports no uncertainty for this step).  Per camera, at the R_opt, t_opt collect returns (whatever
 * ok says), in the solver's own chart R' = R exp([w]x), t' = t + dt, order (w, dt):
 *   e_i = |pi(K, R_opt, t_opt, M_i) - m_i| in pixels, pi the projection of the solve;
 *   w_i = (1 - (e_i / tau)^2)^2, 0 for e_i >= tau;
 *   H = sum_i w_i J_i^T J_i with the analytic 2x6 Jacobian J_i of pi, in fp64;
 *   cov = pixel_var H^-1, 6x6 row-major, by Cholesky.
 * A camera whose factorisation breaks down, or whose smallest relative pivot L_kk^2 / H_kk is below
 * 1e-12 (fewer than 3 weighted points, every point beyond tau), is singular: its covariance is NaN.
 * Every camera is solved on its own: the others of the same submit are unaffected.
 * pixel_var > 0 arms the handle: every later submit ends with the stage on the handle's stream and
 * collect's device_ms includes it.  0 disarms.  Arming allocates the stage's buffers, once, for
 * maxCams and maxPts; destroy frees them.  COSL_E_INVALID for a NULL handle or a pixel_var that is
 * negative or not finite; COSL_E_STATE while a solve is in flight. */
int cosl_pose_solver_set_covariance(cosl_pose_solver* s, double pixel_var);
/* After collect of an armed solve: cov[C][36] (nullable); err[tot] (nullable), e_i of every point in
 * submit order, camera-major; out[C][4] = {sigma2_hat, dof, smallest relative pivot, 1 if the
 * covariance is valid else 0}, with dof = 2 #(w_i > 0) - 6, sigma2_hat = sum w_i e_i^2 / dof (NaN
 * when dof <= 0) and the smallest relative pivot 0 when the factorisation broke down.  COSL_OK also
 * when some cameras are singular (flagged in out).  COSL_E_INVALID for a NULL handle or out;
 * COSL_E_STATE while a solve is in flight, before any armed solve, or after an unarmed submit since
 * (a disarmed handle keeps the last armed result until its next submit). */
int cosl_pose_solver_download_covariance(cosl_pose_solver* s, double* cov, double* err, double* out);
/* Gate and update the map points a frame observes (an extension: poseUpdate3D's point loop after
 * intraCamEstimate; DESIGN.md 5.4).  reserve_mappts allocates, once, the pinned and device buffers for
 * at most maxMapPts map points per submit (all cameras together); 0 frees them.  No submit allocates.
 * COSL_E_INVALID for a NULL handle or maxMapPts < 0, COSL_E_STATE while a solve is in flight. */
int cosl_pose_solver_reserve_mappts(cosl_pose_solver* s, int maxMapPts);
/* cosl_pose_solver_submit_prior plus the map points of each camera: nmap[c] points, Xmap[c] 3 n means
 * (world), Pmap[c] 9 n row-major 3x3 covariances (world, MapPoint::cov's layout), mmap[c] 2 n
 * observations in px, covm[c] 4 n row-major 2x2 covariances [xx, xy, yx, yy] in px^2 (covm and covm[c]
 * nullable: Sigma_m = pixel_var I).  The solve, collect and download_covariance are those of
 * submit_prior with the same arguments, bit for bit.  After the covariance stage, per point j of camera c,
 * at the (R, t) collect returns and its stage covariance P_c (chart R' = R exp([w]x), t' = t + dt):
 *   H_X = d pi / dX = (a; b) R, H_c the stage's analytic 2x6 Jacobian at X0,
 *   R_eff = Sigma_m + H_c P_c H_c^T (the pose uncertainty as measurement noise, linearised at X0);
 *   gate: nu0 = m - pi(X0), S0 = H_X P0 H_X^T + R_eff, d2_0 = nu0^T S0^-1 nu0, e0 = |nu0| in px;
 *   d2_0 < gate (strict): at most 8 fp64 Gauss-Newton steps on (X - X0)^T P0^-1 (X - X0) +
 *   (m - pi(X))^T R_eff^-1 (m - pi(X)), each taken only when it lowers that objective and keeps the
 *   depth (R X + t)_z > 0, stopping at |dX| <= 1e-12 max(1, |X|); the first is the EKF update
 *   X0 + P0 H_X^T S0^-1 nu0.  Then P+ = (P0^-1 + H_X^T R_eff^-1 H_X)^-1 at X+, symmetric, and
 *   d2_1 = nu1^T (H_X P+ H_X^T + R_eff)^-1 nu1 at X+ (reported only).
 *   status 0 updated; 1 gated out; 2 not updatable (depth <= 0 at X0, a non-finite value, S0 not
 *   positive definite), d2_0 NaN; 3 the camera's stage covariance is invalid, d2_0 NaN.  With status
 *   != 0, X and P come back as given (P symmetrised) and d2_1 is NaN.  ok[c] does not change the update.
 * It needs an armed handle (set_covariance) and reserved capacity, else COSL_E_STATE; more map points
 * than reserved, a NULL nmap, Xmap, Pmap or mmap (or entry of a camera with points), a non-finite X or
 * m, a P not symmetric to 1e-12 of its largest diagonal entry or not positive definite, a bad covm
 * (submit_cov's rules) or a gate that is not finite and > 0 give COSL_E_INVALID naming the first bad
 * camera and point, before anything is staged; the handle stays usable.  The update's kernel runs after
 * the covariance stage on the handle's stream, and collect's device_ms includes it. */
int cosl_pose_solver_submit_mappts(cosl_pose_solver* s, int C, const double* K9, const double* R0,
                                   const double* t0, const int* npts, const double* const* Ms,
                                   const double* const* ms, const double* const* covx,
                                   const double* const* prior, const double* const* prevErrs, double tau,
                                   const cosl_pose_opt* opts, const int* nmap, const double* const* Xmap,
                                   const double* const* Pmap, const double* const* mmap,
                                   const double* const* covm, double gate);
/* After collect of a submit_mappts, camera-major in submit order: X[3 n], P[9 n] row-major,
 * stat[3 n] = {d2_0, d2_1, e0} and status[n]; every output nullable.  COSL_E_STATE while a solve is in
 * flight, or when the last submit was not a submit_mappts. */
int cosl_pose_solver_download_mappts(cosl_pose_solver* s, double* X, double* P, double* stat, int* status);
/* PnP RANSAC before the solve (an extension: a robust start where R0, t0 is poor, after solvePnPRobust's EPnP-then-
 * refine pattern; DESIGN.md 5.7).  use[c] != 0 selects camera c of the C cameras of every later submit, of every
 * kind, until the next call; use == NULL disarms.  Per selected camera with n = npts[c] points, in fp64 on the
 * handle's stream between the inputs' copy and the solve:
 *   samples: hypothesis h in [0, nHyp) takes the first 5 distinct idx = u_j mod n of u_j = splitmix64(seed ^
 *   ((c << 40) | (h << 8) | j)), j = 0 .. 255 (splitmix64(x): z = x + 0x9e3779b97f4a7c15, then the standard
 *   SplitMix64 finaliser); none within 256 draws is degenerate;
 *   EPnP (Lepetit et al. 2009) on the 5 points: PCA control points (degenerate when the smallest eigenvalue is below
 *   1e-12 of the largest), the 12x12 M^T M by cyclic Jacobi, betas for N = 1, 2, 3 each refined by 5 Gauss-Newton
 *   steps, absolute orientation with the reflection fix, and of the three the least summed reprojection error over
 *   the sample; a non-finite value is degenerate;
 *   score: point i is an inlier of (R, t) when its depth (R M_i + t)_z > 0 and |m_i - pi(K, R, t, M_i)| < err_thres
 *   (px, Euclidean); a hypothesis scores (inliers, sum over inliers of |e|^2), a degenerate one (-1, 0); covx,
 *   prevErrs and priors do not enter;
 *   select: most inliers, then least sum, then lowest h; the caller's R0, t0 is scored as h = -1 and wins ties.
 * The status of camera c, tested in this order: 3 not selected; 1 n < 5, no hypotheses drawn; 4 R0, t0 kept, no
 * hypothesis beat it; 2 the best hypothesis has fewer than min_inliers inliers, R0, t0 kept; 0 the hypothesis
 * replaced R0, t0.  The solve then starts from that pose and runs unchanged on the same points.  The result does not
 * depend on thread order.  An unarmed handle launches exactly what it did before this call existed.
 * Allocates the hypothesis buffers for nHyp x maxCams once (a later call with a larger nHyp reallocates); no submit
 * allocates.  COSL_E_INVALID for a NULL handle, C not in [1, maxCams], nHyp not in [1, 2^20], err_thres not finite
 * and > 0, or min_inliers < 5, keeping the old setting; COSL_E_STATE while a solve is in flight.  A later submit
 * whose C differs from the armed C gives COSL_E_INVALID. */
int cosl_pose_solver_set_ransac(cosl_pose_solver* s, int C, const uint8_t* use, int nHyp, double err_thres,
                                int min_inliers, uint64_t seed);
/* After collect of a submit that ran RANSAC, per camera: R[9] and t[3], the start pose the solve used; stat[4] =
 * {status, inliers, sum |e|^2, h} of the selection's winner (R0, t0's with h = -1 for status 1, 3 and 4); and
 * inl[tot], camera-major in submit order, 1 where the point is an inlier of the start pose.  Every output
 * nullable.  COSL_E_STATE while a solve is in flight, or when the last submit did not run RANSAC. */
int cosl_pose_solver_download_ransac(cosl_pose_solver* s, double* R, double* t, double* stat, uint8_t* inl);
/* Diagnostics of the same submit, per camera and hypothesis.  *nHyp (nullable) gets the number of hypotheses that
 * submit drew per camera.  The outputs have room for maxHyp hypotheses per camera, camera-major, and each camera's
 * first *nHyp entries are written: idx[5] (-1 where none were drawn or 5 distinct were not found), pose[12] = R | t
 * (unset when degenerate), inliers (-1 when degenerate or not drawn) and sse.  Every output nullable; with all four
 * NULL the call only reports *nHyp.  COSL_E_INVALID when an output is given and maxHyp is below *nHyp, before
 * anything is written; COSL_E_STATE as download_ransac, and also after a set_ransac that reallocated the hypothesis
 * buffers.  A synchronous copy from the device. */
int cosl_pose_solver_download_ransac_hyps(cosl_pose_solver* s, int maxHyp, int* nHyp, int* idx, double* pose,
                                          int* inliers, double* sse);

/* A triangulation handle: batched multi-view triangulation of map points with their 3x3 covariance (an
 * extension: the birth of a MapPoint's M and cov in SingleSLAM::newMapPoints, updateStaticPointPosition and
 * NewMapPointsInterCam, whose triangulation functions are not in this tree; DESIGN.md 5.5).  A handle owns
 * a non-blocking stream, a pinned staging buffer, device buffers, a per-view scratch and a pinned result
 * buffer, all allocated by create for at most maxCams camera entries, maxPts points and maxViews views (all
 * points together) per submit; no submit allocates.  Without a usable device create gives COSL_E_CUDA; there
 * is no CPU path.  COSL_E_INVALID for maxCams < 1, maxPts < 1 or maxViews < 2.
 *
 * submit: a camera table of nCams entries, K9[9 nCams], R[9 nCams] (row-major, world to camera) and
 * t[3 nCams], and camCov (nullable, as camCov[c]): the entry's 6x6 pose covariance, row-major, in the pose
 * solver's chart R' = R exp([w]x), t' = t + dt, order (w, dt), so a download_covariance block is valid as it
 * stands (a BA camCov, in the chart exp([w]x) R, converts as blockdiag(R^T, I) P blockdiag(R, I)).  nPts
 * points in CSR form: point j has the views [viewOff[j], viewOff[j + 1]), 2 to 32 of them, viewOff[0] = 0;
 * view v has the camera entry viewCam[v], the observation m[2 v] in px and covm[4 v] (covm nullable), its
 * row-major 2x2 covariance [xx, xy, yx, yy] in px^2; without covm, Sigma_m = pixel_var I.  A point uses a
 * camera entry at most once; pass the current frame's view last (rho below).  Per point, in fp64, with pi
 * the pose solver's projection, H_X = (a; b) R its Jacobian in X and H_c the covariance stage's 2x6 one:
 *   1. X_lin = A^-1 b, A = sum (I - d d^T), b = sum (I - d d^T) C, d = normalize(R^T K^-1 [m; 1]) and
 *      C = -R^T t per view: the point closest to every ray, by Cholesky;
 *   2. R_v = Sigma_m + H_c(X_lin) P_c H_c(X_lin)^T (Sigma_m without camCov), fixed from here on;
 *   3. from X_lin, at most 10 Gauss-Newton steps s = (sum H_X^T R_v^-1 H_X)^-1 sum H_X^T R_v^-1 nu_v on
 *      f(X) = sum nu_v^T R_v^-1 nu_v, nu_v = m_v - pi_v(X), each taken only when it lowers f and keeps
 *      every depth > 0, else halved at most 4 times; stopped at |s| <= 1e-12 max(1, |X|).  No step is
 *      taken from an X_lin behind a camera;
 *   4. P = (sum H_X^T R_v^-1 H_X)^-1 at X+, by Cholesky, symmetric.  Every 3x3 here counts as positive
 *      definite only with a smallest relative Cholesky pivot L_kk^2 / A_kk of at least 1e-12, and the
 *      Gauss-Newton loop also stops at an information matrix that is not;
 *   5. stat[4] = {f(X+), e_max = max |nu_v| in px, the parallax (the largest angle at X+ between two
 *      rays X+ -> C_v, in radians), rho = sqrt(trace P) / |X+ - C_last|, C_last the point's last view};
 *   6. status 4 degenerate (a smallest relative pivot L_kk^2 / A_kk below 1e-12, i.e. parallel rays; a
 *      non-finite value; R_v or the information matrix not positive definite), else 1 a depth <= 0 at
 *      X_lin or X+, else 2 rho > 1, else 3 e_max >= max_err, else 0.  With status 0, 2 or 3, X, P and
 *      stat are as computed; with 1 or 4 they are NaN.
 * Each point is solved on its own, so a point's output does not depend on the others of the submit.
 * submit checks everything on the calling thread before anything is staged, and gives COSL_E_INVALID
 * naming the first bad camera, point or view (the handle stays usable) for: counts above the reserved
 * sizes; a NULL required array; a non-finite K, R, t or m; an R that is not a rotation (|R^T R - I|_max
 * <= 1e-9, det > 0) or a camCov that is not symmetric to 1e-12 of its largest diagonal entry or not
 * positive definite (the rules of a pose prior, and the message names the entry as a camera's prior); a
 * covm failing submit_cov's rules; a view camera out of range or used twice in one point; a point with
 * fewer than 2 or more than 32 views or a viewOff that is not monotone; a pixel_var that is not finite
 * and > 0; a max_err that is not > 0 (+inf accepts every e_max).  It packs the inputs into pinned memory,
 * so the caller may reuse its arrays when it returns, enqueues one host-to-device copy, tri_kernel and
 * one device-to-host copy on the handle's stream, and returns without waiting for the device.
 *
 * query sets *done = 1 once the request has finished, without waiting.  collect waits for it and writes,
 * per point in submit order, X[3 n], P[9 n] (row-major), stat[4 n] and status[n], every output nullable;
 * *device_ms (nullable) is the device time of the copies and the kernel, from CUDA events.  One request
 * may be in flight per handle: a second submit gives COSL_E_STATE, and so do query and collect with
 * nothing in flight.  destroy waits for a request in flight.  A handle is not re-entrant; different
 * handles share no lock.  Every call makes the handle's device current on the calling thread. */
typedef struct cosl_tri_solver cosl_tri_solver;
int cosl_tri_solver_create(int device, int maxCams, int maxPts, int maxViews, cosl_tri_solver** out);
int cosl_tri_solver_destroy(cosl_tri_solver* s);
int cosl_tri_solver_submit(cosl_tri_solver* s, int nCams, const double* K9, const double* R,
                           const double* t, const double* const* camCov, int nPts, const int* viewOff,
                           const int* viewCam, const double* m, const double* covm, double pixel_var,
                           double max_err);
int cosl_tri_solver_query(cosl_tri_solver* s, int* done);
int cosl_tri_solver_collect(cosl_tri_solver* s, double* X, double* P, double* stat, int* status,
                            double* device_ms);
/* CUDA stream (cudaStream_t as void*) the handle's requests run on; work enqueued there after a submit
 * runs after that request. */
void* cosl_tri_solver_stream(cosl_tri_solver* s);

/* A registration handle: batched Mahalanobis nearest-feature search of map points in the current frame's
 * features (an extension: the geometric half of CoSLAM::activeMapPointRegisterInGroup and
 * curStaticPointRegInGroup, whose getProjectionCovMat is not in this tree; DESIGN.md 5.6).  A handle owns a
 * non-blocking stream, a pinned staging buffer, device buffers (the feature grid and the claim keys among
 * them) and a pinned result buffer, all allocated by create for at most maxCams camera entries, maxPts
 * points, maxQueries query pairs, maxFeats features and maxTrackObs track observations (all points or
 * features together) per submit; no submit allocates.  Without a usable device create gives COSL_E_CUDA;
 * there is no CPU path.  COSL_E_INVALID for maxCams, maxPts, maxQueries or maxFeats < 1 or maxTrackObs < 0.
 *
 * submit: a camera table of nCams entries as cosl_tri_solver_submit's (K9, R, t, camCov in the pose solver's
 * chart, nullable as camCov[c]) with wh[2 nCams], each entry's image width and height in px (1 to 4096).
 * Features in CSR form over the entries: entry c has the features [featOff[c], featOff[c + 1]),
 * featOff[0] = 0; feature f has an undistorted position mf[2 f] (px), covf[4 f] (nullable), its row-major
 * 2x2 covariance Sigma_f in px^2 (pixel_var I without covf), owned[f] (nullable; 0 or 1, 1 when a map point
 * already holds it) and the earlier observations of its track (trkOff nullable: none), [trkOff[f],
 * trkOff[f + 1]), each with a camera entry trkCam[k] and a position trkM[2 k] (px, noise pixel_var I).  nPts
 * points, X[3 j] and PX[9 j] (row-major 3x3, symmetric and positive definite), each with the query entries
 * [qOff[j], qOff[j + 1]) of qCam, at most 32 and each entry at most once per point.  Per query pair (j, c),
 * in fp64, with pi the pose solver's projection, H_X = (a; b) R its Jacobian in X and H_c the covariance
 * stage's 2x6 one:
 *   1. m_hat = pi_c(X_j), S = H_X P_X H_X^T + H_c P_c H_c^T (the second term with the entry's camCov only);
 *   2. d2_f = |L^-1 (m_f - m_hat)|^2 with L L^T = S + Sigma_f over the features of entry c; f* the least
 *      (d2, f) with d2 < gate (+inf allowed: the plain nearest feature), d2_2 the second least such d2;
 *   3. with a finite track_gate, every earlier observation k of f* must have depth > 0 and
 *      d2_k = nu_k^T (H_X P_X H_X^T + H_c P_c H_c^T + pixel_var I)^-1 nu_k < track_gate at its entry;
 *   4. several pairs that hold one feature: the least (d2, point index) keeps it.
 * status, in this order: 7 a non-finite depth, m_hat or S; 1 depth <= 0; 2 m_hat outside [0, W) x [0, H);
 * 3 no feature inside the gate; 4 f* owned; 5 the track check failed; 6 another pair kept f*; else 0,
 * registered.  The result does not depend on the order of points or queries.
 * submit checks everything on the calling thread before anything is staged, and gives COSL_E_INVALID
 * naming the first bad camera, feature, track observation, point or query (the handle stays usable) for:
 * counts above the reserved sizes; a NULL required array; tri's camera-table rules, with its messages; an
 * image size outside [1, 4096]; a featOff, trkOff or qOff that does not start at 0 or is not monotone; a
 * non-finite mf or trkM; a covf failing submit_cov's rules; an owned other than 0 or 1; a track or query
 * camera out of range; an entry queried twice by one point or more than 32 queries; a non-finite X or a P
 * failing the BA point prior's rules; a pixel_var that is not finite and > 0; a gate or track_gate that is
 * not > 0.  It packs the inputs into pinned memory, so the caller may reuse its arrays when it returns,
 * enqueues one host-to-device copy, the binning, search and claim kernels and one device-to-host copy on
 * the handle's stream, and returns without waiting for the device.
 *
 * query sets *done = 1 once the request has finished, without waiting.  collect waits for it and writes,
 * per query pair in submit order, status[Q], feat[Q] (the global feature index f*, -1 for status 1, 2, 3
 * and 7), d2[2 Q] (d2 of f* and d2_2; NaN for 1, 2 and 7, +inf without a feature in the gate) and pred[5 Q]
 * (m_hat and S as xx, xy, yy; NaN for 1 and 7), every output nullable; *device_ms (nullable) is the device
 * time of the copies and the kernels, from CUDA events.  One request may be in flight per handle: a second
 * submit gives COSL_E_STATE, and so do query and collect with nothing in flight.  destroy waits for a
 * request in flight.  A handle is not re-entrant; different handles share no lock.  Every call makes the
 * handle's device current on the calling thread. */
typedef struct cosl_assoc_solver cosl_assoc_solver;
int cosl_assoc_solver_create(int device, int maxCams, int maxPts, int maxQueries, int maxFeats,
                             int maxTrackObs, cosl_assoc_solver** out);
int cosl_assoc_solver_destroy(cosl_assoc_solver* s);
int cosl_assoc_solver_submit(cosl_assoc_solver* s, int nCams, const double* K9, const double* R,
                             const double* t, const double* const* camCov, const int* wh,
                             const int* featOff, const double* mf, const double* covf, const int* owned,
                             const int* trkOff, const int* trkCam, const double* trkM, int nPts,
                             const double* X, const double* PX, const int* qOff, const int* qCam,
                             double pixel_var, double gate, double track_gate);
int cosl_assoc_solver_query(cosl_assoc_solver* s, int* done);
int cosl_assoc_solver_collect(cosl_assoc_solver* s, int* status, int* feat, double* d2, double* pred,
                              double* device_ms);
/* CUDA stream (cudaStream_t as void*) the handle's requests run on; work enqueued there after a submit
 * runs after that request. */
void* cosl_assoc_solver_stream(cosl_assoc_solver* s);

/* ================================================================ bundle adjustment */

/* Flat form of the arguments of
 *   bundleAdjustRobust(nCamsCon, Ks, Rs, Ts, nPtsCon, pts, meas, maxErr, maxIter, nInnerMaxIter)
 * (LibVisualSLAM geometry/SL_BundleAdjust.h; call app/SL_CoSLAMRobustBA.cpp:174-175).
 * Observations are CSR by point: point i owns obs [ptr[i], ptr[i+1]), usually sorted by camera
 * index, the order of vector<vector<Meas2D>> built at app/SL_CoSLAMRobustBA.cpp:109-165; any
 * other order gives the same solution up to the order of the device's floating-point sums.
 * ptr[0] = 0, and a point may have no observation (it is left unchanged).  Moreover,
 * a camera observes a point at most once (as sba's vmask): a problem with a repeated
 * (point, camera) pair is refused with COSL_E_INVALID. */
typedef struct cosl_ba_problem {
  int m;              /* cameras (poses)                                   */
  int n;              /* points                                            */
  int64_t nobs;       /* observations                                      */
  int m_con;          /* first m_con cameras fixed (nCamsCon)              */
  int n_con;          /* first n_con points fixed  (nPtsCon)               */
  double* K;          /* [m][9] row-major intrinsics [fx s cx; 0 fy cy; 0 0 1], read only:
                         K[3], K[6], K[7] are taken as 0 and K[8] as 1 (BundleRTS packs
                         them so), only K[0], K[1], K[2], K[4], K[5] are read          */
  double* R;          /* [m][9] row-major, x_cam = R X + t; updated in place */
  double* t;          /* [m][3] updated in place                           */
  double* X;          /* [n][3] updated in place                           */
  const int64_t* ptr; /* [n+1]                                             */
  const int32_t* cam; /* [nobs] Meas2D::viewId                             */
  const double* xy;   /* [nobs][2] Meas2D::x,y                             */
  uint8_t* outlier;   /* [nobs] out: Meas2D::outlier (may be NULL)         */
} cosl_ba_problem;

typedef struct cosl_ba_options {
  double max_err;     /* maxErr: Tukey scale / outlier threshold in px; <= 0 disables robust
                         weighting (plain sba_motstr_levmar_x behaviour)              */
  int outer_iters;    /* maxIter: robust re-weighting rounds                            */
  int inner_iters;    /* nInnerMaxIter: LM iterations (linear solves) per round         */
  double opts[5];     /* sba opts: {tau for mu0, eps1 |J^T e|_inf, eps2 |dp|, eps3 |e|^2,
                         eps4 relative reduction}; BundleRTS uses {1e-7,1e-12,1e-12,0,1e-16}
                         (app/SL_CoSLAMBA.cpp:323-328)                                  */
  int device;         /* CUDA ordinal of this rank                                      */
  int verbose;
} cosl_ba_options;

/* info[0..9] as sba: {|e0|^2, |e|^2, |J^T e|_inf, |dp|^2, mu/max diag, #iterations, stop reason,
 * #fevals, #jevals, #linear systems}; [10] = total LM trials over all rounds, [11] = seconds spent
 * in the device solve loop (excl. upload), [12] = final weighted cost, [13] = #outliers. */
#define COSL_BA_INFOSZ 16

void cosl_ba_options_default(cosl_ba_options* o);

/* Single-GPU solve, HOST arrays in/out (the drop-in for bundleAdjustRobust). */
int cosl_ba_solve(cosl_ba_problem* prob, const cosl_ba_options* opt, double info[COSL_BA_INFOSZ]);
/* The same call on n_gpus devices of THIS process (devices = CUDA ordinals, NULL = 0..n_gpus-1):
 * one host thread per device, map points sharded over them, one NCCL all-reduce of the reduced
 * camera system per LM trial (SURVEY.md 8e).  n_gpus <= 1 is cosl_ba_solve.  opt->device is
 * ignored when devices is given. */
int cosl_ba_solve_multi(cosl_ba_problem* prob, const cosl_ba_options* opt, int n_gpus,
                        const int* devices, double info[COSL_BA_INFOSZ]);

/* sba_motstr_levmar_x specialised to the KRTS projection (app/SL_CoSLAMBA.cpp:360-363).  Same
 * argument meaning as sba-1.6: n points, ncon fixed, m cameras, mcon fixed, vmask[n*m],
 * p = [m*cnp camera params | n*pnp points] with cnp=11 (fx,cx,cy,ar,s, q1,q2,q3, t1,t2,t3),
 * x = measurements in point-major order, rot0params = m unit quaternions (sbaGlobs::rot0params).
 * func/fjac pointers of the original are not part of this signature (the projection is fixed).
 * Returns number of iterations (>= 0) or a negative COSL_E_*. */
int cosl_sba_motstr_levmar_x(int n, int ncon, int m, int mcon, const char* vmask, double* p,
                             int cnp, int pnp, const double* x, int mnp,
                             const double* rot0params, int itmax, int verbose,
                             const double opts[5], double info[10], int device);
/* The same with sba's covx (an extension of this C-ABI, which had dropped it): covx[k] is the 2x2 covariance
 * (px^2, row-major) of measurement k of x, in x's point-major order; NULL is cosl_sba_motstr_levmar_x.  The
 * least-squares term of measurement k becomes e_k^T covx[k]^-1 e_k, and info[0], info[1] are those sums.  Every
 * covx[k] must be finite, symmetric and positive definite: otherwise COSL_E_INVALID names the first bad one
 * (checked before any device work).  mnp must be 2. */
int cosl_sba_motstr_levmar_x_cov(int n, int ncon, int m, int mcon, const char* vmask, double* p,
                                 int cnp, int pnp, const double* x, const double* covx, int mnp,
                                 const double* rot0params, int itmax, int verbose,
                                 const double opts[5], double info[10], int device);

/* ---- multi-GPU (points sharded across ranks, cameras replicated; one NCCL all-reduce of the
 * packed reduced camera system per LM trial + one small all-reduce of scalars). ---- */
typedef struct cosl_ba_comm cosl_ba_comm; /* opaque */
/* Fill 128 bytes with an ncclUniqueId (rank 0 calls this, then broadcasts the bytes out of band,
 * e.g. through torch.distributed). */
int cosl_nccl_unique_id(uint8_t id[128]);
int cosl_ba_comm_create(const uint8_t id[128], int rank, int nranks, int device,
                        cosl_ba_comm** out);
int cosl_ba_comm_destroy(cosl_ba_comm* c);

/* A solver handle keeps the problem resident on the device so that bench.py can time LM
 * iterations without the upload.  `prob` holds THIS RANK's shard of points/observations (n, nobs,
 * ptr, cam, xy, X local; m, m_con, K, R, t global and identical on all ranks).  n_con applies to
 * the global point order: pass the number of fixed points that fall into this shard. */
typedef struct cosl_ba_solver cosl_ba_solver;
int cosl_ba_solver_create(const cosl_ba_problem* prob, const cosl_ba_options* opt,
                          cosl_ba_comm* comm /* NULL = single GPU */, cosl_ba_solver** out);
/* Re-upload parameters (R, t, X) from the problem struct -- resets the solver to its start. */
int cosl_ba_solver_reset(cosl_ba_solver* s, const cosl_ba_problem* prob);
/* Replace the solver's problem with `prob`, of any size (m, n, nobs, m_con, n_con).  Validates on the
 * calling thread, copies what it needs (the caller may reuse its arrays on return), enqueues the
 * set-up on the solver's stream and returns without waiting for the device.  Afterwards the handle
 * behaves as if cosl_ba_solver_create(prob) had made it: run / run_fixed / submit / download /
 * reset see the loaded problem.  COSL_E_STATE while a submit is in flight; COSL_E_INVALID for a
 * malformed problem (the handle keeps its previous problem) or a multi-rank solver. */
int cosl_ba_solver_load(cosl_ba_solver* s, const cosl_ba_problem* prob);
/* Run the robust loop (outer_iters x inner_iters) on the resident problem. */
int cosl_ba_solver_run(cosl_ba_solver* s, double info[COSL_BA_INFOSZ]);
/* Run exactly `trials` LM trials (linear solves) of one weighted inner loop without any stop test
 * (benchmark mode: LM-iterations/s).  */
int cosl_ba_solver_run_fixed(cosl_ba_solver* s, int trials, double info[COSL_BA_INFOSZ]);
/* Download R, t, X (and outlier flags) into the problem struct's arrays. */
int cosl_ba_solver_download(cosl_ba_solver* s, cosl_ba_problem* prob);
int cosl_ba_solver_destroy(cosl_ba_solver* s);
void* cosl_ba_solver_stream(cosl_ba_solver* s);
/* Non-blocking form of cosl_ba_solver_run.  submit enqueues the same robust loop on the solver's
 * stream and returns at once: the device takes every LM decision (no host read-back until collect).
 * query sets *done = 1 once it has finished, without waiting.  collect waits for it and writes the
 * info fields of run; [11] is the device time from submit to the end of the loop.  download then
 * returns the result.  While a submit is in flight, run, run_fixed, reset, download and submit give
 * COSL_E_STATE; query and collect with nothing in flight give COSL_E_STATE; destroy waits for it.
 * A solver with a multi-rank comm gives COSL_E_INVALID; opt->verbose is ignored. */
int cosl_ba_solver_submit(cosl_ba_solver* s);
int cosl_ba_solver_query(cosl_ba_solver* s, int* done);
int cosl_ba_solver_collect(cosl_ba_solver* s, double info[COSL_BA_INFOSZ]);
/* Ask the BA running on `s` to end at its next decision point.  It may be a submitted BA, or
 * cosl_ba_solver_run executing on another thread.  Returns at once and never waits for the device.
 * A stop applies only to the request that is running or submitted when it is made.  With nothing
 * running it has no effect: it returns COSL_OK and does not stop the next request.  COSL_E_INVALID
 * for a NULL handle or a multi-rank solver (each rank would stop at a different trial, and the
 * per-trial all-reduce would no longer match).
 * The loop checks at every transition into a further stage: into the next linearisation after a
 * finished iteration, into a trial after a linearisation or a rejected trial, and into the next
 * robust round.  The round then ends with stop reason 8 in info[6]; an unfinished iteration is not
 * counted, no further round starts, and the outlier pass still runs on the last accepted iterate, so
 * collect returns COSL_OK and download returns parameters and outlier flags that belong together.
 * run_fixed ignores stops. */
int cosl_ba_solver_stop(cosl_ba_solver* s);
/* Snapshot of the running or last BA (run or submit), without waiting for it:
 * out = {running (0/1), round, iteration in the round, LM trials over all rounds,
 *        cost of the accepted iterate (p_eL2), initial cost of the round, mu, stop requested (0/1)}.
 * The fields come from one decision step, never a mix of two; before the request's first decision
 * fields 1-6 are 0.  After collect (or run) returns, they equal what info reports: round count,
 * info[5], info[10], info[12] / info[1].
 * stop and progress are the only calls that may be made on a handle while another thread is inside
 * run / submit / collect on it. */
int cosl_ba_solver_progress(cosl_ba_solver* s, double out[8]);
/* Marginal covariances of the adjusted cameras and points (an extension: the reference recomputes point
 * covariances by triangulation instead).  At the parameters download returns, with Tukey weights
 * w = (1 - (e / max_err)^2)^2 (0 for e >= max_err; 1 when max_err <= 0) evaluated there, the stage forms
 * H = sum_obs w J^T J over the free parameters and returns diagonal blocks of pixel_var H^-1:
 *   camCov[j]: 6x6, row-major, for (w, t) with R' = exp([w]x) R, t' = t + dt (x_cam = R X + t);
 *   ptCov[i]:  3x3, row-major, for X_i in world coordinates.
 * Fixed cameras and points get zeros.  A free point with fewer than two observations of non-zero weight and no
 * point prior (cosl_ba_solver_set_pt_prior) is left out of H and gets NaN; a point with a prior always enters H.
 * pixel_var > 0 arms: every later cosl_ba_solver_run and cosl_ba_solver_submit ends with the covariance
 * stage on the solver's stream (inside the submitted graph for submit, whose collect then reports its time
 * in info[11] too; not run_fixed).  0 disarms.  Arming allocates the stage's buffers (and so does a load
 * while armed).  COSL_E_INVALID for a multi-rank solver or pixel_var < 0 (or not finite); COSL_E_STATE
 * while a submit is in flight. */
int cosl_ba_solver_set_covariance(cosl_ba_solver* s, double pixel_var);
/* After run / collect of an armed BA: camCov[m][36], ptCov[n][9] (each nullable);
 * out = {pixel_var, sigma2_hat, dof, unconstrained points, device ms of the stage, min relative pivot, camera
 * priors, point priors}: out[6] and out[7] are the numbers of priors set (0 without them).
 * sigma2_hat = sum w |e|^2 / dof over the observations that enter H, dof = 2 #(those with w > 0) -
 * 6 (free cameras) - 3 (points with a covariance); with priors, the numerator gains their sum r^T cov^-1 r and dof
 * gains 6 per camera prior and 3 per point prior.  NaN when dof <= 0: the caller may rescale by
 * sigma2_hat / pixel_var.  The relative pivots are L_ii^2 / S_ii of the Cholesky factor of the reduced
 * camera system (+inf without free cameras).
 * COSL_E_STATE with no covariance for the resident parameters (none armed yet, or load / reset /
 * run_fixed / an unarmed run or submit since) or while a submit is in flight;
 * COSL_E_NUMERIC (nothing written) when the stage found the system singular in the gauge: a pivot
 * break-down or a relative pivot below 1e-12 (e.g. no fixed camera and too few fixed points, or a free
 * camera without an observation of non-zero weight).  The BA itself still returned COSL_OK. */
int cosl_ba_solver_download_covariance(cosl_ba_solver* s, double* camCov, double* ptCov, double out[8]);
/* Measurement covariances of the loaded problem (an extension: sba's covx, DESIGN.md 4.7).  covx[nobs][4]: the
 * 2x2 covariance of each observation in px^2, row-major, in the order of the problem's xy.  The least-squares
 * term of observation k becomes w_k e_k^T covx[k]^-1 e_k: the kernels whiten residual and Jacobian rows by L_k with
 * L_k^T L_k = covx[k]^-1.  The Tukey weights w and the outlier flags stay on the pixel distance |e_k| against
 * max_err.  The costs in info (initial, final, weighted) and the covariance stage's sigma2_hat are whitened; the
 * stage returns pixel_var (J^T W Lambda J)^-1, so with covariances in px^2 pass pixel_var = 1.
 * Validates on the calling thread (every entry finite, symmetric to 1e-12 relative, positive definite): otherwise
 * COSL_E_INVALID names the first bad observation and the handle keeps what it had.  Copies covx (the caller may
 * reuse it on return), enqueues the upload and the factorisation on the solver's stream and returns without
 * waiting.  NULL clears.  The covariances apply to every later run, run_fixed and submit; reset keeps them, load
 * clears them.  COSL_E_STATE while a submit is in flight; COSL_E_INVALID for a NULL handle or a multi-rank solver. */
int cosl_ba_solver_set_obs_cov(cosl_ba_solver* s, const double* covx);
/* Gaussian pose priors on free cameras of the loaded problem (an extension, DESIGN.md 4.8).  Prior k on camera
 * cams[k] has the mean (R[k] row-major 3x3, t[k]) and the 6x6 covariance cov[k] (row-major) for (w, dt) in the chart
 * of camCov: its residual is r = [Log(R R_p^T); t - t_p], and the objective becomes
 *   sum_obs w e^T Lambda e + sum_priors r^T cov^-1 r.
 * cov is in the units of the objective: a camCov of an earlier BA with covariances in px^2 (or with none and
 * pixel_var = 1) is a valid cov as it stands; with unweighted observations of pixel variance s2, pass camCov / s2.
 * Tukey weights and the outlier pass ignore priors.  The priors enter U and ea, every cost in info and progress, the
 * statistics behind mu0, and the covariance stage, whose H gains sum cov^-1 (a problem singular in the gauge may
 * become regular), whose sigma2_hat gains sum r^T cov^-1 r, and whose dof gains 6 per prior; out[6] of
 * cosl_ba_solver_download_covariance is the number of priors.
 * Validates on the calling thread: cams[k] in [m_con, m) and distinct, R[k] a rotation (|R^T R - I|_max <= 1e-9, det
 * > 0), every value finite, cov[k] symmetric to 1e-12 relative and positive definite; otherwise COSL_E_INVALID names
 * the first bad prior and the handle keeps what it had.  Copies the priors (the caller may reuse its arrays on
 * return), enqueues the upload on the solver's stream and returns without waiting.  nPrior == 0 or cams == NULL
 * clears.  The priors apply to every later run, run_fixed and submit; reset keeps them, load clears them.
 * COSL_E_STATE while a submit is in flight; COSL_E_INVALID for a NULL handle, a multi-rank solver or nPrior < 0. */
int cosl_ba_solver_set_cam_prior(cosl_ba_solver* s, int nPrior, const int32_t* cams, const double* R,
                                 const double* t, const double* cov);
/* Gaussian position priors on free points of the loaded problem (an extension, DESIGN.md 4.9).  Prior k on point
 * pts[k] has the mean X[k] (3) and the 3x3 covariance cov[k] (row-major) in world coordinates, the chart of ptCov:
 * its residual is r = X - mu, and the objective gains sum_point_priors r^T cov^-1 r.  Units as for camera priors: a
 * ptCov of an earlier BA with covariances in px^2 (or with none and pixel_var = 1) is a valid cov as it stands; with
 * unweighted observations of pixel variance s2, pass ptCov / s2.  Camera and point priors may be set together.
 * Tukey weights and the outlier pass ignore priors.  The priors enter V and eb, every cost in info and progress, the
 * statistics behind mu0, and the covariance stage: H gains cov^-1 on the point blocks, a point with a prior always
 * gets a finite ptCov (also with zero or one weighted observation; an unobserved one has ptCov = pixel_var cov at
 * its mean), sigma2_hat gains sum r^T cov^-1 r, dof gains 3 per prior, and out[7] of
 * cosl_ba_solver_download_covariance is the number of point priors.  Priors on three non-collinear points fix the
 * gauge of a problem without fixed cameras or points.
 * Validates on the calling thread: pts[k] in [n_con, n) and distinct, every value finite, cov[k] symmetric to 1e-12
 * relative to its largest diagonal entry and positive definite; otherwise COSL_E_INVALID names the first bad prior
 * and the handle keeps what it had.  Copies the priors (the caller may reuse its arrays on return), enqueues the
 * upload on the solver's stream and returns without waiting.  nPrior == 0 or pts == NULL clears.  The priors apply
 * to every later run, run_fixed and submit; reset keeps them, load clears them.  COSL_E_STATE while a submit is in
 * flight; COSL_E_INVALID for a NULL handle, a multi-rank solver or nPrior < 0.  cosl_ba_solve(_multi) and the sba
 * entry points take no priors. */
int cosl_ba_solver_set_pt_prior(cosl_ba_solver* s, int nPrior, const int32_t* pts, const double* X,
                                const double* cov);
/* Per-kernel accumulated device time in ms since create/reset, by name (NULL-terminated list via
 * index): returns name or NULL when idx is out of range. */
const char* cosl_ba_solver_timer(cosl_ba_solver* s, int idx, double* ms, int* calls);
/* enable(1) resets and starts accumulating the per-kernel-class timers above. */
int cosl_ba_solver_profile_enable(cosl_ba_solver* s, int on);
/* Structure of the reduced camera system, for the roofline arithmetic of bench.py:
 * out[0] = order ns, out[1] = doubles in the all-reduce payload [rhs | Schur-structure tiles],
 * out[2] = multiply-adds of the tile Cholesky + substitutions on the used rows,
 * out[3] = Schur pair entries, out[4] = pair work items, out[5] = blocks,
 * out[6] = tiles incl. fill, out[7] = tasks of the solve DAG. */
int cosl_ba_solver_stats(cosl_ba_solver* s, double out[8]);
/* Plan of the reduced-system solve: out = {blocks, Schur-structure tiles, tiles incl. fill, tasks,
 * nested-dissection depth, longest dependency chain (tasks), persistent grid size, small-solve}.
 * small-solve = 1: the system has at most two blocks and one CTA solves it (ba_tile_two). */
int cosl_ba_solver_plan_info(cosl_ba_solver* s, int out[8]);
/* Diagnostic timeline of the persistent solve kernel.  enable != 0: arm tracing for the following
 * solves (returns the task count).  enable == 0: copy the timeline of the LAST solve into
 * out[cap][8] = {SM id, globaltimer ns at ticket, when operands were ready, when done, up to 4
 * phase stamps inside the task} and
 * meta[cap][3] = {task type 0 POTRF / 1 TRSM / 2 UPDATE / 3 BACKWARD / 4 SUM, pivot block, row block},
 * then disarm. */
int cosl_ba_solver_trace(cosl_ba_solver* s, int enable, uint64_t* out, int32_t* meta, int cap);
/* Diagnostic: the task list of the solve plan (16 int32 per task, layout of BaTask in
 * coslam_b200/csrc/ba_plan.h) and the wait lists of the BACKWARD / SUM tasks as (counter, value)
 * pairs; returns the number of tasks. */
int cosl_ba_solver_tasks(cosl_ba_solver* s, int32_t* tasks, int cap, int32_t* lists, int listCap);
/* Diagnostic: solve S x = b with the BA's tile Cholesky on the current device.  S is dense (6mf x 6mf,
 * row-major, only the lower triangle read); the co-visibility of the 6x6 blocks is taken from adj
 * (mf x mf), and entries of S outside those blocks are ignored.  nd_depth < 0: automatic.  *fail = the
 * solver's failure flag (a pivot outside (1e-30, 1e30) or NaN: x is then meaningless, the call still
 * returns COSL_OK).  out as cosl_ba_solver_plan_info, with out[6] = CTAs launched.  Returns COSL_OK or
 * COSL_E_*. */
int cosl_ba_debug_tile_solve(int mf, const uint8_t* adj, int nd_depth, const double* S,
                             const double* b, double* x, int* fail, int out[8]);
/* Diagnostic, like cosl_ba_debug_tile_solve: Z = S^-1 on the tile pattern of adj (fill included) with the
 * covariance stage's factorisation and selected inversion, returned dense (6mf x 6mf, row-major): the
 * blocks (a, c), a >= c, whose tile is in the pattern; zero elsewhere.  *fail = 1 when the factorisation
 * broke down or a relative pivot L_ii^2 / S_ii fell below 1e-12 (Z is then meaningless).
 * out = {blocks, Schur-structure tiles, tiles incl. fill, selected-inversion tasks, nested-dissection
 * depth, steps (one launch each), CTAs of the factorisation, small-solve}. */
int cosl_ba_debug_tile_selinv(int mf, const uint8_t* adj, int nd_depth, const double* S, double* Z,
                              int* fail, int out[8]);

/* ================= post-BA pose-graph spreading (SURVEY.md 8f-2) =================
 * Replaces, for chain graphs, GlobalPoseGraph::computeNewCameraRotations
 * (slam/SL_GlobalPoseEstimation.cpp:52-218) followed by ::computeNewCameraTranslations (:220-359) as
 * RobustBundleRTS::updateNonKeyCameraPoses calls them once per camera
 * (app/SL_CoSLAMRobustBA.cpp:233-250) on the graphs constructCameraGraphs builds (:182-232): one
 * chain per camera, node k -> node k+1, key-frame nodes fixed.  All chains are solved by ONE launch.
 *   chainOff[nChains+1]  first node of each chain (chainOff[0] = 0), N = chainOff[nChains]
 *   fixed[N]             1 = fixed node (CamPoseNode::fixed)
 *   R[9N], t[3N]         node poses, row-major (CamPoseNode::R, ::t)
 *   eR[9N], et[3N]       edge k = rigid transform from node k to node k+1 (CamPoseEdge::R, ::t);
 *                        the slot of a chain's last node is not read
 *   newR[9N], newt[3N]   out: CamPoseNode::newR, ::newt (fixed nodes: copies of R, t)
 * Edges with uncertain scale and the constrained variants (:361-1281) are not on the post-BA path
 * and not provided.  COSL_E_INVALID when a chain with free nodes has no fixed node (the reference's
 * system is rank deficient there). */
int cosl_posegraph_spread_chains(int nChains, const int* chainOff, const uint8_t* fixed,
                                 const double* R, const double* t, const double* eR,
                                 const double* et, double* newR, double* newt, int device);

/* ================= general pose graphs (SURVEY.md 8f-2; the camera-group merge) =================
 * Replaces, on an ARBITRARY edge set, GlobalPoseGraph::computeNewCameraRotations
 * (slam/SL_GlobalPoseEstimation.cpp:52-218: least squares, then the nearest rotation of every free node)
 * together with ::computeNewCameraTranslations4 (:361-525: translations with shared unknown scales),
 * as MergeCameraGroup::recomputeKeyCamPoses calls them (app/SL_MergeCameraGroup.cpp:1083-1086) on the
 * graph _constructGraphForKeyFrms builds (:907-1035).  Both systems are solved by ONE call; the
 * translation system uses the edges' R, not the new rotations, as the reference's does.
 *   fixed[nNodes]          1 = fixed node (CamPoseNode::fixed): copied to newR / newt (:205-216, :505-513)
 *   R[9n], t[3n]           node poses, row-major (CamPoseNode::R, ::t)
 *   id1/id2[nEdges]        edge e runs from node id1[e] to node id2[e] (CamPoseEdge::id1, ::id2)
 *   eR[9e], et[3e]         rigid transform of edge e (CamPoseEdge::R, ::t)
 *   scaleCol[nEdges]       scale column of edge e: t_j - R_e t_i = s[scaleCol[e]] et_e; -1 = known
 *                          scale (t_j - R_e t_i = et_e).  NULL: every scale is known.  The shim maps
 *                          CamPoseEdge::scaleId to columns as :383-403 does.
 *   newR[9n], newt[3n]     out: CamPoseNode::newR, ::newt
 *   scale[nScale]          out: the solved scales (CamPoseEdge::s of the uncertain edges, :515-522)
 * Edges joining two fixed nodes give no rows (:59, :368); parallel edges and edges in both directions
 * are allowed; a disjoint union of graphs is one call.  Never throws.  Returns
 *   COSL_E_INVALID  a node or scale index out of range, a self-loop, a scale column without a row, or a
 *                   connected component with free nodes but no fixed node (the message names one such
 *                   node; the reference's system is rank deficient there);
 *   COSL_E_NUMERIC  a non-positive pivot of the normal equations or a non-finite result;
 *   COSL_E_NOMEM / COSL_E_CUDA  allocation failure / no usable device.
 * A graph without free nodes is answered on the host (copies). */
int cosl_posegraph_solve(int nNodes, const uint8_t* fixed, const double* R, const double* t,
                         int nEdges, const int* id1, const int* id2, const double* eR, const double* et,
                         const int* scaleCol, int nScale, double* newR, double* newt, double* scale,
                         int device);
/* Diagnostic: host time (validation, numbering, planning, CSR lists; ms) of the calling thread's last
 * cosl_posegraph_solve call. */
double cosl_posegraph_last_host_ms(void);

/* ================= pose-graph solver handle =================
 * The two calls above without blocking the calling thread.  It serves the reference's two pose-graph call
 * sites, both run with the BA lock held:
 *   - RobustBundleRTS::output (app/SL_CoSLAMRobustBA.cpp:273-316) after every local BA, and again after a
 *     camera-group merge (app/SL_MergeCameraGroup.cpp:1107): submit_chains after the key-pose write-back
 *     (:279-296), the map-point write-back (:297-310) and other host work, then collect and the non-key
 *     write-back of updateNonKeyCameraPoses;
 *   - MergeCameraGroup::recomputeKeyCamPoses (app/SL_MergeCameraGroup.cpp:1083-1086): submit, collect.
 * A handle owns a non-blocking stream, two timing events, a device buffer from the device's stream-ordered
 * memory pool and pinned buffers for the inputs and the results.  create makes the stream and the events;
 * without a usable device it gives COSL_E_CUDA (there is no CPU path).  The buffers are sized by the first
 * submit and kept while later requests fit; a request that does not fit grows them.  A submit that fits
 * allocates nothing; one that grows them may wait for the device (cudaHostAlloc / cudaFreeHost).
 *
 * submit_chains takes the arguments of cosl_posegraph_spread_chains, submit those of cosl_posegraph_solve,
 * less the outputs and the device.  Each runs the checks and host work of its synchronous call on the
 * calling thread (for submit: validation, numbering, the plan, the CSR lists) and returns that call's code
 * and message for a malformed request (COSL_E_INVALID, COSL_E_NUMERIC when planning fails, COSL_E_NOMEM);
 * the handle stays usable.  It packs the inputs into pinned memory, so the caller may reuse its arrays when
 * it returns, enqueues one host-to-device copy, the synchronous call's kernels with the same launch shapes
 * and one device-to-host copy into pinned memory on the handle's stream, and returns without waiting for
 * the device.  A request the synchronous call answers without the device (a general graph without free
 * nodes, an empty chain table) is in flight all the same, and its collect writes what that call writes
 * (copies of the fixed nodes; nothing).
 *
 * query sets *done = 1 once the request has finished, without waiting.  collect waits for it and writes
 * newR[9N], newt[3N] and, for a general solve, scale[nScale] (nullable when nScale == 0; newR / newt are
 * nullable when N == 0) exactly as the synchronous call does for the same inputs, bit for bit.  It returns
 * the errors only the device detects with the synchronous call's code and message: COSL_E_INVALID for a
 * chain without a fixed node, COSL_E_NUMERIC for a non-positive pivot or a non-finite result; then nothing
 * is written.  *device_ms (nullable) is the device time of the copies and kernels, from CUDA events.
 *
 * One request may be in flight per handle, of either kind: a second submit gives COSL_E_STATE, and so do
 * query and collect with nothing in flight.  destroy waits for a request in flight.  A handle is not
 * re-entrant; different handles, on any threads and devices, share no lock.  Every call makes the handle's
 * device current on the calling thread.  The synchronous calls keep their own per-call buffers and
 * cudaStreamPerThread: threads that call them at the same time do not take turns. */
typedef struct cosl_posegraph_solver cosl_posegraph_solver;
int cosl_posegraph_solver_create(int device, cosl_posegraph_solver** out);
int cosl_posegraph_solver_destroy(cosl_posegraph_solver* s);
int cosl_posegraph_solver_submit_chains(cosl_posegraph_solver* s, int nChains, const int* chainOff,
                                        const uint8_t* fixed, const double* R, const double* t,
                                        const double* eR, const double* et);
int cosl_posegraph_solver_submit(cosl_posegraph_solver* s, int nNodes, const uint8_t* fixed,
                                 const double* R, const double* t, int nEdges, const int* id1,
                                 const int* id2, const double* eR, const double* et,
                                 const int* scaleCol, int nScale);
int cosl_posegraph_solver_query(cosl_posegraph_solver* s, int* done);
int cosl_posegraph_solver_collect(cosl_posegraph_solver* s, double* newR, double* newt,
                                  double* scale, double* device_ms);
/* CUDA stream (cudaStream_t as void*) the handle's requests run on; work enqueued there after a submit
 * runs after that request. */
void* cosl_posegraph_solver_stream(cosl_posegraph_solver* s);

#ifdef __cplusplus
}
#endif
#endif /* COSLAM_B200_H_ */
