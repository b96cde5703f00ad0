/* primitives_cov.cpp -- the stand-ins of ref_stubs/primitives.cpp with working definitions of the three
 * primitives that the reference's covariance-weighted pose solve (intraCamCovEstimate,
 * /root/reference/src/slam/SL_IntraCamPose.cpp:305-360, 457-474, 550-625, 711-795) calls and that abort there,
 * plus an extern "C" entry for it.
 * TEST INFRASTRUCTURE: this file + the UNMODIFIED reference source are compiled into
 * oracle/_ref/libintracam_cov_ref.so by oracle/Makefile.obscov; nothing under coslam_b200/ links it.
 *
 * ref_stubs/primitives.cpp is included as it is, with its three aborting definitions renamed out of the way, so
 * the library runs intraCamEstimate exactly as libintracam_ref.so does and adds:
 *   mat22Inv(A, invA)          the 2x2 inverse [d -b; -c a] / (ad - bc)
 *   mahaDist2(a, b, ivar)      d^T ivar d with d = a - b
 *   getProjectionCovMat(...)   a HARNESS CONVENTION, NOT A RESTATEMENT: LibVisualSLAM's function propagates a map
 *                              point's 3x3 covariance into the image (absent, DESIGN.md 0 row 8f-3).  This one
 *                              returns the 2x2 that ref_intraCamCovEstimate packed into cov[0..3] of the point's
 *                              9-double slot and ignores K, R, t, M and sigma, so that the reference's solve runs on
 *                              caller-given image-plane covariances, as cosl_pose_solver_submit_cov does. */
#include <vector>

#define mat22Inv ref_stubs_mat22Inv_off_path
#define getProjectionCovMat ref_stubs_getProjectionCovMat_off_path
#define mahaDist2 ref_stubs_mahaDist2_off_path
#include "../ref_stubs/primitives.cpp"
#undef mat22Inv
#undef getProjectionCovMat
#undef mahaDist2

void mat22Inv(const double* A, double* invA) {
  const double det = A[0] * A[3] - A[1] * A[2];
  invA[0] = A[3] / det;
  invA[1] = -A[1] / det;
  invA[2] = -A[2] / det;
  invA[3] = A[0] / det;
}

double mahaDist2(const double* a, const double* b, const double* ivar) {
  const double d0 = a[0] - b[0], d1 = a[1] - b[1];
  return d0 * (ivar[0] * d0 + ivar[1] * d1) + d1 * (ivar[2] * d0 + ivar[3] * d1);
}

void getProjectionCovMat(const double*, const double*, const double*, const double*, const double* cov,
                         double* var, double) {
  var[0] = cov[0];
  var[1] = cov[1];
  var[2] = cov[2];
  var[3] = cov[3];
}

/* C entry: the reference's own intraCamCovEstimate with covx[npts][4] (row-major 2x2 in px^2, packed into the
 * reference's 9-double per-point slots for getProjectionCovMat above) and the option block flattened as
 * ref_intraCamEstimate's: {maxIterLM, maxIterRW, epsErrorChangeLM, epsParamChangeLM, epsErrorChangeRW, lambda0} in,
 * {lambda, lambda0, err0, err, errRW, retTypeLM, nIterLM, nIterRW} out. */
extern "C" int ref_intraCamCovEstimate(const double* K, const double* R0, const double* t0, int npts,
                                       const double* prevErrs, const double* covx, const double* Ms,
                                       const double* ms, double tau, double* R_opt, double* t_opt,
                                       const double* optIn, double* optOut) {
  IntraCamPoseOption opt;
  if (optIn) {
    opt.maxIterLM = (int)optIn[0];
    opt.maxIterRW = (int)optIn[1];
    opt.epsErrorChangeLM = optIn[2];
    opt.epsParamChangeLM = optIn[3];
    opt.epsErrorChangeRW = optIn[4];
    opt.lambda0 = optIn[5];
  }
  std::vector<double> covs(9 * (size_t)npts + 1, 0.0);
  for (int i = 0; i < npts; ++i)
    for (int k = 0; k < 4; ++k) covs[9 * (size_t)i + k] = covx[4 * (size_t)i + k];
  const bool ok = intraCamCovEstimate(K, R0, t0, npts, prevErrs, covs.data(), Ms, ms, tau, R_opt, t_opt, &opt);
  if (optOut) {
    optOut[0] = opt.lambda;
    optOut[1] = opt.lambda0;
    optOut[2] = opt.err0;
    optOut[3] = opt.err;
    optOut[4] = opt.errRW;
    optOut[5] = opt.retTypeLM;
    optOut[6] = opt.nIterLM;
    optOut[7] = opt.nIterRW;
  }
  return ok ? 1 : 0;
}
