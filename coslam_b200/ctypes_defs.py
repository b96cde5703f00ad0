"""ctypes mirrors of the PODs declared in include/coslam_b200.h (shared by the product bindings
and by the oracle loader used in tests -- the layouts are identical by construction)."""
import ctypes as C

import numpy as np

COSL_OK = 0
COSL_BA_INFOSZ = 16
COSL_KLT_COMPAT_ITER5 = 1
# ops of cosl_klt_group_step / _submit_step
COSL_KLT_OP_SKIP = 0
COSL_KLT_OP_FIRST = 1
COSL_KLT_OP_TRACK = 2
COSL_KLT_OP_NEXT = 3


class KltConfig(C.Structure):
    """cosl_klt_config == V3D_GPU::KLT_SequenceTrackerConfig (v3d_gpuklt.h:180-199) + compat."""
    _fields_ = [("nIterations", C.c_int), ("nLevels", C.c_int), ("levelSkip", C.c_int),
                ("windowWidth", C.c_int), ("trackBorderMargin", C.c_float),
                ("convergenceThreshold", C.c_float), ("SSD_Threshold", C.c_float),
                ("trackWithGain", C.c_int), ("minDistance", C.c_int),
                ("minCornerness", C.c_float), ("detectBorderMargin", C.c_float),
                ("compat", C.c_int)]

    @staticmethod
    def reference_defaults():
        """KLT_SequenceTrackerConfig() defaults."""
        return KltConfig(12, 3, 2, 5, 4.0, 0.1, 5000.0, 0, 8, 1000.0, 4.0, COSL_KLT_COMPAT_ITER5)

    @staticmethod
    def coslam_live(with_gain=True):
        """What SingleSLAM::initTracker sets (app/SL_SingleSLAM.cpp:291-298) on top of the
        defaults, with Param::* from app/SL_GlobParam.cpp:28-34 and gui/MyApp.cpp:210-211."""
        c = KltConfig.reference_defaults()
        c.minDistance = 8
        c.minCornerness = 3000.0
        c.nLevels = 6
        c.windowWidth = 6
        c.convergenceThreshold = 1.0
        c.SSD_Threshold = 20000.0
        c.trackWithGain = 1 if with_gain else 0
        return c


class KltFeature(C.Structure):
    """cosl_klt_feature == V3D_GPU::KLT_TrackedFeature (v3d_gpuklt.h:166-176)."""
    _fields_ = [("status", C.c_int), ("pos", C.c_float * 2), ("gain", C.c_float), ("fed", C.c_int)]


FEAT_DTYPE = np.dtype([("status", np.int32), ("pos", np.float32, 2), ("gain", np.float32),
                       ("fed", np.int32)])
assert FEAT_DTYPE.itemsize == C.sizeof(KltFeature) == 20


class PoseOpt(C.Structure):
    """cosl_pose_opt == IntraCamPoseOption (slam/SL_IntraCamPose.h:19-57)."""
    _fields_ = [("maxIterLM", C.c_int), ("maxIterRW", C.c_int), ("epsErrorChangeLM", C.c_double),
                ("epsParamChangeLM", C.c_double), ("epsErrorChangeRW", C.c_double),
                ("verboseLM", C.c_int), ("verboseRW", C.c_int), ("lambda0", C.c_double),
                ("lambda_", C.c_double), ("err0", C.c_double), ("err", C.c_double),
                ("errRW", C.c_double), ("retTypeLM", C.c_int), ("npts", C.c_int),
                ("nIterLM", C.c_int), ("nIterRW", C.c_int)]

    @staticmethod
    def defaults():
        o = PoseOpt()
        o.maxIterLM, o.maxIterRW = 100, 5
        o.epsErrorChangeLM, o.epsParamChangeLM, o.epsErrorChangeRW = 1e-7, 1e-6, 1e-6
        o.lambda0 = 1e-3
        return o


class BaProblem(C.Structure):
    _fields_ = [("m", C.c_int), ("n", C.c_int), ("nobs", C.c_int64), ("m_con", C.c_int),
                ("n_con", C.c_int), ("K", C.c_void_p), ("R", C.c_void_p), ("t", C.c_void_p),
                ("X", C.c_void_p), ("ptr", C.c_void_p), ("cam", C.c_void_p), ("xy", C.c_void_p),
                ("outlier", C.c_void_p)]


class BaOptions(C.Structure):
    _fields_ = [("max_err", C.c_double), ("outer_iters", C.c_int), ("inner_iters", C.c_int),
                ("opts", C.c_double * 5), ("device", C.c_int), ("verbose", C.c_int)]

    @staticmethod
    def defaults():
        """RobustBundleRTS defaults (app/SL_CoSLAMRobustBA.h:33-38) + BundleRTS sba opts
        (app/SL_CoSLAMBA.cpp:323-328)."""
        o = BaOptions()
        o.max_err, o.outer_iters, o.inner_iters = 6.0, 5, 10
        o.opts[:] = [1e-3 * 1e-4, 1e-12, 1e-12, 0.0, 1e-16]
        o.device, o.verbose = 0, 0
        return o
