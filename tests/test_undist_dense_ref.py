"""The float64 restatement of the KLT undistortion stage (undist_dense.py, DESIGN.md section 3.5) against
independent anchors: OpenCV's projectPoints / undistortPointsIter for the forward model and the inverse, the
round trip d(inverse(u_d)) = u_d on dense pixel grids, central differences of the inverse for A, Monte-Carlo
draws for the covariance, the identity at k_c = 0, and NaN beyond the fold of a fold-over lens (CPU only)."""
import numpy as np
import pytest

import undist_dense as U


def _grid(W, H, step=1):
    """texel centres (i + 0.5) of a W x H image, every `step` pixels"""
    u, v = np.meshgrid(np.arange(0, W, step) + 0.5, np.arange(0, H, step) + 0.5)
    return u.ravel(), v.ravel()


def _normalised_points(rng, n, r):
    return rng.uniform(-r, r, n), rng.uniform(-r, r, n)


@pytest.mark.parametrize("name", list(U.CALIBS))
def test_forward_model_equals_opencv(name):
    cv2 = pytest.importorskip("cv2")
    K, kc, _, _ = U.CALIBS[name]
    x, y = _normalised_points(np.random.default_rng(1), 4000, 0.8)
    obj = np.stack([x, y, np.ones_like(x)], 1).reshape(-1, 1, 3)
    # OpenCV's projectPoints takes no skew: project with an identity camera, then apply K2 ourselves
    d, _ = cv2.projectPoints(obj, np.zeros(3), np.zeros(3), np.eye(3), kc)
    d = d.reshape(-1, 2)
    fx, s, cx, fy, cy = U.intrinsics(K)
    u, v = U.project(K, kc, x, y)
    assert np.abs(u - (fx * d[:, 0] + s * d[:, 1] + cx)).max() <= 1e-9
    assert np.abs(v - (fy * d[:, 1] + cy)).max() <= 1e-9


@pytest.mark.parametrize("name", ["mild_barrel", "pincushion_tangential"])
def test_inverse_equals_opencv_undistort_points_iter(name):
    cv2 = pytest.importorskip("cv2")
    K, kc, W, H = U.CALIBS[name]
    ud, vd = _grid(W, H, 7)
    u, v, _, ok = U.undistort(K, kc, ud, vd)
    assert ok.all()
    src = np.stack([ud, vd], 1).reshape(-1, 1, 2)
    crit = (cv2.TERM_CRITERIA_COUNT | cv2.TERM_CRITERIA_EPS, 200, 1e-15)
    ref = cv2.undistortPointsIter(src, K, kc, None, K, crit).reshape(-1, 2)
    err = np.abs(np.stack([u, v], 1) - ref).max()
    assert err <= 1e-7, err


@pytest.mark.parametrize("name", list(U.CALIBS))
@pytest.mark.parametrize("size", [(1280, 720), (640, 480)])
def test_round_trip_on_a_dense_grid(name, size):
    K, kc, W0, H0 = U.CALIBS[name]
    W, H = size
    # the calibration scaled to this image size, so that it covers the image as it covers its own
    sc = np.diag([W / W0, H / H0, 1.0])
    Ks = sc @ K
    ud, vd = _grid(W, H)
    u, v, _, ok = U.undistort(Ks, kc, ud, vd)
    assert ok.all(), (name, size, int((~ok).sum()))
    xu, yu = U.normalise(Ks, u, v)
    rd, rv = U.project(Ks, kc, xu, yu)
    err = max(np.abs(rd - ud).max(), np.abs(rv - vd).max())
    assert err <= U.TOL_PX + 1e-12, err  # the stopping rule, and the roundoff of recomputing d in pixels


@pytest.mark.parametrize("name", list(U.CALIBS))
def test_covariance_map_equals_central_differences(name):
    K, kc, W, H = U.CALIBS[name]
    ud, vd = _grid(W, H, 37)
    _, _, J, ok = U.undistort(K, kc, ud, vd)
    assert ok.all()
    A = U.cov_map(K, J)
    h = 1e-2
    cols = []
    for du, dv in ((h, 0.0), (0.0, h)):
        up, vp, _, _ = U.undistort(K, kc, ud + du, vd + dv)
        um, vm, _, _ = U.undistort(K, kc, ud - du, vd - dv)
        cols.append(np.stack([(up - um) / (2 * h), (vp - vm) / (2 * h)], 1))
    num = np.stack(cols, 2)
    assert np.abs(num - A).max() <= 1e-6 * np.abs(A).max()


@pytest.mark.parametrize("name", list(U.CALIBS))
def test_covariance_equals_monte_carlo(name):
    K, kc, W, H = U.CALIBS[name]
    rng = np.random.default_rng(7)
    feats = np.zeros(3, dtype=[("status", "<i4"), ("pos", "<f4", (2,))])
    feats["pos"] = [[0.05, 0.06], [0.93, 0.9], [0.5, 0.5]]     # two corners, where A differs most from I
    Sd = np.array([[0.08, 0.03], [0.03, 0.05]])
    pos, ucov = U.stage(K, kc, W, H, feats, np.tile([Sd[0, 0], Sd[0, 1], Sd[1, 1]], (3, 1)).astype(np.float32))
    assert np.isfinite(ucov).all()
    n = 200_000
    for i in range(3):
        mu = feats["pos"][i].astype(np.float64) * [W, H]
        d = rng.multivariate_normal(mu, Sd, n)
        u, v, _, ok = U.undistort(K, kc, d[:, 0], d[:, 1])
        assert ok.all()
        emp = np.cov(np.stack([u, v]))
        pred = np.array([[ucov[i, 0], ucov[i, 1]], [ucov[i, 1], ucov[i, 2]]])
        assert np.abs(emp - pred).max() <= 0.03 * np.abs(pred).max(), (i, emp, pred)
        assert np.abs(np.array([u.mean(), v.mean()]) - pos[i]).max() < 0.01


@pytest.mark.parametrize("name", list(U.CALIBS))
def test_zero_distortion_is_the_identity(name):
    K, _, W, H = U.CALIBS[name]
    ud, vd = _grid(W, H, 3)
    u, v, J, ok = U.undistort(K, np.zeros(5), ud, vd)
    assert ok.all()
    assert max(np.abs(u - ud).max(), np.abs(v - vd).max()) <= 1e-9
    assert np.abs(U.cov_map(K, J) - np.eye(2)).max() <= 1e-12


def test_fold_over_lens_is_nan_beyond_the_fold():
    """d(r) = r (1 - r^2 / 2) folds at r_u^2 = 2 / 3, where the distorted radius peaks at r_max = 0.5443:
    every pixel inside 0.95 r_max has an answer, and none beyond 1.05 r_max"""
    K = U.camera(400.0, 400.0, 320.0, 240.0)
    kc = np.array([-0.5, 0.0, 0.0, 0.0, 0.0])
    r_max = np.sqrt(2.0 / 3.0) * (1.0 - 1.0 / 3.0)
    ud, vd = _grid(640, 480, 2)
    u, v, _, ok = U.undistort(K, kc, ud, vd)
    xd, yd = U.normalise(K, ud, vd)
    rd = np.hypot(xd, yd)
    inside, beyond = rd < 0.95 * r_max, rd > 1.05 * r_max
    assert inside.sum() > 1000 and beyond.sum() > 1000
    assert ok[inside].all() and np.isfinite(u[inside]).all()
    assert not ok[beyond].any() and np.isnan(u[beyond]).all() and np.isnan(v[beyond]).all()


def test_stage_nan_rules():
    """status < 0 and a NaN input covariance give NaN; a new slot (status 1) without covariance keeps its
    position"""
    K, kc, W, H = U.CALIBS["skew"]
    feats = np.zeros(4, dtype=[("status", "<i4"), ("pos", "<f4", (2,))])
    feats["status"] = [0, -1, 1, 0]
    feats["pos"] = [[0.3, 0.4], [0.3, 0.4], [0.6, 0.2], [0.7, 0.7]]
    cov = np.array([[0.1, 0.0, 0.1], [0.1, 0.0, 0.1], [np.nan] * 3, [0.2, 0.01, 0.1]], np.float32)
    pos, ucov = U.stage(K, kc, W, H, feats, cov)
    assert np.isfinite(pos[[0, 2, 3]]).all() and np.isnan(pos[1]).all()
    assert np.isfinite(ucov[[0, 3]]).all() and np.isnan(ucov[[1, 2]]).all()
    assert U.stage(K, kc, W, H, feats)[1] is None
