"""ctvio_point_covariance / ctvio_feature_table_point_covariance: the covariance of anchored landmarks' world points,
G Sigma_25 G', against references independent of the engine.

A landmark l with inverse depth rho, anchored at time t with the bearing b = (x, y, 1), has the world point
P = R(t) (R_CI b / rho + p_CI) + p(t).  The reference Jacobian G_fd [3, 25] comes from central differences of that
point evaluated with synthetic.spline_pose: each knot rotation of t's segment perturbed on the right (q_k -> q_k
Exp(d)), each knot position additively, rho directly.  Sigma_25 is the joint covariance of the segment's 24 knot dims
and rho: the window covariance's block, the cross column -Sigma W_l' / h_l and the inverse-depth variance.  The windows
are the cases of test_covariance (CASES).
"""
import ctypes as C
import importlib
import os
import subprocess

import numpy as np
import pytest

from helpers import get_state, pkg, syn
from test_covariance import CASES, DENSE_LIMIT, RCOND_MIN, gpu_system, make_case, oracle_case, reference
from test_pose_covariance import (FD_ERR, PriorRecorder, abs_project, bitwise, case_window, check_psd_symmetric,
                                  cov_bound, fd_error_project, project, query_times)

st = importlib.import_module("ctrl-vio_b200.streaming")
P, I32, I64 = C.c_void_p, C.c_int32, C.c_int64
ERR_INVALID, ERR_STATE, ERR_TIME_RANGE = -1, -4, -6
GAUGE = 3  # the runner's gauge: knots 0..3


# ------------------------------------------------------------------------------------------------------------------
# finite-difference reference

def world_points(q, p, rho, t, b, w):
    """P = R(t) (R_CI (x, y, 1) / rho + p_CI) + p(t) for each point"""
    qt, pt = syn.spline_pose(q, p, np.asarray(t, np.int64), w.t0_ns, w.dt_ns)
    bb = np.concatenate([np.asarray(b, float), np.ones((len(t), 1))], 1)
    m = syn.qrot(np.broadcast_to(syn.Q_CtoI, (len(t), 4)), bb) / np.asarray(rho, float)[:, None] + syn.P_CinI
    return syn.qrot(qt, m) + pt


def fd_point_jacobian(q, p, rho, t, b, w, h=1e-6):
    """G_fd [n, 3, 25] and the segment of each point: columns 6k + r over knots s..s+3 (r < 3 rotation, else position),
    column 24 the inverse depth (step h rho)."""
    t = np.asarray(t, np.int64)
    rho = np.asarray(rho, float)
    n = len(t)
    s = (t - w.t0_ns) // w.dt_ns
    rows = np.arange(n)
    G = np.zeros((n, 3, 25))
    for k in range(4):
        for r in range(6):
            out = []
            for sgn in (1.0, -1.0):
                d = np.zeros(3); d[r % 3] = sgn * h
                vals = []
                for i in range(n):
                    qq, pp = q.copy(), p.copy()
                    if r < 3:
                        qq[s[i] + k] = syn.qmul(qq[s[i] + k][None], syn.qexp(d[None]))[0]
                    else:
                        pp[s[i] + k] += d
                    vals.append(world_points(qq, pp, rho[i:i + 1], t[i:i + 1], b[i:i + 1], w)[0])
                out.append(np.array(vals))
            G[rows, :, 6 * k + r] = (out[0] - out[1]) / (2 * h)
    hr = h * rho
    G[:, :, 24] = (world_points(q, p, rho + hr, t, b, w) - world_points(q, p, rho - hr, t, b, w)) / (2 * hr[:, None])
    return G, s


def joint_blocks(cov, cross, var, seg, lm):
    """Sigma_25 [n, 25, 25] from the np x np covariance, the cross columns [nL, np] and the variances"""
    n = len(seg)
    S = np.zeros((n, 25, 25))
    for i, (s, l) in enumerate(zip(seg, lm)):
        S[i, :24, :24] = cov[6 * s:6 * s + 24, 6 * s:6 * s + 24]
        S[i, :24, 24] = S[i, 24, :24] = cross[l, 6 * s:6 * s + 24]
        S[i, 24, 24] = var[l]
    return S


# ------------------------------------------------------------------------------------------------------------------
# CPU part

@pytest.fixture(scope="module")
def point_jac_lib(tmp_path_factory):
    """pose_jacobian / point_jacobian_column of csrc/spline_eval.cuh built for the host"""
    d = tmp_path_factory.mktemp("pointjac")
    src, so = d / "pointjac.cpp", d / "libpointjac.so"
    src.write_text('#include "' + os.path.join(pkg.CSRC_DIR, "spline_eval.cuh") + '"\n' + r'''
using namespace ctvio;
extern "C" int pointjac(int64_t t0, int64_t dt, int nK, const double* q, const double* p, const double* qci,
                        const double* pci, int64_t t, double x, double y, double rho, double* G) {
  SplineParams sp{t0, dt, nK, 1e9 / double(dt)};
  int32_t s; double u;
  if (!spline_index(sp, t, s, u)) return -1;
  KnotPair* tab = new KnotPair[nK];
  for (int k = 0; k + 1 < nK; ++k) make_knot_pair(q, k, tab[k]);
  PoseJacobian pj;
  pose_jacobian<3>(sp, q, p, tab, s, u, pj);
  const M3 R_CI = so3_matrix(Q4{qci[0], qci[1], qci[2], qci[3]});
  for (int c = 0; c < 25; ++c) {
    double col[3];
    point_jacobian_column(pj, R_CI, V3{pci[0], pci[1], pci[2]}, x, y, rho, c, col);
    for (int i = 0; i < 3; ++i) G[i * 25 + c] = col[i];
  }
  delete[] tab;
  return s;
}
''')
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", str(src), "-o", str(so)], check=True)
    lib = C.CDLL(str(so))
    lib.pointjac.restype = C.c_int
    lib.pointjac.argtypes = [I64, I64, C.c_int, P, P, P, P, I64, C.c_double, C.c_double, C.c_double, P]
    return lib


def host_point_jacobian(lib, q, p, t, b, rho, w):
    """G [n, 3, 25] from the kernel's own functions compiled for the host, and the segments"""
    q, p = np.ascontiguousarray(q, float), np.ascontiguousarray(p, float)
    qci, pci = np.ascontiguousarray(syn.Q_CtoI, float), np.ascontiguousarray(syn.P_CinI, float)
    G = np.zeros((len(t), 3, 25))
    seg = np.zeros(len(t), np.int64)
    for i in range(len(t)):
        g = np.zeros((3, 25))
        seg[i] = lib.pointjac(w.t0_ns, w.dt_ns, len(q), q.ctypes.data, p.ctypes.data, qci.ctypes.data, pci.ctypes.data,
                              int(t[i]), float(b[i, 0]), float(b[i, 1]), float(rho[i]), g.ctypes.data)
        G[i] = g
    return G, seg


def point_inputs(w, n_knots, rho_all, n=40, seed=7):
    """n points over the window: landmarks spread over the numbering, anchor times over the spline (knot boundaries and
    both ends included), bearings inside a 90-degree field of view"""
    rng = np.random.default_rng(seed)
    t = query_times(w, n_knots, n)
    lm = np.linspace(0, len(rho_all) - 1, len(t)).astype(np.int32)
    b = rng.uniform(-0.5, 0.5, (len(t), 2))
    return lm, t, b


def test_device_point_jacobian_matches_finite_differences(point_jac_lib):
    """point_jacobian_column (compiled for the host) against G_fd, to FD_ERR of each row's largest entry"""
    w = syn.config_c2()
    q, p = np.ascontiguousarray(w.q0), np.ascontiguousarray(w.p0)
    lm, t, b = point_inputs(w, len(q), w.rho0, 20)
    rho = w.rho0[lm]
    Gfd, s = fd_point_jacobian(q, p, rho, t, b, w)
    G, seg = host_point_jacobian(point_jac_lib, q, p, t, b, rho, w)
    assert np.array_equal(seg, s)
    scale = np.abs(Gfd).max(axis=2, keepdims=True)
    err = np.abs(G - Gfd)
    print(f"worst |G - G_fd| / row scale {float((err / scale).max()):.1e}")
    assert (err <= FD_ERR * scale).all()
    # the inverse-depth column in closed form: -R R_CI b / rho^2
    qt, _ = syn.spline_pose(q, p, t, w.t0_ns, w.dt_ns)
    bb = np.concatenate([b, np.ones((len(t), 1))], 1)
    g_rho = -syn.qrot(qt, syn.qrot(np.broadcast_to(syn.Q_CtoI, (len(t), 4)), bb)) / rho[:, None] ** 2
    assert np.abs(G[:, :, 24] - g_rho).max() <= 1e-12 * np.abs(g_rho).max()


def test_binding_exposes_the_point_covariances():
    for name in ("point_covariance", "feature_table_point_covariance"):
        assert name in pkg.ABI_SYMBOLS and name in pkg.binding.DEVICE_ONLY_SYMBOLS
    assert hasattr(pkg.Estimator, "PointCovariance") and hasattr(pkg.Estimator, "FeatureTablePointCovariance")
    assert "publish_map_covariance" in st.ResidentRunner.__init__.__code__.co_varnames


def test_runner_requires_the_map_for_its_covariance():
    seq = st.config_c5_sequence(2)
    with pytest.raises(ValueError, match="publish_map"):
        st.ResidentRunner(None, seq, triangulate=True, device_features=True, publish_map_covariance=True)


def test_host_mirror_call_compiles(tmp_path):
    src = tmp_path / "point_cov_mirror.cpp"
    src.write_text('#include "' + os.path.join(pkg.PKG_DIR, "host", "trajectory_estimator.hpp") + '"\n'
                   "double f(ctvio_host::TrajectoryEstimator& e) {\n"
                   "  int32_t l[2] = {0, 1};\n"
                   "  int64_t t[2] = {0, 1};\n"
                   "  double b[4] = {0, 0, 0.1, -0.1};\n"
                   "  double cov[2 * 9];\n"
                   "  return e.GetPointCovariance(2, l, t, b, 3, cov);\n"
                   "}\n")
    subprocess.run(["g++", "-std=c++17", "-fsyntax-only", str(src)], check=True)


# ------------------------------------------------------------------------------------------------------------------
# GPU part

def engine_cross(cov, W, hl):
    """the cross columns -Sigma W_l' / h_l [nL, np] (0 for a landmark without information) and their absolute products"""
    act = hl > 0
    inv = np.where(act, 1.0 / np.where(act, hl, 1.0), 0.0)
    return -(W @ cov) * inv[:, None], (np.abs(W) @ np.abs(cov)) * inv[:, None]


def dense_reference(s, free):
    """H^-1 over the free dims by a dense fp64 inverse: (Sigma [np, np], cross [nL, np], var [nL])"""
    A, W, hl = s["A"], s["W"], s["hl"]
    np_, nL = A.shape[0], len(hl)
    H = np.block([[A, W.T], [W, np.diag(hl)]])
    keep = np.concatenate([free, hl > 0])
    Hk = H[np.ix_(keep, keep)]
    sf = 1.0 / (1.0 + np.sqrt(np.diag(Hk)))
    full = sf[:, None] * np.linalg.inv(sf[:, None] * Hk * sf[None, :]) * sf[None, :]
    nf = int(free.sum())
    lm = np.nonzero(hl > 0)[0]
    cov = np.zeros((np_, np_)); cross = np.zeros((nL, np_)); var = np.zeros(nL)
    cov[np.ix_(free, free)] = full[:nf, :nf]
    cross[np.ix_(lm, np.nonzero(free)[0])] = full[nf:, :nf]
    var[lm] = np.diag(full)[nf:]
    return cov, cross, var


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_point_covariance_matches_references(oracle_lib, cuda_lib, name):
    """Per case, about 40 points: C against G_fd Sigma_25 G_fd' with Sigma_25 from the engine's own Covariance(), W and
    h (the projection alone), and against the fp64 inverse of the oracle's H with its cross block (end to end)."""
    s = oracle_case(oracle_lib, name)
    ref = reference(s)
    w = case_window(oracle_lib, name)
    est, _ = make_case(cuda_lib, oracle_lib, name)
    est.SetDeterministic(True)
    cov, var, rc0 = est.Covariance()
    q, p = est.GetKnots()
    rho_all = est.GetInvDepths()
    lm, t, b = point_inputs(w, est.n_knots, rho_all)
    C_, rc = est.PointCovariance(lm, t, b)
    assert rc == rc0 and C_.shape == (len(t), 3, 3)
    check_psd_symmetric(C_)
    Gfd, seg = fd_point_jacobian(q, p, rho_all[lm], t, b, w)
    # 1. the projection alone: Sigma_25 from the engine's Sigma, W and h
    A, W, hl = gpu_system(est)
    nL = len(rho_all)
    cross, cross_abs = engine_cross(cov, W[:nL], hl[:nL])
    S = joint_blocks(cov, cross, var, seg, lm)
    S_abs = joint_blocks(np.abs(cov), cross_abs, var, seg, lm)
    tol1 = 1e-7 * abs_project(Gfd, S_abs) + fd_error_project(Gfd, S)
    err1 = np.abs(C_ - project(Gfd, S))
    assert (err1 <= tol1).all(), float((err1 / np.maximum(tol1, 1e-300)).max())
    # 2. end to end against the fp64 reference, with the covariance bound propagated through |G|
    free, sc = s["free"], ref["sc"]
    Sb = cov_bound(est, s, ref)
    if s["A"].shape[0] + len(s["hl"]) <= DENSE_LIMIT:
        cov_r, cross_r, var_r = dense_reference(s, free)
        # cov_bound's bound holds for every entry of the scaled inverse K^-1 (dense: landmarks included); unscaled with
        # the camera and landmark Jacobi scales
        i = int(np.argmax(free))
        bound = Sb[i, i] / sc[i] ** 2
        sl = 1.0 / (1.0 + np.sqrt(np.maximum(s["hl"], 0.0)))
        d = np.where(free, sc, 0.0)
        cross_b = bound * sl[:, None] * d[None, :]
        var_b = bound * sl ** 2
    else:
        Wo, ho = s["W"], s["hl"]
        cov_r = ref["cov"]
        cross_r, _ = engine_cross(cov_r, Wo, ho)
        inv = np.where(ho > 0, 1.0 / np.where(ho > 0, ho, 1.0), 0.0)
        var_r = np.where(ho > 0, inv + np.einsum("la,ab,lb->l", Wo, cov_r, Wo) * inv ** 2, 0.0)
        dW, dh = np.abs(W[:nL] - Wo), np.abs(hl[:nL] - ho)
        # first-order propagation of the Sigma bound and of the two assemblies' W, h difference
        cross_b = (np.abs(Wo) @ Sb + dW @ np.abs(cov_r) + np.abs(Wo @ cov_r) * (dh * inv)[:, None]) * inv[:, None]
        var_b = (dh * inv ** 2 + (np.einsum("la,ab,lb->l", np.abs(Wo), Sb, np.abs(Wo))
                                  + 2 * np.einsum("la,ab,lb->l", dW, np.abs(cov_r), np.abs(Wo))) * inv ** 2
                 + 2 * np.abs(np.einsum("la,ab,lb->l", Wo, cov_r, Wo)) * dh * inv ** 3)
    Sref = joint_blocks(cov_r, cross_r, var_r, seg, lm)
    Sbnd = joint_blocks(Sb, cross_b, var_b, seg, lm)
    tol = abs_project(Gfd, Sbnd) + 1e-7 * abs_project(Gfd, np.abs(Sref) + S_abs) + fd_error_project(Gfd, Sref)
    err = np.abs(C_ - project(Gfd, Sref))
    r2 = float((err / np.maximum(tol, 1e-300)).max())
    print(f"{name}: {len(t)} points, rcond {rc0:.2e}; worst ratio to bound: projection "
          f"{float((err1 / np.maximum(tol1, 1e-300)).max()):.1e}, end to end {r2:.1e}")
    assert (err <= tol).all(), r2


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["c2", "masked"])
def test_knot_part_is_the_pose_covariance_projected(oracle_lib, cuda_lib, point_jac_lib, name):
    """G_k Sigma_sub G_k' (numpy, G_k from the kernel's own Jacobian functions, Sigma_sub from Covariance()) equals
    A C_6 A' within rounding, A = [-R [m]x, I] and C_6 the body (dtheta, dp) block of PoseCovariance at the anchor time;
    the masked case's points on constant knots get exactly var_rho g_rho g_rho' (the Covariance() variance)."""
    w = case_window(oracle_lib, name)
    est, _ = make_case(cuda_lib, oracle_lib, name)
    est.SetDeterministic(True)
    cov, var, _ = est.Covariance()
    q, p = est.GetKnots()
    rho_all = est.GetInvDepths()
    lm, t, b = point_inputs(w, est.n_knots, rho_all)
    rho = rho_all[lm]
    G, seg = host_point_jacobian(point_jac_lib, q, p, t, b, rho, w)
    Sk = np.stack([cov[6 * x:6 * x + 24, 6 * x:6 * x + 24] for x in seg])
    Gk = G[:, :, :24]
    knot = project(Gk, Sk)
    C6 = est.PoseCovariance(t)[0][:, :6, :6]
    qt = est.QueryTrajectory(t)[0]
    bb = np.concatenate([b, np.ones((len(t), 1))], 1)
    m = syn.qrot(np.broadcast_to(syn.Q_CtoI, (len(t), 4)), bb) / rho[:, None] + syn.P_CinI
    R = st.quat_matrix(qt)
    mx = np.zeros((len(t), 3, 3))
    mx[:, 0, 1], mx[:, 0, 2], mx[:, 1, 2] = -m[:, 2], m[:, 1], -m[:, 0]
    mx -= np.swapaxes(mx, 1, 2)
    Am = np.concatenate([-R @ mx, np.broadcast_to(np.eye(3), (len(t), 3, 3))], 2)
    mag = abs_project(Gk, Sk) + abs_project(Am, np.abs(C6))
    err = np.abs(knot - project(Am, C6))
    print(f"{name}: worst |G_k S G_k' - A C6 A'| / magnitude {float((err / np.maximum(mag, 1e-300)).max()):.1e}")
    assert (err <= 1e-12 * mag).all()
    if name == "masked":  # segments <= 9 use constant knots only: C = var_l g_rho g_rho'
        C_, _ = est.PointCovariance(lm, t, b)
        on = seg <= 9
        assert on.any()
        g = G[on, :, 24]
        want = var[lm[on], None, None] * g[:, :, None] * g[:, None, :]
        assert (np.abs(C_[on] - want) <= 1e-13 * np.abs(want)).all()


@pytest.mark.gpu
def test_gauge_argument(oracle_lib, cuda_lib):
    """The c2 window without fixed knots is rank deficient (only rcond written); with gauge_knot_index = 3 it matches the
    c2 case, whose options fix knots 0..3."""
    free, _ = make_case(cuda_lib, oracle_lib, "c2", fixed_knot_index=-1)
    fixed, _ = make_case(cuda_lib, oracle_lib, "c2")
    for e in (free, fixed):
        e.SetDeterministic(True)
    w = case_window(oracle_lib, "c2")
    lm, t, b = point_inputs(w, free.n_knots, free.GetInvDepths())
    f = cuda_lib.lib.ctvio_point_covariance
    f.argtypes = [P, I32, P, P, P, I32, P, P]
    f.restype = C.c_int
    out = np.full((len(t), 3, 3), 123.5)
    rcond = C.c_double(-1.0)
    rc = f(free.h, len(t), lm.ctypes.data, t.ctypes.data, b.ctypes.data, -1, out.ctypes.data, C.byref(rcond))
    msg = cuda_lib._fn["last_error"]().decode()
    print(f"no gauge: rc {rc}, rcond {rcond.value:.2e}, '{msg}'")
    assert rc == ERR_STATE and "rank deficient" in msg and (out == 123.5).all()
    assert 0.0 <= rcond.value < RCOND_MIN or "pivot" in msg
    Cg, rg = free.PointCovariance(lm, t, b, gauge_knot_index=3)
    Cf, rf = fixed.PointCovariance(lm, t, b)
    d = np.sqrt(np.einsum("nii->ni", Cf))
    scale = d[:, :, None] * d[:, None, :]
    err = np.abs(Cg - Cf)
    print(f"rcond {rg:.3e} vs {rf:.3e}, worst relative {float((err / np.maximum(scale, 1e-300)).max()):.1e}")
    assert (err <= 1e-12 * scale).all()
    assert abs(rg - rf) <= 1e-12 * rf


@pytest.mark.gpu
def test_special_values_and_errors(oracle_lib, cuda_lib):
    """masked case with one extra landmark no factor touches: on four constant knots its point covariance is exactly
    zero, with rho = -1 or NaN a matrix of NaNs; every error path leaves the outputs untouched."""
    w = case_window(oracle_lib, "masked")
    est, _ = make_case(cuda_lib, oracle_lib, "masked")
    est.SetDeterministic(True)
    rho = est.GetInvDepths()
    extra = len(rho)
    t = w.t0_ns + np.arange(14, dtype=np.int64) * w.dt_ns + w.dt_ns // 3
    lm = np.full(len(t), extra, np.int32)
    b = np.tile([0.1, -0.2], (len(t), 1))
    est.SetInvDepths(np.append(rho, 0.3))
    C_, _ = est.PointCovariance(lm, t, b)
    assert not C_[:10].any()                      # four constant knots, rho constant
    assert all(C_[k].any() for k in range(10, 14))
    check_psd_symmetric(C_)
    for bad in (-1.0, np.nan):
        est.SetInvDepths(np.append(rho, bad))
        Cb, _ = est.PointCovariance(np.append(lm[:2], 0), t[:3], np.concatenate([b[:2], b[:1]]))
        assert np.isnan(Cb[:2]).all() and np.isfinite(Cb[2]).all()
    est.SetInvDepths(np.append(rho, 0.3))

    f = cuda_lib.lib.ctvio_point_covariance
    f.argtypes = [P, I32, P, P, P, I32, P, P]
    f.restype = C.c_int
    t_end = w.t0_ns + (est.n_knots - 3) * w.dt_ns
    good_t = np.array([w.t0_ns + 5, t_end - 1], np.int64)
    good_l = np.array([0, extra], np.int32)
    good_b = np.zeros((2, 2))
    out = np.full((2, 3, 3), 123.5)
    rcond = C.c_double(-7.0)

    def call(h=est.h, n=2, l=good_l, tt=good_t, bb=good_b, gauge=-1, o=out):
        a = [None if x is None else x.ctypes.data for x in (l, tt, bb)]
        return f(h, n, *a, gauge, None if o is None else o.ctypes.data, C.byref(rcond))
    cases = [
        (dict(h=None), ERR_INVALID), (dict(n=-1), ERR_INVALID), (dict(l=None), ERR_INVALID),
        (dict(tt=None), ERR_INVALID), (dict(bb=None), ERR_INVALID), (dict(o=None), ERR_INVALID),
        (dict(l=np.array([0, extra + 1], np.int32)), ERR_INVALID), (dict(l=np.array([-1, 0], np.int32)), ERR_INVALID),
        (dict(gauge=-2), ERR_INVALID), (dict(gauge=est.n_knots), ERR_INVALID),
        (dict(tt=np.array([w.t0_ns - 1, t_end - 1], np.int64)), ERR_TIME_RANGE),
        (dict(tt=np.array([w.t0_ns, t_end], np.int64)), ERR_TIME_RANGE),
    ]
    for kw, code in cases:
        assert call(**kw) == code, kw
        assert (out == 123.5).all() and rcond.value == -7.0, kw
    assert call(n=0, l=None, tt=None, bb=None, o=None) == 0 and rcond.value == -7.0
    # the table call without a feature-table window
    g = cuda_lib.lib.ctvio_feature_table_point_covariance
    g.argtypes = [P, I32, I32, P, P]
    g.restype = C.c_int
    assert g(None, 0, -1, out.ctypes.data, C.byref(rcond)) == ERR_INVALID
    assert g(est.h, 2, -1, out.ctypes.data, C.byref(rcond)) == ERR_STATE
    assert g(est.h, 2, est.n_knots, out.ctypes.data, C.byref(rcond)) == ERR_INVALID
    assert (out == 123.5).all() and rcond.value == -7.0
    cfg = pkg.make_config(**w.config_kwargs())
    bare = pkg.Estimator(cuda_lib, cfg)
    with pytest.raises(pkg.CtvioError, match=r"\(-1\)"):  # no landmark yet: every index is out of range
        bare.PointCovariance([0], [w.t0_ns], [[0.0, 0.0]])


@pytest.mark.gpu
def test_no_side_effects_and_transfer_counts(oracle_lib, cuda_lib):
    """Deterministic mode: a solve after the call is bitwise the solve without it (C3 window with its prior); the call
    moves 28 n bytes up and 72 n bytes down."""
    runs = []
    w = case_window(oracle_lib, "c3prior")
    for with_cov in (True, False):
        est, _ = make_case(cuda_lib, oracle_lib, "c3prior")
        est.SetDeterministic(True)
        lm, t, b = point_inputs(w, est.n_knots, est.GetInvDepths(), 20)
        if with_cov:
            x0 = get_state(est)
            est.PointCovariance(lm, t, b, gauge_knot_index=5)
            x1 = get_state(est)
            assert all(np.array_equal(a, c) for a, c in zip(x0[:4], x1[:4])) and x0[4] == x1[4]
            est.TransferStats(reset=True)
            est.PointCovariance(lm, t, b)
            assert est.TransferStats() == (28 * len(t), 72 * len(t))
        s = est.Solve(8)
        runs.append((s, get_state(est)))
    (s1, x1), (s2, x2) = runs
    for fld in ("iterations", "num_successful_steps", "num_unsuccessful_steps", "termination", "initial_cost",
                "final_cost", "final_radius", "num_linear_solves", "num_jacobian_evals"):
        assert getattr(s1, fld) == getattr(s2, fld), fld
    assert all(np.array_equal(a, c) for a, c in zip(x1[:4], x2[:4])) and x1[4] == x2[4]


def anchor_inputs(runner, anchor, ids):
    """(anchor times, bearings) of the window's landmarks as the engine's tables hold them: the anchor slot's frame time
    and the anchor feature's (x, y) from the cloud the runner sent (float32 on the wire, widened on the device)"""
    frame_of = {s: f for f, s in runner.slot_of.items()}
    t = np.array([runner.seq.kf_times[frame_of[int(a)]] for a in anchor], np.int64)
    b = np.zeros((len(ids), 2))
    for k, (a, i) in enumerate(zip(anchor, ids)):
        pts, ch_id = runner.clouds.message(frame_of[int(a)])[:2]
        j = np.nonzero((np.asarray(ch_id, np.float32).astype(np.float64) + 0.5).astype(np.int64) == i)[0]
        assert len(j) == 1
        b[k] = np.asarray(pts, np.float32)[j[0], :2].astype(np.float64)
    return t, b


@pytest.mark.gpu
def test_table_call_is_the_general_call(cuda_lib):
    """C5 resident run (device_features=True), right after GaugeRealign in two windows: FeatureTablePointCovariance is
    bitwise PointCovariance over the same landmarks, the anchor slots' frame times and the stored bearings; it moves
    nothing up and 72 n_lm bytes down; its errors leave the outputs untouched."""
    seq = st.quantize_wire(st.config_c5_sequence(3))
    r = st.ResidentRunner(cuda_lib, seq, triangulate=True, device_features=True)
    e = r.est
    e.SetDeterministic(True)
    seen = []
    realign = e.GaugeRealign

    def probe(*args):
        realign(*args)
        e.TransferStats(reset=True)
        Ct, rt = e.FeatureTablePointCovariance(GAUGE)
        n = e.n_lm
        assert e.TransferStats() == (0, 72 * n)
        ids, anchor, _ = e.FeatureTableLandmarks()
        t, b = anchor_inputs(r, anchor, ids)
        Cg, rg = e.PointCovariance(np.arange(n, dtype=np.int32), t, b, gauge_knot_index=GAUGE)
        assert bitwise(Ct, Cg) and rt == rg
        assert np.isfinite(Ct).all()
        check_psd_symmetric(Ct)
        g = cuda_lib.lib.ctvio_feature_table_point_covariance
        g.argtypes = [P, I32, I32, P, P]
        g.restype = C.c_int
        out = np.full((n, 3, 3), 123.5)
        rc = C.c_double(-7.0)
        for args, code in (((n + 1, GAUGE, out.ctypes.data), ERR_INVALID), ((n, GAUGE, None), ERR_INVALID),
                           ((n, -2, out.ctypes.data), ERR_INVALID), ((n, e.n_knots, out.ctypes.data), ERR_INVALID)):
            assert g(e.h, *args, C.byref(rc)) == code, args
            assert (out == 123.5).all() and rc.value == -7.0
        seen.append((n, rt))

    e.GaugeRealign = probe
    for _ in range(2):
        r.step()
    print("windows (n_lm, rcond):", seen)
    assert len(seen) == 2
    # after the slide the window no longer describes the table
    g = cuda_lib.lib.ctvio_feature_table_point_covariance
    out = np.full((e.n_lm, 3, 3), 123.5)
    assert g(e.h, e.n_lm, GAUGE, out.ctypes.data, None) == ERR_STATE and (out == 123.5).all()


@pytest.mark.gpu
@pytest.mark.parametrize("reanchor", [False, True])
def test_runner_publish_map_covariance_only_reads(cuda_lib, reanchor):
    """Six C5 windows, deterministic: with publish_map_covariance=True the runner solves, marginalizes, slides and
    publishes the map bitwise as with publish_map=True alone.  Every attached point covariance is finite, symmetric,
    PSD, rcond >= 1e-14.  Default slide: every map point has one; reanchor=True: exactly the points re-anchored in
    the slide (anchored in the leaving frame in the window) carry NaN."""
    n = 6
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    kw = dict(triangulate=True, device_features=True, publish_map=True, reanchor=reanchor)
    a = st.ResidentRunner(cuda_lib, seq, **kw)
    b = st.ResidentRunner(cuda_lib, seq, publish_map_covariance=True, **kw)
    for x in (a, b):
        x.est.SetDeterministic(True)
        x.est.lib = PriorRecorder(x.est.lib)
    windows = []
    realign = b.est.GaugeRealign

    def probe(*args):  # the window's landmarks and the slot that leaves with the slide (every C5 frame is a keyframe)
        realign(*args)
        ids, anchor, _ = b.est.FeatureTableLandmarks()
        windows.append((ids, anchor, b.slot_of[b.frames[0]]))
    b.est.GaugeRealign = probe
    maps, covs = [], []
    for _ in range(n):
        a.step()
        b.step()
        assert all(bitwise(u, v) for u, v in zip(a.last_map, b.last_map))
        maps.append(b.last_map)
        covs.append(b.last_map_cov)
    for rec in b.records:
        print(f"window {rec['window']}: point_cov_rcond {rec['point_cov_rcond']:.3e}, ms_point_cov "
              f"{rec['ms_point_cov']:.3f}, {rec['n_map_points']} points, {rec['n_map_points_without_cov']} without"
              + (f", {rec['n_reanchored']} re-anchored" if reanchor else ""))
    for key in ("iterations", "initial_cost", "final_cost", "prior_dim", "n_obs", "n_lm", "n_map_points"):
        assert [x[key] for x in a.records] == [x[key] for x in b.records], key
    assert "point_cov_rcond" not in a.records[0] and a.last_map_cov is None
    assert bitwise(a.q[:a.ncp], b.q[:b.ncp]) and bitwise(a.p[:a.ncp], b.p[:b.ncp])
    assert bitwise(a.est.GetBiases(), b.est.GetBiases())
    assert bitwise(a.est.GetInvDepths(), b.est.GetInvDepths())
    assert bitwise(a.ld, b.ld)
    pa, pb = a.est.lib.priors, b.est.lib.priors
    assert len(pa) == len(pb) > 0
    assert all(bitwise(x, y) for u, v in zip(pa, pb) for x, y in zip(u, v))
    for rec, m, c, (ids, anchor, leaving) in zip(b.records, maps, covs, windows):
        assert rec["point_cov_rcond"] >= RCOND_MIN, rec
        assert c.shape == (len(m[1]), 3, 3)
        no_cov = np.isnan(c).any(axis=(1, 2))
        assert (np.isnan(c[no_cov]).all())
        assert rec["n_map_points_without_cov"] == int(no_cov.sum())
        moved = set(ids[anchor == leaving].tolist())
        numbered = set(ids.tolist())
        want = np.array([i in moved or i not in numbered for i in m[1].tolist()], bool)
        assert np.array_equal(no_cov, want)
        if reanchor:
            assert 0 < no_cov.sum() <= rec["n_reanchored"]
        else:
            assert not no_cov.any()
        check_psd_symmetric(c[~no_cov])
        assert (np.einsum("nii->ni", c[~no_cov]) > 0).all()
