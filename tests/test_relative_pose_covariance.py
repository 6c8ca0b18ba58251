"""ctvio_relative_pose_covariance: the covariance of the pose at t_b in the frame of the pose at t_a, G Sigma_U G', and
the cross-covariance of the two poses, J_a Sigma_U J_b', against references independent of the engine.

The poses are those of ctvio_pose_covariance (the body, or the camera R R_CI, p + R p_CI), the relative pose is
R_ab = R_a' R_b, p_ab = R_a' (p_b - p_a).  The reference Jacobians come from central differences of that relative pose
built with synthetic.spline_pose, over the union U of the knots of the two segments (sorted, 4 to 8 knots): each knot
rotation perturbed on the right (q_k -> q_k Exp(d)), each knot position additively; the rows of G_fd are
Log(R_ab0' R_ab) and p_ab - p_ab0, those of J_fd_a / J_fd_b Log(R_0' R) and p - p_0 of each pose.  The window
covariances are the cases of test_covariance (CASES).
"""
import ctypes as C
import importlib
import os
import subprocess

import numpy as np
import pytest

from helpers import get_state, pkg, syn
from test_covariance import CASES, RCOND_MIN, make_case, oracle_case, reference
from test_pose_covariance import (FD_ERR, PriorRecorder, abs_project, bitwise, case_window, check_psd_symmetric,
                                  cov_bound, project)

st = importlib.import_module("ctrl-vio_b200.streaming")
P, I32, I64 = C.c_void_p, C.c_int32, C.c_int64
ERR_INVALID, ERR_STATE, ERR_TIME_RANGE = -1, -4, -6
GAUGE = 3  # the runner's gauge: knots 0..3
MU = 48    # the largest union: two disjoint segments


# ------------------------------------------------------------------------------------------------------------------
# finite-difference reference

def frame_poses(q, p, t, w, camera):
    """(quaternion, position) at the times t: of the body, or of the camera (R R_CI, p + R p_CI)"""
    qt, pt = syn.spline_pose(q, p, np.asarray(t, np.int64), w.t0_ns, w.dt_ns)
    if camera:
        pt = pt + syn.qrot(qt, np.broadcast_to(syn.P_CinI, pt.shape))
        qt = syn.qmul(qt, np.broadcast_to(syn.Q_CtoI, qt.shape))
    return qt, pt


def relative(qa, pa, qb, pb):
    return syn.qmul(syn.qconj(qa), qb), syn.qrot(syn.qconj(qa), pb - pa)


def union_knots(w, ta, tb):
    """the sorted union of the knots of the segments of ta and tb"""
    sa, sb = (int(ta) - w.t0_ns) // w.dt_ns, (int(tb) - w.t0_ns) // w.dt_ns
    return sorted(set(range(sa, sa + 4)) | set(range(sb, sb + 4)))


def fd_relative_jacobian(q, p, ta, tb, w, camera=False, h=1e-5):
    """G_fd, J_fd_a, J_fd_b [n, 6, MU] over each pair's union (columns 6u + r, r < 3 rotation, else position; zero past
    6 |U|) and the unions.  The step is 10 x test_pose_covariance's: p_ab subtracts two positions of the window's size,
    so rounding dominates the error at 1e-6 (up to 1e-9 of a row on C2); at 1e-5 rounding and truncation together stay
    below 1e-10 of each row."""
    n = len(ta)
    G, Ja, Jb = np.zeros((n, 6, MU)), np.zeros((n, 6, MU)), np.zeros((n, 6, MU))
    knots = []
    for i in range(n):
        U = union_knots(w, ta[i], tb[i])
        knots.append(U)
        tt = np.array([ta[i], tb[i]], np.int64)
        q0, p0 = frame_poses(q, p, tt, w, camera)
        qr0, pr0 = relative(q0[:1], p0[:1], q0[1:], p0[1:])
        for u, k in enumerate(U):
            for r in range(6):
                out = []
                for sgn in (1.0, -1.0):
                    qq, pp = q.copy(), p.copy()
                    d = np.zeros(3); d[r % 3] = sgn * h
                    if r < 3:
                        qq[k] = syn.qmul(qq[k][None], syn.qexp(d[None]))[0]
                    else:
                        pp[k] += d
                    qx, px = frame_poses(qq, pp, tt, w, camera)
                    qr, pr = relative(qx[:1], px[:1], qx[1:], px[1:])
                    out.append(np.concatenate([syn.qlog(syn.qmul(syn.qconj(qr0), qr))[0], (pr - pr0)[0],
                                               syn.qlog(syn.qmul(syn.qconj(q0), qx)).ravel(), (px - p0).ravel()]))
                col = (out[0] - out[1]) / (2 * h)
                c = 6 * u + r
                G[i, :, c], Ja[i, :3, c], Jb[i, :3, c] = col[:6], col[6:9], col[9:12]
                Ja[i, 3:, c], Jb[i, 3:, c] = col[12:15], col[15:18]
    return G, Ja, Jb, knots


def fd_scale(G, Ja, Jb):
    """[n, 6, 1] the size of each row of G_fd for its FD error: its largest entry, or the largest entry of the pose rows
    it is formed from when those cancel (t_a == t_b)"""
    return np.maximum(np.abs(G), np.maximum(np.abs(Ja), np.abs(Jb))).max(axis=2, keepdims=True)


def fd_err_project(A, Ea, S, B, Eb):
    """the part of |A_fd S B_fd' - A S B'| the FD errors Ea, Eb (per row) of A_fd, B_fd can make"""
    Ea, Eb = np.broadcast_to(Ea, A.shape), np.broadcast_to(Eb, B.shape)
    return (np.einsum("nia,nab,njb->nij", Ea, np.abs(S), np.abs(B)) + np.einsum("nia,nab,njb->nij", np.abs(A), np.abs(S), Eb)
            + np.einsum("nia,nab,njb->nij", Ea, np.abs(S), Eb))


def cross(A, S, B):
    return np.einsum("nia,nab,njb->nij", A, S, B)


def abs_cross(A, S, B):
    return np.einsum("nia,nab,njb->nij", np.abs(A), np.abs(S), np.abs(B))


def union_blocks(cov, knots):
    """Sigma_U [n, MU, MU] (zero past 6 |U|)"""
    S = np.zeros((len(knots), MU, MU))
    for i, U in enumerate(knots):
        idx = (6 * np.asarray(U)[:, None] + np.arange(6)[None, :]).ravel()
        S[i, :len(idx), :len(idx)] = cov[np.ix_(idx, idx)]
    return S


def pair_times(w, n_knots, n=50, seed=11):
    """about n pairs over the window: the same segment, overlapping segments 1..3 knots apart, disjoint segments, t_a ==
    t_b and t_a > t_b, both ends of the spline included"""
    rng = np.random.default_rng(seed)
    t_end = w.t0_ns + (n_knots - 3) * w.dt_ns  # the first time outside the spline
    gaps = [0, 1, 2, 3, 4, 7, n_knots // 2]
    ta, tb = [], []
    for i in range(n - 4):
        a = int(rng.integers(w.t0_ns, t_end))
        if i % 8 == 7:
            b = a
        else:
            g = gaps[i % len(gaps)]
            b = min(max(a + g * w.dt_ns + int(rng.integers(-w.dt_ns // 3, w.dt_ns // 3)), w.t0_ns), t_end - 1)
        if i % 3 == 1:
            a, b = b, a
        ta.append(a)
        tb.append(b)
    ta += [w.t0_ns, t_end - 1, w.t0_ns, t_end - 1]
    tb += [t_end - 1, w.t0_ns, w.t0_ns + w.dt_ns - 1, t_end - 1]
    return np.array(ta, np.int64), np.array(tb, np.int64)


def pair_kinds(w, ta, tb):
    sa, sb = (ta - w.t0_ns) // w.dt_ns, (tb - w.t0_ns) // w.dt_ns
    d = np.abs(sa - sb)
    return dict(same=(d == 0) & (ta != tb), overlap=(d >= 1) & (d <= 3), disjoint=d >= 4, equal=ta == tb,
                reversed=ta > tb)


# ------------------------------------------------------------------------------------------------------------------
# CPU part

@pytest.fixture(scope="module")
def rel_jac_lib(tmp_path_factory):
    """relative_pose_jacobian_column with pose_jacobian / pose_jacobian_column / frame_pose / relative_pose of
    csrc/spline_eval.cuh built for the host, composed as relative_pose_cov_kernel composes them"""
    d = tmp_path_factory.mktemp("reljac")
    src, so = d / "reljac.cpp", d / "libreljac.so"
    src.write_text('#include "' + os.path.join(pkg.CSRC_DIR, "spline_eval.cuh") + '"\n' + r'''
using namespace ctvio;
extern "C" int reljac(int64_t t0, int64_t dt, int nK, const double* q, const double* p, const double* qci,
                      const double* pci, int64_t ta, int64_t tb, int camera, double* G, double* JaJb, int32_t* knots) {
  SplineParams sp{t0, dt, nK, 1e9 / double(dt)};
  int32_t sa, sb; double ua, ub;
  if (!spline_index(sp, ta, sa, ua) || !spline_index(sp, tb, sb, ub)) return -1;
  KnotPair* tab = new KnotPair[nK];
  for (int k = 0; k + 1 < nK; ++k) make_knot_pair(q, k, tab[k]);
  const M3 R_CI = so3_matrix(Q4{qci[0], qci[1], qci[2], qci[3]});
  const V3 p_CI{pci[0], pci[1], pci[2]};
  M3 R[2];
  V3 pos[2];
  for (int side = 0; side < 2; ++side) {
    PoseJacobian pj;
    pose_jacobian<3>(sp, q, p, tab, side ? sb : sa, side ? ub : ua, pj);
    for (int c = 0; c < 24; ++c) {
      double col[12];
      pose_jacobian_column(pj, camera != 0, R_CI, p_CI, c, col);
      for (int i = 0; i < 6; ++i) JaJb[side * 144 + i * 24 + c] = col[i];
    }
    frame_pose(pj, camera != 0, R_CI, p_CI, R[side], pos[side]);
  }
  const RelativePose rel = relative_pose(R[0], pos[0], R[1], pos[1]);
  const int nu = 4 + relative_union_offset(sa, sb);
  for (int c = 0; c < 6 * nu; ++c) {
    double g[6];
    relative_pose_jacobian_column(rel, JaJb, relative_union_first(sa, sb), JaJb + 144, relative_union_first(sb, sa), c, g);
    for (int i = 0; i < 6; ++i) G[i * 48 + c] = g[i];
  }
  for (int u = 0; u < nu; ++u) knots[u] = relative_union_knot(sa, sb, u);
  delete[] tab;
  return nu;
}
''')
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", str(src), "-o", str(so)], check=True)
    lib = C.CDLL(str(so))
    lib.reljac.restype = C.c_int
    lib.reljac.argtypes = [I64, I64, C.c_int, P, P, P, P, I64, I64, C.c_int, P, P, P]
    return lib


def host_relative_jacobian(lib, q, p, ta, tb, w, camera):
    """G [n, 6, MU] from the kernel's own functions compiled for the host, and the unions"""
    q, p = np.ascontiguousarray(q, float), np.ascontiguousarray(p, float)
    qci, pci = np.ascontiguousarray(syn.Q_CtoI, float), np.ascontiguousarray(syn.P_CinI, float)
    G = np.zeros((len(ta), 6, MU))
    knots = []
    for i in range(len(ta)):
        g, jj, k = np.zeros((6, MU)), np.zeros(2 * 144), np.zeros(8, np.int32)
        nu = lib.reljac(w.t0_ns, w.dt_ns, len(q), q.ctypes.data, p.ctypes.data, qci.ctypes.data, pci.ctypes.data,
                        int(ta[i]), int(tb[i]), int(camera), g.ctypes.data, jj.ctypes.data, k.ctypes.data)
        assert nu >= 4
        G[i] = g
        knots.append(k[:nu].tolist())
    return G, knots


def test_pair_times_cover_every_kind():
    for w in (syn.config_c2(), syn.config_c4()):
        ta, tb = pair_times(w, len(w.q0))
        assert all(k.any() for k in pair_kinds(w, ta, tb).values())
        assert {len(union_knots(w, a, b)) for a, b in zip(ta, tb)} == {4, 5, 6, 7, 8}


def test_device_relative_jacobian_matches_finite_differences(rel_jac_lib):
    """The Jacobian relative_pose_cov_kernel builds (the same inline functions, compiled for the host) against G_fd in
    both frames, for pairs in the same segment, in overlapping and disjoint segments, with t_a == t_b and t_a > t_b,
    to FD_ERR of each row's size (fd_scale)"""
    w = syn.config_c2()
    q, p = np.ascontiguousarray(w.q0), np.ascontiguousarray(w.p0)
    ta, tb = pair_times(w, len(q), 24)
    for camera in (False, True):
        Gfd, Ja, Jb, kfd = fd_relative_jacobian(q, p, ta, tb, w, camera)
        G, knots = host_relative_jacobian(rel_jac_lib, q, p, ta, tb, w, camera)
        assert knots == kfd
        scale = fd_scale(Gfd, Ja, Jb)
        err = np.abs(G - Gfd)
        print(f"camera {camera}: worst |G - G_fd| / row size {float((err / scale).max()):.1e}")
        assert (err <= FD_ERR * scale).all(), float((err / scale).max())
        # t_a == t_b: the relative pose does not move, G is zero to rounding
        eq = ta == tb
        assert eq.any() and np.abs(G[eq]).max() <= 1e-14 * scale[eq].max()


def test_binding_exposes_the_relative_pose_covariance():
    assert ("relative_pose_covariance" in pkg.ABI_SYMBOLS
            and "relative_pose_covariance" in pkg.binding.DEVICE_ONLY_SYMBOLS)
    assert hasattr(pkg.Estimator, "RelativePoseCovariance")
    assert "publish_odometry_covariance" in st.ResidentRunner.__init__.__code__.co_varnames


def test_host_mirror_call_compiles(tmp_path):
    src = tmp_path / "rel_pose_cov_mirror.cpp"
    src.write_text('#include "' + os.path.join(pkg.PKG_DIR, "host", "trajectory_estimator.hpp") + '"\n'
                   "double f(ctvio_host::TrajectoryEstimator& e) {\n"
                   "  int64_t ta[2] = {0, 1}, tb[2] = {1, 0};\n"
                   "  double cov[2 * 36], cross[2 * 36];\n"
                   "  return e.GetRelativePoseCovariance(2, ta, tb, 3, true, cov) +\n"
                   "         e.GetRelativePoseCovariance(2, ta, tb, -1, false, cov, cross);\n"
                   "}\n")
    subprocess.run(["g++", "-std=c++17", "-fsyntax-only", str(src)], check=True)


# ------------------------------------------------------------------------------------------------------------------
# GPU part

@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_relative_pose_covariance_matches_references(oracle_lib, cuda_lib, name):
    """Per case, about 50 pairs of every kind, both frames: cov6 against G_fd Sigma_U G_fd' and cross6 against
    J_fd_a Sigma_U J_fd_b' (Sigma the engine's Covariance(), the one the call forms), and both against the fp64
    reference end to end, the covariance bound propagated through the Jacobians; cov6 exactly symmetric and PSD."""
    s = oracle_case(oracle_lib, name)
    ref = reference(s)
    w = case_window(oracle_lib, name)
    est, _ = make_case(cuda_lib, oracle_lib, name)
    est.SetDeterministic(True)
    cov, _, rc0 = est.Covariance(want_rho=False)
    q, p = est.GetKnots()
    ta, tb = pair_times(w, est.n_knots)
    Sbound = cov_bound(est, s, ref)
    worst = np.zeros(4)
    for camera in (False, True):
        C6, X6, rc = est.RelativePoseCovariance(ta, tb, camera_frame=camera, want_cross=True)
        C6b, none, rcb = est.RelativePoseCovariance(ta, tb, camera_frame=camera)
        assert rc == rc0 == rcb and none is None and C6.shape == X6.shape == (len(ta), 6, 6)
        assert bitwise(C6, C6b)
        check_psd_symmetric(C6)
        G, Ja, Jb, knots = fd_relative_jacobian(q, p, ta, tb, w, camera)
        E = FD_ERR * fd_scale(G, Ja, Jb)
        Ea, Eb = FD_ERR * np.abs(Ja).max(axis=2, keepdims=True), FD_ERR * np.abs(Jb).max(axis=2, keepdims=True)
        S, Sref, Sb = union_blocks(cov, knots), union_blocks(ref["cov"], knots), union_blocks(Sbound, knots)
        checks = []
        for got, A, EA, B, EB in ((C6, G, E, G, E), (X6, Ja, Ea, Jb, Eb)):
            # 1. the projection alone
            tol1 = 1e-7 * abs_cross(A, S, B) + fd_err_project(A, EA, S, B, EB)
            err1 = np.abs(got - cross(A, S, B))
            # 2. end to end against the fp64 reference
            tol2 = (abs_cross(A, Sb, B) + 1e-7 * abs_cross(A, np.abs(Sref) + np.abs(S), B)
                    + fd_err_project(A, EA, Sref, B, EB))
            err2 = np.abs(got - cross(A, Sref, B))
            for err, tol in ((err1, tol1), (err2, tol2)):
                r = np.where(tol > 0, err / np.maximum(tol, 1e-300), np.where(err > 0, np.inf, 0.0))
                checks.append(float(r.max()))
        worst = np.maximum(worst, checks)
        assert (np.array(checks) <= 1.0).all(), (camera, checks)
    print(f"{name}: {len(ta)} pairs, rcond {rc0:.2e}; worst ratio to bound: cov6 projection {worst[0]:.1e}, "
          f"end to end {worst[1]:.1e}; cross6 projection {worst[2]:.1e}, end to end {worst[3]:.1e}")


def hat(v):
    m = np.zeros(v.shape[:-1] + (3, 3))
    m[..., 0, 1], m[..., 0, 2], m[..., 1, 2] = -v[..., 2], v[..., 1], -v[..., 0]
    return m - np.swapaxes(m, -1, -2)


def pose_joint_and_relative_jacobian(est, ta, tb, camera, cross6):
    """[[P_a, X], [X', P_b]] [n, 12, 12] from the (dtheta, dp) blocks of PoseCovariance at t_a and t_b and cross6, and
    the relative-pose Jacobian [A_a A_b] [n, 6, 12] built here from QueryTrajectory:
    A_a = [[-R_ab', 0], [[p_ab]x, -R_a']], A_b = [[I, 0], [0, R_a']]"""
    Pa = est.PoseCovariance(ta, camera_frame=camera)[0][:, :6, :6]
    Pb = est.PoseCovariance(tb, camera_frame=camera)[0][:, :6, :6]
    joint = np.block([[Pa, cross6], [np.swapaxes(cross6, 1, 2), Pb]])
    R_CI, p_CI = st.quat_matrix(np.asarray(syn.Q_CtoI, float))[0], np.asarray(syn.P_CinI, float)
    poses = []
    for t in (ta, tb):
        qt, pt = est.QueryTrajectory(t)[:2]
        R = st.quat_matrix(qt)
        if camera:
            pt = pt + R @ p_CI
            R = R @ R_CI
        poses.append((R, pt))
    (Ra, pa), (Rb, pb) = poses
    RaT = np.swapaxes(Ra, 1, 2)
    A = np.zeros((len(ta), 6, 12))
    A[:, :3, :3] = -np.swapaxes(RaT @ Rb, 1, 2)
    A[:, 3:, :3] = hat(np.einsum("nij,nj->ni", RaT, pb - pa))
    A[:, 3:, 3:6] = -RaT
    A[:, :3, 6:9] = np.eye(3)
    A[:, 3:, 9:] = RaT
    return joint, A


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["c2", "masked"])
def test_consistent_with_the_pose_covariance(oracle_lib, cuda_lib, rel_jac_lib, name):
    """The joint covariance of the two poses, [[P_a, X], [X', P_b]] from the (dtheta, dp) blocks of PoseCovariance at
    t_a and t_b and cross6, projected through the relative-pose Jacobian built here from QueryTrajectory,
    [A_a A_b] with A_a = [[-R_ab', 0], [[p_ab]x, -R_a']], A_b = [[I, 0], [0, R_a']], is cov6 within rounding."""
    w = case_window(oracle_lib, name)
    est, _ = make_case(cuda_lib, oracle_lib, name)
    est.SetDeterministic(True)
    cov, _, _ = est.Covariance(want_rho=False)
    q, p = est.GetKnots()
    ta, tb = pair_times(w, est.n_knots)
    for camera in (False, True):
        C6, X6, _ = est.RelativePoseCovariance(ta, tb, camera_frame=camera, want_cross=True)
        joint, A = pose_joint_and_relative_jacobian(est, ta, tb, camera, X6)
        G, knots = host_relative_jacobian(rel_jac_lib, q, p, ta, tb, w, camera)
        mag = abs_project(A, joint) + abs_project(G, union_blocks(np.abs(cov), knots))
        err = np.abs(C6 - project(A, joint))
        print(f"{name} camera {camera}: worst |cov6 - A joint A'| / magnitude "
              f"{float((err / np.maximum(mag, 1e-300)).max()):.1e}")
        assert (err <= 1e-12 * mag).all()


@pytest.mark.gpu
def test_constant_knots_and_equal_times(oracle_lib, cuda_lib):
    """masked case (knots 0..12 fixed): a pair whose two segments are <= 9 uses constant knots only and gets exact zero
    matrices (cov6 and cross6); t_a == t_b gives entries below 1e-12 of that pose's covariance."""
    est, _ = make_case(cuda_lib, oracle_lib, "masked")
    est.SetDeterministic(True)
    w = case_window(oracle_lib, "masked")
    t = w.t0_ns + np.arange(14, dtype=np.int64) * w.dt_ns + w.dt_ns // 3
    ta, tb = np.concatenate([t[:10], t[9::-1], t[10:]]), np.concatenate([t[9::-1], t[:10], t[:9:-1]])
    fixed, _ = make_case(cuda_lib, oracle_lib, "c2")
    fixed.SetDeterministic(True)
    te = pair_times(case_window(oracle_lib, "c2"), fixed.n_knots)[0]
    for camera in (False, True):
        C6, X6, _ = est.RelativePoseCovariance(ta, tb, camera_frame=camera, want_cross=True)
        assert not C6[:20].any() and not X6[:20].any()
        assert all(C6[k].any() and X6[k].any() for k in range(20, len(ta)))
        check_psd_symmetric(C6)
        Ce, _, _ = fixed.RelativePoseCovariance(te, te, camera_frame=camera)
        Pe = fixed.PoseCovariance(te, camera_frame=camera)[0][:, :6, :6]
        d = np.sqrt(np.einsum("nii->ni", Pe))
        scale = d[:, :, None] * d[:, None, :]  # 0 on the gauge segment, where cov6 must be exactly 0
        print(f"camera {camera}: t_a == t_b, worst |cov6| / pose scale "
              f"{float((np.abs(Ce) / np.maximum(scale, 1e-300)).max()):.1e}")
        assert (np.abs(Ce) <= 1e-12 * scale).all()


@pytest.mark.gpu
def test_errors_gauge_and_rank_deficiency(oracle_lib, cuda_lib):
    """Every error path leaves the outputs and rcond untouched; n = 0 returns OK; without a gauge the c2 window is rank
    deficient and only rcond is written; with gauge_knot_index = 3 it matches the c2 case, whose options fix knots
    0..3; the whole trajectory as the gauge gives exact zeros."""
    est, _ = make_case(cuda_lib, oracle_lib, "c2")
    f = cuda_lib.lib.ctvio_relative_pose_covariance
    f.argtypes = [P, I32, P, P, I32, I32, P, P, P]
    f.restype = C.c_int
    w = case_window(oracle_lib, "c2")
    t_end = w.t0_ns + (est.n_knots - 3) * w.dt_ns
    ga, gb = np.array([w.t0_ns + 5, t_end - 1], np.int64), np.array([t_end - 1, w.t0_ns + 5], np.int64)
    out, xout = np.full((2, 6, 6), 123.5), np.full((2, 6, 6), 123.5)
    rcond = C.c_double(-7.0)

    def call(h=est.h, n=2, ta=ga, tb=gb, gauge=-1, cam=0, o=out, x=xout):
        return f(h, n, *[None if a is None else a.ctypes.data for a in (ta, tb)], gauge, cam,
                 *[None if a is None else a.ctypes.data for a in (o, x)], C.byref(rcond))
    cases = [
        (dict(h=None), ERR_INVALID), (dict(n=-1), ERR_INVALID), (dict(ta=None), ERR_INVALID),
        (dict(tb=None), ERR_INVALID), (dict(o=None), ERR_INVALID), (dict(cam=2), ERR_INVALID),
        (dict(cam=-1), ERR_INVALID), (dict(gauge=-2), ERR_INVALID), (dict(gauge=est.n_knots), ERR_INVALID),
        (dict(ta=np.array([w.t0_ns - 1, t_end - 1], np.int64)), ERR_TIME_RANGE),
        (dict(tb=np.array([w.t0_ns, t_end], np.int64)), ERR_TIME_RANGE),
    ]
    for kw, code in cases:
        assert call(**kw) == code, kw
        assert (out == 123.5).all() and (xout == 123.5).all() and rcond.value == -7.0, kw
    assert call(n=0, ta=None, tb=None, o=None, x=None) == 0 and rcond.value == -7.0
    assert call(gauge=est.n_knots - 1) == 0  # the whole trajectory constant: every matrix exactly zero
    assert not out.any() and not xout.any()
    cfg = pkg.make_config(**w.config_kwargs())
    bare = pkg.Estimator(cuda_lib, cfg)
    with pytest.raises(pkg.CtvioError, match=r"\(-4\)"):
        bare.RelativePoseCovariance(ga, gb)

    free, _ = make_case(cuda_lib, oracle_lib, "c2", fixed_knot_index=-1)
    fixed, _ = make_case(cuda_lib, oracle_lib, "c2")
    for e in (free, fixed):
        e.SetDeterministic(True)
    ta, tb = pair_times(w, free.n_knots)
    out, xout = np.full((len(ta), 6, 6), 123.5), np.full((len(ta), 6, 6), 123.5)
    rcond = C.c_double(-1.0)
    rc = call(h=free.h, n=len(ta), ta=ta, tb=tb, o=out, x=xout)
    msg = cuda_lib._fn["last_error"]().decode()
    print(f"no gauge: rc {rc}, rcond {rcond.value:.2e}, '{msg}'")
    assert rc == ERR_STATE and "rank deficient" in msg and (out == 123.5).all() and (xout == 123.5).all()
    assert 0.0 <= rcond.value < RCOND_MIN or "pivot" in msg
    for camera in (False, True):
        Cg, Xg, rg = free.RelativePoseCovariance(ta, tb, gauge_knot_index=GAUGE, camera_frame=camera, want_cross=True)
        Cf, Xf, rf = fixed.RelativePoseCovariance(ta, tb, camera_frame=camera, want_cross=True)
        # the scale of each entry: the two poses' joint covariance through the relative-pose Jacobian
        joint, A = pose_joint_and_relative_jacobian(fixed, ta, tb, camera, Xf)
        d = np.sqrt(np.einsum("nii->ni", joint))
        sc, sx = abs_project(A, d[:, :, None] * d[:, None, :]), d[:, :6, None] * d[:, None, 6:]
        print(f"camera {camera}: rcond {rg:.3e} vs {rf:.3e}, worst relative "
              f"{float((np.abs(Cg - Cf) / np.maximum(sc, 1e-300)).max()):.1e} (cov6), "
              f"{float((np.abs(Xg - Xf) / np.maximum(sx, 1e-300)).max()):.1e} (cross6)")
        assert (np.abs(Cg - Cf) <= 1e-12 * sc).all()
        assert (np.abs(Xg - Xf) <= 1e-12 * sx).all()
        assert abs(rg - rf) <= 1e-12 * rf


@pytest.mark.gpu
def test_no_side_effects_and_transfer_counts(oracle_lib, cuda_lib):
    """Deterministic mode: a solve after the call is bitwise the solve without it (C3 window with its prior); the call
    moves 16 n bytes up and 288 n bytes down, 576 n with cross6."""
    runs = []
    w = case_window(oracle_lib, "c3prior")
    for with_cov in (True, False):
        est, _ = make_case(cuda_lib, oracle_lib, "c3prior")
        est.SetDeterministic(True)
        ta, tb = pair_times(w, est.n_knots, 20)
        if with_cov:
            x0 = get_state(est)
            est.RelativePoseCovariance(ta, tb, gauge_knot_index=5, camera_frame=True, want_cross=True)
            x1 = get_state(est)
            assert all(np.array_equal(a, b) for a, b in zip(x0[:4], x1[:4])) and x0[4] == x1[4]
            est.TransferStats(reset=True)
            est.RelativePoseCovariance(ta, tb)
            assert est.TransferStats(reset=True) == (16 * len(ta), 288 * len(ta))
            est.RelativePoseCovariance(ta, tb, want_cross=True)
            assert est.TransferStats() == (16 * len(ta), 576 * len(ta))
        s = est.Solve(8)
        runs.append((s, get_state(est)))
    (s1, x1), (s2, x2) = runs
    for fld in ("iterations", "num_successful_steps", "num_unsuccessful_steps", "termination", "initial_cost",
                "final_cost", "final_radius", "num_linear_solves", "num_jacobian_evals"):
        assert getattr(s1, fld) == getattr(s2, fld), fld
    assert all(np.array_equal(a, b) for a, b in zip(x1[:4], x2[:4])) and x1[4] == x2[4]


@pytest.mark.gpu
def test_runner_publish_odometry_covariance_only_reads(cuda_lib):
    """Six C5 windows, deterministic: with publish_odometry_covariance=True the runner solves, marginalizes and slides
    bitwise as without it, and its records differ only in the new keys, the timings and the call's own transfers.
    Every window clears rcond >= 1e-14 and its consecutive-keyframe covariances are finite, symmetric and PSD."""
    n = 6
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    a = st.ResidentRunner(cuda_lib, seq, triangulate=True, device_features=True)
    b = st.ResidentRunner(cuda_lib, seq, triangulate=True, device_features=True, publish_odometry_covariance=True)
    covs = []
    for x in (a, b):
        x.est.SetDeterministic(True)
        x.est.lib = PriorRecorder(x.est.lib)
    for _ in range(n):
        a.step()
        b.step()
        covs.append(b.last_rel_cov)
    for rec in b.records:
        print(f"window {rec['window']}: rel_cov_rcond {rec['rel_cov_rcond']:.3e}, ms_rel_cov {rec['ms_rel_cov']:.3f}"
              + (f", {rec['rel_cov_error']}" if "rel_cov_error" in rec else ""))
    new = {"rel_cov_rcond", "ms_rel_cov"}
    timing = {"ms", "ms_build_and_predict", "ms_solve", "ms_realign_marginalize", "ms_readback", "device_ms",
              "init_device_ms", "h2d_bytes", "d2h_bytes"}
    assert a.last_rel_cov is None
    for ra, rb, c in zip(a.records, b.records, covs):
        assert set(rb) == set(ra) | new and not new & set(ra)
        for key in set(ra) - timing:
            assert bitwise(ra[key], rb[key]) if isinstance(ra[key], float) else ra[key] == rb[key], key
        m = c.shape[0]
        assert c.shape == (st.WIN_KF - 1, 6, 6) and m == st.WIN_KF - 1
        if ra["window"] > 0:
            assert (rb["h2d_bytes"] - ra["h2d_bytes"], rb["d2h_bytes"] - ra["d2h_bytes"]) == (16 * m, 288 * m)
        assert rb["rel_cov_rcond"] >= RCOND_MIN, rb
        assert np.isfinite(c).all() and (np.einsum("nii->ni", c) > 0).all()
        check_psd_symmetric(c)
    assert bitwise(a.q[:a.ncp], b.q[:b.ncp]) and bitwise(a.p[:a.ncp], b.p[:b.ncp])
    assert bitwise(a.est.GetBiases(), b.est.GetBiases())
    assert bitwise(a.est.GetInvDepths(), b.est.GetInvDepths())
    assert bitwise(a.ld, b.ld)
    pa, pb = a.est.lib.priors, b.est.lib.priors
    assert len(pa) == len(pb) > 0
    assert all(bitwise(x, y) for u, v in zip(pa, pb) for x, y in zip(u, v))
