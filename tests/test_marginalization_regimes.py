"""The marginalization (K7, ctvio_marginalize) in every regime of its eigen-solver, against fp64 references.

launch_jacobi_eig (csrc/marginalize.cu) picks its code path from the matrix size n, and runs twice per marginalization:
on the dropped block Amm (size m) and on the Schur complement (size n).  With the rotation log ctvio_marginalize passes:

    n          path
    1-15       jacobi_eig_block_kernel<true> (A in shared memory) + jacobi_apply_log_kernel
    16-128     jacobi_blocked_kernel + jacobi_blocked_apply_kernel (jacobi_blocked.cu; 8-wide blocks, their count
               rounded up to even: n = 113..128 pad to 16 blocks, which still fit one SM's shared memory).
               CTVIO_JACOBI=elementwise takes the row above / below instead.
    129-168    jacobi_eig_block_kernel<true> + replay (the padded matrix and the pair table fit 224 KiB)
    169-312    jacobi_eig_block_kernel<false> (A in global memory) + replay; the replay stages 16 rounds of the log
               in shared memory, above the 48 KiB default from n = 245 on
    >= 313     jacobi_eig_kernel: no log, V accumulated in place (the per-thread block table of the logged kernel
               holds n <= 312)

(a) the eigen-solver alone (ctvio_debug_eig, the same launcher) against LAPACK at both sides of every boundary;
(b) the whole marginalization against the CPU oracle on windows whose dropped size m and kept size n sit in chosen
    regimes; (c) the oracle itself against a numpy dense pseudo-inverse Schur complement on the same windows, so that a
    mismatch in (b) cannot come from the oracle.
"""
import ctypes as C
import functools
import types

import numpy as np
import pytest

from helpers import dense_jacobian, pkg, syn

# ------------------------------------------------------------------------------------------------------------------
# (a) the eigen-solver alone

SIZES = [1, 2, 3, 7, 15, 16, 17, 24, 25, 33, 111, 112, 113, 128, 129, 167, 168, 169, 244, 245, 246, 300, 312, 313, 400]
FAMILIES = ["separated", "rank_deficient", "clustered", "diagonal", "zero", "negative_definite"]


def expected_path(n, mode):
    if mode == "default" and 16 <= n <= 128:
        return "blocked"
    return "logged" if n <= 312 else "nolog"


def eig_case(n, family, seed):
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    if family == "separated":     # unit gaps over [-n/2, n/2]: every eigenvector is well defined
        ev = np.arange(n) - n // 2 + rng.uniform(-0.25, 0.25, n)
    elif family == "rank_deficient":  # what a streaming prior looks like: a few directions at the rounding floor
        ev = 10.0 ** rng.uniform(-6, 6, n)
        k = min(6, n)
        ev[:k] = 10.0 ** rng.uniform(-14, -10, k) * rng.choice([-1.0, 1.0], k)
    elif family == "clustered":   # exactly repeated eigenvalues (triples) and clusters 1e-12 apart
        base = 10.0 ** rng.uniform(-2, 2, (n + 2) // 3)
        ev = np.repeat(base, 3)[:n]
        ev[1::3] *= 1.0 + 1e-12
    elif family == "diagonal":    # nothing to rotate: zero rotations logged, V = I
        return np.diag(rng.uniform(-3, 3, n))
    elif family == "zero":
        return np.zeros((n, n))
    elif family == "negative_definite":
        ev = -(10.0 ** rng.uniform(-3, 3, n))
    a = (q * ev) @ q.T
    return 0.5 * (a + a.T)


def debug_eig(cuda_lib, a):
    n = a.shape[0]
    f = cuda_lib.lib.ctvio_debug_eig
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    a = np.ascontiguousarray(a)
    v, ev = np.zeros((n, n)), np.zeros(n)
    rc = f(n, a.ctypes.data, v.ctypes.data, ev.ctypes.data, 0)
    return rc, v, ev


def debug_counters(cuda_lib):
    """n of the last decomposition of the element-wise logged kernel and of the blocked kernel (the no-log kernel
    writes neither)."""
    out = {}
    for key, sym in (("logged", "ctvio_debug_jacobi"), ("blocked", "ctvio_debug_jacobi_blocked")):
        buf = (C.c_int * 8)()
        assert getattr(cuda_lib.lib, sym)(buf) == 0
        out[key] = buf[1]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("n", SIZES)
def test_eigen_solver_regimes_match_lapack(cuda_lib, n, family, monkeypatch):
    """Every code path of launch_jacobi_eig at both sides of each boundary, against LAPACK (numpy.linalg.eigh, fp64):
    return code, sorted eigenvalues, V'V = I, V diag(ev) V' = A, eigenvectors of the separated family up to sign,
    bit-identical repeated runs.  Tolerances: 1e-13 |A| for the eigenvalues, 1e-12 for orthogonality and (relative to
    |A|) reconstruction, widened linearly above n = 128 (n / 128 times as many rotations act on every entry).
    Measured worst cases on an H100 (eigenvalues / V'V / reconstruction): 1-15 1e-15 / 2e-15 / 2e-15; blocked 7e-14 /
    8e-14 / 2e-14; logged 16-312 1.3e-14 / 1.0e-14 / 2e-15; no-log (313, 400) 1.5e-13 / 2.4e-13 / 5e-14; separated
    eigenvectors 1 - |v . v_lapack| <= 5e-15."""
    a = eig_case(n, family, seed=1000 * n + FAMILIES.index(family))
    scale = max(np.linalg.norm(a, 2), 1e-300)
    ref_ev, ref_v = np.linalg.eigh(a)
    grow = max(1.0, n / 128)
    for mode in ("default", "elementwise") if 16 <= n <= 128 else ("default",):
        if mode == "elementwise":
            monkeypatch.setenv("CTVIO_JACOBI", "elementwise")
        path = expected_path(n, mode)
        if path == "nolog":  # this kernel writes no counter: make sure a stale one cannot read n
            assert debug_eig(cuda_lib, np.eye(2))[0] == 0
        rc, v, ev = debug_eig(cuda_lib, a)
        assert rc == 0, (mode, rc)
        cnt = debug_counters(cuda_lib)
        if path == "nolog":
            assert cnt["logged"] == 2 and cnt["blocked"] != n, (mode, cnt)
        else:
            assert cnt[path] == n, (mode, path, cnt)
        rc2, v2, ev2 = debug_eig(cuda_lib, a)
        assert rc2 == 0 and np.array_equal(v, v2) and np.array_equal(ev, ev2), mode
        if family in ("diagonal", "zero"):  # exact: no rotation at all
            assert np.array_equal(ev, np.diag(a)) and np.array_equal(v, np.eye(n)), mode
            continue
        order = np.argsort(ev)
        ev_err = np.abs(ev[order] - ref_ev).max() / scale
        orth = np.abs(v.T @ v - np.eye(n)).max()
        rec = np.abs((v * ev) @ v.T - a).max() / scale
        vec = (1.0 - np.abs(np.einsum("ij,ij->j", v[:, order], ref_v))).max() if family == "separated" else 0.0
        print(f"n={n} {family} {path}: eigenvalues {ev_err:.1e}, V'V {orth:.1e}, V S V' {rec:.1e}, vectors {vec:.1e}")
        assert ev_err <= 1e-13 * grow, (mode, ev_err)
        assert orth <= 1e-12 * grow, (mode, orth)
        assert rec <= 1e-12 * grow, (mode, rec)
        assert vec <= 1e-10, (mode, vec)


# ------------------------------------------------------------------------------------------------------------------
# (b), (c) the whole marginalization on windows built for a chosen (m, n)
#
# Windows follow config_c3_sequence: keyframes every 100 ms from 31 ms, control points every 50 ms, landmarks anchored
# in keyframe 0 only and observed in the next `track` keyframes, and keyframe 0's factors flagged for marginalization
# the way c3_window_a flags them (its landmarks' image factors, the IMU samples before keyframe 1, bias factor 0).  So
# m = 12 (control points 0, 1) + 6 (bias node 0) + landmarks, and n = 6 (control points 2 .. 2 track + 4) + 6 + 1.
# Amm is well conditioned on these windows once its rows and columns are scaled to unit diagonal (condition number ~8;
# unscaled ~1e10 from the units alone), so the pseudo-inverse is the inverse and the references are well defined.
#
# Not covered here, and why: m = 0 cannot occur (every recorded factor drops a block: an image factor its inverse depth,
# an IMU sample its bias node, a bias factor its first node, an old prior only takes part when it has a dropped block);
# n < 16 needs all control points but the last dropped, and then Amm is singular to ~1e-10 (scaled) along the common
# accelerometer bias / vertical acceleration direction, so no two implementations agree on the prior.  The n < 16 solver
# path is covered by (a).

MARG_CASES = {
    # name: (landmarks in keyframe 0, track length, control points, expected m, expected n)
    "m68-n61": (50, 3, 11, 68, 61),           # both blocked
    "m268-n73": (250, 4, 13, 268, 73),        # Amm through the logged kernel with A in global memory + 61 KiB replay
    "m358-n61": (340, 3, 11, 358, 61),        # Amm through the no-log kernel, the prior through the blocked one
    "m150-n169": (132, 12, 29, 150, 169),     # Amm with A in shared memory, the prior with A in global memory
    "m10-n43": (10, 1, 8, 10, 43),            # small Amm (diagonal: one inverse depth per landmark), blocked prior
}


@functools.lru_cache(maxsize=None)
def marg_case(name):
    lms, track, n_knots, _, _ = MARG_CASES[name]
    n_kf = track + 1
    kf = syn.KF_OFFSET_NS + np.arange(n_kf, dtype=np.int64) * 100_000_000
    w = syn.make_window(name, n_knots, kf, [lms] + [0] * (n_kf - 1), track, seed=syn.SEED0 + 70 + lms, fix_ld=False)
    if name == "m10-n43":   # image factors only, no control point dropped
        img = np.ones(w.n_obs, np.int32); imu = np.zeros(len(w.imu_t), np.int32); bias = np.zeros(len(w.bf_i), np.int32)
        nowk = later = 0
    else:
        img = (w.anchor_frame[w.lm] == 0).astype(np.int32)
        imu = (w.imu_t < w.kf_times[1]).astype(np.int32)
        bias = np.zeros(len(w.bf_i), np.int32); bias[0] = 1
        later = int((w.kf_times[1] - w.t0_ns) // w.dt_ns)
        nowk = int((w.kf_times[0] - w.t0_ns) // w.dt_ns)
    return types.SimpleNamespace(name=name, w=w, img=img, imu=imu, bias=bias, nowk=nowk, later=later)


def marg_dims(c):
    """(m, n) from the window's structure alone: the parameter blocks the flagged factors touch (an image factor its
    padded knot windows at both frame times, an IMU sample its 4 control points, a bias factor two bias nodes) and the
    rule that drops control points < later, the bias nodes of IMU samples and of a bias factor's first node, and every
    flagged landmark."""
    w = c.w
    smax = w.n_knots - 4
    knots = set()
    fi = c.img.astype(bool)
    for t in np.unique(np.concatenate([w.ti[fi], w.tj[fi]])):
        s1 = (int(t) - w.t0_ns) // w.dt_ns
        s2 = min((int(t) + w.rs_padding_ns - w.t0_ns) // w.dt_ns, smax)
        knots.update(range(s1, s2 + 4))
    fm = c.imu.astype(bool)
    for s in np.unique((w.imu_t[fm] - w.t0_ns) // w.dt_ns):
        knots.update(range(int(s), int(s) + 4))
    fb = c.bias.astype(bool)
    bias_drop = set(w.imu_node[fm].tolist()) | set(w.bf_i[fb].tolist())
    bias_keep = set(w.bf_j[fb].tolist()) - bias_drop
    dk = sum(1 for k in knots if c.later > c.nowk and k < c.later)
    m = 6 * dk + 6 * len(bias_drop) + len(np.unique(w.lm[fi]))
    n = 6 * (len(knots) - dk) + 6 * len(bias_keep) + (1 if fi.any() else 0)
    return m, n


def marg_estimator(lib, c):
    opt = pkg.make_options(fix_ld=False, ld_lower=0.0, ld_upper=syn.LD_UPPER, is_marg_state=True,
                           ctrl_to_be_opt_now=c.nowk, ctrl_to_be_opt_later=c.later)
    return pkg.setup_estimator(lib, c.w, image_marg=c.img, imu_marg=c.imu, bias_marg=c.bias, options=opt)


def dense_schur(e, c, pr):
    """numpy restatement of the marginalization from the factor probes at e's state (Cauchy scale 1 for image factors):
    A = J'J, b = J'r over the flagged factors, dense pseudo-inverse Schur complement onto the prior's columns."""
    w = c.w
    Jd, rd = dense_jacobian(e, w, cauchy=1.0)
    npd, nK = e.np_dim, e.n_knots
    rows = np.concatenate([np.repeat(c.img.astype(bool), 2), np.repeat(c.imu.astype(bool), 6),
                           np.repeat(c.bias.astype(bool), 6)])
    J, r = Jd[rows], rd[rows]
    A, b = J.T @ J, J.T @ r
    drop = np.zeros(npd + e.n_lm, bool)
    if c.later > c.nowk:
        drop[:6 * c.later] = True
    fm, fb = c.imu.astype(bool), c.bias.astype(bool)
    for node in set(w.imu_node[fm].tolist()) | set(w.bf_i[fb].tolist()):
        drop[6 * nK + 6 * node:6 * nK + 6 * node + 6] = True
    drop[npd + np.unique(w.lm[c.img.astype(bool)])] = True
    used = np.abs(J).sum(0) > 0
    col_of = {}
    for t, i, cc in zip(pr.blk_type, pr.blk_index, pr.blk_col):
        base = {0: 6 * i, 1: 6 * i + 3, 2: 6 * nK + 6 * i, 3: 6 * nK + 6 * i + 3, 4: npd - 1}[int(t)]
        for d in range(1 if t == 4 else 3):
            col_of[base + d] = cc + d
    keep = np.array(sorted(col_of, key=lambda g: col_of[g]))
    di = np.nonzero(drop & used)[0]
    # (a padded knot window can reach a control point the factor's Jacobian is zero on: kept, but not `used`)
    assert not drop[keep].any() and set(np.nonzero(used & ~drop)[0]) <= set(keep)
    Amm = A[np.ix_(di, di)]
    Amr = A[np.ix_(di, keep)]
    Ainv = np.linalg.pinv(0.5 * (Amm + Amm.T), rcond=1e-15, hermitian=True)
    d = 1.0 / np.sqrt(np.diag(Amm))
    evs = np.linalg.eigvalsh(Amm * d[:, None] * d[None, :])  # condition number net of the units of the blocks
    return dict(Ap=A[np.ix_(keep, keep)] - Amr.T @ Ainv @ Amr, bp=b[keep] - Amr.T @ Ainv @ b[di], m=len(di), n=len(keep),
                scaled_cond=evs[-1] / evs[0])


@functools.lru_cache(maxsize=None)
def _oracle_prior(oracle_lib, name):
    c = marg_case(name)
    o = marg_estimator(oracle_lib, c)
    pr = o.SaveMarginalizationInfo()
    assert pr is not None
    return o, pr


@pytest.mark.parametrize("name", list(MARG_CASES))
def test_window_structure_puts_m_and_n_in_their_regimes(name):
    assert marg_dims(marg_case(name)) == MARG_CASES[name][3:]


@pytest.mark.parametrize("name", list(MARG_CASES))
def test_oracle_marginalization_equals_dense_schur(oracle_lib, name):
    """The oracle's SaveMarginalizationInfo against the numpy dense pseudo-inverse Schur complement, at the windows the
    GPU is compared on below (Amm well conditioned there, so the pseudo-inverse is the inverse)."""
    c = marg_case(name)
    o, pr = _oracle_prior(oracle_lib, name)
    ref = dense_schur(o, c, pr)
    assert (ref["m"], ref["n"]) == marg_dims(c) == (ref["m"], pr.n)
    assert 0 < ref["scaled_cond"] < 1e3, ref["scaled_cond"]
    JtJ, Jtr = pr.J.T @ pr.J, pr.J.T @ pr.r
    sc = np.abs(ref["Ap"]).max()
    assert np.abs(JtJ - ref["Ap"]).max() <= 1e-7 * sc, np.abs(JtJ - ref["Ap"]).max() / sc
    assert np.abs(Jtr - ref["bp"]).max() <= 1e-7 * np.abs(ref["bp"]).max()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(MARG_CASES))
def test_marginalization_regimes_match_oracle(oracle_lib, cuda_lib, name):
    """ctvio_marginalize against the oracle at the same state, with m and n in the regimes named by the case: block list
    exactly, linearisation points, J'J and J'r at 1e-7 of their largest entry (J_lin and r_lin themselves are only
    defined up to an orthogonal factor, and the eps = 1e-30 pseudo-inverse makes r_lin noise / sqrt(noise) along
    rounding-level eigen-directions).  Both decompositions ran on the intended kernels, and a second marginalization
    from the same state is bit-identical.  Measured on an H100: J'J <= 4e-13, J'r <= 1.3e-11 of the largest entry."""
    c = marg_case(name)
    o, po = _oracle_prior(oracle_lib, name)
    m, n = MARG_CASES[name][3:]
    g = marg_estimator(cuda_lib, c)
    q, p = o.GetKnots()
    g.SetKnots(q, p); g.SetBiases(o.GetBiases()); g.SetInvDepths(o.GetInvDepths()); g.SetLineDelay(o.GetLineDelay())
    pg = g.SaveMarginalizationInfo()
    assert pg is not None and pg.n == po.n == n
    want = {}
    for k in (m, n):  # the counters hold the size of the last decomposition each kernel ran
        if expected_path(k, "default") != "nolog":
            want[expected_path(k, "default")] = k
    cnt = debug_counters(cuda_lib)
    assert all(cnt[key] == v for key, v in want.items()), (want, cnt)
    assert np.array_equal(pg.blk_type, po.blk_type) and np.array_equal(pg.blk_index, po.blk_index)
    assert np.array_equal(pg.blk_col, po.blk_col) and np.allclose(pg.blk_x0, po.blk_x0, rtol=0, atol=1e-15)
    Ag, Ao = pg.J.T @ pg.J, po.J.T @ po.J
    bg, bo = pg.J.T @ pg.r, po.J.T @ po.r
    err_A = np.abs(Ag - Ao).max() / np.abs(Ao).max()
    err_b = np.abs(bg - bo).max() / np.abs(bo).max()
    print(f"{name}: J'J {err_A:.2e}, J'r {err_b:.2e} of the largest entry")
    assert err_A <= 1e-7 and err_b <= 1e-7, (err_A, err_b)
    pg2 = g.SaveMarginalizationInfo()
    assert np.array_equal(pg.J, pg2.J) and np.array_equal(pg.r, pg2.r)
