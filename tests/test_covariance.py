"""ctvio_covariance: the camera-side block of H^-1 and the inverse-depth variances, against fp64 references.

H = [[A, W'], [W, diag(h)]] is the undamped Gauss-Newton matrix of the factor set (A the camera block, W the landmark
couplings, h the landmark diagonals).  The references invert it in numpy over the free dimensions: densely where
np + nL <= 3000, else through the Schur complement S = A - W' diag(1/h) W.  Comparisons run in the Jacobi-scaled
space the engine factors in (K = D H D, D = 1 / (1 + sqrt(diag H))), where the inverse's forward error is bounded by
kappa(K) (4 npad u + 2 eta) |K^-1|_max, eta the normwise difference between the engine's and the oracle's H.

    case        window (test_lm_step_regimes)  options                                np    nb  K5 path (H100)
    c2          c2                             fixed_knot_index 3                     247   4   DAG
    c3prior     C3 window B with its prior     line delay free, fixed_knot_index 3    259   5   DAG
    masked      c2                             knots 0..12 fixed, gyro biases locked  247   4   DAG
    c4          c4                             fixed_knot_index 3                     889   14  DAG
    coop16      coop16                         fixed_knot_index 3                     985   16  barrier kernel

Without fixed knots these windows are rank deficient: yaw and translation are unobservable, and the C3 window's prior
(from the marginalization of the window before it, solved and gauge-realigned) does not pin them either - numerically
its pivot ratio stays below 1e-14 - so that case fixes knots as well.
"""
import ctypes as C
import functools

import numpy as np
import pytest

from helpers import c3_window_a, get_state, pkg, syn
from test_lm_step_regimes import debug_lm_step, regime_window

U = 2.0 ** -53
DENSE_LIMIT = 3000
RCOND_MIN = 1e-14

CASES = {
    # name: (window, options)
    "c2": ("c2", {"fixed_knot_index": 3}),
    "c3prior": ("c3prior", {"fixed_knot_index": 3}),
    "masked": ("c2", {"fixed_knot_index": 12, "lock_wb": True}),
    "c4": ("c4", {"fixed_knot_index": 3}),
    "coop16": ("coop16", {"fixed_knot_index": 3}),
}


# ------------------------------------------------------------------------------------------------------------------
# windows

@functools.lru_cache(maxsize=None)
def c3_prior_inputs(oracle_lib):
    """C3 window B with the prior the oracle marginalizes out of window A (after 15 LM iterations and the gauge
    realignment), at window A's solved state: (window, prior, state)."""
    e, seq, wa, nowk = c3_window_a(oracle_lib)
    R0 = syn.qrot(wa.q0[nowk][None], np.eye(3)).T.copy()
    e.Solve(15)
    e.GaugeRealign(nowk, R0, wa.p0[nowk].copy())
    pr = e.SaveMarginalizationInfo()
    isb = (pr.blk_type == pkg.BLK_BG) | (pr.blk_type == pkg.BLK_BA)
    pr.blk_index[isb] -= 1  # bias nodes are window-relative: the window slides by one keyframe
    wb = syn.subwindow(seq, 1, 11)
    q, p = e.GetKnots()
    b = np.zeros((11, 6)); b[:10] = e.GetBiases()[1:]; b[10] = b[9]
    rho = wb.rho0.copy()
    ga, gb = wa.meta["lm_global"], wb.meta["lm_global"]
    common = np.intersect1d(ga, gb)
    rho[np.searchsorted(gb, common)] = e.GetInvDepths()[np.searchsorted(ga, common)]
    return wb, pr, (q, p, b, rho, e.GetLineDelay())


def case_options(name, w):
    win, opt = CASES[name]
    opt = dict(opt)
    if win == "c3prior":
        opt.update(fix_ld=False, ld_lower=0.0, ld_upper=syn.LD_UPPER)
    else:
        opt.setdefault("fix_ld", w.fix_ld)
        opt.update(ld_lower=w.ld_lower, ld_upper=w.ld_upper)
    return opt


def make_case(lib, oracle_lib, name, **override):
    """The case's estimator on `lib`; override replaces options (e.g. no fixed knots)."""
    win, _ = CASES[name]
    if win == "c3prior":
        w, pr, (q, p, b, rho, ld) = c3_prior_inputs(oracle_lib)
    else:
        w = regime_window(win)
    opt = {**case_options(name, w), **override}
    est = pkg.setup_estimator(lib, w, options=pkg.make_options(**opt))
    if win == "c3prior":
        est.SetKnots(q, p); est.SetBiases(b); est.SetInvDepths(rho); est.SetLineDelay(ld)
        est.AddMarginalizationFactor(pr)
    return est, opt


def const_mask(est, opt):
    """Dims the solve holds constant (ctvio_options rules)."""
    nK, nB = est.n_knots, est.n_bias
    m = np.zeros(6 * (nK + nB) + 1, bool)
    k = opt.get("fixed_knot_index", -1)
    if k >= 0:
        m[:6 * (k + 1)] = True
    for b in range(nB):
        if opt.get("lock_wb"):
            m[6 * nK + 6 * b:6 * nK + 6 * b + 3] = True
        if opt.get("lock_ab"):
            m[6 * nK + 6 * b + 3:6 * nK + 6 * b + 6] = True
    if opt.get("fix_ld"):
        m[-1] = True
    return m


@functools.lru_cache(maxsize=None)
def oracle_case(oracle_lib, name):
    est, opt = make_case(oracle_lib, oracle_lib, name)
    H, g, hl, gl, _ = est.NormalEquations()
    W = np.zeros((est.n_lm, est.np_dim))
    f = oracle_lib.raw("landmark_coupling")
    f.restype = C.c_int
    assert f(est.h, W.ctypes.data_as(C.c_void_p)) == 0
    return dict(A=H, W=W, hl=hl, free=~const_mask(est, opt) & (np.diag(H) > 0))


# ------------------------------------------------------------------------------------------------------------------
# references

def scaled_system(A, W, hl, free):
    """Jacobi scales and the scaled reduced system K_S = D (A - W' diag(1/h) W) D over the free camera dims."""
    sc = 1.0 / (1.0 + np.sqrt(np.maximum(np.diag(A), 0.0)))
    lm = hl > 0
    Wf = W[np.ix_(lm, free)]
    S = A[np.ix_(free, free)] - (Wf / hl[lm, None]).T @ Wf
    d = sc[free]
    return sc, d[:, None] * S * d[None, :]


def reference(s):
    """Sigma_cc (np x np, zero off the free dims), var_rho (diag of H^-1, None above DENSE_LIMIT) and kappa_inf(K)
    of the scaled system they came from, plus K^-1's max entry."""
    A, W, hl, free = s["A"], s["W"], s["hl"], s["free"]
    np_, nL = A.shape[0], len(hl)
    sc, KS = scaled_system(A, W, hl, free)
    cov = np.zeros((np_, np_))
    var = None
    if np_ + nL <= DENSE_LIMIT:
        H = np.block([[A, W.T], [W, np.diag(hl)]])
        keep = np.concatenate([free, hl > 0])
        Hk = H[np.ix_(keep, keep)]
        sf = 1.0 / (1.0 + np.sqrt(np.diag(Hk)))
        K = sf[:, None] * Hk * sf[None, :]
        Kinv = np.linalg.inv(K)
        full = sf[:, None] * Kinv * sf[None, :]
        nf = int(free.sum())
        cov[np.ix_(free, free)] = full[:nf, :nf]
        var = np.zeros(nL)
        var[hl > 0] = np.diag(full)[nf:]
        kappa = np.abs(K).sum(1).max() * np.abs(Kinv).sum(1).max()
    else:
        Kinv = np.linalg.inv(KS)
        d = sc[free]
        cov[np.ix_(free, free)] = d[:, None] * Kinv * d[None, :]
        kappa = np.abs(KS).sum(1).max() * np.abs(Kinv).sum(1).max()
    return dict(cov=cov, var=var, kappa=kappa, sc=sc, KS=KS, kinv_max=np.abs(Kinv).max())


def pivot_rcond(KS):
    """The engine's rank estimate on the reference: (min L_ii / max L_ii)^2 of the Cholesky factor of K_S."""
    try:
        d = np.diag(np.linalg.cholesky(KS))
    except np.linalg.LinAlgError:
        return 0.0
    return float((d.min() / d.max()) ** 2)


# ------------------------------------------------------------------------------------------------------------------
# CPU part

@pytest.mark.parametrize("name", list(CASES))
def test_cases_are_full_rank_and_their_references_agree(oracle_lib, name):
    """Every case has rcond >= 1e-14 on the reference, and the two references (dense H^-1 and the Schur route) agree
    within kappa 50 u on the camera block."""
    s = oracle_case(oracle_lib, name)
    ref = reference(s)
    rc = pivot_rcond(ref["KS"])
    print(f"{name}: np {s['A'].shape[0]}, nL {len(s['hl'])}, kappa_inf {ref['kappa']:.2e}, pivot rcond {rc:.2e}")
    assert rc >= RCOND_MIN
    if ref["var"] is not None:
        free = s["free"]
        d = ref["sc"][free]
        Kinv = np.linalg.inv(ref["KS"])
        err = np.abs(d[:, None] * Kinv * d[None, :] - ref["cov"][np.ix_(free, free)]) / (d[:, None] * d[None, :])
        assert err.max() <= 50 * ref["kappa"] * U * ref["kinv_max"], err.max()


def test_window_without_gauge_is_rank_deficient_on_the_reference(oracle_lib):
    est, opt = make_case(oracle_lib, oracle_lib, "c2", fixed_knot_index=-1)
    H, _, hl, _, _ = est.NormalEquations()
    W = np.zeros((est.n_lm, est.np_dim))
    f = oracle_lib.raw("landmark_coupling")
    f.restype = C.c_int
    assert f(est.h, W.ctypes.data_as(C.c_void_p)) == 0
    _, KS = scaled_system(H, W, hl, ~const_mask(est, opt) & (np.diag(H) > 0))
    assert pivot_rcond(KS) < RCOND_MIN


P, I32 = C.c_void_p, C.c_int32


def test_covariance_rejects_a_null_handle():
    lib = C.CDLL(pkg.load().path)
    lib.ctvio_last_error.restype = C.c_char_p
    lib.ctvio_covariance.argtypes = [P, P, P, P]
    lib.ctvio_covariance.restype = C.c_int
    rcond = C.c_double(-7.0)
    out = np.full(4, -7.0)
    assert lib.ctvio_covariance(None, out.ctypes.data, out.ctypes.data, C.byref(rcond)) == -1  # CTVIO_ERR_INVALID
    assert lib.ctvio_last_error() == b"null handle"
    assert rcond.value == -7.0 and (out == -7.0).all()
    assert lib.ctvio_covariance(None, None, None, None) == -1


def test_binding_exposes_the_covariance():
    assert "covariance" in pkg.ABI_SYMBOLS and "covariance" in pkg.binding.DEVICE_ONLY_SYMBOLS
    assert hasattr(pkg.Estimator, "Covariance")


# ------------------------------------------------------------------------------------------------------------------
# GPU part

def gpu_system(est):
    """The engine's own A, W (line delay in the last column), h_l at the current state (deterministic mode: the same
    sums ctvio_covariance forms)."""
    o = debug_lm_step(est, 1e4)
    return o["A"], o["W"], o["hl"]


def check_against_reference(name, est, s, cov, var):
    ref = reference(s)
    free = s["free"]
    sc = ref["sc"]
    A, W, hl = gpu_system(est)
    A = np.triu(A) + np.triu(A, 1).T
    nL = len(s["hl"])
    # eta: the two assemblies' normwise difference in the scaled space
    dH = np.block([[A - s["A"], (W[:nL] - s["W"]).T], [W[:nL] - s["W"], np.diag(hl[:nL] - s["hl"])]])
    H = np.block([[s["A"], s["W"].T], [s["W"], np.diag(s["hl"])]])
    keep = np.concatenate([free, s["hl"] > 0])
    sf = 1.0 / (1.0 + np.sqrt(np.diag(H)[keep]))
    K = sf[:, None] * H[np.ix_(keep, keep)] * sf[None, :]
    eta = np.abs(sf[:, None] * dH[np.ix_(keep, keep)] * sf[None, :]).sum(1).max() / np.abs(K).sum(1).max()
    npad = (A.shape[0] + 63) // 64 * 64
    bound = ref["kappa"] * (4 * npad * U + 2 * eta) * ref["kinv_max"]
    dd = sc[free][:, None] * sc[free][None, :]
    r_cov = (np.abs(cov[np.ix_(free, free)] - ref["cov"][np.ix_(free, free)]) / dd).max() / bound
    # constant / untouched dims exactly zero, symmetric to the bit
    assert not cov[~free].any() and not cov[:, ~free].any()
    assert np.array_equal(cov, cov.T)
    # self-checks on the engine's own reduced system: |Sigma_s K_S - I|, eigenvalues of Sigma_s
    _, KS = scaled_system(A, W[:nL], hl[:nL], free)
    d = sc[free]
    Ss = cov[np.ix_(free, free)] / (d[:, None] * d[None, :])
    kap_s = np.abs(KS).sum(1).max() * np.abs(Ss).sum(1).max()
    r_id = np.abs(Ss @ KS - np.eye(len(d))).max() / (kap_s * 4 * npad * U)
    lam = np.linalg.eigvalsh(Ss)
    assert lam[0] >= -kap_s * 4 * npad * U * np.abs(Ss).max(), lam[0]
    r_var = 0.0
    if ref["var"] is not None:
        sl = 1.0 / (1.0 + np.sqrt(s["hl"]))
        act = s["hl"] > 0
        r_var = (np.abs(var[:nL] - ref["var"])[act] / sl[act] ** 2).max() / bound
    print(f"{name}: kappa_inf {ref['kappa']:.2e}, eta {eta:.1e}: worst ratio to bound  cov {r_cov:.1e}  var {r_var:.1e}  "
          f"|Sigma S - I| {r_id:.1e}")
    assert r_cov <= 1 and r_var <= 1 and r_id <= 1, (r_cov, r_var, r_id)


def chol_path(lib):
    out = {}
    for key in ("cluster", "plain", "coop"):
        f = getattr(lib.lib, f"ctvio_debug_chol_{key}_launches")
        f.restype = C.c_longlong
        out[key] = f()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_covariance_matches_fp64_reference(oracle_lib, cuda_lib, name):
    """cov_cc and var_rho against the references, rcond >= 1e-14, constant dims and a landmark without factors exactly
    0, two calls bitwise equal (deterministic mode)."""
    s = oracle_case(oracle_lib, name)
    est, opt = make_case(cuda_lib, oracle_lib, name)
    est.SetDeterministic(True)
    nL = est.n_lm
    est.SetInvDepths(np.append(est.GetInvDepths(), 0.3))  # one landmark no factor touches
    before = chol_path(cuda_lib)
    cov, var, rcond = est.Covariance()
    after = chol_path(cuda_lib)
    ran = [k for k in before if after[k] != before[k]]
    print(f"{name}: K5 path {ran}, rcond {rcond:.2e}")
    assert rcond >= RCOND_MIN
    assert var[nL] == 0.0 and np.isfinite(var).all() and (var[:nL][s["hl"] > 0] > 0).all()
    cov2, var2, rcond2 = est.Covariance()
    assert np.array_equal(cov, cov2) and np.array_equal(var, var2) and rcond == rcond2
    cov3, var3, _ = est.Covariance(want_cc=False)
    assert cov3 is None and np.array_equal(var3, var)
    check_against_reference(name, est, s, cov, var)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "coop"])
def test_covariance_is_the_same_on_every_cholesky_path(oracle_lib, cuda_lib, monkeypatch, mode):
    """c2 through the plain tile-DAG launch (CTVIO_CHOL_CLUSTER=0: bitwise the cluster launch) and the barrier kernel
    (CTVIO_CHOL=coop: the other factor layout, held to the reference)."""
    s = oracle_case(oracle_lib, "c2")
    est, _ = make_case(cuda_lib, oracle_lib, "c2")
    est.SetDeterministic(True)
    cov0, var0, rc0 = est.Covariance()
    monkeypatch.setenv("CTVIO_CHOL_CLUSTER" if mode == "plain" else "CTVIO_CHOL", "0" if mode == "plain" else "coop")
    before = chol_path(cuda_lib)
    cov, var, rc = est.Covariance()
    after = chol_path(cuda_lib)
    assert after[mode] == before[mode] + 1, (before, after)
    if mode == "plain":
        assert np.array_equal(cov, cov0) and np.array_equal(var, var0) and rc == rc0
    check_against_reference("c2 " + mode, est, s, cov, var)


@pytest.mark.gpu
def test_rank_deficient_window_fails_and_writes_only_rcond(oracle_lib, cuda_lib):
    est, _ = make_case(cuda_lib, oracle_lib, "c2", fixed_knot_index=-1)
    f = cuda_lib.lib.ctvio_covariance
    f.argtypes = [P, P, P, P]
    f.restype = C.c_int
    cov = np.full((est.np_dim, est.np_dim), 123.5)
    var = np.full(est.n_lm, 123.5)
    rcond = C.c_double(-1.0)
    rc = f(est.h, cov.ctypes.data, var.ctypes.data, C.byref(rcond))
    msg = cuda_lib._fn["last_error"]().decode()
    print(f"rank deficient: rc {rc}, rcond {rcond.value:.2e}, '{msg}'")
    assert rc == -4 and "rank deficient" in msg  # CTVIO_ERR_STATE
    assert 0.0 <= rcond.value < RCOND_MIN or "pivot" in msg
    assert (cov == 123.5).all() and (var == 123.5).all()
    with pytest.raises(pkg.CtvioError, match="rank deficient"):
        est.Covariance()


@pytest.mark.gpu
def test_covariance_has_no_side_effects(oracle_lib, cuda_lib):
    """Deterministic mode: the state after the call is bitwise the state before it, and a following Solve is bitwise
    the Solve without the call (C3 window with its prior: the prior is part of both solves)."""
    runs = []
    for with_cov in (True, False):
        est, _ = make_case(cuda_lib, oracle_lib, "c3prior")
        est.SetDeterministic(True)
        x0 = get_state(est)
        if with_cov:
            est.Covariance()
            x1 = get_state(est)
            for a, b in zip(x0[:4], x1[:4]):
                assert np.array_equal(a, b)
            assert x0[4] == x1[4]
        s = est.Solve(8)
        runs.append((s, get_state(est)))
    (s1, x1), (s2, x2) = runs
    for fld in ("iterations", "num_successful_steps", "num_unsuccessful_steps", "termination", "initial_cost",
                "final_cost", "final_radius", "num_linear_solves", "num_jacobian_evals"):
        assert getattr(s1, fld) == getattr(s2, fld), fld
    for a, b in zip(x1[:4], x2[:4]):
        assert np.array_equal(a, b)
    assert x1[4] == x2[4]


@pytest.mark.gpu
def test_covariance_state_errors_and_transfer_stats(cuda_lib, oracle_lib):
    cfg = pkg.make_config(**regime_window("c2").config_kwargs())
    bare = pkg.Estimator(cuda_lib, cfg)
    with pytest.raises(pkg.CtvioError, match=r"\(-4\)"):
        bare.Covariance()
    est, _ = make_case(cuda_lib, oracle_lib, "c2")
    est.Covariance()
    est.TransferStats(reset=True)
    est.Covariance(want_cc=False, want_rho=False)
    assert est.TransferStats()[1] == 0
    est.Covariance()
    assert est.TransferStats()[1] == 8 * (est.np_dim ** 2 + est.n_lm)
