"""One LM step's linear algebra (K4 Schur reduction, K5 Cholesky + solves, K6 back-substitution) in every regime of the
reduced system, against fp64 references.

The reduced camera system has np = 6 (n_knots + n_bias) + 1 rows (the line delay last), padded to npad = 64 nb.  K4
(scale_copy_kernel + schur_tile_kernel) builds it tile by tile: each 64x64 tile of the lower triangle gets the
landmarks whose knot-dim range touches both of its blocks, cut into parts of `part` landmarks (engine.cu, prepare), and
a CTA reduces its part 32 landmarks (one chunk) at a time.  K5 picks its kernel from nb and the SM count:

    nb (nb + 1) / 2 <= SMs   chol_dag_kernel, one CTA per tile: in clusters of 8 (grid rounded up to a multiple of 8)
                             if the runtime accepts the cluster launch, else a plain cooperative launch
                             (CTVIO_CHOL_CLUSTER=0 forces the plain one)
    otherwise                chol_coop_kernel with grid-wide barriers, grid min(SMs, t0 (t0 + 1) / 2), t0 = nb - 1
                             (CTVIO_CHOL=coop forces it at any size)

Windows: make_window(n_knots, keyframes every 100 ms, tracks of 4 keyframes, seed 5) unless stated; on an H100 SXM
(132 SMs) nb <= 15 takes the tile DAG.

    case        n_knots, n_kf  np    nb  why
    c1          4, 5 (no IMU)  31    1   C1: one tile; the DAG grid of 1 padded to a cluster of 8; no IMU, so a
                                         landmark's observations share one K1 round
    pad1        16, 5          127   2   one padding row
    ld-fixed    23, 9          193   4   the line-delay row alone in the last block (63 padding rows), fixed ...
    ld-free     23, 9          193   4   ... and free
    c2          30, 11         247   4   C2 size: the whole pivot chain in one cluster
    chain5      36, 13         295   5   first block count whose pivot chain (2 nb - 1 CTAs) crosses a cluster
    long        40, 15         331   6   tracks of 12 keyframes: landmarks spanning 3 or more blocks
    masked      30, 11         247   4   knots 0..12 constant (dims 0..77 end inside block 1) and gyro biases locked:
                                         masked dimensions inside blocks
    c4          100, 48        889   14  C4 size, 4 700 landmarks: tiles cut into several parts, parts of several
                                         32-landmark chunks
    dag15       106, 49        931   15  the largest tile-DAG grid (120 CTAs)
    coop16      112, 52        985   16  the barrier kernel chosen automatically
    coop20      140, 66        1237  20  the barrier kernel's grid capped at the SM count

Each case runs at the radii 1e4 (Ceres' initial radius), 1e-3 (heavily damped) and 1e16 (max_radius), through
ctvio_debug_lm_step (engine.cu), which returns every stage's inputs and outputs.  The CPU part pins the numpy
references: the numpy Schur step from the oracle's normal equations equals the dense full-system step.
"""
import ctypes as C
import functools

import numpy as np
import pytest

from helpers import get_state, pkg, syn

U = 2.0 ** -53
RADII = (1e4, 1e-3, 1e16)
H100_SMS = 132          # the CPU part's structure assertions; the GPU part reads the SM count of its device
DENSE_LIMIT = 3000      # np + nL up to which the dense full-system reference is formed
KF0 = syn.KF_OFFSET_NS

REGIMES = {
    # name: (n_knots, n_kf, landmarks anchored per keyframe, track length, options, np, nb)
    "c1": (4, 5, None, 4, {}, 31, 1),
    "pad1": (16, 5, 40, 4, {}, 127, 2),
    "ld-fixed": (23, 9, 30, 4, {}, 193, 4),
    "ld-free": (23, 9, 30, 4, {"fix_ld": False}, 193, 4),
    "c2": (30, 11, 30, 4, {}, 247, 4),
    "chain5": (36, 13, 25, 4, {}, 295, 5),
    "long": (40, 15, 15, 12, {}, 331, 6),
    "masked": (30, 11, 30, 4, {"fixed_knot_index": 12, "lock_wb": True}, 247, 4),
    "c4": (100, 48, 100, 4, {}, 889, 14),
    "dag15": (106, 49, 10, 4, {}, 931, 15),
    "coop16": (112, 52, 10, 4, {}, 985, 16),
    "coop20": (140, 66, 8, 4, {}, 1237, 20),
}


def gamma(k):
    k = np.asarray(k, float)
    return k * U / (1.0 - k * U)


@functools.lru_cache(maxsize=None)
def regime_window(name):
    n_knots, n_kf, per, track, opt, _, _ = REGIMES[name]
    if name == "c1":
        return syn.config_c1()
    kf = KF0 + np.arange(n_kf, dtype=np.int64) * 100_000_000
    return syn.make_window(name, n_knots, kf, [per] * (n_kf - 1) + [0], track, seed=5,
                           fix_ld=opt.get("fix_ld", True))


def regime_options(name):
    w = regime_window(name)
    opt = dict(REGIMES[name][4])
    opt.setdefault("fix_ld", w.fix_ld)
    return pkg.make_options(ld_lower=w.ld_lower, ld_upper=w.ld_upper, **opt)


def const_mask(name):
    """The constant camera dims of the case (trajectory_estimator.cpp rules, as ctvio_set_options applies them)."""
    w = regime_window(name)
    opt = REGIMES[name][4]
    nK, nB = w.n_knots, w.bias0.shape[0]
    m = np.zeros(6 * (nK + nB) + 1, bool)
    k = opt.get("fixed_knot_index", -1)
    if k >= 0:
        m[:6 * (k + 1)] = True
    for b in range(nB):
        if opt.get("lock_wb"):
            m[6 * nK + 6 * b:6 * nK + 6 * b + 3] = True
    if opt.get("fix_ld", w.fix_ld):
        m[-1] = True
    return m


def knot_ranges(w):
    """Per landmark the knot-dim range [lo, hi) of its coupling row: the padded knot windows of all its observation
    times (engine.cu, prepare)."""
    nK = w.n_knots
    smax, maxt = nK - 4, w.t0_ns + (nK - 3) * w.dt_ns

    def window(t):
        s1 = (t - w.t0_ns) // w.dt_ns
        t2 = t + w.rs_padding_ns
        s2 = np.where(t2 >= maxt, smax, (t2 - w.t0_ns) // w.dt_ns)
        return s1, np.minimum(s2 + 3, nK - 1)

    fi, li = window(w.ti)
    fj, lj = window(w.tj)
    nL = len(w.rho0)
    lo = np.full(nL, np.iinfo(np.int64).max)
    hi = np.zeros(nL, np.int64)
    np.minimum.at(lo, w.lm, 6 * np.minimum(fi, fj))
    np.maximum.at(hi, w.lm, 6 * (np.maximum(li, lj) + 1))
    return lo, hi


def schur_structure(name, n_sm):
    """K4's work list as prepare() builds it: per tile the landmarks touching both blocks, cut into parts."""
    w = regime_window(name)
    np_ = 6 * (w.n_knots + w.bias0.shape[0]) + 1
    npad = (np_ + 63) // 64 * 64
    T = npad // 64
    lo, hi = knot_ranges(w)
    count = np.zeros((T, T), np.int64)
    span = 0
    for l0, h0 in zip(lo, hi):
        b0, b1 = l0 // 64, (h0 - 1) // 64
        span = max(span, b1 - b0 + 1)
        for x in range(b0, b1 + 1):
            count[x, b0:x + 1] += 1
    total = int(count.sum())
    part = max(32, ((total // (2 * n_sm) + 31) // 32) * 32)
    tiles = count[np.tril_indices(T)]
    items = int(sum((c + part - 1) // part for c in tiles))
    return dict(np=np_, npad=npad, nb=T, part=part, items=items, max_parts=int(max((c + part - 1) // part for c in tiles)),
                max_chunks=int(min(int(tiles.max()), part) + 31) // 32, max_span=span, lo=lo, hi=hi)


# ------------------------------------------------------------------------------------------------------------------
# references

def sym_upper(a):
    return np.triu(a) + np.triu(a, 1).T


def clamp_diag(m):
    return np.clip(m, 1e-6, 1e32)


@functools.lru_cache(maxsize=None)
def oracle_system(oracle_lib, name):
    """The oracle's normal equations and landmark couplings at the window's initial state."""
    o = pkg.setup_estimator(oracle_lib, regime_window(name), options=regime_options(name))
    H, g, hl, gl, _ = o.NormalEquations()
    W = np.zeros((o.n_lm, o.np_dim))
    f = oracle_lib.raw("landmark_coupling")
    f.restype = C.c_int
    assert f(o.h, W.ctypes.data_as(C.c_void_p)) == 0
    return dict(A=H, gc=g, hl=hl, gl=gl, W=W)


def full_system_step(s, free, radius):
    """Dense LM step over [free camera dims | landmarks] without Schur: Jacobi scaling, clamped damping.  Rows that no
    factor touches (zero diagonal) are left out: their step is 0.  Returns (delta camera, delta landmarks, kappa_inf)."""
    A, W, hl, gc, gl = s["A"], s["W"], s["hl"], s["gc"], s["gl"]
    np_, nL = A.shape[0], len(hl)
    H = np.block([[A, W.T], [W, np.diag(hl)]])
    g = np.concatenate([gc, gl])
    keep = np.concatenate([free, np.ones(nL, bool)]) & (np.diag(H) > 0)
    Hk, gk = H[np.ix_(keep, keep)], g[keep]
    sc = 1.0 / (1.0 + np.sqrt(np.diag(Hk)))
    K = sc[:, None] * Hk * sc[None, :]
    K[np.diag_indices_from(K)] += clamp_diag(np.diag(K)) / radius
    Kinv = np.linalg.inv(K)
    d = np.zeros(np_ + nL)
    d[keep] = -sc * (Kinv @ (sc * gk))
    kappa = np.abs(K).sum(1).max() * np.abs(Kinv).sum(1).max()
    return d[:np_], d[np_:], kappa, (keep, sc, K)


def schur_step(s, free, radius):
    """The same step through the Schur complement onto the camera dims (numpy fp64, the formulas of kernels_linear.cu)."""
    A, W, hl, gc, gl = s["A"], s["W"], s["hl"], s["gc"], s["gl"]
    np_ = A.shape[0]
    cam = free & (np.diag(A) > 0)
    sc = np.where(cam, 1.0 / (1.0 + np.sqrt(np.maximum(np.diag(A), 0))), 0.0)
    sl = 1.0 / (1.0 + np.sqrt(hl))
    M = sc[:, None] * A * sc[None, :]
    M[np.diag_indices(np_)] += clamp_diag(np.diag(M)) / radius
    hs = sl * sl * hl
    hh = hs + clamp_diag(hs) / radius
    V = (sl / np.sqrt(hh))[:, None] * W * sc[None, :]
    lc = sl / np.sqrt(hh) * gl
    M = M - V.T @ V
    rhs = sc * gc - V.T @ lc
    y = np.zeros(np_)
    y[cam] = np.linalg.solve(M[np.ix_(cam, cam)], rhs[cam])
    dc = -sc * y
    wy = W @ (sc * y)
    dl = -sl * (sl * gl - sl * wy) / hh
    return dc, dl


# ------------------------------------------------------------------------------------------------------------------
# CPU part

@pytest.mark.parametrize("name", list(REGIMES))
def test_window_structure_puts_the_reduced_system_in_its_regime(name):
    st = schur_structure(name, H100_SMS)
    assert (st["np"], st["nb"]) == REGIMES[name][5:], (st["np"], st["nb"])
    assert st["npad"] == 64 * st["nb"]
    print(f"{name}: np {st['np']}, nb {st['nb']}, part {st['part']}, {st['items']} K4 items, "
          f"<= {st['max_parts']} parts per tile, <= {st['max_chunks']} chunks per part, landmarks span <= {st['max_span']} blocks")
    if name in ("ld-fixed", "ld-free"):
        assert st["np"] % 64 == 1  # the line-delay row alone in the last block
    if name == "masked":
        m = const_mask(name)
        assert m[:78].all() and not m[78] and 64 < 78 < 128       # the knot mask ends inside block 1
        assert any(m[i] != m[i - 1] for i in range(1, len(m)) if i % 64)


def test_regimes_cover_multi_part_tiles_multi_chunk_parts_and_long_landmarks():
    st = {n: schur_structure(n, H100_SMS) for n in REGIMES}
    assert any(s["max_parts"] > 1 for s in st.values())
    assert st["c4"]["max_chunks"] > 1 and st["c4"]["max_parts"] > 1
    assert st["long"]["max_span"] >= 3
    assert {s["nb"] for s in st.values()} >= {1, 2, 4, 5, 14, 15, 16, 20}


@pytest.mark.parametrize("name", [n for n in REGIMES if n != "c4"])
def test_numpy_schur_step_equals_full_system_step(oracle_lib, name):
    """The references the GPU is held to, pinned against each other: from the oracle's A, W, h_l, g, the numpy Schur
    step equals the dense full-system step within max(1e-10, 50 kappa u) (relative, max norm).  The oracle's coupling
    rows live inside the knot ranges K4's work lists assume."""
    s = oracle_system(oracle_lib, name)
    free = ~const_mask(name)
    lo, hi = knot_ranges(regime_window(name))
    cols = np.arange(s["W"].shape[1])
    outside = (cols[None, :] < lo[:, None]) | ((cols[None, :] >= hi[:, None]) & (cols[None, :] != len(cols) - 1))
    assert not (s["W"] * outside).any()
    assert not s["A"][~free].any() and not s["W"][:, ~free].any()   # constant dims have no Jacobian columns
    for radius in RADII:
        dc_f, dl_f, kappa, _ = full_system_step(s, free, radius)
        dc_s, dl_s = schur_step(s, free, radius)
        ref = np.concatenate([dc_f, dl_f])
        err = np.abs(np.concatenate([dc_s, dl_s]) - ref).max() / np.abs(ref).max()
        bound = max(1e-10, 50 * kappa * U)
        print(f"{name} radius {radius:g}: kappa {kappa:.1e}, Schur vs full {err:.1e} (bound {bound:.1e})")
        assert err <= bound, (radius, err, bound)


# ------------------------------------------------------------------------------------------------------------------
# GPU part

def device_sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def chol_counters(lib):
    out = {}
    for key in ("cluster", "plain", "coop"):
        f = getattr(lib.lib, f"ctvio_debug_chol_{key}_launches")
        f.restype = C.c_longlong
        out[key] = f()
    return out


def debug_lm_step(est, radius):
    f = est.lib.lib.ctvio_debug_lm_step
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.POINTER(C.c_int64)]
    n = C.c_int64(0)
    assert f(est.h, radius, None, C.byref(n)) == 0
    buf = np.full(n.value, np.nan)
    before = chol_counters(est.lib)
    rc = f(est.h, radius, buf.ctypes.data, C.byref(n))
    assert rc == 0, est.lib._fn["last_error"]()
    after = chol_counters(est.lib)
    ran = [k for k in before if after[k] != before[k]]
    assert len(ran) == 1 and after[ran[0]] == before[ran[0]] + 1, (before, after)
    np_, npad, nL = int(buf[0]), int(buf[1]), int(buf[2])
    o = {"np": np_, "npad": npad, "nL": nL, "items": int(buf[3]), "gd": buf[4], "dHd": buf[5], "dir_max": buf[6],
         "chol_fail": int(buf[7]), "path": ran[0], "raw": buf}
    pos = 16
    for key, shape in (("A", (np_, np_)), ("gc", np_), ("hl", nL), ("gl", nL), ("W", (nL, np_)), ("cmask", np_),
                       ("sc", np_), ("sl", nL), ("hh", nL), ("M", (npad, npad)), ("rhs", npad), ("y", npad),
                       ("dc", np_), ("dl", nL)):
        size = int(np.prod(shape))
        o[key] = buf[pos:pos + size].reshape(shape)
        o[key + "_off"] = pos
        pos += size
    assert pos == len(buf)
    o["free"] = o["cmask"] == 0
    return o


def worst(err, bound):
    """max err / bound; entries with a zero bound must be exact"""
    z = bound == 0
    assert not err[z].any()
    return float((err[~z] / bound[~z]).max()) if (~z).any() else 0.0


def check_k4(o, ranges, radius):
    """K4 against its own inputs: M = S A S + clamp(diag)/radius - sum_l v_l v_l', v_l = sl / sqrt(hh) W_l S, and
    rhs = S g_c - sum_l v_l is_l g_l, formed in extended precision.  |M - M_ref| <= gamma_{k+4} (|S||A||S| + D +
    sum_l |v_l||v_l|') element by element, k = landmarks in the entry: true for any summation order."""
    np_, npad, nL, free = o["np"], o["npad"], o["nL"], o["free"]
    ld = np_ - 1
    L = np.longdouble
    sc = np.where(free, o["sc"], 0.0)
    A = sym_upper(o["A"])
    # hh: the damped landmark diagonal, same operations as scale_copy_kernel
    hs = o["sl"] * o["sl"] * o["hl"]
    hh_ref = np.where(o["hl"] > 0, hs + clamp_diag(hs) / radius, 0.0)
    assert np.all(np.abs(o["hh"] - hh_ref) <= 2 * U * np.abs(hh_ref)), "hh"
    SAS = (sc[:, None] * A) * sc[None, :]
    D = np.where(free, clamp_diag(np.diag(SAS)) / radius, 0.0)
    Mref = (sc[:, None].astype(L) * A.astype(L)) * sc[None, :].astype(L)
    Mref[np.diag_indices(np_)] += D
    B = np.abs(SAS) + np.diag(D)
    K = np.zeros((np_, np_), np.int64)
    rhs_ref = sc.astype(L) * o["gc"].astype(L)
    rB = np.abs(sc * o["gc"])
    rK = np.zeros(np_, np.int64)
    lo, hi = ranges
    isl = np.where(o["hh"] > 0, o["sl"].astype(L) / np.sqrt(o["hh"].astype(L)), 0)
    for l in range(nL):
        idx = np.concatenate([np.arange(lo[l], hi[l]), [ld]])
        v = isl[l] * o["W"][l, idx].astype(L) * sc[idx].astype(L)
        ix = np.ix_(idx, idx)
        Mref[ix] -= np.multiply.outer(v, v)
        av = np.abs(v.astype(float))
        B[ix] += np.multiply.outer(av, av)
        K[ix] += 1
        c = isl[l] * L(o["gl"][l])
        rhs_ref[idx] -= v * c
        rB[idx] += av * abs(float(c))
        rK[idx] += 1
    M, rhs = o["M"], o["rhs"]
    lower = np.tril(np.ones((np_, np_), bool))
    both = free[:, None] & free[None, :] & lower
    err = np.abs(M[:np_, :np_] - Mref.astype(float))
    r_m = worst(err[both], gamma(K[both] + 4) * B[both])
    r_r = worst(np.abs(rhs[:np_] - rhs_ref.astype(float))[free], gamma(rK[free] + 4) * rB[free])
    # padding rows and constant dims: exactly the identity / zero (bitwise: no -0.0 either)
    bits = M.view(np.int64)
    one = np.float64(1.0).view(np.int64)
    fixed = np.concatenate([~free, np.ones(npad - np_, bool)])
    lower_pad = np.tril(np.ones((npad, npad), bool))
    rows = fixed[:, None] & lower_pad
    cols = fixed[None, :] & lower_pad
    want = np.where(np.eye(npad, dtype=bool), one, 0)
    assert np.array_equal(bits[rows], want[rows]) and np.array_equal(bits[cols], want[cols])
    assert np.array_equal(rhs.view(np.int64)[fixed], np.zeros(fixed.sum(), np.int64))
    return r_m, r_r


def lower_sym(M):
    return np.tril(M) + np.tril(M, -1).T


def check_k5(o, Msym, Minv_norm):
    """Normwise backward error <= npad u (residual in extended precision); padding exactly 0; forward error against
    numpy's Cholesky solve within 4 kappa npad u.  Returns (backward ratio, forward ratio, kappa, numpy solution)."""
    npad = o["npad"]
    y, rhs = o["y"], o["rhs"]
    L = np.longdouble
    res = (Msym.astype(L) @ y.astype(L) - rhs.astype(L)).astype(float)
    nM = np.abs(Msym).sum(1).max()
    back = np.abs(res).max() / (nM * np.abs(y).max() + np.abs(rhs).max())
    assert np.array_equal(y[o["np"]:].view(np.int64), np.zeros(npad - o["np"], np.int64))
    import scipy.linalg
    try:
        y_np = scipy.linalg.cho_solve(scipy.linalg.cho_factor(Msym, lower=True), rhs)
    except np.linalg.LinAlgError:  # numerically singular (max_radius without a gauge prior): kappa makes the bound loose
        y_np = np.linalg.solve(Msym, rhs)
    kappa = nM * Minv_norm
    fwd = np.abs(y - y_np).max() / np.abs(y_np).max()
    return back / (npad * U), fwd / (4 * kappa * npad * U), kappa, y_np


def check_k6(o, ranges):
    """dc bitwise = -sc o y on free dims and 0 on constant ones; dl against the back-substitution formula on the GPU's
    y (extended precision, gamma_{k+6} componentwise); g'd and d'Hd over the full Hessian within gamma_n bounds."""
    np_, nL, free = o["np"], o["nL"], o["free"]
    y, sc, dc, dl = o["y"][:np_], o["sc"], o["dc"], o["dl"]
    assert np.array_equal(dc[free], -(sc[free] * y[free])) and not dc[~free].any()
    L = np.longdouble
    sy = np.where(free, sc * y, 0.0)
    W = o["W"]
    wy = W.astype(L) @ sy.astype(L)
    sl, gl, hh, hl = o["sl"], o["gl"], o["hh"], o["hl"]
    dl_ref = -sl.astype(L) * (sl.astype(L) * gl - sl.astype(L) * wy) / hh.astype(L)
    k = (W != 0).sum(1)
    bnd = gamma(k + 6) * np.abs(sl) * (np.abs(sl * gl) + np.abs(sl) * (np.abs(W) @ np.abs(sy))) / hh
    r_dl = worst(np.abs(dl - dl_ref.astype(float)), bnd)
    g = np.concatenate([o["gc"], gl])
    d = np.concatenate([dc, dl])
    n = np_ + nL
    gd_ref = float((g.astype(L) * d.astype(L)).sum())
    r_gd = abs(o["gd"] - gd_ref) / (gamma(n) * np.abs(g) @ np.abs(d))
    A = sym_upper(o["A"])
    dHd_ref = float(dc.astype(L) @ (A.astype(L) @ dc.astype(L)) + 2 * (dl.astype(L) @ (W.astype(L) @ dc.astype(L)))
                    + (hl.astype(L) * dl.astype(L) ** 2).sum())
    hb = np.abs(dc) @ (np.abs(A) @ np.abs(dc)) + 2 * np.abs(dl) @ (np.abs(W) @ np.abs(dc)) + (np.abs(hl) * dl ** 2).sum()
    r_dhd = abs(o["dHd"] - dHd_ref) / (gamma(n) * hb)
    assert o["dir_max"] == max(np.abs(dc).max(), np.abs(dl).max(), 0.0)
    return r_dl, r_gd, r_dhd


def check_assembly(o, s):
    """GPU A, g_c, h_l, g_l, W (with wld) against the oracle at the same state, at the tolerances of
    test_normal_equations_match_oracle."""
    A = sym_upper(o["A"])
    for key, g_, ref, rtol in (("A", A, s["A"], 1e-9), ("W", o["W"], s["W"], 1e-9), ("gc", o["gc"], s["gc"], 1e-8),
                               ("hl", o["hl"], s["hl"], 1e-10), ("gl", o["gl"], s["gl"], 1e-8)):
        atol = (1e-11 if key in ("A", "W") else 1e-10) * np.abs(ref).max()
        assert np.allclose(g_, ref, rtol=rtol, atol=atol), (key, np.abs(g_ - ref).max() / np.abs(ref).max())
    H = np.block([[A, o["W"].T], [o["W"], np.diag(o["hl"])]])
    Ho = np.block([[s["A"], s["W"].T], [s["W"], np.diag(s["hl"])]])
    return H, Ho


def expected_k5(nb, n_sm, mode):
    if mode == "coop" or nb * (nb + 1) // 2 > n_sm:
        return {"coop"}
    return {"plain"} if mode == "plain" else {"cluster", "plain"}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(REGIMES))
def test_lm_step_regime_matches_fp64_references(oracle_lib, cuda_lib, name, monkeypatch):
    """Every stage of one LM step against its reference (see the check_* functions) at the three radii: in deterministic
    mode for the default K5 path, the plain tile-DAG launch and the barrier kernel (cluster and plain DAG bitwise equal,
    DAG and barrier kernel within the forward bound), two deterministic calls bitwise equal at every stage, a default-mode
    call within the same bounds, and the full step against a dense full-system solve of the oracle's normal equations
    where np + nL <= 3000: relative error <= max(1e-10, kappa (50 u + 2 eta)), eta the normwise difference between the
    two assemblies.  The K5 path is asserted from launch counters, the number of K4 work items from the window."""
    n_sm = device_sm_count()
    st = schur_structure(name, n_sm)
    s = oracle_system(oracle_lib, name)
    w = regime_window(name)
    g = pkg.setup_estimator(cuda_lib, w, options=regime_options(name))
    ranges = (st["lo"], st["hi"])
    report = []
    for radius in RADII:
        outs = {}
        monkeypatch.delenv("CTVIO_CHOL", raising=False)
        monkeypatch.delenv("CTVIO_CHOL_CLUSTER", raising=False)
        g.SetDeterministic(False)
        nondet = debug_lm_step(g, radius) if radius == RADII[0] else None
        g.SetDeterministic(True)
        for mode in ("default", "plain", "coop"):
            monkeypatch.delenv("CTVIO_CHOL", raising=False)
            monkeypatch.delenv("CTVIO_CHOL_CLUSTER", raising=False)
            if mode == "plain":
                if expected_k5(st["nb"], n_sm, "default") == {"coop"}:
                    continue
                monkeypatch.setenv("CTVIO_CHOL_CLUSTER", "0")
            if mode == "coop":
                monkeypatch.setenv("CTVIO_CHOL", "coop")
            outs[mode] = debug_lm_step(g, radius)
            assert outs[mode]["path"] in expected_k5(st["nb"], n_sm, mode), (mode, outs[mode]["path"])
        monkeypatch.delenv("CTVIO_CHOL", raising=False)
        monkeypatch.delenv("CTVIO_CHOL_CLUSTER", raising=False)
        o = outs["default"]
        assert (o["np"], o["npad"], o["items"]) == (st["np"], st["npad"], st["items"])
        assert np.array_equal(o["free"], ~const_mask(name))
        if radius == RADII[0]:
            again = debug_lm_step(g, radius)
            assert np.array_equal(again["raw"], o["raw"]), "deterministic mode: two calls differ"
        for mode, x in outs.items():  # the evaluation and K4 do not depend on the K5 path
            assert np.array_equal(x["raw"][16:x["y_off"]], o["raw"][16:o["y_off"]]), mode
        H, Ho = check_assembly(o, s)
        r_m, r_r = check_k4(o, ranges, radius)
        Msym = lower_sym(o["M"])
        Minv_norm = np.abs(np.linalg.inv(Msym)).sum(1).max()
        lam_min = np.linalg.eigvalsh(Msym)[0]
        if o["chol_fail"]:
            # only a numerically singular system may fail (the damping at max_radius is at the rounding level)
            assert lam_min <= o["npad"] * U * np.abs(Msym).sum(1).max(), (radius, lam_min)
            report.append(f"radius {radius:g}: K4 {r_m:.2f}/{r_r:.2f}; K5 reported a non-positive pivot "
                          f"(lambda_min {lam_min:.1e}): numerically singular, not checked further")
            continue
        ratios = {}
        for mode, x in outs.items():
            b, f, kappa, y_np = check_k5(x, Msym, Minv_norm)
            assert b <= 1 and f <= 1, (mode, b, f, kappa)
            ratios[mode] = (b, f)
        if "plain" in outs:
            assert np.array_equal(outs["plain"]["raw"], o["raw"]), "cluster and plain DAG launches differ"
        r_dl, r_gd, r_dhd = check_k6(o, ranges)
        assert r_dl <= 1 and r_gd <= 1 and r_dhd <= 1, (r_dl, r_gd, r_dhd)
        if nondet is not None:
            check_assembly(nondet, s)
            nm, nr = check_k4(nondet, ranges, radius)
            nb_, nf, _, _ = check_k5(nondet, lower_sym(nondet["M"]), np.abs(np.linalg.inv(lower_sym(nondet["M"]))).sum(1).max())
            ndl, ngd, ndhd = check_k6(nondet, ranges)
            assert max(nm, nr, nb_, nf, ndl, ngd, ndhd) <= 1, (nm, nr, nb_, nf, ndl, ngd, ndhd)
        e2e = ""
        if o["np"] + o["nL"] <= DENSE_LIMIT:
            dc_f, dl_f, kappa_f, (keep, sf, K) = full_system_step(s, o["free"], radius)
            eta = np.abs(sf[:, None] * (H - Ho)[np.ix_(keep, keep)] * sf[None, :]).sum(1).max() / np.abs(K).sum(1).max()
            ref = np.concatenate([dc_f, dl_f])
            err = np.abs(np.concatenate([o["dc"], o["dl"]]) - ref).max() / np.abs(ref).max()
            bound = max(1e-10, kappa_f * (50 * U + 2 * eta))
            assert err <= bound, (radius, err, bound, kappa_f, eta)
            e2e = f", full system {err / bound:.2f} (kappa {kappa_f:.1e})"
        paths = "/".join(sorted({x["path"] for x in outs.values()}))
        report.append(f"radius {radius:g}: K5 {paths}; K4 M {r_m:.2f} rhs {r_r:.2f}; "
                      + ", ".join(f"K5 {m} back {b:.2f} fwd {f:.2e}" for m, (b, f) in ratios.items())
                      + f"; K6 dl {r_dl:.2f} gd {r_gd:.2f} dHd {r_dhd:.2f}{e2e}")
    print(f"\n{name} (np {st['np']}, nb {st['nb']}, {n_sm} SMs, part {st['part']}, {st['items']} K4 items): worst ratio to bound")
    for line in report:
        print("  " + line)


def _perturbed_c1(seed, scale):
    w = syn.config_c1()
    rng = np.random.default_rng(seed)
    w.p0 = w.p0 + scale * rng.standard_normal(w.p0.shape)
    w.rho0 = w.rho0 * np.exp(np.clip(scale * rng.standard_normal(w.rho0.shape), -3, 3))
    return w


@pytest.mark.gpu
@pytest.mark.parametrize("speculation", ["always", "never"])
def test_deterministic_mode_is_bitwise_reproducible_on_far_start_c1(cuda_lib, monkeypatch, speculation):
    """C1 started far from the optimum (the window of test_lm_driver_with_rejected_steps_matches_oracle), deterministic
    mode, Solve(12) twice: equal summaries and bit-identical states.  All of C1's keyframes lie in one knot interval, so
    the four observations of a landmark share one visual-kernel round; their landmark sums must still be added in one
    fixed order.  (Deterministic mode always takes the plain driver; the speculation switch must not matter.)"""
    monkeypatch.setenv("CTVIO_SPECULATION", speculation)
    runs = []
    for _ in range(2):
        g = pkg.setup_estimator(cuda_lib, _perturbed_c1(4, 5.0))
        g.SetDeterministic(True)
        s = g.Solve(12)
        runs.append((s, get_state(g)))
    (s1, x1), (s2, x2) = runs
    for f in ("iterations", "num_successful_steps", "num_unsuccessful_steps", "termination", "initial_cost",
              "final_cost", "final_radius", "num_linear_solves", "num_jacobian_evals", "kernel_launches"):
        assert getattr(s1, f) == getattr(s2, f), f
    for a, b in zip(x1[:4], x2[:4]):
        assert np.array_equal(a, b)
    assert x1[4] == x2[4]
