"""The factor kernels' normal-equation assembly (K1 visual_kernel<true>, K2 imu_kernel<true>, K3 small_factors_kernel +
prior_add_jtj_kernel) entry by entry against an extended-precision J'J, in every regime of their work lists.

Reference.  Every factor's residual and Jacobian come from the oracle's per-factor probes (EvalImageFactors with the
Cauchy corrector of the solve, EvalImuFactors) or, for the bias factors and the prior, from their formulas restated in
numpy.  With the constant mask of the options applied to the columns, the rows are accumulated block-sparsely in
np.longdouble (x86 80-bit): for each set of factors that share their camera columns, [J r]'[J r] by one matmul, scattered
into A | g; per row, J_rho [J r] into the landmark's W | wld | g_l and J_rho^2 into h_l.  Alongside, with the same
index sets (a column that a factor reaches twice, e.g. through two aliased knot windows, counts twice):

    C_ij = sum_r |J_ri| |J_rj|        m_ij = the number of such terms        E_ij = sum_r ||J_r||_inf (|J_ri| + |J_rj|)

(the residual is column np of A | g, ||J_r||_inf includes it and J_rho).  Any summation order of the device's terms
in fp64 is within gamma_{m+2} C of the exact sum; the device's rows differ from the oracle's by at most tau ||J_r||_inf
per entry, tau = 1e-9 (the probe parity tests' tolerance), which moves a product by at most tau E.  So

    |X_gpu - X_ref|_ij <= gamma_{m_ij + 2} C_ij + tau E_ij        for X = A, g, h_l, g_l, W, wld,

and an entry with C_ij = 0 (constant dims, dims no factor reaches) is exactly 0 on the device.  A mis-mapped, dropped,
doubled or unmasked contribution is off by the order of C_ij, about 1e9 bounds.  The cost: gamma_{N+2} sum |c_f| +
tau sum_f ||r_f||_inf ||r_f||_1 + gamma_3 b per image factor (the rounding of 1 + s / b and the log, b = cauchy^2).

Regimes (windows from synthetic.make_window; image factors added per (anchor time, observation time) pair, projected
through the ground-truth spline; nothing has to be consistent with the initial state, only the assembly is checked):

    one-factor      one image factor and one IMU sample: K1 item of count 1, K2 item of count 1 (odd: the next
                    sample's rows zeroed)
    same-window     C1: every keyframe in one knot interval, wi0 == wj0 (every local pair aliased, doubled diagonal);
                    4 knots, so the window is also clipped at the spline end
    overlap         anchor / observation windows 1, 2, 3, 4 and 5 or more knots apart
    spline-ends     frames in the first and the last interval, one whose padded time passes maxt (smax clamp): TMA
                    copies of 4 knots / 3 knot pairs
    global-shutter  no rolling-shutter padding: slot always 0, the fifth window knot unused
    ld-zero         line delay free at 0 ...
    ld-upper        ... and at its upper bound, rows up to 1023: observations evaluated in slot 1 through the delay
    chunk-64        groups of 129, 256 and 257 in a window of few groups: the cap halved to 64, equal chunks
    chunk-128       70 groups of 128: more than one chunk per SM at cap 64, so the cap stays 128 (items of exactly 128)
    outliers        10 % of the observations moved 5-50 px, at the ground-truth state: Cauchy weights of the moved ones
                    < 0.2 among inliers at the noise level
    imu-1khz        1 kHz samples: runs of 50 (items 32 + 18) and of 33 (32 + 1)
    imu-nodes       bias-node changes inside knot intervals, samples at t0, at knot times (u = 0) and at maxt - 1,
                    handed over out of time order
    masks-fixed     fixed_knot_index ending inside knot windows, lock_ab
    masks-traj      lock_traj, lock_wb, line delay free
    prior           a 61-dim prior with rotation, position, gyro-bias, accel-bias and line-delay blocks, some on constant
                    dims, and bias factors under lock_wb

The CPU part pins the reference against the oracle's own assembly (tau = 0: both use the oracle's Jacobians) and the
numpy restatements of the K1 / K2 work-item rules, and checks that each case reaches its regime at 132 SMs.  The GPU
part checks deterministic mode (two calls bitwise equal) and default mode against the reference, and the device's
work items against the same rules at its SM count.
"""
import ctypes as C
import functools

import numpy as np
import pytest

from helpers import pkg, syn
from test_lm_step_regimes import H100_SMS, debug_lm_step, device_sm_count, gamma

L = np.longdouble
TAU = 1e-9
MS = 1_000_000
KF0 = syn.KF_OFFSET_NS
CAUCHY = 2.0
VIS_CAP, VIS_MIN_CHUNK, IMU_CAP = 128, 64, 32  # kVisObsPerRound, kVisMinChunk, kImuMaxPerItem (kernels.h)
ROW_MAX_LD_NS = int(syn.LD_UPPER * 1e9)


# ------------------------------------------------------------------------------------------------------------------
# windows

def base_window(name, n_knots, kf, seed, **kw):
    """knots, biases, 200 Hz IMU and bias factors of make_window, no image factors"""
    w = syn.make_window(name, n_knots, np.asarray(kf, np.int64), [0] * len(kf), 1, seed=seed, **kw)
    w.meta["rng"] = np.random.default_rng(seed + 1000)
    return w


def max_t(w):
    return w.t0_ns + (w.n_knots - 3) * w.dt_ns


def row_cap(w, t):
    """largest row whose time stays inside the spline at any line delay up to LD_UPPER"""
    return np.minimum(1023, (max_t(w) - 1 - np.asarray(t, np.int64)) // ROW_MAX_LD_NS).astype(np.int32)


def add_obs(w, pairs, per_lm=4):
    """pairs of (anchor time, observation time, count): count observations of count / per_lm new landmarks, anchored at
    a random bearing and depth, projected into the observation time through the ground-truth spline (+ pixel noise)"""
    rng = w.meta["rng"]
    gs = w.rs_padding_ns == 0
    ld_ns = np.int64(int(w.ld_gt * 1e9))
    cols = {k: [getattr(w, k)] for k in ("ti", "rowi", "pi", "tj", "rowj", "pj", "lm")}
    rho_gt, rho0 = [w.rho_gt], [w.rho0]
    l0 = len(w.rho0)
    for ta, tb, count in pairs:
        nl = -(-count // per_lm)
        x, y = rng.uniform(-0.8, 0.8, nl), rng.uniform(-0.6, 0.6, nl)
        depth = rng.uniform(2.0, 10.0, nl)
        ra = np.zeros(nl, np.int32) if gs else np.minimum(syn._row_of(y), row_cap(w, ta))
        qa, pa = syn.spline_pose(w.q_gt, w.p_gt, ta + ra.astype(np.int64) * ld_ns, w.t0_ns, w.dt_ns)
        pG = syn.qrot(qa, syn.qrot(syn.Q_CtoI[None], np.stack([x, y, np.ones(nl)], -1) * depth[:, None]) + syn.P_CinI) + pa
        xy, rb = project(w, pG, tb, ld_ns, gs)
        k = np.repeat(np.arange(nl), per_lm)[:count]
        noise = lambda: rng.normal(0, 1 / 740, (count, 2))
        cols["ti"].append(np.full(count, ta, np.int64)); cols["rowi"].append(ra[k]); cols["pi"].append(np.stack([x, y], -1)[k] + noise())
        cols["tj"].append(np.full(count, tb, np.int64)); cols["rowj"].append(rb[k]); cols["pj"].append(xy[k] + noise())
        cols["lm"].append((l0 + k).astype(np.int32))
        rho_gt.append(1 / depth); rho0.append(1 / depth * (1 + rng.normal(0, 0.1, nl)))
        l0 += nl
    for key, v in cols.items():
        setattr(w, key, np.ascontiguousarray(np.concatenate(v).astype(v[0].dtype)))
    w.rho_gt, w.rho0 = np.concatenate(rho_gt), np.concatenate(rho0)
    return w


def project(w, pG, t, ld_ns, gs):
    """rolling-shutter projection at frame time t, rows kept inside the spline (fixed-point iteration on the row)"""
    cap = row_cap(w, t)
    row = np.zeros(len(pG), np.int32) if gs else np.full(len(pG), min(512, int(cap)), np.int32)
    for _ in range(1 if gs else 4):
        q, p = syn.spline_pose(w.q_gt, w.p_gt, t + row.astype(np.int64) * ld_ns, w.t0_ns, w.dt_ns)
        pC = syn.qrot(syn.qconj(syn.Q_CtoI)[None], syn.qrot(syn.qconj(q), pG - p) - syn.P_CinI)
        xy = pC[:, :2] / pC[:, 2:3]
        if not gs:
            row = np.minimum(syn._row_of(xy[:, 1]), cap)
    return xy, row


def set_imu(w, t, rng, order=None):
    """replace the IMU samples by samples at times t (gyro / accel from the ground truth + noise)"""
    t = np.asarray(t, np.int64)
    om, a, _ = syn.spline_imu(w.q_gt, w.p_gt, t, w.t0_ns, w.dt_ns)
    qi, _ = syn.spline_pose(w.q_gt, w.p_gt, t, w.t0_ns, w.dt_ns)
    acc = syn.qrot(syn.qconj(qi), a + syn.GRAVITY)
    node = np.clip(np.searchsorted(w.kf_times, t, side="right") - 1, 0, len(w.kf_times) - 1).astype(np.int32)
    w.bf_sqrt_info = syn.bias_sqrt_info(t, w.kf_times)
    o = np.arange(len(t)) if order is None else order
    w.imu_t, w.imu_gyro = t[o], (om + rng.normal(0, syn.SIGMA_G, om.shape))[o]
    w.imu_accel, w.imu_node = (acc + rng.normal(0, syn.SIGMA_A, acc.shape))[o], node[o]
    return w


def kf_every(n, step_ms, offset=KF0):
    return offset + np.arange(n, dtype=np.int64) * step_ms * MS


def case_one_factor():
    kf = kf_every(3, 100)
    w = add_obs(base_window("one-factor", 12, kf, 11), [(kf[0], kf[1], 1)])
    w.imu_t, w.imu_gyro, w.imu_accel, w.imu_node = w.imu_t[[9]], w.imu_gyro[[9]], w.imu_accel[[9]], w.imu_node[[9]]
    w.bf_i, w.bf_j, w.bf_sqrt_info = w.bf_i[:0], w.bf_j[:0], w.bf_sqrt_info[:0]
    return w, {}


def case_same_window():
    return syn.config_c1(), {}


def case_overlap():
    kf = kf_every(9, 50)
    pairs = [(kf[i], kf[i + d], 24) for i in (0, 2) for d in range(1, 7)]
    return add_obs(base_window("overlap", 16, kf, 12), pairs), {}


def case_spline_ends():
    n_knots = 10
    mt = (n_knots - 3) * syn.DT_NS
    kf = np.array([5 * MS, 100 * MS, 200 * MS, mt - 45 * MS, mt - 20 * MS], np.int64)
    w = base_window("spline-ends", n_knots, kf, 13)
    return add_obs(w, [(kf[0], kf[1], 20), (kf[0], kf[3], 20), (kf[1], kf[4], 20), (kf[3], kf[4], 20), (kf[4], kf[3], 20),
                       (kf[4], kf[0], 8)]), {}


def case_global_shutter():
    kf = kf_every(6, 100)
    w = base_window("global-shutter", 14, kf, 14, global_shutter=True)
    return add_obs(w, [(kf[i], kf[j], 30) for i, j in ((0, 1), (0, 3), (1, 2), (2, 5), (4, 5))]), {}


def _ld_window(name, seed):
    kf = kf_every(6, 100)
    w = base_window(name, 14, kf, seed, fix_ld=False)
    w = add_obs(w, [(kf[i], kf[j], 40) for i, j in ((0, 1), (0, 2), (1, 3), (2, 4), (3, 5))])
    top = np.arange(w.n_obs) % 3 == 0  # a third of the rows at the bottom of the image
    w.rowi = np.where(top, row_cap(w, w.ti), w.rowi).astype(np.int32)
    w.rowj = np.where(top, row_cap(w, w.tj), w.rowj).astype(np.int32)
    return w


def case_ld_zero():
    return _ld_window("ld-zero", 15), {"fix_ld": False, "ld": 0.0}


def case_ld_upper():
    return _ld_window("ld-upper", 16), {"fix_ld": False, "ld": syn.LD_UPPER}


def case_chunk_64():
    kf = kf_every(5, 100)
    return add_obs(base_window("chunk-64", 14, kf, 17), [(kf[0], kf[1], 129), (kf[0], kf[2], 256), (kf[1], kf[3], 257)]), {}


def case_chunk_128():
    kf = kf_every(20, 50)
    pairs = [(kf[i], kf[i + d], 128) for i in range(20) for d in range(1, 5) if i + d < 20]
    return add_obs(base_window("chunk-128", 24, kf, 18), pairs), {}


def case_outliers():
    kf = kf_every(11, 100)
    w = syn.make_window("outliers", 30, kf, [60, 60, 60] + [0] * 8, 4, seed=19)
    rng = np.random.default_rng(19)
    k = rng.choice(w.n_obs, w.n_obs // 10, replace=False)
    ang = rng.uniform(0, 2 * np.pi, len(k))
    px = rng.uniform(5, 50, len(k)) / syn.FY
    w.pj = w.pj.copy()
    w.pj[k] += px[:, None] * np.stack([np.cos(ang), np.sin(ang)], -1)
    w.meta["moved"] = k
    return w, {"state": "gt"}  # at the ground truth only the moved observations are far from the noise level


def case_imu_1khz():
    kf = kf_every(6, 100, offset=33 * MS)   # node changes 33 ms into intervals 2, 4, ...: runs of 33 + 17
    w = base_window("imu-1khz", 14, kf, 20)
    w = set_imu(w, np.arange(0, max_t(w), MS), w.meta["rng"])
    return add_obs(w, [(kf[0], kf[1], 30), (kf[1], kf[3], 30)]), {}


def case_imu_nodes():
    kf = np.array([31, 131, 175, 231, 340, 420], np.int64) * MS
    w = base_window("imu-nodes", 14, kf, 21)
    t = np.concatenate([np.arange(0, max_t(w), 5 * MS), [max_t(w) - 1]])
    w = set_imu(w, t, w.meta["rng"], order=w.meta["rng"].permutation(len(t)))
    return add_obs(w, [(kf[0], kf[2], 30), (kf[2], kf[4], 30)]), {}


def case_masks_fixed():
    kf = kf_every(8, 100)
    w = syn.make_window("masks-fixed", 24, kf, [30, 30, 30, 30, 0, 0, 0, 0], 4, seed=22)
    return w, {"fixed_knot_index": 12, "lock_ab": True}


def case_masks_traj():
    kf = kf_every(8, 100)
    w = syn.make_window("masks-traj", 24, kf, [30, 30, 30, 0, 0, 0, 0, 0], 4, seed=23, fix_ld=False)
    return w, {"lock_traj": True, "lock_wb": True, "fix_ld": False, "ld": 21e-6}


def case_prior():
    kf = kf_every(6, 100)
    w = syn.make_window("prior", 16, kf, [30, 30, 0, 0, 0, 0], 4, seed=24, fix_ld=False)
    rng = np.random.default_rng(24)
    types, index, x0 = [], [], []
    for k in range(6):
        types += [pkg.BLK_ROT, pkg.BLK_POS]; index += [k, k]
        x0.append(syn.qmul(w.q0[k], syn.qexp(rng.normal(0, 0.01, 3))))
        x0.append(np.append(w.p0[k] + rng.normal(0, 0.01, 3), 0.0))
    for b in range(4):
        types += [pkg.BLK_BG, pkg.BLK_BA]; index += [b, b]
        x0.append(np.append(w.bias0[b, :3] + rng.normal(0, 1e-3, 3), 0.0))
        x0.append(np.append(w.bias0[b, 3:] + rng.normal(0, 1e-3, 3), 0.0))
    types.append(pkg.BLK_LD); index.append(0); x0.append([w.ld0 + 2e-6, 0, 0, 0])
    sizes = [1 if t == pkg.BLK_LD else 3 for t in types]
    col = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int32)
    n = int(sum(sizes))
    J = rng.normal(0, 1, (n, n)) * np.exp(rng.uniform(-3, 3, n))[None, :] + 20 * np.eye(n)
    w.meta["prior"] = pkg.PriorData(n=n, J=J, r=rng.normal(0, 1, n), blk_type=np.array(types, np.int32),
                                    blk_index=np.array(index, np.int32), blk_col=col, blk_x0=np.array(x0, float))
    return w, {"fixed_knot_index": 2, "lock_wb": True, "fix_ld": False, "ld": w.ld0}


CASES = {
    "one-factor": case_one_factor, "same-window": case_same_window, "overlap": case_overlap,
    "spline-ends": case_spline_ends, "global-shutter": case_global_shutter, "ld-zero": case_ld_zero,
    "ld-upper": case_ld_upper, "chunk-64": case_chunk_64, "chunk-128": case_chunk_128, "outliers": case_outliers,
    "imu-1khz": case_imu_1khz, "imu-nodes": case_imu_nodes, "masks-fixed": case_masks_fixed,
    "masks-traj": case_masks_traj, "prior": case_prior,
}


@functools.lru_cache(maxsize=None)
def case(name):
    w, opt = CASES[name]()
    opt = dict(opt)
    ld = opt.pop("ld", None)
    w.meta["state"] = opt.pop("state", "init")
    opt.setdefault("fix_ld", w.fix_ld)
    return w, opt, ld


def make_estimator(lib, name):
    w, opt, ld = case(name)
    e = pkg.setup_estimator(lib, w, state=w.meta["state"],
                            options=pkg.make_options(ld_lower=w.ld_lower, ld_upper=w.ld_upper, **opt))
    if ld is not None:
        e.SetLineDelay(ld)
    if "prior" in w.meta:
        e.AddMarginalizationFactor(w.meta["prior"])
    return e


def const_mask(name):
    """constant camera dims (trajectory_estimator.cpp rules as prepare applies them)"""
    w, opt, _ = case(name)
    nK, nB = w.n_knots, w.bias0.shape[0]
    m = np.zeros(6 * (nK + nB) + 1, bool)
    if opt.get("lock_traj"):
        m[:6 * nK] = True
    k = opt.get("fixed_knot_index", -1)
    if k >= 0:
        m[:6 * (k + 1)] = True
    for b in range(nB):
        m[6 * nK + 6 * b:6 * nK + 6 * b + 3] |= bool(opt.get("lock_wb"))
        m[6 * nK + 6 * b + 3:6 * nK + 6 * b + 6] |= bool(opt.get("lock_ab"))
    m[-1] = opt["fix_ld"]
    return m


# ------------------------------------------------------------------------------------------------------------------
# work-item rules (engine.cu, prepare)

def knot_window(w, t):
    s1 = (np.asarray(t, np.int64) - w.t0_ns) // w.dt_ns
    t2 = np.asarray(t, np.int64) + w.rs_padding_ns
    s2 = np.where(t2 >= max_t(w), w.n_knots - 4, (t2 - w.t0_ns) // w.dt_ns)
    return s1, s2


def visual_items(w, n_sm):
    """K1 items (start, count, wi0, wj0): frame-pair groups in (wi0, wj0) order, the cap halved from 128 while all chunks
    at half the cap still fit on the SMs (down to 64), each group cut into equal chunks"""
    wi0, _ = knot_window(w, w.ti)
    wj0, _ = knot_window(w, w.tj)
    keys, counts = np.unique(np.stack([wi0, wj0], 1), axis=0, return_counts=True)
    cap = VIS_CAP
    while cap // 2 >= VIS_MIN_CHUNK and sum(-(-c // (cap // 2)) for c in counts) <= n_sm:
        cap //= 2
    items, start = [], 0
    for (a, b), c in zip(keys, counts):
        per = -(-c // -(-c // cap))
        items += [(s, min(per, start + c - s), a, b) for s in range(start, start + c, per)]
        start += c
    return np.array(items, np.int64).reshape(-1, 4), cap


def imu_items(w):
    """K2 items (start, count, s, node): the samples stably sorted by (start knot, bias node), runs cut at 32"""
    s = (w.imu_t - w.t0_ns) // w.dt_ns
    order = np.lexsort((w.imu_node, s))
    items = []
    for k, n in enumerate(order):
        if not items or items[-1][2] != s[n] or items[-1][3] != w.imu_node[n] or items[-1][1] >= IMU_CAP:
            items.append([k, 0, int(s[n]), int(w.imu_node[n])])
        items[-1][1] += 1
    return np.array(items, np.int64).reshape(-1, 4)


def regime_facts(name, n_sm):
    """what the case is there for, asserted from the window and the work-item rules; returns a one-line summary"""
    w, opt, ld = case(name)
    vis, cap = visual_items(w, n_sm)
    imu = imu_items(w)
    nK = w.n_knots
    wi0, si2 = knot_window(w, w.ti)
    wj0, sj2 = knot_window(w, w.tj)
    lns = int((w.ld0 if ld is None else ld) * 1e9)
    slot_i = (w.ti + w.rowi.astype(np.int64) * lns - w.t0_ns) // w.dt_ns - wi0
    slot_j = (w.tj + w.rowj.astype(np.int64) * lns - w.t0_ns) // w.dt_ns - wj0
    assert set(np.unique(np.concatenate([slot_i, slot_j]))) <= {0, 1}
    assert (np.maximum(si2 - wi0, sj2 - wj0) <= 1).all()
    dist = np.abs(vis[:, 3] - vis[:, 2])
    counts = vis[:, 1]
    if name == "one-factor":
        assert vis.tolist() == [[0, 1, wi0[0], wj0[0]]] and imu[:, 1].tolist() == [1]
    elif name == "same-window":
        assert (vis[:, 2] == vis[:, 3]).all() and (vis[:, 2] == nK - 4).all()
        assert (np.bincount(w.lm) > 1).any()   # several observations of a landmark in one round
    elif name == "overlap":
        assert {1, 2, 3, 4} <= set(dist.tolist()) and dist.max() >= 5
    elif name == "spline-ends":
        assert (vis[:, 2:] == 0).any() and (vis[:, 2:] == nK - 4).any()
        assert ((np.concatenate([w.ti, w.tj]) + w.rs_padding_ns) >= max_t(w)).any()     # the smax clamp
    elif name == "global-shutter":
        assert w.rs_padding_ns == 0 and not slot_i.any() and not slot_j.any()
    elif name in ("ld-zero", "ld-upper"):
        assert not opt["fix_ld"] and max(w.rowi.max(), w.rowj.max()) >= 1000
        assert (slot_i.any() or slot_j.any()) == (name == "ld-upper")
    elif name == "chunk-64":
        assert cap == 64 and sorted(set(counts.tolist())) == [43, 49, 52, 64]
    elif name == "chunk-128":
        assert cap == 128 and (counts == 128).all() and len(vis) <= n_sm < 2 * len(vis)
    elif name == "imu-1khz":
        runs = [tuple(imu[k:k + 2, 1]) for k in range(len(imu) - 1) if tuple(imu[k, 2:]) == tuple(imu[k + 1, 2:])]
        assert (32, 18) in runs and (32, 1) in runs
    elif name == "imu-nodes":
        assert w.imu_t.min() == w.t0_ns and w.imu_t.max() == max_t(w) - 1 and (np.diff(w.imu_t) < 0).any()
        assert ((w.imu_t - w.t0_ns) % w.dt_ns == 0).sum() > 3
        assert len(imu) > len(np.unique(imu[:, 2]))   # a bias-node change inside a knot interval
    elif name == "masks-fixed":
        k = opt["fixed_knot_index"]
        assert ((vis[:, 2:] <= k) & (vis[:, 2:] + 4 > k)).any() and ((imu[:, 2] <= k) & (imu[:, 2] + 3 > k)).any()
    elif name == "prior":
        pr = w.meta["prior"]
        assert set(pr.blk_type.tolist()) == {0, 1, 2, 3, 4}
        col2g = prior_col2g(pr, nK, w.bias0.shape[0], const_mask(name))
        assert (col2g < 0).any() and (col2g >= 0).any() and len(w.bf_i) > 0
    return (f"{len(vis)} K1 items (cap {cap}, counts {counts.min()}..{counts.max()}, window distance "
            f"{dist.min()}..{dist.max()}), {len(imu)} K2 items (counts {imu[:, 1].min()}..{imu[:, 1].max()})"
            if len(imu) else f"{len(vis)} K1 items (cap {cap}), no K2 items")


# ------------------------------------------------------------------------------------------------------------------
# reference

def prior_col2g(pr, nK, nB, cmask):
    col2g = np.full(pr.n, -1, np.int64)
    for t, i, c in zip(pr.blk_type, pr.blk_index, pr.blk_col):
        g = {0: 6 * i, 1: 6 * i + 3, 2: 6 * nK + 6 * i, 3: 6 * nK + 6 * i + 3, 4: 6 * nK + 6 * nB}[int(t)]
        for d in range(1 if t == pkg.BLK_LD else 3):
            if not cmask[g + d]:
                col2g[c + d] = g + d
    return col2g


def prior_dx(pr, q, p, bias, ld):
    """marginalization_factor.cpp:326-373: x - x0, rotations 2 sign(w) vec(x0^-1 x)"""
    dx = np.zeros(pr.n)
    for t, i, c, x0 in zip(pr.blk_type, pr.blk_index, pr.blk_col, pr.blk_x0):
        if t == pkg.BLK_ROT:
            d = syn.qmul(syn.qconj(x0) / (x0 @ x0), q[i])
            dx[c:c + 3] = (2.0 if d[3] >= 0 else -2.0) * d[:3]
        elif t == pkg.BLK_LD:
            dx[c] = ld - x0[0]
        else:
            x = {pkg.BLK_POS: p[i], pkg.BLK_BG: bias[i, :3], pkg.BLK_BA: bias[i, 3:]}[int(t)]
            dx[c:c + 3] = x - x0[:3]
    return dx


class Reference:
    """A | g over [camera dims | residual], landmark rows W | wld | g_l and h_l, in long double, with C, m, E."""

    def __init__(self, np_, nL):
        self.np, self.nL = np_, nL
        D = np_ + 1
        self.A = {"X": np.zeros((D, D), L), "C": np.zeros((D, D)), "m": np.zeros((D, D)), "E": np.zeros((D, D))}
        self.W = {"X": np.zeros((nL, D), L), "C": np.zeros((nL, D)), "m": np.zeros((nL, D)), "E": np.zeros((nL, D))}
        self.h = {"X": np.zeros(nL, L), "C": np.zeros(nL), "m": np.zeros(nL), "E": np.zeros(nL)}
        self.cost, self.cost_abs, self.cost_eval, self.n_terms = L(0), 0.0, 0.0, 0

    def rows(self, cols, J, r, lm=None, jrho=None):
        """rows sharing the camera columns cols (a column may repeat); J (n, k), r (n,)"""
        cols = np.append(cols, self.np)
        Jx = np.concatenate([J, r[:, None]], 1)
        nr = np.abs(Jx).max(1) if jrho is None else np.maximum(np.abs(Jx).max(1), np.abs(jrho))
        aJ = np.abs(Jx)
        ix = (cols[:, None], cols[None, :])
        JL = Jx.astype(L)
        np.add.at(self.A["X"], ix, JL.T @ JL)
        np.add.at(self.A["C"], ix, aJ.T @ aJ)
        np.add.at(self.A["m"], ix, float(len(r)))
        v = nr @ aJ
        np.add.at(self.A["E"], ix, v[:, None] + v[None, :])
        if lm is None:
            return
        ixl = (lm[:, None], cols[None, :])
        ar = np.abs(jrho)
        np.add.at(self.W["X"], ixl, jrho.astype(L)[:, None] * JL)
        np.add.at(self.W["C"], ixl, ar[:, None] * aJ)
        np.add.at(self.W["m"], ixl, 1.0)
        np.add.at(self.W["E"], ixl, nr[:, None] * (ar[:, None] + aJ))
        np.add.at(self.h["X"], lm, jrho.astype(L) ** 2)
        np.add.at(self.h["C"], lm, ar ** 2)
        np.add.at(self.h["m"], lm, 1.0)
        np.add.at(self.h["E"], lm, 2 * nr * ar)

    def factor_costs(self, c, r, extra=0.0):
        """per-factor costs c (long double), their residual rows r (n, k)"""
        self.cost += c.sum()
        self.cost_abs += float(np.abs(c).sum())
        self.cost_eval += float((np.abs(r).max(1) * np.abs(r).sum(1)).sum()) + extra
        self.n_terms += len(c)

    def parts(self):
        """{quantity: (reference, C, m, E)} in the layout of the device's outputs"""
        np_ = self.np
        A, W, h = self.A, self.W, self.h
        return {"A": tuple(A[k][:np_, :np_] for k in "XCmE"), "g": tuple(A[k][:np_, np_] for k in "XCmE"),
                "h_l": tuple(h[k] for k in "XCmE"), "g_l": tuple(W[k][:, np_] for k in "XCmE"),
                "W": tuple(W[k][:, :np_] for k in "XCmE")}


@functools.lru_cache(maxsize=None)
def reference(oracle_lib, name):
    w, opt, _ = case(name)
    o = make_estimator(oracle_lib, name)
    nK, nB, nL = w.n_knots, o.n_bias, o.n_lm
    np_ = o.np_dim
    cm = const_mask(name)
    ref = Reference(np_, nL)
    live = lambda cols, J: np.where(cm[cols][None, :], 0.0, J)
    # image factors: per (s_i, s_j) the 48 knot columns and the line delay
    if o.n_img:
        r, s, J, _ = o.EvalImageFactors(True, CAUCHY)
        r_raw = o.EvalImageFactors(False, 0.0)[0]
        sq = (r_raw.astype(L) ** 2).sum(1)
        b = L(CAUCHY) ** 2
        ref.factor_costs(L(0.5) * b * np.log1p(sq / b), r_raw, extra=len(sq) * float(gamma(3)) * CAUCHY ** 2)
        jk = J[:, :96].reshape(-1, 2, 4, 2, 2, 3)              # obs, side, knot, (rot, pos), row, xyz
        Jrow = np.moveaxis(jk, 4, 1).reshape(-1, 2, 48)        # obs, row, (side, knot, rot|pos, xyz)
        Jrow = np.concatenate([Jrow, J[:, 98:100, None]], 2)   # + line delay
        keys, inv = np.unique(s, axis=0, return_inverse=True)
        for g, (si, sj) in enumerate(keys):
            sel = np.nonzero(inv.ravel() == g)[0]
            cols = np.concatenate([6 * (sd + k) + np.arange(6) for sd in (si, sj) for k in range(4)] + [[np_ - 1]])
            ref.rows(cols, live(cols, Jrow[sel].reshape(-1, 49)), r[sel].ravel(), np.repeat(w.lm[sel], 2),
                     J[sel, 96:98].ravel())
    # IMU factors: per (s, node) the 24 knot columns and the 6 bias columns
    if o.n_imu:
        r, s, J, _ = o.EvalImuFactors(True)
        ref.factor_costs(L(0.5) * (r.astype(L) ** 2).sum(1), r)
        Jk = J[:, :144].reshape(-1, 4, 2, 6, 3)                # sample, knot, (rot, pos), row, xyz
        Jrow = np.moveaxis(Jk, 3, 1).reshape(-1, 6, 24)
        Jb = np.zeros((len(r), 6, 6))
        Jb[:, [0, 1, 2], [0, 1, 2]] = J[:, 144:147]
        Jb[:, [3, 4, 5], [3, 4, 5]] = J[:, 153:156]
        Jrow = np.concatenate([Jrow, Jb], 2)
        node = w.imu_node
        keys, inv = np.unique(np.stack([s, node], 1), axis=0, return_inverse=True)
        for g, (sk, nd) in enumerate(keys):
            sel = np.nonzero(inv.ravel() == g)[0]
            cols = np.concatenate([6 * sk + np.arange(24), 6 * nK + 6 * nd + np.arange(6)])
            ref.rows(cols, live(cols, Jrow[sel].reshape(-1, 30)), r[sel].ravel())
    # bias random-walk factors (trajectory_value_factor.h:45-99)
    bias = o.GetBiases()
    for i, j, si in zip(w.bf_i, w.bf_j, w.bf_sqrt_info):
        cols = np.concatenate([6 * nK + 6 * i + np.arange(6), 6 * nK + 6 * j + np.arange(6)])
        r = si * (bias[j] - bias[i])
        ref.factor_costs(L(0.5) * (r.astype(L) ** 2).sum(keepdims=True), r[None])
        ref.rows(cols, live(cols, np.concatenate([-np.diag(si), np.diag(si)], 1)), r)
    # prior: res = r + J dx over all its columns, Jacobian columns on constant dims dropped
    if "prior" in w.meta:
        pr = w.meta["prior"]
        q, p = o.GetKnots()
        dx = prior_dx(pr, q, p, bias, o.GetLineDelay())
        res = pr.r.astype(L) + pr.J.astype(L) @ dx.astype(L)
        col2g = prior_col2g(pr, nK, nB, cm)
        keep = col2g >= 0
        ref.factor_costs(L(0.5) * (res ** 2).sum(keepdims=True), res.astype(float)[None])
        ref.rows(col2g[keep], pr.J[:, keep], res.astype(float))
    return ref


def worst(x, parts, tau):
    """max over entries of |x - ref| / bound; entries with C = 0 must be exactly 0"""
    X, Cb, m, E = parts
    x = np.asarray(x, float)
    z = Cb == 0
    bad = np.count_nonzero(x[z])
    assert bad == 0, f"{bad} structural zeros are not zero (largest {np.abs(x[z]).max():.3e})"
    if not (~z).any():
        return 0.0
    err = np.abs(x[~z].astype(L) - X[~z]).astype(float)
    return float((err / (gamma(m[~z] + 2) * Cb[~z] + tau * E[~z])).max())


def cost_ratio(c, ref, tau):
    bound = gamma(ref.n_terms + 2) * ref.cost_abs + tau * ref.cost_eval
    return float(abs(L(c) - ref.cost)) / bound


def check_against_reference(ref, out, tau):
    """ratios of the device's (or oracle's) A, g, h_l, g_l, W (with wld), cost(s) to their bounds"""
    P = ref.parts()
    r = {k: worst(out[k], P[k], tau) for k in P if k in out}
    for k in ("cost", "cost_eval"):
        if k in out:
            r[k] = cost_ratio(out[k], ref, tau)
    return r


# ------------------------------------------------------------------------------------------------------------------
# CPU part

@pytest.mark.parametrize("name", list(CASES))
def test_work_item_rules_put_each_case_in_its_regime(name):
    print(f"\n{name}: {regime_facts(name, H100_SMS)}")


def test_cases_cover_the_cauchy_tail_and_long_imu_runs():
    """the synthetic generator alone stays near the identity of the loss and below 32 samples per IMU run"""
    w, _, _ = case("overlap")
    assert imu_items(w)[:, 1].max() <= 10
    assert imu_items(case("imu-1khz")[0])[:, 1].max() == IMU_CAP
    assert len(case("outliers")[0].meta["moved"]) == case("outliers")[0].n_obs // 10


@pytest.mark.parametrize("name", list(CASES))
def test_reference_equals_oracle_assembly(oracle_lib, name):
    """the long-double reference against the oracle's NormalEquations / landmark coupling / costs within the same
    bounds with tau = 0 (the oracle's own Jacobians on both sides)"""
    ref = reference(oracle_lib, name)
    o = make_estimator(oracle_lib, name)
    A, g, hl, gl, cost = o.NormalEquations()
    W = np.zeros((o.n_lm, o.np_dim))
    f = oracle_lib.raw("landmark_coupling")
    f.restype = C.c_int
    assert f(o.h, W.ctypes.data_as(C.c_void_p)) == 0
    r = check_against_reference(ref, {"A": A, "g": g, "h_l": hl, "g_l": gl, "W": W, "cost": cost,
                                      "cost_eval": o.EvalCost()}, 0.0)
    print(f"\n{name}: oracle vs reference, worst ratio " + ", ".join(f"{k} {v:.2g}" for k, v in r.items()))
    assert max(r.values()) <= 1, r


def test_cauchy_weights_of_the_outlier_case(oracle_lib):
    """rho'(s) = 1 / (1 + s / b): every moved observation of the outlier case sits deep in the Cauchy tail, the others
    at the noise level (the plain generator's weights at its initial state are printed beside them)"""
    def weights(name):
        r = make_estimator(oracle_lib, name).EvalImageFactors(False, 0.0)[0]
        return 1 / (1 + (r ** 2).sum(1) / CAUCHY ** 2)
    plain, out = weights("overlap"), weights("outliers")
    moved = out[case("outliers")[0].meta["moved"]]
    rest = np.delete(out, case("outliers")[0].meta["moved"])
    print(f"\nCauchy weights: overlap min {plain.min():.2e} median {np.median(plain):.2f}; outliers moved "
          f"{moved.min():.2e}..{moved.max():.2e}, not moved median {np.median(rest):.2f}")
    assert moved.max() < 0.2 and moved.min() < 1e-2 and np.median(rest) > 0.5


# ------------------------------------------------------------------------------------------------------------------
# GPU part

def device_outputs(g, deterministic):
    A, gc, hl, gl, cost = g.NormalEquations()
    o = debug_lm_step(g, 1e4)
    if deterministic:  # the two entry points run the same evaluation
        assert np.array_equal(np.triu(A), np.triu(o["A"])) and np.array_equal(gc, o["gc"])
    return {"A": A, "g": gc, "h_l": hl, "g_l": gl, "W": o["W"], "cost": cost, "cost_eval": g.EvalCost()}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_factor_kernels_match_extended_precision_reference(oracle_lib, cuda_lib, name):
    n_sm = device_sm_count()
    facts = regime_facts(name, n_sm)
    w, _, _ = case(name)
    ref = reference(oracle_lib, name)
    g = make_estimator(cuda_lib, name)
    st = g.DebugStructure()
    vis, _ = visual_items(w, n_sm)
    assert np.array_equal(st["items"], vis), "K1 work items"
    assert np.array_equal(st["imu_items"], imu_items(w)), "K2 work items"
    g.SetDeterministic(True)
    det = device_outputs(g, True)
    again = device_outputs(g, True)
    for k in ("A", "g", "h_l", "g_l", "W", "cost", "cost_eval"):
        assert np.array_equal(det[k], again[k]), f"deterministic mode: two calls differ in {k}"
    g.SetDeterministic(False)
    fast = device_outputs(g, False)
    rd = check_against_reference(ref, det, TAU)
    rf = check_against_reference(ref, fast, TAU)
    print(f"\n{name} ({n_sm} SMs): {facts}\n  worst ratio, deterministic: "
          + ", ".join(f"{k} {v:.2g}" for k, v in rd.items()) + "\n  worst ratio, default:       "
          + ", ".join(f"{k} {v:.2g}" for k, v in rf.items()))
    assert max(rd.values()) <= 1 and max(rf.values()) <= 1, (rd, rf)
