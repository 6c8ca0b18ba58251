"""BASELINE config 5: streaming sliding window over a long synthetic sequence.

Mirrors the reference's per-image cycle (odometry_manager.cpp:253-281) through the public Estimator API:

  1. ExtendTrajectory(t_img + 40 ms)   trajectory_manager.cpp:108-120: new control points = copies of the last one
  2. InitTrajectory                     :288-315: IMU-only predictor over [max_bef_ns, maxTime), control points
                                        <= max_bef_idx fixed, biases locked, Solve(8)   (skipped for the first window)
  3. UpdateTrajectory(..., 15)          :317-483: prior + image + IMU + bias factors, Solve(15),
     double2vector                      :485-516: 4-DoF re-alignment to the pre-solve pose of the first control point
  4. UpdateVIOPrior(marg_flag)          :122-286: MARGIN_OLD marginalizes the oldest keyframe (its control points,
                                        bias node 0, the landmarks anchored in it) into the next prior;
                                        MARGIN_SECOND_NEW keeps the prior untouched
  5. SlideWindow                        drop the oldest / the second-newest frame

The host-side slicing of the synthetic sequence (the "feature tracker / feature manager") is not part of the timed
region; everything that crosses the C-ABI is.  The same class drives the CUDA engine and (tests / bench CPU leg) the
oracle.  Used by tests (GPU vs oracle over a few windows) and by bench.py ("c5").
"""
from __future__ import annotations

import time

import numpy as np

from . import synthetic as syn
from .binding import BLK_BA, BLK_BG, BLK_LD, BLK_POS, BLK_RHO, BLK_ROT, CtvioError, Estimator, PriorData

KF_DT_NS = 50_000_000       # 20 Hz keyframes
WINDOW_SIZE = 10            # visual_odometry/parameters.h:8
WIN_KF = WINDOW_SIZE + 1    # keyframes per window
EXTEND_NS = 40_000_000      # odometry_manager.cpp:246, 251
# keyframe phase inside a knot interval: (offset + 40 ms) mod 50 ms > 40 ms, so that the spline's end before the
# extension lies BEFORE the new image and InitTrajectory has IMU samples to work with (with 20 Hz images and 50 ms
# knots any other phase leaves the predictor without data)
C5_KF_OFFSET_NS = 7_000_000
MARGIN_OLD, MARGIN_SECOND_NEW = 0, 1


def config_c5_sequence(n_windows: int, seed=syn.SEED0 + 5, anchors=30, track_len=10):
    """n_windows + 10 keyframes at 20 Hz, `anchors` new landmarks per keyframe tracked over the next 10 keyframes,
    free line delay (online calibration)."""
    n_kf = n_windows + WIN_KF - 1
    kf = C5_KF_OFFSET_NS + np.arange(n_kf, dtype=np.int64) * KF_DT_NS
    n_knots = int((kf[-1] + 200_000_000) // syn.DT_NS) + 4
    per_frame = [anchors] * (n_kf - 1) + [0]
    return syn.make_window("C5-seq", n_knots, kf, per_frame, track_len, seed=seed, fix_ld=False)


class StreamingRunner:
    """One estimator engine driven through the reference's per-image cycle.

    perm_seed: shuffle the order in which factors are handed to the estimator (the summation order of the CPU
    oracle) -- used by the sensitivity tests; the window problem is mathematically unchanged.
    second_new_every: every N-th frame is treated as a non-keyframe: when it is the second-newest frame of the window
    the step takes the MARGIN_SECOND_NEW branch (no marginalization, the frame is dropped instead of the oldest).
    min_parallax: when set, the branch of every step (the first one included) comes from the features instead:
    keyframe_decision over the window's tracker messages (the reference's addFeatureCheckParallax), MARGIN_OLD for a
    keyframe.  The record then also carries n_tracked and mean_parallax (None without parallax features).
    """

    def __init__(self, lib, seq: "syn.Window", iters=15, init_iters=8, device=0, second_new_every=0, perm_seed=None,
                 predictor=True, min_parallax=None):
        from . import make_config, make_options
        self.lib, self.seq, self.iters, self.init_iters = lib, seq, iters, init_iters
        self.predictor = predictor
        self.second_new_every = second_new_every
        self.min_parallax = min_parallax
        self.clouds = FrameClouds(seq) if min_parallax is not None else None
        self.rng = None if perm_seed is None else np.random.default_rng(perm_seed)
        s = seq
        self.frames = list(range(WIN_KF))                       # source keyframe ids in the window
        self.next_frame = WIN_KF
        # the spline so far: control points 0 .. ncp-1 (the initializer's output covers the first window)
        self.ncp = self._cp_needed(int(s.kf_times[WIN_KF - 1]) + EXTEND_NS)
        self.q = s.q0.copy(); self.p = s.p0.copy()
        self.bias = s.bias0.copy()                              # per source keyframe
        self.rho = s.rho0.copy()                                # per landmark (source ids)
        self.ld = s.ld0
        self.prior = None                                       # PriorData with GLOBAL knot / SOURCE frame / landmark ids
        cfg = make_config(device=device, **s.config_kwargs())
        self.est = Estimator(lib, cfg)
        self._make_options = make_options
        self.records = []
        self.step_index = 0

    # -- spline bookkeeping ------------------------------------------------------------------------
    def _cp_needed(self, t_ns):
        """smallest control-point count with maxTimeNs() >= t_ns (se3_spline.h:201-207)."""
        s = self.seq
        n = 4
        while s.t0_ns + (n - 3) * s.dt_ns < t_ns:
            n += 1
        return n

    def _knot_of(self, t_ns):
        return int((t_ns - self.seq.t0_ns) // self.seq.dt_ns)

    def _perm(self, n):
        return np.arange(n) if self.rng is None else self.rng.permutation(n)

    def _second_new_rule(self):
        """the second_new_every rule: MARGIN_SECOND_NEW when the second-newest frame is an N-th frame"""
        n = self.second_new_every
        return MARGIN_SECOND_NEW if n and (self.frames[-2] % n) == n - 1 else MARGIN_OLD

    @staticmethod
    def _decision_record(n_tracked, parallax_num, parallax_sum):
        return dict(n_tracked=n_tracked, mean_parallax=parallax_sum / parallax_num if parallax_num else None)

    # -- prior re-indexing (index identity <-> window-relative indices) -----------------------------
    def _prior_to_window(self, ks, frames, lm_global):
        pr = self.prior
        if pr is None:
            return None
        out = PriorData(n=pr.n, J=pr.J, r=pr.r, blk_type=pr.blk_type.copy(), blk_index=pr.blk_index.copy(),
                        blk_col=pr.blk_col.copy(), blk_x0=pr.blk_x0)
        knots = (out.blk_type == BLK_ROT) | (out.blk_type == BLK_POS)
        out.blk_index[knots] -= ks
        biases = (out.blk_type == BLK_BG) | (out.blk_type == BLK_BA)
        if biases.any():
            pos = np.searchsorted(frames, out.blk_index[biases])
            assert np.all(np.asarray(frames)[np.clip(pos, 0, len(frames) - 1)] == out.blk_index[biases]), \
                "a bias node of the prior left the window"
            out.blk_index[biases] = pos
        isrho = out.blk_type == BLK_RHO
        if isrho.any():
            pos = np.searchsorted(lm_global, out.blk_index[isrho])
            assert np.all(lm_global[np.clip(pos, 0, len(lm_global) - 1)] == out.blk_index[isrho])
            out.blk_index[isrho] = pos
        assert out.blk_index.min() >= 0
        return out

    def _prior_to_global(self, pr, ks, frames, lm_global):
        if pr is None:
            return None
        knots = (pr.blk_type == BLK_ROT) | (pr.blk_type == BLK_POS)
        pr.blk_index[knots] += ks
        biases = (pr.blk_type == BLK_BG) | (pr.blk_type == BLK_BA)
        pr.blk_index[biases] = np.asarray(frames)[pr.blk_index[biases]]
        isrho = pr.blk_type == BLK_RHO
        pr.blk_index[isrho] = lm_global[pr.blk_index[isrho]]
        return pr

    # -- one image ------------------------------------------------------------------------------------
    def step(self, k=None):
        s = self.seq
        first = self.step_index == 0
        t_wall = 0.0
        e = self.est
        max_bef_ns = max_bef_idx = None
        if not first:
            # the new image joins the window (AddImageToWindow), then ExtendTrajectory
            self.frames.append(self.next_frame)
            self.bias[self.next_frame] = self.bias[self.frames[-2]]   # Bgs_[WINDOW_SIZE] starts from the newest estimate
            self.next_frame += 1
            t_img = int(s.kf_times[self.frames[-1]])
            max_bef_ns = s.t0_ns + (self.ncp - 3) * s.dt_ns
            max_bef_idx = self.ncp - 1
            ncp_new = self._cp_needed(t_img + EXTEND_NS)
            self.q[self.ncp:ncp_new] = self.q[self.ncp - 1]
            self.p[self.ncp:ncp_new] = self.p[self.ncp - 1]
            self.ncp = ncp_new
        frames = np.asarray(self.frames, np.int64)
        kf = s.kf_times[frames]
        t_newest = int(kf[-1])
        max_t = s.t0_ns + (self.ncp - 3) * s.dt_ns
        ks = self._knot_of(int(kf[0]))                # min_idx of UpdateTrajectory = first control point of the window
        nloc = self.ncp - ks
        nowk, later = 0, self._knot_of(int(kf[1])) - ks
        decision = None
        if self.min_parallax is not None:
            # the feature manager's keyframe decision (visual_odometry.cpp:180-183), over the tracker's messages
            is_kf, n_tracked, num, psum = keyframe_decision([self.clouds.message(f) for f in self.frames], self.min_parallax)
            marg_flag = MARGIN_OLD if is_kf else MARGIN_SECOND_NEW
            decision = self._decision_record(n_tracked, num, psum)
        else:
            marg_flag = self._second_new_rule()

        # ---- host-side "tracker / feature manager": slice the sequence (not timed) ----
        w = syn.subwindow_frames(s, frames, imu_max_ns=min(max_t, t_newest + 1), window_size=WINDOW_SIZE)
        lm_global = w.meta["lm_global"]
        rho = np.ascontiguousarray(self.rho[lm_global])
        img_marg = ((w.anchor_frame[w.lm] == 0) & (rho[w.lm] > 0)).astype(np.int32)   # :216-218
        imu_marg = (w.imu_t < kf[1]).astype(np.int32)                                  # :243-253
        bias_marg = np.zeros(len(w.bf_i), np.int32); bias_marg[0] = 1                 # :256-263
        if marg_flag != MARGIN_OLD:
            img_marg[:] = 0; imu_marg[:] = 0; bias_marg[:] = 0
        pi_, pm = self._perm(w.n_obs), self._perm(len(w.imu_t))
        q = np.ascontiguousarray(self.q[ks:self.ncp]); p = np.ascontiguousarray(self.p[ks:self.ncp])
        b = np.ascontiguousarray(self.bias[frames])
        prior = self._prior_to_window(ks, self.frames, lm_global)
        init_sel = None
        if not first and self.predictor:
            init_sel = np.nonzero((w.imu_t >= max_bef_ns) & (w.imu_t < max_t))[0]
        h2d = 0
        # the host buffers the front end hands over (factor order as the reference's containers would give it): built
        # here, outside the timed region, like the rest of the slicing
        img_args = tuple(np.ascontiguousarray(a[pi_]) for a in (w.ti, w.rowi, w.pi, w.tj, w.rowj, w.pj, w.lm, img_marg))
        imu_args = tuple(np.ascontiguousarray(a[pm]) for a in (w.imu_t, w.imu_gyro, w.imu_accel, w.imu_node, imu_marg))
        init_args = None
        if init_sel is not None and len(init_sel) > 0:
            init_args = (np.ascontiguousarray(w.imu_t[init_sel]), np.ascontiguousarray(w.imu_gyro[init_sel]),
                         np.ascontiguousarray(w.imu_accel[init_sel]), np.full(len(init_sel), len(frames) - 1, np.int32))
        opt_init = None if init_args is None else self._make_options(fixed_knot_index=max_bef_idx - ks, lock_wb=True, lock_ab=True,
                                                                    fix_ld=True)
        opt_main = self._make_options(fix_ld=False, ld_lower=0.0, ld_upper=syn.LD_UPPER, is_marg_state=(marg_flag == MARGIN_OLD),
                                      ctrl_to_be_opt_now=nowk, ctrl_to_be_opt_later=later)

        # ---- timed region: everything that crosses the C-ABI ----
        stats = e.lib.has("transfer_stats")
        if stats:
            e.TransferStats(reset=True)
        t_start = time.perf_counter()
        e.SetTimeOrigin(s.t0_ns + ks * s.dt_ns)
        e.SetKnots(q, p); e.SetBiases(b); e.SetInvDepths(rho); e.SetLineDelay(self.ld)
        h2d += q.nbytes + p.nbytes + b.nbytes + rho.nbytes + 8
        init_summary = None
        if init_args is not None:
            # InitTrajectory: IMU only, new control points only, biases locked at the newest keyframe's estimate
            e.SetOptions(opt_init)
            e.ClearFactors()
            e.AddMarginalizationFactor(None)
            e.AddIMUMeasurementAnalytic(*init_args)
            h2d += len(init_sel) * 64
            init_summary = e.Solve(self.init_iters)
        # UpdateTrajectory
        e.SetOptions(opt_main)
        e.ClearFactors()
        e.AddMarginalizationFactor(prior)
        e.AddImageFeatureDelayAnalytic(*img_args)
        e.AddIMUMeasurementAnalytic(*imu_args)
        e.AddBiasFactor(w.bf_i, w.bf_j, w.bf_sqrt_info, bias_marg)
        h2d += w.n_obs * 64 + len(w.imu_t) * 64 + len(w.bf_i) * 56 + (0 if prior is None else prior.n * prior.n * 8)
        # pre-solve pose of the window's first control point (R0, t0 of UpdateTrajectory:329-331) -- AFTER InitTrajectory
        q_pre, p_pre = (q[nowk], p[nowk])
        R0 = syn.qrot(q_pre[None], np.eye(3)).T.copy(); t0 = p_pre.copy()
        t_built = time.perf_counter()
        summ = e.Solve(self.iters)
        t_solved = time.perf_counter()
        e.GaugeRealign(nowk, R0, t0)
        new_prior = e.SaveMarginalizationInfo() if marg_flag == MARGIN_OLD else None
        t_marged = time.perf_counter()
        qs, ps = e.GetKnots(); bs = e.GetBiases(); rs = e.GetInvDepths(); ld = e.GetLineDelay()
        t_wall = time.perf_counter() - t_start
        d2h = qs.nbytes + ps.nbytes + bs.nbytes + rs.nbytes + 8 + (0 if new_prior is None else new_prior.J.nbytes)
        if stats:
            h2d, d2h = e.TransferStats(reset=True)  # the engine's own count (includes its index tables)

        # ---- carry the solution over (the reference updates the parameter blocks in place) ----
        self.q[ks:self.ncp] = qs; self.p[ks:self.ncp] = ps
        self.bias[frames] = bs
        self.rho[lm_global] = rs
        self.ld = ld
        if marg_flag == MARGIN_OLD:
            self.prior = self._prior_to_global(new_prior, ks, self.frames, lm_global)
            self.frames.pop(0)                      # slideWindowOld
        else:
            self.frames.pop(-2)                     # slideWindowNew: the prior stays as it is
        # 0.5 |r_lin|^2 of the prior this window was solved with: the part of the cost that is set by the eps = 1e-30
        # pseudo-inverse's noise eigen-directions (tests compare costs with this constant removed)
        prior_const = 0.0 if prior is None else 0.5 * float(np.dot(prior.r, prior.r))
        rec = dict(window=self.step_index, ms=1e3 * t_wall, prior_const=prior_const,
                   ms_build_and_predict=1e3 * (t_built - t_start), ms_solve=1e3 * (t_solved - t_built),
                   ms_realign_marginalize=1e3 * (t_marged - t_solved), ms_readback=1e3 * (t_start + t_wall - t_marged), iterations=summ.iterations, final_cost=summ.final_cost,
                   initial_cost=summ.initial_cost, termination=summ.termination, n_obs=w.n_obs, n_imu=len(w.imu_t),
                   n_knots=nloc, n_lm=len(lm_global), device_ms=summ.device_ms, marg_flag=marg_flag,
                   init_iterations=None if init_summary is None else init_summary.iterations,
                   init_n_imu=0 if init_sel is None else len(init_sel),
                   init_device_ms=0.0 if init_summary is None else init_summary.device_ms,
                   prior_dim=0 if self.prior is None else self.prior.n, h2d_bytes=h2d, d2h_bytes=d2h)
        if decision is not None:
            rec.update(decision)
        self.records.append(rec)
        self.step_index += 1
        return rec

    def run(self, n_windows, first=0):
        for _ in range(n_windows):
            self.step()
        return self.records

    def state_error(self):
        """RMS translation error of the optimised part of the spline against the generator's truth (sanity metric)."""
        s = self.seq
        ks = self._knot_of(int(s.kf_times[self.frames[0]]))
        return float(np.sqrt(np.mean(np.sum((self.p[ks:self.ncp - 2] - s.p_gt[ks:self.ncp - 2]) ** 2, axis=1))))


def c3_window_a(lib, perm_seed=None, device=0):
    """BASELINE config 3, window A: the C3 source sequence restricted to keyframes 0..10 with the line delay free and
    the factors of keyframe 0 flagged for marginalization (trajectory_manager.cpp:206-263).  perm_seed shuffles the order
    in which factors are handed over (sensitivity tests).  Returns (estimator, sequence, window, first control point)."""
    from . import make_options, setup_estimator
    seq = syn.config_c3_sequence()
    wa = syn.subwindow(seq, 0, 10)
    later = int((wa.kf_times[1] - wa.t0_ns) // wa.dt_ns)
    nowk = int((wa.kf_times[0] - wa.t0_ns) // wa.dt_ns)
    img_marg = (wa.anchor_frame[wa.lm] == 0).astype(np.int32)
    imu_marg = (wa.imu_t < wa.kf_times[1]).astype(np.int32)
    bias_marg = np.zeros(len(wa.bf_i), np.int32); bias_marg[0] = 1
    if perm_seed is not None:
        rng = np.random.default_rng(perm_seed)
        pm = rng.permutation(wa.n_obs)
        for f in ("ti", "rowi", "pi", "tj", "rowj", "pj", "lm"):
            setattr(wa, f, np.ascontiguousarray(getattr(wa, f)[pm]))
        img_marg = img_marg[pm]
        pi = rng.permutation(len(wa.imu_t))
        for f in ("imu_t", "imu_gyro", "imu_accel", "imu_node"):
            setattr(wa, f, np.ascontiguousarray(getattr(wa, f)[pi]))
        imu_marg = imu_marg[pi]
    opt = make_options(fix_ld=False, ld_lower=0.0, ld_upper=syn.LD_UPPER, is_marg_state=True,
                       ctrl_to_be_opt_now=nowk, ctrl_to_be_opt_later=later)
    e = setup_estimator(lib, wa, image_marg=img_marg, imu_marg=imu_marg, bias_marg=bias_marg, options=opt, device=device)
    return e, seq, wa, nowk


# =====================================================================================================================
# Device-resident window (SURVEY 8f-1) fed by the wire formats (8f-4)

IMU_RECORD = np.dtype({"names": ["timestamp", "gyro", "accel", "orientation"],
                       "formats": [np.int64, (np.float64, 3), (np.float64, 3), (np.float64, 4)],
                       "offsets": [0, 8, 32, 64], "itemsize": 96})  # utils/parameter_struct.h:58-65 (Eigen alignment)


def quantize_wire(seq: "syn.Window"):
    """What survives the tracker's sensor_msgs::PointCloud: float32 bearings (rows are integers already).  Applied to
    the source sequence so that the classic (host-buffer) and the resident (wire-format) paths see identical numbers."""
    import copy
    s = copy.copy(seq)
    s.pi = seq.pi.astype(np.float32).astype(np.float64)
    s.pj = seq.pj.astype(np.float32).astype(np.float64)
    return s


class FrameClouds:
    """The tracker's per-frame messages rebuilt from the synthetic sequence: frame f carries the anchor observation of
    every landmark anchored in f followed by the observations of older landmarks seen in f (feature id = landmark id)."""

    def __init__(self, seq: "syn.Window"):
        self.seq = seq
        n_f = len(seq.kf_times)
        order_a = np.argsort(seq.anchor_frame, kind="stable")
        self.anchor_idx = np.empty(len(seq.anchor_frame), np.int32)     # landmark -> index inside its anchor frame's cloud
        counts_a = np.bincount(seq.anchor_frame, minlength=n_f)
        start_a = np.concatenate([[0], np.cumsum(counts_a)])
        self.anchor_idx[order_a] = np.arange(len(order_a)) - start_a[seq.anchor_frame[order_a]]
        order_o = np.argsort(seq.obs_frame, kind="stable")
        counts_o = np.bincount(seq.obs_frame, minlength=n_f)
        start_o = np.concatenate([[0], np.cumsum(counts_o)])
        self.obs_idx = np.empty(seq.n_obs, np.int32)                     # observation -> index inside its frame's cloud
        self.obs_idx[order_o] = np.arange(len(order_o)) - start_o[seq.obs_frame[order_o]] + counts_a[seq.obs_frame[order_o]]
        self._order_a, self._start_a, self._order_o, self._start_o = order_a, start_a, order_o, start_o
        # first observation of every landmark (its anchor bearing / row are replicated in every factor of the landmark)
        first = np.full(len(seq.anchor_frame), -1, np.int64)
        lms, idx = np.unique(seq.lm, return_index=True)
        first[lms] = idx
        self._first_obs = first

    def message(self, f):
        """(points float32 [n,3], id, u, v, vx, vy float32 [n]) of frame f."""
        s = self.seq
        la = self._order_a[self._start_a[f]:self._start_a[f + 1]]       # landmarks anchored here
        oo = self._order_o[self._start_o[f]:self._start_o[f + 1]]       # observations made here
        fo = self._first_obs[la]
        ok = fo >= 0
        xy = np.zeros((len(la), 2)); row = np.zeros(len(la))
        xy[ok] = s.pi[fo[ok]]; row[ok] = s.rowi[fo[ok]]
        xy = np.concatenate([xy, s.pj[oo]]); row = np.concatenate([row, s.rowj[oo].astype(np.float64)])
        ids = np.concatenate([la, s.lm[oo]]).astype(np.float32)
        n = len(ids)
        pts = np.ones((n, 3), np.float32); pts[:, :2] = xy
        z = np.zeros(n, np.float32)
        return pts, ids, (syn.FX * xy[:, 0] + syn.U0).astype(np.float32) if hasattr(syn, "FX") else z, row.astype(np.float32), z, z


def keyframe_decision(messages, min_parallax):
    """FeatureManager::addFeatureCheckParallax + compensatedParallax2 (feature_manager.cpp:28-87, :424-456) over the
    window's tracker messages (FrameClouds.message tuples), oldest to newest, the new image last: the host-buffer
    path's feature manager and the reference of ctvio_check_keyframe.  Ids and bearings are read as the wire carries
    them (float32; id = int(id + 0.5) as FeatureMsg2Image), ids are unique within a message.
    Returns (is_keyframe, n_tracked, parallax_num, parallax_sum):
      n_tracked     features of the new image whose id occurs in any other message (last_track_num);
      parallax_num  features of message fc-1 whose id also occurs in message fc-2 (fc = len(messages) - 1), 0 if fc < 2;
      parallax_sum  the sum of their bearing distances sqrt(du^2 + dv^2) (z == 1: compensated == plain);
      is_keyframe   fc < 2, n_tracked < 20 or no parallax feature, else parallax_sum / parallax_num >= min_parallax."""
    fc = len(messages) - 1
    ids = [(np.asarray(m[1], np.float32).astype(np.float64) + 0.5).astype(np.int64) for m in messages]
    others = np.concatenate(ids[:fc]) if fc > 0 else np.zeros(0, np.int64)
    n_tracked = int(np.isin(ids[fc], others).sum())
    parallax_num, parallax_sum = 0, 0.0
    if fc >= 2:
        id_i, id_j = ids[fc - 2], ids[fc - 1]
        xy_i = np.asarray(messages[fc - 2][0], np.float32)[:, :2].astype(np.float64)
        xy_j = np.asarray(messages[fc - 1][0], np.float32)[:, :2].astype(np.float64)
        order = np.argsort(id_i, kind="stable")
        pos = np.clip(np.searchsorted(id_i[order], id_j), 0, max(len(id_i) - 1, 0))
        hit = (id_i[order][pos] == id_j) if len(id_i) else np.zeros(len(id_j), bool)
        i = order[pos[hit]]
        du = xy_i[i, 0] - xy_j[hit, 0]
        dv = xy_i[i, 1] - xy_j[hit, 1]
        parallax_num = int(hit.sum())
        parallax_sum = float(np.sum(np.sqrt(du * du + dv * dv)))
    if fc < 2 or n_tracked < 20 or parallax_num == 0:
        return True, n_tracked, parallax_num, parallax_sum
    return bool(parallax_sum / parallax_num >= min_parallax), n_tracked, parallax_num, parallax_sum


class FeatureTable:
    """FeatureManager's feature list (feature_manager.cpp:28-59, :111-158, :341-423) over the tracker's messages
    (FrameClouds.message tuples) put into frame slots: the host restatement of the device's resident feature table
    (ctvio_feature_table_*), and the reference for those calls.

    One entry per landmark (FeaturePerId), in creation order: the feature id, the anchor slot, the feature index of its
    observation in each of the 16 frame slots (-1: none; the anchor's own observation included), its number in the last
    window (-1: not numbered), its inverse depth (-1: not initialised) and its solved status (solve_flag == SovelSucc,
    carried across a re-anchoring slide).  slide: landmarks leave with their anchor frame (no re-anchoring, the
    convention of subwindow_frames); an id seen again after its landmark left starts a new entry.  slide_reanchor: they
    are re-anchored as the reference does (removeBackShiftDepth / removeFront)."""

    N_SLOTS = 16

    def __init__(self):
        self.id = np.zeros(0, np.int64)
        self.anchor = np.zeros(0, np.int32)
        self.idx = np.full((0, self.N_SLOTS), -1, np.int32)
        self.lm = np.zeros(0, np.int32)
        self.rho = np.zeros(0)
        self.solved = np.zeros(0, bool)
        self.held = set()            # frame slots whose cloud the table holds
        self.numbered = np.zeros(0, np.int64)   # entries of the last window, in landmark order
        self.slots = None            # the last window's frame slots, oldest to newest
        self.bearing = {}            # frame slot -> bearings (x, y) of its cloud, as the wire carries them (float32)

    def add(self, slot, message):
        """the insertion half of addFeatureCheckParallax for the message put into `slot`: returns (n_tracked, n_new)"""
        assert slot not in self.held, "the table still holds this slot"
        ids = (np.asarray(message[1], np.float32).astype(np.float64) + 0.5).astype(np.int64)
        pos = {int(i): k for k, i in enumerate(self.id)}
        hit = np.array([pos.get(int(i), -1) for i in ids], np.int64)
        tracked = hit >= 0
        self.idx[hit[tracked], slot] = np.nonzero(tracked)[0]
        order = np.argsort(ids[~tracked], kind="stable")       # new entries in ascending id (std::map) order
        new_i = np.nonzero(~tracked)[0][order]
        n = len(new_i)
        idx = np.full((n, self.N_SLOTS), -1, np.int32)
        idx[:, slot] = new_i
        self.id = np.concatenate([self.id, ids[new_i]])
        self.anchor = np.concatenate([self.anchor, np.full(n, slot, np.int32)])
        self.idx = np.concatenate([self.idx, idx])
        self.lm = np.concatenate([self.lm, np.full(n, -1, np.int32)])
        self.rho = np.concatenate([self.rho, np.full(n, -1.0)])
        self.solved = np.concatenate([self.solved, np.zeros(n, bool)])
        self.held.add(slot)
        self.bearing[slot] = np.asarray(message[0], np.float32)[:, :2].astype(np.float64)
        return int(tracked.sum()), n

    def used_num(self, slots):
        return (self.idx[:, np.asarray(slots)] >= 0).sum(axis=1)

    def window(self, slots, window_size, rho):
        """setDepth of the last window's landmarks from `rho` (their solved inverse depths), then getDepthVector's
        numbering: candidates used_num >= 2 && start_frame < window_size - 2 in table order.  Returns the inverse
        depths of the new numbering (entries never initialised: -1)."""
        assert set(slots) == self.held and len(set(slots)) == len(slots)
        old = self.lm >= 0
        self.rho[old] = np.asarray(rho)[self.lm[old]]
        position = np.full(self.N_SLOTS, -1, np.int64)
        position[np.asarray(slots)] = np.arange(len(slots))
        start = position[self.anchor]
        cand = (self.used_num(slots) >= 2) & (start < window_size - 2)
        self.numbered = np.nonzero(cand)[0]
        self.lm[:] = -1
        self.lm[self.numbered] = np.arange(len(self.numbered))
        self.slots = np.asarray(slots, np.int32)
        return self.rho[self.numbered].copy()

    def landmarks(self):
        """(feature id, anchor slot, used_num) of each numbered landmark"""
        e = self.numbered
        return self.id[e], self.anchor[e], self.used_num(self.slots)[e]

    def observation_csr(self):
        """(obs_offset, obs_slot, obs_idx) of the window's landmarks: the anchor first, then the other observations in
        window order"""
        offset, slot, idx = [0], [], []
        for e in self.numbered:
            obs = [self.anchor[e]] + [s for s in self.slots if s != self.anchor[e] and self.idx[e, s] >= 0]
            slot += obs
            idx += [self.idx[e, s] for s in obs]
            offset.append(len(slot))
        return np.asarray(offset, np.int32), np.asarray(slot, np.int32), np.asarray(idx, np.int32)

    def factors(self, rho, marg_oldest):
        """image factors (trajectory_manager.cpp:206-236, :359-385), landmark-major and in window order within a
        landmark: (slot_i, idx_i, slot_j, idx_j, landmark, marg).  marg: anchor in the oldest frame and rho > 0."""
        off, slot, idx = self.observation_csr()
        out = [[] for _ in range(6)]
        for l in range(len(self.numbered)):
            a = off[l]
            m = int(bool(marg_oldest) and slot[a] == self.slots[0] and rho[l] > 0)
            for k in range(a + 1, off[l + 1]):
                for lst, v in zip(out, (slot[a], idx[a], slot[k], idx[k], l, m)):
                    lst.append(v)
        return tuple(np.asarray(x, np.int32) for x in out)

    def slide(self, slot, rho):
        """removeFailures (landmarks of the last window whose inverse depth in `rho` is < 0), then the landmarks
        anchored in `slot` leave and every other one loses its observation there.  Returns the number removed."""
        assert slot in self.held
        fail = np.zeros(len(self.id), bool)
        old = self.lm >= 0
        fail[old] = np.asarray(rho)[self.lm[old]] < 0
        keep = ~fail & (self.anchor != slot)
        self.id, self.anchor, self.idx = self.id[keep], self.anchor[keep], self.idx[keep]
        self.lm, self.rho, self.solved = self.lm[keep], self.rho[keep], self.solved[keep]
        self.idx[:, slot] = -1
        self.held.discard(slot)
        return int((~keep).sum())

    def slide_reanchor(self, slots, marg_old, rho, cam_R=None, cam_t=None, init_depth=5.0):
        """the reference of ctvio_feature_table_slide_reanchor.  slots: the window before the slide, oldest to newest;
        the leaving slot is slots[0] (marg_old) or slots[-2].  removeFailures as slide(), then an entry anchored in the
        leaving slot:
          marg_old (removeBackShiftDepth): with >= 2 observations left in the listed slots, its anchor becomes the
            earliest listed slot holding one and its inverse depth 1 / p_1.z (1 / init_depth when p_1.z is not > 0), with
            p_w = cam_R[0] (x, y, 1) depth + cam_t[0], p_1 = cam_R[1]^T (p_w - cam_t[1]), depth = 1 / its inverse depth
            (from `rho` when numbered in the last window, else its stored one), (x, y) the old anchor's bearing; else it
            leaves.  cam_R [>= 2, 3, 3], cam_t [>= 2, 3]: the camera poses of slots[0] and slots[1].
          not marg_old (removeFront): with an observation in the newest slot its anchor moves there and its inverse depth
            is kept; else it leaves.
        A re-anchored entry keeps its place, loses its number and stays solved when it was numbered.  Every other entry
        loses its observation in the leaving slot.  Returns (n_removed, n_reanchored)."""
        slots = [int(x) for x in slots]
        assert set(slots) == self.held and len(set(slots)) == len(slots) and len(slots) >= 2
        leave = slots[0] if marg_old else slots[-2]
        rho = np.asarray(rho, np.float64)
        numbered = (self.lm >= 0) & (self.lm < len(rho))
        r_now = self.rho.copy()
        r_now[numbered] = rho[self.lm[numbered]]
        fail = numbered & (r_now < 0)
        keep = ~fail & (self.anchor != leave)
        moved = np.zeros(len(self.id), bool)
        rest = self.idx[:, slots] >= 0
        rest[:, slots.index(leave)] = False
        for e in np.nonzero(~fail & (self.anchor == leave))[0]:
            if marg_old:
                if rest[e].sum() < 2:
                    continue
                x, y = self.bearing[leave][self.idx[e, leave]]
                with np.errstate(divide="ignore", invalid="ignore"):
                    depth = 1.0 / r_now[e]
                    p_w = np.asarray(cam_R[0]) @ np.array([x * depth, y * depth, depth]) + np.asarray(cam_t[0])
                    z = (np.asarray(cam_R[1]).T @ (p_w - np.asarray(cam_t[1])))[2]
                self.rho[e] = 1.0 / (z if z > 0 else init_depth)
                self.anchor[e] = slots[int(np.argmax(rest[e]))]
            else:
                if not rest[e, -1]:
                    continue
                self.rho[e] = r_now[e]
                self.anchor[e] = slots[-1]
            moved[e] = keep[e] = True
            self.solved[e] |= numbered[e]
            self.lm[e] = -1
        self.id, self.anchor, self.idx = self.id[keep], self.anchor[keep], self.idx[keep]
        self.lm, self.rho, self.solved = self.lm[keep], self.rho[keep], self.solved[keep]
        self.idx[:, leave] = -1
        self.held.discard(leave)
        return int((~keep).sum()), int(moved.sum())

    def map(self, slots, window_size, rho, cam_R, cam_t):
        """GetLandmarksInWindow / GetMarginCloud (visual_odometry.cpp:310-372) over the window's frame slots after the
        slide, oldest to newest: the reference of ctvio_feature_table_map.  rho: the resident inverse depths of the last
        window's numbering; cam_R [n_frames, 3, 3], cam_t [n_frames, 3]: the camera pose of each listed frame.
        Per entry: start = window position of its anchor, used_num = 1 + its observations in the other listed slots,
        depth = 1 / (its resident inverse depth when numbered in the last window, else its stored one).  Stable
        (IsLandMarkStable): used_num >= 2, start < window_size - 2, not start > window_size * 3 / 4, not depth <= 0 (NaN
        passes).  Margin cloud: stable, start == 0, used_num <= 2 and solve_flag == SovelSucc (numbered in the last
        window, or solved before a re-anchoring slide).  Returns (xyz [n, 3] world points R_c (x, y, 1) depth + t_c,
        feature ids [n], in_margin_cloud [n]) of the stable entries in table order."""
        assert set(slots) == self.held and len(set(slots)) == len(slots)
        slots = np.asarray(slots)
        position = np.full(self.N_SLOTS, -1, np.int64)
        position[slots] = np.arange(len(slots))
        start = position[self.anchor]
        used = self.used_num(slots)
        rho = np.asarray(rho, np.float64)
        numbered = (self.lm >= 0) & (self.lm < len(rho))
        r = self.rho.copy()
        r[numbered] = rho[self.lm[numbered]]
        with np.errstate(divide="ignore"):
            depth = 1.0 / r
        stable = (used >= 2) & (start < window_size - 2) & ~(start > window_size * 3.0 / 4.0) & ~(depth <= 0)
        margin = stable & (start == 0) & (used <= 2) & (numbered | self.solved)
        e = np.nonzero(stable)[0]
        xy = np.array([self.bearing[a][self.idx[k, a]] for k, a in zip(e, self.anchor[e])]).reshape(-1, 2)
        d = depth[e]
        pc = np.stack([xy[:, 0] * d, xy[:, 1] * d, d], -1)
        s = start[e]
        xyz = np.einsum("kij,kj->ki", np.asarray(cam_R)[s], pc) + np.asarray(cam_t)[s]
        return xyz, self.id[e].astype(np.int32), margin[e]


def quat_matrix(q):
    """rotation matrices [n, 3, 3] of unit quaternions [n, 4] (x, y, z, w)"""
    q = np.asarray(q, np.float64).reshape(-1, 4)
    return np.stack([syn.qrot(q, np.broadcast_to(np.eye(3)[j], (len(q), 3))) for j in range(3)], -1)


def camera_poses(q_imu, p_imu):
    """the camera pose of IMU poses (x, y, z, w quaternions [n, 4], positions [n, 3]) through the configured extrinsic
    (GetCameraPose): R_c = R R_CI, t_c = p + R p_CI, R_CI from the configured quaternion.  Returns (R_c [n, 3, 3],
    t_c [n, 3])."""
    R = quat_matrix(q_imu)
    R_CI = quat_matrix(syn.Q_CtoI)[0]
    return R @ R_CI, np.asarray(p_imu, np.float64).reshape(-1, 3) + R @ syn.P_CinI


class ResidentRunner(StreamingRunner):
    """The same per-image cycle with the window living in HBM: the new image's PointCloud and the new IMUData records go
    up as they are, control points are extended / dropped on the device, inverse depths are re-indexed on the device,
    the prior is handed over device-to-device, and the factor payload is gathered from the resident tables (only index
    tables cross the boundary).

    Both branches of the reference's slide: by default every frame is a keyframe (MARGIN_OLD, the C5 configuration);
    second_new_every takes the base class's rule; min_parallax takes the decision on the device (CheckKeyframe over the
    window's frame slots, right after the new cloud is ingested).  MARGIN_SECOND_NEW solves without marginalization
    flags, keeps the prior and drops the second-newest frame (SlideWindowSecondNew).  Frame slots come from a small
    allocator (a window that skipped frames can span more than 16 source frames): frame f takes slot f % 16 when that
    slot is free, else the lowest free one, so a MARGIN_OLD-only run uses exactly the slots f % 16.

    triangulate=True: new landmarks enter with inverse depth -1 and get their initial depth from TriangulateWindow (the
    reference's FeatureManager::triangulate in AddImageToWindow, visual_odometry.cpp:185-191) on the device, after the
    predictor solve, from the resident spline at each observation's row time.  The reference takes the newest frame's
    pose from its own IMU propagation (RI_, PI_, :189-190); here it is the predictor-solved spline, which carries the same
    IMU information.  Default (False): new landmarks take the sequence's initial guess rho0, as before.
    triangulate_probe (tests): called as probe(runner, obs_offset, obs_slot, obs_idx, rho_before) right after
    TriangulateWindow, on the engine state the call used.

    device_features=True (requires triangulate=True): the feature list lives on the device (the resident feature table,
    FeatureTable is its host restatement).  Each cloud joins it right after ingestion (FeatureTableAdd), the window's
    landmarks are numbered and their inverse depths re-laid out by FeatureTableWindow, the triangulation and the image
    factors come from the table, and the leaving frame's slot leaves it at the end of the step (FeatureTableSlide).  No
    host association is used: the caller passes only frame slots.  Default (False): the host derives the landmark
    numbering and the factor index tables from the sequence's ground-truth association, as before.

    publish_map=True (requires device_features=True): right after FeatureTableSlide, inside the timed region, the
    landmark map and keyframe poses the reference publishes after every image (GetLandmarksInWindow, GetMarginCloud,
    PublishVioKeyFrame) come from the device (FeatureTableMap over the post-slide window).  The arrays (xyz, ids,
    in_margin, cam_q, cam_p) are kept on last_map, and the record gains n_map_points and n_margin_points.

    reanchor=True (requires device_features=True): the table slides as the reference's feature list does
    (FeatureTableSlideReanchor: removeBackShiftDepth / removeFront), after GaugeRealign and the marginalization and
    before SlideWindow / SlideWindowSecondNew, while the leaving frame's time is still inside the spline.  The landmarks
    anchored in the leaving frame are re-anchored instead of dropped; the record gains n_reanchored.  On C5 the solve
    diverges in window 8: as in the reference, every MARGIN_OLD marginalizes all factors of the landmarks anchored in the
    oldest frame, so a re-anchored landmark's observations enter the prior again at every slide (DESIGN §6).
    Default (False): FeatureTableSlide after the window's slide, as before.

    publish_covariance=True: right after GaugeRealign and before the marginalization, inside the timed region, the
    covariance of the camera pose and velocity the reference publishes as its TF (odometry_manager.cpp:287-288, at
    maxTimeNs() - 50 ms) comes from the device (PoseCovariance with camera_frame=True).  The main solve fixes no knots,
    so the call holds knots 0..3 (the window's first segment) constant as its own gauge.  The 12 x 12 matrix is kept on
    last_pose_cov and the record gains pose_cov_rcond and ms_pose_cov; a window the call finds rank deficient records
    pose_cov_rcond = nan, its message as pose_cov_error, and keeps last_pose_cov = None.

    publish_map_covariance=True (requires publish_map=True): right after GaugeRealign, next to the pose covariance and
    with the same gauge (knots 0..3), the covariance of every landmark's world point in the window's numbering comes
    from the device (FeatureTablePointCovariance, ids from FeatureTableLandmarks).  After FeatureTableMap the matrices
    are attached to the map points by feature id and kept on last_map_cov [n_points, 3, 3]: a point whose entry had no
    number in the window, or was anchored in the leaving frame (re-anchored by reanchor=True), has no covariance and
    gets NaN.  The record gains point_cov_rcond, ms_point_cov and n_map_points_without_cov; a window the call finds rank
    deficient records point_cov_rcond = nan and its message as point_cov_error, and keeps last_map_cov = None.  With
    publish_covariance as well, the window covariance is formed twice (once per call).

    publish_odometry_covariance=True: right after GaugeRealign, next to the pose covariance and with the same gauge
    (knots 0..3) and frame (the camera), the covariance of the relative camera pose of each consecutive keyframe pair
    (kf[i], kf[i+1]) of the window, the odometry edges a pose graph fuses, comes from the device
    (RelativePoseCovariance).  Unlike the absolute pose covariance it does not grow with the distance from the gauge.
    The matrices are kept on last_rel_cov [n_frames - 1, 6, 6] and the record gains rel_cov_rcond and ms_rel_cov; a
    window the call finds rank deficient records rel_cov_rcond = nan and its message as rel_cov_error, and keeps
    last_rel_cov = None.  Each covariance call forms the window covariance anew."""

    POSE_COV_LAG_NS = 50_000_000
    POSE_COV_GAUGE_KNOT = 3

    def __init__(self, lib, seq, triangulate=False, device_features=False, publish_map=False, reanchor=False,
                 publish_covariance=False, publish_map_covariance=False, publish_odometry_covariance=False, **kw):
        if device_features and not triangulate:
            raise ValueError("device_features requires triangulate=True: new landmarks enter with inverse depth -1")
        if publish_map and not device_features:
            raise ValueError("publish_map requires device_features=True: the map is read from the resident feature table")
        if reanchor and not device_features:
            raise ValueError("reanchor requires device_features=True: landmarks are re-anchored in the resident feature table")
        if publish_map_covariance and not publish_map:
            raise ValueError("publish_map_covariance requires publish_map=True: the covariances belong to the map's points")
        super().__init__(lib, seq, **kw)
        self.triangulate = triangulate
        self.device_features = device_features
        self.publish_map = publish_map
        self.reanchor = reanchor
        self.publish_covariance = publish_covariance
        self.publish_map_covariance = publish_map_covariance
        self.publish_odometry_covariance = publish_odometry_covariance
        self.last_map = None
        self.last_pose_cov = None
        self.last_map_cov = None
        self.last_rel_cov = None
        self.triangulate_probe = None
        if self.clouds is None:
            self.clouds = FrameClouds(seq)
        self.n_slots = 16
        self.slot_of = {}          # source frame -> frame slot, for the frames in the engine's table
        self.imu_sent = 0          # samples of the source sequence already ingested
        self.prev_lm_global = None
        self.prev_ks = None
        self.readback = None
        self.prior_dim = 0         # dimension of the engine's active prior

    def _assign_slot(self, f):
        """frame slot of a new frame: f % n_slots when free, else the lowest free slot"""
        used = set(self.slot_of.values())
        s = f % self.n_slots
        if s in used:
            s = min(set(range(self.n_slots)) - used)
        self.slot_of[f] = s
        return s

    def _imu_records(self, lo, hi):
        s = self.seq
        rec = np.zeros(hi - lo, IMU_RECORD)
        rec["timestamp"] = s.imu_t[lo:hi]; rec["gyro"] = s.imu_gyro[lo:hi]; rec["accel"] = s.imu_accel[lo:hi]
        rec["orientation"][:, 3] = 1.0
        return rec

    def step(self, k=None):
        s = self.seq
        e = self.est
        first = self.step_index == 0
        t_push = 0.0
        if first:
            # the initializer's window: state, the 11 clouds and the IMU samples so far go up once
            e.SetTimeOrigin(s.t0_ns)
            e.SetKnots(self.q[:self.ncp], self.p[:self.ncp]); e.SetBiases(self.bias[self.frames]); e.SetLineDelay(self.ld)
            for f in self.frames:
                e.IngestFeatureCloud(self._assign_slot(f), int(s.kf_times[f]), *self.clouds.message(f))
                if self.device_features:
                    e.FeatureTableAdd(self.slot_of[f])
            self.base_knot = 0      # global index of the engine's knot 0
        else:
            self.frames.append(self.next_frame)
            self._assign_slot(self.next_frame)
            self.next_frame += 1
        frames = np.asarray(self.frames, np.int64)
        frame_slots = np.array([self.slot_of[f] for f in self.frames], np.int32)   # window position -> frame slot
        kf = s.kf_times[frames]
        t_newest = int(kf[-1])
        t0 = time.perf_counter()
        max_bef_ns = max_bef_idx = None
        if not first:
            f = self.frames[-1]
            e.IngestFeatureCloud(int(frame_slots[-1]), t_newest, *self.clouds.message(f))
            if self.device_features:
                e.FeatureTableAdd(int(frame_slots[-1]))   # addFeatureCheckParallax's insertion, by feature id
        decision = None
        if self.min_parallax is not None:
            # addFeatureCheckParallax on the device, over the clouds already in the frame table
            is_kf, n_tracked, num, psum = e.CheckKeyframe(frame_slots, self.min_parallax)
            marg_flag = MARGIN_OLD if is_kf else MARGIN_SECOND_NEW
            decision = self._decision_record(n_tracked, num, psum)
        else:
            marg_flag = self._second_new_rule()
        marg = marg_flag == MARGIN_OLD
        if not first:
            max_bef_ns = s.t0_ns + (self.ncp - 3) * s.dt_ns
            max_bef_idx = self.ncp - 1
            self.ncp = e.ExtendKnotsTo(t_newest + EXTEND_NS) + self.base_knot
        hi = int(np.searchsorted(s.imu_t, t_newest, side="right"))
        if hi > self.imu_sent:
            opt_min = s.t0_ns + self._knot_of(int(kf[0])) * s.dt_ns
            e.IngestImu(self._imu_records(self.imu_sent, hi), 8, 32, drop_before_ns=opt_min)
            self.imu_sent = hi
        t_push = time.perf_counter() - t0
        max_t = s.t0_ns + (self.ncp - 3) * s.dt_ns
        ks = self._knot_of(int(kf[0]))
        assert ks == self.base_knot, (ks, self.base_knot)
        nloc = self.ncp - ks
        nowk, later = 0, self._knot_of(int(kf[1])) - ks

        # bias random walk between consecutive keyframes of the window (trajectory_manager.cpp:420-450)
        bf_i = np.arange(len(kf) - 1, dtype=np.int32)
        bf_sqrt_info = syn.bias_sqrt_info(s.imu_t, kf)
        bias_marg = np.zeros(len(bf_i), np.int32); bias_marg[0] = 1
        if not marg:
            bias_marg[:] = 0
        if not self.device_features:
            # ---- host-side index work of the "feature manager" (ids only, not timed like the classic runner's slicing) ----
            w = syn.subwindow_frames(s, frames, imu_max_ns=min(max_t, t_newest + 1), window_size=WINDOW_SIZE)
            lm_global = w.meta["lm_global"]
            if self.prev_lm_global is None:
                old_index = np.full(len(lm_global), -1, np.int32)
            else:
                pos = np.searchsorted(self.prev_lm_global, lm_global)
                pos = np.clip(pos, 0, len(self.prev_lm_global) - 1)
                old_index = np.where(self.prev_lm_global[pos] == lm_global, pos, -1).astype(np.int32)
            # new landmarks (old_index < 0): the sequence's initial guess, or -1 (not initialised) when triangulated below
            init_rho = np.full(len(lm_global), -1.0) if self.triangulate else s.rho0[lm_global]
            img_marg = (w.anchor_frame[w.lm] == 0).astype(np.int32)  # (inverse depths are positive in the synthetic sequences)
            if not marg:
                img_marg[:] = 0
            # factor -> (frame slot, index in that frame's cloud) of its two observations
            sel = self._factor_selection(frames, lm_global)
            g_lm = lm_global[w.lm]
            slot_i = frame_slots[w.anchor_frame[w.lm]]
            idx_i = self.clouds.anchor_idx[g_lm]
            slot_j = frame_slots[w.obs_frame]
            idx_j = self.clouds.obs_idx[sel]
            if self.triangulate:
                tri_csr = self._observation_csr(frames, w, lm_global, slot_j, idx_j, frame_slots)
        R0 = t0_ = None
        if self.readback is not None:
            qn, pn = self.readback[0][ks - self.prev_ks], self.readback[1][ks - self.prev_ks]
        else:
            qn, pn = self.q[ks], self.p[ks]
        R0 = syn.qrot(qn[None], np.eye(3)).T.copy(); t0_ = np.array(pn, float)

        # ---- timed region ----
        e.TransferStats(reset=True) if not first else None
        t_start = time.perf_counter()
        if self.device_features:
            n_lm = e.FeatureTableWindow(frame_slots, WINDOW_SIZE)   # setDepth + getDepthVector, on the device
        else:
            e.RemapLandmarks(old_index, init_rho)
            n_lm = len(lm_global)
        init_summary = None
        if not first and self.predictor:
            e.SetOptions(self._make_options(fixed_knot_index=max_bef_idx - ks, lock_wb=True, lock_ab=True, fix_ld=True))
            e.ClearFactors()
            e.EnablePrior(False)
            n_init = e.AddImuFromTable(max_bef_ns, max_t, fixed_node=len(frames) - 1)
            if n_init > 0:
                init_summary = e.Solve(self.init_iters)
        n_tri = n_fb = None
        if self.triangulate:
            # FeatureManager::triangulate on the predictor-solved spline (window 0: the initializer's), before the
            # image factors that read the depths
            if self.device_features:
                n_tri, n_fb = e.TriangulateWindowFromTable()
            else:
                rho_before = e.GetInvDepths() if self.triangulate_probe is not None else None
                n_tri, n_fb = e.TriangulateWindow(*tri_csr)
                if self.triangulate_probe is not None:
                    self.triangulate_probe(self, *tri_csr, rho_before)
        e.SetOptions(self._make_options(fix_ld=False, ld_lower=0.0, ld_upper=syn.LD_UPPER, is_marg_state=marg,
                                        ctrl_to_be_opt_now=nowk, ctrl_to_be_opt_later=later))
        e.ClearFactors()
        e.EnablePrior(True)
        if self.device_features:
            n_obs = e.AddImageFeaturesFromTable(marg)
        else:
            e.AddImageFeaturesFromSlots(slot_i, idx_i, slot_j, idx_j, w.lm, img_marg)
            n_obs = w.n_obs
        opt_min = s.t0_ns + ks * s.dt_ns
        if marg:
            n_imu = e.AddImuFromTable(opt_min, min(max_t, t_newest + 1), kf_times=kf, marg_before_ns=int(kf[1]))
        else:
            n_imu = e.AddImuFromTable(opt_min, min(max_t, t_newest + 1), kf_times=kf)
        e.AddBiasFactor(bf_i, bf_i + 1, bf_sqrt_info, bias_marg)
        if not self.device_features:
            n_imu = len(w.imu_t)
        t_built = time.perf_counter()
        summ = e.Solve(self.iters)
        t_solved = time.perf_counter()
        e.GaugeRealign(nowk, R0, t0_)
        pose_cov = None
        if self.publish_covariance:                    # the covariance of the published camera pose, before the slide
            t_cov = time.perf_counter()
            try:
                self.last_pose_cov, rc = e.PoseCovariance([max_t - self.POSE_COV_LAG_NS],
                                                          gauge_knot_index=self.POSE_COV_GAUGE_KNOT, camera_frame=True)
                pose_cov = dict(pose_cov_rcond=rc)
            except CtvioError as err:
                self.last_pose_cov = None
                pose_cov = dict(pose_cov_rcond=float("nan"), pose_cov_error=str(err))
            pose_cov["ms_pose_cov"] = 1e3 * (time.perf_counter() - t_cov)
        rel_cov = None
        if self.publish_odometry_covariance:           # the odometry edges between the window's keyframes, before the slide
            t_cov = time.perf_counter()
            try:
                self.last_rel_cov, _, rc = e.RelativePoseCovariance(kf[:-1], kf[1:],
                                                                    gauge_knot_index=self.POSE_COV_GAUGE_KNOT,
                                                                    camera_frame=True)
                rel_cov = dict(rel_cov_rcond=rc)
            except CtvioError as err:
                self.last_rel_cov = None
                rel_cov = dict(rel_cov_rcond=float("nan"), rel_cov_error=str(err))
            rel_cov["ms_rel_cov"] = 1e3 * (time.perf_counter() - t_cov)
        point_cov = lm_cov = None
        if self.publish_map_covariance:                # the covariances of the window's landmark points, before the slide
            t_cov = time.perf_counter()
            try:
                cov, rc = e.FeatureTablePointCovariance(gauge_knot_index=self.POSE_COV_GAUGE_KNOT)
                lm_ids, lm_anchor, _ = e.FeatureTableLandmarks()
                lm_cov = (cov, lm_ids, lm_anchor)
                point_cov = dict(point_cov_rcond=rc)
            except CtvioError as err:
                point_cov = dict(point_cov_rcond=float("nan"), point_cov_error=str(err))
            point_cov["ms_point_cov"] = 1e3 * (time.perf_counter() - t_cov)
        if marg:
            n_out = C_int32(); nb_out = C_int32()
            e.lib.call("marginalize", e.h, byref(n_out), byref(nb_out))
            if n_out.value > 0:
                e.AdoptPrior()           # device-to-device
            self.prior_dim = n_out.value
        t_marged = time.perf_counter()
        qs, ps = e.GetKnots(); ld = e.GetLineDelay()   # the trajectory is the product the caller publishes
        n_removed = n_reanchored = None
        if self.reanchor:                              # removeFailures + removeBackShiftDepth / removeFront
            n_removed, n_reanchored = e.FeatureTableSlideReanchor(frame_slots, marg)
        if marg:
            drop_knots = later
            e.SlideWindow(drop_knots, 1, 1)            # slideWindowOld: oldest frame's control points and bias node leave
        else:
            drop_knots = 0
            e.SlideWindowSecondNew()                   # slideWindowNew: the second-newest frame leaves, the prior stays
        if self.device_features and not self.reanchor:  # the leaving frame's landmarks and observations leave the table
            n_removed = e.FeatureTableSlide(self.slot_of[self.frames[0 if marg else -2]])
        if self.publish_map:                           # the landmark map and keyframe poses of the post-slide window
            self.last_map = e.FeatureTableMap(np.delete(frame_slots, 0 if marg else len(frame_slots) - 2), WINDOW_SIZE)
        if self.publish_map_covariance:
            self.last_map_cov = None if lm_cov is None else self._map_covariance(lm_cov, frame_slots[0 if marg else -2])
            point_cov["n_map_points_without_cov"] = (len(self.last_map[1]) if self.last_map_cov is None else
                                                     int(np.isnan(self.last_map_cov[:, 0, 0]).sum()))
        t_wall = time.perf_counter() - t_start
        h2d, d2h = (0, 0) if first else e.TransferStats(reset=True)

        del self.slot_of[self.frames.pop(0 if marg else -2)]
        self.q[ks:self.ncp] = qs; self.p[ks:self.ncp] = ps
        self.ld = ld
        self.readback, self.prev_ks = (qs, ps), ks
        if not self.device_features:
            self.prev_lm_global = lm_global
        self.base_knot = ks + drop_knots
        rec = dict(window=self.step_index, ms=1e3 * (t_wall + t_push), prior_const=0.0,
                   ms_build_and_predict=1e3 * (t_built - t_start + t_push), ms_solve=1e3 * (t_solved - t_built),
                   ms_realign_marginalize=1e3 * (t_marged - t_solved), ms_readback=1e3 * (t_start + t_wall - t_marged),
                   iterations=summ.iterations, final_cost=summ.final_cost, initial_cost=summ.initial_cost,
                   termination=summ.termination, n_obs=n_obs, n_imu=n_imu, n_knots=nloc, n_lm=n_lm,
                   device_ms=summ.device_ms, marg_flag=marg_flag,
                   init_iterations=None if init_summary is None else init_summary.iterations, init_n_imu=0,
                   init_device_ms=0.0 if init_summary is None else init_summary.device_ms, prior_dim=self.prior_dim,
                   h2d_bytes=h2d, d2h_bytes=d2h)
        if decision is not None:
            rec.update(decision)
        if pose_cov is not None:
            rec.update(pose_cov)
        if point_cov is not None:
            rec.update(point_cov)
        if rel_cov is not None:
            rec.update(rel_cov)
        if self.device_features:
            # n_new_lm: the window's landmarks without a depth yet (-1), which are exactly the ones TriangulateWindow wrote
            rec.update(n_triangulated=n_tri, n_fallback=n_fb, n_new_lm=n_tri + n_fb, n_removed=n_removed)
            if self.reanchor:
                rec.update(n_reanchored=n_reanchored)
            if self.publish_map:
                rec.update(n_map_points=len(self.last_map[1]), n_margin_points=int(self.last_map[2].sum()))
        elif self.triangulate:
            rec.update(n_triangulated=n_tri, n_fallback=n_fb, n_new_lm=int(np.sum(old_index < 0)))
        self.records.append(rec)
        self.step_index += 1
        return rec

    def _map_covariance(self, lm_cov, leaving_slot):
        """[n_points, 3, 3]: the window's point covariances attached to last_map's points by feature id; NaN for a point
        whose entry had no number in the window or was anchored in the leaving slot (re-anchored since)"""
        cov, ids, anchor = lm_cov
        keep = anchor != leaving_slot
        of_id = dict(zip(ids[keep].tolist(), np.nonzero(keep)[0].tolist()))
        out = np.full((len(self.last_map[1]), 3, 3), np.nan)
        for k, i in enumerate(self.last_map[1].tolist()):
            l = of_id.get(i)
            if l is not None:
                out[k] = cov[l]
        return out

    def _observation_csr(self, frames, w, lm_global, slot_j, idx_j, frame_slots=None):
        """(obs_offset, obs_slot, obs_idx) of TriangulateWindow: per window landmark its anchor, then its observations
        in frame order (the factors are landmark-major and frame-ordered within a landmark).  frame_slots: the frame
        slot of each window position (default: frame % n_slots, the slots of a MARGIN_OLD-only run)."""
        assert np.all(np.diff(w.lm) >= 0)
        if frame_slots is None:
            frame_slots = frames % self.n_slots
        n_lm = len(lm_global)
        counts = np.bincount(w.lm, minlength=n_lm)
        obs_offset = np.concatenate([[0], np.cumsum(counts + 1)]).astype(np.int32)
        first_factor = np.cumsum(counts) - counts
        obs_slot = np.empty(obs_offset[-1], np.int32)
        obs_idx = np.empty(obs_offset[-1], np.int32)
        obs_slot[obs_offset[:-1]] = frame_slots[w.anchor_frame]
        obs_idx[obs_offset[:-1]] = self.clouds.anchor_idx[lm_global]
        pos = obs_offset[w.lm] + 1 + np.arange(len(w.lm)) - first_factor[w.lm]
        obs_slot[pos] = slot_j
        obs_idx[pos] = idx_j
        return obs_offset, obs_slot, obs_idx

    def _factor_selection(self, frames, lm_global):
        """indices (into the source sequence's observation arrays) of the window's factors, in subwindow_frames order"""
        s = self.seq
        pos = -np.ones(len(s.kf_times), np.int64); pos[frames] = np.arange(len(frames))
        keep = np.zeros(len(s.rho_gt), bool); keep[lm_global] = True
        return np.nonzero(keep[s.lm] & (pos[s.obs_frame] >= 0))[0]

    def sync_state_to_host(self):
        """full state read-back (tests): biases of the window's frames and inverse depths of its landmarks.
        Call right after step(): the engine's window has already slid by one keyframe."""
        e = self.est
        b = e.GetBiases()
        self.bias[np.asarray(self.frames[:len(b) - 1])] = b[:-1]
        return b


class CycleRunner:
    """ResidentRunner(triangulate=True, device_features=True) through the library's per-image cycle: window 0 is one
    ctvio_odometry_start, every later window one ctvio_process_image, fed with the sequence's clouds and IMU records.
    The frame slots, the window's frames, the knot range of each frame and the bias nodes are the library's; the runner
    only keeps what a caller publishes: the trajectory (q, p, ld), the records and the last map.

    Options as ResidentRunner's: second_new_every (through marg_flag_override), min_parallax (the device's keyframe
    decision), publish_map, reanchor, iters / init_iters.  want_knots / want_map=False leave the knot / map outputs
    unrequested (the trajectory is then not carried into q / p, and last_map stays None).  Not supported: the host
    association (device_features=False), the rho0 mode (triangulate=False), predictor=False and a perm_seed.

    covariances: any subset of ("pose", "odometry", "map") ("map" requires publish_map=True), the library's covariance
    publications (ctvio_cycle_covariances): the window covariance is formed once per image, with the gauge of
    ResidentRunner (knots 0..3, opt.covariance_gauge_knot), and projected to ResidentRunner's three publications.
    They are kept on last_pose_cov [1, 12, 12], last_rel_cov [n_frames - 1, 6, 6] and last_map_cov [n_points, 3, 3]
    (None when the cycle could not form them), and the record gains pose_cov_rcond / rel_cov_rcond / point_cov_rcond
    (nan with *_error when the window is rank deficient) and n_map_points_without_cov.  ResidentRunner's
    publish_*covariance keywords are not taken: name the publications in covariances instead."""

    COVARIANCES = ("pose", "odometry", "map")

    def __init__(self, lib, seq, iters=15, init_iters=8, device=0, second_new_every=0, min_parallax=None,
                 publish_map=False, reanchor=False, want_knots=True, want_map=True, triangulate=True,
                 device_features=True, predictor=True, perm_seed=None, publish_covariance=False,
                 publish_map_covariance=False, publish_odometry_covariance=False, covariances=()):
        from . import binding, make_config
        if not triangulate or not device_features:
            raise ValueError("CycleRunner runs the device feature table with triangulation only "
                             "(triangulate=True, device_features=True)")
        if not predictor:
            raise ValueError("CycleRunner always runs the IMU predictor (predictor=True)")
        if perm_seed is not None:
            raise ValueError("CycleRunner takes the factors from the resident tables: no perm_seed")
        if publish_covariance or publish_map_covariance or publish_odometry_covariance:
            raise ValueError("CycleRunner takes the covariance publications as covariances=('pose', 'odometry', 'map'), "
                             "not as ResidentRunner's publish_*covariance keywords")
        if isinstance(covariances, str):
            raise ValueError("covariances is a collection of names, e.g. covariances=('pose',)")
        covariances = tuple(covariances)
        unknown = [c for c in covariances if c not in self.COVARIANCES]
        if unknown:
            raise ValueError(f"unknown covariances {unknown}: pick from {self.COVARIANCES}")
        if "map" in covariances and not publish_map:
            raise ValueError("covariances=('map', ...) requires publish_map=True: the covariances belong to the map's points")
        if min_parallax is not None and second_new_every:
            raise ValueError("min_parallax and second_new_every both choose the branch: pick one")
        if min_parallax is not None and not min_parallax > 0:
            raise ValueError("min_parallax must be > 0 (None: every image is a keyframe)")
        self.lib, self.seq = lib, seq
        self.second_new_every = second_new_every
        self.want_knots, self.want_map = want_knots, want_map and publish_map
        s = seq
        self.clouds = FrameClouds(seq)
        self.frames = list(range(WIN_KF))
        self.next_frame = WIN_KF
        self.q = s.q0.copy(); self.p = s.p0.copy(); self.ld = s.ld0
        self.bias = s.bias0.copy()
        self.ncp = StreamingRunner._cp_needed(self, int(s.kf_times[WIN_KF - 1]) + EXTEND_NS)
        self.est = Estimator(lib, make_config(device=device, **s.config_kwargs()))
        self.opt = binding.CycleOptions()
        lib.call("cycle_default_options", C_byref(self.opt))
        self.opt.window_size = WINDOW_SIZE
        self.opt.solve_iterations = iters
        self.opt.predictor_iterations = init_iters
        self.opt.min_parallax = 0.0 if min_parallax is None else float(min_parallax)
        self.opt.extend_ns = EXTEND_NS
        self.opt.ld_lower, self.opt.ld_upper = 0.0, syn.LD_UPPER
        self.opt.sigma_wb_discrete, self.opt.sigma_ab_discrete = syn.SIGMA_BG, syn.SIGMA_BA
        self.opt.reanchor = int(reanchor)
        self.opt.publish_map = int(publish_map)
        self.covariances = covariances
        self.opt.publish_pose_covariance = int("pose" in covariances)
        self.opt.publish_odometry_covariance = int("odometry" in covariances)
        self.opt.publish_map_covariance = int("map" in covariances)
        self.reanchor, self.publish_map = reanchor, publish_map
        self.last_map = None
        self.last_pose_cov = self.last_rel_cov = self.last_map_cov = None
        self.last_cov_info = None
        self.records = []
        self.step_index = 0
        self.imu_sent = 0

    def _override(self):
        """the second_new_every rule of StreamingRunner, or -1 (the device decides)"""
        n = self.second_new_every
        if not n:
            return -1
        return MARGIN_SECOND_NEW if (self.frames[-2] % n) == n - 1 else MARGIN_OLD

    def _imu_records(self, t_newest):
        s = self.seq
        hi = int(np.searchsorted(s.imu_t, t_newest, side="right"))
        lo, self.imu_sent = self.imu_sent, max(hi, self.imu_sent)
        return ResidentRunner._imu_records(self, lo, hi) if hi > lo else None

    def step(self, k=None):
        s, e = self.seq, self.est
        first = self.step_index == 0
        if not first:
            self.frames.append(self.next_frame)
            self.next_frame += 1
        t_newest = int(s.kf_times[self.frames[-1]])
        imu = self._imu_records(t_newest)
        e.TransferStats(reset=True)
        t0 = time.perf_counter()
        if first:
            f = self.frames
            res, arr = e.OdometryStart(self.opt, s.t0_ns, self.q[:self.ncp], self.p[:self.ncp],
                                       [self.clouds.message(i) for i in f], s.kf_times[f], self.bias[f], self.ld, imu,
                                       marg_flag_override=self._override(), want_knots=self.want_knots,
                                       want_map=self.want_map)
        else:
            res, arr = e.ProcessImage(t_newest, self.clouds.message(self.frames[-1]), imu,
                                      marg_flag_override=self._override(), want_knots=self.want_knots,
                                      want_map=self.want_map)
        cov_rec = self._covariances(res["n_map_points"]) if self.covariances else None
        t_wall = time.perf_counter() - t0
        h2d, d2h = e.TransferStats(reset=True)
        marg_flag = res["marg_flag"]
        ks = int((res["knot_t0_ns"] - s.t0_ns) // s.dt_ns)
        self.ncp = ks + res["n_knots"]
        if "q" in arr:
            self.q[ks:self.ncp] = arr["q"]; self.p[ks:self.ncp] = arr["p"]; self.ld = arr["line_delay"]
        if "map" in arr:
            self.last_map = arr["map"]
        self.frames.pop(0 if marg_flag == MARGIN_OLD else -2)
        sv, pr = res["solve"], res["predictor"]
        rec = dict(window=self.step_index, ms=1e3 * t_wall, host_ms=res["host_ms"], prior_const=0.0,
                   iterations=sv["iterations"], final_cost=sv["final_cost"], initial_cost=sv["initial_cost"],
                   termination=sv["termination"], n_obs=res["n_image_factors"], n_imu=res["n_imu_factors"],
                   n_knots=res["n_knots"], n_lm=res["n_landmarks"], device_ms=sv["device_ms"], marg_flag=marg_flag,
                   init_iterations=None if res["n_predictor_imu"] == 0 or first else pr["iterations"],
                   init_device_ms=pr["device_ms"], prior_dim=res["prior_dim"], h2d_bytes=h2d, d2h_bytes=d2h,
                   n_triangulated=res["n_triangulated"], n_fallback=res["n_fallback"], n_removed=res["n_removed"],
                   frame_slot=res["frame_slot"])
        if self.opt.min_parallax > 0:
            rec.update(StreamingRunner._decision_record(res["n_tracked"], res["parallax_num"], res["parallax_sum"]))
        if self.reanchor:
            rec.update(n_reanchored=res["n_reanchored"])
        if self.publish_map:
            rec.update(n_map_points=res["n_map_points"], n_margin_points=res["n_margin_points"])
        if cov_rec is not None:
            rec.update(cov_rec)
        self.records.append(rec)
        self.step_index += 1
        return rec

    def _covariances(self, n_map_points):
        """the last cycle's covariance publications onto last_*_cov, and their record entries"""
        cov12, cov6, cov9, info = self.est.CycleCovariances()
        self.last_cov_info = info
        self.last_pose_cov = None if cov12 is None else cov12[None]
        self.last_rel_cov, self.last_map_cov = cov6, cov9
        rec = {}
        for name, key, got in (("pose", "pose_cov", cov12), ("odometry", "rel_cov", cov6), ("map", "point_cov", cov9)):
            if name in self.covariances:
                rec[key + "_rcond"] = info["rcond"] if got is not None else float("nan")
                if got is None:
                    rec[key + "_error"] = info.get("error", "")
        if "map" in self.covariances:
            rec["n_map_points_without_cov"] = info["n_map_points_without_cov"] if cov9 is not None else n_map_points
        return rec

    def checkpoint(self):
        """The run after the last step(): the library's blob (ctvio_odometry_checkpoint) with the runner's own host-side
        counters and carried trajectory, as a dict for restore() / resume()."""
        return dict(blob=self.est.Checkpoint(), frames=list(self.frames), next_frame=self.next_frame,
                    imu_sent=self.imu_sent, step_index=self.step_index, ncp=self.ncp, q=self.q.copy(), p=self.p.copy(),
                    ld=self.ld)

    def restore(self, state):
        """Continue from a checkpoint() on this runner's engine: the next step() is the image after it.  The records
        and the last publications of the steps since are dropped."""
        if state["step_index"] < 1:
            raise ValueError("a checkpoint is taken after a step")
        self.est.Restore(state["blob"])
        self.frames = list(state["frames"])
        self.next_frame, self.imu_sent = state["next_frame"], state["imu_sent"]
        self.step_index, self.ncp = state["step_index"], state["ncp"]
        self.q, self.p, self.ld = state["q"].copy(), state["p"].copy(), state["ld"]
        self.records = []
        self.last_map = self.last_pose_cov = self.last_rel_cov = self.last_map_cov = self.last_cov_info = None
        return self

    @classmethod
    def resume(cls, lib, seq, state, **kw):
        """A runner on a fresh engine that continues a checkpoint() of a run over `seq`; kw: the options of that run
        (the engine's deterministic mode is not part of the checkpoint)."""
        return cls(lib, seq, **kw).restore(state)

    def run(self, n_windows, first=0):
        for _ in range(n_windows):
            self.step()
        return self.records

    def state_error(self):
        """RMS translation error of the optimised part of the spline against the generator's truth (sanity metric)."""
        s = self.seq
        ks = int((s.kf_times[self.frames[0]] - s.t0_ns) // s.dt_ns)
        return float(np.sqrt(np.mean(np.sum((self.p[ks:self.ncp - 2] - s.p_gt[ks:self.ncp - 2]) ** 2, axis=1))))


from ctypes import byref, c_int32 as C_int32  # noqa: E402  (used by ResidentRunner.step)
from ctypes import byref as C_byref  # noqa: E402  (used by CycleRunner)
