"""Re-anchoring slide of the resident feature table (ctvio_feature_table_slide_reanchor): the landmarks anchored in the
leaving frame are re-anchored as the reference's feature list does it (removeBackShiftDepth / removeFront,
feature_manager.cpp:341-423) instead of leaving with it.

CPU: streaming.FeatureTable.slide_reanchor is driven side by side with a literal restatement of the reference's
std::list<FeaturePerId> over the C5 sequence, checked against the geometry of a noise-free global-shutter sequence, and
pinned at the rule boundaries.  GPU: the device call against FeatureTable, its error paths, full tables, and the whole
ResidentRunner(reanchor=True)."""
import ctypes as C
import importlib
import types

import numpy as np
import pytest

from helpers import pkg, syn

st = importlib.import_module("ctrl-vio_b200.streaming")

WS = st.WINDOW_SIZE
INIT_DEPTH = 5.0


def msg(ids, xy=(0.0, 0.0)):
    """a tracker message as FrameClouds.message returns it: float32 points (z = 1), id, u, v, vx, vy channels"""
    ids = np.asarray(ids, np.float32)
    n = len(ids)
    pts = np.ones((n, 3), np.float32)
    pts[:, :2] = np.broadcast_to(np.asarray(xy, np.float32), (n, 2))
    z = np.zeros(n, np.float32)
    return pts, ids, z, z, z, z


def spline_camera_poses(q, p, times, t0_ns, dt_ns):
    """camera poses at the given times from syn.spline_pose of the knots, the extrinsic composed on the host"""
    qi, pi = syn.spline_pose(np.asarray(q), np.asarray(p), np.asarray(times, np.int64), t0_ns, dt_ns)
    return st.camera_poses(qi, pi)


# ---------------------------------------------------------------------------------------------------------------------
# the reference's feature list, restated literally (visual_struct.h:66-100, feature_manager.h/.cpp, visual_odometry.*)

SOLVE_INITIAL, SOLVE_SUCC, SOLVE_FAIL = 0, 1, 2


class FeaturePerId:
    def __init__(self, feature_id, start_frame):
        self.feature_id = feature_id
        self.start_frame = start_frame
        self.feature_per_frame = []         # FeaturePerFrame::point (x, y, 1)
        self.estimated_depth = -1.0
        self.solve_flag = SOLVE_INITIAL

    def end_frame(self):
        return self.start_frame + len(self.feature_per_frame) - 1


class ReferenceFeatureManager:
    def __init__(self, window_size=WS):
        self.feature = []                   # std::list<FeaturePerId>
        self.ws = window_size

    def add_feature(self, frame_count, message):
        """the insertion half of addFeatureCheckParallax (feature_manager.cpp:28-59): the image is a std::map by id"""
        pts = np.asarray(message[0], np.float32).astype(np.float64)
        ids = (np.asarray(message[1], np.float32).astype(np.float64) + 0.5).astype(np.int64)
        for k in np.argsort(ids, kind="stable"):
            fid = int(ids[k])
            point = np.array([pts[k, 0], pts[k, 1], 1.0])
            it = next((f for f in self.feature if f.feature_id == fid), None)
            if it is None:
                self.feature.append(FeaturePerId(fid, frame_count))
                self.feature[-1].feature_per_frame.append(point)
            else:
                it.feature_per_frame.append(point)

    def is_candidate(self, f):
        return len(f.feature_per_frame) >= 2 and f.start_frame < self.ws - 2

    def get_depth_vector(self):
        with np.errstate(divide="ignore"):
            return np.array([1.0 / f.estimated_depth for f in self.feature if self.is_candidate(f)])

    def set_depth(self, x):
        k = 0
        for f in self.feature:
            if not self.is_candidate(f):
                continue
            with np.errstate(divide="ignore"):
                f.estimated_depth = 1.0 / x[k]
            k += 1
            f.solve_flag = SOLVE_FAIL if f.estimated_depth < 0 else SOLVE_SUCC

    def remove_failures(self):
        self.feature = [f for f in self.feature if f.solve_flag != SOLVE_FAIL]

    def remove_back_shift_depth(self, marg_R, marg_P, new_R, new_P, init_depth=INIT_DEPTH):
        kept = []
        for f in self.feature:
            if f.start_frame != 0:
                f.start_frame -= 1
            else:
                uv_i = f.feature_per_frame.pop(0)
                if len(f.feature_per_frame) < 2:
                    continue
                with np.errstate(invalid="ignore"):
                    pts_i = uv_i * f.estimated_depth
                    w_pts_i = marg_R @ pts_i + marg_P
                    pts_j = new_R.T @ (w_pts_i - new_P)
                dep_j = pts_j[2]
                f.estimated_depth = dep_j if dep_j > 0 else init_depth
            kept.append(f)
        self.feature = kept

    def remove_front(self, frame_count):
        kept = []
        for f in self.feature:
            if f.start_frame == frame_count:
                f.start_frame -= 1
            else:
                if f.end_frame() < frame_count - 1:
                    kept.append(f)
                    continue
                j = frame_count - 1 - f.start_frame
                f.feature_per_frame.pop(j)
                if len(f.feature_per_frame) == 0:
                    continue
            kept.append(f)
        self.feature = kept

    def stable(self, f):
        """IsLandMarkStable (visual_odometry.h:82-93)"""
        return self.is_candidate(f) and not f.start_frame > self.ws * 3.0 / 4.0 and not f.estimated_depth <= 0

    def landmarks_in_window(self, Rs, Ps):
        """GetLandmarksInWindow: (feature ids, world points)"""
        ids, xyz = [], []
        for f in self.feature:
            if self.stable(f):
                i = f.start_frame
                ids.append(f.feature_id)
                xyz.append(Rs[i] @ (f.feature_per_frame[0] * f.estimated_depth) + Ps[i])
        return np.asarray(ids, np.int64), np.asarray(xyz).reshape(-1, 3)

    def margin_cloud(self):
        """GetMarginCloud's feature ids"""
        return np.asarray([f.feature_id for f in self.feature if self.stable(f) and self.is_candidate(f) and
                           f.start_frame == 0 and len(f.feature_per_frame) <= 2 and f.solve_flag == SOLVE_SUCC], np.int64)


def table_depths(t, rho):
    """each entry's depth as the reference holds it after setDepth: 1 / (resident rho when numbered, else stored)"""
    numbered = t.lm >= 0
    r = t.rho.copy()
    r[numbered] = np.asarray(rho)[t.lm[numbered]]
    with np.errstate(divide="ignore"):
        return 1.0 / r


def same_depths(a, b):
    a, b = np.asarray(a), np.asarray(b)
    both_nan = np.isnan(a) & np.isnan(b)
    close = np.isclose(a, b, rtol=1e-15, atol=0.0) | (a == b)
    return a.shape == b.shape and bool(np.all(both_nan | close))


def decision_rule(seq, mode, n):
    clouds = st.FrameClouds(seq)
    if mode == "min_parallax":
        means = []
        for k in range(n):
            _, _, num, s = st.keyframe_decision([clouds.message(f) for f in range(k, k + st.WIN_KF)], 0.0)
            means.append(s / num)
        m = float(np.median(means))
        return lambda frames: st.keyframe_decision([clouds.message(f) for f in frames], m)[0]
    every = {"margin_old": 0, "second_new_every_2": 2, "second_new_every_3": 3}[mode]
    return lambda frames: not (every and frames[-2] % every == every - 1)


def solved_depths(seq, ids, rng, noise=0.05, negative=0.01):
    """a stand-in for the solve: truth with relative noise, about `negative` of them negative (removeFailures)"""
    rho = seq.rho_gt[ids] * (1.0 + noise * rng.standard_normal(len(ids)))
    rho[rng.random(len(ids)) < negative] *= -1
    return rho


@pytest.mark.parametrize("mode", ["margin_old", "second_new_every_2", "second_new_every_3", "min_parallax"])
def test_table_matches_literal_reference(mode):
    n = 40
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    clouds = st.FrameClouds(seq)
    decide = decision_rule(seq, mode, n)
    rng = np.random.default_rng(7)
    r = types.SimpleNamespace(n_slots=16, slot_of={})
    t, ref = st.FeatureTable(), ReferenceFeatureManager()
    frames = list(range(st.WIN_KF))
    for i, f in enumerate(frames):
        t.add(st.ResidentRunner._assign_slot(r, f), clouds.message(f))
        ref.add_feature(i, clouds.message(f))
    nxt, rho, flags, n_moved, n_margin = st.WIN_KF, np.zeros(0), set(), 0, []
    for k in range(n):
        if k:
            frames.append(nxt)
            t.add(st.ResidentRunner._assign_slot(r, nxt), clouds.message(nxt))
            ref.add_feature(WS, clouds.message(nxt))
            nxt += 1
        slots = np.array([r.slot_of[f] for f in frames], np.int32)
        marg = bool(decide(frames))
        flags.add(marg)
        rho_h = t.window(slots, WS, rho)
        assert same_depths(rho_h, ref.get_depth_vector()), k           # getDepthVector in the same numbering
        rho = solved_depths(seq, t.id[t.numbered], rng)
        ref.set_depth(rho)
        R_c, t_c = spline_camera_poses(seq.q_gt, seq.p_gt, seq.kf_times[frames], seq.t0_ns, seq.dt_ns)
        ref.remove_failures()
        if marg:
            ref.remove_back_shift_depth(R_c[0], t_c[0], R_c[1], t_c[1])
        else:
            ref.remove_front(WS)
        n_before = len(t.id)
        removed, moved = t.slide_reanchor(slots, marg, rho, R_c, t_c, INIT_DEPTH)
        n_moved += moved
        assert n_before - removed == len(t.id) == len(ref.feature), k
        leave = r.slot_of.pop(frames.pop(0 if marg else -2))
        post = np.array([r.slot_of[f] for f in frames], np.int32)
        position = np.full(16, -1); position[post] = np.arange(len(post))
        assert t.id.tolist() == [f.feature_id for f in ref.feature], k
        assert position[t.anchor].tolist() == [f.start_frame for f in ref.feature], k
        assert t.used_num(post).tolist() == [len(f.feature_per_frame) for f in ref.feature], k
        assert same_depths(table_depths(t, rho), [f.estimated_depth for f in ref.feature]), k
        # the observations themselves: the table's bearings in the listed slots are the reference's points, in order
        for e, f in zip(range(len(t.id)), ref.feature):
            xy = [t.bearing[s][t.idx[e, s]] for s in post if t.idx[e, s] >= 0]
            assert np.array_equal(np.asarray(xy), np.asarray(f.feature_per_frame)[:, :2]), (k, e)
        # the published map and the margin cloud
        R_p, t_p = spline_camera_poses(seq.q_gt, seq.p_gt, seq.kf_times[frames], seq.t0_ns, seq.dt_ns)
        xyz, ids, margin = t.map(post, WS, rho, R_p, t_p)
        ids_r, xyz_r = ref.landmarks_in_window(R_p, t_p)
        assert np.array_equal(ids, ids_r), k
        assert np.allclose(xyz, xyz_r, rtol=1e-12, atol=1e-12), k
        assert np.array_equal(ids[margin], ref.margin_cloud()), k
        n_margin.append(int(margin.sum()))
        assert leave not in t.held
    assert n_moved > 0
    if mode == "margin_old":
        assert flags == {True} and max(n_margin) > 0
    elif mode != "second_new_every_2":
        assert flags == {True, False}


def test_shifted_depth_is_the_true_depth_in_the_new_anchor():
    """noise-free global-shutter C5-like sequence, ground-truth knots and inverse depths: every re-anchored inverse depth
    is the landmark's true inverse depth in the new anchor camera, and the new anchor's own bearing at that depth lands
    on the landmark.  The only error is the float32 rounding of the bearings the wire carries (2^-24 relative, times
    the lever of the depth shift): the bound is 1e-6 relative (measured: 2.1e-10 for the inverse depths, 4.1e-8 for the
    points, which also carry the new anchor's rounded bearing)."""
    n = 12
    n_kf = n + st.WIN_KF - 1
    kf = st.C5_KF_OFFSET_NS + np.arange(n_kf, dtype=np.int64) * st.KF_DT_NS
    n_knots = int((kf[-1] + 200_000_000) // syn.DT_NS) + 4
    seq = syn.make_window("C5-gs", n_knots, kf, [30] * (n_kf - 1) + [0], 10, seed=syn.SEED0 + 5, fix_ld=False,
                          global_shutter=True, pixel_sigma=0.0)
    clouds = st.FrameClouds(seq)
    R_all, t_all = spline_camera_poses(seq.q_gt, seq.p_gt, seq.kf_times, seq.t0_ns, seq.dt_ns)
    # every landmark's world point from its (float64) anchor bearing and true depth
    first = np.full(len(seq.rho_gt), -1); lms, i0 = np.unique(seq.lm, return_index=True); first[lms] = i0
    a = seq.anchor_frame
    xy1 = np.concatenate([seq.pi[first], np.ones((len(first), 1))], 1)
    p_world = np.einsum("lij,lj->li", R_all[a], xy1 / seq.rho_gt[:, None]) + t_all[a]
    r = types.SimpleNamespace(n_slots=16, slot_of={})
    t = st.FeatureTable()
    frames = list(range(st.WIN_KF))
    for f in frames:
        t.add(st.ResidentRunner._assign_slot(r, f), clouds.message(f))
    nxt, rho, worst, worst_point, checked = st.WIN_KF, np.zeros(0), 0.0, 0.0, 0
    for k in range(n):
        if k:
            frames.append(nxt)
            t.add(st.ResidentRunner._assign_slot(r, nxt), clouds.message(nxt))
            nxt += 1
        slots = np.array([r.slot_of[f] for f in frames], np.int32)
        t.window(slots, WS, rho)
        # the solve's stand-in: each landmark's true inverse depth in its current anchor camera
        slot_frame = {s: f for f, s in r.slot_of.items()}
        g = np.array([slot_frame[int(s)] for s in t.anchor[t.numbered]], np.int64)
        pc = np.einsum("lji,lj->li", R_all[g], p_world[t.id[t.numbered]] - t_all[g])
        rho = 1.0 / pc[:, 2]
        before = dict(zip(t.id.tolist(), t.anchor.tolist()))
        _, moved = t.slide_reanchor(slots, True, rho, R_all[frames], t_all[frames], INIT_DEPTH)
        r.slot_of.pop(frames.pop(0))
        frame_of = {s: f for f, s in r.slot_of.items()}
        m = np.array([before[i] != a_ for i, a_ in zip(t.id.tolist(), t.anchor.tolist())])
        assert m.sum() == moved > 0
        for e in np.nonzero(m)[0]:
            g = frame_of[int(t.anchor[e])]
            assert g == frames[0]                                       # contiguous tracks: the next frame
            pc = R_all[g].T @ (p_world[t.id[e]] - t_all[g])
            worst = max(worst, abs(t.rho[e] * pc[2] - 1.0))
            x, y = t.bearing[int(t.anchor[e])][t.idx[e, t.anchor[e]]]
            p = R_all[g] @ (np.array([x, y, 1.0]) / t.rho[e]) + t_all[g]
            worst_point = max(worst_point, np.linalg.norm(p - p_world[t.id[e]]) / pc[2])
            checked += 1
    print("re-anchored", checked, "worst relative inverse-depth error", worst, "worst relative point error", worst_point)
    assert checked > 1000
    assert worst <= 1e-6 and worst_point <= 1e-6


def chain(n_slots, ids_per_slot):
    t = st.FeatureTable()
    for s in range(n_slots):
        t.add(s, msg(ids_per_slot[s], xy=(0.1, -0.2)))
    return t


def test_rule_boundaries_margin_old():
    # landmark 1: anchor + 1 observation; 2: anchor + 2; 3: anchor + 2, NaN inverse depth; 4: anchor + 2, negative (a
    # failure); 5: anchor + 2, a depth that the shift takes behind the next camera; 6: anchored in slot 1
    t = chain(3, [[1, 2, 3, 4, 5], [1, 2, 3, 4, 5, 6], [2, 3, 4, 5, 6]])
    slots = [0, 1, 2]
    t.window(slots, WS, np.zeros(0))
    assert t.id[t.numbered].tolist() == [1, 2, 3, 4, 5, 6]
    rho = np.array([0.5, 0.25, np.nan, -0.5, -1e-300, 0.125])
    rho[4] = 1.0 / 0.01                                              # depth 0.01 m
    R = np.stack([np.eye(3)] * 3)
    tc = np.array([[0.0, 0.0, 0.0], [0.0, 0.0, 1.0], [0.0, 0.0, 2.0]])   # the next camera 1 m further along z
    removed, moved = t.slide_reanchor(slots, True, rho, R, tc, INIT_DEPTH)
    assert (removed, moved) == (2, 3)                                # 1 (too few) and 4 (failed) leave
    assert t.id.tolist() == [2, 3, 5, 6] and t.anchor.tolist() == [1, 1, 1, 1]
    assert t.rho[0] == 1.0 / (4.0 - 1.0)                             # 1 / (depth - 1 m)
    assert t.rho[1] == 1.0 / INIT_DEPTH                              # NaN falls back
    assert t.rho[2] == 1.0 / INIT_DEPTH                              # behind the camera falls back
    assert t.lm.tolist() == [-1, -1, -1, 5] and t.solved.tolist() == [True, True, True, False]
    assert t.idx[:, 0].tolist() == [-1] * 4 and 0 not in t.held
    # the re-anchored landmarks at start 0 with two observations are in the margin cloud through their solved status
    # (they have lost their number); landmark 6 through its number
    xyz, ids, margin = t.map([1, 2], WS, rho, R[1:], tc[1:])
    assert ids.tolist() == [2, 3, 5, 6] and margin.tolist() == [True, True, True, True]
    t.solved[:] = False
    assert t.map([1, 2], WS, rho, R[1:], tc[1:])[2].tolist() == [False, False, False, True]


def test_reanchor_skips_a_gap_to_the_earliest_observation():
    t = chain(4, [[1], [], [1], [1]])
    t.window([0, 1, 2, 3], WS, np.zeros(0))
    R, tc = np.stack([np.eye(3)] * 4), np.zeros((4, 3))
    assert t.slide_reanchor([0, 1, 2, 3], True, np.array([0.5]), R, tc) == (0, 1)
    assert t.anchor.tolist() == [2] and t.rho.tolist() == [0.5]


def test_rule_boundaries_margin_second_new():
    # slot 2 (second newest) leaves: 7 is anchored there and seen in the newest slot, 8 is not, 9 is anchored earlier
    t = chain(4, [[9], [9], [7, 8, 9], [7, 9]])
    slots = [0, 1, 2, 3]
    rho_h = t.window(slots, WS, np.zeros(0))
    assert t.id[t.numbered].tolist() == [9, 7]                       # 7: start 2 < WS - 2, used_num 2
    rho = np.array([0.5, 0.2])
    t.rho[t.id == 8] = 0.75
    removed, moved = t.slide_reanchor(slots, False, rho)
    assert (removed, moved) == (1, 1)
    assert t.id.tolist() == [9, 7] and t.anchor.tolist() == [0, 3]
    assert t.rho.tolist()[1] == 0.2 and t.lm.tolist()[1] == -1 and t.solved.tolist() == [False, True]
    assert t.idx[:, 2].tolist() == [-1, -1] and t.idx[0, 3] == 1
    rho2 = t.window([0, 1, 3], WS, rho)
    assert t.id[t.numbered].tolist() == [9] and rho2.tolist() == [0.5]


def test_runner_reanchor_requires_device_features():
    with pytest.raises(ValueError):
        st.ResidentRunner(None, None, triangulate=True, reanchor=True)


# ---------------------------------------------------------------------------------------------------------------------
# GPU

def bitwise(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def engine(cuda_lib, seq):
    return pkg.Estimator(cuda_lib, pkg.make_config(**seq.config_kwargs()))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["margin_old", "second_new_every_3", "min_parallax"])
def test_device_reanchor_matches_host_restatement(cuda_lib, mode):
    n = 40
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    clouds = st.FrameClouds(seq)
    decide = decision_rule(seq, mode, n)
    e = engine(cuda_lib, seq)
    e.SetKnots(seq.q0, seq.p0); e.SetBiases(seq.bias0[:2]); e.SetLineDelay(seq.ld0)
    r = types.SimpleNamespace(n_slots=16, slot_of={})
    t = st.FeatureTable()
    rng = np.random.default_rng(5)

    def add(f):
        s = st.ResidentRunner._assign_slot(r, f)
        m_ = clouds.message(f)
        e.IngestFeatureCloud(s, int(seq.kf_times[f]), *m_)
        assert e.FeatureTableAdd(s) == t.add(s, m_)

    frames = list(range(st.WIN_KF))
    for f in frames:
        add(f)
    nxt, rho, flags, moved_ids, worst, total_moved = st.WIN_KF, np.zeros(0), set(), set(), 0.0, 0
    for k in range(n):
        if k:
            frames.append(nxt); add(nxt); nxt += 1
        slots = np.array([r.slot_of[f] for f in frames], np.int32)
        marg = bool(decide(frames))
        flags.add(marg)
        rho_h = t.window(slots, WS, rho)
        n_lm = e.FeatureTableWindow(slots, WS)
        assert n_lm == len(t.numbered)
        ids, anchor, used = e.FeatureTableLandmarks()
        hi, ha, hu = t.landmarks()
        assert np.array_equal(ids, hi) and np.array_equal(anchor, ha) and np.array_equal(used, hu), k
        # bitwise, except the depths a re-anchoring slide computed (device spline against syn.spline_pose)
        rho_d = e.GetInvDepths()
        shifted = np.isin(hi, list(moved_ids))
        assert bitwise(rho_d[~shifted], rho_h[~shifted]), k
        assert np.allclose(rho_d[shifted], rho_h[shifted], rtol=1e-12, atol=0.0), k
        if shifted.any():
            worst = max(worst, float(np.max(np.abs(rho_d[shifted] / rho_h[shifted] - 1.0))))
        rho = solved_depths(seq, hi, rng)
        e.SetInvDepths(rho)
        q, p = e.GetKnots()
        R_c, t_c = spline_camera_poses(q, p, seq.kf_times[frames], seq.t0_ns, seq.dt_ns)
        before = dict(zip(t.id.tolist(), t.anchor.tolist()))
        out = e.FeatureTableSlideReanchor(slots, marg, INIT_DEPTH)
        assert out == t.slide_reanchor(slots, marg, rho, R_c, t_c, INIT_DEPTH), k
        total_moved += out[1]
        moved_ids |= {i for i, a in zip(t.id.tolist(), t.anchor.tolist()) if before[i] != a}
        r.slot_of.pop(frames.pop(0 if marg else -2))
        post = np.array([r.slot_of[f] for f in frames], np.int32)
        xyz, mid, margin, _, cp = e.FeatureTableMap(post, WS)
        R_p, t_p = spline_camera_poses(q, p, seq.kf_times[frames], seq.t0_ns, seq.dt_ns)
        xyz_h, mid_h, margin_h = t.map(post, WS, rho, R_p, t_p)
        assert np.array_equal(mid, mid_h) and np.array_equal(margin, margin_h), k
        scale = max(np.abs(xyz_h).max(initial=0.0), 1.0)
        assert np.abs(xyz - xyz_h).max(initial=0.0) <= 1e-12 * scale, k
    assert total_moved > 0
    assert flags == ({True} if mode == "margin_old" else {True, False})
    print(mode, "re-anchored", total_moved, "worst relative difference of a shifted inverse depth", worst)


def raw_reanchor(e, slots, marg_old, init_depth):
    slots = np.ascontiguousarray(slots, np.int32)
    nr, na = C.c_int32(-5), C.c_int32(-5)
    rc = e.lib.raw("feature_table_slide_reanchor")(e.h, C.c_int32(len(slots)), pkg.binding._addr(slots),
                                                   C.c_int32(marg_old), C.c_double(init_depth), C.byref(nr), C.byref(na))
    return rc, nr.value, na.value


@pytest.mark.gpu
def test_error_paths_leave_table_and_state_unchanged(cuda_lib):
    seq = st.config_c5_sequence(1)
    clouds = st.FrameClouds(seq)
    e = engine(cuda_lib, seq)
    t = st.FeatureTable()
    for s in range(4):
        m = clouds.message(s)
        e.IngestFeatureCloud(s, int(seq.kf_times[s]), *m)
        assert e.FeatureTableAdd(s) == t.add(s, m)
    INVALID, STATE, TIME_RANGE = -1, -4, -6
    slots = [0, 1, 2, 3]

    def refused(code, *a):
        rc, nr, na = raw_reanchor(e, *a)
        assert rc == code and nr == -5 and na == -5, (rc, a)

    refused(STATE, slots, 1, INIT_DEPTH)                             # knots not set (MARGIN_OLD)
    e.SetKnots(seq.q0, seq.p0); e.SetBiases(seq.bias0[:2]); e.SetLineDelay(seq.ld0)
    refused(INVALID, [0], 1, INIT_DEPTH)
    refused(INVALID, np.arange(17) % 16, 1, INIT_DEPTH)
    refused(INVALID, [0, 1, 2, 16], 1, INIT_DEPTH)
    refused(INVALID, [0, 1, -1, 3], 0, INIT_DEPTH)
    refused(INVALID, [0, 1, 1, 3], 1, INIT_DEPTH)
    for bad in (0.0, -1.0, np.nan, np.inf):
        refused(INVALID, slots, 1, bad)
    refused(STATE, [0, 1, 2], 1, INIT_DEPTH)                         # not the held slots
    refused(STATE, [0, 1, 2, 3, 4], 0, INIT_DEPTH)
    rho_h = t.window(slots, WS, np.zeros(0))
    assert e.FeatureTableWindow(slots, WS) == len(rho_h) > 0
    rho = seq.rho_gt[t.id[t.numbered]]
    e.SetInvDepths(np.concatenate([rho, [1.0]]))                     # a different landmark count
    refused(STATE, slots, 1, INIT_DEPTH)
    refused(STATE, slots, 0, INIT_DEPTH)
    e.SetInvDepths(rho)
    q0, p0 = e.GetKnots()
    e.SlideWindow(1, 1, 1)                                           # the oldest frame's time leaves the spline
    refused(TIME_RANGE, slots, 1, INIT_DEPTH)
    assert bitwise(e.GetInvDepths(), rho)
    # after every refusal, the table and the depths are the restatement's: a MARGIN_SECOND_NEW slide needs no pose
    assert e.FeatureTableSlideReanchor(slots, 0, INIT_DEPTH) == t.slide_reanchor(slots, 0, rho)
    post = [0, 1, 3]
    rho_h = t.window(post, WS, rho)
    assert e.FeatureTableWindow(post, WS) == len(rho_h)
    assert bitwise(e.GetInvDepths(), rho_h)
    ids, anchor, used = e.FeatureTableLandmarks()
    hi, ha, hu = t.landmarks()
    assert np.array_equal(ids, hi) and np.array_equal(anchor, ha) and np.array_equal(used, hu)
    assert bitwise(e.GetKnots()[0], q0[1:]) and bitwise(e.GetKnots()[1], p0[1:])


def full_table_run(cuda_lib, seed=11):
    """16 slots x 1024 features with overlapping ids: a MARGIN_OLD and a MARGIN_SECOND_NEW re-anchoring slide, with the
    window, depths, landmarks and map after each; returns every device output"""
    rng = np.random.default_rng(seed)
    seq = st.config_c5_sequence(6)                                   # 16 keyframes
    e = engine(cuda_lib, seq)
    e.SetKnots(seq.q0, seq.p0)
    t = st.FeatureTable()
    for s in range(16):
        ids = rng.choice(20000, 1024, replace=False)                 # float32 carries ids < 2^24 exactly
        m = msg(ids, rng.uniform(-0.5, 0.5, (1024, 2)))
        e.IngestFeatureCloud(s, int(seq.kf_times[s]), *m)
        assert e.FeatureTableAdd(s) == t.add(s, m)
    q, p = e.GetKnots()
    R_c, t_c = spline_camera_poses(q, p, seq.kf_times[:16], seq.t0_ns, seq.dt_ns)
    slots = list(range(16))
    out, rho = [], np.zeros(0)
    for marg in (True, False):
        rho_h = t.window(slots, 16, rho)
        n_lm = e.FeatureTableWindow(slots, 16)
        assert n_lm == len(t.numbered)
        rho = rng.uniform(-0.05, 1.0, n_lm)
        e.SetInvDepths(rho)
        pos = np.asarray(slots)
        r = e.FeatureTableSlideReanchor(slots, marg, INIT_DEPTH)
        assert r == t.slide_reanchor(slots, marg, rho, R_c[pos], t_c[pos], INIT_DEPTH)
        assert r[1] > 10
        out.append(r)
        slots.pop(0 if marg else -2)
        out.append(e.FeatureTableMap(slots, 16))
        rho_h = t.window(slots, 16, rho)
        assert e.FeatureTableWindow(slots, 16) == len(rho_h)
        out += [e.FeatureTableLandmarks(), e.GetInvDepths()]
        assert np.allclose(out[-1], rho_h, rtol=1e-12, atol=0.0)
        rho = out[-1]
    return out


@pytest.mark.gpu
def test_full_tables_are_bitwise_reproducible(cuda_lib):
    a, b = full_table_run(cuda_lib), full_table_run(cuda_lib)
    for x, y in zip(a, b):
        if isinstance(x, tuple) and isinstance(x[0], np.ndarray):
            assert all(bitwise(u, v) if u.dtype == np.float64 else np.array_equal(u, v) for u, v in zip(x, y))
        elif isinstance(x, np.ndarray):
            assert bitwise(x, y)
        else:
            assert x == y


# the triangulating runner's bound (test_resident_triangulation.STATE_ERROR_BOUND) and the published map's
# (test_resident_map.GT_MEDIAN_BOUND_M)
STATE_ERROR_BOUND = 0.15
GT_MEDIAN_BOUND_M = 0.3


def true_world_points(seq):
    """every landmark's world point from its anchor observation (bearing, row time) and true inverse depth"""
    first = np.full(len(seq.rho_gt), -1); lms, i0 = np.unique(seq.lm, return_index=True); first[lms] = i0
    t = seq.ti[first] + (seq.rowi[first].astype(np.int64) * np.int64(int(seq.ld_gt * 1e9)))
    R, tc = spline_camera_poses(seq.q_gt, seq.p_gt, t, seq.t0_ns, seq.dt_ns)
    xy1 = np.concatenate([seq.pi[first], np.ones((len(first), 1))], 1)
    return np.einsum("lij,lj->li", R, xy1 / seq.rho_gt[:, None]) + tc


@pytest.mark.gpu
def test_whole_runner_with_reanchoring(cuda_lib):
    """ResidentRunner(reanchor=True) on C5 against the default device-feature runner.  Measured on an H100 80GB HBM3
    (400 W, DESIGN §6) on the 40-window C5 sequence: the solve tracks the default runner through window 7 (0.119 m
    against 0.105 m, within the triangulating runner's bound) and diverges in window 8 (on this 9-window sequence window
    8 still held: 0.045 m).  Like the reference's UpdateVIOPrior, every MARGIN_OLD flags all factors of the landmarks anchored in
    the oldest frame for marginalization; a re-anchored landmark keeps its later observations in the window, so each of
    them is marginalized into the prior again at every following slide (up to 9 times on C5, where every landmark is
    tracked over the whole window).  By window 8 the prior is that over-confident; with the image factors' marginalization
    flags switched off the same runner ends at 0.085 m after 16 windows (the default: 0.190 m).  The test pins windows
    0-7 and the structure of window 8's map, and prints the rest."""
    n = 9
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    r = st.ResidentRunner(cuda_lib, seq, triangulate=True, device_features=True, reanchor=True, publish_map=True)
    d = st.ResidentRunner(cuda_lib, seq, triangulate=True, device_features=True)
    p_true = true_world_points(seq)
    dist, err = [], []
    for _ in range(n):
        r.step()
        d.step()
        xyz, ids, _, _, _ = r.last_map
        dist.append(np.linalg.norm(xyz - p_true[ids], axis=1))
        err.append((r.state_error(), d.state_error()))
    lm_re, lm_def = [x["n_lm"] for x in r.records], [x["n_lm"] for x in d.records]
    margin = [x["n_margin_points"] for x in r.records]
    med = float(np.median(np.concatenate(dist[:8])))
    print(f"state_error per window (reanchor, default): {[(round(a, 4), round(b, 4)) for a, b in err]}; "
          f"n_lm {lm_re} vs {lm_def}; n_obs {[x['n_obs'] for x in r.records]} vs {[x['n_obs'] for x in d.records]}; "
          f"iterations {[x['iterations'] for x in r.records]} vs {[x['iterations'] for x in d.records]}; "
          f"reanchored {[x['n_reanchored'] for x in r.records]}; margin {margin}; map median (windows 0-7) {med:.4f} m")
    for k in range(8):
        assert np.isfinite(r.records[k]["final_cost"]) and np.isfinite(err[k][0]), k
    assert err[7][0] <= STATE_ERROR_BOUND, err
    assert lm_re[0] == lm_def[0] and all(a > b for a, b in zip(lm_re[1:], lm_def[1:]))
    assert all(x["marg_flag"] == st.MARGIN_OLD for x in r.records)
    assert [x["n_reanchored"] for x in r.records[:8]] == [30 * (k + 1) for k in range(8)]
    # a landmark anchored in frame a is seen in a .. a+10; re-anchored slide by slide, it is down to its last two
    # observations (start 0, used_num 2: the margin cloud) after the slide that drops frame a+8, so the first margin
    # cloud is the 30 landmarks of frame 0, after window 8's slide
    assert margin == [0] * 8 + [30]
    assert med <= GT_MEDIAN_BOUND_M
