"""The published landmark map of the resident window (ctvio_feature_table_map: GetLandmarksInWindow, GetMarginCloud and
the keyframe poses of PublishVioKeyFrame) and ResidentRunner(publish_map=True).

streaming.FeatureTable.map, the host restatement, is pinned on hand-built tables at every boundary of
IsLandMarkStable and GetMarginCloud (CPU).  On the GPU the device call is compared with it after every slide of the
device-feature runner, with poses from an independent evaluator (the knots read back through syn.spline_pose and a host
extrinsic composition); its error paths, reproducibility, transfer count and read-only behaviour are checked, and the
published map is compared with the one the sequence's ground truth gives."""
import ctypes as C
import importlib

import numpy as np
import pytest

from helpers import pkg, syn

st = importlib.import_module("ctrl-vio_b200.streaming")

WS = st.WINDOW_SIZE


def msg(ids, xy):
    """a tracker message (FrameClouds.message layout): float32 points (x, y, 1), id, u, v, vx, vy channels"""
    ids = np.asarray(ids, np.float32)
    n = len(ids)
    pts = np.ones((n, 3), np.float32)
    pts[:, :2] = np.asarray(xy, np.float32).reshape(n, 2)
    z = np.zeros(n, np.float32)
    return pts, ids, z, z, z, z


def bearing(i):
    return (0.01 * i, -0.02 * i + 0.1)


def wire(i):
    """id i's bearing as the message carries it (float32)"""
    return tuple(float(np.float32(v)) for v in bearing(i))


def table_of(tracks, n_slots):
    """FeatureTable over slots 0 .. n_slots-1 from {id: [slots]} (the first slot the anchor); each slot's cloud lists
    its ids in ascending order"""
    t = st.FeatureTable()
    for s in range(n_slots):
        ids = sorted(i for i, sl in tracks.items() if s in sl)
        t.add(s, msg(ids, [bearing(i) for i in ids]))
    return t


def identity_poses(n):
    return np.broadcast_to(np.eye(3), (n, 3, 3)), np.zeros((n, 3))


def test_stable_rule_boundaries_window_10():
    tracks = {
        1: [0],              # used_num 1
        2: [0, 1],           # used_num 2
        3: [0, 1, 2],        # used_num 3
        4: [7, 8],           # start = WS - 3
        5: [8, 9],           # start = WS - 2
        6: [3, 5, 11],       # observations in non-adjacent slots count
    }
    t = table_of(tracks, 12)
    assert t.id.tolist() == [1, 2, 3, 6, 4, 5]                      # table order: creation order (anchor slot, id)
    t.rho[:] = 0.5
    xyz, ids, margin = t.map(list(range(12)), WS, np.zeros(0), *identity_poses(12))
    assert ids.tolist() == [2, 3, 6, 4]
    assert not margin.any()                                          # nothing was numbered in a window
    x, y = wire(2)
    assert xyz[0].tolist() == [x * 2.0, y * 2.0, 2.0]                 # identity pose: the anchor bearing times depth 2


def test_three_quarter_rule_binds_at_window_16():
    tracks = {1: [12, 13], 2: [13, 14], 3: [11, 15]}
    t = table_of(tracks, 16)
    t.rho[:] = 1.0
    # start 12 == 16 * 3 / 4 passes, start 13 > 12 does not (though 13 < 16 - 2)
    assert t.map(list(range(16)), 16, np.zeros(0), *identity_poses(16))[1].tolist() == [3, 1]
    # at window_size 10 the same table's starts 11..13 fail the candidate rule first
    assert t.map(list(range(16)), WS, np.zeros(0), *identity_poses(16))[1].tolist() == []


def test_depth_values_and_numbering():
    tracks = {i: [0, 1] for i in range(1, 9)}
    t = table_of(tracks, 2)
    # stored inverse depths: -1 (never initialised), inf (depth 0), 0 (depth inf), NaN, 0.25
    t.rho[:] = [-1.0, np.inf, 0.0, np.nan, 0.25, -1.0, -1.0, 0.25]
    # entries 5, 6 and 7 were numbered 0, 1, 2 in the last window: their resident values replace the stored ones
    t.lm[:] = [-1, -1, -1, -1, -1, 0, 1, 2]
    rho = np.array([0.5, -0.5, np.nan])
    xyz, ids, margin = t.map([0, 1], 4, rho, *identity_poses(2))
    assert ids.tolist() == [3, 4, 5, 6, 8]                            # depth -1, 0 and the resident -2 fail; NaN passes
    assert margin.tolist() == [False, False, False, True, True]      # numbered: entry 6 (0.5) and entry 8 (NaN)
    assert xyz[2].tolist() == [wire(5)[0] * 4, wire(5)[1] * 4, 4.0]   # stored 0.25
    assert xyz[3].tolist() == [wire(6)[0] * 2, wire(6)[1] * 2, 2.0]   # resident 0.5, not the stored -1
    assert not np.isfinite(xyz[0]).any()                              # depth inf (inverse depth 0)
    assert np.isnan(xyz[1]).all() and np.isnan(xyz[4]).all()          # NaN depths


def test_margin_cloud_conditions():
    # all numbered in the last window with positive depths unless said otherwise
    tracks = {1: [0, 1], 2: [0, 1, 2], 3: [1, 2], 4: [0, 2], 5: [0, 1]}
    t = table_of(tracks, 3)
    t.rho[:] = 0.5
    t.lm[:] = [0, 1, 2, -1, 3]                                       # table order 1, 2, 4, 5, 3: id 5 is not numbered
    xyz, ids, margin = t.map([0, 1, 2], WS, np.full(4, 0.5), *identity_poses(3))
    assert ids.tolist() == [1, 2, 4, 5, 3]
    # 1: start 0, used 2, numbered; 2: used 3; 4: used 2 across a gap; 5: not numbered (no SovelSucc); 3: start 1
    assert margin.tolist() == [True, False, True, False, False]
    # a resident inverse-depth count shorter than the numbering: the entry keeps its stored value and is not numbered
    assert t.map([0, 1, 2], WS, np.full(1, 0.5), *identity_poses(3))[2].tolist() == [True, False, False, False, False]


def test_world_point_against_analytic_pose():
    t = table_of({7: [0, 1], 9: [1, 2]}, 3)
    t.rho[:] = [0.2, 0.4]
    th = np.array([0.0, 0.3, -0.7])
    R = np.zeros((3, 3, 3))
    R[:, 0, 0] = R[:, 1, 1] = np.cos(th); R[:, 0, 1] = -np.sin(th); R[:, 1, 0] = np.sin(th); R[:, 2, 2] = 1.0
    tc = np.array([[0.0, 0.0, 0.0], [1.0, 2.0, 3.0], [-1.0, 0.5, 2.0]])
    xyz, ids, _ = t.map([0, 1, 2], WS, np.zeros(0), R, tc)
    assert ids.tolist() == [7, 9]
    x, y = wire(9)
    d = 2.5
    c, s = np.cos(0.3), np.sin(0.3)
    want = [c * x * d - s * y * d + 1.0, s * x * d + c * y * d + 2.0, d + 3.0]
    assert np.allclose(xyz[1], want, rtol=0, atol=1e-14)


def test_camera_poses_compose_the_extrinsic():
    q = np.array([[0.0, 0.0, np.sin(0.2), np.cos(0.2)], [0.0, 0.0, 0.0, 1.0]])
    p = np.array([[1.0, 2.0, 3.0], [0.0, 0.0, 0.0]])
    R, t = st.camera_poses(q, p)
    Rz = np.array([[np.cos(0.4), -np.sin(0.4), 0], [np.sin(0.4), np.cos(0.4), 0], [0, 0, 1]])
    R_CI = st.quat_matrix(syn.Q_CtoI)[0]
    assert np.allclose(R[0], Rz @ R_CI, atol=1e-15) and np.allclose(t[0], p[0] + Rz @ syn.P_CinI, atol=1e-15)
    assert np.allclose(R[1], R_CI, atol=0) and np.allclose(t[1], syn.P_CinI, atol=0)
    assert np.allclose(R_CI, syn.R_CtoI, atol=1e-5)


def test_publish_map_requires_device_features():
    with pytest.raises(ValueError):
        st.ResidentRunner(None, None, triangulate=True, publish_map=True)


# ---------------------------------------------------------------------------------------------------------------------
# GPU

def bitwise(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def spline_camera_poses(q, p, times, t0_ns, dt_ns):
    """the independent evaluator: syn.spline_pose of the knots, then the extrinsic on the host"""
    qi, pi = syn.spline_pose(np.asarray(q), np.asarray(p), np.asarray(times, np.int64), t0_ns, dt_ns)
    return st.camera_poses(qi, pi)


class MapMirror:
    """Mirrors the runner's resident-table calls into a FeatureTable (asserting each count on the way) and checks every
    FeatureTableMap against FeatureTable.map, with camera poses from the knots read back right then."""

    NAMES = ("IngestFeatureCloud", "FeatureTableAdd", "FeatureTableWindow", "FeatureTableSlide", "FeatureTableMap")

    def __init__(self, runner, gt=False):
        self.r, self.t, self.msgs = runner, st.FeatureTable(), {}
        self.n_points, self.n_margin, self.gt_dist, self.worst = [], [], [], 0.0
        self.gt = gt
        e = runner.est
        orig = {n: getattr(e, n) for n in self.NAMES}

        def ingest(slot, t_ns, *m):
            orig["IngestFeatureCloud"](slot, t_ns, *m)
            self.msgs[slot] = m

        def add(slot):
            out = orig["FeatureTableAdd"](slot)
            assert out == self.t.add(slot, self.msgs[slot])
            return out

        def window(slots, ws):
            rho = e.GetInvDepths()
            n = orig["FeatureTableWindow"](slots, ws)
            self.t.window(slots, ws, rho)
            assert n == len(self.t.numbered)
            return n

        def slide(slot):
            rho = e.GetInvDepths()
            n = orig["FeatureTableSlide"](slot)
            assert n == self.t.slide(slot, rho)
            return n

        def fmap(slots, ws):
            out = orig["FeatureTableMap"](slots, ws)
            self.check(slots, ws, out)
            return out
        for n, f in zip(self.NAMES, (ingest, add, window, slide, fmap)):
            setattr(e, n, f)

    def check(self, slots, ws, out):
        r, e, s = self.r, self.r.est, self.r.seq
        xyz, ids, margin, cq, cp = out
        rho = e.GetInvDepths()
        q, p = e.GetKnots()
        t0 = s.t0_ns + (r.ncp - e.n_knots) * s.dt_ns               # the engine's knot 0 after the slide
        frame_of = {sl: f for f, sl in r.slot_of.items()}
        times = s.kf_times[[frame_of[int(x)] for x in slots]]
        R_c, t_c = spline_camera_poses(q, p, times, t0, s.dt_ns)
        xyz_h, ids_h, margin_h = self.t.map(slots, ws, rho, R_c, t_c)
        assert np.array_equal(ids, ids_h) and np.array_equal(margin, margin_h)
        scale = max(np.abs(xyz_h).max(initial=0.0), np.abs(t_c).max(), 1.0)
        err = max(np.abs(xyz - xyz_h).max(initial=0.0), np.abs(cp - t_c).max(), np.abs(st.quat_matrix(cq) - R_c).max())
        self.worst = max(self.worst, err / scale)
        assert err <= 1e-12 * scale, (err, scale)
        self.n_points.append(len(ids))
        self.n_margin.append(int(margin.sum()))
        if self.gt:
            self.gt_dist.append(self.gt_map_distance(slots, ws, times, xyz, ids))

    def gt_map_distance(self, slots, ws, times, xyz, ids):
        """distances between the published points and the map the restatement gives from the ground-truth knots and
        rho_gt (landmarks stable on both sides)"""
        s, t = self.r.seq, self.t
        stored = t.rho
        t.rho = s.rho_gt[t.id]
        rho_gt = np.zeros(len(t.numbered))
        rho_gt[t.lm[t.lm >= 0]] = s.rho_gt[t.id[t.lm >= 0]]
        try:
            R_g, t_g = spline_camera_poses(s.q_gt, s.p_gt, times, s.t0_ns, s.dt_ns)
            xyz_g, ids_g, _ = t.map(slots, ws, rho_gt, R_g, t_g)
        finally:
            t.rho = stored
        both, i, j = np.intersect1d(ids, ids_g, return_indices=True)
        return np.linalg.norm(xyz[i] - xyz_g[j], axis=1)


def median_parallax(seq, n):
    clouds = st.FrameClouds(seq)
    means = []
    for k in range(n):
        _, _, num, s = st.keyframe_decision([clouds.message(f) for f in range(k, k + st.WIN_KF)], 0.0)
        means.append(s / num)
    return float(np.median(means))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["margin_old", "second_new_every_2", "min_parallax"])
def test_device_map_matches_restatement_after_every_slide(cuda_lib, mode):
    n = 40
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    kw = {"margin_old": {}, "second_new_every_2": dict(second_new_every=2),
          "min_parallax": dict(min_parallax=median_parallax(seq, n))}[mode]
    r = st.ResidentRunner(cuda_lib, seq, triangulate=True, device_features=True, publish_map=True, **kw)
    m = MapMirror(r)
    r.run(n)
    assert len(m.n_points) == n
    assert [x["n_map_points"] for x in r.records] == m.n_points
    assert [x["n_margin_points"] for x in r.records] == m.n_margin
    # (C5's margin cloud is empty: a landmark leaves with its anchor frame, so an entry at start 0 after the slide was
    #  anchored in the frame after it and is tracked across the window; the flag is covered by the tests below)
    assert min(m.n_points) > 0
    flags = {x["marg_flag"] for x in r.records}
    assert flags == ({st.MARGIN_OLD} if mode == "margin_old" else {st.MARGIN_OLD, st.MARGIN_SECOND_NEW})
    print(mode, "points", m.n_points, "margin", m.n_margin, "worst relative difference", m.worst)


def raw_map(e, slots, ws, capacity, n_arrays=None, null_points=False, sentinel=-7.25):
    """ctvio_feature_table_map with every output filled with a sentinel; returns (rc, n_points, outputs)"""
    slots = np.ascontiguousarray(slots, np.int32)
    na = max(capacity, 1) if n_arrays is None else n_arrays
    nf = max(len(slots), 1)
    xyz, ids, flag = np.full((na, 3), sentinel), np.full(na, -7, np.int32), np.full(na, 77, np.uint8)
    cq, cp = np.full((nf, 4), sentinel), np.full((nf, 3), sentinel)
    n = C.c_int32(-5)
    a = pkg.binding._addr
    rc = e.lib.raw("feature_table_map")(e.h, C.c_int32(len(slots)), a(slots), C.c_int32(ws), C.c_int32(capacity),
                                        None if null_points else a(xyz), a(ids), a(flag), C.byref(n), a(cq), a(cp))
    return rc, n.value, (xyz, ids, flag, cq, cp)


def untouched(out, sentinel=-7.25):
    xyz, ids, flag, cq, cp = out
    return (xyz == sentinel).all() and (ids == -7).all() and (flag == 77).all() and (cq == sentinel).all() and \
        (cp == sentinel).all()


@pytest.mark.gpu
def test_error_paths_write_nothing(cuda_lib):
    seq = st.config_c5_sequence(1)
    clouds = st.FrameClouds(seq)
    e = pkg.Estimator(cuda_lib, pkg.make_config(**seq.config_kwargs()))
    t = st.FeatureTable()
    for s in range(3):
        m = clouds.message(s)
        e.IngestFeatureCloud(s, int(seq.kf_times[s]), *m)
        assert e.FeatureTableAdd(s) == t.add(s, m)
    INVALID, STATE, TIME_RANGE = -1, -4, -6

    def refused(code, *a, **k):
        rc, n, out = raw_map(e, *a, **k)
        assert rc == code and n == -5 and untouched(out), (rc, n)

    refused(STATE, [0, 1, 2], WS, 100)                               # knots not set
    e.SetKnots(seq.q0, seq.p0)
    e.SetLineDelay(seq.ld0)
    refused(INVALID, [], WS, 100)
    refused(INVALID, np.arange(17) % 16, WS, 100)
    refused(INVALID, [0, 1, 16], WS, 100)
    refused(INVALID, [0, -1, 2], WS, 100)
    refused(INVALID, [0, 1, 1], WS, 100)
    refused(INVALID, [0, 1, 2], 2, 100)
    refused(INVALID, [0, 1, 2], WS, -1)
    refused(INVALID, [0, 1, 2], WS, 100, null_points=True)
    refused(STATE, [0, 1], WS, 100)                                  # not the held slots
    refused(STATE, [0, 1, 2, 3], WS, 100)
    rho_h = t.window([0, 1, 2], WS, np.zeros(0))
    n_lm = e.FeatureTableWindow([0, 1, 2], WS)
    assert n_lm == len(rho_h) > 0
    rho = np.linspace(0.1, 0.5, n_lm)
    e.SetInvDepths(np.concatenate([rho, [1.0]]))                     # a different landmark count
    refused(STATE, [0, 1, 2], WS, 100)
    e.SetInvDepths(rho)
    # MARGIN_SECOND_NEW: slot 1 leaves, so the landmarks anchored in slot 0 keep used_num 2 (the margin cloud)
    assert e.FeatureTableSlide(1) == t.slide(1, rho)
    refused(STATE, [0, 1, 2], WS, 100)                               # slot 1 has left
    post = [0, 2]
    R_c, t_c = spline_camera_poses(seq.q0, seq.p0, seq.kf_times[post], seq.t0_ns, seq.dt_ns)
    xyz_h, ids_h, margin_h = t.map(post, WS, rho, R_c, t_c)
    n = len(ids_h)
    assert n > 1 and margin_h.any()
    # a capacity one below the count: refused, the count is reported, nothing else is written
    rc, n_dev, out = raw_map(e, post, WS, n - 1, n_arrays=n)
    assert rc == INVALID and n_dev == n and untouched(out)
    rc, n_dev, out = raw_map(e, post, WS, 0, n_arrays=1, null_points=True)
    assert rc == INVALID and n_dev == n and untouched(out)
    rc, n_dev, (xyz, ids, flag, cq, cp) = raw_map(e, post, WS, n)
    assert rc == 0 and n_dev == n
    assert np.array_equal(ids, ids_h) and np.array_equal(flag.astype(bool), margin_h)
    assert np.abs(xyz - xyz_h).max() <= 1e-12 * np.abs(xyz_h).max()
    assert np.abs(cp - t_c).max() <= 1e-12 * np.abs(t_c).max() and np.abs(st.quat_matrix(cq) - R_c).max() <= 1e-12
    # NULL pose arrays are allowed
    nn = C.c_int32()
    xyz2, ids2, flag2 = np.zeros((n, 3)), np.zeros(n, np.int32), np.zeros(n, np.uint8)
    a = pkg.binding._addr
    slots = np.asarray(post, np.int32)
    assert e.lib.raw("feature_table_map")(e.h, C.c_int32(2), a(slots), C.c_int32(WS), C.c_int32(n), a(xyz2), a(ids2),
                                          a(flag2), C.byref(nn), None, None) == 0
    assert nn.value == n and bitwise(xyz2, xyz) and np.array_equal(ids2, ids)
    # a listed frame time outside the spline
    m = clouds.message(3)
    e.IngestFeatureCloud(3, int(seq.kf_times[-1]) + 10 ** 10, *m)
    assert e.FeatureTableAdd(3) == t.add(3, m)
    refused(TIME_RANGE, [0, 2, 3], WS, 100)
    # the refused calls changed nothing: the table slides as the restatement's does
    assert e.FeatureTableSlide(3) == t.slide(3, rho)
    assert bitwise(e.GetInvDepths(), rho)
    xyz3, ids3, margin3, _, _ = e.FeatureTableMap(post, WS)
    assert bitwise(xyz3, xyz) and np.array_equal(ids3, ids) and np.array_equal(margin3, margin_h)


def full_table(cuda_lib, seed=11):
    rng = np.random.default_rng(seed)
    seq = st.config_c5_sequence(6)                                   # 16 keyframes
    e = pkg.Estimator(cuda_lib, pkg.make_config(**seq.config_kwargs()))
    e.SetKnots(seq.q0, seq.p0)
    t = st.FeatureTable()
    for s in range(16):
        ids = rng.choice(20000, 1024, replace=False)
        m = msg(ids, rng.uniform(-0.5, 0.5, (1024, 2)))
        e.IngestFeatureCloud(s, int(seq.kf_times[s]), *m)
        assert e.FeatureTableAdd(s) == t.add(s, m)
    slots = np.arange(16, dtype=np.int32)
    t.window(slots, 16, np.zeros(0))
    n_lm = e.FeatureTableWindow(slots, 16)
    assert n_lm == len(t.numbered)
    rho = rng.uniform(-0.05, 1.0, n_lm)
    e.SetInvDepths(rho)
    assert e.FeatureTableSlide(0) == t.slide(0, rho)
    return e, t, seq, slots[1:], rho


@pytest.mark.gpu
def test_full_tables_bitwise_and_transfer_count(cuda_lib):
    e, t, seq, slots, rho = full_table(cuda_lib)
    e.TransferStats(reset=True)
    a = e.FeatureTableMap(slots, 16)
    h2d, d2h = e.TransferStats(reset=True)
    n = len(a[1])
    assert n > 1000 and a[2].any() and not a[2].all()
    assert h2d == 0 and d2h == 8 + 56 * len(slots) + 32 * n
    b = e.FeatureTableMap(slots, 16)
    assert all(bitwise(x, y) if x.dtype == np.float64 else np.array_equal(x, y) for x, y in zip(a, b))
    e2, *_ = full_table(cuda_lib)
    c = e2.FeatureTableMap(slots, 16)
    assert all(bitwise(x, y) if x.dtype == np.float64 else np.array_equal(x, y) for x, y in zip(a, c))
    q, p = e.GetKnots()
    R_c, t_c = spline_camera_poses(q, p, seq.kf_times[slots], seq.t0_ns, seq.dt_ns)
    xyz_h, ids_h, margin_h = t.map(slots, 16, rho, R_c, t_c)
    assert np.array_equal(a[1], ids_h) and np.array_equal(a[2], margin_h)
    assert np.abs(a[0] - xyz_h).max() <= 1e-12 * np.abs(xyz_h).max()


@pytest.mark.gpu
def test_publish_map_only_reads(cuda_lib):
    n = 8
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    a = st.ResidentRunner(cuda_lib, seq, triangulate=True, device_features=True)
    b = st.ResidentRunner(cuda_lib, seq, triangulate=True, device_features=True, publish_map=True)
    for x in (a, b):
        x.est.SetDeterministic(True)
        x.run(n)
    for key in ("n_obs", "n_lm", "n_triangulated", "n_fallback", "iterations", "marg_flag", "prior_dim", "n_removed"):
        assert [x[key] for x in a.records] == [x[key] for x in b.records], key
    assert all(x["n_map_points"] > 0 for x in b.records) and "n_map_points" not in a.records[0]
    assert a.frames == b.frames and a.ncp == b.ncp
    assert bitwise(a.q[:a.ncp], b.q[:b.ncp]) and bitwise(a.p[:a.ncp], b.p[:b.ncp])
    assert bitwise(a.est.GetBiases(), b.est.GetBiases())
    assert bitwise(a.est.GetInvDepths(), b.est.GetInvDepths())
    assert bitwise(a.ld, b.ld)


# median distance (m) between the published map and the ground-truth map over the triangulating C5 run: measured
# 0.227 m (90th percentile 0.81 m, 8 400 points) on an H100 80GB HBM3 (DESIGN §6)
GT_MEDIAN_BOUND_M = 0.3


@pytest.mark.gpu
def test_published_map_near_ground_truth(cuda_lib):
    n = 40
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    r = st.ResidentRunner(cuda_lib, seq, triangulate=True, device_features=True, publish_map=True)
    m = MapMirror(r, gt=True)
    r.run(n)
    d = np.concatenate(m.gt_dist)
    med = float(np.median(d))
    print("ground-truth map distance: median", med, "90th percentile", float(np.percentile(d, 90)), "points", len(d))
    assert len(d) > 1000 and med <= GT_MEDIAN_BOUND_M
