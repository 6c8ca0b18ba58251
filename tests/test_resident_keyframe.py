"""The keyframe decision (ctvio_check_keyframe, the reference's addFeatureCheckParallax) on the resident frame table, and
the MARGIN_SECOND_NEW slide of the device-resident window (ctvio_slide_window_second_new).

The host restatement streaming.keyframe_decision is pinned on hand-built clouds (CPU); the device call is compared with
it over a C5 sequence, and the resident runner taking both branches is compared with the host-buffer runner, which
test_c5_streaming_windows_match_oracle[3] pins to the oracle."""
import importlib
import types

import numpy as np
import pytest

from helpers import pkg, rot_angle_between, syn

st = importlib.import_module("ctrl-vio_b200.streaming")

MIN_PARALLAX_REF = 10.0 / 740.0   # keyframe_parallax / focal length (cam_tumrs.yaml)


def msg(ids, xy):
    """a tracker message as FrameClouds.message returns it: float32 points (z = 1), id, u, v, vx, vy channels"""
    ids = np.asarray(ids, np.float32)
    n = len(ids)
    pts = np.ones((n, 3), np.float32)
    pts[:, :2] = np.broadcast_to(np.asarray(xy, np.float32), (n, 2))
    z = np.zeros(n, np.float32)
    return pts, ids, z, z, z, z


def test_fewer_than_three_frames_is_a_keyframe():
    a = msg(np.arange(40), (0.0, 0.0))
    b = msg(np.arange(40), (0.5, 0.5))
    assert st.keyframe_decision([a], 1e9) == (True, 0, 0, 0.0)
    kf, n_tracked, num, s = st.keyframe_decision([a, b], 1e9)
    assert kf and n_tracked == 40 and num == 0 and s == 0.0


def test_twenty_tracked_features_decide_by_parallax():
    older = msg(np.arange(30), (0.0, 0.0))
    prev = msg(np.arange(30), (0.375, 0.5))                    # parallax 0.625 for every feature
    new_ids = lambda k: np.concatenate([np.arange(k), 1000 + np.arange(15)])
    few = st.keyframe_decision([older, prev, msg(new_ids(19), (0.1, 0.1))], 1.0)
    assert few == (True, 19, 30, 30 * 0.625)                   # 19 tracked: a keyframe whatever the parallax
    enough = st.keyframe_decision([older, prev, msg(new_ids(20), (0.1, 0.1))], 1.0)
    assert enough == (False, 20, 30, 30 * 0.625)               # 20 tracked: 0.625 < 1.0 decides
    assert st.keyframe_decision([older, prev, msg(new_ids(20), (0.1, 0.1))], 0.625)[0]


def test_no_common_feature_before_the_new_frame_is_a_keyframe():
    older = msg(np.arange(30), (0.0, 0.0))
    prev = msg(30 + np.arange(30), (0.0, 0.0))
    kf, n_tracked, num, s = st.keyframe_decision([older, prev, msg(np.arange(60), (0.0, 0.0))], 1e9)
    assert kf and n_tracked == 60 and num == 0 and s == 0.0


def test_known_mean_just_below_and_above_the_threshold():
    # 16 features with parallax 0.625 and 16 with 0.3125, exact in float32 and float64: mean 0.46875
    ids = np.arange(32)
    older = msg(ids, (0.0, 0.0))
    xy = np.where((ids < 16)[:, None], [[0.375, 0.5]], [[0.1875, 0.25]])
    prev = msg(ids, xy)
    new = msg(ids[::-1], (0.0, 0.0))
    mean = 0.46875
    kf, n_tracked, num, s = st.keyframe_decision([older, prev, new], mean * (1 - 1e-12))
    assert (kf, n_tracked, num, s) == (True, 32, 32, 32 * mean)
    assert st.keyframe_decision([older, prev, new], mean)[0]
    assert not st.keyframe_decision([older, prev, new], mean * (1 + 1e-12))[0]


def test_ids_seen_only_in_an_older_frame_count_as_tracked():
    oldest = msg(np.arange(25), (0.0, 0.0))
    older = msg(100 + np.arange(40), (0.0, 0.0))
    prev = msg(100 + np.arange(40), (0.0, 0.25))
    new = msg(np.arange(25), (0.0, 0.0))                         # none of its ids is in the two frames before it
    kf, n_tracked, num, s = st.keyframe_decision([oldest, older, prev, new], 0.2)
    assert (kf, n_tracked, num, s) == (True, 25, 40, 40 * 0.25)
    assert not st.keyframe_decision([oldest, older, prev, new], 0.3)[0]


def test_frame_slot_allocator():
    runner = types.SimpleNamespace(n_slots=16, slot_of={})
    assign = lambda f: st.ResidentRunner._assign_slot(runner, f)
    assert [assign(f) for f in range(11)] == list(range(11))
    for f in range(11, 40):                                      # MARGIN_OLD only: always f % 16
        del runner.slot_of[f - 11]
        assert assign(f) == f % 16
    runner.slot_of = {f: f % 16 for f in (20, 22, 24, 26, 28, 30, 33, 34, 35)}   # a window spanning 16 frames
    assert assign(36) == 0                                       # 36 % 16 is frame 20's: the lowest free slot
    assert assign(37) == 5                                       # 37 % 16 is free


# ---------------------------------------------------------------------------------------------------------------------
# GPU

N_SLOTS = 16


def consecutive_windows(seq, n_windows):
    """(frames, messages) of each window of n_windows consecutive-keyframe windows"""
    clouds = st.FrameClouds(seq)
    out = []
    for k in range(n_windows):
        frames = list(range(k, k + st.WIN_KF))
        out.append((frames, [clouds.message(f) for f in frames]))
    return clouds, out


def median_mean_parallax(windows):
    means = []
    for _, msgs in windows:
        _, _, num, s = st.keyframe_decision(msgs, 0.0)
        means.append(s / num)
    return float(np.median(means))


@pytest.mark.gpu
def test_device_keyframe_decision_matches_host(cuda_lib):
    n_windows = 40
    seq = st.quantize_wire(st.config_c5_sequence(n_windows))
    clouds, windows = consecutive_windows(seq, n_windows)
    thresholds = (MIN_PARALLAX_REF, median_mean_parallax(windows))
    e = pkg.Estimator(cuda_lib, pkg.make_config(**seq.config_kwargs()))
    ingested = set()
    outcomes = {m: set() for m in thresholds}
    for frames, msgs in windows:
        for f, m in zip(frames, msgs):
            if f not in ingested:                                  # rotating slots, every frame once
                e.IngestFeatureCloud(f % N_SLOTS, int(seq.kf_times[f]), *m)
                ingested.add(f)
        slots = np.asarray(frames) % N_SLOTS
        for m in thresholds:
            kf_h, nt_h, num_h, sum_h = st.keyframe_decision(msgs, m)
            kf_d, nt_d, num_d, sum_d = e.CheckKeyframe(slots, m)
            assert (nt_d, num_d) == (nt_h, num_h), (frames[0], m)
            assert abs(sum_d - sum_h) <= 1e-12 * abs(sum_h)
            if abs(sum_h / num_h - m) > 1e-9 * m:
                assert kf_d == kf_h, (frames[0], m, sum_h / num_h)
            outcomes[m].add(kf_d)
            again = e.CheckKeyframe(slots, m)
            assert again[:3] == (kf_d, nt_d, num_d)
            assert np.float64(again[3]).view(np.int64) == np.float64(sum_d).view(np.int64)   # bitwise
    assert outcomes[thresholds[1]] == {True, False}
    print(f"thresholds {thresholds}: outcomes {outcomes}")


@pytest.mark.gpu
def test_device_keyframe_decision_edge_cases(cuda_lib):
    """the hand-built clouds of the CPU tests, an empty cloud and a slot never ingested, on the device"""
    seq = st.config_c5_sequence(1)
    e = pkg.Estimator(cuda_lib, pkg.make_config(**seq.config_kwargs()))
    ids = np.arange(32)
    xy = np.where((ids < 16)[:, None], [[0.375, 0.5]], [[0.1875, 0.25]])
    prev = msg(ids, xy)
    clouds = [msg(ids, (0.0, 0.0)), prev, msg(ids[::-1], (0.0, 0.0)), msg([], (0.0, 0.0)), msg(1000 + np.arange(19), (0, 0))]
    for s, m in enumerate(clouds):
        e.IngestFeatureCloud(s, 0, *m)
    mean = 0.46875
    for m in (mean * (1 - 1e-12), mean, mean * (1 + 1e-12)):
        assert e.CheckKeyframe([0, 1, 2], m) == st.keyframe_decision(clouds[:3], m)
    assert e.CheckKeyframe([2], 1.0) == (True, 0, 0, 0.0)
    assert e.CheckKeyframe([0, 2], 1.0) == (True, 32, 0, 0.0)
    assert e.CheckKeyframe([0, 1, 3], 1.0) == (True, 0, 32, 32 * mean)       # empty new cloud
    assert e.CheckKeyframe([3, 9, 2], 1.0) == (True, 0, 0, 0.0)              # empty and never-ingested slots
    assert e.CheckKeyframe([0, 1, 4], 0.0) == st.keyframe_decision([clouds[0], clouds[1], clouds[4]], 0.0)


@pytest.mark.gpu
def test_keyframe_and_second_new_error_paths(cuda_lib):
    seq = st.config_c5_sequence(1)
    e = pkg.Estimator(cuda_lib, pkg.make_config(**seq.config_kwargs()))
    for s in range(3):
        e.IngestFeatureCloud(s, 0, *msg(np.arange(30), (0.0, 0.01 * s)))
    invalid = r"\(-1\)"
    with pytest.raises(pkg.CtvioError, match=invalid):
        e.CheckKeyframe(np.zeros(0, np.int32), 0.01)
    with pytest.raises(pkg.CtvioError, match=invalid):
        e.CheckKeyframe(np.arange(17) % 16, 0.01)
    for slots in ([0, 1, 16], [-1, 1, 2], [0, 1, 1], [2, 0, 2]):
        with pytest.raises(pkg.CtvioError, match=invalid):
            e.CheckKeyframe(slots, 0.01)
    for m in (-1e-3, float("nan"), float("inf")):
        with pytest.raises(pkg.CtvioError, match=invalid):
            e.CheckKeyframe([0, 1, 2], m)
    kf, n_tracked, num, s = e.CheckKeyframe([0, 1, 2], 0.01)      # the valid call still works
    assert (kf, n_tracked, num) == (False, 30, 30) and np.isclose(s, 30 * float(np.float32(0.01)), rtol=1e-12)
    # SlideWindowSecondNew: fewer than 2 bias nodes
    state = r"\(-4\)"
    with pytest.raises(pkg.CtvioError, match=state):
        e.SlideWindowSecondNew()
    e.SetKnots(seq.q0[:8], seq.p0[:8])
    e.SetBiases(seq.bias0[:1])
    with pytest.raises(pkg.CtvioError, match=state):
        e.SlideWindowSecondNew()


def bias_prior(node):
    """a 3-column prior on the gyro bias of one node"""
    return pkg.PriorData(n=3, J=np.eye(3), r=np.zeros(3), blk_type=np.array([pkg.binding.BLK_BG], np.int32),
                         blk_index=np.array([node], np.int32), blk_col=np.zeros(1, np.int32), blk_x0=np.zeros((1, 4)))


@pytest.mark.gpu
def test_second_new_slide_moves_one_bias_node(cuda_lib):
    seq = st.config_c5_sequence(1)
    e = pkg.Estimator(cuda_lib, pkg.make_config(**seq.config_kwargs()))
    nB = 6
    q, p = seq.q0[:10].copy(), seq.p0[:10].copy()
    b = np.random.default_rng(3).normal(size=(nB, 6))
    e.SetKnots(q, p); e.SetBiases(b)
    e.AddMarginalizationFactor(bias_prior(nB - 2))
    with pytest.raises(pkg.CtvioError, match=r"\(-4\)"):
        e.SlideWindowSecondNew()
    assert np.array_equal(e.GetBiases(), b)                  # nothing changed
    e.AddMarginalizationFactor(bias_prior(0))
    e.SlideWindowSecondNew()
    expect = b.copy(); expect[nB - 2] = b[nB - 1]
    assert np.array_equal(e.GetBiases(), expect)
    qs, ps = e.GetKnots()
    assert np.array_equal(qs, q) and np.array_equal(ps, p)


def run_deterministic(a, b, n):
    """both runners in deterministic mode.  In the default mode the order of the atomic accumulation varies from run to
    run, and over 8 windows two runs of the same host-buffer chain already differ by up to ~4e-6 x scale at the spline's
    extended end, more than the tolerance; in deterministic mode the two paths give bitwise equal states."""
    for r in (a, b):
        r.est.SetDeterministic(True)
        r.run(n)


def assert_states_agree(a, b):
    """the tolerances of test_resident_window_matches_host_buffer_path"""
    assert [x["iterations"] for x in a.records] == [x["iterations"] for x in b.records]
    assert [x["prior_dim"] for x in a.records] == [x["prior_dim"] for x in b.records]
    assert [x["marg_flag"] for x in a.records] == [x["marg_flag"] for x in b.records]
    assert {x["marg_flag"] for x in b.records} == {st.MARGIN_OLD, st.MARGIN_SECOND_NEW}
    assert np.isclose(a.records[0]["final_cost"], b.records[0]["final_cost"], rtol=1e-9)
    scale = np.abs(a.p[:a.ncp]).max()
    print(f"max |dp| / scale {np.abs(a.p[:a.ncp] - b.p[:b.ncp]).max() / scale:.2e}, "
          f"max rotation {rot_angle_between(a.q[:a.ncp], b.q[:b.ncp]).max():.2e} rad, |dld| {abs(a.ld - b.ld):.2e}")
    assert np.abs(a.p[:a.ncp] - b.p[:b.ncp]).max() <= 1e-6 * scale
    assert rot_angle_between(a.q[:a.ncp], b.q[:b.ncp]).max() <= 1e-6
    assert abs(a.ld - b.ld) <= 1e-10
    assert a.frames == b.frames


@pytest.mark.gpu
@pytest.mark.parametrize("every,n", [(3, 8), (2, 14)])
def test_resident_second_new_slide_matches_host_buffer_path(cuda_lib, every, n):
    """every=2 skips so many frames that the window ends up spanning 17 source frames: slots leave the f % 16 rule"""
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    a = st.StreamingRunner(cuda_lib, seq, second_new_every=every)
    b = st.ResidentRunner(cuda_lib, seq, second_new_every=every)
    run_deterministic(a, b, n)
    assert_states_agree(a, b)
    assert sorted(b.slot_of) == b.frames and len(set(b.slot_of.values())) == len(b.frames)
    if every == 2:
        assert b.frames[-1] - b.frames[0] + 1 > N_SLOTS
        assert any(slot != f % N_SLOTS for f, slot in b.slot_of.items())
    print("marg flags", [x["marg_flag"] for x in b.records], "window frames", b.frames, "slots", b.slot_of)


@pytest.mark.gpu
def test_device_decided_cycle_matches_host_buffer_path(cuda_lib):
    n = 8
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    _, windows = consecutive_windows(seq, n)
    m = median_mean_parallax(windows)
    a = st.StreamingRunner(cuda_lib, seq, min_parallax=m)
    b = st.ResidentRunner(cuda_lib, seq, min_parallax=m)
    run_deterministic(a, b, n)
    assert_states_agree(a, b)
    for ra, rb in zip(a.records, b.records):
        assert ra["n_tracked"] == rb["n_tracked"]
        assert np.isclose(ra["mean_parallax"], rb["mean_parallax"], rtol=1e-12, atol=0.0)
    print(f"min_parallax {m:.6f}: flags {[x['marg_flag'] for x in b.records]}, "
          f"means {[round(x['mean_parallax'], 6) for x in b.records]}")
