"""The resident feature table (ctvio_feature_table_*, FeatureManager's feature list on the device) and the resident runner
that takes its landmarks, triangulation and image factors from it.

streaming.FeatureTable, the host restatement, is pinned on hand-built clouds and tied to the host path's association
(subwindow_frames + _observation_csr) on the C5 sequence (CPU); the device calls are compared with it after every call,
and ResidentRunner(device_features=True) is compared bitwise with the host-association runner (GPU)."""
import importlib
import types

import numpy as np
import pytest

from helpers import pkg, syn

st = importlib.import_module("ctrl-vio_b200.streaming")

WS = st.WINDOW_SIZE


def msg(ids, xy=(0.0, 0.0)):
    """a tracker message as FrameClouds.message returns it: float32 points (z = 1), id, u, v, vx, vy channels"""
    ids = np.asarray(ids, np.float32)
    n = len(ids)
    pts = np.ones((n, 3), np.float32)
    pts[:, :2] = np.broadcast_to(np.asarray(xy, np.float32), (n, 2))
    z = np.zeros(n, np.float32)
    return pts, ids, z, z, z, z


def filled(slots_msgs):
    t = st.FeatureTable()
    for s, m in slots_msgs:
        t.add(s, m)
    return t


def test_new_entries_in_ascending_id_order():
    t = st.FeatureTable()
    assert t.add(3, msg([42, 7, 19, 3])) == (0, 4)
    assert t.id.tolist() == [3, 7, 19, 42]
    assert [t.idx[e, 3] for e in range(4)] == [3, 1, 2, 0]           # index in the cloud, not in the table
    assert t.add(5, msg([100, 19, 50, 3])) == (2, 2)
    assert t.id.tolist() == [3, 7, 19, 42, 50, 100]                  # appended after the live entries, ascending
    assert t.anchor.tolist() == [3, 3, 3, 3, 5, 5]
    assert t.idx[0, 5] == 3 and t.idx[2, 5] == 1 and t.idx[1, 5] == -1
    assert (t.rho == -1).all() and (t.lm == -1).all()


def test_tracked_counts_live_entries_only():
    t = filled([(0, msg([1, 2, 3])), (1, msg([1, 2, 4]))])
    assert t.slide(0, np.zeros(0)) == 3                               # 1, 2, 3 leave with their anchor
    assert t.id.tolist() == [4]
    n_tracked, n_new = t.add(2, msg([1, 2, 4, 5]))
    assert (n_tracked, n_new) == (1, 3)                               # 1 and 2 come back as new landmarks
    assert t.id.tolist() == [4, 1, 2, 5] and t.anchor.tolist() == [1, 2, 2, 2]
    # the keyframe decision's count differs: there, an id counts when it occurs in any listed slot
    _, kf_tracked, _, _ = st.keyframe_decision([msg([1, 2, 4]), msg([1, 2, 4, 5])], 1.0)
    assert kf_tracked == 3


def window_of(t, slots, ws=WS, rho=None):
    rho = np.zeros(0) if rho is None else rho
    return t.window(slots, ws, rho)


def test_candidate_rule_boundaries():
    # 12 frames in slots 0..11; landmark k anchored in slot k and seen in slot k+1 (used_num 2), landmark 100 + k seen
    # only in its anchor slot (used_num 1)
    t = st.FeatureTable()
    for s in range(12):
        t.add(s, msg(([s - 1] if s else []) + [s, 100 + s]))
    window_of(t, list(range(12)), ws=WS)
    ids, anchor, used = t.landmarks()
    assert ids.tolist() == list(range(WS - 2))                       # start_frame 0 .. WS-3 with used_num 2
    assert (used == 2).all() and anchor.tolist() == list(range(WS - 2))
    assert WS - 2 not in ids.tolist()                                 # start_frame WS-2 is not a candidate
    # with a slot dropped from between anchor and observation, used_num falls to 1
    t2 = st.FeatureTable()
    for s in range(4):
        t2.add(s, msg(([s - 1] if s else []) + [s]))
    t2.slide(1, np.zeros(0))                                          # landmark 0 loses its only observation
    window_of(t2, [0, 2, 3])
    assert t2.landmarks()[0].tolist() == [2]


def test_non_candidate_keeps_its_depth():
    t = filled([(0, msg([1, 2])), (1, msg([1, 2])), (2, msg([1]))])
    rho = window_of(t, [0, 1, 2])
    assert t.landmarks()[0].tolist() == [1, 2] and (rho == -1).all()
    rho = np.array([0.25, 0.5])
    t.slide(1, rho)                                                  # landmark 2 falls to used_num 1
    rho2 = window_of(t, [0, 2], rho=rho)
    assert t.landmarks()[0].tolist() == [1] and rho2.tolist() == [0.25]
    assert t.rho.tolist() == [0.25, 0.5]                             # setDepth reached the non-candidate too
    t.add(3, msg([2, 9]))
    rho3 = window_of(t, [0, 2, 3], rho=np.array([0.125]))
    assert t.landmarks()[0].tolist() == [1, 2] and rho3.tolist() == [0.125, 0.5]


def test_remove_failures_only_negative():
    t = filled([(0, msg([1, 2, 3, 4])), (1, msg([1, 2, 3, 4, 5]))])
    window_of(t, [0, 1])
    t.add(2, msg([5]))
    assert t.slide(2, np.array([-1e-300, 0.0, np.nan, 0.5])) == 1    # only rho < 0 is SolveFail
    assert t.id.tolist() == [2, 3, 4, 5]


@pytest.mark.parametrize("leaving", ["oldest", "second_newest"])
def test_slide(leaving):
    t = filled([(4, msg([1, 2])), (7, msg([1, 2, 3])), (9, msg([2, 3, 5]))])
    slot = 4 if leaving == "oldest" else 7
    removed = t.slide(slot, np.zeros(0))
    if leaving == "oldest":
        assert removed == 2 and t.id.tolist() == [3, 5]
    else:
        assert removed == 1 and t.id.tolist() == [1, 2, 5]
        assert t.idx[:, 7].tolist() == [-1, -1, -1]
        assert t.idx[1, 9] == 0 and t.idx[0, 9] == -1
    assert slot not in t.held
    t.add(slot, msg([2, 8]))                                         # the slot is free again


def host_association(r, seq, frames, slots):
    """what the host path derives: (landmark ids, factor lists, CSR)"""
    fr = np.asarray(frames)
    w = syn.subwindow_frames(seq, fr, window_size=WS)
    lm_global = w.meta["lm_global"]
    sel = st.ResidentRunner._factor_selection(r, fr, lm_global)
    slot_j, idx_j = slots[w.obs_frame], r.clouds.obs_idx[sel]
    csr = st.ResidentRunner._observation_csr(r, fr, w, lm_global, slot_j, idx_j, slots)
    fac = (slots[w.anchor_frame[w.lm]], r.clouds.anchor_idx[lm_global[w.lm]], slot_j, idx_j, w.lm,
           (w.anchor_frame[w.lm] == 0).astype(np.int32))
    return lm_global, fac, csr


def run_table_over_sequence(seq, n, every, check):
    """drive FeatureTable through the runner's slot allocation and slides; check(k, r, table, frames, slots, marg, rho)"""
    clouds = st.FrameClouds(seq)
    r = types.SimpleNamespace(n_slots=16, slot_of={}, clouds=clouds, seq=seq)
    t = st.FeatureTable()
    frames = list(range(st.WIN_KF))
    for f in frames:
        t.add(st.ResidentRunner._assign_slot(r, f), clouds.message(f))
    nxt, rho = st.WIN_KF, np.zeros(0)
    for k in range(n):
        if k:
            frames.append(nxt)
            t.add(st.ResidentRunner._assign_slot(r, nxt), clouds.message(nxt))
            nxt += 1
        slots = np.array([r.slot_of[f] for f in frames], np.int32)
        marg = not (every and frames[-2] % every == every - 1)
        rho = t.window(slots, WS, rho)
        rho = np.where(rho < 0, 0.2 + 1e-3 * np.arange(len(rho)), rho)   # a "triangulated" depth for the new ones
        check(k, r, t, frames, slots, marg, rho)
        t.slide(r.slot_of.pop(frames.pop(0 if marg else -2)), rho)


@pytest.mark.parametrize("every,n", [(0, 40), (2, 14), (3, 40)])
def test_table_matches_host_association_on_c5(every, n):
    """The table's numbering, factors, marg flags and CSR equal the host path's.  The one difference is the documented
    deviation: after a MARGIN_SECOND_NEW slide the landmarks anchored in the dropped frame come back in the next cloud
    as new entries (the host path forgets them for good); with second_new_every=3 they become candidates from window 7
    on.  The comparison then drops exactly those re-created entries from the table's side."""
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    anchor_frame = seq.anchor_frame
    n_recreated = []

    def check(k, r, t, frames, slots, marg, rho):
        ids, anchor, _ = t.landmarks()
        slot_frame = {s: f for f, s in r.slot_of.items()}
        first = np.array([anchor_frame[i] == slot_frame[a] for i, a in zip(ids, anchor)], bool)   # not re-created
        n_recreated.append(int((~first).sum()))
        lm_global, fac_h, csr_h = host_association(r, seq, frames, slots)
        assert np.array_equal(ids[first], lm_global), k
        keep = np.nonzero(first)[0]
        renum = np.full(len(ids), -1); renum[keep] = np.arange(len(keep))
        fac_t = t.factors(rho, marg)
        sel = first[fac_t[4]]
        fac_t = fac_t[:4] + (renum[fac_t[4][sel]], fac_t[5][sel])
        fac_t = tuple(x[sel] if i < 4 else x for i, x in enumerate(fac_t))
        for a, b in zip(fac_t[:5], fac_h[:5]):
            assert np.array_equal(a, b), k
        assert np.array_equal(fac_t[5], fac_h[5] * int(marg)), k
        off, osl, oix = t.observation_csr()
        cnt = np.diff(off)[keep]
        assert np.array_equal(np.concatenate([[0], np.cumsum(cnt)]), csr_h[0]), k
        o = np.concatenate([np.arange(off[e], off[e + 1]) for e in keep]) if len(keep) else np.zeros(0, int)
        assert np.array_equal(osl[o], csr_h[1]) and np.array_equal(oix[o], csr_h[2]), k

    run_table_over_sequence(seq, n, every, check)
    if every == 3:
        assert n_recreated[:7] == [0] * 7 and max(n_recreated) > 0
    else:
        assert max(n_recreated) == 0                                  # the two conventions agree exactly


# ---------------------------------------------------------------------------------------------------------------------
# GPU

def engine(cuda_lib, seq=None):
    seq = seq or st.config_c5_sequence(1)
    return pkg.Estimator(cuda_lib, pkg.make_config(**seq.config_kwargs()))


def assert_landmarks(e, t, n):
    assert n == len(t.numbered)
    ids, anchor, used = e.FeatureTableLandmarks()
    hi, ha, hu = t.landmarks()
    assert np.array_equal(ids, hi) and np.array_equal(anchor, ha) and np.array_equal(used, hu)


def bitwise(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["second_new_every", "min_parallax"])
def test_device_table_matches_host_restatement(cuda_lib, mode):
    n = 40
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    clouds = st.FrameClouds(seq)
    if mode == "min_parallax":
        means = []
        for k in range(n):
            _, _, num, s = st.keyframe_decision([clouds.message(f) for f in range(k, k + st.WIN_KF)], 0.0)
            means.append(s / num)
        m = float(np.median(means))
        decide = lambda frames: st.keyframe_decision([clouds.message(f) for f in frames], m)[0]
    else:
        decide = lambda frames: not (frames[-2] % 3 == 2)
    # e: the device table; g: the same clouds and state, fed the numpy table's CSR and factor list through the
    # index-array calls, so that the device-built CSR and factor descriptors are compared through what reads them
    e, g = engine(cuda_lib, seq), engine(cuda_lib, seq)
    for x in (e, g):
        x.SetKnots(seq.q0, seq.p0); x.SetBiases(seq.bias0[:2]); x.SetLineDelay(seq.ld0)
    r = types.SimpleNamespace(n_slots=16, slot_of={})
    t = st.FeatureTable()
    rng = np.random.default_rng(5)

    def add(f):
        s = st.ResidentRunner._assign_slot(r, f)
        m_ = clouds.message(f)
        for x in (e, g):
            x.IngestFeatureCloud(s, int(seq.kf_times[f]), *m_)
        assert e.FeatureTableAdd(s) == t.add(s, m_)

    frames = list(range(st.WIN_KF))
    for f in frames:
        add(f)
    nxt, rho, flags = st.WIN_KF, np.zeros(0), set()
    for k in range(n):
        if k:
            frames.append(nxt); add(nxt); nxt += 1
        slots = np.array([r.slot_of[f] for f in frames], np.int32)
        marg = decide(frames)
        flags.add(marg)
        rho_h = t.window(slots, WS, rho)
        n_lm = e.FeatureTableWindow(slots, WS)
        assert_landmarks(e, t, n_lm)
        assert bitwise(e.GetInvDepths(), rho_h), k
        # the device CSR: triangulating from it equals TriangulateWindow over the numpy CSR, bit for bit
        g.SetInvDepths(rho_h)
        assert e.TriangulateWindowFromTable() == g.TriangulateWindow(*t.observation_csr()), k
        rho_tri = e.GetInvDepths()
        assert bitwise(rho_tri, g.GetInvDepths()), k
        # a "solve": new depths, a few of them negative (removeFailures)
        rho = rho_tri * (1.0 + 0.01 * rng.standard_normal(len(rho_tri)))
        rho[rng.random(len(rho)) < 0.01] *= -1
        for x in (e, g):
            x.SetInvDepths(rho)
            x.ClearFactors()
        # the device factor descriptors: (slot, index) pairs and landmark numbers in the same order as the numpy list,
        # seen through the residuals and Jacobians they produce (every landmark has its own depth)
        fac = t.factors(rho, marg)
        n_f = e.AddImageFeaturesFromTable(marg)
        g.AddImageFeaturesFromSlots(*fac)
        assert n_f == len(fac[0])
        re_, se, Je, ce = e.EvalImageFactors()
        rg, sg, Jg, cg = g.EvalImageFactors()
        assert bitwise(re_, rg) and np.array_equal(se, sg) and bitwise(Je, Jg), k
        assert np.isclose(ce, cg, rtol=1e-12, atol=0.0), k        # (the summed cost: atomic order varies)
        leave = r.slot_of.pop(frames.pop(0 if marg else -2))
        assert e.FeatureTableSlide(leave) == t.slide(leave, rho), k
    assert flags == {True, False}


class Forbidden:
    def __getitem__(self, _):
        raise AssertionError("the device-feature runner read the host association")


def forbid_host_association(monkeypatch, runner):
    def boom(*a, **k):
        raise AssertionError("the device-feature runner read the host association")
    monkeypatch.setattr(st.syn, "subwindow_frames", boom)
    monkeypatch.setattr(st.ResidentRunner, "_factor_selection", boom)
    monkeypatch.setattr(st.ResidentRunner, "_observation_csr", boom)
    runner.clouds.anchor_idx = Forbidden()
    runner.clouds.obs_idx = Forbidden()


def run_deterministic(monkeypatch, a, b, n):
    """both runners in deterministic mode (the default mode's atomic accumulation order varies from run to run); the
    device-feature runner `b` runs with the host association made unreadable"""
    a.est.SetDeterministic(True)
    a.run(n)
    with monkeypatch.context() as mp:
        forbid_host_association(mp, b)
        b.est.SetDeterministic(True)
        b.run(n)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["c5", "second_new_every_2", "min_parallax"])
def test_device_feature_runner_matches_host_association_bitwise(cuda_lib, monkeypatch, case):
    n = {"c5": 8, "second_new_every_2": 14, "min_parallax": 8}[case]
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    kw = {}
    if case == "second_new_every_2":
        kw = dict(second_new_every=2)
    elif case == "min_parallax":
        clouds = st.FrameClouds(seq)
        means = []
        for k in range(n):
            _, _, num, s = st.keyframe_decision([clouds.message(f) for f in range(k, k + st.WIN_KF)], 0.0)
            means.append(s / num)
        kw = dict(min_parallax=float(np.median(means)))
    a = st.ResidentRunner(cuda_lib, seq, triangulate=True, **kw)
    b = st.ResidentRunner(cuda_lib, seq, triangulate=True, device_features=True, **kw)
    run_deterministic(monkeypatch, a, b, n)
    for key in ("n_obs", "n_lm", "n_triangulated", "n_fallback", "iterations", "marg_flag", "prior_dim"):
        assert [x[key] for x in a.records] == [x[key] for x in b.records], key
    if case != "c5":
        assert {x["marg_flag"] for x in b.records} == {st.MARGIN_OLD, st.MARGIN_SECOND_NEW}
    assert a.frames == b.frames and a.ncp == b.ncp
    assert bitwise(a.q[:a.ncp], b.q[:b.ncp]) and bitwise(a.p[:a.ncp], b.p[:b.ncp])
    assert bitwise(a.est.GetBiases(), b.est.GetBiases())
    assert bitwise(a.est.GetInvDepths(), b.est.GetInvDepths())
    assert bitwise(a.ld, b.ld)
    print(case, "n_lm", [x["n_lm"] for x in b.records], "n_obs", [x["n_obs"] for x in b.records],
          "removed", [x["n_removed"] for x in b.records])


def test_device_feature_runner_requires_triangulation():
    with pytest.raises(ValueError):
        st.ResidentRunner(None, None, triangulate=False, device_features=True)


@pytest.mark.gpu
def test_error_paths_leave_table_and_state_unchanged(cuda_lib):
    seq = st.config_c5_sequence(1)
    e = engine(cuda_lib, seq)
    t = st.FeatureTable()
    clouds = [msg([1, 2, 3, 4]), msg([1, 2, 3, 5]), msg([2, 3, 5, 6])]
    for s, m in enumerate(clouds):
        e.IngestFeatureCloud(s, int(seq.kf_times[s]), *m)
    invalid, state = r"\(-1\)", r"\(-4\)"

    def raises(code, fn, *a):
        with pytest.raises(pkg.CtvioError, match=code):
            fn(*a)

    raises(state, e.TriangulateWindowFromTable)                    # knots not set
    e.SetKnots(seq.q0[:20], seq.p0[:20]); e.SetLineDelay(seq.ld0)
    raises(state, e.TriangulateWindowFromTable)                    # no window yet
    raises(state, e.AddImageFeaturesFromTable, 1)
    raises(state, e.FeatureTableLandmarks, 0)
    for s in range(3):
        assert e.FeatureTableAdd(s) == t.add(s, clouds[s])
    raises(invalid, e.FeatureTableAdd, 16)
    raises(invalid, e.FeatureTableAdd, -1)
    raises(invalid, e.FeatureTableAdd, 7)                           # no cloud ingested
    raises(state, e.FeatureTableAdd, 1)                             # the table holds it
    raises(state, e.IngestFeatureCloud, 1, 0, *msg([7, 8]))         # its cloud stays while the table holds the slot
    raises(invalid, e.FeatureTableWindow, np.zeros(0, np.int32), WS)
    raises(invalid, e.FeatureTableWindow, np.arange(17) % 16, WS)
    raises(invalid, e.FeatureTableWindow, [0, 1, 16], WS)
    raises(invalid, e.FeatureTableWindow, [0, 1, 1], WS)
    raises(invalid, e.FeatureTableWindow, [0, 1, 2], 2)
    raises(state, e.FeatureTableWindow, [0, 1], WS)                 # not the held slots
    raises(state, e.FeatureTableWindow, [0, 1, 2, 3], WS)
    raises(invalid, e.FeatureTableSlide, 16)
    raises(state, e.FeatureTableSlide, 5)
    rho_h = t.window([0, 1, 2], WS, np.zeros(0))
    n = e.FeatureTableWindow([0, 1, 2], WS)
    assert_landmarks(e, t, n)
    assert bitwise(e.GetInvDepths(), rho_h)
    raises(invalid, e.TriangulateWindowFromTable, 0.0)
    raises(invalid, e.TriangulateWindowFromTable, -5.0)
    raises(invalid, e.FeatureTableLandmarks, n + 1)
    rho = np.array([0.5, 0.25, 0.125, 0.0625])[:n]
    e.SetInvDepths(np.concatenate([rho, [1.0]]))                    # a different landmark count
    raises(state, e.TriangulateWindowFromTable)
    raises(state, e.AddImageFeaturesFromTable, 1)
    raises(state, e.FeatureTableWindow, [0, 1, 2], WS)
    raises(state, e.FeatureTableSlide, 0)
    e.SetInvDepths(rho)
    e.ClearFactors()
    e.AddImageFeatureDelayAnalytic([0], [0], [[0.0, 0.0]], [0], [0], [[0.0, 0.0]], [0])
    raises(state, e.AddImageFeaturesFromTable, 1)                   # host-payload factors present
    e.ClearFactors()
    assert e.AddImageFeaturesFromTable(1) == len(t.factors(rho, True)[0])
    # after all the refused calls the table is the host restatement's, step for step
    assert e.FeatureTableSlide(0) == t.slide(0, rho)
    raises(state, e.AddImageFeaturesFromTable, 1)                   # the window is stale after a slide
    raises(invalid, e.FeatureTableAdd, 0)                           # the slid slot's cloud left with it
    e.IngestFeatureCloud(0, int(seq.kf_times[3]), *msg([5, 6, 7]))
    assert e.FeatureTableAdd(0) == t.add(0, msg([5, 6, 7]))
    rho_h = t.window([1, 2, 0], WS, rho)
    assert_landmarks(e, t, e.FeatureTableWindow([1, 2, 0], WS))
    assert bitwise(e.GetInvDepths(), rho_h)


def full_table_run(cuda_lib, seed):
    """16 slots x 1024 features with overlapping ids; returns every device output"""
    rng = np.random.default_rng(seed)
    e = engine(cuda_lib)
    t = st.FeatureTable()
    out = []
    for s in range(16):
        ids = rng.choice(20000, 1024, replace=False)             # float32 carries ids < 2^24 exactly
        m = msg(ids)
        e.IngestFeatureCloud(s, 0, *m)
        r = e.FeatureTableAdd(s)
        assert r == t.add(s, m)
        out.append(r)
    slots = np.arange(16, dtype=np.int32)
    rho_h = t.window(slots, 16, np.zeros(0))
    n = e.FeatureTableWindow(slots, 16)
    assert_landmarks(e, t, n)
    assert bitwise(e.GetInvDepths(), rho_h)
    out += [e.FeatureTableLandmarks(), e.GetInvDepths()]
    rho = rng.uniform(-0.05, 1.0, n)
    e.SetInvDepths(rho)
    out.append(e.AddImageFeaturesFromTable(1))
    for s in (0, 7):
        r = e.FeatureTableSlide(s)
        assert r == t.slide(s, rho)
        out.append(r)
    rest = np.array([s for s in slots if s not in (0, 7)], np.int32)
    rho_h = t.window(rest, 16, rho)
    n2 = e.FeatureTableWindow(rest, 16)
    assert_landmarks(e, t, n2)
    assert bitwise(e.GetInvDepths(), rho_h)
    out += [e.FeatureTableLandmarks(), e.GetInvDepths()]
    return out


@pytest.mark.gpu
def test_full_tables_are_bitwise_reproducible(cuda_lib):
    a, b = full_table_run(cuda_lib, 11), full_table_run(cuda_lib, 11)
    for x, y in zip(a, b):
        if isinstance(x, tuple) and isinstance(x[0], np.ndarray):
            assert all(np.array_equal(u, v) for u, v in zip(x, y))
        elif isinstance(x, np.ndarray):
            assert bitwise(x, y)
        else:
            assert x == y


@pytest.mark.gpu
def test_remove_failures_after_a_negative_depth(cuda_lib):
    """one inverse depth set negative (SetInvDepths) between the solve and the slide: that landmark leaves the table"""
    n = 3
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    runner = st.ResidentRunner(cuda_lib, seq, triangulate=True, device_features=True)
    runner.run(n - 1)
    e = runner.est
    # the next image's table calls, as step() makes them
    f = runner.next_frame
    runner.frames.append(f)
    s = runner._assign_slot(f)
    e.IngestFeatureCloud(s, int(seq.kf_times[f]), *runner.clouds.message(f))
    e.FeatureTableAdd(s)
    slots = np.array([runner.slot_of[x] for x in runner.frames], np.int32)
    e.ExtendKnotsTo(int(seq.kf_times[f]) + st.EXTEND_NS)
    e.FeatureTableWindow(slots, WS)
    e.TriangulateWindowFromTable()
    ids, anchors, _ = e.FeatureTableLandmarks()
    rho = e.GetInvDepths()
    assert (rho > 0).all()
    leaving = int(slots[0])
    victim = len(rho) - 1                                        # anchored late: not in the leaving slot
    assert anchors[victim] != leaving
    rho[victim] = -0.1
    e.SetInvDepths(rho)
    anchored = int(np.sum(anchors == leaving))
    assert anchored > 0
    assert e.FeatureTableSlide(leaving) >= anchored + 1
    ids_after = e.FeatureTableLandmarks(e.FeatureTableWindow(slots[1:], WS))[0].tolist()
    assert ids[victim] not in ids_after
    same_anchor = [int(i) for k, i in enumerate(ids) if anchors[k] == anchors[victim] and k != victim]
    assert same_anchor and set(same_anchor) <= set(ids_after)     # its neighbours stay
    assert not set(ids[anchors == leaving].tolist()) & set(ids_after)
