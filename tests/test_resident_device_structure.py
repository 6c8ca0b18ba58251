"""The structure build of a factor set with table-built image factors, on the device (structure.cu), against the host
build of the same factors added through ctvio_add_image_features_from_slots.

Every case builds one factor set on two engines with the same state and clouds: `e` takes the image factors from the
resident feature table (device build), `g` takes the same factors in the same caller order as slot-named factors (host
build).  ctvio_debug_structure returns what each built - sorted descriptors, sorted-to-caller map, K1 items, landmark
layout, K4 items and entries, active mask and, after ctvio_marginalize, its block positions - and every array must be
equal.  Solves and priors built on the two structures must be bitwise equal, the table path must read back only the
documented count block, and its errors must be the host build's."""
import ctypes as C
import importlib

import numpy as np
import pytest

from helpers import pkg

st = importlib.import_module("ctrl-vio_b200.streaming")

WS = st.WINDOW_SIZE
CAP = 1024  # features per frame slot (a descriptor names feature k of slot s as s * CAP + k)
ARRAYS = ("desc", "orig", "items", "lo", "hi", "woff", "schur_items", "entries", "active", "pos_cam", "pos_lm", "marg_img")


def engine(lib, seq):
    return pkg.Estimator(lib, pkg.make_config(**seq.config_kwargs()))


def bitwise(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def count_block_bytes(n_knots):
    """what the device structure build reads back (include/ctvio.h, ctvio_debug_structure)"""
    return 32 + 4 * ((n_knots + 31) // 32)


def assert_same_structure(e, g, ctx=""):
    a, b = e.DebugStructure(), g.DebugStructure()
    for k in ARRAYS:
        if a[k] is None or b[k] is None:
            assert a[k] is None and b[k] is None, (k, ctx)
        else:
            assert a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), (k, ctx)
    n = len(a["orig"])
    assert np.array_equal(np.sort(a["orig"]), np.arange(n)), ctx
    return a


def caller_order(s):
    """the caller-order descriptors of a built structure (sorted descriptors through the sorted-to-caller map)"""
    d = np.empty_like(s["desc"])
    d[s["orig"]] = s["desc"]
    return d


def slots_args(desc):
    d = np.asarray(desc, np.int64).reshape(-1, 4)
    return d[:, 0] // CAP, d[:, 0] % CAP, d[:, 1] // CAP, d[:, 1] % CAP, d[:, 2], d[:, 3]


def fac_desc(fac):
    si, ii, sj, ij, lm, mg = (np.asarray(x, np.int64) for x in fac)
    return np.stack([si * CAP + ii, sj * CAP + ij, lm, mg], axis=1)


def get_prior(x, n, nb):
    J, r, x0 = np.zeros((n, n)), np.zeros(n), np.zeros((nb, 4))
    ty, ix, co = np.zeros(nb, np.int32), np.zeros(nb, np.int32), np.zeros(nb, np.int32)
    x.lib.call("get_prior", x.h, J.ctypes.data_as(C.c_void_p), r.ctypes.data_as(C.c_void_p), ty.ctypes.data_as(C.c_void_p),
               ix.ctypes.data_as(C.c_void_p), co.ctypes.data_as(C.c_void_p), x0.ctypes.data_as(C.c_void_p))
    return J, r, ty, ix, co, x0


def assert_same_state(e, g, ctx=""):
    qe, pe = e.GetKnots()
    qg, pg = g.GetKnots()
    assert bitwise(qe, qg) and bitwise(pe, pg), ctx
    assert bitwise(e.GetBiases(), g.GetBiases()), ctx
    assert bitwise(e.GetInvDepths(), g.GetInvDepths()), ctx
    assert bitwise(e.GetLineDelay(), g.GetLineDelay()), ctx


# ---- C5 windows through the resident runner: its estimator is a twin of a table engine and a slots engine ----------
class Twin:
    """Every call of the runner goes to both engines; the table engine's image factors reach the slots engine as
    slot-named factors in the same caller order.  Before each solve the two structures are compared, after each
    marginalization the block positions and the priors."""

    def __init__(self, e, g):
        self.e, self.g = e, g
        self.windows = 0
        self.lib = self  # the runner calls e.lib.call("marginalize", e.h, ...)
        self.h = None

    def __getattr__(self, name):
        fe, fg = getattr(self.e, name), getattr(self.g, name)
        if not callable(fe):
            return fe

        def both(*a, **k):
            r = fe(*a, **k)
            fg(*a, **k)
            return r
        return both

    def AddImageFeaturesFromTable(self, marg):
        n = self.e.AddImageFeaturesFromTable(marg)
        if n:
            self.g.AddImageFeaturesFromSlots(*slots_args(caller_order(self.e.DebugStructure())))
        return n

    def Solve(self, iters):
        if self.e.n_img:
            assert_same_structure(self.e, self.g, self.windows)
            self.windows += 1
        r = self.e.Solve(iters)
        assert self.g.Solve(iters).iterations == r.iterations
        return r

    def call(self, name, h, *args):
        assert name == "marginalize"
        self.e.lib.call(name, self.e.h, *args)
        n, nb = C.c_int32(), C.c_int32()
        self.g.lib.call(name, self.g.h, C.byref(n), C.byref(nb))
        assert_same_structure(self.e, self.g, ("marg", self.windows))
        if n.value > 0:
            pe, pg = get_prior(self.e, n.value, nb.value), get_prior(self.g, n.value, nb.value)
            assert all(bitwise(x, y) if x.dtype == np.float64 else np.array_equal(x, y) for x, y in zip(pe, pg))


def c5_kw(case, seq, n):
    if case == "second_new_every_2":
        return dict(second_new_every=2)
    if case == "reanchor":
        return dict(reanchor=True, second_new_every=2)
    if case == "min_parallax":
        clouds = st.FrameClouds(seq)
        means = []
        for k in range(n):
            _, _, num, s = st.keyframe_decision([clouds.message(f) for f in range(k, k + st.WIN_KF)], 0.0)
            means.append(s / num)
        return dict(min_parallax=float(np.median(means)))
    return {}


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["margin_old", "second_new_every_2", "min_parallax", "reanchor"])
def test_c5_windows_device_structure_equals_host_build(cuda_lib, case):
    n = 9
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    runner = st.ResidentRunner(cuda_lib, seq, triangulate=True, device_features=True, **c5_kw(case, seq, n))
    twin = Twin(runner.est, engine(cuda_lib, seq))
    runner.est = twin
    twin.SetDeterministic(True)
    runner.run(n)
    assert twin.windows == n
    assert_same_state(twin.e, twin.g, case)
    if case == "margin_old":
        assert {x["marg_flag"] for x in runner.records} == {st.MARGIN_OLD}
    elif case != "reanchor":
        assert {x["marg_flag"] for x in runner.records} == {st.MARGIN_OLD, st.MARGIN_SECOND_NEW}


# ---- hand-built tables -----------------------------------------------------------------------------------------------
def msg(ids):
    ids = np.asarray(ids, np.float32)
    pts = np.ones((len(ids), 3), np.float32)
    pts[:, 0] = 1e-4 * (ids % 97)
    pts[:, 1] = -1e-4 * (ids % 89)
    z = np.zeros(len(ids), np.float32)
    v = (ids % 480).astype(np.float32)
    return pts, ids, z, v, z, z


class Pair:
    """table engine e, slots engine g and the host restatement t of the feature table, over the same clouds"""

    def __init__(self, lib, seq, n_knots=None):
        self.seq = seq
        self.e, self.g = engine(lib, seq), engine(lib, seq)
        self.t = st.FeatureTable()
        k = n_knots or len(seq.q0)
        for x in self.both:
            x.SetKnots(seq.q0[:k], seq.p0[:k]); x.SetBiases(seq.bias0[:2]); x.SetLineDelay(seq.ld0)

    @property
    def both(self):
        return (self.e, self.g)

    def add(self, slot, t_ns, ids):
        m = msg(ids)
        for x in self.both:
            x.IngestFeatureCloud(slot, int(t_ns), *m)
        assert self.e.FeatureTableAdd(slot) == self.t.add(slot, m)

    def window(self, slots, ws, rho_fn):
        """numbers the window on both tables; rho_fn(anchor slots) -> the inverse depths both engines take"""
        self.t.window(slots, ws, np.zeros(0))
        n_lm = self.e.FeatureTableWindow(slots, ws)
        _, anchor, _ = self.e.FeatureTableLandmarks()
        rho = rho_fn(anchor)
        for x in self.both:
            x.SetInvDepths(rho)
        return rho

    def factors(self, rho, marg, options=None):
        for x in self.both:
            x.SetOptions(options or pkg.make_options())
            x.ClearFactors()
        n = self.e.AddImageFeaturesFromTable(marg)
        fac = self.t.factors(rho, marg)
        assert n == len(fac[0])
        self.g.AddImageFeaturesFromSlots(*fac)
        return fac


def full_pair(lib, seed, first_cloud=CAP):
    seq = st.config_c5_sequence(8)
    assert len(seq.kf_times) >= 16
    rng = np.random.default_rng(seed)
    p = Pair(lib, seq)
    for s in range(16):
        p.add(s, seq.kf_times[s], rng.choice(20000, first_cloud if s == 0 else CAP, replace=False))
    return p, rng


@pytest.mark.gpu
@pytest.mark.parametrize("marg_oldest", [0, 1])
def test_full_tables(cuda_lib, marg_oldest):
    p, rng = full_pair(cuda_lib, 7)
    slots = np.arange(16, dtype=np.int32)
    rho = p.window(slots, 16, lambda anchor: rng.uniform(-0.05, 1.0, len(anchor)))
    opt = pkg.make_options(is_marg_state=bool(marg_oldest), ctrl_to_be_opt_now=0, ctrl_to_be_opt_later=2)
    fac = p.factors(rho, marg_oldest, opt)
    assert len(fac[0]) > 3000
    s = assert_same_structure(p.e, p.g)
    assert s["pos_cam"] is None
    assert s["marg_img"] is None
    assert (s["desc"][:, 3] != 0).any() == bool(marg_oldest)


@pytest.mark.gpu
def test_full_tables_solve_and_prior(cuda_lib):
    # slot 0 holds 200 features, so that the marginalized landmarks (anchored there, positive depth) stay few
    p, rng = full_pair(cuda_lib, 3, first_cloud=200)
    slots = np.arange(16, dtype=np.int32)
    rho = p.window(slots, 16, lambda anchor: np.where(anchor == 0, 0.3, 1.0) * rng.uniform(0.2, 1.0, len(anchor)))
    opt = pkg.make_options(is_marg_state=True, ctrl_to_be_opt_now=0, ctrl_to_be_opt_later=2, fixed_knot_index=1)
    p.factors(rho, 1, opt)
    assert_same_structure(p.e, p.g)
    for x in p.both:
        x.SetDeterministic(True)
    se, sg = p.e.Solve(4), p.g.Solve(4)
    assert se.iterations == sg.iterations and bitwise(se.final_cost, sg.final_cost)
    for x in p.both:
        x.GaugeRealign(0, np.eye(3), np.zeros(3))
    pe, pg = p.e.SaveMarginalizationInfo(), p.g.SaveMarginalizationInfo()
    assert pe is not None and pg is not None and pe.n == pg.n
    assert bitwise(pe.J, pg.J) and bitwise(pe.r, pg.r) and bitwise(pe.blk_x0, pg.blk_x0)
    assert np.array_equal(pe.blk_type, pg.blk_type) and np.array_equal(pe.blk_index, pg.blk_index)
    s = assert_same_structure(p.e, p.g)
    assert s["marg_img"] is not None and len(s["marg_img"]) > 0
    assert_same_state(p.e, p.g)


def small_pair(lib, times_of_slot, ids_of_slot, n_knots=None):
    seq = st.config_c5_sequence(4)
    p = Pair(lib, seq, n_knots)
    for s, (t, ids) in enumerate(zip(times_of_slot, ids_of_slot)):
        p.add(s, t, ids)
    return p


@pytest.mark.gpu
def test_two_frames_share_a_padded_knot_window(cuda_lib):
    seq = st.config_c5_sequence(4)
    dt = int(seq.config_kwargs()["dt_ns"])
    base = int(seq.config_kwargs()["t0_ns"]) + 10 * dt + dt // 10
    # frames 0 / 1 and 2 / 3 start in the same knot interval: each pair shares the first knot of its padded window
    times = [base, base + dt // 5, base + 2 * dt, base + 2 * dt + dt // 7, base + 4 * dt]
    ids = [np.arange(0, 300), np.arange(100, 400), np.arange(200, 500), np.arange(0, 500, 2), np.arange(250, 600)]
    p = small_pair(cuda_lib, times, ids)
    rho = p.window(np.arange(5, dtype=np.int32), 16, lambda anchor: np.full(len(anchor), 0.5))
    fac = p.factors(rho, 1, pkg.make_options(is_marg_state=True, ctrl_to_be_opt_later=2))
    s = assert_same_structure(p.e, p.g)
    pairs = {(a, b) for a, b in zip(fac[0], fac[2])}
    groups = {(int(w0), int(w1)) for w0, w1 in s["items"][:, 2:]}
    assert len(groups) < len(pairs)  # slot pairs that share their windows form one group
    for x in p.both:
        x.SaveMarginalizationInfo()
    assert_same_structure(p.e, p.g)


@pytest.mark.gpu
def test_window_without_image_factors(cuda_lib):
    seq = st.config_c5_sequence(4)
    p = small_pair(cuda_lib, seq.kf_times[:3], [np.arange(0, 50), np.arange(50, 100), np.arange(100, 150)])
    rho = p.window(np.arange(3, dtype=np.int32), WS, lambda anchor: np.zeros(len(anchor)))
    assert len(p.factors(rho, 1)[0]) == 0
    s = assert_same_structure(p.e, p.g)
    assert len(s["orig"]) == 0 and len(s["items"]) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("table_first", [True, False])
def test_mixed_table_and_slot_factors(cuda_lib, table_first):
    p, rng = full_pair(cuda_lib, 5)
    slots = np.arange(16, dtype=np.int32)
    rho = p.window(slots, 16, lambda anchor: rng.uniform(0.1, 1.0, len(anchor)))
    for x in p.both:
        x.ClearFactors()
    fac = fac_desc(p.t.factors(rho, 1))
    extra = fac[rng.choice(len(fac), 500, replace=False)][::-1].copy()  # not landmark-sorted
    extra[:, 3] = rng.integers(0, 2, len(extra))
    assert (np.diff(extra[:, 2]) < 0).any()
    if table_first:
        p.e.AddImageFeaturesFromTable(1)
        p.e.AddImageFeaturesFromSlots(*slots_args(extra))
        p.g.AddImageFeaturesFromSlots(*slots_args(np.concatenate([fac, extra])))
    else:
        p.e.AddImageFeaturesFromSlots(*slots_args(extra))
        p.e.AddImageFeaturesFromTable(1)
        p.g.AddImageFeaturesFromSlots(*slots_args(np.concatenate([extra, fac])))
    assert_same_structure(p.e, p.g)
    # a second table call appends to the same set
    p.e.AddImageFeaturesFromTable(0)
    p.g.AddImageFeaturesFromSlots(*slots_args(fac_desc(p.t.factors(rho, 0))))
    assert_same_structure(p.e, p.g)


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0, 2, 5])
def test_fixed_knot_index_mask(cuda_lib, offset):
    seq = st.config_c5_sequence(4)
    kw = seq.config_kwargs()
    fixed = int((seq.kf_times[0] - kw["t0_ns"]) // kw["dt_ns"]) + offset  # inside the knots the factors touch
    p = small_pair(cuda_lib, seq.kf_times[:6], [np.arange(k * 40, k * 40 + 200) for k in range(6)])
    rho = p.window(np.arange(6, dtype=np.int32), WS, lambda anchor: np.full(len(anchor), 0.4))
    p.factors(rho, 0, pkg.make_options(fixed_knot_index=fixed))
    s = assert_same_structure(p.e, p.g)
    assert not s["active"][:6 * (fixed + 1)].any()
    for x in p.both:  # a rebuild of the masks alone (options changed, same factors) keeps them equal
        x.SetOptions(pkg.make_options(fixed_knot_index=-1, fix_ld=False))
    s2 = assert_same_structure(p.e, p.g)
    assert s2["active"][:6 * (fixed + 1)].any()


# ---- traffic ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", ["c5", "full"])
def test_table_path_reads_back_only_the_count_block(cuda_lib, case):
    if case == "full":
        p, rng = full_pair(cuda_lib, 9)
        slots = np.arange(16, dtype=np.int32)
        rho = p.window(slots, 16, lambda anchor: rng.uniform(0.1, 1.0, len(anchor)))
    else:
        seq = st.quantize_wire(st.config_c5_sequence(2))
        clouds = st.FrameClouds(seq)
        p = Pair(cuda_lib, seq)
        for f in range(st.WIN_KF):
            m = clouds.message(f)
            for x in p.both:
                x.IngestFeatureCloud(f, int(seq.kf_times[f]), *m)
            assert p.e.FeatureTableAdd(f) == p.t.add(f, m)
        rho = p.window(np.arange(st.WIN_KF, dtype=np.int32), WS, lambda anchor: np.full(len(anchor), 0.25))
    for x in p.both:
        x.ClearFactors()
        x.SetDeterministic(True)
        x.TransferStats(reset=True)
    n = p.e.AddImageFeaturesFromTable(1)
    assert n > 0 and p.e.TransferStats(reset=True)[1] == 0
    p.g.AddImageFeaturesFromSlots(*p.t.factors(rho, 1))
    p.g.TransferStats(reset=True)
    p.e.Solve(2)
    p.g.Solve(2)
    de, dg = p.e.TransferStats()[1], p.g.TransferStats()[1]
    assert de - dg == count_block_bytes(len(p.seq.q0)), (de, dg)
    assert_same_state(p.e, p.g)


@pytest.mark.gpu
def test_runner_window_traffic(cuda_lib):
    n = 4
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    runner = st.ResidentRunner(cuda_lib, seq, triangulate=True, device_features=True)
    runner.run(n)
    d2h = [r["d2h_bytes"] for r in runner.records[1:]]
    assert max(d2h) < 2048, d2h


# ---- errors ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_errors_are_the_host_builds(cuda_lib):
    seq = st.config_c5_sequence(4)
    times = seq.kf_times[:6]
    dt = int(seq.config_kwargs()["dt_ns"])
    t0 = int(seq.config_kwargs()["t0_ns"])
    n_knots = int((times[4] - t0) // dt) + 4  # the newest frame's padded window leaves the spline
    p = small_pair(cuda_lib, times, [np.arange(k * 40, k * 40 + 200) for k in range(6)], n_knots=n_knots)
    rho = p.window(np.arange(6, dtype=np.int32), WS, lambda anchor: np.full(len(anchor), 0.4))
    p.factors(rho, 1, pkg.make_options(is_marg_state=True, ctrl_to_be_opt_later=1))
    for x in p.both:
        x.SetDeterministic(True)
    msgs = []
    for x in p.both:
        with pytest.raises(pkg.CtvioError, match=r"\(-6\)") as err:
            x.Solve(2)
        msgs.append(str(err.value).split(":", 1)[1])
    assert msgs[0] == msgs[1]
    for x in p.both:
        x.ExtendKnotsTo(int(times[-1]) + st.EXTEND_NS)
    assert_same_structure(p.e, p.g)
    se, sg = p.e.Solve(3), p.g.Solve(3)
    assert se.iterations == sg.iterations
    assert_same_state(p.e, p.g)
    pe, pg = p.e.SaveMarginalizationInfo(), p.g.SaveMarginalizationInfo()
    assert bitwise(pe.J, pg.J) and bitwise(pe.r, pg.r)
    # a landmark out of range: the same error from both builds
    nL = len(p.e.GetInvDepths())
    bad = fac_desc(p.t.factors(rho, 0))[:3].copy()
    bad[1, 2] = nL
    for x in p.both:
        x.AddImageFeaturesFromSlots(*slots_args(bad))
        with pytest.raises(pkg.CtvioError, match=r"\(-1\).*landmark index out of range"):
            x.Solve(1)


# ---- CPU -------------------------------------------------------------------------------------------------------------
def test_structure_probe_null_handle():
    raw = C.CDLL(pkg.load().path)
    f = raw.ctvio_debug_structure
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    n = C.c_int64(0)
    assert f(None, None, C.byref(n)) == -1
    raw.ctvio_last_error.restype = C.c_char_p
    assert raw.ctvio_last_error() == b"null argument"
    assert f(None, None, None) == -1
