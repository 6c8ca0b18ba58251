"""The covariance publications of the per-image odometry cycle (ctvio_cycle_covariances) and CycleRunner(covariances=).

CPU: the info struct and the renamed option fields match the header's layout (compiled with the host C compiler), the
new option checks and the getter's argument errors reach ctvio_last_error, the symbol lists, CycleRunner's checks of
covariances=.
GPU (C5): in deterministic mode the cycle's pose, odometry-edge and map-point covariances are bitwise ResidentRunner's
with its three publications, per window, in every case of test_odometry_cycle.py; the publications leave no trace in
the cycle and add no host wait; transfers stay at most the runner's; a rank-deficient window (no gauge) is reported and
the cycle carries on; the getter's state errors; default mode within tolerance."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from helpers import pkg

st = pkg.streaming if hasattr(pkg, "streaming") else __import__("importlib").import_module("ctrl-vio_b200.streaming")
bd = pkg.binding
P, I32, I64, F64 = C.c_void_p, C.c_int32, C.c_int64, C.c_double
ALL = ("pose", "odometry", "map")
ERR_INVALID, ERR_STATE = -1, -4


# ---------------------------------------------------------------------------------------------------------- CPU
@pytest.fixture(scope="module")
def raw():
    lib = C.CDLL(pkg.load().path)
    lib.ctvio_last_error.restype = C.c_char_p
    lib.ctvio_set_knots.argtypes = [P, I32, P, P]
    lib.ctvio_cycle_default_options.argtypes = [P]
    lib.ctvio_odometry_start.argtypes = [P, P, I64, I32, P, P, I32, P, P, F64, P, I32, P, P]
    lib.ctvio_cycle_covariances.argtypes = [P, P, P, P, P, I32, P, P]
    return lib


def _defaults(raw):
    o = bd.CycleOptions()
    assert raw.ctvio_cycle_default_options(C.byref(o)) == 0
    return o


def _reset_error(raw):
    assert raw.ctvio_set_knots(None, 0, None, None) < 0
    assert raw.ctvio_last_error() == b"need >= 4 knots"


def _start_rc(raw, opt):
    q = np.zeros((4, 4)); q[:, 3] = 1; p = np.zeros((4, 3)); b = np.zeros((11, 6))
    msgs = (bd.ImageMsg * 11)()
    res = bd.CycleResult()
    return raw.ctvio_odometry_start(None, C.byref(opt), 0, 4, q.ctypes.data, p.ctypes.data, 11, msgs, b.ctypes.data, 0.0,
                                    None, -1, None, C.byref(res))


def test_info_and_options_layout_match_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc") or shutil.which("g++")
    assert cc, "a host C compiler is needed to read the header's layout"
    structs = {"ctvio_cycle_covariance_info": bd.CycleCovarianceInfo, "ctvio_cycle_options": bd.CycleOptions}
    lines = []
    for name, cls in structs.items():
        lines.append(f'printf("{name} %zu\\n", sizeof({name}));')
        for f, _ in cls._fields_:
            lines.append(f'printf("{name}.{f} %zu\\n", offsetof({name}, {f}));')
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "ctvio.h"\nint main(void) {\n' + "\n".join(lines) +
                   "\nreturn 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-x", "c" if not cc.endswith("++") else "c++", str(src), "-I",
                    os.path.join(pkg.REPO_ROOT, "include"), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    got = dict(l.rsplit(" ", 1) for l in out.split("\n") if l)
    for name, cls in structs.items():
        assert int(got[name]) == C.sizeof(cls), name
        for f, _ in cls._fields_:
            assert int(got[f"{name}.{f}"]) == getattr(cls, f).offset, (name, f)
    # the four option words took the place of reserved[4]: the struct keeps its size
    assert C.sizeof(bd.CycleOptions) == bd.CycleOptions.publish_map.offset + 4 + 16


def test_default_options(raw):
    o = _defaults(raw)
    assert (o.publish_pose_covariance, o.publish_odometry_covariance, o.publish_map_covariance) == (0, 0, 0)
    assert o.covariance_gauge_knot == st.ResidentRunner.POSE_COV_GAUGE_KNOT == 3


@pytest.mark.parametrize("field, value, message", [
    ("publish_pose_covariance", 2, "the publish_*_covariance options must be 0 or 1"),
    ("publish_odometry_covariance", -1, "the publish_*_covariance options must be 0 or 1"),
    ("publish_map_covariance", 7, "the publish_*_covariance options must be 0 or 1"),
    ("covariance_gauge_knot", -2, "covariance_gauge_knot must be -1..3"),
    ("covariance_gauge_knot", 4, "covariance_gauge_knot must be -1..3"),
])
def test_option_errors_reach_last_error(raw, field, value, message):
    opt = _defaults(raw)
    setattr(opt, field, value)
    _reset_error(raw)
    assert _start_rc(raw, opt) == ERR_INVALID
    assert raw.ctvio_last_error().decode() == message


def test_map_covariance_requires_the_map(raw):
    opt = _defaults(raw)
    opt.publish_map_covariance = 1
    opt.publish_map = 0
    _reset_error(raw)
    assert _start_rc(raw, opt) == ERR_INVALID
    assert raw.ctvio_last_error().decode() == "publish_map_covariance requires publish_map"
    for gauge in (-1, 0, 3):   # the valid range passes the option checks (and stops at the null handle)
        opt = _defaults(raw)
        opt.publish_map_covariance = opt.publish_pose_covariance = opt.publish_odometry_covariance = 1
        opt.covariance_gauge_knot = gauge
        _reset_error(raw)
        assert _start_rc(raw, opt) == ERR_INVALID
        assert raw.ctvio_last_error().decode() == "null handle"


def test_getter_null_handle(raw):
    info = bd.CycleCovarianceInfo()
    _reset_error(raw)
    assert raw.ctvio_cycle_covariances(None, None, None, None, None, 0, None, C.byref(info)) == ERR_INVALID
    assert raw.ctvio_last_error().decode() == "null handle"


def test_symbols_are_device_only():
    assert "cycle_covariances" in pkg.ABI_SYMBOLS and "cycle_covariances" in bd.DEVICE_ONLY_SYMBOLS


@pytest.mark.parametrize("kw", [dict(covariances=("pose", "velocity")), dict(covariances="pose"),
                                dict(covariances=("map",)), dict(covariances=ALL),
                                dict(covariances=("map",), publish_map=False)])
def test_cycle_runner_checks_covariances(kw):
    with pytest.raises(ValueError):
        st.CycleRunner(None, None, **kw)


@pytest.mark.parametrize("kw", [dict(publish_covariance=True), dict(publish_map_covariance=True),
                                dict(publish_odometry_covariance=True)])
def test_cycle_runner_points_to_covariances(kw):
    with pytest.raises(ValueError, match=r"covariances="):
        st.CycleRunner(None, None, publish_map=True, **kw)


# ---------------------------------------------------------------------------------------------------------- GPU
def _seq(n):
    return st.quantize_wire(st.config_c5_sequence(n + 1))


def _median_parallax(seq, n):
    clouds = st.FrameClouds(seq)
    vals = []
    for w in range(1, n):
        _, _, num, s = st.keyframe_decision([clouds.message(f) for f in range(w, w + st.WIN_KF)], 0.0)
        if num:
            vals.append(s / num)
    return float(np.median(vals))


BASE = dict(triangulate=True, device_features=True, publish_map=True)
REF_COV = dict(publish_covariance=True, publish_odometry_covariance=True, publish_map_covariance=True)


def _runners(lib, seq, deterministic=True, gauge=None, **kw):
    """ResidentRunner with its three publications, CycleRunner with covariances=ALL, the plain CycleRunner"""
    ref = st.ResidentRunner(lib, seq, **BASE, **REF_COV, **kw)
    cyc = st.CycleRunner(lib, seq, **BASE, covariances=ALL, **kw)
    plain = st.CycleRunner(lib, seq, **BASE, **kw)
    if gauge is not None:
        ref.POSE_COV_GAUGE_KNOT = gauge
        cyc.opt.covariance_gauge_knot = gauge
    for r in (ref, cyc, plain):
        r.est.SetDeterministic(deterministic)
    return ref, cyc, plain


def _step_counted(runner):
    """one step and the host waits it made (the counter is per thread: reset right before)"""
    runner.est.SyncStats(reset=True)
    rec = runner.step()
    return rec, runner.est.SyncStats(reset=True)


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def _same_float(a, b):
    return (np.isnan(a) and np.isnan(b)) or a == b


STATE_KEYS = ("marg_flag", "n_obs", "n_lm", "n_imu", "n_triangulated", "n_fallback", "iterations", "termination",
              "prior_dim", "n_removed", "initial_cost", "final_cost", "n_map_points", "n_margin_points")


def _get_prior(e):
    J = np.zeros(1 << 20); r = np.zeros(1 << 12); bt = np.zeros(1 << 12, np.int32); bi = np.zeros(1 << 12, np.int32)
    bc = np.zeros(1 << 12, np.int32); x0 = np.zeros(1 << 14)
    e.lib.call("get_prior", e.h, *(bd._addr(a) for a in (J, r, bt, bi, bc, x0)))
    return J, r, bt, bi, bc, x0


def _no_trace(cyc, plain):
    """the cycle with the publications is bitwise the cycle without them"""
    for a, b in zip(cyc.records, plain.records):
        for k in STATE_KEYS + (("n_reanchored",) if "n_reanchored" in a else ()):
            assert a[k] == b[k], (a["window"], k, a[k], b[k])
    assert cyc.frames == plain.frames
    assert np.array_equal(cyc.q[:cyc.ncp], plain.q[:plain.ncp]) and np.array_equal(cyc.p[:cyc.ncp], plain.p[:plain.ncp])
    assert cyc.ld == plain.ld
    assert np.array_equal(cyc.est.GetBiases(), plain.est.GetBiases())
    assert np.array_equal(cyc.est.GetInvDepths(), plain.est.GetInvDepths())
    assert np.array_equal(cyc.est.GetKnots()[0], plain.est.GetKnots()[0])
    for x, y in zip(cyc.last_map, plain.last_map):
        assert np.array_equal(x, y)
    for x, y in zip(_get_prior(cyc.est), _get_prior(plain.est)):
        assert np.array_equal(x, y)


def _run_parity(lib, seq, n, **kw):
    ref, cyc, plain = _runners(lib, seq, **kw)
    for w in range(n):
        ra = ref.step()
        rb, waits_cov = _step_counted(cyc)
        _, waits_plain = _step_counted(plain)
        assert waits_cov == waits_plain, (w, waits_cov, waits_plain)
        assert _same(ref.last_pose_cov, cyc.last_pose_cov), w
        assert _same(ref.last_rel_cov, cyc.last_rel_cov), w
        assert _same(ref.last_map_cov, cyc.last_map_cov), w
        for key in ("pose_cov_rcond", "rel_cov_rcond", "point_cov_rcond"):
            assert _same_float(ra[key], rb[key]), (w, key, ra[key], rb[key])
        assert ra["n_map_points_without_cov"] == rb["n_map_points_without_cov"], w
        assert ra["n_map_points"] == rb["n_map_points"]
    _no_trace(cyc, plain)
    return ref, cyc, plain


@pytest.mark.gpu
def test_every_frame_keyframe_bitwise():
    ref, cyc, _ = _run_parity(pkg.load(), _seq(8), 8)
    assert all(r["pose_cov_rcond"] >= 1e-14 for r in cyc.records)
    assert cyc.last_map_cov.shape == (cyc.records[-1]["n_map_points"], 3, 3)
    assert cyc.last_rel_cov.shape == (st.WIN_KF - 1, 6, 6)


@pytest.mark.gpu
def test_second_new_every_bitwise():
    _, cyc, _ = _run_parity(pkg.load(), _seq(14), 14, second_new_every=2)
    assert {r["marg_flag"] for r in cyc.records} == {st.MARGIN_OLD, st.MARGIN_SECOND_NEW}


@pytest.mark.gpu
def test_min_parallax_decision_bitwise():
    seq = _seq(8)
    _, cyc, _ = _run_parity(pkg.load(), seq, 8, min_parallax=_median_parallax(seq, 8))
    assert {r["marg_flag"] for r in cyc.records} == {st.MARGIN_OLD, st.MARGIN_SECOND_NEW}


@pytest.mark.gpu
def test_reanchor_bitwise_before_divergence():
    _, cyc, _ = _run_parity(pkg.load(), _seq(8), 8, reanchor=True)
    assert sum(r["n_reanchored"] for r in cyc.records) > 0
    # re-anchored points have no covariance: NaN rows
    assert sum(r["n_map_points_without_cov"] for r in cyc.records) > 0


@pytest.mark.gpu
def test_transfers_at_most_the_runners():
    lib = pkg.load()
    seq = _seq(6)
    ref = st.ResidentRunner(lib, seq, **BASE, **REF_COV)
    cyc = st.CycleRunner(lib, seq, **BASE, covariances=ALL)
    ref.run(6); cyc.run(6)
    # as test_odometry_cycle.py: the messages' bytes, which the runner counts before its timed region, are left out
    clouds = st.FrameClouds(seq)
    sent = np.searchsorted(seq.imu_t, seq.kf_times, side="right")
    for w, (a, b) in enumerate(zip(ref.records, cyc.records)):
        if w == 0:
            continue
        f = st.WIN_KF - 1 + w
        msg = 20 * len(clouds.message(f)[1]) + 8 + 96 * int(sent[f] - sent[f - 1])
        assert b["h2d_bytes"] - msg <= a["h2d_bytes"], (w, a["h2d_bytes"], b["h2d_bytes"], msg)
        assert b["d2h_bytes"] - 8 <= a["d2h_bytes"], (w, a["d2h_bytes"], b["d2h_bytes"])


@pytest.mark.gpu
def test_rank_deficient_window_is_reported_and_the_cycle_goes_on():
    """Without a gauge (covariance_gauge_knot = -1) window 0 has neither a prior nor a fixed knot: rank deficient."""
    seq = _seq(6)
    ref, cyc, plain = _run_parity(pkg.load(), seq, 6, gauge=-1)
    a, b = ref.records[0], cyc.records[0]
    for key in ("pose_cov", "rel_cov", "point_cov"):
        assert np.isnan(a[key + "_rcond"]) and np.isnan(b[key + "_rcond"])
        assert "rank deficient" in a[key + "_error"] and "rank deficient" in b[key + "_error"]
    # the first window's info, read again from the getter of a fresh run stopped after window 0
    lib = pkg.load()
    one = st.CycleRunner(lib, seq, **BASE, covariances=ALL)
    one.opt.covariance_gauge_knot = -1
    one.est.SetDeterministic(True)
    one.step()
    cov12, cov6, cov9, info = one.est.CycleCovariances()
    assert cov12 is None and cov6 is None and cov9 is None
    assert info["status"] == ERR_STATE and info["available"] == 0 and info["requested"] == 7
    assert info["gauge_knot"] == -1
    assert "rank deficient" in info["error"]
    # the pivot-ratio test, or a non-positive pivot (then rcond may pass the threshold), as the separate calls decide
    assert not info["rcond"] >= 1e-14 or "non-positive pivot" in info["error"]
    # the runner's message carries the same rcond and reason
    assert f"rcond {info['rcond']:.3e}" in a["pose_cov_error"]
    assert ("non-positive pivot" in a["pose_cov_error"]) == ("non-positive pivot" in info["error"])


@pytest.mark.gpu
def test_getter_state_errors():
    lib = pkg.load()
    seq = _seq(2)
    cyc = st.CycleRunner(lib, seq, **BASE, covariances=ALL)
    e = cyc.est
    fn = e.lib._fn["cycle_covariances"]
    last = e.lib._fn["last_error"]
    info = bd.CycleCovarianceInfo()
    # before any cycle
    assert fn(e.h, None, None, None, None, C.c_int32(0), None, C.byref(info)) == ERR_STATE
    assert last().decode() == "ctvio_cycle_covariances: not available: no odometry cycle has run"
    assert info.available == 0 and info.status == ERR_STATE and np.isnan(info.rcond)
    with pytest.raises(bd.CtvioError, match="no odometry cycle has run"):
        e.CycleCovariances()
    cyc.step()
    n_map = cyc.records[0]["n_map_points"]
    assert n_map > 1
    # too small a map capacity
    buf = np.zeros((n_map, 3, 3))
    assert fn(e.h, None, None, None, None, C.c_int32(n_map - 1), bd._addr(buf), C.byref(info)) == ERR_INVALID
    assert "map_capacity is smaller" in last().decode()
    assert info.available == 7 and info.n_map_points == n_map
    # NULL outputs, and the capacity that fits
    assert fn(e.h, None, None, None, None, C.c_int32(0), None, None) == 0
    assert fn(e.h, None, None, None, None, C.c_int32(n_map), bd._addr(buf), C.byref(info)) == 0
    assert np.array_equal(buf, cyc.last_map_cov, equal_nan=True)
    # a rejected start changes nothing: the publications stay available and the run goes on
    bad = bd.CycleOptions()
    C.memmove(C.byref(bad), C.byref(cyc.opt), C.sizeof(bad))
    bad.covariance_gauge_knot = 9
    with pytest.raises(bd.CtvioError, match="covariance_gauge_knot must be -1..3"):
        e.OdometryStart(bad, seq.t0_ns, cyc.q[:cyc.ncp], cyc.p[:cyc.ncp], [], [], cyc.bias[:0], cyc.ld)
    cov12, _, _, info2 = e.CycleCovariances()
    assert np.array_equal(cov12[None], cyc.last_pose_cov) and info2["available"] == 7
    cyc.step()
    # after a cycle without the flags: not available
    plain = st.CycleRunner(lib, seq, **BASE)
    plain.step()
    assert plain.est.lib._fn["cycle_covariances"](plain.est.h, None, None, None, None, C.c_int32(0), None,
                                                  C.byref(info)) == ERR_STATE
    assert last().decode() == "ctvio_cycle_covariances: not available: the cycle's options publish no covariances"
    assert info.requested == 0 and info.available == 0


@pytest.mark.gpu
def test_pose_time_and_pairs_are_the_runners():
    lib = pkg.load()
    seq = _seq(3)
    cyc = st.CycleRunner(lib, seq, **BASE, covariances=("pose", "odometry"))
    for _ in range(3):
        frames = list(cyc.frames) + ([cyc.next_frame] if cyc.step_index else [])
        rec = cyc.step()
        info = cyc.last_cov_info
        kf = seq.kf_times[np.asarray(frames)]
        assert np.array_equal(info["pair_t_ns"], np.stack([kf[:-1], kf[1:]], 1))
        # ResidentRunner's TF time: maxTimeNs() of the solved window - 50 ms (ncp: the solved window's knot count)
        assert info["pose_t_ns"] == seq.t0_ns + (cyc.ncp - 3) * seq.dt_ns - st.ResidentRunner.POSE_COV_LAG_NS
        assert info["n_map_points"] == 0 and cyc.last_map_cov is None
        assert "point_cov_rcond" not in rec and rec["pose_cov_rcond"] == info["rcond"]


@pytest.mark.gpu
def test_default_mode_within_tolerance():
    lib = pkg.load()
    seq = _seq(4)
    ref, cyc, _ = _runners(lib, seq, deterministic=False)
    for w in range(4):
        ref.step(); cyc.step()
        for a, b in ((ref.last_pose_cov, cyc.last_pose_cov), (ref.last_rel_cov, cyc.last_rel_cov),
                     (ref.last_map_cov, cyc.last_map_cov)):
            assert a.shape == b.shape
            assert np.array_equal(np.isnan(a), np.isnan(b)), w
            # default mode sums in a run-dependent order, in the solve as in Sigma: relative to each matrix's scale
            for x, y in zip(a.reshape(a.shape[0], -1), b.reshape(b.shape[0], -1)):
                ok = ~np.isnan(x)
                if ok.any():
                    assert np.abs(x[ok] - y[ok]).max() <= 1e-2 * np.abs(x[ok]).max() + 1e-300, w
