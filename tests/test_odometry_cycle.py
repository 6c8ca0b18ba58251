"""The per-image odometry cycle (ctvio_odometry_start / ctvio_process_image) and its runner, CycleRunner.

CPU: every new entry point reports its own argument errors through ctvio_last_error without touching a device, the
ctypes mirrors of the new structs match the header's layout (compiled with the host C compiler), and CycleRunner refuses
the options it does not support.
GPU: CycleRunner is bitwise ResidentRunner(triangulate=True, device_features=True, publish_map=True) in deterministic
mode, per window and after the run (state, frames, the last prior, the map), in both branches of the keyframe decision
and with the re-anchoring slide; the two new kernels (bias random-walk weights, realignment from the device snapshot)
against their host definitions; default mode within the resident parity tolerance; transfers; misuse."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from helpers import pkg, syn

st = pkg.streaming if hasattr(pkg, "streaming") else __import__("importlib").import_module("ctrl-vio_b200.streaming")
bd = pkg.binding
P, I32, I64, F64 = C.c_void_p, C.c_int32, C.c_int64, C.c_double


# ---------------------------------------------------------------------------------------------------------- CPU
@pytest.fixture(scope="module")
def raw():
    lib = C.CDLL(pkg.load().path)
    lib.ctvio_last_error.restype = C.c_char_p
    lib.ctvio_set_knots.argtypes = [P, I32, P, P]
    return lib


def _defaults(raw):
    o = bd.CycleOptions()
    raw.ctvio_cycle_default_options.argtypes = [P]
    assert raw.ctvio_cycle_default_options(C.byref(o)) == 0
    return o


def _start(raw, h, opt, n_frames=11, frames=None, imu=None, override=-1, result=True):
    fn = raw.ctvio_odometry_start
    fn.argtypes = [P, P, I64, I32, P, P, I32, P, P, F64, P, I32, P, P]
    q = np.zeros((4, 4)); q[:, 3] = 1; p = np.zeros((4, 3)); b = np.zeros((n_frames, 6))
    msgs = frames if frames is not None else (bd.ImageMsg * n_frames)()
    res = bd.CycleResult()
    return fn(h, None if opt is None else C.byref(opt), 0, 4, q.ctypes.data, p.ctypes.data, n_frames, msgs, b.ctypes.data,
              0.0, None if imu is None else C.byref(imu), override, None, C.byref(res) if result else None)


def _process(raw, h, img, imu=None, override=-1):
    fn = raw.ctvio_process_image
    fn.argtypes = [P, P, P, I32, P, P]
    res = bd.CycleResult()
    return fn(h, None if img is None else C.byref(img), None if imu is None else C.byref(imu), override, None, C.byref(res))


def _expect(raw, rc, message):
    assert rc < 0
    assert raw.ctvio_last_error().decode() == message


def _reset_error(raw):
    assert raw.ctvio_set_knots(None, 0, None, None) < 0
    assert raw.ctvio_last_error() == b"need >= 4 knots"


def test_start_errors_reach_last_error(raw):
    opt = _defaults(raw)
    _reset_error(raw); _expect(raw, _start(raw, None, opt), "null handle")
    _reset_error(raw); _expect(raw, _start(raw, None, None), "null options")
    for ws in (1, 16, -3):
        bad = _defaults(raw); bad.window_size = ws
        _reset_error(raw); _expect(raw, _start(raw, None, bad, n_frames=ws + 1 if ws > 0 else 1), "window_size must be 2..15")
    _reset_error(raw); _expect(raw, _start(raw, None, opt, n_frames=10), "n_frames must be window_size + 1")
    imu = bd.ImuMsgs(n=1, stride_bytes=40, off_gyro=8, off_accel=32, data=None)
    _reset_error(raw); _expect(raw, _start(raw, None, opt, imu=imu), "bad IMU record layout")
    _reset_error(raw); _expect(raw, _start(raw, None, opt, override=2), "marg_flag_override must be -1, 0 or 1")
    _reset_error(raw); _expect(raw, _start(raw, None, opt, result=False), "null result")
    bad = _defaults(raw); bad.init_depth = 0.0
    _reset_error(raw); _expect(raw, _start(raw, None, bad), "init_depth must be positive")


def test_process_image_errors_reach_last_error(raw):
    img = bd.ImageMsg(t_ns=0, n_points=0)
    _reset_error(raw); _expect(raw, _process(raw, None, img), "null handle")
    _reset_error(raw); _expect(raw, _process(raw, None, None), "null image message")
    bad = bd.ImageMsg(t_ns=0, n_points=2000)
    _reset_error(raw); _expect(raw, _process(raw, None, bad), "n_points must be 0..1024")
    imu = bd.ImuMsgs(n=3, stride_bytes=96, off_gyro=80, off_accel=32, data=None)
    _reset_error(raw); _expect(raw, _process(raw, None, img, imu), "bad IMU record layout")
    _reset_error(raw); _expect(raw, _process(raw, None, img, override=-2), "marg_flag_override must be -1, 0 or 1")


def test_other_new_entry_points_report_null_handle(raw):
    raw.ctvio_sync_stats.argtypes = [P, P, I32]
    _reset_error(raw); _expect(raw, raw.ctvio_sync_stats(None, None, 0), "null handle")
    raw.ctvio_debug_bias_weights.argtypes = [P, I32, P, F64, F64, P]
    _reset_error(raw); _expect(raw, raw.ctvio_debug_bias_weights(None, 2, None, 1.0, 1.0, None), "null handle")
    raw.ctvio_cycle_default_options.argtypes = [P]
    _reset_error(raw); _expect(raw, raw.ctvio_cycle_default_options(None), "null options")


def test_default_options_are_the_runner_values(raw):
    o = _defaults(raw)
    assert (o.window_size, o.solve_iterations, o.predictor_iterations, o.fix_ld) == (st.WINDOW_SIZE, 15, 8, 0)
    assert o.min_parallax == 0.0 and o.init_depth == 5.0 and o.extend_ns == st.EXTEND_NS
    assert (o.ld_lower, o.ld_upper) == (0.0, syn.LD_UPPER)
    assert (o.sigma_wb_discrete, o.sigma_ab_discrete) == (syn.SIGMA_BG, syn.SIGMA_BA)
    assert (o.reanchor, o.publish_map) == (0, 1)


STRUCTS = {
    "ctvio_image_msg": bd.ImageMsg, "ctvio_imu_msgs": bd.ImuMsgs, "ctvio_cycle_options": bd.CycleOptions,
    "ctvio_cycle_outputs": bd.CycleOutputs, "ctvio_cycle_result": bd.CycleResult, "ctvio_summary": bd.Summary,
}


def test_struct_layouts_match_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc") or shutil.which("g++")
    assert cc, "a host C compiler is needed to read the header's layout"
    lines = []
    for name, cls in STRUCTS.items():
        lines.append(f'printf("{name} %zu\\n", sizeof({name}));')
        for f, _ in cls._fields_:
            lines.append(f'printf("{name}.{f} %zu\\n", offsetof({name}, {f}));')
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "ctvio.h"\nint main(void) {\n' + "\n".join(lines) +
                   "\nreturn 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-x", "c" if not cc.endswith("++") else "c++", str(src), "-I",
                    os.path.join(pkg.REPO_ROOT, "include"), "-o", str(exe)], check=True)
    got = dict(l.rsplit(" ", 1) for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n") if l)
    for name, cls in STRUCTS.items():
        assert int(got[name]) == C.sizeof(cls), name
        for f, _ in cls._fields_:
            assert int(got[f"{name}.{f}"]) == getattr(cls, f).offset, (name, f)


def test_symbols_are_device_only():
    for n in ("odometry_start", "process_image", "cycle_default_options", "sync_stats", "debug_bias_weights"):
        assert n in pkg.ABI_SYMBOLS and n in bd.DEVICE_ONLY_SYMBOLS


@pytest.mark.parametrize("kw", [dict(triangulate=False), dict(device_features=False), dict(predictor=False),
                                dict(perm_seed=1), dict(publish_covariance=True), dict(publish_map_covariance=True),
                                dict(publish_odometry_covariance=True), dict(min_parallax=0.01, second_new_every=2),
                                dict(min_parallax=0.0)])
def test_cycle_runner_rejects_unsupported_options(kw):
    with pytest.raises(ValueError):
        st.CycleRunner(None, None, **kw)


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


def _pair(lib, seq, deterministic=True, **kw):
    base = dict(triangulate=True, device_features=True, publish_map=True)
    ref = st.ResidentRunner(lib, seq, **base, **kw)
    cyc = st.CycleRunner(lib, seq, **base, **kw)
    if deterministic:
        ref.est.SetDeterministic(True); cyc.est.SetDeterministic(True)
    priors = []
    adopt = ref.est.AdoptPrior

    def capture():   # the runner adopts right away: keep what ctvio_get_prior returns before (the last one only)
        priors[:] = [_get_prior(ref.est)]
        adopt()
    ref.est.AdoptPrior = capture
    return ref, cyc, priors


def _get_prior(e):
    # the last marginalization's prior through ctvio_get_prior, into buffers larger than any C5 prior (zeros beyond)
    J = np.zeros(1 << 20); r = np.zeros(1 << 12); bt = np.zeros(1 << 12, np.int32); bi = np.zeros(1 << 12, np.int32)
    bc = np.zeros(1 << 12, np.int32); x0 = np.zeros(1 << 14)
    e.lib.call("get_prior", e.h, *(bd._addr(a) for a in (J, r, bt, bi, bc, x0)))
    return J, r, bt, bi, bc, x0


KEYS = ("marg_flag", "n_obs", "n_lm", "n_imu", "n_triangulated", "n_fallback", "iterations", "termination", "prior_dim",
        "n_removed", "initial_cost", "final_cost", "n_map_points", "n_margin_points")


def _compare_bitwise(ref, cyc, priors, n):
    for a, b in zip(ref.records, cyc.records):
        for k in KEYS + (("n_reanchored",) if "n_reanchored" in a else ()):
            assert a[k] == b[k], (a["window"], k, a[k], b[k])
        if "n_tracked" in a:
            assert (a["n_tracked"], a["mean_parallax"]) == (b["n_tracked"], b["mean_parallax"])
    assert len(ref.records) == len(cyc.records) == n
    assert ref.frames == cyc.frames
    assert np.array_equal(ref.q[:ref.ncp], cyc.q[:cyc.ncp]) and np.array_equal(ref.p[:ref.ncp], cyc.p[:cyc.ncp])
    assert ref.ld == cyc.ld
    assert np.array_equal(ref.est.GetBiases(), cyc.est.GetBiases())
    assert np.array_equal(ref.est.GetInvDepths(), cyc.est.GetInvDepths())
    assert np.array_equal(ref.est.GetKnots()[0], cyc.est.GetKnots()[0])
    for x, y in zip(ref.last_map, cyc.last_map):
        assert np.array_equal(x, y)
    if priors:
        for a, b in zip(priors[-1], _get_prior(cyc.est)):
            assert np.array_equal(a, b)


@pytest.mark.gpu
def test_every_frame_keyframe_bitwise():
    lib = pkg.load()
    seq = _seq(8)
    ref, cyc, priors = _pair(lib, seq)
    ref.run(8); cyc.run(8)
    _compare_bitwise(ref, cyc, priors, 8)
    assert all(r["marg_flag"] == st.MARGIN_OLD for r in cyc.records)


@pytest.mark.gpu
def test_second_new_every_bitwise():
    lib = pkg.load()
    seq = _seq(14)
    ref, cyc, priors = _pair(lib, seq, second_new_every=2)
    ref.run(14); cyc.run(14)
    _compare_bitwise(ref, cyc, priors, 14)
    assert {r["marg_flag"] for r in cyc.records} == {st.MARGIN_OLD, st.MARGIN_SECOND_NEW}


@pytest.mark.gpu
def test_min_parallax_decision_bitwise():
    lib = pkg.load()
    seq = _seq(8)
    ref, cyc, priors = _pair(lib, seq, min_parallax=_median_parallax(seq, 8))
    ref.run(8); cyc.run(8)
    _compare_bitwise(ref, cyc, priors, 8)
    assert {r["marg_flag"] for r in cyc.records} == {st.MARGIN_OLD, st.MARGIN_SECOND_NEW}


@pytest.mark.gpu
def test_reanchor_bitwise_before_divergence():
    lib = pkg.load()
    seq = _seq(8)
    ref, cyc, priors = _pair(lib, seq, reanchor=True)
    ref.run(8); cyc.run(8)
    _compare_bitwise(ref, cyc, priors, 8)
    assert sum(r["n_reanchored"] for r in cyc.records) > 0


@pytest.mark.gpu
def test_bias_weights_kernel_matches_host():
    lib = pkg.load()
    seq = _seq(6)
    cyc = st.CycleRunner(lib, seq, publish_map=True)
    e = cyc.est
    s = seq
    for w in range(6):
        cyc.step()
        ingested = s.imu_t[:cyc.imu_sent]
        kf = s.kf_times[np.asarray(cyc.frames)]
        cases = [kf,                                              # the window's frames (C5: no sample on a frame time)
                 np.r_[kf[:3], ingested[-8], ingested[-3]],       # samples exactly on the keyframe times
                 np.r_[kf[-2], kf[-2] + 1, kf[-2] + 2, kf[-1]]]   # an interval without samples: zeros
        for k in cases:
            k = np.asarray(k, np.int64)
            got = e.DebugBiasWeights(k, syn.SIGMA_BG, syn.SIGMA_BA)
            want = syn.bias_sqrt_info(ingested, k)
            assert np.array_equal(got, want), (w, got - want)
        assert np.all(e.DebugBiasWeights(np.r_[kf[-2], kf[-2] + 1, kf[-2] + 2, kf[-1]].astype(np.int64),
                                         syn.SIGMA_BG, syn.SIGMA_BA)[1] == 0.0)


@pytest.mark.gpu
def test_snapshot_realign_matches_host_realign():
    # window 0 of the cycle against the separate calls with the host's R0 / t0: the realigned knots are equal bitwise
    lib = pkg.load()
    seq = _seq(2)
    ref, cyc, _ = _pair(lib, seq)
    ref.step(); cyc.step()
    assert np.array_equal(ref.q[:ref.ncp], cyc.q[:cyc.ncp]) and np.array_equal(ref.p[:ref.ncp], cyc.p[:cyc.ncp])


@pytest.mark.gpu
def test_default_mode_within_resident_tolerance():
    lib = pkg.load()
    seq = _seq(8)
    ref, cyc, _ = _pair(lib, seq, deterministic=False)
    ref.run(8); cyc.run(8)
    for a, b in zip(ref.records, cyc.records):
        assert a["marg_flag"] == b["marg_flag"] and a["n_obs"] == b["n_obs"] and a["n_lm"] == b["n_lm"]
        # default mode sums in a run-dependent order: two runs of one runner differ as much
        assert abs(a["final_cost"] - b["final_cost"]) <= 1e-3 * abs(a["final_cost"])
    assert np.abs(ref.p[:ref.ncp] - cyc.p[:cyc.ncp]).max() < 1e-2
    assert cyc.state_error() <= 1.5 * ref.state_error() + 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("want", [True, False])
def test_transfers_at_most_the_runners(want):
    lib = pkg.load()
    seq = _seq(6)
    ref = st.ResidentRunner(lib, seq, triangulate=True, device_features=True, publish_map=True)
    cyc = st.CycleRunner(lib, seq, publish_map=True, want_knots=want, want_map=want)
    ref.run(6); cyc.run(6)
    # the runner counts from its timed region on, after the new cloud and IMU records went up and the feature table's
    # 8-byte add result came back: those bytes (5 float32 per point + the frame time, 96-byte IMU records; 8 down) are
    # left out of the cycle's count as well
    clouds = st.FrameClouds(seq)
    sent = np.searchsorted(seq.imu_t, seq.kf_times, side="right")
    for w, (a, b) in enumerate(zip(ref.records, cyc.records)):
        if w == 0:
            continue
        f = st.WIN_KF - 1 + w
        msg = 20 * len(clouds.message(f)[1]) + 8 + 96 * int(sent[f] - sent[f - 1])
        assert b["h2d_bytes"] - msg <= a["h2d_bytes"], (a["window"], a["h2d_bytes"], b["h2d_bytes"], msg)
        assert b["d2h_bytes"] - 8 <= a["d2h_bytes"], (a["window"], a["d2h_bytes"], b["d2h_bytes"])


@pytest.mark.gpu
def test_misuse():
    lib = pkg.load()
    seq = _seq(3)
    cyc = st.CycleRunner(lib, seq, publish_map=True)
    e = cyc.est
    # process_image before start
    m = st.FrameClouds(seq).message(11)
    with pytest.raises(bd.CtvioError, match=r"\(-4\)"):
        e.ProcessImage(int(seq.kf_times[11]), m)
    cyc.run(2)   # a valid start (and one image) afterwards
    # the existing calls still work on the engine after a cycle
    q, p = e.GetKnots()
    assert q.shape[0] == e.n_knots and np.isfinite(q).all()
    qq, pp, _, _, _ = e.QueryTrajectory(np.array([seq.kf_times[cyc.frames[-1]]], np.int64))
    assert np.isfinite(qq).all() and np.isfinite(pp).all() and np.isfinite(e.GetBiases()).all()
    # slot exhaustion: the separate calls fill every free slot, the next image finds none and nothing changes
    q_before, p_before = e.GetKnots()
    clouds = st.FrameClouds(seq)
    n_filled = 0
    for k in range(16):
        try:
            e.IngestFeatureCloud(k, int(seq.kf_times[-1]), *clouds.message(len(seq.kf_times) - 1))
            e.FeatureTableAdd(k)
            n_filled += 1
        except bd.CtvioError:
            pass   # a slot the cycle's window holds
    assert n_filled > 0
    with pytest.raises(bd.CtvioError, match="no free frame slot"):
        e.ProcessImage(int(seq.kf_times[-1]), clouds.message(len(seq.kf_times) - 1))
    q_after, p_after = e.GetKnots()
    assert np.array_equal(q_before, q_after) and np.array_equal(p_before, p_after)
    assert e.SyncStats(reset=True) >= 0
