"""Checkpoint and restore of the odometry cycle's run (ctvio_odometry_checkpoint / ctvio_odometry_restore) and the
runner's CycleRunner.checkpoint / restore / resume.

CPU: the argument errors reach ctvio_last_error without a device, and the ctypes prototypes match the header.
GPU (C5, deterministic mode unless said otherwise): a run continued from a checkpoint on a fresh engine is bitwise the
uninterrupted run, per window and after it (knots, biases, inverse depths, line delay, the last prior, the map, the
covariance publications, and the final checkpoint itself, which holds the active prior); rewinding one engine repeats
its run bitwise; taking checkpoints changes nothing; default mode stays within the resident parity tolerance; malformed
blobs and foreign configurations are refused without a trace; state errors; transfers; the size query."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from helpers import pkg

st = __import__("importlib").import_module("ctrl-vio_b200.streaming")
bd = pkg.binding
P, I64 = C.c_void_p, C.c_int64
ERR_INVALID, ERR_STATE = -1, -4


# ---------------------------------------------------------------------------------------------------------- CPU
@pytest.fixture(scope="module")
def raw():
    lib = C.CDLL(pkg.load().path)
    lib.ctvio_last_error.restype = C.c_char_p
    lib.ctvio_set_knots.argtypes = [P, C.c_int32, P, P]
    for name, args in bd.PROTOTYPES.items():
        getattr(lib, "ctvio_" + name).argtypes = args
    return lib


def _expect(raw, rc, message):
    assert rc == ERR_INVALID
    assert raw.ctvio_last_error().decode() == message


def _reset_error(raw):
    assert raw.ctvio_set_knots(None, 0, None, None) < 0
    assert raw.ctvio_last_error() == b"need >= 4 knots"


def test_argument_errors_reach_last_error(raw):
    n = I64(-7)
    buf = C.create_string_buffer(64)
    _reset_error(raw); _expect(raw, raw.ctvio_odometry_checkpoint(None, None, 0, None), "null len")
    _reset_error(raw); _expect(raw, raw.ctvio_odometry_checkpoint(None, buf, -1, C.byref(n)), "capacity must be >= 0")
    _reset_error(raw); _expect(raw, raw.ctvio_odometry_checkpoint(None, None, 0, C.byref(n)), "null handle")
    assert n.value == -7   # nothing written
    _reset_error(raw); _expect(raw, raw.ctvio_odometry_restore(None, None, 8), "null buffer")
    _reset_error(raw); _expect(raw, raw.ctvio_odometry_restore(None, buf, -1), "len must be >= 0")
    _reset_error(raw); _expect(raw, raw.ctvio_odometry_restore(None, buf, 64), "null handle")


_CTYPES = {"ctvio_handle": C.c_void_p, "void*": C.c_void_p, "const void*": C.c_void_p, "int64_t": C.c_int64,
           "int64_t*": C.POINTER(C.c_int64)}


def test_prototypes_match_header():
    hdr = open(os.path.join(pkg.REPO_ROOT, "include", "ctvio.h")).read()
    lib = pkg.load()
    for name, args in bd.PROTOTYPES.items():
        m = re.search(r"\bint ctvio_" + name + r"\(([^)]*)\);", hdr)
        assert m, name
        params = [re.sub(r"\s*\*\s*", "* ", p.strip()).rsplit(" ", 1)[0].strip() for p in m.group(1).split(",")]
        assert [_CTYPES[p] for p in params] == args, (name, params)
        assert lib._fn[name].argtypes == args
        assert name in bd.ABI_SYMBOLS and name in bd.DEVICE_ONLY_SYMBOLS


def test_runner_restore_needs_a_step():
    r = st.CycleRunner.__new__(st.CycleRunner)
    with pytest.raises(ValueError):
        r.restore(dict(step_index=0))


# ---------------------------------------------------------------------------------------------------------- GPU
def _seq(n):
    return st.quantize_wire(st.config_c5_sequence(n + 1))


def _runner(lib, seq, deterministic=True, **kw):
    r = st.CycleRunner(lib, seq, publish_map=True, **kw)
    r.est.SetDeterministic(deterministic)
    return r


def _median_parallax(seq, n):
    clouds = st.FrameClouds(seq)
    vals = []
    for w in range(1, n):
        _, _, num, s = st.keyframe_decision([clouds.message(f) for f in range(w, w + st.WIN_KF)], 0.0)
        if num:
            vals.append(s / num)
    return float(np.median(vals))


def _get_prior(e):
    J = np.zeros(1 << 20); r = np.zeros(1 << 12); bt = np.zeros(1 << 12, np.int32); bi = np.zeros(1 << 12, np.int32)
    bc = np.zeros(1 << 12, np.int32); x0 = np.zeros(1 << 14)
    e.lib.call("get_prior", e.h, *(bd._addr(a) for a in (J, r, bt, bi, bc, x0)))
    return J, r, bt, bi, bc, x0


# measured per call, not part of what the run computes
TIMING = ("ms", "host_ms", "device_ms", "init_device_ms", "h2d_bytes", "d2h_bytes")


def _same_value(x, y):
    if isinstance(x, float) and isinstance(y, float) and np.isnan(x) and np.isnan(y):
        return True
    return x == y


def _same_records(ref_records, got_records):
    assert len(ref_records) == len(got_records)
    for a, b in zip(ref_records, got_records):
        assert set(a) == set(b)
        for k in a:
            if k not in TIMING:
                assert _same_value(a[k], b[k]), (a["window"], k, a[k], b[k])


def _same_run(ref, got):
    assert ref.frames == got.frames and ref.ncp == got.ncp and ref.step_index == got.step_index
    assert np.array_equal(ref.q[:ref.ncp], got.q[:got.ncp]) and np.array_equal(ref.p[:ref.ncp], got.p[:got.ncp])
    assert ref.ld == got.ld
    assert np.array_equal(ref.est.GetBiases(), got.est.GetBiases())
    assert np.array_equal(ref.est.GetInvDepths(), got.est.GetInvDepths())
    assert np.array_equal(ref.est.GetKnots()[0], got.est.GetKnots()[0])
    assert np.array_equal(ref.est.GetKnots()[1], got.est.GetKnots()[1])
    assert np.array_equal(ref.est.GetLineDelay(), got.est.GetLineDelay())
    for x, y in zip(ref.last_map, got.last_map):
        assert np.array_equal(x, y)
    for x, y in ((ref.last_pose_cov, got.last_pose_cov), (ref.last_rel_cov, got.last_rel_cov),
                 (ref.last_map_cov, got.last_map_cov)):
        assert (x is None) == (y is None)
        if x is not None:
            assert np.array_equal(x, y, equal_nan=True)
    if any(r["marg_flag"] == st.MARGIN_OLD for r in got.records):
        for x, y in zip(_get_prior(ref.est), _get_prior(got.est)):
            assert np.array_equal(x, y)
    # everything the next cycle would read, the active prior included
    _same_blob(ref.est.Checkpoint(), got.est.Checkpoint())


SECTIONS = ("meta", "prior_blocks", "knot_q", "knot_p", "bias", "rho", "line_delay", "prior_J", "prior_r", "prior_x0",
            "imu_t", "imu_ga", "imu_carry", "ft_id", "ft_anchor", "ft_mask", "ft_lm", "ft_rho", "ft_key", "ft_idx", "clouds")


def _same_blob(a, b):
    """two checkpoints byte for byte, naming the sections that differ"""
    if a == b:
        return
    table = lambda x: np.frombuffer(x, np.uint64, 2 * len(SECTIONS), 40).reshape(-1, 2)
    ta, tb = table(a), table(b)
    differ = [name for name, (oa, na), (ob, nb) in zip(SECTIONS, ta, tb)
              if (na != nb) or a[int(oa):int(oa + na)] != b[int(ob):int(ob + nb)]]
    assert False, ("the checkpoints differ", len(a), len(b), differ)


def _continue_from(lib, seq, k, n, kw, deterministic=True):
    """an uninterrupted run of n windows, and one checkpointed after window k and continued on a fresh engine"""
    ref = _runner(lib, seq, deterministic, **kw)
    ref.run(n)
    first = _runner(lib, seq, deterministic, **kw)
    first.run(k + 1)
    state = first.checkpoint()
    first.est.close()
    got = st.CycleRunner.resume(lib, seq, state, publish_map=True, **kw)
    got.est.SetDeterministic(deterministic)
    assert got.step_index == k + 1
    got.run(n - k - 1)
    return ref, got


def _first_second_new(lib, seq, n, kw):
    probe = _runner(lib, seq, **kw)
    probe.run(n)
    flags = [r["marg_flag"] for r in probe.records]
    probe.est.close()
    assert st.MARGIN_OLD in flags and st.MARGIN_SECOND_NEW in flags
    return next(w for w in range(1, n - 2) if flags[w] == st.MARGIN_SECOND_NEW)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["start", "second_new", "min_parallax", "reanchor", "covariances"])
def test_continuation_on_a_fresh_engine_is_bitwise(case):
    lib = pkg.load()
    n = 8 if case == "reanchor" else 14
    seq = _seq(n)
    kw, k = {}, 0
    if case == "second_new":
        kw = dict(second_new_every=3)
        k = _first_second_new(lib, seq, n, kw)
    elif case == "min_parallax":
        kw = dict(min_parallax=_median_parallax(seq, n))
        k = _first_second_new(lib, seq, n, kw)
    elif case == "reanchor":
        kw, k = dict(reanchor=True), 3
    elif case == "covariances":
        kw, k = dict(covariances=("pose", "odometry", "map")), 5
    ref, got = _continue_from(lib, seq, k, n, kw)
    if case in ("second_new", "min_parallax"):
        assert ref.records[k]["marg_flag"] == st.MARGIN_SECOND_NEW
    if case == "reanchor":
        assert sum(r["n_reanchored"] for r in ref.records[k + 1:]) > 0
    if case == "covariances":
        assert any(r["pose_cov_rcond"] > 0 for r in got.records)
    _same_records(ref.records[k + 1:], got.records)
    _same_run(ref, got)


@pytest.mark.gpu
def test_rewind_on_one_engine_repeats_the_run():
    lib = pkg.load()
    n, k = 12, 4
    seq = _seq(n)
    r = _runner(lib, seq, second_new_every=3)
    r.run(k + 1)
    state = r.checkpoint()
    r.run(n - k - 1)
    first_records, first_blob = list(r.records), r.est.Checkpoint()
    q, p, ld, last_map = r.q.copy(), r.p.copy(), r.ld, r.last_map
    r.restore(state)
    r.run(n - k - 1)
    _same_records(first_records[k + 1:], r.records)
    assert np.array_equal(q, r.q) and np.array_equal(p, r.p) and ld == r.ld
    for x, y in zip(last_map, r.last_map):
        assert np.array_equal(x, y)
    _same_blob(r.est.Checkpoint(), first_blob)


@pytest.mark.gpu
def test_checkpoints_leave_the_run_unchanged_and_the_size_query_is_exact():
    lib = pkg.load()
    n = 10
    seq = _seq(n)
    plain = _runner(lib, seq, second_new_every=3)
    plain.run(n)
    r = _runner(lib, seq, second_new_every=3)
    fn = lib._fn["odometry_checkpoint"]
    for _ in range(n):
        r.step()
        need = I64()
        assert fn(r.est.h, None, 0, C.byref(need)) == 0
        buf = C.create_string_buffer(need.value + 64)
        got = I64()
        assert fn(r.est.h, buf, need.value + 64, C.byref(got)) == 0
        assert got.value == need.value
        short = C.create_string_buffer(need.value - 1)
        assert fn(r.est.h, short, need.value - 1, C.byref(got)) == ERR_INVALID and got.value == need.value
    _same_records(plain.records, r.records)
    _same_run(plain, r)


@pytest.mark.gpu
def test_default_mode_continuation_within_resident_tolerance():
    lib = pkg.load()
    n, k = 8, 3
    seq = _seq(n)
    ref, got = _continue_from(lib, seq, k, n, {}, deterministic=False)
    for a, b in zip(ref.records[k + 1:], got.records):
        assert a["marg_flag"] == b["marg_flag"] and a["n_obs"] == b["n_obs"] and a["n_lm"] == b["n_lm"]
        # default mode sums in a run-dependent order: two runs of one runner differ as much
        assert abs(a["final_cost"] - b["final_cost"]) <= 1e-3 * abs(a["final_cost"])
    assert np.abs(ref.p[:ref.ncp] - got.p[:got.ncp]).max() < 1e-2
    assert got.state_error() <= 1.5 * ref.state_error() + 1e-3


def _restore_rc(e, blob):
    return e.lib._fn["odometry_restore"](e.h, blob, len(blob))


@pytest.mark.gpu
def test_malformed_blobs_and_foreign_configs_are_refused_without_a_trace():
    lib = pkg.load()
    n, k = 6, 3
    seq = _seq(n)
    ref = _runner(lib, seq)
    ref.run(k + 2)
    r = _runner(lib, seq)
    r.run(k + 1)
    blob = r.est.Checkpoint()
    hdr = bd.Estimator.CHECKPOINT_HEADER_BYTES
    bad = []
    for at in (hdr + 137, len(blob) // 2, len(blob) - 5):   # a frame time of the counts section, the device sections, the last cloud
        b = bytearray(blob); b[at] ^= 0x10; bad.append((bytes(b), "checksum mismatch"))
    bad.append((blob[:-8], "the length differs from the blob's own (truncated or padded)"))
    b = bytearray(blob); b[0] ^= 1; bad.append((bytes(b), "not a checkpoint (bad magic number)"))
    b = bytearray(blob); b[8] = 2; bad.append((bytes(b), "format version 2 (this library reads version 1 only)"))
    for b, why in bad:
        assert _restore_rc(r.est, b) == ERR_INVALID
        assert lib._fn["last_error"]().decode() == "ctvio_odometry_restore: " + why
    _same_blob(r.est.Checkpoint(), blob)
    # an engine of another configuration refuses the blob and keeps its own (empty) run
    cfg = pkg.make_config(device=0, **seq.config_kwargs())
    cfg.image_weight *= 2
    other = bd.Estimator(lib, cfg)
    assert _restore_rc(other, blob) == ERR_INVALID
    assert lib._fn["last_error"]().decode() == "ctvio_odometry_restore: the configuration differs from the engine's"
    n_len = I64()
    assert lib._fn["odometry_checkpoint"](other.h, None, 0, C.byref(n_len)) == ERR_STATE
    other.close()
    # the refused restores left nothing behind: the next cycle is the uninterrupted run's
    r.step()
    _same_records(ref.records[k + 1:], r.records[k + 1:])
    _same_run(ref, r)


@pytest.mark.gpu
def test_state_errors():
    lib = pkg.load()
    seq = _seq(3)
    r = _runner(lib, seq)
    n = I64()
    fn = lib._fn["odometry_checkpoint"]
    assert fn(r.est.h, None, 0, C.byref(n)) == ERR_STATE   # before a start
    r.run(2)
    assert fn(r.est.h, None, 0, C.byref(n)) == 0 and n.value > 0
    # a cycle that stops on an error (knot outputs too small, reported after the cycle ran)
    f = r.next_frame
    m, _keep = bd.Estimator._image_msg(int(seq.kf_times[f]), r.clouds.message(f))
    q = np.zeros((1, 4)); p = np.zeros((1, 3))
    out = bd.CycleOutputs(knot_capacity=1, q_xyzw=q.ctypes.data, p_xyz=p.ctypes.data)
    res = bd.CycleResult()
    assert lib._fn["process_image"](r.est.h, C.byref(m), None, -1, C.byref(out), C.byref(res)) == ERR_INVALID
    assert fn(r.est.h, None, 0, C.byref(n)) == ERR_STATE
    assert "stopped on an error" in lib._fn["last_error"]().decode()


@pytest.mark.gpu
def test_transfers_are_the_blob_one_way():
    lib = pkg.load()
    seq = _seq(4)
    r = _runner(lib, seq)
    r.run(3)
    r.est.TransferStats(reset=True)
    blob = r.est.Checkpoint()
    assert r.est.TransferStats(reset=True) == (0, len(blob))
    fresh = st.CycleRunner(lib, seq, publish_map=True)
    fresh.est.SetDeterministic(True)
    fresh.est.TransferStats(reset=True)
    fresh.est.Restore(blob)
    assert fresh.est.TransferStats(reset=True) == (len(blob), 4)   # the device check's verdict comes back
    _same_blob(fresh.est.Checkpoint(), blob)
