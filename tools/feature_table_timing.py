"""Host wall clock of the resident feature table's calls for one window (FeatureTableAdd + FeatureTableWindow +
AddImageFeaturesFromTable + FeatureTableSlide, each ending in its own stream synchronise), against the host work they
replace, at two sizes:
  c5    the C5 sequence's windows (11 frame slots of ~300 features): the host side is ResidentRunner's index construction
        (subwindow_frames, old index, factor selection, observation CSR) + RemapLandmarks + AddImageFeaturesFromSlots,
        and separately streaming.FeatureTable (the numpy restatement) doing the table's work;
  full  16 frame slots x 1024 features with overlapping ids, one slot replaced per window: the device calls and
        FeatureTable.
Then whole ResidentRunner(triangulate=True) windows with and without device_features (median ms per window and the
per-window h2d / d2h bytes of TransferStats), and (separate, traced run) the kernels of one window's table calls, from
torch.profiler.  Prints the card name and power limit, medians and 10th-90th percentiles.
Both sides hold the same table throughout: after each window the device's re-laid-out inverse depths are checked
bitwise against the numpy table's and both sides get |rho| (outside the timed region; it stands in for triangulation
and the solve, so removeFailures drops nothing), and every device count is asserted equal to the numpy one.
Usage: python tools/feature_table_timing.py [--windows N] [--passes N]"""
import argparse
import importlib
import json
import os
import sys
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
pkg = importlib.import_module("ctrl-vio_b200")
st = importlib.import_module("ctrl-vio_b200.streaming")
syn = st.syn
from keyframe_timing import spread  # noqa: E402
from triangulate_timing import device_info  # noqa: E402

WS = st.WINDOW_SIZE


def bitwise(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def solved(e, table, rho_t):
    """outside the timed region: check the device's re-laid-out depths against the numpy table's, then give both sides
    the same positive depths (|rho|: what triangulation and the solve leave), so that neither side's removeFailures
    drops the window's landmarks and both tables stay the same size"""
    assert len(rho_t) == len(table.numbered) and bitwise(e.GetInvDepths(), rho_t)
    rho_t = np.abs(rho_t)
    e.SetInvDepths(rho_t)
    return rho_t


def n_factors(table, slots):
    return int(table.used_num(slots)[table.numbered].sum()) - len(table.numbered)


def timed(samples, key, fn):
    t0 = time.perf_counter()
    r = fn()
    samples.setdefault(key, []).append(1e6 * (time.perf_counter() - t0))
    return r


def c5_pass(lib, seq, n, samples, warmup, counts):
    """one pass over the sequence's windows (MARGIN_OLD): device table calls, and the host path's work on a second
    engine, per window; every device count is checked against the numpy table's"""
    clouds = st.FrameClouds(seq)
    e = pkg.Estimator(lib, pkg.make_config(**seq.config_kwargs()))
    h = pkg.Estimator(lib, pkg.make_config(**seq.config_kwargs()))
    r = types.SimpleNamespace(n_slots=16, slot_of={}, clouds=clouds, seq=seq)
    table = st.FeatureTable()
    frames = list(range(st.WIN_KF))
    for f in frames:
        s = st.ResidentRunner._assign_slot(r, f)
        for x in (e, h):
            x.IngestFeatureCloud(s, int(seq.kf_times[f]), *clouds.message(f))
        e.FeatureTableAdd(s)
        table.add(s, clouds.message(f))
    prev_lm, nxt = None, st.WIN_KF
    rho_t = np.zeros(0)
    for k in range(n):
        rec = {}
        if k:
            frames.append(nxt)
            s = st.ResidentRunner._assign_slot(r, nxt)
            m = clouds.message(nxt)
            for x in (e, h):
                x.IngestFeatureCloud(s, int(seq.kf_times[nxt]), *m)
            nxt += 1
            added = timed(rec, "device_add", lambda: e.FeatureTableAdd(s))
            assert added == timed(rec, "numpy_table", lambda: table.add(s, m))
        slots = np.array([r.slot_of[f] for f in frames], np.int32)
        n_lm = timed(rec, "device_window", lambda: e.FeatureTableWindow(slots, WS))
        rho_t = timed(rec, "numpy_table_window", lambda: table.window(slots, WS, rho_t))
        assert n_lm == len(table.numbered)
        rho_t = solved(e, table, rho_t)
        e.ClearFactors()
        n_f = timed(rec, "device_factors", lambda: e.AddImageFeaturesFromTable(True))
        assert n_f == len(timed(rec, "numpy_table_factors", lambda: table.factors(rho_t, True))[0])
        counts.append((n_lm, n_f))

        def host_indices():
            fr = np.asarray(frames, np.int64)
            w = syn.subwindow_frames(seq, fr, window_size=WS)
            lm = w.meta["lm_global"]
            if prev_lm is None:
                old = np.full(len(lm), -1, np.int32)
            else:
                pos = np.clip(np.searchsorted(prev_lm, lm), 0, len(prev_lm) - 1)
                old = np.where(prev_lm[pos] == lm, pos, -1).astype(np.int32)
            sel = st.ResidentRunner._factor_selection(r, fr, lm)
            slot_j, idx_j = slots[w.obs_frame], clouds.obs_idx[sel]
            csr = st.ResidentRunner._observation_csr(r, fr, w, lm, slot_j, idx_j, slots)
            args = (slots[w.anchor_frame[w.lm]], clouds.anchor_idx[lm[w.lm]], slot_j, idx_j, w.lm,
                    (w.anchor_frame[w.lm] == 0).astype(np.int32))
            return lm, old, args, csr
        lm, old, args, _ = timed(rec, "host_indices", host_indices)
        timed(rec, "host_remap", lambda: h.RemapLandmarks(old, np.full(len(lm), -1.0)))
        h.ClearFactors()
        timed(rec, "host_add_from_slots", lambda: h.AddImageFeaturesFromSlots(*args))
        prev_lm = lm
        leave = r.slot_of.pop(frames.pop(0))
        removed = timed(rec, "device_slide", lambda: e.FeatureTableSlide(leave))
        assert removed == timed(rec, "numpy_table_slide", lambda: table.slide(leave, rho_t))
        if k >= max(warmup, 1):
            for key, v in rec.items():
                samples.setdefault(key, []).extend(v)
    return e


def full_pass(lib, n, samples, warmup, counts, seed=11):
    rng = np.random.default_rng(seed)
    seq = st.config_c5_sequence(1)
    e = pkg.Estimator(lib, pkg.make_config(**seq.config_kwargs()))
    table = st.FeatureTable()

    def cloud():
        ids = rng.choice(20000, 1024, replace=False).astype(np.float32)
        pts = np.ones((1024, 3), np.float32)
        z = np.zeros(1024, np.float32)
        return pts, ids, z, z, z, z
    order = list(range(16))
    for s in order:
        m = cloud()
        e.IngestFeatureCloud(s, 0, *m)
        e.FeatureTableAdd(s)
        table.add(s, m)
    rho_t = np.zeros(0)
    for k in range(n):
        rec = {}
        slots = np.array(order, np.int32)
        n_lm = timed(rec, "device_window", lambda: e.FeatureTableWindow(slots, 16))
        rho_t = timed(rec, "numpy_table_window", lambda: table.window(slots, 16, rho_t))
        assert n_lm == len(table.numbered)
        rho_t = solved(e, table, rho_t)
        e.ClearFactors()
        n_f = timed(rec, "device_factors", lambda: e.AddImageFeaturesFromTable(True))
        assert n_f == n_factors(table, slots)   # (the numpy factor list, a Python loop over ~10^5 factors, is not timed)
        counts.append((len(table.id), n_lm, n_f))
        leave = order.pop(0)
        removed = timed(rec, "device_slide", lambda: e.FeatureTableSlide(leave))
        assert removed == timed(rec, "numpy_table_slide", lambda: table.slide(leave, rho_t))
        m = cloud()
        e.IngestFeatureCloud(leave, 0, *m)
        order.append(leave)
        added = timed(rec, "device_add", lambda: e.FeatureTableAdd(leave))
        assert added == timed(rec, "numpy_table", lambda: table.add(leave, m))
        if k >= warmup:
            for key, v in rec.items():
                samples.setdefault(key, []).extend(v)
    return e


def summarize(name, samples, extra=None):
    dev = np.sum([samples[k] for k in ("device_add", "device_window", "device_factors", "device_slide")], axis=0)
    out = dict(case=name, device_window_total=spread(dev), **{k: spread(v) for k, v in samples.items()})
    if "host_indices" in samples:
        host = np.sum([samples[k] for k in ("host_indices", "host_remap", "host_add_from_slots")], axis=0)
        out["host_path_total"] = spread(host)
    out.update(extra or {})
    print(json.dumps(out))


def runner_windows(lib, seq, n, skip):
    out = {}
    for df in (False, True):
        r = st.ResidentRunner(lib, seq, triangulate=True, device_features=df)
        step_us = []
        for _ in range(n):
            t0 = time.perf_counter()
            r.step()
            step_us.append(1e6 * (time.perf_counter() - t0))
        recs = r.records[skip:]
        # timed_window: the record's ms (C-ABI calls; the host association is outside it); whole_step: all of step()
        out["device_features" if df else "host_association"] = dict(
            timed_window_us=spread([1e3 * x["ms"] for x in recs]), whole_step_us=spread(step_us[skip:]),
            h2d_bytes_median=float(np.median([x["h2d_bytes"] for x in recs])),
            d2h_bytes_median=float(np.median([x["d2h_bytes"] for x in recs])))
    print(json.dumps(dict(case="resident_runner_windows", windows=n - skip, **out)))


def trace_window(lib, seq):
    """kernels and copies of one window's table calls (traced run of its own, after the timings), on a table in the
    state the runner keeps it: the window before it numbered, given positive depths and slid"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    clouds = st.FrameClouds(seq)
    e = pkg.Estimator(lib, pkg.make_config(**seq.config_kwargs()))
    table = st.FeatureTable()
    for f in range(st.WIN_KF + 1):
        e.IngestFeatureCloud(f, int(seq.kf_times[f]), *clouds.message(f))
    for f in range(st.WIN_KF):
        e.FeatureTableAdd(f)
        table.add(f, clouds.message(f))
    slots = np.arange(st.WIN_KF, dtype=np.int32)
    e.FeatureTableWindow(slots, WS)
    rho_t = solved(e, table, table.window(slots, WS, np.zeros(0)))
    assert e.FeatureTableSlide(0) == table.slide(0, rho_t)
    table.add(st.WIN_KF, clouds.message(st.WIN_KF))
    slots = np.arange(1, st.WIN_KF + 1, dtype=np.int32)
    kernels, copies = [], []

    def traced(fn):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            out = fn()
            torch.cuda.synchronize()
        ev = [x for x in prof.events() if x.device_type == torch.autograd.DeviceType.CUDA]
        kernels.extend((x.name, round(x.device_time, 2)) for x in ev if "emcpy" not in x.name and "emset" not in x.name)
        copies.extend(x.name for x in ev if "emcpy" in x.name or "emset" in x.name)
        return out
    traced(lambda: e.FeatureTableAdd(st.WIN_KF))
    n_lm = traced(lambda: e.FeatureTableWindow(slots, WS))
    rho_t = solved(e, table, table.window(slots, WS, rho_t))     # between the traced calls
    e.ClearFactors()
    n_f = traced(lambda: e.AddImageFeaturesFromTable(True))
    assert n_lm == len(table.numbered) and n_f == n_factors(table, slots)
    assert traced(lambda: e.FeatureTableSlide(1)) == table.slide(1, rho_t)
    print(json.dumps(dict(traced_kernels_us=kernels, count=len(kernels), copies=copies, n_landmarks=n_lm, n_factors=n_f)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=60)
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    print(json.dumps(dict(device=device_info())))
    lib = pkg.load()
    seq = st.quantize_wire(st.config_c5_sequence(args.windows + 1))
    samples, counts = {}, []
    for _ in range(args.passes):
        c5_pass(lib, seq, args.windows, samples, args.warmup, counts)
    c = np.asarray(counts)
    summarize("c5", samples, dict(landmarks_per_window=[int(c[:, 0].min()), int(np.median(c[:, 0])), int(c[:, 0].max())],
                                  factors_per_window=[int(c[:, 1].min()), int(np.median(c[:, 1])), int(c[:, 1].max())]))
    samples, counts = {}, []
    full_pass(lib, args.windows, samples, args.warmup, counts)
    c = np.asarray(counts)[args.warmup:]
    summarize("full", samples, dict(entries_landmarks_factors_median=[int(x) for x in np.median(c, axis=0)],
                                    entries_landmarks_factors_min=[int(x) for x in c.min(axis=0)]))
    runner_windows(lib, seq, min(args.windows, 40), args.warmup)
    trace_window(lib, seq)


if __name__ == "__main__":
    main()
