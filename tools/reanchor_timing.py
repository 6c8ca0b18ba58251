"""Host wall clock of the resident feature table's two slides, each call ending in its own stream synchronise:
FeatureTableSlide (landmarks leave with their anchor frame) against FeatureTableSlideReanchor in both branches
(MARGIN_OLD: removeBackShiftDepth with the two camera poses from the resident spline; MARGIN_SECOND_NEW: removeFront), at
two sizes:
  c5    the C5 sequence's windows (11 frame slots of ~300 features), each variant on its own engine as its runner would
        hold the table (depths: truth, so that removeFailures drops nothing);
  full  16 frame slots x 1024 features with overlapping ids, a fresh table per repetition.
Then whole ResidentRunner(triangulate=True, device_features=True) windows with and without reanchor: the record's ms,
n_lm, n_obs, LM iterations, and state_error() at the end.  Prints the card name and power limit, medians and
10th-90th percentiles.
Usage: python tools/reanchor_timing.py [--windows N] [--reps N] [--warmup N]"""
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
from keyframe_timing import spread  # noqa: E402
from triangulate_timing import device_info  # noqa: E402

WS = st.WINDOW_SIZE
VARIANTS = ("slide", "reanchor_margin_old", "reanchor_second_new")


def slide_call(e, variant, slots):
    """the timed call; returns the leaving window position"""
    if variant == "slide":
        e.FeatureTableSlide(int(slots[0]))
        return 0
    marg = variant == "reanchor_margin_old"
    e.FeatureTableSlideReanchor(slots, marg)
    return 0 if marg else len(slots) - 2


def c5_pass(lib, seq, variant, n, warmup):
    clouds = st.FrameClouds(seq)
    e = pkg.Estimator(lib, pkg.make_config(**seq.config_kwargs()))
    e.SetKnots(seq.q0, seq.p0)
    r = types.SimpleNamespace(n_slots=16, slot_of={})
    frames = list(range(st.WIN_KF))
    for f in frames:
        s = st.ResidentRunner._assign_slot(r, f)
        e.IngestFeatureCloud(s, int(seq.kf_times[f]), *clouds.message(f))
        e.FeatureTableAdd(s)
    nxt, samples, n_lm = st.WIN_KF, [], []
    for k in range(n):
        if k:
            frames.append(nxt)
            s = st.ResidentRunner._assign_slot(r, nxt)
            e.IngestFeatureCloud(s, int(seq.kf_times[nxt]), *clouds.message(nxt))
            e.FeatureTableAdd(s)
            nxt += 1
        slots = np.array([r.slot_of[f] for f in frames], np.int32)
        e.FeatureTableWindow(slots, WS)
        ids = e.FeatureTableLandmarks()[0]
        e.SetInvDepths(seq.rho_gt[ids])
        n_lm.append(len(ids))
        t0 = time.perf_counter()
        pos = slide_call(e, variant, slots)
        dt = 1e6 * (time.perf_counter() - t0)
        r.slot_of.pop(frames.pop(pos))
        if k >= warmup:
            samples.append(dt)
    return dict(case="c5", variant=variant, call=spread(samples), landmarks_per_window_median=float(np.median(n_lm)))


def full_reps(lib, variant, reps, warmup, seed=11):
    rng = np.random.default_rng(seed)
    seq = st.config_c5_sequence(6)                                    # 16 keyframes
    e = pkg.Estimator(lib, pkg.make_config(**seq.config_kwargs()))
    e.SetKnots(seq.q0, seq.p0)
    slots = np.arange(16, dtype=np.int32)
    samples, moved = [], []
    for k in range(reps + warmup):
        for s in slots:
            ids = rng.choice(20000, 1024, replace=False).astype(np.float32)
            pts = np.ones((1024, 3), np.float32)
            pts[:, :2] = rng.uniform(-0.5, 0.5, (1024, 2))
            z = np.zeros(1024, np.float32)
            e.IngestFeatureCloud(int(s), int(seq.kf_times[s]), pts, ids, z, z, z, z)
            e.FeatureTableAdd(int(s))
        n_lm = e.FeatureTableWindow(slots, 16)
        e.SetInvDepths(rng.uniform(0.05, 1.0, n_lm))
        t0 = time.perf_counter()
        pos = slide_call(e, variant, slots)
        dt = 1e6 * (time.perf_counter() - t0)
        # empty the table for the next repetition (outside the timed region)
        rest = np.delete(slots, pos)
        e.SetInvDepths(np.full(e.FeatureTableWindow(rest, 16), -1.0))  # every numbered entry fails ...
        for s in rest:
            e.FeatureTableSlide(int(s))                                # ... and every slot leaves
        if k >= warmup:
            samples.append(dt)
    return dict(case="full", variant=variant, call=spread(samples))


def runner_windows(lib, seq, n, skip):
    out = {}
    for re in (False, True):
        r = st.ResidentRunner(lib, seq, triangulate=True, device_features=True, reanchor=re)
        r.run(n)
        recs = r.records[skip:]
        out["reanchor" if re else "default"] = dict(
            ms=spread([1e3 * x["ms"] for x in recs]),
            n_lm_median=float(np.median([x["n_lm"] for x in recs])),
            n_obs_median=float(np.median([x["n_obs"] for x in recs])),
            iterations_mean=float(np.mean([x["iterations"] for x in recs])),
            state_error_m=r.state_error())
    print(json.dumps(dict(case="resident_runner_windows", windows=n - skip, **out)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=60)
    ap.add_argument("--reps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    print(json.dumps(dict(device=device_info())))
    lib = pkg.load()
    seq = st.quantize_wire(st.config_c5_sequence(args.windows + 1))
    for v in VARIANTS:
        print(json.dumps(c5_pass(lib, seq, v, args.windows, args.warmup)))
    for v in VARIANTS:
        print(json.dumps(full_reps(lib, v, args.reps, args.warmup)))
    runner_windows(lib, st.quantize_wire(st.config_c5_sequence(41)), 40, args.warmup)


if __name__ == "__main__":
    main()
