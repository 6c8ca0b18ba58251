"""Timing of the device structure build (structure.cu) against the library before it, in one process.

    python tools/structure_timing.py PREV.so [NEW.so] [--windows 60] [--rounds 3] [--reps 30] [--out build/structure_timing.json]

PREV.so: a build of libctvio_b200.so whose structure build of table-built factors runs on the host (the descriptors read
back by ctvio_add_image_features_from_table); NEW.so defaults to the in-tree build.  Both are loaded with RTLD_DEEPBIND
as tools/pdl_ab.py does.
  - whole ResidentRunner(triangulate=True, device_features=True) windows of the wire-quantized C5 sequence, builds
    alternating per round (the first 5 windows of each run skipped): ms per window, its spread, d2h bytes per window;
  - per call, at one C5 window and at full tables (16 slots x 1 024 features): host wall clock of
    AddImageFeaturesFromTable, wall clock and summary.device_ms of the Solve that follows (it builds the structure);
  - a separate torch.profiler run of one such add + solve with the new build: the kernels of the structure build and
    their durations.
Prints one JSON line with the card's name and power limit and writes it to --out.
"""
import argparse
import ctypes
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
pkg = importlib.import_module("ctrl-vio_b200")
st = importlib.import_module("ctrl-vio_b200.streaming")
from pdl_ab import card, stats  # noqa: E402

STRUCTURE_KERNELS = ("structure_kernel", "schur_lists_kernel", "marg_discover_kernel", "offset_positions_kernel",
                     "gather_factors_kernel", "feature_table_factors_kernel")


def load(path):
    """as pdl_ab.load; the previous build lacks ctvio_debug_structure"""
    ctypes.CDLL(path, mode=os.RTLD_LOCAL | os.RTLD_DEEPBIND | os.RTLD_NOW)
    return pkg.CtvioLib(path, optional=("debug_structure",))


def c5_engine(lib):
    """one C5 window of the resident table: 11 clouds, numbered and triangulated"""
    seq = st.quantize_wire(st.config_c5_sequence(2))
    clouds = st.FrameClouds(seq)
    e = pkg.Estimator(lib, pkg.make_config(**seq.config_kwargs()))
    e.SetKnots(seq.q0, seq.p0); e.SetBiases(seq.bias0[:st.WIN_KF]); e.SetLineDelay(seq.ld0)
    for f in range(st.WIN_KF):
        e.IngestFeatureCloud(f, int(seq.kf_times[f]), *clouds.message(f))
        e.FeatureTableAdd(f)
    e.FeatureTableWindow(np.arange(st.WIN_KF, dtype=np.int32), st.WINDOW_SIZE)
    e.TriangulateWindowFromTable()
    return e


def full_engine(lib, seed=11):
    """full tables: 16 slots x 1 024 features with overlapping ids, one window over all of them"""
    seq = st.config_c5_sequence(8)
    rng = np.random.default_rng(seed)
    e = pkg.Estimator(lib, pkg.make_config(**seq.config_kwargs()))
    e.SetKnots(seq.q0, seq.p0); e.SetBiases(seq.bias0[:2]); e.SetLineDelay(seq.ld0)
    for s in range(16):
        ids = rng.choice(20000, 1024, replace=False).astype(np.float32)
        pts = np.ones((1024, 3), np.float32)
        pts[:, 0] = 1e-4 * (ids % 97); pts[:, 1] = -1e-4 * (ids % 89)
        z = np.zeros(1024, np.float32)
        e.IngestFeatureCloud(s, int(seq.kf_times[s]), pts, ids, z, (ids % 480).astype(np.float32), z, z)
        e.FeatureTableAdd(s)
    n = e.FeatureTableWindow(np.arange(16, dtype=np.int32), 16)
    e.SetInvDepths(rng.uniform(0.1, 1.0, n))
    return e


def per_call(e, reps, iters=3):
    """AddImageFeaturesFromTable wall clock, then the Solve that builds the structure (wall clock, device_ms)"""
    e.SetOptions(pkg.make_options())
    e.SaveState()
    add, solve, dev, d2h = [], [], [], []
    for r in range(reps + 3):
        e.RestoreState()
        e.ClearFactors()
        e.TransferStats(reset=True)
        t0 = time.perf_counter()
        n = e.AddImageFeaturesFromTable(1)
        t1 = time.perf_counter()
        s = e.Solve(iters)
        t2 = time.perf_counter()
        if r >= 3:
            add.append(1e3 * (t1 - t0)); solve.append(1e3 * (t2 - t1)); dev.append(s.device_ms)
            d2h.append(e.TransferStats(reset=True)[1])
    return {"n_factors": n, "add_ms": stats([add]), "solve_wall_ms": stats([solve]), "solve_device_ms": stats([dev]),
            "d2h_bytes_add_and_solve": int(np.median(d2h))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("prev")
    ap.add_argument("new", nargs="?", default=None)
    ap.add_argument("--windows", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=os.path.join(ROOT, "build", "structure_timing.json"))
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("structure_timing.py needs a CUDA device")
    new = os.path.abspath(args.new) if args.new else pkg.load().path
    libs = {"prev": load(os.path.abspath(args.prev)), "new": load(new)}
    res = {"card": card(), "prev": args.prev, "new": new}

    # ---- whole C5 windows, alternating builds ----
    seq = st.quantize_wire(st.config_c5_sequence(args.windows))
    ms = {k: [] for k in libs}
    d2h = {k: [] for k in libs}
    for r in range(args.rounds):
        for k in (("prev", "new") if r % 2 == 0 else ("new", "prev")):
            rr = st.ResidentRunner(libs[k], seq, triangulate=True, device_features=True, device=0)
            rr.run(args.windows)
            ms[k].append([x["ms"] for x in rr.records[5:]])
            d2h[k] += [x["d2h_bytes"] for x in rr.records[5:]]
            del rr
    res["c5_window_ms"] = {k: stats(v) for k, v in ms.items()}
    res["c5_window_d2h_bytes_median"] = {k: float(np.median(v)) for k, v in d2h.items()}
    res["c5_window_median_change"] = res["c5_window_ms"]["new"]["median"] / res["c5_window_ms"]["prev"]["median"] - 1.0

    # ---- per call: add from the table + the structure-building solve ----
    for name, make in (("c5", c5_engine), ("full", full_engine)):
        res[name + "_per_call"] = {k: per_call(make(lib), args.reps) for k, lib in libs.items()}

    # ---- kernels of one add + solve (separate, traced run) ----
    from torch.profiler import ProfilerActivity, profile

    kern = {}
    for name, make in (("c5", c5_engine), ("full", full_engine)):
        e = make(libs["new"])
        e.SetOptions(pkg.make_options())
        e.ClearFactors()
        e.AddImageFeaturesFromTable(1)
        e.Solve(1)  # warm-up
        e.ClearFactors()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            e.AddImageFeaturesFromTable(1)
            e.Solve(1)
            torch.cuda.synchronize()
        rows = {}
        for ev in prof.events():
            if ev.device_type.name == "CUDA" and any(s in ev.name for s in STRUCTURE_KERNELS):
                key = next(s for s in STRUCTURE_KERNELS if s in ev.name)
                rows.setdefault(key, []).append(ev.time_range.elapsed_us() / 1e3)
        kern[name] = {k: {"calls": len(v), "ms": float(np.sum(v))} for k, v in rows.items()}
    res["kernels_ms"] = kern

    line = json.dumps(res)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(line + "\n")
    print(line)
    c = res["c5_window_ms"]
    print(f"C5 ms/window  prev {c['prev']['median']:.4f} [{c['prev']['round_median_min']:.4f}, {c['prev']['round_median_max']:.4f}]"
          f"  new {c['new']['median']:.4f} [{c['new']['round_median_min']:.4f}, {c['new']['round_median_max']:.4f}]"
          f"  change {100 * res['c5_window_median_change']:+.2f} %  d2h/window {res['c5_window_d2h_bytes_median']}")
    for name in ("c5", "full"):
        for k in libs:
            p = res[name + "_per_call"][k]
            print(f"{name:4s} {k:4s} n={p['n_factors']}  add {p['add_ms']['median']:.4f} ms  solve wall "
                  f"{p['solve_wall_ms']['median']:.4f} ms  device {p['solve_device_ms']['median']:.4f} ms  d2h "
                  f"{p['d2h_bytes_add_and_solve']} B")
    print("kernels:", json.dumps(kern))


if __name__ == "__main__":
    main()
