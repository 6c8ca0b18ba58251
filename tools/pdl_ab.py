"""A/B of two builds of libctvio_b200.so in one process: C2 solve(15) device_ms, C5 resident ms per window, C4 solve ms.

    python tools/pdl_ab.py A.so B.so [--rounds 5] [--solves 20] [--c5-windows 120] [--c4-solves 4] [--c4x]

Both libraries are loaded through CtvioLib.  They export the same symbol names, so each is first opened with
RTLD_DEEPBIND: its own calls bind to its own definitions, not to the copy that was loaded first.
C2: the estimator set up as bench.py sets it up, `--rounds` rounds that alternate the builds (A then B, B then A, ...),
each `--solves` timed solves with a 256 MiB buffer written between solves to flush L2 (as bench.py does); the median
and spread (min / max of the round medians, and of all solves) of summary.device_ms per build.
C5: whole windows of the device-resident streaming runner (bench.py's gpu_resident), alternating builds per round; the
first 5 windows of each run are skipped as bench.py skips them.
C4 (10 000 landmarks, speculation off): solve ms per build, alternating; --c4x adds the 100 000-landmark window.
Prints one JSON line with the card's name and power limit; writes it to --out as well (default build/pdl_ab.json).
"""
import argparse
import ctypes
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("ctrl-vio_b200")
syn = pkg.synthetic
MAX_ITERS = 15


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20)
        out["power_limit_w"] = float(r.stdout.strip())
    except Exception:
        pass
    return out


def load(path):
    ctypes.CDLL(path, mode=os.RTLD_LOCAL | os.RTLD_DEEPBIND | os.RTLD_NOW)
    return pkg.CtvioLib(path)


def stats(rounds):
    med = [float(np.median(r)) for r in rounds]
    allv = [x for r in rounds for x in r]
    return {"median": float(np.median(allv)), "round_medians": med, "round_median_min": min(med),
            "round_median_max": max(med), "min": float(min(allv)), "max": float(max(allv)), "n": len(allv)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("a")
    ap.add_argument("b")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--solves", type=int, default=20)
    ap.add_argument("--c5-windows", type=int, default=120)
    ap.add_argument("--c5-rounds", type=int, default=3)
    ap.add_argument("--c4-solves", type=int, default=4)
    ap.add_argument("--c4x", action="store_true")
    ap.add_argument("--out", default=os.path.join(ROOT, "build", "pdl_ab.json"))
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("pdl_ab.py needs a CUDA device")
    libs = {"A": load(os.path.abspath(args.a)), "B": load(os.path.abspath(args.b))}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    res = {"card": card(), "A": args.a, "B": args.b}

    # ---- C2 ----
    w = syn.config_c2(seed=syn.SEED0 + 2)
    est = {}
    for k, lib in libs.items():
        est[k] = pkg.setup_estimator(lib, w, device=0)
        est[k].SaveState()

    def c2_solve(k, it):
        est[k].RestoreState()
        flush.fill_(it & 0xFF)
        torch.cuda.synchronize()
        return est[k].Solve(MAX_ITERS)

    for k in libs:
        for it in range(3):
            c2_solve(k, it)
    c2 = {k: [] for k in libs}
    iters = {k: set() for k in libs}
    for r in range(args.rounds):
        for k in (("A", "B") if r % 2 == 0 else ("B", "A")):
            ms = []
            for it in range(args.solves):
                s = c2_solve(k, it)
                ms.append(s.device_ms)
                iters[k].add((s.iterations, s.num_jacobian_evals))
            c2[k].append(ms)
    res["c2_device_ms"] = {k: dict(stats(v), iterations_passes=sorted(iters[k])) for k, v in c2.items()}
    res["c2_median_change"] = res["c2_device_ms"]["B"]["median"] / res["c2_device_ms"]["A"]["median"] - 1.0
    del est

    # ---- C5: device-resident streaming windows ----
    if args.c5_windows > 0:
        st = importlib.import_module("ctrl-vio_b200.streaming")
        seq = st.quantize_wire(st.config_c5_sequence(args.c5_windows))
        c5 = {k: [] for k in libs}
        dev5 = {k: [] for k in libs}
        for r in range(args.c5_rounds):
            for k in (("A", "B") if r % 2 == 0 else ("B", "A")):
                rr = st.ResidentRunner(libs[k], seq, device=0)
                rr.run(args.c5_windows)
                c5[k].append([x["ms"] for x in rr.records[5:]])
                dev5[k].append([x["device_ms"] for x in rr.records[5:]])
                del rr
        res["c5_resident_ms_per_window"] = {k: stats(v) for k, v in c5.items()}
        res["c5_resident_solve_device_ms"] = {k: stats(v) for k, v in dev5.items()}
        res["c5_median_change"] = (res["c5_resident_ms_per_window"]["B"]["median"] /
                                   res["c5_resident_ms_per_window"]["A"]["median"] - 1.0)

    # ---- C4 (and C4x): speculation is off above 20 k observations ----
    for name, n_lm in (("c4", 10_000), ("c4x", 100_000)):
        if args.c4_solves <= 0 or (name == "c4x" and not args.c4x):
            continue
        w4 = syn.config_c4(n_landmarks=n_lm)
        e4 = {}
        for k, lib in libs.items():
            e4[k] = pkg.setup_estimator(lib, w4, device=0)
            e4[k].SaveState()
        ms = {k: [] for k in libs}
        for r in range(2 + args.c4_solves):
            for k in (("A", "B") if r % 2 == 0 else ("B", "A")):
                e4[k].RestoreState()
                flush.fill_(r & 0xFF)
                torch.cuda.synchronize()
                s = e4[k].Solve(MAX_ITERS)
                if r >= 2:
                    ms[k].append(s.device_ms)
        res[name + "_solve_device_ms"] = {k: stats([v]) for k, v in ms.items()}
        del e4

    line = json.dumps(res)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(line + "\n")
    print(line)
    c = res["c2_device_ms"]
    print(f"C2 device_ms  A median {c['A']['median']:.4f} [{c['A']['round_median_min']:.4f}, {c['A']['round_median_max']:.4f}]"
          f"  B median {c['B']['median']:.4f} [{c['B']['round_median_min']:.4f}, {c['B']['round_median_max']:.4f}]"
          f"  change {100 * res['c2_median_change']:+.2f} %")
    if "c5_resident_ms_per_window" in res:
        c = res["c5_resident_ms_per_window"]
        print(f"C5 ms/window  A median {c['A']['median']:.4f}  B median {c['B']['median']:.4f}"
              f"  change {100 * res['c5_median_change']:+.2f} %")


if __name__ == "__main__":
    main()
