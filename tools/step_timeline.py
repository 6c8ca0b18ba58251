"""Kernel timeline of one warmed-up C2 solve(15) on the engine stream, per LM step, from a torch.profiler trace.

    python tools/step_timeline.py [--lib PATH] [--out DIR] [--solves N]

The estimator is set up as bench.py sets it up (config_c2, SaveState / RestoreState, a 256 MiB buffer written between
solves to flush L2).  For each profiled solve it prints every kernel / memset of the engine stream (the stream of
gradient_norm_kernel) with its duration and the gap since the previous operation on that stream, grouped per LM step
(a step starts at each visual_kernel), the median in-solve duration of every kernel of a step on all streams, the
evaluation phase per step (first start to last end of its factor kernels), and the summed gaps of the critical chain (engine-stream operations from the
solve's first one up to the end of the last gradient_norm_kernel, which is where summary.device_ms ends for this solve:
it runs all 15 iterations, so no speculated step is left behind) as a fraction of summary.device_ms.  For each gap it names the operation on another stream that ended last before the gap closed,
when that one ended inside the gap: such a gap is a cross-stream wait, not a launch boundary.  A negative gap is overlap:
a kernel chained by programmatic dependent launch starts before its predecessor ends and waits for it in
griddepcontrol.wait, so its duration includes that wait; only positive gaps are summed.
The trace (chrome JSON) and a JSON summary go to DIR (default build/step_timeline, ignored by git).  Card name and
power limit are printed with the numbers.  Not a bench value: the profiler slows the host side.
"""
import argparse
import gzip
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
FACTOR_KERNELS = ("visual_kernel", "imu_kernel", "small_factors_kernel", "prior_add_jtj_kernel")


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


def short(name):
    n = name.replace("void ", "").replace("ctvio::", "").replace("(anonymous namespace)::", "")
    return n.split("(")[0]


def gpu_ops(trace_path):
    op = gzip.open if trace_path.endswith(".gz") else open
    with op(trace_path, "rt") as f:
        ev = json.load(f)["traceEvents"]
    ops = []
    for e in ev:
        if e.get("ph") != "X" or e.get("cat") not in ("kernel", "gpu_memset", "gpu_memcpy"):
            continue
        ops.append({"name": short(e["name"]) if e["cat"] == "kernel" else e["cat"], "ts": float(e["ts"]),
                    "dur": float(e["dur"]), "stream": int(e["args"].get("stream", -1))})
    ops.sort(key=lambda o: o["ts"])
    return ops


def analyse(ops, device_ms):
    eng = {o["stream"] for o in ops if o["name"] == "gradient_norm_kernel"}
    assert len(eng) == 1, f"gradient_norm_kernel on streams {eng}"
    eng = eng.pop()
    main = [o for o in ops if o["stream"] == eng]
    last_gn = max(i for i, o in enumerate(main) if o["name"] == "gradient_norm_kernel")
    chain = main[:last_gn + 1]
    other = [o for o in ops if o["stream"] != eng]
    steps, rows, gaps = [], [], 0.0
    for i, o in enumerate(chain):
        gap = 0.0 if i == 0 else o["ts"] - (chain[i - 1]["ts"] + chain[i - 1]["dur"])
        gaps += max(gap, 0.0)
        waited = None
        if i > 0 and gap > 0:
            prev_end = chain[i - 1]["ts"] + chain[i - 1]["dur"]
            ends = [x for x in other if prev_end < x["ts"] + x["dur"] <= o["ts"] + 0.5]
            if ends:
                w = max(ends, key=lambda x: x["ts"] + x["dur"])
                waited = f"{w['name']}@s{w['stream']}"
        if o["name"].startswith("visual_kernel"):
            steps.append([])
        row = {"name": o["name"], "dur_us": o["dur"], "gap_us": gap, "after_other_stream": waited}
        (steps[-1] if steps else rows).append(row)
    span_us = chain[-1]["ts"] + chain[-1]["dur"] - chain[0]["ts"]
    # every stream's kernels per LM step (a step's window opens when the engine-stream operation in front of its
    # visual_kernel ends: the fork onto the other streams is recorded there), and the evaluation phase: first start to
    # last end of the step's factor kernels (fork -> join)
    vis = [i for i, o in enumerate(chain) if o["name"].startswith("visual_kernel")]
    opens = [chain[i - 1]["ts"] + chain[i - 1]["dur"] if i > 0 else chain[i]["ts"] for i in vis]
    opens.append(chain[-1]["ts"] + chain[-1]["dur"])
    per_kernel, eval_us = {}, []
    for a, b in zip(opens, opens[1:]):
        ks = [o for o in ops if a <= o["ts"] < b]
        for o in ks:
            per_kernel.setdefault(o["name"], []).append(o["dur"])
        fac = [o for o in ks if o["name"].split("<")[0] in FACTOR_KERNELS]
        eval_us.append(max(o["ts"] + o["dur"] for o in fac) - min(o["ts"] for o in fac))
    by_pair = {}
    for s in steps:
        for a, b in zip(s, s[1:]):
            by_pair.setdefault(f"{a['name']} -> {b['name']}", []).append(b["gap_us"])
    return {"engine_stream": eng, "pre_steps": rows, "steps": steps, "chain_gap_us": gaps, "chain_span_us": span_us,
            "device_ms": device_ms, "gap_fraction_of_device_ms": gaps * 1e-3 / device_ms,
            "median_gap_by_boundary_us": {k: float(np.median(v)) for k, v in by_pair.items()},
            "median_dur_by_kernel_us": {k: float(np.median(v)) for k, v in per_kernel.items()},
            "eval_phase_us": eval_us, "eval_phase_median_us": float(np.median(eval_us)),
            "other_stream_ops": sorted({f"{o['name']}@s{o['stream']}" for o in other})}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="libctvio_b200.so to load (default: the in-tree build)")
    ap.add_argument("--out", default=os.path.join(ROOT, "build", "step_timeline"))
    ap.add_argument("--solves", type=int, default=3, help="profiled solves (one trace each)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--tag", default="")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    if not torch.cuda.is_available():
        raise SystemExit("step_timeline.py needs a CUDA device")
    os.makedirs(args.out, exist_ok=True)
    lib = pkg.CtvioLib(args.lib) if args.lib else pkg.load()
    w = syn.config_c2(seed=syn.SEED0 + 2)
    est = pkg.setup_estimator(lib, w, device=0)
    est.SaveState()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def one():
        est.RestoreState()
        flush.fill_(7)
        torch.cuda.synchronize()
        s = est.Solve(MAX_ITERS)
        torch.cuda.synchronize()
        return s

    for _ in range(args.warmup):
        one()
    plain = [one().device_ms for _ in range(10)]
    dev = card()
    results = []
    for k in range(args.solves):
        est.RestoreState()
        flush.fill_(7)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            s = est.Solve(MAX_ITERS)
            torch.cuda.synchronize()
        path = os.path.join(args.out, f"trace{args.tag}_{k}.json")
        prof.export_chrome_trace(path)
        r = analyse(gpu_ops(path), s.device_ms)
        r.update(iterations=s.iterations, passes=s.num_jacobian_evals, kernel_launches=s.kernel_launches, trace=path)
        results.append(r)
    summary = {"card": dev, "unprofiled_device_ms": plain, "unprofiled_device_ms_median": float(np.median(plain)),
               "solves": results}
    with open(os.path.join(args.out, f"summary{args.tag}.json"), "w") as f:
        json.dump(summary, f, indent=1)

    print(f"card: {dev['name']}, power limit {dev['power_limit_w']} W; lib {lib.path}")
    print(f"unprofiled device_ms: median {np.median(plain):.3f} (min {min(plain):.3f}, max {max(plain):.3f}) over 10 solves")
    r = results[0]
    print(f"engine stream {r['engine_stream']}; other streams: {', '.join(r['other_stream_ops'])}")
    for j, s in enumerate(r["steps"]):
        tot = sum(x["dur_us"] + max(x["gap_us"], 0) for x in s)
        print(f"-- pass {j} ({tot:.1f} us incl. gaps)")
        for x in s:
            wait = f"  [after {x['after_other_stream']}]" if x["after_other_stream"] else ""
            print(f"   {x['name']:<34s} {x['dur_us']:8.2f} us  gap {x['gap_us']:7.2f} us{wait}")
    print("median gap before each boundary (us):")
    for k, v in sorted(r["median_gap_by_boundary_us"].items(), key=lambda kv: -kv[1]):
        print(f"   {v:7.2f}  {k}")
    print("median in-solve duration per kernel over the LM steps, all streams (us):")
    for k, v in sorted(r["median_dur_by_kernel_us"].items(), key=lambda kv: -kv[1]):
        print(f"   {v:8.2f}  {k}")
    print(f"evaluation phase (first start -> last end of the step's factor kernels): median "
          f"{r['eval_phase_median_us']:.2f} us over {len(r['eval_phase_us'])} steps")
    for k, r in enumerate(results):
        print(f"solve {k}: device_ms {r['device_ms']:.3f} (profiled), {r['iterations']} iterations, {r['passes']} passes; "
              f"critical-chain gaps {r['chain_gap_us']:.1f} us = {100 * r['gap_fraction_of_device_ms']:.1f} % of device_ms "
              f"(chain span {r['chain_span_us']:.1f} us)")


if __name__ == "__main__":
    main()
