"""Host wall clock of ctvio_check_keyframe (launch, result read-back and the call's own stream synchronise) at two sizes:
  c5    one C5 window: 11 frame slots of ~300 features each (the clouds of config_c5_sequence);
  full  the largest window the resident tables hold: 16 frame slots x 1024 features, every id seen in every slot.
Also the host restatement keyframe_decision on the same clouds, for scale.  Prints the card name and power limit, the
median and 10th-90th percentile over the repetitions and (separate, traced run) the kernels one call launches, from
torch.profiler.  Usage: python tools/keyframe_timing.py [--reps N] [--warmup N]"""
import argparse
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
from triangulate_timing import device_info  # noqa: E402

MIN_PARALLAX = 10.0 / 740.0


def c5_case(lib):
    seq = st.quantize_wire(st.config_c5_sequence(1))
    clouds = st.FrameClouds(seq)
    frames = list(range(st.WIN_KF))
    msgs = [clouds.message(f) for f in frames]
    e = pkg.Estimator(lib, pkg.make_config(**seq.config_kwargs()))
    for f, m in zip(frames, msgs):
        e.IngestFeatureCloud(f, int(seq.kf_times[f]), *m)
    return e, np.arange(len(frames), dtype=np.int32), msgs


def full_case(lib):
    seq = st.config_c5_sequence(1)
    rng = np.random.default_rng(11)
    n_slots, n = 16, 1024
    msgs = []
    for s in range(n_slots):
        ids = rng.permutation(n).astype(np.float32)           # every id in every slot, in a different order
        pts = np.ones((n, 3), np.float32)
        pts[:, :2] = rng.normal(scale=0.3, size=(n, 2))
        z = np.zeros(n, np.float32)
        msgs.append((pts, ids, z, z, z, z))
    e = pkg.Estimator(lib, pkg.make_config(**seq.config_kwargs()))
    for s, m in enumerate(msgs):
        e.IngestFeatureCloud(s, 0, *m)
    return e, np.arange(n_slots, dtype=np.int32), msgs


def spread(samples):
    s = np.asarray(samples)
    return dict(median_us=round(float(np.median(s)), 1), p10_us=round(float(np.percentile(s, 10)), 1),
                p90_us=round(float(np.percentile(s, 90)), 1), min_us=round(float(s.min()), 1), reps=len(s))


def time_case(name, e, slots, msgs, reps, warmup):
    import torch
    out = {}
    for label, fn in (("check_keyframe", lambda: e.CheckKeyframe(slots, MIN_PARALLAX)),
                      ("host_keyframe_decision", lambda: st.keyframe_decision(msgs, MIN_PARALLAX))):
        samples = []
        torch.cuda.synchronize()
        for it in range(warmup + reps):
            t0 = time.perf_counter()
            fn()
            t1 = time.perf_counter()
            if it >= warmup:
                samples.append(1e6 * (t1 - t0))
        out[label] = spread(samples)
    dev, host = e.CheckKeyframe(slots, MIN_PARALLAX), st.keyframe_decision(msgs, MIN_PARALLAX)
    res = dict(case=name, n_slots=int(len(slots)), n_features=int(sum(len(m[1]) for m in msgs)),
               device_result=list(dev), host_result=list(host), **out)
    print(json.dumps(res))
    return res


def trace_launches(e, slots):
    """kernels of one CheckKeyframe call (traced run of its own, after the timings)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        e.CheckKeyframe(slots, MIN_PARALLAX)
        torch.cuda.synchronize()
    ev = [x for x in prof.events() if x.device_type == torch.autograd.DeviceType.CUDA]
    kernels = [x.name for x in ev if "emcpy" not in x.name and "emset" not in x.name]
    copies = [x.name for x in ev if "emcpy" in x.name or "emset" in x.name]
    print(json.dumps(dict(traced_kernels=kernels, count=len(kernels), copies=copies)))
    return kernels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=50)
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    print(json.dumps(dict(device=device_info())))
    lib = pkg.load()
    cases = {"c5": c5_case(lib), "full": full_case(lib)}
    for name, (e, slots, msgs) in cases.items():
        time_case(name, e, slots, msgs, reps=args.reps, warmup=args.warmup)
    for name, (e, slots, _) in cases.items():
        k = trace_launches(e, slots)
        if len(k) != 1:
            print(f"{name}: expected 1 kernel, traced {len(k)}")


if __name__ == "__main__":
    main()
