"""Host wall clock of ctvio_triangulate_window against the host composition it replaces (QueryTrajectory of every
observation time -> Triangulate with the caller's poses -> RemapLandmarks with the depths), both ending in a device
synchronise, at two sizes:
  c5    one C5 window (11 frames, ~300 landmarks) whose ~30 newest landmarks are not initialised;
  full  the largest window the resident tables hold: 16 frame slots x 1024 features, 1024 landmarks seen in all 16.
Prints the card name and power limit, the spread over the repetitions, and (separate, traced run) the kernels one
TriangulateWindow call launches, from torch.profiler.  Usage: python tools/triangulate_timing.py [--reps N] [--warmup N]"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
pkg = importlib.import_module("ctrl-vio_b200")
syn = pkg.synthetic
st = importlib.import_module("ctrl-vio_b200.streaming")
import test_resident_triangulation as trt  # noqa: E402  (the CSR / payload / full-table builders of the tests)


def device_info():
    import torch
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        phys = vis.split(",")[0] if vis else "0"
        r = subprocess.run(["nvidia-smi", f"--id={phys}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20)
        out["power_limit_w"] = float(r.stdout.strip())
    except Exception:
        pass
    return out


def c5_case(lib):
    seq = st.quantize_wire(st.config_c5_sequence(1))
    frames = np.arange(st.WIN_KF)
    w = syn.subwindow_frames(seq, frames, window_size=st.WINDOW_SIZE)
    e, clouds = trt.resident_engine(lib, seq, frames, seq.q0, seq.p0, syn.LD_TRUE)
    off, slot, idx = trt.resident_csr(seq, clouds, frames, w)
    rho = w.rho0.copy()
    rho[w.anchor_frame == w.anchor_frame.max()] = -1.0  # the landmarks of the newest anchoring frame
    t, row, xy = trt.payload_from_clouds(seq, clouds, {int(f) % trt.N_SLOTS: int(f) for f in frames}, slot, idx)
    return e, off, slot, idx, rho, t, row, xy


def full_case(lib):
    seq = st.config_c5_sequence(st.WIN_KF)
    frames, msgs, off, slot, idx, _ = trt.full_tables(seq, np.random.default_rng(5))
    e = pkg.Estimator(lib, pkg.make_config(**seq.config_kwargs()))
    e.SetKnots(seq.q_gt, seq.p_gt); e.SetLineDelay(syn.LD_TRUE)
    for f, m in zip(frames, msgs):
        e.IngestFeatureCloud(int(f), int(seq.kf_times[f]), *m)
    rho = np.full(len(off) - 1, -1.0)
    t = np.asarray(seq.kf_times[slot], np.int64)
    row = np.array([int(msgs[s][3][i]) for s, i in zip(slot, idx)], np.int64)
    xy = np.array([msgs[s][0][i, :2] for s, i in zip(slot, idx)], np.float64)
    return e, off, slot, idx, rho, t, row, xy


def host_path_inputs(off, rho, t, row, xy, ld):
    """what a caller without the device path uploads: the observations of the landmarks to initialise"""
    new = np.nonzero(~(rho > 0))[0]
    used = np.diff(off)[new]
    sub_off = np.concatenate([[0], np.cumsum(used)]).astype(np.int32)
    sel = np.concatenate([np.arange(off[l], off[l + 1]) for l in new])
    times = t[sel] + row[sel] * np.int64(int(ld * 1e9))
    pts = np.column_stack([xy[sel], np.ones(len(sel))])
    old_index = np.where(rho > 0, np.arange(len(rho)), -1).astype(np.int32)
    return new, sub_off, times, pts, old_index


def time_case(name, e, off, slot, idx, rho, t, row, xy, reps, warmup):
    import torch
    ld = e.GetLineDelay()
    new, sub_off, times, pts, old_index = host_path_inputs(off, rho, t, row, xy, ld)
    ric = trt.quat_to_R(syn.Q_CtoI)[0].reshape(9)
    tic = np.asarray(syn.P_CinI, float)
    depth0 = np.full(len(new), -1.0)
    init = np.zeros(len(rho))

    def device_path():
        return e.TriangulateWindow(off, slot, idx, 5.0)

    def host_path():
        q, p = e.QueryTrajectory(times)[:2]
        R = trt.quat_to_R(q).reshape(-1, 9)
        d = e.Triangulate(R, p, ric, tic, sub_off[:-1], sub_off, pts, depth0, window_size=len(times) + 3, init_depth=5.0)
        d[np.diff(sub_off) < 2] = 5.0
        init[new] = 1.0 / d
        e.RemapLandmarks(old_index, init)

    out = {}
    for label, fn in (("triangulate_window", device_path), ("host_composition", host_path)):
        samples = []
        for it in range(warmup + reps):
            e.SetInvDepths(rho)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            t1 = time.perf_counter()
            if it >= warmup:
                samples.append(1e6 * (t1 - t0))
        s = np.asarray(samples)
        out[label] = dict(median_us=round(float(np.median(s)), 1), p10_us=round(float(np.percentile(s, 10)), 1),
                          p90_us=round(float(np.percentile(s, 90)), 1), min_us=round(float(s.min()), 1), reps=reps)
    res = dict(case=name, n_landmarks=int(len(off) - 1), n_observations=int(off[-1]), n_new=int(len(new)),
               n_new_observations=int(len(times)), **out)
    print(json.dumps(res))
    return res


def trace_launches(e, off, slot, idx, rho):
    """kernels of one TriangulateWindow call (traced run of its own, after the timings)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    e.SetInvDepths(rho)
    e.SetKnots(*e.GetKnots())  # knot-pair table stale: the call rebuilds it first
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        e.TriangulateWindow(off, slot, idx, 5.0)
        torch.cuda.synchronize()
    kernels = [ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA and
               "emcpy" not in ev.name and "emset" not in ev.name]
    print(json.dumps(dict(traced_kernels=kernels, count=len(kernels))))
    return kernels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=30)
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    print(json.dumps(dict(device=device_info())))
    lib = pkg.load()
    cases = {"c5": c5_case(lib), "full": full_case(lib)}
    for name, c in cases.items():
        time_case(name, *c, reps=args.reps, warmup=args.warmup)
    for name, c in cases.items():
        e, off, slot, idx, rho = c[:5]
        k = trace_launches(e, off, slot, idx, rho)
        if not 1 <= len(k) <= 2:
            print(f"{name}: expected 1 or 2 kernels (knot-pair table + triangulation), traced {len(k)}")


if __name__ == "__main__":
    main()
