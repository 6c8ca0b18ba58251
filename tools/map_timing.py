"""Host wall clock of ctvio_feature_table_map (one launch, the call's own stream synchronise, the copy out of mapped
memory) against the host composition it replaces: GetInvDepths, FeatureTableLandmarks (taken before the slide, which
it refuses to follow), QueryTrajectory of the listed frame times, the extrinsic on the host and FeatureTable.map over
the host's own copy of the clouds.  The host's table bookkeeping (FeatureTable add / window / slide), which such a
caller needs as well, is not timed.  Two sizes:
  c5    ResidentRunner(device_features=True, publish_map=True) over the wire-quantized C5 sequence: both sides are timed
        at every slide; then whole runner windows with and without publish_map (the record's ms);
  full  16 frame slots x 1024 features with overlapping ids: window, positive and negative depths, the oldest slot
        slides, both sides are timed, a new cloud takes the freed slot.
Every device map is checked against the host one (ids and margin flags equal, points within 1e-12 of the scene
scale).  Prints the card name and power limit, medians and 10th-90th percentiles (us).
Usage: python tools/map_timing.py [--windows N] [--warmup N]"""
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
from keyframe_timing import spread  # noqa: E402
from triangulate_timing import device_info  # noqa: E402


def clock(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, 1e6 * (time.perf_counter() - t0)


class Timer:
    """times the device map and the host composition at the same engine state"""

    def __init__(self, e, table, frame_time):
        self.e, self.t, self.frame_time = e, table, frame_time
        self.device, self.host, self.counts, self.landmarks_us = [], [], [], 0.0

    def before_slide(self):
        _, self.landmarks_us = clock(lambda: self.e.FeatureTableLandmarks())

    def compare(self, device_map, slots, ws):
        out, dev_us = clock(lambda: device_map(slots, ws))
        e, t = self.e, self.t

        def host():
            rho = e.GetInvDepths()
            q, p, *_ = e.QueryTrajectory(np.array([self.frame_time(s) for s in slots], np.int64))
            return t.map(slots, ws, rho, *st.camera_poses(q, p))
        (xyz, ids, margin), host_us = clock(host)
        assert np.array_equal(out[1], ids) and np.array_equal(out[2], margin)
        assert np.abs(out[0] - xyz).max(initial=0.0) <= 1e-12 * max(np.abs(xyz).max(initial=0.0), 1.0)
        self.device.append(dev_us)
        self.host.append(host_us + self.landmarks_us)
        self.counts.append((len(ids), int(margin.sum())))
        return out


def c5_case(lib, n, warmup):
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    r = st.ResidentRunner(lib, seq, triangulate=True, device_features=True, publish_map=True)
    e, table, msgs = r.est, st.FeatureTable(), {}
    frame_of = lambda s: next(f for f, x in r.slot_of.items() if x == s)
    tm = Timer(e, table, lambda s: int(seq.kf_times[frame_of(s)]))
    orig = {k: getattr(e, k) for k in ("IngestFeatureCloud", "FeatureTableAdd", "FeatureTableWindow",
                                       "FeatureTableSlide", "FeatureTableMap")}

    def ingest(slot, t_ns, *m):
        orig["IngestFeatureCloud"](slot, t_ns, *m)
        msgs[slot] = m

    def add(slot):
        table.add(slot, msgs[slot])
        return orig["FeatureTableAdd"](slot)

    def window(slots, ws):
        table.window(slots, ws, e.GetInvDepths())
        return orig["FeatureTableWindow"](slots, ws)

    def slide(slot):
        tm.before_slide()
        table.slide(slot, e.GetInvDepths())
        return orig["FeatureTableSlide"](slot)
    e.IngestFeatureCloud, e.FeatureTableAdd, e.FeatureTableWindow, e.FeatureTableSlide = ingest, add, window, slide
    e.FeatureTableMap = lambda slots, ws: tm.compare(orig["FeatureTableMap"], slots, ws)
    r.run(n)
    c = np.asarray(tm.counts)
    print(json.dumps(dict(case="c5", windows=n - warmup, device_map_us=spread(tm.device[warmup:]),
                          host_composition_us=spread(tm.host[warmup:]),
                          map_points_min_median_max=[int(c[:, 0].min()), int(np.median(c[:, 0])), int(c[:, 0].max())],
                          margin_points_median=float(np.median(c[:, 1])))))
    out = {}
    for pm in (False, True):
        rr = st.ResidentRunner(lib, seq, triangulate=True, device_features=True, publish_map=pm)
        rr.run(n)
        out["publish_map" if pm else "without_map"] = spread([1e3 * x["ms"] for x in rr.records[warmup:]])
    print(json.dumps(dict(case="c5_runner_window_us", windows=n - warmup, **out)))


def full_case(lib, n, warmup, seed=11):
    rng = np.random.default_rng(seed)
    seq = st.config_c5_sequence(6)                                   # 16 keyframe times
    e = pkg.Estimator(lib, pkg.make_config(**seq.config_kwargs()))
    e.SetKnots(seq.q0, seq.p0)
    table = st.FeatureTable()
    tm = Timer(e, table, lambda s: int(seq.kf_times[s]))

    def cloud():
        ids = rng.choice(20000, 1024, replace=False).astype(np.float32)
        pts = np.ones((1024, 3), np.float32)
        pts[:, :2] = rng.uniform(-0.5, 0.5, (1024, 2))
        z = np.zeros(1024, np.float32)
        return pts, ids, z, z, z, z
    order = list(range(16))
    for s in order:
        m = cloud()
        e.IngestFeatureCloud(s, int(seq.kf_times[s]), *m)
        e.FeatureTableAdd(s)
        table.add(s, m)
    for _ in range(n):
        slots = np.array(order, np.int32)
        table.window(slots, 16, e.GetInvDepths())
        n_lm = e.FeatureTableWindow(slots, 16)
        rho = rng.uniform(-0.05, 1.0, n_lm)
        e.SetInvDepths(rho)
        tm.before_slide()
        leave = order.pop(0)
        table.slide(leave, rho)
        e.FeatureTableSlide(leave)
        tm.compare(e.FeatureTableMap, np.array(order, np.int32), 16)
        m = cloud()
        e.IngestFeatureCloud(leave, int(seq.kf_times[leave]), *m)
        e.FeatureTableAdd(leave)
        table.add(leave, m)
        order.append(leave)
    c = np.asarray(tm.counts)[warmup:]
    print(json.dumps(dict(case="full", windows=n - warmup, device_map_us=spread(tm.device[warmup:]),
                          host_composition_us=spread(tm.host[warmup:]),
                          entries_median=int(np.median([len(table.id)])), map_points_median=int(np.median(c[:, 0])),
                          margin_points_median=float(np.median(c[:, 1])))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    print(json.dumps(dict(device=device_info())))
    lib = pkg.load()
    c5_case(lib, args.windows, args.warmup)
    full_case(lib, args.windows, args.warmup)
    print(json.dumps(dict(device=device_info())))


if __name__ == "__main__":
    main()
