"""Host wall clock per C5 window of the covariance publications: CycleRunner() against
CycleRunner(covariances=("pose", "odometry", "map")) (Sigma formed once per image, inside ctvio_process_image) against
ResidentRunner with its three publications (Sigma formed once per covariance call, three times per image), all with
triangulate, device_features and publish_map, default mode.

60 windows per run, the first 5 skipped, three runs of each alternating in one process; prints the medians with the
10th-90th percentiles and the extremes, host waits on the device per window (ctvio_sync_stats), ResidentRunner's own
time in its three covariance calls, and the card's name and power limit read in the same run, as one JSON line.
Needs an H100."""
import importlib
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("ctrl-vio_b200")
st = importlib.import_module("ctrl-vio_b200.streaming")

N_WIN, SKIP, RUNS = 60, 5, 3
BASE = dict(triangulate=True, device_features=True, publish_map=True)
KINDS = ("cycle", "cycle_cov", "resident_cov")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def make(kind, lib, seq):
    if kind == "cycle":
        return st.CycleRunner(lib, seq, **BASE)
    if kind == "cycle_cov":
        return st.CycleRunner(lib, seq, **BASE, covariances=("pose", "odometry", "map"))
    return st.ResidentRunner(lib, seq, **BASE, publish_covariance=True, publish_odometry_covariance=True,
                             publish_map_covariance=True)


def run(kind, lib, seq, n_win=N_WIN):
    r = make(kind, lib, seq)
    ms, waits, cov_ms = [], [], []
    for _ in range(n_win):
        r.est.SyncStats(reset=True)
        rec = r.step()
        waits.append(r.est.SyncStats(reset=True))
        ms.append(rec["ms"])
        cov_ms.append(sum(rec.get(k, 0.0) for k in ("ms_pose_cov", "ms_rel_cov", "ms_point_cov")))
    r.est.close()
    return ms[SKIP:], waits[SKIP:], cov_ms[SKIP:]


def main():
    lib = pkg.load()
    seq = st.quantize_wire(st.config_c5_sequence(N_WIN + 1))
    warm = st.quantize_wire(st.config_c5_sequence(8))
    for kind in KINDS:   # warm-up: module load, allocations
        run(kind, lib, warm, n_win=8)
    res = {k: ([], [], []) for k in KINDS}
    for _ in range(RUNS):
        for kind in KINDS:
            for acc, v in zip(res[kind], run(kind, lib, seq)):
                acc.extend(v)
    out = {"card": card(), "windows_per_run": N_WIN, "skipped": SKIP, "runs": RUNS}
    for kind, (ms, wt, cov) in res.items():
        a = np.asarray(ms)
        out[kind] = {"ms_median": float(np.median(a)), "ms_p10": float(np.percentile(a, 10)),
                     "ms_p90": float(np.percentile(a, 90)), "ms_min": float(a.min()), "ms_max": float(a.max()),
                     "host_waits_per_window_median": float(np.median(wt)), "host_waits_per_window_max": int(np.max(wt))}
        if kind == "resident_cov":
            out[kind]["ms_in_covariance_calls_median"] = float(np.median(cov))
    out["added_ms_per_image_cycle_cov_minus_cycle"] = out["cycle_cov"]["ms_median"] - out["cycle"]["ms_median"]
    out["saved_ms_per_image_resident_cov_minus_cycle_cov"] = (out["resident_cov"]["ms_median"] -
                                                              out["cycle_cov"]["ms_median"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
