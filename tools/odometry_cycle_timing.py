"""Host wall clock per C5 window of CycleRunner (one ctvio_process_image per image) against ResidentRunner (the same
cycle through the separate entry points), same options (triangulate, device_features, publish_map), default mode.

60 windows per run, the first 5 skipped, three runs of each alternating; prints the medians with the 10th-90th
percentiles, the library's count of host waits on the device per window (ctvio_sync_stats) and the card's name and
power limit, as one JSON line.  Needs an H100."""
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


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def run(kind, lib, seq, n_win=N_WIN):
    base = dict(triangulate=True, device_features=True, publish_map=True)
    r = (st.CycleRunner if kind == "cycle" else st.ResidentRunner)(lib, seq, **base)
    ms, waits = [], []
    for w in range(n_win):
        r.est.SyncStats(reset=True)
        rec = r.step()
        waits.append(r.est.SyncStats(reset=True))
        ms.append(rec["ms"])
    r.est.close()
    return ms[SKIP:], waits[SKIP:]


def main():
    lib = pkg.load()
    seq = st.quantize_wire(st.config_c5_sequence(N_WIN + 1))
    res = {"cycle": ([], []), "resident": ([], [])}
    run("cycle", lib, st.quantize_wire(st.config_c5_sequence(8)), n_win=8)   # warm-up: module load, allocations
    for _ in range(RUNS):
        for kind in ("resident", "cycle"):
            ms, wt = run(kind, lib, seq)
            res[kind][0].extend(ms); res[kind][1].extend(wt)
    out = {"card": card(), "windows_per_run": N_WIN, "skipped": SKIP, "runs": RUNS}
    for kind, (ms, wt) in res.items():
        a = np.asarray(ms)
        out[kind] = {"ms_median": float(np.median(a)), "ms_p10": float(np.percentile(a, 10)),
                     "ms_p90": float(np.percentile(a, 90)), "host_waits_per_window_median": float(np.median(wt)),
                     "host_waits_per_window_max": int(np.max(wt))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
