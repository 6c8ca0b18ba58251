"""Blob size and host wall clock of ctvio_odometry_checkpoint and ctvio_odometry_restore per C5 window.

One CycleRunner (triangulate, device_features, publish_map, default mode) over 60 windows, the first 5 skipped: after
every image the run is checkpointed (Estimator.Checkpoint: the size query and the checkpoint) and the blob restored on
a second engine of the same configuration (Estimator.Restore).  Each call ends with a stream synchronisation, so the
host clock around it covers its device work.  Prints the blob size and both times (median, 10th-90th percentiles,
extremes) and the card's name and power limit read in the same run, as one JSON line.  Needs an H100."""
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("ctrl-vio_b200")
st = importlib.import_module("ctrl-vio_b200.streaming")

N_WIN, SKIP = 60, 5


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def stats(v):
    a = np.asarray(v, float)
    return {"median": float(np.median(a)), "p10": float(np.percentile(a, 10)), "p90": float(np.percentile(a, 90)),
            "min": float(a.min()), "max": float(a.max())}


def main():
    lib = pkg.load()
    seq = st.quantize_wire(st.config_c5_sequence(N_WIN + 1))
    r = st.CycleRunner(lib, seq, publish_map=True)
    other = pkg.Estimator(lib, pkg.make_config(device=0, **seq.config_kwargs()))
    size, ck_ms, rs_ms = [], [], []
    for w in range(N_WIN):
        r.step()
        t0 = time.perf_counter()
        blob = r.est.Checkpoint()
        t1 = time.perf_counter()
        other.Restore(blob)
        t2 = time.perf_counter()
        if w >= SKIP:
            size.append(len(blob)); ck_ms.append(1e3 * (t1 - t0)); rs_ms.append(1e3 * (t2 - t1))
    out = {"card": card(), "windows": N_WIN, "skipped": SKIP, "blob_bytes": stats(size), "checkpoint_ms": stats(ck_ms),
           "restore_ms": stats(rs_ms)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
