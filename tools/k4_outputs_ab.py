"""Output comparison of two builds of libctvio_b200.so in one process: does a change of the LM step keep its results?

    python tools/k4_outputs_ab.py A.so B.so [--repeats 3]

Both libraries are loaded as tools/pdl_ab.py loads them (RTLD_DEEPBIND: each binds to its own definitions).
Deterministic mode: C2 solve(15) (the bench window) and C3 window A solve(15) + 4-DoF re-alignment + marginalization of
keyframe 0 on each build; knots, biases, inverse depths, line delay, summary (iterations, passes, initial / final
cost) and the prior (J, r, block layout) must be bit-identical between the builds.
Default mode: C2 solve(15) `--repeats` times per build, alternating; the largest difference of each output between the
builds, next to the largest difference between two runs of one build (the run-to-run spread of the atomics' order).
Prints one JSON line with the card's name and power limit; writes it to --out as well (default build/k4_outputs_ab.json).
Exit status 1 if a deterministic-mode output differs or the iteration / pass counts differ.
"""
import argparse
import importlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
pkg = importlib.import_module("ctrl-vio_b200")
syn = pkg.synthetic
from pdl_ab import card, load  # noqa: E402

MAX_ITERS = 15


def state(est, s):
    q, p = est.GetKnots()
    return {"knots_q": q, "knots_p": p, "biases": est.GetBiases(), "inv_depths": est.GetInvDepths(),
            "line_delay": np.array([est.GetLineDelay()]),
            "summary": np.array([s.iterations, s.num_jacobian_evals, s.initial_cost, s.final_cost], np.float64)}


def c2_run(lib, deterministic):
    est = pkg.setup_estimator(lib, syn.config_c2(seed=syn.SEED0 + 2), device=0)
    est.SetDeterministic(deterministic)
    return state(est, est.Solve(MAX_ITERS))


def c3_run(lib):
    st = importlib.import_module("ctrl-vio_b200.streaming")
    e, _, wa, nowk = st.c3_window_a(lib, device=0)
    e.SetDeterministic(True)
    R0 = syn.qrot(wa.q0[nowk][None], np.eye(3)).T.copy()
    t0 = wa.p0[nowk].copy()
    out = state(e, e.Solve(MAX_ITERS))
    e.GaugeRealign(nowk, R0, t0)
    pr = e.SaveMarginalizationInfo()
    out.update({"prior_J": pr.J, "prior_r": pr.r, "prior_blocks": np.concatenate(
        [pr.blk_type, pr.blk_index, pr.blk_col]).astype(np.float64), "prior_x0": pr.blk_x0})
    return out


def bitwise_equal(a, b):
    return {k: bool(a[k].shape == b[k].shape and np.array_equal(a[k].view(np.int64), b[k].view(np.int64))) for k in a}


def max_diff(a, b):
    return {k: float(np.abs(a[k] - b[k]).max()) if a[k].size else 0.0 for k in a if k != "summary"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("a")
    ap.add_argument("b")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "build", "k4_outputs_ab.json"))
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("k4_outputs_ab.py needs a CUDA device")
    libs = {"A": load(os.path.abspath(args.a)), "B": load(os.path.abspath(args.b))}
    res = {"card": card(), "A": args.a, "B": args.b}

    det = {k: {"c2": c2_run(lib, True), "c3": c3_run(lib)} for k, lib in libs.items()}
    res["deterministic_bitwise_equal"] = {w: bitwise_equal(det["A"][w], det["B"][w]) for w in ("c2", "c3")}

    runs = {k: [] for k in libs}
    for r in range(args.repeats):
        for k in (("A", "B") if r % 2 == 0 else ("B", "A")):
            runs[k].append(c2_run(libs[k], False))
    counts = {k: sorted({(int(x["summary"][0]), int(x["summary"][1])) for x in v}) for k, v in runs.items()}
    between = [max_diff(a, b) for a in runs["A"] for b in runs["B"]]
    within = [max_diff(v[i], v[j]) for v in runs.values() for i in range(len(v)) for j in range(i + 1, len(v))]
    keys = between[0].keys()
    res["default_mode"] = {
        "iterations_passes": counts,
        "max_diff_between_builds": {k: max(d[k] for d in between) for k in keys},
        "max_diff_within_a_build": {k: max((d[k] for d in within), default=0.0) for k in keys},
        "final_cost": {k: [float(x["summary"][3]) for x in v] for k, v in runs.items()},
    }
    ok = all(all(v.values()) for v in res["deterministic_bitwise_equal"].values()) and counts["A"] == counts["B"]
    res["ok"] = ok
    line = json.dumps(res)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(line + "\n")
    print(line)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
