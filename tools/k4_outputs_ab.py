"""Output comparison of two builds of libctvio_b200.so in one process: does a change of the LM step keep its results?

    python tools/k4_outputs_ab.py A.so B.so [--repeats 3]

Both libraries are loaded as tools/pdl_ab.py loads them (RTLD_DEEPBIND: each binds to its own definitions).
Deterministic mode: C2 solve(15) (the bench window) and C3 window A solve(15) + 4-DoF re-alignment + marginalization of
keyframe 0 on each build; knots, biases, inverse depths, line delay, summary (iterations, passes, initial / final
cost) and the prior (J, r, block layout) must be bit-identical between the builds.
Structure (deterministic mode): the C2 solve, the C3 window with its re-alignment and marginalization, a C4 solve
(host-built image factors); C5 windows of the resident runner with table-built factors (device build) and with
host-derived factors; one C5 window mixing table-built and slot-named factors.  Every ctvio_debug_structure array (after
the marginalization: its block positions too), the bytes each phase moved (ctvio_transfer_stats), the kernel launches
and the window's outputs must be equal between the builds.
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


def structure(est, out, tag=""):
    """ctvio_debug_structure's arrays into out (the call itself prepares; bytes are read before it)"""
    out["transfer" + tag] = np.array(est.TransferStats(reset=True), np.float64)
    for k, v in est.DebugStructure().items():
        out["structure_" + k + tag] = np.zeros(0) if v is None else np.asarray(v, np.float64)
    est.TransferStats(reset=True)
    return out


def solved(est, s):
    out = state(est, s)
    out["launches"] = np.array([s.kernel_launches], np.float64)
    return out


def prior(pr):
    if pr is None:
        return {"prior_n": np.zeros(1)}
    return {"prior_J": pr.J, "prior_r": pr.r, "prior_x0": pr.blk_x0,
            "prior_blocks": np.concatenate([pr.blk_type, pr.blk_index, pr.blk_col]).astype(np.float64)}


def c2_structure(lib):
    est = pkg.setup_estimator(lib, syn.config_c2(seed=syn.SEED0 + 2), device=0)
    est.SetDeterministic(True)
    est.TransferStats(reset=True)
    return structure(est, solved(est, est.Solve(MAX_ITERS)))


def c3_structure(lib):
    st = importlib.import_module("ctrl-vio_b200.streaming")
    e, _, wa, nowk = st.c3_window_a(lib, device=0)
    e.SetDeterministic(True)
    e.TransferStats(reset=True)
    out = structure(e, solved(e, e.Solve(MAX_ITERS)), "_solve")
    e.GaugeRealign(nowk, syn.qrot(wa.q0[nowk][None], np.eye(3)).T.copy(), wa.p0[nowk].copy())
    out.update(prior(e.SaveMarginalizationInfo()))
    return structure(e, out, "_marg")


def c4_structure(lib):
    est = pkg.setup_estimator(lib, syn.config_c4(n_landmarks=10_000), device=0)
    est.SetDeterministic(True)
    est.TransferStats(reset=True)
    return structure(est, solved(est, est.Solve(MAX_ITERS)))


def c5_structure(lib, device_features, n=6):
    st = importlib.import_module("ctrl-vio_b200.streaming")
    seq = st.quantize_wire(st.config_c5_sequence(n + 1))
    rr = st.ResidentRunner(lib, seq, device=0, triangulate=device_features, device_features=device_features)
    rr.est.SetDeterministic(True)
    out = {}

    class Recorder:
        """the engine's library, recording the structure after every solve and marginalization (before the slide
        moves the spline under the factors)"""

        def __getattr__(self, name):
            return getattr(lib, name)

        def call(self, name, *a):
            rc = lib.call(name, *a)
            if name in ("solve", "marginalize"):
                tag = "_%d_%s" % (len(out), name)
                for k, v in rr.est.DebugStructure().items():
                    out["structure_" + k + tag] = np.zeros(0) if v is None else np.asarray(v, np.float64)
            return rc
    rr.est.lib = Recorder()
    rr.run(n)
    # every window's numeric record entries except the timings, in one row
    out["records"] = np.array([float(v) for r in rr.records for k, v in sorted(r.items())
                                if isinstance(v, (int, float)) and not k.startswith("ms") and "device_ms" not in k])
    q, p = rr.est.GetKnots()
    out.update(knots_q=q, knots_p=p, biases=rr.est.GetBiases(), inv_depths=rr.est.GetInvDepths())
    return out


def mixed_structure(lib):
    """one C5 window on the resident feature table: its factors from the table, then 500 of them again, not
    landmark-sorted, as slot-named factors"""
    st = importlib.import_module("ctrl-vio_b200.streaming")
    seq = st.config_c5_sequence(8)
    e = pkg.Estimator(lib, pkg.make_config(**seq.config_kwargs()))
    e.SetKnots(seq.q0, seq.p0); e.SetBiases(seq.bias0[:2]); e.SetLineDelay(seq.ld0)
    rng = np.random.default_rng(5)
    for s in range(16):
        ids = rng.choice(20000, 1024, replace=False).astype(np.float32)
        pts = np.ones((len(ids), 3), np.float32)
        pts[:, 0], pts[:, 1] = 1e-4 * (ids % 97), -1e-4 * (ids % 89)
        z = np.zeros(len(ids), np.float32)
        e.IngestFeatureCloud(s, int(seq.kf_times[s]), pts, ids, z, (ids % 480).astype(np.float32), z, z)
        e.FeatureTableAdd(s)
    n_lm = e.FeatureTableWindow(np.arange(16, dtype=np.int32), 16)
    e.SetInvDepths(rng.uniform(0.2, 1.0, n_lm))
    e.SetOptions(pkg.make_options(is_marg_state=True, ctrl_to_be_opt_now=0, ctrl_to_be_opt_later=2))
    e.ClearFactors()
    e.AddImageFeaturesFromTable(1)
    s = e.DebugStructure()
    d = np.empty_like(s["desc"])
    d[s["orig"]] = s["desc"]
    extra = d[rng.choice(len(d), 500, replace=False)][::-1]
    e.AddImageFeaturesFromSlots(extra[:, 0] // 1024, extra[:, 0] % 1024, extra[:, 1] // 1024, extra[:, 1] % 1024,
                                extra[:, 2], rng.integers(0, 2, len(extra)))
    e.SetDeterministic(True)
    e.TransferStats(reset=True)
    out = structure(e, solved(e, e.Solve(4)), "_solve")
    e.GaugeRealign(0, np.eye(3), np.zeros(3))
    out.update(prior(e.SaveMarginalizationInfo()))
    return structure(e, out, "_marg")


STRUCTURE_CASES = {"c2": c2_structure, "c3": c3_structure, "c4": c4_structure,
                   "c5_table": lambda lib: c5_structure(lib, True), "c5_host": lambda lib: c5_structure(lib, False),
                   "mixed": mixed_structure}


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
    for w, run in STRUCTURE_CASES.items():
        a, b = run(libs["A"]), run(libs["B"])
        res["deterministic_bitwise_equal"]["structure_" + w] = bitwise_equal(a, b)

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
