"""debug: phase clocks of CTA 0 of visual_kernel<true> and imu_kernel<true> (needs tools/build_timing.sh).

    python tools/vis_timing.py [TIMING_LIB]

The stamps are those of the last launch of each kernel in a solve(2) (thread 0 of CTA 0), in SM cycles.
"""
import ctypes as C, importlib, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("ctrl-vio_b200"); syn = pkg.synthetic
path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(pkg.LIB_PATH), "libctvio_b200_timing.so")
LIB = pkg.CtvioLib(os.path.abspath(path), "ctvio_")
for name in ("c2", "c4"):
    w = syn.config_c2() if name == "c2" else syn.config_c4()
    est = pkg.setup_estimator(LIB, w)
    est.Solve(2)
    ck = (C.c_longlong * 8)()
    LIB.lib.ctvio_debug_vis_clk(ck)
    d = np.diff(np.array(ck[:6], dtype=np.int64))
    print(name, "K1 CTA 0 (last round), cycles: staging %d | evaluation (thread 0) %d | barrier wait %d | syrk %d | cost+flush %d" % tuple(d))
    LIB.lib.ctvio_debug_imu_clk(ck)
    d = np.diff(np.array(ck[:6], dtype=np.int64))
    print(name, "K2 CTA 0, cycles: evaluation (thread 0) %d | barrier wait %d | syrk %d | shared-memory reduction %d | flush %d" % tuple(d))
