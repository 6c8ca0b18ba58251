import importlib, os, sys, numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("ctrl-vio_b200"); st = importlib.import_module("ctrl-vio_b200.streaming")
lib = pkg.load()
seq = st.quantize_wire(st.config_c5_sequence(4))
a = st.StreamingRunner(lib, seq); b = st.ResidentRunner(lib, seq)
for k in range(3):
    ra = a.step(); rb = b.step()
    print(k, "classic init_it", ra["init_iterations"], "cost %.6f -> %.6f it %d" % (ra["initial_cost"], ra["final_cost"], ra["iterations"]), "| resident init_it", rb["init_iterations"], "cost %.6f -> %.6f it %d" % (rb["initial_cost"], rb["final_cost"], rb["iterations"]), "n_imu", ra["n_imu"], rb["n_imu"], "prior", ra["prior_dim"], rb["prior_dim"])
    print("   dp", np.abs(a.p[:a.ncp]-b.p[:b.ncp]).max(), "ld", a.ld, b.ld)
