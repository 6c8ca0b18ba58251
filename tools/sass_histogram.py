"""Per-kernel SASS opcode histogram of libctvio_b200.so (cuobjdump -sass): the mnemonics that prove which hardware paths the
kernels use (DMMA = fp64 tensor cores via mma.sync.m8n8k4, UBLKCP / SYNCS = TMA bulk copy + mbarrier, RED/ATOM = atomics,
UCGABAR_* = thread-block-cluster barrier, ST = generic stores (the distributed-shared-memory stores of K5 among them),
ACQBULK / PREEXIT = griddepcontrol.wait / .launch_dependents of the kernels chained by programmatic dependent launch)."""
import collections, os, re, subprocess, sys
so = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "ctrl-vio_b200", "csrc", "libctvio_b200.so")
out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
kern = None
hist = collections.OrderedDict()
arch = set()
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        kern = re.sub(r"\(.*", "", name).replace("ctvio::", "").replace("(anonymous namespace)::", "")
        hist[kern] = collections.Counter()
        continue
    m = re.search(r"arch = (sm_\w+)", line)
    if m:
        arch.add(m.group(1))
    m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and kern:
        op = m.group(1)
        hist[kern][op.split(".")[0]] += 1
        if op.startswith("DMMA") or op.startswith("UBLKCP") or op.startswith("SYNCS") or op.startswith("RED") or op.startswith("ATOM"):
            hist[kern][op] += 0
keys = ["DMMA", "DFMA", "DMUL", "DADD", "MUFU", "UBLKCP", "SYNCS", "RED", "REDG", "ATOM", "ATOMG", "ATOMS", "BAR", "WARPSYNC", "LDS", "STS", "LDG", "STG", "SHFL", "UCGABAR_ARV", "UCGABAR_WAIT", "ST", "ACQBULK", "PREEXIT"]
print("architectures:", sorted(arch))
print("%-52s" % "kernel" + "".join("%8s" % k for k in keys) + "   total")
for k, h in hist.items():
    tot = sum(v for kk, v in h.items() if "." not in kk)
    print("%-52s" % k[:52] + "".join("%8d" % h.get(x, 0) for x in keys) + "%8d" % tot)
