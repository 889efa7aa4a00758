"""SASS opcode histogram of every kernel in the built objects (runs on the CPU box: cuobjdump only).
usage: python tools/sass_hist.py > sass_histograms.md
Evidence that the hot kernels are Hopper-native: HGMMA (wgmma), UTMALDG (TMA tensor loads), UBLKCP (TMA bulk copy), HMMA (mma.sync),
LDGSTS (cp.async), IDP.4A (dp4a) and no F2I.U8.F16."""
import collections, glob, os, re, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEY = ["HGMMA", "UTMALDG", "UBLKCP", "LDGSTS", "IDP", "MUFU", "F2FP", "HMUL2", "HMMA", "SYNCS", "FENCE", "CCTL", "MEMBAR", "F2I"]
print("# SASS opcode histograms of the shipped kernels (cuobjdump -sass ggllm.cpp_b200/csrc/*.o)\n")
print("Per kernel: total instructions, then the counts of the opcodes that identify the hardware path.\n")
for obj in sorted(glob.glob(os.path.join(ROOT, "ggllm.cpp_b200", "csrc", "*.o"))):
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
    kernels, cur = collections.OrderedDict(), None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = m.group(1); kernels[cur] = collections.Counter(); continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+(?:\.[A-Z0-9_]+)*)", line)
        if m and cur:
            kernels[cur][m.group(1)] += 1
    if not kernels:
        continue
    print("## %s\n" % os.path.basename(obj))
    print("| kernel | instructions | " + " | ".join(KEY) + " |")
    print("|---|---|" + "---|" * len(KEY))
    for name, c in kernels.items():
        dem = subprocess.run(["cu++filt", name], capture_output=True, text=True).stdout.strip() or name
        dem = re.sub(r"\(.*", "", dem).replace("(anonymous namespace)::", "").replace("<unnamed>::", "")[:70]
        tot = sum(c.values())
        cols = [sum(v for k, v in c.items() if k.split(".")[0] == key or k.startswith(key + ".")) for key in KEY]
        if tot >= 64:
            print("| `%s` | %d | %s |" % (dem, tot, " | ".join(str(v) if v else "" for v in cols)))
    print()
