"""Per-kernel SASS opcode counts of the built library (cuobjdump -sass): the mnemonics that prove which hardware paths a
kernel uses (HGMMA = wgmma, UTMALDG/UTMASTG = TMA tensor copies, UBLKCP = 1-D TMA bulk copy, SYNCS = mbarrier,
LDGSTS = cp.async).  Usage: python tools/sass_opcodes.py > sass_opcodes.md"""
import collections, os, re, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = os.path.join(ROOT, "sopro_b200", "lib", "libsopro_b200.so")
out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
demangle = lambda n: subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip()
WATCH = ["HGMMA", "UTMALDG", "UTMASTG", "UBLKCP", "SYNCS", "FFMA", "LDGSTS", "LDS", "STS",
         "SHFL", "HMMA", "BAR", "ATOMS", "RED", "MUFU"]
cur, counts, size = None, collections.OrderedDict(), {}
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1)
        counts[cur] = collections.Counter()
        size[cur] = 0
        continue
    m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)", line)
    if m and cur:
        counts[cur][m.group(1).split(".")[0]] += 1
        size[cur] += 1
print("# SASS opcode counts per kernel (sm_90a, `cuobjdump -sass sopro_b200/lib/libsopro_b200.so`)\n")
print("| kernel | instr | " + " | ".join(WATCH) + " |")
print("|---|---|" + "---|" * len(WATCH))
for k, c in counts.items():
    name = demangle(k)
    name = re.sub(r"\(.*$", "", name).replace("__nv_bfloat16", "bf16")
    print(f"| `{name}` | {size[k]} | " + " | ".join(str(c.get(w, 0)) for w in WATCH) + " |")
