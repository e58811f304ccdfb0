"""Per-kernel SASS evidence (runs here, no GPU): counts of the mnemonics that prove the Hopper / NVLink paths.

    python tools/sass_summary.py > profiles/sass_summary.txt
"""
import collections
import re
import subprocess
import sys

SO = sys.argv[1] if len(sys.argv) > 1 else "pipegoose_b200/_C.so"
KEEP = ("HGMMA", "UTMALDG", "UTMASTG", "UBLKCP", "SYNCS", "LDGMC", "STGMC", "REDGMC",
        "REDG", "ATOMG", "MUFU", "LDG", "STG", "HMMA", "USETMAXREG", "ACQBULK", "PREEXIT", "CCTL")
sass = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True).stdout
demangle = {}
names = sorted(set(re.findall(r"Function : (\S+)", sass)))
if names:
    out = subprocess.run(["c++filt"] + names, capture_output=True, text=True).stdout.splitlines()
    demangle = dict(zip(names, out))
cur, counts = None, collections.OrderedDict()
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = demangle.get(m.group(1), m.group(1))
        cur = re.sub(r"\(.*", "", cur).replace("void ", "")
        counts.setdefault(cur, collections.Counter())
        continue
    m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)((?:\.[A-Z0-9_x]+)*)", line)
    if m and cur is not None:
        op, mods = m.group(1), m.group(2)
        for k in KEEP:
            if op == k or op.startswith(k):
                key = k
                if k in ("STG", "LDG") and ".MC" in mods:   # multimem.st shows as a multicast-qualified store
                    key = k + ".MC"
                counts[cur][key] += 1
                break
print("# SASS evidence per kernel (cuobjdump -sass pipegoose_b200/_C.so; sm_90a) — tools/sass_summary.py")
print("# HGMMA = wgmma.mma_async, UTMALDG/UTMASTG = TMA tensor load/store,")
print("# UBLKCP = cp.async.bulk, SYNCS = mbarrier ops, LDGMC = multimem.ld_reduce (NVLS),")
print("# (multimem.st compiles to STG.E.128.STRONG.SYS on the multicast address: the aperture, not the opcode, selects NVLS),")
print("# REDG = red.global (peer or local), USETMAXREG = setmaxnreg, ACQBULK / PREEXIT = griddepcontrol (PDL)")
print()
merged = collections.OrderedDict()
for k, c in counts.items():
    base = re.sub(r"<.*", "", k)
    merged.setdefault(base, collections.Counter()).update(c)
for k in sorted(merged):
    c = merged[k]
    if not c:
        continue
    print(k)
    print("    " + ", ".join(f"{n}={v}" for n, v in sorted(c.items())))
