"""Instruction-mnemonic counts per kernel of libhs_b200.so (cuobjdump -sass): the evidence for which memory paths a
kernel uses -- STG.E.128 (the halves of the 32-byte sector stores), LDGSTS (cp.async), UBLKCP (TMA bulk copy), SYNCS (mbarrier),
SHFL (warp shuffles), REDG/ATOMG, MUFU, DFMA ...      python tools/sass_counts.py > profiles/rNN_sass_counts.txt"""
import collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "happy-simulator_b200", "libhs_b200.so")
out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
cur, cnt = None, collections.defaultdict(collections.Counter)
for line in out.splitlines():
    m = re.match(r"\s+Function : (\S+)", line)
    if m:
        cur = m.group(1); continue
    m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and cur:
        op = m.group(1)
        base = op.split(".")[0]
        cnt[cur][base] += 1
        if base in ("CCTL", "STG", "LDG", "LDGSTS", "UBLKCP", "STS", "LDS", "SYNCS", "REDG", "ATOMG", "SHFL", "MUFU", "UTMALDG", "UTMASTG"):
            cnt[cur][op] += 1
KEYS = ["STG.E.NA.EFL2.256", "STG.E.ENL2.256", "STG.E.128", "STG.E.64", "STG.E", "LDG.E.128", "LDG.E.64", "LDG.E", "LDGSTS.E.128", "LDGSTS",
        "UBLKCP", "CCTL.E.PF1", "SYNCS", "SHFL", "REDG", "ATOMG", "STS.128", "LDS.128", "DFMA", "DMUL", "DADD", "MUFU", "IMAD", "BRA", "BSSY"]
print(f"# {os.path.relpath(lib, ROOT)}: SASS mnemonic counts per kernel (cuobjdump -sass, sm_90a)")
for fn in sorted(cnt):
    if "hs_" not in fn:
        continue
    c = cnt[fn]
    name = subprocess.run(["c++filt", fn], capture_output=True, text=True).stdout.strip().split("(")[0]
    tot = sum(v for k, v in c.items() if "." not in k)
    print(f"{name:60s} total {tot:6d}  " + "  ".join(f"{k}:{c[k]}" for k in KEYS if c.get(k)))
