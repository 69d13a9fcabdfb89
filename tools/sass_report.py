#!/usr/bin/env python3
"""profiles/<tag>_sass_tma.txt: what the built libkvgpu.so contains, per kernel — the SASS mnemonics that prove the
sm_90a features the design relies on (UBLKCP = TMA bulk copy, SYNCS = mbarrier, REDUX = warp reduction,
MATCH = match.any, REDG / ATOMG = fire-and-forget / returning global atomics, ACQBULK/griddepcontrol = programmatic
dependent launch), with registers and shared memory.   python tools/sass_report.py <tag>"""
import collections, os, re, subprocess, sys
tag = sys.argv[1] if len(sys.argv) > 1 else "h100"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = os.path.join(ROOT, "kubevirt-gpu-device-plugin_b200", "libkvgpu.so")
sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
res = subprocess.run(["cuobjdump", "-res-usage", lib], capture_output=True, text=True).stdout
arch = sorted(set(re.findall(r"arch = (sm_\w+)", sass)))
usage = {}
for m in re.finditer(r"Function (\S+):\n\s+REG:(\d+) STACK:(\d+) SHARED:(\d+)", res):
    usage[m.group(1)] = (int(m.group(2)), int(m.group(3)), int(m.group(4)))
want = ["UBLKCP", "SYNCS", "REDUX", "MATCH", "REDG", "ATOMG", "ATOMS", "MEMBAR", "ACQBULK", "CCTL", "LDS", "STS", "LDG", "STG"]
rows, cur, cnt, n = [], None, None, 0
def flush():
    if cur:
        rows.append((cur, n, dict(cnt)))
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        flush()
        cur, cnt, n = m.group(1), collections.Counter(), 0
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_]+)", line)
    if m and cur:
        n += 1
        op = m.group(1)
        for w in want:
            if op == w or op.startswith(w + "."):
                cnt[w] += 1
flush()
def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return dict(zip(names, out))
dm = demangle([r[0] for r in rows])
os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
out = os.path.join(ROOT, "profiles", "%s_sass_tma.txt" % tag)
with open(out, "w") as f:
    f.write("# cuobjdump -sass / -res-usage of kubevirt-gpu-device-plugin_b200/libkvgpu.so  (arch: %s)\n" % ", ".join(arch))
    f.write("# UBLKCP = cp.async.bulk (TMA 1-D bulk copy), SYNCS = mbarrier ops, REDUX = redux.sync, MATCH = match.any\n")
    f.write("%-78s %6s %4s %6s | %s\n" % ("kernel", "instr", "regs", "smem", " ".join("%-7s" % w for w in want)))
    for name, n, c in sorted(rows, key=lambda r: dm[r[0]]):
        short = re.sub(r"\(.*", "", dm[name]).replace("kvg::", "")
        short = re.sub(r"^void ", "", short)
        reg, stack, sh = usage.get(name, (0, 0, 0))
        f.write("%-78s %6d %4d %6d | %s\n" % (short[:78], n, reg, sh, " ".join("%-7d" % c.get(w, 0) for w in want)))
    tma = [(dm[r[0]], r[2].get("UBLKCP", 0)) for r in rows if r[2].get("UBLKCP", 0)]
    f.write("\n# kernels with TMA bulk copies: %d (%d UBLKCP sites)\n" % (len(tma), sum(t[1] for t in tma)))
    f.write("# every kernel starts with griddepcontrol.launch_dependents + griddepcontrol.wait (pdl_enter): %d of %d kernels contain ACQBULK / the PDL pair\n"
            % (sum(1 for r in rows if r[2].get("ACQBULK", 0)), len(rows)))
print(open(out).read()[:6000])
