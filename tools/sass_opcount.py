"""Static SASS opcode counts per (noinline) device function of one kernel: python sass_opcount.py <libualm.so> <kernel> [ops...]"""
import collections, os, re, subprocess, sys, tempfile
so, kname = sys.argv[1:3]
ops = sys.argv[3:] or ["LDL", "STL", "LDG", "LD", "ST", "STG", "LDS", "STS", "DFMA", "DMUL", "DADD", "CALL"]
d = tempfile.mkdtemp(); subprocess.run(["cuobjdump", "-xelf", "all", os.path.abspath(so)], cwd=d, capture_output=True)
for cub in sorted(os.listdir(d)):   # the cubin that holds the kernel (the library carries one per translation unit)
    lines = subprocess.run(["nvdisasm", "-c", os.path.join(d, cub)], capture_output=True, text=True).stdout.split("\n")
    start = [i for i, l in enumerate(lines) if l.startswith(".text.") and kname in l]
    if start: start = start[0]; break
cur, agg = "kernel body", collections.defaultdict(collections.Counter)
for l in lines[start + 1:]:
    if l.startswith(".text.") or l.lstrip().startswith(".section"): break
    if l.startswith("$") and l.endswith(":"): cur = l[:-1].split("$")[-1]
    m = re.match(r"^\s+/\*[0-9a-f]{4,6}\*/\s+(@!?U?P\d+\s+)?([A-Z0-9_]+)", l)
    if m: agg[cur][m.group(2)] += 1; agg[cur]["_n"] += 1
for f, a in sorted(agg.items(), key=lambda kv: -kv[1]["_n"]):
    nm = subprocess.run(["c++filt", f], capture_output=True, text=True).stdout.strip().split("(")[0]
    print("%-48s %6d  " % (nm[:48], a["_n"]) + " ".join("%s=%d" % (o, a[o]) for o in ops if a[o]))
