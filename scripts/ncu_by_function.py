"""Per-function breakdown of an ncu report of the throughput kernel: executed warp instructions and stall samples per
source function of cuipm_fast_core.h.  ncu's source page exports SASS rows only for code in headers, so the rows are
joined with nvdisasm's line table of the same cubin (extracted from libcuipm.so) by instruction index.
usage: python scripts/ncu_by_function.py <report.ncu-rep> <kernel-substring e.g. Li21ELi3E> [--lines N]"""
import bisect, collections, csv, os, re, subprocess, sys, tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
rep, ksub = sys.argv[1], sys.argv[2]
nlines = int(sys.argv[sys.argv.index("--lines") + 1]) if "--lines" in sys.argv else 0
# --cubin <file> --core <cuipm_fast_core.h of that build>: the binary / source the report was taken with (default: the tree's)
if "--cubin" in sys.argv:
    cubin = sys.argv[sys.argv.index("--cubin") + 1]
else:
    tmp = tempfile.mkdtemp()
    subprocess.run(["cuobjdump", "-xelf", "all", os.path.join(ROOT, "acados_b200", "csrc", "libcuipm.so")], cwd=tmp, stdout=subprocess.DEVNULL)
    cubin = os.path.join(tmp, "cuipm_fast.sm_90a.cubin")
dis = subprocess.run(["nvdisasm", "--print-line-info", cubin], stdout=subprocess.PIPE, text=True).stdout
core = sys.argv[sys.argv.index("--core") + 1] if "--core" in sys.argv else os.path.join(ROOT, "acados_b200", "csrc", "cuipm_fast_core.h")
src = open(core).read().split("\n")
marks = []
for i, l in enumerate(src, 1):
    m = re.search(r"FK_DEV\s+[\w:<>&\s\*]*?\b(\w+)\s*\(", l)
    if m and "define" not in l:
        marks.append((i, m.group(1)))
starts = [m[0] for m in marks]
# instruction index -> (file, line) for the kernel
loc, kern, cf, cl = [], None, None, None
for l in dis.split("\n"):
    m = re.match(r'\s*//## File "(.*)", line (\d+)', l)
    if m:
        cf, cl = m.group(1), int(m.group(2)); continue
    m = re.match(r"\.text\.(\S+):", l)
    if m:
        kern = m.group(1); continue
    if re.match(r"\s+/\*[0-9a-f]{4,}\*/", l) and kern and ksub in kern:
        loc.append((cf, cl, l.strip()))
csvtxt = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "sass"], stdout=subprocess.PIPE, text=True).stdout
rows = list(csv.reader(csvtxt.split("\n")))
hdr = next(r for r in rows if r and r[0] == "Address")
body = [r for r in rows[rows.index(hdr) + 1:] if len(r) == len(hdr)]
ci = {h: i for i, h in enumerate(hdr)}
assert len(body) == len(loc), (len(body), len(loc))
ex, st, byline, stline = collections.Counter(), collections.Counter(), collections.Counter(), collections.Counter()
reasons = ["stall_wait", "stall_short_sb", "stall_long_sb", "stall_no_inst", "stall_branch_resolving", "stall_selected", "stall_math", "stall_mio", "stall_dispatch"]
fr = collections.defaultdict(collections.Counter)      # function -> reason -> samples
opst = collections.defaultdict(collections.Counter)    # reason -> opcode of the stalled instruction -> samples
wf, wfx = collections.Counter(), collections.Counter()  # shared-memory wavefronts / excessive ones per function
opmix = collections.Counter()
for r, (f, ln, txt) in zip(body, loc):
    e, s = int(r[ci["Instructions Executed"]]), int(r[ci["Warp Stall Sampling (All Samples)"]])
    if f and f.endswith("cuipm_fast_core.h"):
        j = bisect.bisect_right(starts, ln) - 1
        fn = marks[j][1] if j >= 0 else "?"
        byline[ln] += e; stline[ln] += s
    else:
        fn = "other:" + os.path.basename(str(f))
    ex[fn] += e; st[fn] += s
    op = re.sub(r"^(@!?U?P\d+\s+)?", "", r[ci["Source"]].strip()).split()[0].split(".")[0]
    opmix[op] += e
    for rs in reasons:
        c = int(r[ci[rs]] or 0)
        fr[fn][rs] += c
        opst[rs][op] += c
    wf[fn] += int(r[ci["L1 Wavefronts Shared"]] or 0); wfx[fn] += int(r[ci["L1 Wavefronts Shared Excessive"]] or 0)
te, ts = sum(ex.values()), sum(st.values())
print(f"executed warp instructions {te:.4g}, stall samples {ts}")
print(f"{'function':22s} {'instr %':>8s} {'stall %':>8s}")
for fn, e in ex.most_common(25):
    print(f"{fn:22s} {100*e/te:8.2f} {100*st[fn]/max(ts,1):8.2f}")
print("stall samples by reason (share of all samples) per function:")
print(f"{'function':22s} " + " ".join(f"{r[6:12]:>7s}" for r in reasons))
for fn, e in ex.most_common(12):
    print(f"{fn:22s} " + " ".join(f"{100*fr[fn][r]/max(ts,1):7.2f}" for r in reasons))
for rs in reasons[:3]:
    tot = sum(opst[rs].values())
    print(f"{rs}: stalled instruction is " + ", ".join(f"{o} {100*c/max(tot,1):.0f}%" for o, c in opst[rs].most_common(8)))
tw = sum(wf.values())
print("shared-memory wavefronts (share, excessive share of own): " + ", ".join(f"{fn} {100*c/max(tw,1):.0f}% ({100*wfx[fn]/max(c,1):.0f}%)" for fn, c in wf.most_common(8)))
print("instruction mix:", ", ".join(f"{o} {100*c/te:.1f}%" for o, c in opmix.most_common(16)))
if nlines:
    print("hottest lines (instr %, stall %):")
    for ln, e in byline.most_common(nlines):
        print(f"  {ln:5d} {100*e/te:6.2f} {100*stline[ln]/max(ts,1):6.2f}  {src[ln-1].strip()[:110]}")
    print("lines with most stall samples (instr %, stall %):")
    for ln, e in stline.most_common(nlines):
        print(f"  {ln:5d} {100*byline[ln]/te:6.2f} {100*e/max(ts,1):6.2f}  {src[ln-1].strip()[:110]}")
