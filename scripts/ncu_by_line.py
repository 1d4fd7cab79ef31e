#!/usr/bin/env python
"""Stall samples / warp instructions of an ncu capture by SOURCE LINE (needs -lineinfo + --import-source on).
Usage: ncu_by_line.py rep.ncu-rep [top_n]   -> per file: totals; top lines; for kuka_coop.cuh / kuka_device.cuh: per function (by line ranges
found from 'KC_F void kc_...' / 'KK_DEV void kuka_...' definitions)."""
import collections, csv, io, re, subprocess, sys
rep = sys.argv[1]; topn = int(sys.argv[2]) if len(sys.argv) > 2 else 25
txt = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "cuda,sass"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(txt)))
cur_file, hdr = None, None
by_line = collections.defaultdict(lambda: [0, 0, collections.Counter(), ""])   # (file, line) -> samples, inst, stalls, text
cur_line = None
for r in rows:
    if not r:
        continue
    if r[0] in ("File Name", "File Path"):
        cur_file = r[1].split("/")[-1]; continue
    if r[0] == "Line No":
        hdr = r; isamp = hdr.index("# Samples"); iex = hdr.index("Instructions Executed")
        stalls = [(i, h.replace("stall_", "")) for i, h in enumerate(hdr) if h.startswith("stall_") and "Not Issued" not in h]
        continue
    if hdr is None or len(r) < len(hdr):
        continue
    if r[0] != "":
        cur_line = (cur_file, int(r[0])); by_line[cur_line][3] = r[1].strip()
        continue
    if cur_line is None:
        continue
    try:
        sm, ex = int(r[isamp] or 0), int(r[iex] or 0)
    except ValueError:
        continue
    e = by_line[cur_line]; e[0] += sm; e[1] += ex
    for i, n in stalls:
        v = int(r[i] or 0)
        if v: e[2][n] += v
tot_s = sum(e[0] for e in by_line.values()); tot_i = sum(e[1] for e in by_line.values())
print("total stall samples %d, warp instructions %d" % (tot_s, tot_i))
files = collections.defaultdict(lambda: [0, 0])
for (f, l), e in by_line.items():
    files[f][0] += e[0]; files[f][1] += e[1]
for f, (s_, i_) in sorted(files.items(), key=lambda x: -x[1][0]):
    print("file %-28s samples %5.1f %%  instructions %5.1f %%" % (f, 100.0 * s_ / tot_s, 100.0 * i_ / tot_i))
# function ranges
import os
root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "robotics-rl-srl_b200", "csrc")
for fname in ("kuka_coop.cuh", "kuka_device.cuh", "kuka_kernels.cu", "distractor_kernels.cu"):
    try:
        src = open(os.path.join(root, fname)).read().split("\n")
    except Exception:
        continue
    starts = [(n + 1, re.search(r"(kc_\w+|kuka_\w+|reset_\w+|env_\w+|apply_\w+)\s*\(", l).group(1)) for n, l in enumerate(src)
              if re.match(r"^(KC_F|KK_DEV|template|__global__).*\b(kc_\w+|kuka_\w+|reset_\w+|env_\w+|apply_\w+)\s*\(", l) and not l.strip().endswith(";")]
    starts = [(n, name) for n, name in starts]
    agg = collections.OrderedDict()
    for (f, l), e in by_line.items():
        if f != fname: continue
        name = "(file scope)"
        for n, nm in starts:
            if n <= l: name = nm
        a = agg.setdefault(name, [0, 0, collections.Counter()]); a[0] += e[0]; a[1] += e[1]; a[2].update(e[2])
    for name, a in sorted(agg.items(), key=lambda x: -x[1][0]):
        if a[0] * 1000 < tot_s: continue
        top = ", ".join("%s %d%%" % (k, 100 * v / max(1, a[0])) for k, v in a[2].most_common(4))
        print("  %-14s %-24s samples %5.1f %%  instructions %5.1f %%  cycles/instr %.1f  [%s]" % (fname, name, 100.0 * a[0] / tot_s, 100.0 * a[1] / tot_i,
              (a[0] / tot_s) / max(1e-9, a[1] / tot_i) * 1.0, top))
print("-- top lines")
for (f, l), e in sorted(by_line.items(), key=lambda x: -x[1][0])[:topn]:
    top = ", ".join("%s %d%%" % (k, 100 * v / max(1, e[0])) for k, v in e[2].most_common(3))
    print("%5.2f%% %5.2f%%i  %s:%d  %s   [%s]" % (100.0 * e[0] / tot_s, 100.0 * e[1] / tot_i, f, l, e[3][:90], top))
