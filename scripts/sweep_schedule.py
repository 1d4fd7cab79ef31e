"""Static schedule of the fast PGS sweep loops of a Kuka kernel, from the SASS of a built library (CPU only, no GPU needed).

The fast loop of kuka_physics_step (csrc/kuka_device.cuh) has two copies: the quiet one (no env of the warp watches a contact) and the
watch one.  Each is an innermost loop whose body is one sweep: the button rows and the 12 motor rows, one `FFMA.SAT` each.  This script
runs `cuobjdump -sass` on the library, finds those loops in one kernel (default: the bench kernel, KukaButtonGymEnv rollout with four
lanes per env), and prints each loop's instruction count and static stall sum: the stall counts that ptxas wrote into the control bits of
the loop's instructions, i.e. the cycles one warp spends issuing one sweep when no variable-latency wait (memory, scoreboard) holds it.
On the single warp per scheduler this kernel runs, that sum is the floor of a sweep's time.

    python scripts/sweep_schedule.py [LIBRARY] [--kernel PATTERN] [--json]
"""
import argparse, json, os, re, shutil, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_LIB = os.path.join(ROOT, "robotics-rl-srl_b200", "csrc", "libsrl_sim_b200.so")
# kuka_kernel<JOINTS = false, TWOB = false, PREFETCH = false, COOP = true, TRACE = false>: what bench.py's Kuka rollout launches
DEFAULT_KERNEL = "kuka_kernelILb0ELb0ELb0ELb1ELb0EE"

_FUNC = re.compile(r"^\s*Function : (\S+)")
_INST = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;\s*/\* 0x([0-9a-f]{16}) \*/")
_CTRL = re.compile(r"^\s*/\* 0x([0-9a-f]{16}) \*/\s*$")
_BRA = re.compile(r"(?:^|\s)BRA(?:\.\S+)?\s+(?:!?U?P\d, )?(?:`\()?0x([0-9a-f]+)")


def find_cuobjdump():
    for c in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if c and os.path.exists(c):
            return c
    return None


def parse_sass(text, pattern):
    """Instructions of the first function whose name contains `pattern`: list of (address, text, stall cycles)."""
    insts, cur, pending = None, False, None
    for line in text.splitlines():
        m = _FUNC.match(line)
        if m:
            if cur:
                break
            cur = pattern in m.group(1)
            if cur:
                insts = []
            continue
        if not cur:
            continue
        m = _INST.match(line)
        if m:
            pending = (int(m.group(1), 16), m.group(2))
            continue
        m = _CTRL.match(line)
        if m and pending is not None:
            hi = int(m.group(1), 16)
            insts.append((pending[0], pending[1], (hi >> 41) & 0xF))   # control bits 105..108 of the 128-bit word: stall count
            pending = None
    return insts


def sweep_loops(insts):
    """Innermost loops (back edge to an earlier address, no other loop nested inside) with at least 12 FFMA.SAT."""
    idx = {a: i for i, (a, _, _) in enumerate(insts)}
    loops = []
    for i, (a, t, _) in enumerate(insts):
        m = _BRA.search(t)
        if m:
            tgt = int(m.group(1), 16)
            if tgt <= a and tgt in idx:
                loops.append((idx[tgt], i))
    inner = [l for l in loops if not any(o != l and l[0] <= o[0] and o[1] <= l[1] for o in loops)]
    out = []
    for s, e in sorted(set(inner)):
        body = insts[s:e + 1]
        nsat = sum(1 for _, t, _ in body if re.search(r"\bFFMA\.SAT\b", t))
        if nsat >= 12:
            out.append({"start": "0x%04x" % body[0][0], "end": "0x%04x" % body[-1][0], "instructions": len(body),
                        "stall_cycles": sum(st for _, _, st in body), "ffma_sat": nsat})
    # the quiet copy is the sweep and a back edge; the watch copy adds the watched rows' updates and the test
    out.sort(key=lambda l: l["instructions"])
    for k, l in enumerate(out):
        l["copy"] = "quiet" if k == 0 else "watch" if k == len(out) - 1 else "other"
    return out


def schedule(lib, pattern=DEFAULT_KERNEL):
    tool = find_cuobjdump()
    if tool is None:
        raise FileNotFoundError("cuobjdump not found")
    text = subprocess.run([tool, "-sass", lib], capture_output=True, text=True, check=True).stdout
    insts = parse_sass(text, pattern)
    if not insts:
        raise LookupError("no function matching %r in %s" % (pattern, lib))
    return sweep_loops(insts)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("lib", nargs="?", default=DEFAULT_LIB)
    ap.add_argument("--kernel", default=DEFAULT_KERNEL, help="substring of the mangled kernel name")
    ap.add_argument("--json", action="store_true")
    args = ap.parse_args()
    loops = schedule(args.lib, args.kernel)
    by = {l["copy"]: l for l in loops}
    ratio = by["watch"]["stall_cycles"] / by["quiet"]["stall_cycles"] if "watch" in by and "quiet" in by else None
    if args.json:
        print(json.dumps({"kernel": args.kernel, "loops": loops, "watch_over_quiet": ratio}))
        return
    print("%s in %s" % (args.kernel, os.path.relpath(args.lib)))
    print("%-6s %-15s %13s %22s %9s" % ("loop", "addresses", "instructions", "static cycles (stalls)", "FFMA.SAT"))
    for l in loops:
        print("%-6s %-15s %13d %22d %9d" % (l["copy"], l["start"] + "-" + l["end"][2:], l["instructions"], l["stall_cycles"], l["ffma_sat"]))
    if ratio is not None:
        print("watch / quiet static cycles: %.2f" % ratio)


if __name__ == "__main__":
    sys.exit(main())
