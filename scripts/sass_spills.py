"""Static SASS of the level kernel by source function: instructions, local-memory loads/stores (register spills) and moves.

    nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 --expt-relaxed-constexpr -Xptxas -v \\
         -cubin -o /tmp/tracker.cubin dvo_slam_b200/csrc/tracker.cu
    python scripts/sass_spills.py /tmp/tracker.cubin
    python scripts/sass_spills.py /tmp/tracker.cubin --loops     # the innermost pixel loops of stages A and B

Counts instructions in the code (both template instances of stage B), not executed ones.  Every instruction is attributed
through `nvdisasm -g` to the source line it came from and the line to the function that lexically contains it (inlined
code counts for the function it was written in; see instruction_accounting.function_map)."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from instruction_accounting import CSRC, function_map  # noqa: E402


PIXEL_FUNCS = {"residual_pixel": "A", "record_pixel": "B"}


def disassemble(cubin, kernel):
    """The kernel's instructions in address order as (address, opcode, function) and the index each label points at."""
    nvdisasm = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvdisasm")
    sass = subprocess.run([nvdisasm, "-g", "-c", cubin], capture_output=True, text=True, check=True).stdout
    maps, ins, labels = {}, [], {}
    section, fname, line = None, None, 0
    for ln in sass.splitlines():
        m = re.match(r"\s*\.section\s+\.text\.(\S+?),", ln)
        if m:
            section = m.group(1)
            continue
        if section is None or kernel not in section:
            continue
        m = re.match(r'\s*//## File "(.*)", line (\d+)', ln)
        if m:
            fname, line = os.path.basename(m.group(1)), int(m.group(2))
            continue
        m = re.match(r"^(\.L_x_\d+):", ln)
        if m:
            labels[m.group(1)] = len(ins)
            continue
        m = re.match(r"\s*/\*([0-9a-f]+)\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)(.*)", ln)
        if not m:
            continue
        if fname not in maps:
            p = os.path.join(CSRC, fname or "")
            maps[fname] = function_map(p) if os.path.isfile(p) else {}
        target = re.search(r"`\((\.L_x_\d+)\)", m.group(4)) if m.group(3).startswith("BRA") else None
        ins.append((int(m.group(1), 16), m.group(3), (fname, maps[fname].get(line, "(other)")), target and target.group(1)))
    return ins, labels


def pixel_loops(cubin, kernel):
    """Static counts of the innermost pixel loops: every backward branch closes a loop [target, branch]; a loop is a pixel
    loop of stage A / B when it holds code of residual_pixel / record_pixel, and innermost when no smaller pixel loop
    overlaps it.  CALL in a stage-B loop marks the instance that dumps the residual records (dvo_b200_residual_image).  Generic `LD` is the gather path's load from global memory or the window through generic addresses."""
    ins, labels = disassemble(cubin, kernel)
    loops = [(labels[t], i) for i, (_, _, _, t) in enumerate(ins) if t in labels and labels[t] <= i]
    found = []
    for lo, hi in loops:
        body = ins[lo:hi + 1]
        stages = {PIXEL_FUNCS[f] for _, _, (_, f), _ in body if f in PIXEL_FUNCS}
        if stages:
            found.append((lo, hi, "".join(sorted(stages))))
    cols = ("inst", "LDL", "STL", "LD", "BRA", "VOTE", "CALL", "gather")
    print("%-8s %-14s" % ("stage", "loop") + "".join("%8s" % k for k in cols))
    for lo, hi, st in found:
        if any(h2 - l2 < hi - lo and l2 <= hi and lo <= h2 for l2, h2, _ in found):
            continue   # an outer loop: it contains (or, entered in its middle, overlaps) a smaller pixel loop
        c = collections.Counter()
        for _, op, (_, f), _ in ins[lo:hi + 1]:
            base = op.split(".")[0]
            c["inst"] += 1
            c[base] += base in cols
            c["gather"] += f.startswith("gather_taps")
        print("%-8s %#06x-%#06x" % (st, ins[lo][0], ins[hi][0]) + "".join("%8d" % c[k] for k in cols))


def main():
    args = [a for a in sys.argv[1:] if a != "--loops"]
    cubin = args[0]
    kernel = args[1] if len(args) > 1 else "k_level_persistent"
    if "--loops" in sys.argv:
        pixel_loops(cubin, kernel)
        return
    ins, _ = disassemble(cubin, kernel)
    acc = collections.defaultdict(collections.Counter)
    for _, op, key, _ in ins:
        c = acc[key]
        c["inst"] += 1
        c[op.split(".")[0]] += op.split(".")[0] in ("LDL", "STL", "MOV")
        c["IMAD.MOV"] += op.startswith("IMAD.MOV")
    cols = ("inst", "LDL", "STL", "MOV", "IMAD.MOV")
    print("%-22s %-28s" % ("file", "function") + "".join("%9s" % k for k in cols))
    total = collections.Counter()
    for (f, fn), c in sorted(acc.items(), key=lambda kv: -kv[1]["inst"]):
        total.update(c)
        print("%-22s %-28s" % (f, fn) + "".join("%9d" % c[k] for k in cols))
    print("%-51s" % "total" + "".join("%9d" % total[k] for k in cols))


if __name__ == "__main__":
    main()
