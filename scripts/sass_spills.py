"""Static SASS of the level kernel by source function: instructions, local-memory loads/stores (register spills) and moves.

    nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 --expt-relaxed-constexpr -Xptxas -v \\
         -cubin -o /tmp/tracker.cubin dvo_slam_b200/csrc/tracker.cu
    python scripts/sass_spills.py /tmp/tracker.cubin

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


def main():
    cubin = sys.argv[1]
    kernel = sys.argv[2] if len(sys.argv) > 2 else "k_level_persistent"
    nvdisasm = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvdisasm")
    sass = subprocess.run([nvdisasm, "-g", "-c", cubin], capture_output=True, text=True, check=True).stdout
    maps, acc = {}, collections.defaultdict(collections.Counter)
    section, fname, line = None, None, 0
    for ln in sass.splitlines():
        m = re.match(r"\s*\.section\s+\.text\.(\S+?),", ln)
        if m:
            section = m.group(1)
            continue
        m = re.match(r'\s*//## File "(.*)", line (\d+)', ln)
        if m:
            fname, line = os.path.basename(m.group(1)), int(m.group(2))
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", ln)
        if not m or section is None or kernel not in section:
            continue
        if fname not in maps:
            p = os.path.join(CSRC, fname or "")
            maps[fname] = function_map(p) if os.path.isfile(p) else {}
        c = acc[(fname, maps[fname].get(line, "(other)"))]
        op = m.group(2)
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
