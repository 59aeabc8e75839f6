"""Compare two `nvcc -Xptxas -v` logs of the library kernel by kernel.

    python tools/ptxas_compare.py parent.log this.log

Each log holds the output of compiling every csrc/*.cu with the library's flags plus `-Xptxas -v`
(`nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xptxas -v -c ...`).  Every kernel
entry becomes one line `demangled name | registers, barriers, stack, static shared memory | stack frame, spills`,
sorted.  The trailing periodic-boundary template argument PBC of the kernels that have one is written as an int in
both logs (it was a bool, false / true, before triclinic cells made it none / box / cell = 0 / 1 / 2), so a kernel
that existing calls run keeps its name across that change.  pair_bwd3_kernel's trailing lattice-gradient argument
LAT and tc_knn_kernel's trailing slot-group argument WIDE are dropped from the name when they are false, for the same
reason, and so is the trailing segment-form argument SEG of the cell-grid kernels (SEG_KERNELS).  Prints a unified diff of the two listings: a line present
in both is an instantiation whose registers, spills, stack and shared memory are unchanged."""
import difflib
import re
import subprocess
import sys

PBC_KERNELS = ("pair_kernel<", "pair_dense_tiled_kernel<", "pair_bwd1_kernel<", "pair_bwd3_kernel<",
               "knn_warp_select_kernel<", "knn_block_sort_kernel<", "tc_knn_kernel<", "tc_pair_kernel<",
               "radius_count_kernel<", "radius_scatter_kernel<", "radius_query_kernel<")

SEG_KERNELS = {"knn_grid_setup_kernel<": 4, "radius_count_kernel<": 5, "radius_scatter_kernel<": 5,   # template arguments
               "radius_query_kernel<": 4, "radius_query_wide_kernel<": 4, "knn_ring_kernel<": 5,      # with SEG
               "knn_scan_kernel<": 4}


def entries(path):
    out, cur, owner = [], None, None
    for line in open(path):
        m = re.search(r"Compiling entry function '(_Z\w+)'", line)
        p = re.search(r"Function properties for (\w+)", line)
        if m:
            cur = [m.group(1), "", ""]
            out.append(cur)
        elif p:
            owner = p.group(1)      # a non-inlined device function's properties can follow the entry's own
        elif cur is not None and owner == cur[0] and "bytes stack frame" in line:
            cur[2] = line.split(":", 1)[-1].strip()
        elif cur is not None and "Used" in line and "registers" in line:
            cur[1] = line.split(":", 1)[-1].strip()
    names = subprocess.run(["cu++filt"], input="\n".join(e[0] for e in out), capture_output=True, text=True,
                           check=True).stdout.splitlines()
    lines = []
    for (_, regs, frame), name in zip(out, names):
        if "pair_bwd3_kernel<" in name or "tc_knn_kernel<" in name:     # the trailing LAT / WIDE argument: dropped when false
            name = re.sub(r"(\(int\)\d), \(bool\)([01])>\(",    # before it), written as `true` otherwise
                          lambda m: m.group(1) + (">(" if m.group(2) == "0" else ", (bool)true>("), name, count=1)
        if any(k in name and name.split(">(", 1)[0].count(",") + 1 == n for k, n in SEG_KERNELS.items()):
            name = re.sub(r", \(bool\)([01])>\(", lambda m: ">(" if m.group(1) == "0" else ", (bool)true>(", name, count=1)
        if any(k in name for k in PBC_KERNELS):
            name = re.sub(r", \(bool\)([01])>\(", r", (int)\1>(", name, count=1)
        lines.append(f"{name} | {regs} | {frame}\n")
    return sorted(lines)


def main():
    a, b = entries(sys.argv[1]), entries(sys.argv[2])
    sys.stdout.writelines(difflib.unified_diff(a, b, sys.argv[1], sys.argv[2], n=0))
    print(f"# {len(a)} kernel entries before ({len(set(a))} distinct), {len(b)} after ({len(set(b))} distinct); "
          f"{sum(1 for x in a if x not in set(b))} of the entries before are missing or changed after")


if __name__ == "__main__":
    main()
