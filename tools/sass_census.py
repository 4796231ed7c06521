"""Opcode census of the built library (cuobjdump -sass): which kernels use FFMA/DFMA (only inside IEEE division
sequences under --fmad=false), REDUX/MATCH (warp-aggregated binning).
usage: python tools/sass_census.py > sass_census.md"""
import collections, os, re, subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sass = subprocess.run(["cuobjdump", "-sass", os.path.join(ROOT, "nanort_b200", "libnanort_b200.so")],
                      capture_output=True, text=True).stdout
cur, ops = None, collections.OrderedDict()
for l in sass.splitlines():
    m = re.match(r"\s*Function : (\S+)", l)
    if m:
        cur = m.group(1)
        ops[cur] = []
        continue
    m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(@!?U?P\d\s+)?([A-Z0-9_.]+)", l)
    if cur and m:
        ops[cur].append(m.group(2))
WANT = ["traverse_fast3_kernel", "traverse_packet_kernel", "traverse_conformance_kernelINS_7AosRaysELb0", "scene_unified_kernelILi64ELi8E", "scene_list_kernel", "traverse_f64_kernel", "bin_large_kernel", "subtree_kernel",
        "instance_setup_kernel"]
print("| kernel | SASS instrs | FFMA/DFMA | ... of them within a division / sqrt sequence | FMUL+FADD (DMUL+DADD) | MUFU | REDUX | MATCH |")
print("|---|---|---|---|---|---|---|---|")
seen = set()
for name, lst in ops.items():
    if not any(w in name for w in WANT):
        continue
    dem = subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip()
    dem = re.sub(r"nrt::\(anonymous namespace\)::|nrt::", "", dem).split("(")[0][:160]
    if dem in seen or "Li512" in name:  # the deep-stack twin of a 64-entry instantiation
        continue
    seen.add(dem)
    c = collections.Counter(x.split(".")[0] for x in lst)
    fma = [i for i, x in enumerate(lst) if x.startswith("FFMA") or x.startswith("DFMA")]
    anchors = [i for i, x in enumerate(lst) if x.startswith("MUFU") or x.startswith("FCHK")]
    # the division slow path is a local subroutine whose FFMAs carry explicit rounding modes (.RZ/.RM/.RP)
    inside = sum(1 for i in fma if (anchors and min(abs(i - a) for a in anchors) <= 28) or re.search(r"\.R[ZMP]", lst[i]))
    print(f"| `{dem}` | {len(lst)} | {len(fma)} | {inside} | {c['FMUL'] + c['FADD']} ({c['DMUL'] + c['DADD']}) | {c['MUFU']} | "
          f"{c['REDUX']} | {c['MATCH']} |")
