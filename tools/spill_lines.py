"""Local-memory (spill) instructions of a kernel by source line: the CPU-side check behind DESIGN.md 9's "keep the register tile out
of local memory".  Compiles one .cu of csrc/ to a cubin with -lineinfo, disassembles it with `nvdisasm -g` and counts LDL / STL per
(file, line) inside the entry whose mangled name contains the given substring.

    python tools/spill_lines.py fwd_fast.cu fwd_fast_kernelILi10ELi50 [-DNAME ...]
"""
import collections, os, re, subprocess, sys, tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cvxpylayers_b200.build import ARCH_FLAGS  # noqa: E402
src, sub, defs = sys.argv[1], sys.argv[2], [a for a in sys.argv[3:] if a.startswith("-D")]
with tempfile.TemporaryDirectory() as td:
    cub = os.path.join(td, "k.cubin")
    r = subprocess.run(["nvcc", *ARCH_FLAGS, "-lineinfo", "-O3", "-std=c++17", "-Xptxas=-v", *defs, "-cubin", "-o", cub,
                        os.path.join(ROOT, "cvxpylayers_b200", "csrc", src)], capture_output=True, text=True)
    if r.returncode:
        sys.exit(r.stderr)
    lines = r.stderr.splitlines()
    for i, l in enumerate(lines):
        if "Compiling entry function" in l and sub in l:
            print("\n".join(x.replace("ptxas info    : ", "") for x in lines[i:i + 4]))
    out = subprocess.run(["nvdisasm", "-g", cub], capture_output=True, text=True).stdout
fun, cur, cnt = None, None, collections.Counter()
for l in out.splitlines():
    m = re.match(r"\s*\.text\.(\S+):", l)
    if m:
        fun = m.group(1)
    m = re.search(r'//## File "([^"]+)", line (\d+)', l)
    if m:
        cur = (os.path.basename(m.group(1)), int(m.group(2)))
        continue
    if fun and sub in fun and re.search(r"\b(LDL|STL)(\.\w+)*\b", l):
        cnt[cur] += 1
print(f"{sum(cnt.values())} local-memory instructions in *{sub}*:")
for (f, ln), c in sorted(cnt.items()):
    print(f"  {f}:{ln}  {c}")
