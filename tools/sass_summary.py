"""Per-kernel SASS evidence for the shipped library: counts of the instructions that prove the Hopper paths are in
the binary (UBLKCP = cp.async.bulk / TMA, SYNCS = mbarrier, DMMA = FP64 tensor-core mma, plus DFMA / LDS / STS / BAR / RED /
local-memory spills), the arch of the cubin and the hash of the .so, so that a stored profile ties the measured binary to the
sources.     python tools/sass_summary.py > sass_summary.txt"""
import hashlib, os, re, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = os.path.join(ROOT, "cvxpylayers_b200", "libbcone.so")
sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
print("library:", os.path.relpath(so, ROOT), "sha256", hashlib.sha256(open(so, "rb").read()).hexdigest()[:16], "bytes", os.path.getsize(so))
print("git HEAD:", subprocess.run(["git", "-C", ROOT, "rev-parse", "--short", "HEAD"], capture_output=True, text=True).stdout.strip())
archs = sorted(set(re.findall(r"arch = (sm_\w+)", sass)))
print("cubin archs:", ", ".join(archs))
keys = ["UBLKCP", "SYNCS", "DMMA", "DFMA", "LDS", "STS", "BAR.SYNC", "SHFL", "ATOM", "RED", "LDL", "STL", "MUFU"]
print(f"{'kernel':72s} " + " ".join(f"{k:>8s}" for k in keys))
cur, counts = None, {}
for line in sass.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        cur = m.group(1); counts[cur] = dict.fromkeys(keys, 0); continue
    if cur is None:
        continue
    for k in keys:
        if re.search(r"\b" + re.escape(k) + r"\b", line) or (k in ("UBLKCP", "SYNCS", "DMMA", "SHFL", "ATOM", "MUFU", "LDS", "STS", "LDL", "STL", "RED", "DFMA") and re.search(r"\s" + k + r"[.\s]", line)):
            counts[cur][k] += 1
            break
for fn, c in counts.items():
    name = subprocess.run(["c++filt", fn], capture_output=True, text=True).stdout.strip()
    name = re.sub(r"\(.*", "", name)
    print(f"{name[:72]:72s} " + " ".join(f"{c[k]:8d}" for k in keys))
