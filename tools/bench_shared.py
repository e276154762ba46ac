"""Batch-shared A and P against the replicated batch: solve, adjoint and forward mode, same data, same process, alternated.

For each workload the matrices of instance 0 are used by every instance (b and c stay per instance).  "replicated" passes
``A.expand(B, -1).contiguous()`` to the existing entry points, "shared" passes the one copy (bcone_*_shared).  Times are CUDA
events around `reps` calls, best of `rounds` alternated rounds.  The replicated inputs are built once, outside the timed region;
their size is reported as `replicated_input_bytes`.  Peak device bytes are torch's allocator peak over one call (the outputs it
allocates, such as the per-instance dA / dP of the replicated adjoint); the engine's own per-stream scratch is not counted by torch
(DESIGN.md §4 gives its size).  The card name and power limit of
the run are printed with the lines.

    python tools/bench_shared.py [--configs C2,C3,C5] [--rounds 3] [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cvxpylayers_b200 import problems as pr  # noqa: E402
from cvxpylayers_b200.engine import Engine, make_settings  # noqa: E402

BATCH = {"C2": 4096, "C3": 2048, "C5": 256}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20)
        name, pl = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
        return name, pl
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown"


def timed(fn, reps):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def run(name, rounds, reps, dev):
    B = BATCH[name]
    base = pr.CONFIGS[name](B=B, seed=0)
    st = base.structure
    rng = np.random.default_rng(1)
    A1 = torch.tensor(base.A_vals[0], device=dev)
    P1 = None if base.P_vals is None else torch.tensor(base.P_vals[0], device=dev)
    if name == "C2":
        bt = pr.plant(st, np.repeat(base.A_vals[:1], B, 0), np.repeat(base.P_vals[:1], B, 0), rng, active_frac=0.2)
        b, c = torch.tensor(bt.b, device=dev), torch.tensor(bt.c, device=dev)
    else:
        b = torch.tensor(base.b[:1] + 1e-3 * rng.standard_normal((B, st.m)) * (np.abs(base.b[:1]).max() + 1.0), device=dev)
        c = torch.tensor(base.c[:1] * (1.0 + 1e-3 * rng.standard_normal((B, st.n))), device=dev)
    eng = Engine(st, dev)
    S = make_settings({"lsqr_precond": 2} if name == "C2" else {"lsqr_precond": 1})
    sol = eng.solve(A1, b, c, P1, S)
    dx, dy = torch.randn((B, st.n), dtype=torch.float64, device=dev), torch.randn((B, st.m), dtype=torch.float64, device=dev)
    tA = torch.randn(st.nnzA, dtype=torch.float64, device=dev)
    tP = None if P1 is None else torch.randn(st.nnzP, dtype=torch.float64, device=dev)
    zb = torch.zeros((B, st.m), dtype=torch.float64, device=dev)
    # the replicated batch is materialised once, outside the timed region: only the calls are compared
    A_rep, P_rep = A1.expand(B, -1).contiguous(), None if P1 is None else P1.expand(B, -1).contiguous()
    tA_rep, tP_rep = tA.expand(B, -1).contiguous(), None if tP is None else tP.expand(B, -1).contiguous()
    rep_args = lambda: (A_rep, P_rep)  # noqa: E731

    def solve_rep():
        A, P = rep_args()
        eng.solve(A, b, c, P, S)

    def vjp_rep():
        A, P = rep_args()
        eng.vjp(A, b, c, sol.x, sol.y, sol.s, dx, dy, P, S)

    def jvp_rep():
        A, P = rep_args()
        eng.jvp(A, b, c, sol.x, sol.y, sol.s, tA_rep, zb, dx, P, tP_rep, S)

    fns = {
        ("solve", "replicated"): solve_rep,
        ("solve", "shared"): lambda: eng.solve(A1, b, c, P1, S),
        ("vjp", "replicated"): vjp_rep,
        ("vjp", "shared"): lambda: eng.vjp(A1, b, c, sol.x, sol.y, sol.s, dx, dy, P1, S),
        ("jvp", "replicated"): jvp_rep,
        ("jvp", "shared"): lambda: eng.jvp(A1, b, c, sol.x, sol.y, sol.s, tA, zb, dx, P1, tP, S),
    }
    for f in fns.values():   # warm-up (allocations, per-stream slabs)
        f()
    best = {k: float("inf") for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():   # alternated: replicated, shared, replicated, ... within each round
            best[k] = min(best[k], timed(f, reps))
    out = []
    for what in ("solve", "vjp", "jvp"):
        r, s = best[(what, "replicated")], best[(what, "shared")]
        out.append({"config": name, "B": B, "what": what, "replicated_ms": round(r, 3), "shared_ms": round(s, 3),
                    "speedup": round(r / s, 3), "replicated_peak_bytes": peak(fns[(what, "replicated")]),
                    "shared_peak_bytes": peak(fns[(what, "shared")]),
                    "replicated_input_bytes": B * (st.nnzA + st.nnzP) * 8 * (2 if what == "jvp" else 1), "path": eng.path_info()})
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--configs", default="C2,C3,C5")
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--out", default=None)
    a = p.parse_args()
    dev = torch.device("cuda", 0)
    name, pl = card()
    lines = []
    for cfg in a.configs.split(","):
        for rec in run(cfg, a.rounds, a.reps, dev):
            rec.update({"gpu": name, "power_limit": pl})
            lines.append(json.dumps(rec))
            print(lines[-1], flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
