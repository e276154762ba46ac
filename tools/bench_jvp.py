"""Forward-mode derivative (bcone_jvp) next to the adjoint (bcone_vjp) on the same solutions: CUDA-event time per call,
mean LSQR iterations, and time per LSQR iteration (call time / mean iterations), both with lsqr_precond = 1.
One JSON line per config on stdout, with the card's name and power limit read in the same run.

    python tools/bench_jvp.py [--configs C2,C3,C5,EXP] [--reps 10] [--warmup 2]

On C2 the adjoint takes the fused single-pass kernel (bwd_fast.cu) while the forward mode always runs the generic LSQR kernel
(bwd.cu), so the two times there compare different kernels."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench import device_info  # noqa: E402
from cvxpylayers_b200 import problems as pr  # noqa: E402
from cvxpylayers_b200.engine import Engine, make_settings  # noqa: E402

BATCH = {"C2": 4096, "C3": 2048, "C5": 256, "EXP": 64}


def _t(a, dev):
    return None if a is None else torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device=dev)


def _time(fn, reps: int) -> float:
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / reps


def run(name: str, reps: int, warmup: int, dev) -> dict:
    B = BATCH[name]
    bt = pr.CONFIGS[name](B=B)
    st = bt.structure
    eng = Engine(st, dev)
    A, b, c, P = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev)
    sol = eng.solve(A, b, c, P, make_settings({"eps": 1e-8, "max_iters": 200000}))
    torch.cuda.synchronize()
    solved = int((sol.status == 1).sum())
    rng = np.random.default_rng(0)
    dA, db, dc = _t(rng.standard_normal(bt.A_vals.shape), dev), _t(rng.standard_normal(bt.b.shape), dev), _t(rng.standard_normal(bt.c.shape), dev)
    dP = _t(rng.standard_normal(bt.P_vals.shape), dev) if bt.P_vals is not None else None
    wx, wy = _t(rng.standard_normal((B, st.n)), dev), _t(rng.standard_normal((B, st.m)), dev)
    stg = make_settings({"lsqr_precond": 1})
    jout = [None]
    vout = [None]

    def jvp():
        jout[0] = eng.jvp(A, b, c, sol.x, sol.y, sol.s, dA, db, dc, P, dP, stg)

    def vjp():
        vout[0] = eng.vjp(A, b, c, sol.x, sol.y, sol.s, wx, wy, P, stg)

    for _ in range(warmup):
        jvp()
        vjp()
    torch.cuda.synchronize()
    tj, tv = [], []
    for _ in range(3):   # alternate the two so that both see the same clocks
        tj.append(_time(jvp, reps))
        tv.append(_time(vjp, reps))
    tj, tv = float(np.median(tj)), float(np.median(tv))
    ij, iv = float(jout[0][3].double().mean()), float(vout[0][4].double().mean())
    # with lsqr_precond = 1 a structure that has the block-preconditioned kernel runs the fused one
    vjp_path = Engine.BWD_PATHS[0] if eng.path_info()["bwd"] == Engine.BWD_PATHS[0] else Engine.BWD_PATHS[1]
    return {"tool": "bench_jvp", "config": name, "B": B, "n": st.n, "m": st.m, "solved": solved, "lsqr_precond": 1,
            "vjp_path": vjp_path, "jvp_path": "bwd_kernel (generic LSQR, JVP)",
            "jvp_ms": round(tj, 4), "vjp_ms": round(tv, 4), "jvp_lsqr_iters_mean": round(ij, 2), "vjp_lsqr_iters_mean": round(iv, 2),
            "jvp_us_per_lsqr_iter": round(1e3 * tj / max(ij, 1e-9), 3), "vjp_us_per_lsqr_iter": round(1e3 * tv / max(iv, 1e-9), 3),
            "reps": reps, "device": device_info(dev.index)}


def main():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--configs", default="C2,C3,C5,EXP")
    p.add_argument("--reps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=2)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_jvp needs a CUDA device")
    dev = torch.device("cuda", 0)
    for name in a.configs.split(","):
        print(json.dumps(run(name, a.reps, a.warmup, dev)), flush=True)


if __name__ == "__main__":
    main()
