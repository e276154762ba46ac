"""Instances whose CSR values do not fit in shared memory (the values-off-chip tier) next to the on-chip kernels and the CPU
oracle.  One JSON line per workload on stdout, with the card's name and power limit read in the same run:
CUDA-event time of the solve, the adjoint (bcone_vjp) and the forward mode (bcone_jvp), both with lsqr_precond = 1; mean
iterations; solved count; kernel paths; and the C oracle (oracle/cone_oracle.c, SCS-like, one instance per host core) on a
sample of the same instances with the same settings, as instances per second next to the GPU's.

    python tools/bench_large.py [--workloads qp_c2_tri,qp_c2_eig,qp_n200_eig,portfolio400] [--reps 3] [--warmup 1] [--sample 32]

qp_c2_tri / qp_c2_eig are the same 1024 QPs (BASELINE C2's n = 100 / m = 200) in the SOC form of cvxpy's DIFFCP path, with the
triangular factor (25,052 values per instance: on chip) and with cvxpy's dense eigen factor (30,002 values: off chip) -- the
direct cost of the tier on identical problems.  qp_n200_eig: n = 200 / m = 400 (120,002 values, 960 KB per instance: a full
grid's values exceed the L2).  portfolio400: socp_portfolio with 400 assets, 5 x 20 factor rows (40,800 values in CSR)."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench import device_info  # noqa: E402
from cvxpylayers_b200 import problems as pr  # noqa: E402
from cvxpylayers_b200.engine import Engine, make_settings  # noqa: E402
from oracle import oracle as orc  # noqa: E402

WORKLOADS = {
    "qp_c2_tri": lambda: pr.qp_as_socp(pr.dense_qp(1024, 100, 200, 50, seed=0)),
    "qp_c2_eig": lambda: pr.qp_as_socp(pr.dense_qp(1024, 100, 200, 50, seed=0), factor="eigen"),
    "qp_n200_eig": lambda: pr.qp_as_socp(pr.dense_qp(512, 200, 400, 100, seed=0), factor="eigen"),
    "portfolio400": lambda: pr.socp_portfolio(1024, n_assets=400, n_soc=5, k=20, seed=0),
}
FWD = {"eps": 1e-6, "max_iters": 200000}
BWD = {"lsqr_precond": 1}


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


def run(name: str, reps: int, warmup: int, sample: int, dev) -> dict:
    bt = WORKLOADS[name]()
    st, B = bt.structure, bt.B
    eng = Engine(st, dev)
    A, b, c = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev)
    fs, bs = make_settings(FWD), make_settings(BWD)
    rng = np.random.default_rng(0)
    wx, wy = _t(rng.standard_normal((B, st.n)), dev), _t(rng.standard_normal((B, st.m)), dev)
    tA, tb, tc = _t(rng.standard_normal((B, st.nnzA)), dev), _t(rng.standard_normal((B, st.m)), dev), _t(rng.standard_normal((B, st.n)), dev)
    out = {}

    def solve():
        out["sol"] = eng.solve(A, b, c, settings=fs)

    def vjp():
        s = out["sol"]
        out["vjp"] = eng.vjp(A, b, c, s.x, s.y, s.s, wx, wy, settings=bs)

    def jvp():
        s = out["sol"]
        out["jvp"] = eng.jvp(A, b, c, s.x, s.y, s.s, tA, tb, tc, settings=bs)

    for _ in range(warmup):
        solve(); vjp(); jvp()   # noqa: E702
    torch.cuda.synchronize()
    t_solve, t_vjp, t_jvp = _time(solve, reps), _time(vjp, reps), _time(jvp, reps)
    sol = out["sol"]
    solved = int((sol.status == 1).sum())
    # the C oracle on the host cores, same settings, on the first `sample` instances
    k = slice(0, min(sample, B))
    nk = k.stop
    t0 = time.perf_counter()
    xo, yo, so, sto, ito = orc.solve_batch(st, bt.A_vals[k], bt.b[k], bt.c[k], None, **FWD)
    t1 = time.perf_counter()
    orc.vjp_batch(st, bt.A_vals[k], bt.b[k], bt.c[k], xo, yo, so, _np(wx)[k], _np(wy)[k], None, **BWD)
    t2 = time.perf_counter()
    gpu_ips = lambda ms: round(B / (ms * 1e-3), 1)  # noqa: E731
    return {"tool": "bench_large", "workload": name, "B": B, "n": st.n, "m": st.m, "nnzA": st.nnzA, "value_bytes_per_instance": 8 * st.nnzA,
            "paths": eng.path_info(), "kernel_info": eng.kernel_info(), "solved": solved, "fwd_settings": FWD, "bwd_settings": BWD,
            "solve_ms": round(t_solve, 3), "vjp_ms": round(t_vjp, 3), "jvp_ms": round(t_jvp, 3),
            "iters_mean": round(float(sol.iters.double().mean()), 1),
            "vjp_lsqr_iters_mean": round(float(out["vjp"][4].double().mean()), 1), "jvp_lsqr_iters_mean": round(float(out["jvp"][3].double().mean()), 1),
            "gpu_solve_inst_per_s": gpu_ips(t_solve), "gpu_vjp_inst_per_s": gpu_ips(t_vjp),
            "oracle": {"sample": nk, "host_threads": orc.max_threads(), "solved": int((sto == 1).sum()), "iters_mean": round(float(ito.mean()), 1),
                       "solve_inst_per_s": round(nk / (t1 - t0), 1), "vjp_inst_per_s": round(nk / (t2 - t1), 1)},
            "reps": reps, "device": device_info(dev.index)}


def _np(t):
    return t.cpu().numpy()


def main():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--workloads", default=",".join(WORKLOADS))
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--warmup", type=int, default=1)
    p.add_argument("--sample", type=int, default=32)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_large needs a CUDA device")
    dev = torch.device("cuda", 0)
    for name in a.workloads.split(","):
        print(json.dumps(run(name, a.reps, a.warmup, a.sample, dev)), flush=True)


if __name__ == "__main__":
    main()
