"""Solution polishing in the slab tier (csrc/polish_large.cu) next to the forward: C4 (sparse LP, n = 1000, m = 2000, B = 512),
problems.sparse_qp (n = 300, m = 600, diagonal P, B = 4096) and a dense QP (n = 256, m = 512, B = 1024).  Per workload and
forward eps (1e-3, 1e-4): the forward's time and median iteration count, the polish time, the attempted and accepted fractions,
the max and median error to the planted optimum before and after polishing, and the DMMA FLOP count of the attempted instances
with the achieved FP64 rate of the polish kernel; then a forward at eps 1e-6 for comparison.  Times are CUDA events, median of
`reps` calls after one warm-up.  The card name, power limit, max SM clock, the polish grid and slab bytes are recorded in the
same run.  Lines are written as they are measured.

    python tools/bench_polish_large.py [--reps 3] [--out profiles/bench_polish_large_h100.jsonl] [--only C4,sparse_qp,dense_qp]
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
from cvxpylayers_b200.engine import Engine, Solution, make_settings  # noqa: E402


def card():
    out = {"name": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        out["power_limit"], out["clocks_max_sm"] = (v.strip() for v in q.splitlines()[0].split(","))
    except Exception as e:  # noqa: BLE001
        out["nvidia_smi"] = f"unavailable: {e}"
    return out


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def dmma_flops(n, nl, p_diag):
    """FP64 FLOPs of the O(n^3) work of one attempted instance: Cholesky + inverse of P + d I (n^3 / 3 each, dense P only),
    W = A_L L^{-T} (nl n^2, dense P only), S = W W' (nl^2 n: the lower half of S, n deep) and Cholesky + inverse of S."""
    f = nl * nl * n + 2.0 * nl ** 3 / 3.0
    if not p_diag:
        f += 2.0 * n ** 3 / 3.0 + nl * n * n
    return f


def workloads(only):
    w = {
        "C4": lambda: pr.sparse_lp(512, 1000, 2000, seed=0),
        "sparse_qp": lambda: pr.sparse_qp(4096, 300, 600, seed=0),
        "dense_qp": lambda: pr.dense_qp(1024, 256, 512, 64, seed=0),
    }
    return {k: v for k, v in w.items() if not only or k in only}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    dev = "cuda"
    f = open(a.out, "w") if a.out else None

    def emit(line):
        s = json.dumps(line)
        print(s, flush=True)
        if f:
            f.write(s + "\n")
            f.flush()

    emit({"card": card()})
    for name, make in workloads([s for s in a.only.split(",") if s]).items():
        bt = make()
        st_ = bt.structure
        eng = Engine(st_, dev)
        info = eng.polish_info()
        p_diag = st_.P_indptr is None or bool(np.all(np.repeat(np.arange(st_.n), np.diff(st_.P_indptr)) == st_.P_indices))
        emit({"config": name, "B": bt.B, "n": st_.n, "m": st_.m, "polish_plan": info, "p_diag": p_diag})
        T = lambda v: None if v is None else torch.tensor(v, dtype=torch.float64, device=dev)  # noqa: E731
        A, P, b, c = T(bt.A_vals), T(bt.P_vals), T(bt.b), T(bt.c)
        z = st_.cones.z

        def err(x, y):
            e = np.maximum(np.abs(x - bt.x_star).max(1), np.abs(y - bt.y_star).max(1))
            return float(e.max()), float(np.median(e))

        for eps in (1e-3, 1e-4):
            st = make_settings({"eps": eps})
            sol = eng.solve(A, b, c, P, st)
            t_fwd = timed(lambda: eng.solve(A, b, c, P, st, out=sol), a.reps)
            base = Solution(*(t.clone() for t in (sol.x, sol.y, sol.s, sol.status, sol.iters, sol.resid)))
            work = Solution(*(t.clone() for t in (base.x, base.y, base.s, base.status, base.iters, base.resid)))

            def reset():
                for u, v in ((work.x, base.x), (work.y, base.y), (work.s, base.s), (work.resid, base.resid)):
                    u.copy_(v)

            def pol():
                reset()
                return eng.polish(A, b, c, work, P)

            t_copy = timed(reset, a.reps)
            t_pol = timed(pol, a.reps) - t_copy
            flags = pol().cpu().numpy()
            torch.cuda.synchronize()
            xb, yb, sb = (t.cpu().numpy() for t in (base.x, base.y, base.s))
            nl = z + (yb[:, z:] > sb[:, z:]).sum(1)
            att = flags >= 0
            flops = float(sum(dmma_flops(st_.n, int(k), p_diag) for k in nl[att]))
            e0, e1 = err(xb, yb), err(work.x.cpu().numpy(), work.y.cpu().numpy())
            emit({"config": name, "B": bt.B, "eps": eps, "forward_ms": t_fwd, "median_iters": float(np.median(base.iters.cpu().numpy())),
                  "solved": float((base.status.cpu().numpy() == 1).mean()), "polish_ms": t_pol,
                  "attempted": float(att.mean()), "accepted": float((flags == 1).mean()), "rejected": float((flags == 0).mean()),
                  "median_live_rows": float(np.median(nl)), "planted_live_rows_median": float(np.median(z + (bt.y_star[:, z:] > 0).sum(1))),
                  "max_err_unpolished": e0[0], "median_err_unpolished": e0[1], "max_err_polished": e1[0], "median_err_polished": e1[1],
                  "dmma_gflop_attempted": flops / 1e9, "polish_tflops": flops / (t_pol * 1e-3) / 1e12 if t_pol > 0 else None})
        st6 = make_settings({"eps": 1e-6})
        sol6 = eng.solve(A, b, c, P, st6)
        t6 = timed(lambda: eng.solve(A, b, c, P, st6, out=sol6), a.reps)
        e6 = err(sol6.x.cpu().numpy(), sol6.y.cpu().numpy())
        emit({"config": name, "B": bt.B, "eps": 1e-6, "forward_ms": t6, "median_iters": float(np.median(sol6.iters.cpu().numpy())),
              "solved": float((sol6.status.cpu().numpy() == 1).mean()), "max_err": e6[0], "median_err": e6[1]})
    if f:
        f.close()


if __name__ == "__main__":
    main()
