"""Solution refinement (bcone_refine) next to the forward on C2, C3, C5 and EXP: the eps-1e-4 forward, refinement with 1, 2 and
3 steps from its solution (lsqr_precond = 1), and the eps-1e-8 forward, each with its error (max over x and y) to the planted
optimum where the batch has one (C2, C5) and to the eps-1e-8 forward's solution, as the largest and the median over the
instances the 3-step refinement accepted.
Times are CUDA events around one call, median of `reps` calls after one warm-up; refinement times exclude the copy that resets
its input.  The card name and power limit are printed with the lines.

    python tools/bench_refine.py [--reps 5] [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_polish import card, timed  # noqa: E402

from cvxpylayers_b200 import problems as pr  # noqa: E402
from cvxpylayers_b200.engine import Engine, Solution, make_settings  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = "cuda"
    lines = [{"card": card()}]
    configs = (("C2", lambda: pr.config_c2(4096)), ("C3", lambda: pr.socp_portfolio(2048)), ("C5", lambda: pr.sdp(256)),
               ("EXP", lambda: pr.exp_sum(64)))
    for name, make in configs:
        bt = make()
        eng = Engine(bt.structure, dev)
        T = lambda v: None if v is None else torch.tensor(v, dtype=torch.float64, device=dev)  # noqa: E731
        A, P, b, c = T(bt.A_vals), T(bt.P_vals), T(bt.b), T(bt.c)
        st8 = make_settings({"eps": 1e-8, "max_iters": 400000})
        sol8 = eng.solve(A, b, c, P, st8)
        t8 = timed(lambda: eng.solve(A, b, c, P, st8, out=sol8), a.reps)
        refs = {"eps_1e-8": (sol8.x.cpu().numpy(), sol8.y.cpu().numpy())}
        if bt.x_star is not None:
            refs["planted"] = (bt.x_star, bt.y_star)

        def errs(s_):
            return {k: np.maximum(np.abs(s_.x.cpu().numpy() - xr).max(1), np.abs(s_.y.cpu().numpy() - yr).max(1)) for k, (xr, yr) in refs.items()}

        st4 = make_settings({"eps": 1e-4, "lsqr_precond": 1})
        sol = eng.solve(A, b, c, P, st4)
        t4 = timed(lambda: eng.solve(A, b, c, P, st4, out=sol), a.reps)
        base = Solution(*(t.clone() for t in (sol.x, sol.y, sol.s, sol.status, sol.iters, sol.resid)))
        work = Solution(*(t.clone() for t in (base.x, base.y, base.s, base.status, base.iters, base.resid)))

        def reset():
            for u, v in ((work.x, base.x), (work.y, base.y), (work.s, base.s), (work.resid, base.resid)):
                u.copy_(v)

        t_copy = timed(reset, a.reps)
        ref_rows, e_ref = [], []
        for k in (1, 2, 3):
            t_k = timed(lambda: (reset(), eng.refine(A, b, c, work, P, st4, k)), a.reps) - t_copy
            reset()
            flags = eng.refine(A, b, c, work, P, st4, k).cpu().numpy()
            e_ref.append(errs(work))
            ref_rows.append({"steps": k, "refine_ms": t_k, "accepted": float((flags == 1).mean()), "rejected": float((flags == 0).mean()),
                             "not_attempted": float((flags == -1).mean())})
        mask = flags == 1   # (the instances the 3-step refinement accepted)

        def summary(e):
            return {k: {"max": float(v[mask].max()), "median": float(np.median(v[mask]))} for k, v in e.items()} if mask.any() else None

        for row, e in zip(ref_rows, e_ref):
            row["err"] = summary(e)
        lines.append({"config": name, "B": bt.B, "lsqr_precond": 1, "forward_eps_1e-4_ms": t4, "forward_eps_1e-8_ms": t8,
                      "err_eps_1e-4": summary(errs(base)), "err_eps_1e-8": summary(errs(sol8)), "refine": ref_rows})
        print(json.dumps(lines[-1]), flush=True)
    out = "\n".join(json.dumps(l_) for l_ in lines)
    print(out)
    if a.out:
        with open(a.out, "w") as f:
            f.write(out + "\n")


if __name__ == "__main__":
    main()
