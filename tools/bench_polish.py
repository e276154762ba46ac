"""Solution polishing (bcone_polish) next to the forward on C1 and C2: polish time (replicated and batch-shared A / P), the
forward at the same eps, the fraction of instances accepted at eps 1e-4 and 1e-3, the largest error to the planted optimum with
and without polishing, and the time of an eps-1e-8 forward for comparison.  Times are CUDA events around `reps` calls, median
of the calls after one warm-up.  The card name and power limit are printed with the lines.

    python tools/bench_polish.py [--reps 5] [--out FILE]
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
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name()


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = "cuda"
    lines = [{"card": card()}]
    for name, bt in (("C1", pr.dense_qp(4096, 10, 20, 0, seed=0)), ("C2", pr.config_c2(4096))):
        eng = Engine(bt.structure, dev)
        T = lambda v: torch.tensor(v, dtype=torch.float64, device=dev)  # noqa: E731
        A, P, b, c = T(bt.A_vals), T(bt.P_vals), T(bt.b), T(bt.c)
        masks = {}
        for eps in (1e-4, 1e-3):
            st = make_settings({"eps": eps})
            sol = eng.solve(A, b, c, P, st)
            t_fwd = timed(lambda: eng.solve(A, b, c, P, st, out=sol), a.reps)
            base = Solution(*(t.clone() for t in (sol.x, sol.y, sol.s, sol.status, sol.iters, sol.resid)))
            work = Solution(*(t.clone() for t in (base.x, base.y, base.s, base.status, base.iters, base.resid)))

            def pol(shared=False):
                for u, v in ((work.x, base.x), (work.y, base.y), (work.s, base.s)):
                    u.copy_(v)
                return eng.polish(A[0] if shared else A, b, c, work, P[0] if shared else P)

            t_copy = timed(lambda: [u.copy_(v) for u, v in ((work.x, base.x), (work.y, base.y), (work.s, base.s))], a.reps)
            t_pol = timed(pol, a.reps) - t_copy
            t_pol_sh = timed(lambda: pol(True), a.reps) - t_copy   # (A[0] for every instance: timing only, not planted)
            flags = pol().cpu().numpy()
            acc = masks[eps] = flags == 1
            # (over the accepted instances: a rejected one keeps its input, and a few planted C1 / C2 instances are degenerate)
            err = lambda s_: float(max(np.abs(s_.x.cpu().numpy() - bt.x_star)[acc].max(), np.abs(s_.y.cpu().numpy() - bt.y_star)[acc].max()))  # noqa: E731
            lines.append({"config": name, "B": bt.B, "eps": eps, "forward_ms": t_fwd, "polish_ms": t_pol, "polish_shared_ms": t_pol_sh,
                          "accepted": float((flags == 1).mean()), "rejected": float((flags == 0).mean()),
                          "not_attempted": float((flags == -1).mean()), "max_err_accepted_unpolished": err(base),
                          "max_err_accepted_polished": err(work)})
        st8 = make_settings({"eps": 1e-8, "max_iters": 400000})
        sol8 = eng.solve(A, b, c, P, st8)
        e8 = np.maximum(np.abs(sol8.x.cpu().numpy() - bt.x_star).max(1), np.abs(sol8.y.cpu().numpy() - bt.y_star).max(1))
        lines.append({"config": name, "B": bt.B, "eps": 1e-8, "forward_ms": timed(lambda: eng.solve(A, b, c, P, st8, out=sol8), a.reps),
                      "max_err_over_accepted_at_eps_1e-4": float(e8[masks[1e-4]].max()),
                      "max_err_over_accepted_at_eps_1e-3": float(e8[masks[1e-3]].max())})
    out = "\n".join(json.dumps(l_) for l_ in lines)
    print(out)
    if a.out:
        with open(a.out, "w") as f:
            f.write(out + "\n")


if __name__ == "__main__":
    main()
