"""LSMR (settings.lsmr = 1, diffcp's mode = "lsmr") against LSQR for the adjoint (bcone_vjp) and the forward mode (bcone_jvp) on
the same solutions: CUDA-event time per call (10 calls per timing, the two solvers alternated, median of three), mean iteration
counts, and the error against the exact least-squares solution on sampled instances for lsqr_precond 0 and 1.
One JSON line per (config, lsqr_precond) on stdout, with the card's name and power limit read in the same run.

    python tools/bench_lsmr.py [--configs C2:1,C2:2,C3:1,C5:1,EXP:1] [--reps 10] [--warmup 2] [--sample 4]

The timed lsqr_precond is the one after the colon; the errors are always reported for 0 and 1 (keys err_p0 / err_p1: the largest
relative difference of db, dc (adjoint) and dx, dy, ds (forward mode) to numpy.linalg.lstsq on the explicit system, over the
sampled instances, at the default iteration limit 2N)."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import device_info  # noqa: E402
from cvxpylayers_b200 import problems as pr  # noqa: E402
from cvxpylayers_b200.engine import Engine, make_settings  # noqa: E402
from tests.jvp_ref import dense_M, jvp_rhs  # noqa: E402

BATCH = {"C2": 4096, "C3": 2048, "C5": 256, "EXP": 64}
MODES = ("lsqr", "lsmr")


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


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _errors(eng, bt, A, b, c, P, x, y, s, wx, wy, tA, tb, tc, tP, idx, pc):
    """-> {mode: (adjoint error, forward-mode error)} on the sampled instances ``idx`` against exact least squares."""
    st, n = bt.structure, bt.structure.n
    xs, ys, ss = (v.cpu().numpy() for v in (x, y, s))
    wxs, wys = wx.cpu().numpy(), wy.cpu().numpy()
    exact = []
    for i in idx:
        Pd = bt.P_dense(i) if bt.P_vals is not None else None
        M, D, piy = dense_M(st, bt.A_dense(i), Pd, bt.b[i], bt.c[i], xs[i], ys[i], ss[i])
        dz = np.concatenate([wxs[i], D.T @ wys[i], [-(xs[i] @ wxs[i] + ys[i] @ wys[i])]])
        r = np.linalg.lstsq(M.T, dz, rcond=None)[0]
        tbt = pr.Batch(st, tA.cpu().numpy(), tb.cpu().numpy(), tc.cpu().numpy(), None if tP is None else tP.cpu().numpy())
        g = jvp_rhs(bt.A_dense(i), xs[i], piy, tbt.A_dense(i), None if tP is None else tbt.P_dense(i), tbt.b[i], tbt.c[i])
        z = np.linalg.lstsq(M, g, rcond=None)[0]
        zx, zy, zt = z[:n], z[n:-1], z[-1]
        Dzy = D @ zy
        exact.append((piy * r[-1] - r[n:-1], xs[i] * r[-1] - r[:n], zx - xs[i] * zt, Dzy - ys[i] * zt, Dzy - zy - ss[i] * zt))
    out = {}
    for mode in MODES:
        stg = make_settings({"mode": mode, "lsqr_precond": pc})
        _, _, db, dc, _ = eng.vjp(A, b, c, x, y, s, wx, wy, P, stg)
        jx, jy, js, _ = eng.jvp(A, b, c, x, y, s, tA, tb, tc, P, tP, stg)
        db, dc, jx, jy, js = (v.cpu().numpy() for v in (db, dc, jx, jy, js))
        ea = max(max(_rel(db[i], e[0]), _rel(dc[i], e[1])) for i, e in zip(idx, exact))
        ej = max(max(_rel(jx[i], e[2]), _rel(jy[i], e[3]), _rel(js[i], e[4])) for i, e in zip(idx, exact))
        out[mode] = (ea, ej)
    return out


def run(name: str, pc: int, reps: int, warmup: int, sample: int, dev) -> dict:
    B = BATCH[name]
    bt = pr.CONFIGS[name](B=B)
    st = bt.structure
    eng = Engine(st, dev)
    A, b, c, P = _t(bt.A_vals, dev), _t(bt.b, dev), _t(bt.c, dev), _t(bt.P_vals, dev)
    sol = eng.solve(A, b, c, P, make_settings({"eps": 1e-8, "max_iters": 200000}))
    torch.cuda.synchronize()
    solved = int((sol.status == 1).sum())
    rng = np.random.default_rng(0)
    tA, tb, tc = _t(rng.standard_normal(bt.A_vals.shape), dev), _t(rng.standard_normal(bt.b.shape), dev), _t(rng.standard_normal(bt.c.shape), dev)
    tP = _t(rng.standard_normal(bt.P_vals.shape), dev) if bt.P_vals is not None else None
    wx, wy = _t(rng.standard_normal((B, st.n)), dev), _t(rng.standard_normal((B, st.m)), dev)
    res = {"tool": "bench_lsmr", "config": name, "B": B, "n": st.n, "m": st.m, "solved": solved, "lsqr_precond": pc}
    calls, outs = {}, {}
    for mode in MODES:
        stg = make_settings({"mode": mode, "lsqr_precond": pc})

        def vjp(stg=stg, mode=mode):
            outs["vjp", mode] = eng.vjp(A, b, c, sol.x, sol.y, sol.s, wx, wy, P, stg)

        def jvp(stg=stg, mode=mode):
            outs["jvp", mode] = eng.jvp(A, b, c, sol.x, sol.y, sol.s, tA, tb, tc, P, tP, stg)

        calls["vjp", mode], calls["jvp", mode] = vjp, jvp
    for fn in calls.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in calls}
    for _ in range(3):   # alternate the solvers so that both see the same clocks
        for k, fn in calls.items():
            times[k].append(_time(fn, reps))
    if pc == 2 and eng.path_info()["bwd"].startswith("bwd_block_kernel"):
        res["lsmr_block_fallbacks"] = eng.fallback_count()   # (of the last block-preconditioned call: an LSMR adjoint)
    for (kind, mode), v in times.items():
        res[f"{kind}_{mode}_ms"] = round(float(np.median(v)), 4)
        res[f"{kind}_{mode}_iters_mean"] = round(float(outs[kind, mode][4 if kind == "vjp" else 3].double().mean()), 2)
    idx = list(np.random.default_rng(1).choice(B, size=min(sample, B), replace=False))
    if sample > 0:
        for p in (0, 1):
            e = _errors(eng, bt, A, b, c, P, sol.x, sol.y, sol.s, wx, wy, tA, tb, tc, tP, idx, p)
            for mode in MODES:
                res[f"err_p{p}_vjp_{mode}"], res[f"err_p{p}_jvp_{mode}"] = float(f"{e[mode][0]:.3e}"), float(f"{e[mode][1]:.3e}")
    res.update({"bwd_path": eng.path_info()["bwd"], "sample": [int(i) for i in idx], "reps": reps, "device": device_info(dev.index)})
    return res


def main():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--configs", default="C2:1,C2:2,C3:1,C5:1,EXP:1")
    p.add_argument("--reps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--sample", type=int, default=4)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lsmr needs a CUDA device")
    dev = torch.device("cuda", 0)
    for item in a.configs.split(","):
        name, pc = item.split(":") if ":" in item else (item, "1")
        print(json.dumps(run(name, int(pc), a.reps, a.warmup, a.sample, dev)), flush=True)


if __name__ == "__main__":
    main()
