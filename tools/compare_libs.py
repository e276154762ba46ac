"""Two builds of libbcone.so side by side: do they plan and launch the same, and do they compute the same?

    python tools/compare_libs.py LIB_A LIB_B [--configs C1,C2,...] [--small-cta 0,1,2] [--timing]

For every `problems.CONFIGS` entry and every BCONE_SMALL_CTA mode, each library (loaded through BCONE_LIB in a process of its
own, because the mode is read when the handle is created) prints kernel_info(), path_info() and the launch_count() delta of one
solve and of one vjp and one jvp for every lsqr_precond (0, 1, 2) and least-squares method (LSQR, LSMR), with the fallback_count()
of the block-preconditioned vjp (lsqr_precond = 2), at a batch below and at a batch above what the grid keeps resident (SMs x CTAs
per SM).  The lines of the two libraries must be equal.  The vjp and the jvp run at a fixed point (the planted optimum, or library
A's solution where the workload has none) and are deterministic, so their outputs must be bit-identical; the forward forms K with floating-point atomics on some paths (fwd.cu, factor_and_g),
so its solutions are compared at 1e-8 relative, the tolerance tests/test_gpu_large.py uses for the same reason.

--timing instead prints, per library and alternating between them (order swapped every round), the host-clock time per call of
solve + vjp on C2 at a batch of one instance per SM (where the host's launch cost is visible): to completion, to enqueue 200
calls back to back, and to enqueue one call on an idle device; with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FWD = {"eps": 1e-4, "max_iters": 100000}
BWD = [{"lsqr_precond": pc, "mode": mode} for pc in (0, 1, 2) for mode in ("lsqr", "lsmr")]


def _setup(name, B, dev):
    import numpy as np
    import torch

    from cvxpylayers_b200 import problems as pr

    bt = pr.CONFIGS[name](B=B)
    t = lambda a: None if a is None else torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device=dev)  # noqa: E731
    return bt.structure, {k: t(getattr(bt, k)) for k in ("A_vals", "b", "c", "P_vals", "x_star", "y_star", "s_star")}


def worker(configs, outdir, at):
    """Runs in a process whose BCONE_LIB / BCONE_SMALL_CTA are set: one JSON line per (config, batch), outputs saved to outdir.
    at: the directory of the other library's outputs, whose solution is the point of differentiation where none is planted."""
    import torch

    from cvxpylayers_b200.engine import Engine, make_settings

    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    fs = make_settings(FWD)
    for name in configs:
        st, _ = _setup(name, 1, dev)
        info = Engine(st, dev).kernel_info()
        for B in (8, sms * max(info["fwd_ctas_per_sm"], info["bwd_ctas_per_sm"]) + 8):
            st, d = _setup(name, B, dev)
            eng = Engine(st, dev)
            g = torch.Generator(device="cpu").manual_seed(1)
            rnd = lambda *shape: torch.randn(shape, dtype=torch.float64, generator=g).to(dev)  # noqa: E731
            dx, dy, tA, tb, tc = rnd(B, st.n), rnd(B, st.m), rnd(B, st.nnzA), rnd(B, st.m), rnd(B, st.n)
            tP = rnd(B, st.nnzP) if st.nnzP else None
            counts, l0 = [], eng.launch_count()
            sol = eng.solve(d["A_vals"], d["b"], d["c"], d["P_vals"], fs)
            counts.append(eng.launch_count() - l0)
            pt = [d["x_star"], d["y_star"], d["s_star"]]
            if pt[0] is None:
                pt = torch.load(os.path.join(at, f"{name}_{B}.pt"))["solve"] if at else [sol.x, sol.y, sol.s]
            exact, fallbacks = [], []
            for args in BWD:
                bs = make_settings(args)
                # (a structure without a geometry for the call -- the forward mode, or LSMR's adjoint: both libraries must refuse it alike)
                for call in ("vjp", "jvp"):
                    l1 = eng.launch_count()
                    try:
                        out = (eng.vjp(d["A_vals"], d["b"], d["c"], *pt, dx, dy, d["P_vals"], bs) if call == "vjp" else
                               eng.jvp(d["A_vals"], d["b"], d["c"], *pt, tA, tb, tc, d["P_vals"], tP, bs))
                        counts.append(eng.launch_count() - l1)
                    except RuntimeError as ex:
                        out = ()
                        counts.append(str(ex))
                    if call == "vjp" and args["lsqr_precond"] == 2:
                        fallbacks.append(eng.fallback_count())
                    exact += [v for v in out if v is not None]
            torch.cuda.synchronize()
            torch.save({"solve": [sol.x, sol.y, sol.s], "status": [sol.status, sol.iters], "exact": exact},
                       os.path.join(outdir, f"{name}_{B}.pt"))
            print(json.dumps({"config": name, "B": B, "kernel_info": eng.kernel_info(), "path_info": eng.path_info(),
                              "launches_solve_then_vjp_jvp_per_setting": counts, "fallback_count_lsqr_lsmr": fallbacks,
                              "solved": int((sol.status == 1).sum())}), flush=True)


def timing(reps=200):
    import torch

    from bench import device_info
    from cvxpylayers_b200.engine import Engine, make_settings

    dev = torch.device("cuda", 0)
    B = torch.cuda.get_device_properties(dev).multi_processor_count
    st, d = _setup("C2", B, dev)
    eng = Engine(st, dev)
    fs = make_settings({"eps": 1e-4, "max_iters": 10000, "lsqr_precond": 1, "adaptive_check": 1})
    out, g = eng.alloc_solution(B), None
    dx, dy = torch.ones((B, st.n), dtype=torch.float64, device=dev), torch.ones((B, st.m), dtype=torch.float64, device=dev)

    def step():
        nonlocal g
        eng.solve(d["A_vals"], d["b"], d["c"], d["P_vals"], fs, out=out)
        g = eng.vjp(d["A_vals"], d["b"], d["c"], out.x, out.y, out.s, dx, dy, d["P_vals"], fs, out=g)

    for _ in range(20):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        step()
    t_enqueue = time.perf_counter() - t0   # host time to enqueue (the launches return before the kernels finish)
    torch.cuda.synchronize()
    t_all = time.perf_counter() - t0
    idle = []   # the same calls on an idle device, one at a time: host cost of a call without queueing effects (median)
    for _ in range(reps):
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        step()
        idle.append(time.perf_counter() - t1)
    print(json.dumps({"tool": "compare_libs --timing", "lib": os.environ.get("BCONE_LIB"), "config": "C2", "B": B, "calls": reps,
                      "us_per_solve_plus_vjp": round(1e6 * t_all / reps, 2), "host_enqueue_us_per_solve_plus_vjp": round(1e6 * t_enqueue / reps, 2),
                      "host_enqueue_us_idle_device_median": round(1e6 * sorted(idle)[reps // 2], 2),
                      "device": device_info(0)}), flush=True)


def _run(lib, extra_env, args, capture=True):
    env = {**os.environ, "BCONE_LIB": os.path.abspath(lib), **extra_env}
    r = subprocess.run([sys.executable, os.path.abspath(__file__), *args], env=env, text=True, stdout=subprocess.PIPE if capture else None)
    if r.returncode != 0:
        raise SystemExit(f"worker failed for {lib} ({extra_env})")
    return r.stdout.splitlines() if capture else []


def main():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("libs", nargs="*")
    p.add_argument("--configs", default=None)
    p.add_argument("--small-cta", default="0,1,2")
    p.add_argument("--timing", action="store_true")
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    p.add_argument("--at", default=None, help=argparse.SUPPRESS)
    a = p.parse_args()
    if a.worker:
        return timing() if a.worker == "timing" else worker(a.configs.split(","), a.worker, a.at)
    import torch

    from cvxpylayers_b200 import problems as pr

    if len(a.libs) != 2:
        p.error("two library paths")
    if a.timing:
        for r in range(a.rounds):
            for lib in (a.libs if r % 2 == 0 else a.libs[::-1]):   # (order swapped every round: whichever runs second must not matter)
                _run(lib, {}, ["--worker", "timing"], capture=False)
        return
    configs = a.configs or ",".join(pr.CONFIGS)
    bad = 0
    for mode in a.small_cta.split(","):
        with tempfile.TemporaryDirectory() as ta, tempfile.TemporaryDirectory() as tb:
            la = _run(a.libs[0], {"BCONE_SMALL_CTA": mode}, ["--worker", ta, "--configs", configs])
            lb = _run(a.libs[1], {"BCONE_SMALL_CTA": mode}, ["--worker", tb, "--configs", configs, "--at", ta])
            for x, y in zip(la, lb):
                rec = json.loads(x)
                fa, fb = (torch.load(os.path.join(td, f"{rec['config']}_{rec['B']}.pt")) for td in (ta, tb))
                exact = len(fa["exact"]) == len(fb["exact"]) and all(torch.equal(u, v) for u, v in zip(fa["exact"], fb["exact"]))
                status, iters = (torch.equal(u, v) for u, v in zip(fa["status"], fb["status"]))
                fwd_err = max(float((u - v).abs().max() / max(1.0, float(u.abs().max())))   # (an unsolved instance is NaN in both)
                              for u, v in zip(map(torch.nan_to_num, fa["solve"]), map(torch.nan_to_num, fb["solve"])))
                ok = x == y and exact and status and fwd_err <= 1e-8
                bad += not ok
                print(json.dumps({"BCONE_SMALL_CTA": int(mode), **rec, "same_lines": x == y, "vjp_jvp_bit_identical": exact,
                                  "status_equal": status, "iters_equal": iters, "solve_max_rel_diff": fwd_err, "ok": ok}), flush=True)
                if x != y:
                    print("  A:", x, "\n  B:", y, flush=True)
            bad += len(la) != len(lb)
    print(f"compare_libs: {'all equal' if not bad else f'{bad} MISMATCHES'}")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
