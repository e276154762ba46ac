"""Forward-kernel time of the register-tiled kernel on its compile-time geometry (100 x 200 -> fwd_fast_kernel<10,50>) and on
runtime geometries (fwd_fast_kernel<0,0>) of similar size, so the headline is not a one-shape number (VERDICT r1 weak 11).
One JSON line per shape: ms per 4096-batch, us per instance-iteration."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import Engine, make_settings

dev = torch.device("cuda", 0)
B = 4096
sms = torch.cuda.get_device_properties(dev).multi_processor_count   # one resident instance per SM
args = make_settings({"eps": 1e-4, "max_iters": 10000, "adaptive_check": 1})
t = lambda a: None if a is None else torch.as_tensor(a, dtype=torch.float64, device=dev)
for (n, m, z) in [(100, 200, 50), (90, 200, 40), (100, 190, 50), (80, 160, 40), (96, 192, 48)]:
    bt = pr.dense_qp(B, n, m, z, seed=1)
    eng = Engine(bt.structure, dev)
    A, b, c, P = t(bt.A_vals), t(bt.b), t(bt.c), t(bt.P_vals)
    for _ in range(3):
        sol = eng.solve(A, b, c, P, args)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    for _ in range(5):
        sol = eng.solve(A, b, c, P, args)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 5
    its = float(sol.iters.float().mean())
    print(json.dumps({"n": n, "m": m, "z": z, "kernel": eng.path_info()["fwd"], "geometry": "compile-time <10,50>" if (n, m) == (100, 200) else "runtime <0,0>",
                      "fwd_ms_per_4096": round(ms, 3), "iters_mean": round(its, 2), "solved": int((sol.status == 1).sum()),
                      "us_per_instance": round(ms * 1e3 * sms / B, 1), "us_per_instance_iteration": round(ms * 1e3 * sms / B / its, 3),
                      "flops_scale_vs_100x200": round(n * m / 20000, 3)}))
