"""Per-phase cycle counts of the generic forward kernel (fwd.cu) for any config: python tools/phase_generic.py C5 [B]"""
import ctypes as C, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import Engine, make_settings

name = sys.argv[1] if len(sys.argv) > 1 else "C5"
B = int(sys.argv[2]) if len(sys.argv) > 2 else {"C3": 2048, "C5": 256, "EXP": 1024, "C1": 4096, "C4": torch.cuda.get_device_properties(0).multi_processor_count}[name]
dev = torch.device("cuda", 0)
bt = pr.CONFIGS[name](B=B)
st = bt.structure
t = lambda a: None if a is None else torch.as_tensor(a, dtype=torch.float64, device=dev)
eng = Engine(st, dev)
args = make_settings({"eps": 1e-4, "max_iters": 100000})
A, b, c, P = t(bt.A_vals), t(bt.b), t(bt.c), t(bt.P_vals)
sol = eng.solve(A, b, c, P, args)
eng.lib.bcone_set_profile(eng.h, 1, None)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(); sol = eng.solve(A, b, c, P, args); e1.record(); torch.cuda.synchronize()
out = (C.c_uint64 * 32)()
eng.lib.bcone_set_profile(eng.h, 1, out)
v = np.array(list(out), dtype=np.float64) / B
MHZ = torch.cuda.clock_rate(0)   # SM clock over the last sample period, read right after the profiled call
its = sol.iters.float().mean().item()
print(name, "B", B, "kernel ms", e0.elapsed_time(e1), "SM clock MHz", MHZ, "geometry", eng.kernel_info(), "iters mean", its, "max", int(sol.iters.max()))
for k, nm in {0: "load", 1: "equilibration", 2: "K+chol+inv+g", 3: "iterations", 4: "checks"}.items():
    print(f"{nm:16s} {v[k]:12.0f} cycles/instance {v[k] / MHZ:9.1f} us")
print(f"per iteration: {v[3] / its:.0f} cycles = {v[3] / its / MHZ:.2f} us; per check: {v[4] / max(1.0, its / 25):.0f} cycles")
