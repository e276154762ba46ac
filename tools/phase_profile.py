"""Per-phase cycle shares of the forward and block-backward kernels (clock64 stamps by thread 0).
The indented sub-phase rows ([eq], [K], [it]) are only filled by a library built with -DBC_SUBPROF."""
import ctypes as C, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from cvxpylayers_b200 import problems as pr
from cvxpylayers_b200.engine import Engine, make_settings

B = int(sys.argv[1]) if len(sys.argv) > 1 else 1184
dev = torch.device("cuda", 0)
bt = pr.config_c2(B=B)
st = bt.structure
t = lambda a: None if a is None else torch.as_tensor(a, dtype=torch.float64, device=dev)
eng = Engine(st, dev)
args = make_settings({"eps": 1e-4, "max_iters": 10000, "lsqr_precond": 2, "adaptive_check": 1})
A, b, c, P = t(bt.A_vals), t(bt.b), t(bt.c), t(bt.P_vals)
g = torch.Generator(device="cpu").manual_seed(1)
dx = torch.randn((B, st.n), dtype=torch.float64, generator=g).to(dev)
dy = torch.randn((B, st.m), dtype=torch.float64, generator=g).to(dev)
sol = eng.solve(A, b, c, P, args); eng.vjp(A, b, c, sol.x, sol.y, sol.s, dx, dy, P, args)
eng.lib.bcone_set_profile(eng.h, 1, None)
sol = eng.solve(A, b, c, P, args); eng.vjp(A, b, c, sol.x, sol.y, sol.s, dx, dy, P, args)
out = (C.c_uint64 * 32)()
eng.lib.bcone_set_profile(eng.h, 1, out)
v = np.array(list(out), dtype=np.float64) / B   # cycles per instance
MHZ = torch.cuda.clock_rate(0)   # SM clock over the last sample period, read right after the profiled calls
print(torch.cuda.get_device_name(0), "SM clock", MHZ, "MHz")
names = {5: "  [chol P] factor", 6: "  [chol P] inverse", 16: "  [eq] A sweep", 17: "  [eq] P part", 18: "  [eq] scale update",
         19: "  [K] A'RA", 20: "  [K] + P", 21: "  [K] chol+inv", 22: "  [K] g", 23: "  [it] A'w", 24: "  [it] Li rows", 25: "  [it] Li cols",
         26: "  [it] A p", 27: "  [it] reduce", 28: "  [it] update+proj", 0: "fwd load", 1: "fwd equilibration", 2: "fwd K+chol+inv+g", 3: "fwd iterations", 4: "fwd checks",
         8: "bwd load", 9: "bwd Px + chol/inv P", 10: "bwd W", 11: "bwd S", 12: "bwd chol/inv S", 13: "bwd q+LSQR", 14: "bwd solve+write"}
for k, nm in names.items():
    print(f"{nm:26s} {v[k]:10.0f} cycles/instance  {v[k] / MHZ:7.1f} us")
print("fwd total us", v[:5].sum() / MHZ, "bwd total us", v[8:15].sum() / MHZ, "iters", sol.iters.float().mean().item())
if v[29]:   # slot 29: a counter, not cycles (register-tiled forward only)
    print("fwd factorisations per instance", v[29])
