"""Solution refinement (refine_kernel) on the paths a memory or race checker should see, meant to run under compute-sanitizer:
    compute-sanitizer --tool memcheck python tools/sanitize_refine.py
    compute-sanitizer --tool racecheck python tools/sanitize_refine.py
A dense (soc_sizes) and a CSR (psd_warm) pattern, each with every 5th row not attempted (status FAILED) and a batch of more than
twice what the 128-register build keeps resident (BCONE_SMALL_CTA=0), so every CTA refines several instances in turn and takes
the early exit of a not-attempted row between them; then the values-off-chip build (BCONE_VALUES_GLOBAL=1 on the exponential
structure).  One step with a short LSQR keeps the run short under the checker."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from cvxpylayers_b200.engine import Engine, Solution, make_settings  # noqa: E402
from tests import cone_planted as cp  # noqa: E402

dev = torch.device("cuda", 0)
t = lambda a: None if a is None else torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device=dev)  # noqa: E731
cases = [("soc_sizes", 600, {"BCONE_SMALL_CTA": "0"}), ("psd_warm", 600, {"BCONE_SMALL_CTA": "0"}), ("exp", 8, {"BCONE_VALUES_GLOBAL": "1"})]
for name, B, env in cases:
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    bt = cp.make(name, B)
    eng = Engine(bt.structure, dev)   # (the environment is read when the plans are made)
    for k, v in saved.items():
        if v is None:
            os.environ.pop(k)
        else:
            os.environ[k] = v
    rng = np.random.default_rng(0)
    x, y, s = (t(a + 1e-4 * rng.standard_normal(a.shape)) for a in (bt.x_star, bt.y_star, bt.s_star))
    status = torch.ones(B, dtype=torch.int32, device=dev)
    status[torch.arange(B, device=dev) % 5 == 2] = -4
    sol = Solution(x, y, s, status, torch.zeros_like(status), torch.zeros((B, 3), dtype=torch.float64, device=dev))
    flags = eng.refine(t(bt.A_vals), t(bt.b), t(bt.c), sol, t(bt.P_vals), make_settings({"lsqr_precond": 1, "lsqr_iter_lim": 20}), 1)
    torch.cuda.synchronize()
    info = eng.refine_info()
    f = flags.cpu().numpy()
    print(name, "B", B, "resident CTAs", info["num_sms"] * (info["small_ctas_per_sm"] if info["last_small"] == 1 else info["ctas_per_sm"]),
          "info", info, "flags", {int(k): int(v) for k, v in zip(*np.unique(f, return_counts=True))}, flush=True)
    assert (f[np.arange(B) % 5 == 2] == -1).all()
