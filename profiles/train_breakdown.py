"""Where a DP training step of the cell spends its time (host-synchronised phases; diagnostic only)."""
import os, sys, time, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from mac_network_b200 import _lib
from mac_network_b200.config import MACConfig
from mac_network_b200.dp import DPTrainer
from mac_network_b200.params import init_params, perturb_biases
from mac_network_b200.synthetic import SHAPES, make_inputs
from mac_network_b200.mac_cell import mac_network
from mac_network_b200.autograd import mac_backward
B, S, N, d, L = SHAPES["headline"]
cfg = MACConfig.args("args", netLength=L)
pv = perturb_biases(init_params(cfg, L, seed=100), seed=101)
for prec, tc in (("fp32", False), ("bf16", True), ("bf16", False), ("fp32", True)):
    tr = DPTrainer(cfg, L, param_values=pv, seed=7, prec=prec, bwd_tc=tc)
    batch = {k: torch.from_numpy(v).cuda() for k, v in make_inputs(B, S, N, d, seed=1).items()}
    tm = torch.randn(B, d, device="cuda"); tcn = torch.randn(B, d, device="cuda")
    lib = _lib.load()
    for it in range(3):
        torch.cuda.synchronize(); t0 = time.perf_counter(); n0 = lib.mac_b200_launch_count()
        cell = tr.cell_for("k", batch); cell.seed = it + 1
        torch.cuda.synchronize(); t1 = time.perf_counter()
        c, m = mac_network(cell, L)
        t1h = time.perf_counter(); torch.cuda.synchronize(); t2 = time.perf_counter(); n1 = lib.mac_b200_launch_count()
        mac_backward(cell, tcn / B, tm / B, bucket=tr.bucket, tc=tc)
        t2h = time.perf_counter(); torch.cuda.synchronize(); t3 = time.perf_counter(); n2 = lib.mac_b200_launch_count()
        tr.apply(); torch.cuda.synchronize(); t4 = time.perf_counter()
    print(json.dumps({"prec": prec, "bwd_tc": tc, "cell_for_ms": (t1 - t0) * 1e3, "fwd_ms": (t2 - t1) * 1e3, "fwd_host_ms": (t1h - t1) * 1e3,
                      "fwd_launches": n1 - n0, "bwd_ms": (t3 - t2) * 1e3, "bwd_host_ms": (t2h - t2) * 1e3, "bwd_launches": n2 - n1,
                      "apply_ms": (t4 - t3) * 1e3}), flush=True)
    del tr; torch.cuda.empty_cache()
