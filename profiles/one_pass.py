"""ONE headline-shaped inference pass (B=64, S=40, N=196, d=512, netLength=12) in the throughput form the bench uses (bf16,
fused read step, tensor-core write + projY), without CUDA graphs, between cudaProfilerStart/Stop after three warm passes:
    ncu --profile-from-start off --metrics gpu__time_duration.sum,launch__grid_size --clock-control none --csv --log-file X python profiles/one_pass.py
    ncu --profile-from-start off --set full --clock-control none --import-source on -k regex:read_step_kernel -c 1 -o Y python profiles/one_pass.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mac_network_b200.config import MACConfig                               # noqa: E402
from mac_network_b200.mac_cell import MACCell, MACParams, mac_network       # noqa: E402
from mac_network_b200.params import init_params, perturb_biases             # noqa: E402
from mac_network_b200.synthetic import SHAPES, make_inputs                  # noqa: E402

variant = sys.argv[1] if len(sys.argv) > 1 else "args"
B, S, N, d, L = SHAPES["gqa" if variant == "gqa" else "headline"]
cfg = MACConfig.args(variant, netLength=L)
params = MACParams(cfg, L, values=perturb_biases(init_params(cfg, L, seed=100), seed=101))
x = {k: torch.from_numpy(v).cuda() for k, v in make_inputs(B, S, N, d, seed=1234).items()}
cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], x["knowledgeBase"],
               1.0, 1.0, 1.0, B, False, config=cfg, params=params, prec="bf16", small_tc=True, fold_y=False)
for _ in range(3):
    mac_network(cell, L)
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStart()
mac_network(cell, L)
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStop()
