"""The e4m3 read step (prec="fp8", csrc/read_step_fp8.cuh) against the bf16 one (csrc/read_step.cuh) at the headline shape
(B=64, N=196, d=512, netLength=12).  Usage:  python profiles/read_step_fp8.py OUT_DIR [--rounds 8]

  read step:  one inference read step as the cell runs it (mac_read_fwd_inv with y given: the read-step kernel + kb_attend),
              launched back to back over 6 input sets (knowledge base, inv, y, control, outputs) whose bytes exceed the 50 MB
              L2, CUDA events around 60 launches; bf16 and fp8 alternate `--rounds` times.
  passes/s:   whole inference passes (bench.py's resident form: 8 resident batches, CUDA graphs, 12 passes in flight on 12
              streams, the small_tc projections), bf16 and fp8 alternating `--rounds` times, each window >= 0.5 s.
  errors:     one headline pass of each precision against the fp64 oracle (worst per-step max-norm relative error).
Also records the card (name, power limit, max SM clock from nvidia-smi).  Writes OUT_DIR/read_step_fp8_h100.json."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import bench
from mac_network_b200 import _lib as L
from mac_network_b200.config import MACConfig
from mac_network_b200.mac_cell import MACParams
from mac_network_b200.params import init_params, perturb_biases
from mac_network_b200.synthetic import SHAPES

PRECS = ("bf16", "fp8")


def device_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock, "torch_device": torch.cuda.get_device_name(0)}


def spread(xs):
    xs = [float(x) for x in xs]
    return {"median": float(np.median(xs)), "min": min(xs), "max": max(xs), "rounds": [round(x, 4) for x in xs]}


def read_step_launchers(B, N, d, nsets=6):
    """For each precision, closures that run one read step on one of `nsets` input sets (same knowledge bases for both)."""
    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(5)
    W = {k: (torch.randn(*shp, device="cuda", generator=g) * sc).contiguous() for k, shp, sc in (
        ("Wx", (d, d), d ** -0.5), ("bx", (d,), 0.1), ("Wy", (d, d), d ** -0.5), ("by", (d,), 0.1),
        ("Wm", (2 * d, d), (2 * d) ** -0.5), ("bm", (d,), 0.1), ("Wm2", (d, d), d ** -0.5), ("bm2", (d,), 0.1),
        ("wr", (d,), 4 * d ** -0.5))}
    keep = []
    for k in ("Wx", "Wm", "Wm2"):
        o = torch.empty((W[k].shape[1], W[k].shape[0]), dtype=torch.bfloat16, device="cuda")
        L.check(lib.mac_pack_weight_bf16(L.ptr(W[k]), L.ptr(o), W[k].shape[0], W[k].shape[1], L.stream_ptr()))
        keep.append(o)
    for w in (W["Wm"][:d], W["Wm2"]):
        o = torch.empty((d, d), dtype=torch.uint8, device="cuda")
        s = torch.empty(d, device="cuda")
        L.check(lib.mac_pack_weight_fp8(L.ptr(w), L.ptr(o), L.ptr(s), d, d, L.stream_ptr()))
        keep += [o, s]
    rw = L.ReadWeights(*[W[k].data_ptr() for k in ("Wx", "bx", "Wy", "by", "Wm", "bm", "Wm2", "bm2", "wr")], 0.1,
                       *[t.data_ptr() for t in keep[:3]], None, None, None, None, *[t.data_ptr() for t in keep[3:]])
    wsb = lib.mac_read_workspace_bytes(B, N, d, 1)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    fns = {p: [] for p in PRECS}
    read_bytes = {}
    for _ in range(nsets):
        kb = torch.nn.functional.elu(torch.randn(B, N, d, device="cuda", generator=g)).to(torch.bfloat16).contiguous()
        y, c = torch.randn(B, d, device="cuda", generator=g), torch.randn(B, d, device="cuda", generator=g)
        info, att = torch.empty(B, d, device="cuda"), torch.empty(B, N, device="cuda")
        for prec in PRECS:
            code = L.PREC[prec]
            nb = lib.mac_read_invariant_bytes(B, N, d, code)
            inv = torch.empty(nb, dtype=torch.uint8, device="cuda")
            L.check(lib.mac_read_invariant(None, L.ptr(kb), ctypes.byref(rw), code, L.ptr(inv), nb, B, N, d, L.stream_ptr()))

            def step(inv=inv, kb=kb, y=y, c=c, info=info, att=att, code=code):
                L.check(lib.mac_read_fwd_inv(None, L.ptr(kb), L.ptr(inv), L.ptr(y), L.ptr(y), L.ptr(c), ctypes.byref(rw), code,
                                             L.ptr(info), L.ptr(att), L.ptr(ws), wsb, B, N, d, L.stream_ptr()))
            fns[prec].append(step)
            keep += [kb, y, c, info, att, inv]
    M = B * N
    # bytes one step reads from memory: P (or P8), Q, the knowledge base, both weights, y, control; writes att, info
    read_bytes["bf16"] = 3 * M * d * 2 + 2 * d * d * 2
    read_bytes["fp8"] = M * d + M * 4 + 2 * M * d * 2 + 2 * d * d + 2 * d * 4
    return fns, read_bytes, keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--steps", type=int, default=24, help="passes per timed window of the passes/s measurement")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    B, S, N, d, L_steps = SHAPES["headline"]
    out = {"device": device_info(), "shape_B_S_N_d_L": [B, S, N, d, L_steps], "rounds": args.rounds}

    # ---- one read step, alternating
    fns, read_bytes, keep = read_step_launchers(B, N, d)
    us = {p: [] for p in PRECS}
    for _ in range(args.rounds):
        for p in PRECS:
            us[p].append(bench.time_kernel(fns[p], iters=60) * 1e6)
    M = B * N
    out["read_step_fused_us"] = {p: dict(spread(us[p]), algorithmic_tflops=4.0 * M * d * d / np.median(us[p]) / 1e6,
                                         bytes_read=read_bytes[p]) for p in PRECS}
    out["read_step_fused_us"]["note"] = ("one inference read step (read-step kernel + kb_attend) per launch, 60 launches back to "
                                         "back over 6 input sets (> 50 MB L2), CUDA events; median / min / max over rounds")
    out["read_step_speedup_fp8"] = float(np.median(us["bf16"]) / np.median(us["fp8"]))
    del fns, keep
    torch.cuda.synchronize()

    # ---- whole passes at 12 in flight, alternating
    cfg = MACConfig.args("args", netLength=L_steps)
    params = MACParams(cfg, L_steps, values=perturb_biases(init_params(cfg, L_steps, seed=100), seed=101))
    nstreams = 12
    slots = {p: [bench.Slot(cfg, params, (B, S, N, d, L_steps), 1234 + s, p, True, fold_y=False, small_tc=True)
                 for s in range(bench.NSLOTS)] for p in PRECS}
    side = [torch.cuda.Stream() for _ in range(nstreams - 1)]
    main_stream = torch.cuda.current_stream()

    def runner(ss):
        def run(n):
            fork = torch.cuda.Event()
            fork.record(main_stream)
            for st in side:
                st.wait_event(fork)
            for k in range(n):
                j = k % nstreams
                if j == 0:
                    ss[k % len(ss)].run()
                else:
                    with torch.cuda.stream(side[j - 1]):
                        ss[k % len(ss)].run()
            for st in side:
                ev = torch.cuda.Event()
                ev.record(st)
                main_stream.wait_event(ev)
        return run
    runs = {p: runner(slots[p]) for p in PRECS}
    for p in PRECS:
        runs[p](2 * nstreams)
    torch.cuda.synchronize()
    pps = {p: [] for p in PRECS}
    for _ in range(args.rounds):
        for p in PRECS:
            t, _ = bench.timed_blocks(runs[p], args.steps, torch.cuda.synchronize, None, min_total_s=0.5)
            pps[p].append(args.steps / t)
    out["passes_per_s"] = {p: dict(spread(pps[p]), reasoning_steps_per_s=float(np.median(pps[p])) * L_steps,
                                   launches_per_pass=int(slots[p][0].launches)) for p in PRECS}
    out["passes_per_s"]["note"] = ("resident inputs (8 batches > 50 MB L2), CUDA graphs, 12 passes in flight on 12 streams, "
                                   "small_tc batch-sized projections; median / min / max over rounds of >= 0.5 s")
    out["passes_speedup_fp8"] = float(np.median(pps["fp8"]) / np.median(pps["bf16"]))
    del slots, runs
    torch.cuda.synchronize()

    # ---- errors against the fp64 oracle (one headline pass each)
    from tests._util import max_rel
    from tests.test_gpu_fullshape import PER_STEP, headline_case
    from tests.test_gpu_parity import run_gpu
    cfg_e, inputs, pv, ref = headline_case()
    out["max_rel_vs_fp64_oracle"] = {}
    for p in PRECS:
        got, _ = run_gpu(cfg_e, pv, inputs, L_steps, prec=p)
        out["max_rel_vs_fp64_oracle"][p] = {k: max(max_rel(got[k][i], ref[k][i]) for i in range(L_steps)) for k in PER_STEP}
    out["max_rel_vs_fp64_oracle"]["note"] = ("worst per-step max-norm relative error over the 12 steps, headline shape, "
                                             "init_params weights (tests/test_gpu_fullshape.py::headline_case)")
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "read_step_fp8_h100.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
