"""A training step through torch.autograd (`modules.MACModel` + `answer_loss` + `loss.backward()` + `torch.optim.Adam`) against
`DPTrainer.train_step_full` (hand-ordered backward, fused clip / Adam / EMA).  Usage:
    python profiles/torch_modules.py OUT_DIR [--rounds 5] [--window 1.0]

At the CLEVR training shape (B=64, S=40, 1024x14x14, d=512, L=12) with every unit on tensor cores (prec="bf16",
bwd_tc=True, bf16 stem and encoder), both arms on device-resident batches (NCHW images) rotating over three batches.  One
process, the arms alternating `--rounds` times, every window at least `--window` seconds of host clock ending in a
synchronise.  Also: the library launches per step of each arm (mac_b200_launch_count), and the host time of one step
(host clock from a drained device to the return of step(); both arms read the scalar logit biases back once after the
weights move, so this includes the device work enqueued before that read).  Records the card (name, power
limit, max SM clock from nvidia-smi).  Writes OUT_DIR/torch_modules_h100.json.  Fails without a GPU."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from mac_network_b200 import _lib as L
from mac_network_b200.config import MACConfig
from mac_network_b200.dp import DPTrainer
from mac_network_b200.modules import MACModel, answer_loss
from profiles.model_pipeline import compare, device_info
from profiles.train_pipeline import A, E, SHAPE, V, host_batches

PRECS = dict(prec="bf16", bwd_tc=True, stem_prec="bf16", enc_prec="bf16")


def device_batches(sh):
    names = {"questions": "questions", "questionLengths": "questionLengths", "answers": "answers", "images": "images_nchw"}
    return [{names[k]: torch.from_numpy(v).cuda() for k, v in b.items()} for b in host_batches(sh)]


def trainer_step(t, batches, sh):
    state = {"i": 0}

    def step():
        b = batches[state["i"] % len(batches)]
        state["i"] += 1
        t.train_step_full((sh["B"], sh["S"]), b, global_batch=sh["B"])
    return step


def module_step(m, opt, batches):
    state = {"i": 0}

    def step():
        b = batches[state["i"] % len(batches)]
        state["i"] += 1
        opt.zero_grad()
        logits, _ = m(b["questions"], b["questionLengths"], images_nchw=b["images_nchw"])
        answer_loss(logits, b["answers"]).backward()
        torch.nn.utils.clip_grad_norm_(m.parameters(), 8.0)
        opt.step()
    return step


def arm(step):
    def go(n):
        for _ in range(n):
            step()
        torch.cuda.synchronize()
    return go


def launches(step, lib):
    torch.cuda.synchronize()
    n0 = lib.mac_b200_launch_count()
    step()
    torch.cuda.synchronize()
    return int(lib.mac_b200_launch_count() - n0)


def enqueue_ms(step, n=10):
    """Host time of one step call (median of n), the device drained before each."""
    out = []
    for _ in range(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        step()
        out.append(time.perf_counter() - t0)
    torch.cuda.synchronize()
    return 1e3 * float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=1.0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("torch_modules.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    os.makedirs(a.out_dir, exist_ok=True)
    sh, lib = SHAPE, L.load()
    cfg = MACConfig.args(sh["variant"], netLength=sh["L"])
    batches = device_batches(sh)
    t = DPTrainer(cfg, sh["L"], seed=7, classifier=(A, [512]), encoder=(V, E), stem=(sh["C"], 2), **PRECS)
    m = MACModel.from_trainer(t)
    opt = torch.optim.Adam(m.parameters(), lr=1e-4, eps=1e-8)
    steps = {"DPTrainer.train_step_full": trainer_step(t, batches, sh), "MACModel+torch.optim.Adam": module_step(m, opt, batches)}
    out = {"device": device_info(), "rounds": a.rounds, "window_s": a.window, "shape": sh, "precisions": PRECS,
           "module_step": "zero_grad, forward, answer_loss, backward, clip_grad_norm_(8.0), Adam.step",
           "arms": compare({k: arm(s) for k, s in steps.items()}, a.rounds, a.window),
           "launches_per_step": {k: launches(s, lib) for k, s in steps.items()},
           "enqueue_ms": {k: enqueue_ms(s) for k, s in steps.items()}}
    base = out["arms"]["DPTrainer.train_step_full"]["ms_per_batch"]
    out["module_over_trainer"] = out["arms"]["MACModel+torch.optim.Adam"]["ms_per_batch"] / base
    path = os.path.join(a.out_dir, "torch_modules_h100.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
