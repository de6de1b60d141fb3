"""Whole-model training from host buffers: serving.TrainPipeline against a loop of MACnet.runBatch(train=True), as a caller
has to write it without the pipeline.  Usage:  python profiles/train_pipeline.py OUT_DIR [--rounds 5] [--window 1.0]

  arms:    at the CLEVR training shape (B=64, S=40 with question lengths mixed in 20..40, 1024x14x14, d=512, L=12), for
           "all_tc" (prec="bf16", bwd_tc=True, bf16 stem and encoder) and "tc32" (the parity form, bf16x3 stem):
           (a) runBatch(train=True) over numpy batches; (b) the pipeline over numpy batches; (c) the pipeline over batches
           whose images are pinned tensors.  One process, the arms alternating `--rounds` times, every window at least
           `--window` seconds of host clock ending in a synchronise, the inputs rotating over three host batches.  The
           pipeline arms read each step's result after the next submit, as a training loop would.
  ingest:  mac_ingest_nchw_train alone (both patch forms, keep 0.82) against permute().contiguous() + mac_im2col3x3 /
           mac_im2col3x3_split, with the bytes each has to move over its time, beside the H100's 3.35 TB/s of HBM bandwidth.
Records the card (name, power limit, max SM clock from nvidia-smi).  Writes OUT_DIR/train_pipeline_h100.json.  Fails
without a GPU."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from mac_network_b200 import _lib as L
from mac_network_b200.config import MACConfig
from mac_network_b200.model import MACnet
from mac_network_b200.serving import TrainPipeline
from profiles.model_pipeline import HBM_TBS, compare, device_info, timed

SHAPE = dict(variant="args", B=64, S=40, C=1024, H=14, W=14, L=12)
CONFIGS = {"all_tc": dict(train_prec="bf16", bwd_tc=True, stem_prec="bf16", enc_prec="bf16"),
           "tc32": dict(train_prec="tc32", bwd_tc=True, stem_prec="bf16x3")}
V, E, A = 90, 300, 28
KEEP = 0.82


def host_batches(sh, n=3, seed=0):
    """n batches whose longest question fills S (one trained cell shape), the others 20..40 words."""
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        lengths = rng.randint(sh["S"] // 2, sh["S"] + 1, size=(sh["B"],)).astype(np.int32)
        lengths[0] = sh["S"]
        q = rng.randint(1, V + 1, size=(sh["B"], sh["S"])).astype(np.int32)
        q[np.arange(sh["S"])[None, :] >= lengths[:, None]] = 0
        out.append({"questions": q, "questionLengths": lengths, "answers": rng.randint(0, A, size=(sh["B"],)).astype(np.int32),
                    "images": np.maximum(rng.standard_normal((sh["B"], sh["C"], sh["H"], sh["W"])), 0).astype(np.float32)})
    return out


def run_batch_arm(net, batches):
    def go(n):
        for i in range(n):
            b = batches[i % len(batches)]
            net.runBatch(None, b, {"images": b["images"]}, train=True)
        torch.cuda.synchronize()
    return go


def pipeline_arm(pipe, batches):
    def go(n):
        prev = None
        for i in range(n):
            t = pipe.submit(batches[i % len(batches)])
            if prev is not None:
                pipe.result(prev)
            prev = t
        pipe.result(prev)
        pipe.drain()
    return go


def ingest_part(sh, rounds, iters=30):
    lib = L.load()
    B, C, H, W = sh["B"], sh["C"], sh["H"], sh["W"]
    x = torch.relu(torch.randn(B, C, H, W, device="cuda"))
    nhwc = torch.empty((B, H, W, C), device="cuda")
    M, K = B * H * W, 9 * C
    cols = torch.empty((M, 2 * K), dtype=torch.bfloat16, device="cuda")
    s = L.stream_ptr()

    def baseline(split):
        def go():
            t = x.permute(0, 2, 3, 1).contiguous()
            if split:
                L.check(lib.mac_im2col3x3_split(L.ptr(t), L.ptr(cols), KEEP, 7, 32, 1, B, H, W, C, s))
            else:
                L.check(lib.mac_im2col3x3(L.ptr(t), L.ptr(cols), 1, KEEP, 7, 32, 1, B, H, W, C, s))
        return go

    def ingest(form):
        return lambda: L.check(lib.mac_ingest_nchw_train(L.ptr(x), L.ptr(nhwc), L.ptr(cols), form, KEEP, 7, 32, 1, B, C, H, W, s))
    n_in = x.numel()
    fns = {  # permute r+w, the patch pass reads its input once and writes the patches
        "permute_contiguous_im2col_bf16": (baseline(False), n_in * 4 * 3 + M * K * 2),
        "ingest_train_bf16": (ingest(0), n_in * 4 * 2 + M * K * 2),
        "permute_contiguous_im2col_split": (baseline(True), n_in * 4 * 3 + M * K * 4),
        "ingest_train_split": (ingest(1), n_in * 4 * 2 + M * K * 4)}
    us = {k: [] for k in fns}
    for fn, _ in fns.values():
        fn()
    for _ in range(rounds):
        for k, (fn, _) in fns.items():
            us[k].append(timed(fn, iters))
    out = {}
    for k, (_, nbytes) in fns.items():
        med = float(np.median(us[k]))
        out[k] = {"us": med, "us_min": min(us[k]), "us_max": max(us[k]), "min_bytes": nbytes,
                  "tb_per_s_of_min_bytes": nbytes / med / 1e6, "share_of_hbm_bound": nbytes / med / 1e6 / HBM_TBS}
    out["note"] = ("keep %.2f.  min_bytes: what the operation has to read and write once (fp32 NCHW read, fp32 NHWC written, "
                   "bf16 patches written; the baseline's patch pass re-reads its input up to nine times, mostly from L2, "
                   "counted once).  The bound is HBM bandwidth, %.2f TB/s on the data sheet of a 700 W card" % (KEEP, HBM_TBS))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_pipeline.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    os.makedirs(a.out_dir, exist_ok=True)
    sh = SHAPE
    out = {"device": device_info(), "rounds": a.rounds, "window_s": a.window, "shape": sh, "stem_dropout": KEEP,
           "ingest": ingest_part(sh, a.rounds), "configs": {}}
    print(json.dumps({"ingest": out["ingest"]}), flush=True)
    cfg = MACConfig.args(sh["variant"], netLength=sh["L"])
    batches = host_batches(sh)
    pins = [dict(b, images=torch.from_numpy(b["images"]).pin_memory()) for b in batches]
    for name in a.configs.split(","):
        net = MACnet(cfg, sh["L"], V, A, wrd_emb_dim=E, image_in_dim=sh["C"], classifier_dims=(512,), seed=7, prec="bf16",
                     **CONFIGS[name])
        pipe = TrainPipeline(net, (sh["B"], sh["S"], sh["H"], sh["W"]), depth=2)
        arms = {"runBatch_numpy": run_batch_arm(net, batches), "pipeline_numpy": pipeline_arm(pipe, batches),
                "pipeline_pinned": pipeline_arm(pipe, pins)}
        r = compare(arms, a.rounds, a.window)
        base = r["runBatch_numpy"]["ms_per_batch"]
        for v in r.values():
            v["questions_per_s"] = v["batches_per_s"] * sh["B"]
            v["ms_saved_per_step"] = base - v["ms_per_batch"]
            v["speedup_over_runBatch"] = base / v["ms_per_batch"]
        out["configs"][name] = {"trainer": CONFIGS[name], "stage_threads": pipe.stage_threads, "arms": r}
        print(json.dumps({name: out["configs"][name]}), flush=True)
        del pipe, arms, net
        torch.cuda.empty_cache()
    path = os.path.join(a.out_dir, "train_pipeline_h100.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out["device"]))


if __name__ == "__main__":
    main()
