"""Whole-model serving from host buffers: serving.ModelPipeline against a loop of MACnet.runBatch(train=False), as a caller
has to write it without the pipeline.  Usage:  python profiles/model_pipeline.py OUT_DIR [--rounds 5] [--window 1.0]

  arms:    at the CLEVR shape (B=64, S=40, 1024x14x14, d=512, L=12) and the GQA shape (B=64, S=30, 2048x7x7, d=512, L=6), for
           prec="bf16" and for prec="fp8" + eval_stem_prec="fp8" + eval_enc_prec="bf16":  (a) runBatch over numpy batches;
           (b) ModelPipeline with 1, 2 and 4 slots, host cast on and off (the cast exists with the bf16 stem only).  One
           process, the arms alternating `--rounds` times, every window at least `--window` seconds of host clock ending in
           a synchronise (a shorter one is timed again with more batches), the inputs rotating over three host batches
           (154 MB at the CLEVR shape: more than the L2 holds).
  stages:  device time of each stage of one un-overlapped pass (CUDA events around back-to-back launches): ingest, stem
           (ingest included), encoder, cell, output unit + top-k.
  ingest:  mac_ingest_nchw alone against permute().contiguous() + mac_im2col3x3, with the bytes each has to move over its
           time, beside the H100's 3.35 TB/s of HBM bandwidth (the bound of a copy kernel).
Records the card (name, power limit, max SM clock from nvidia-smi).  Writes OUT_DIR/model_pipeline_h100.json.  Fails
without a GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from mac_network_b200 import _lib as L
from mac_network_b200.config import MACConfig
from mac_network_b200.model import MACnet
from mac_network_b200.serving import ModelPipeline

HBM_TBS = 3.35
SHAPES = {"clevr": dict(variant="args", B=64, S=40, C=1024, H=14, W=14, L=12),
          "gqa": dict(variant="gqa", B=64, S=30, C=2048, H=7, W=7, L=6)}
MODELS = {"bf16": dict(prec="bf16"), "fp8": dict(prec="fp8", eval_stem_prec="fp8", eval_enc_prec="bf16")}
V, E, A = 90, 300, 28


def device_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock, "torch_device": torch.cuda.get_device_name(0)}


def host_batches(sh, n=3, seed=0):
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        lengths = rng.randint(sh["S"] // 2, sh["S"] + 1, size=(sh["B"],)).astype(np.int32)
        lengths[0] = sh["S"]
        q = rng.randint(1, V + 1, size=(sh["B"], sh["S"])).astype(np.int32)
        q[np.arange(sh["S"])[None, :] >= lengths[:, None]] = 0
        img = np.maximum(rng.standard_normal((sh["B"], sh["C"], sh["H"], sh["W"])), 0).astype(np.float32)
        out.append({"questions": q, "questionLengths": lengths, "images": img,
                    "answers": np.zeros(sh["B"], dtype=np.int32)})
    return out


def pinned(batches):
    return [{k: torch.from_numpy(v).pin_memory() for k, v in b.items() if k != "answers"} for b in batches]


def run_batch_arm(net, batches):
    def go(n):
        for i in range(n):
            b = batches[i % len(batches)]
            net.runBatch(None, b, {"images": b["images"]}, train=False)
        torch.cuda.synchronize()
    return go


def pipeline_arm(pipe, batches):
    def go(n):
        for i in range(n):
            pipe.submit(batches[i % len(batches)], next_batch=batches[(i + 1) % len(batches)])
        pipe.drain()
    return go


def wall(go, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    go(n)
    return (time.perf_counter() - t0) / n


def compare(arms, rounds, window_s):
    """arms: name -> go(n).  Warm up, size each window from a short run, alternate the arms `rounds` times (s per batch); a
    round that comes in under window_s (the sizing run was slower) is timed again with more batches, so every window that
    is kept lasted at least window_s."""
    iters = {}
    for name, go in arms.items():
        go(6)
        iters[name] = max(8, int(np.ceil(1.2 * window_s / wall(go, 8))))
    rows, windows = {name: [] for name in arms}, {name: [] for name in arms}
    for _ in range(rounds):
        for name, go in arms.items():
            per = wall(go, iters[name])
            while per * iters[name] < window_s:
                iters[name] = int(np.ceil(1.3 * window_s / per))
                per = wall(go, iters[name])
            rows[name].append(per)
            windows[name].append(per * iters[name])
    return {name: {"ms_per_batch": 1e3 * float(np.median(v)), "ms_min": 1e3 * min(v), "ms_max": 1e3 * max(v),
                   "batches_per_s": 1.0 / float(np.median(v)), "batches_per_window": iters[name],
                   "window_s": round(min(windows[name]), 3)} for name, v in rows.items()}


def timed(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3            # us


def stages(net, sh, batch, rounds, iters=20):
    """One eager slot's units, stage by stage on one stream: device time of back-to-back launches, nothing overlapped."""
    from mac_network_b200.mac_cell import mac_network
    from mac_network_b200.output_unit import answer_topk
    pipe = ModelPipeline(net, (sh["B"], sh["S"], sh["H"], sh["W"]), slots=1, use_graph=False, host_cast=False)
    pipe.result(pipe.submit(batch))
    s = pipe.slots[0]
    x = s.x
    B, C, H, W = x["images"].shape
    words, cntx, vecq = s.enc.forward(x["questions"], x["questionLengths"])
    memory = s.cell._hm[net.L]
    mode = 1 if s.stem.prec == "bf16" else 0
    out = (torch.empty((B * H * W, 9 * C), dtype=torch.bfloat16, device="cuda") if mode else
           torch.empty((B, H, W, C), device="cuda"))
    lib = L.load()
    fns = {"ingest": lambda: L.check(lib.mac_ingest_nchw(L.ptr(x["images"]), 0, L.ptr(out), mode, B, C, H, W, L.stream_ptr())),
           "stem": lambda: s.stem.forward_nchw(x["images"]),
           "encoder": lambda: s.enc.forward(x["questions"], x["questionLengths"]),
           "cell": lambda: mac_network(s.cell, net.L),
           "output_topk": lambda: answer_topk(s.out.logits(memory, vecq), 1)}
    us = {k: [] for k in fns}
    with torch.cuda.stream(s.stream):
        for fn in fns.values():
            fn()
        for _ in range(rounds):
            for k, fn in fns.items():
                us[k].append(timed(fn, iters))
    res = {k: {"us": float(np.median(v)), "us_min": min(v), "us_max": max(v)} for k, v in us.items()}
    res["sum_without_ingest_us"] = sum(res[k]["us"] for k in ("stem", "encoder", "cell", "output_topk"))
    res["note"] = ("eager launches on one stream, CUDA events around %d calls; `stem` includes `ingest`; at small kernels "
                   "this is launch-bound and an upper bound of the captured graph's time" % iters)
    return res


def ingest_part(sh, rounds, iters=30):
    lib = L.load()
    B, C, H, W = sh["B"], sh["C"], sh["H"], sh["W"]
    x = torch.relu(torch.randn(B, C, H, W, device="cuda"))
    x16 = x.to(torch.bfloat16)
    cols = torch.empty((B * H * W, 9 * C), dtype=torch.bfloat16, device="cuda")
    nhwc = torch.empty((B, H, W, C), device="cuda")
    s = L.stream_ptr()

    def baseline():
        t = x.permute(0, 2, 3, 1).contiguous()
        L.check(lib.mac_im2col3x3(L.ptr(t), L.ptr(cols), 1, 1.0, 0, 32, 0, B, H, W, C, s))
    n_in, n_cols = x.numel(), cols.numel()
    fns = {"permute_contiguous_im2col_bf16": (baseline, n_in * 4 * 3 + n_cols * 2),      # permute r+w, im2col reads once + writes
           "ingest_patch_bf16_from_fp32": (lambda: L.check(lib.mac_ingest_nchw(L.ptr(x), 0, L.ptr(cols), 1, B, C, H, W, s)),
                                           n_in * 4 + n_cols * 2),
           "ingest_patch_bf16_from_bf16": (lambda: L.check(lib.mac_ingest_nchw(L.ptr(x16), 1, L.ptr(cols), 1, B, C, H, W, s)),
                                           n_in * 2 + n_cols * 2),
           "permute_contiguous": (lambda: x.permute(0, 2, 3, 1).contiguous(), n_in * 8),
           "ingest_nhwc_f32": (lambda: L.check(lib.mac_ingest_nchw(L.ptr(x), 0, L.ptr(nhwc), 0, B, C, H, W, s)), n_in * 8)}
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
    out["note"] = ("min_bytes: what the operation has to read and write once (the baseline's im2col re-reads its input up "
                   "to nine times, mostly from L2; only one read is counted).  The bound is HBM bandwidth, %.2f TB/s on "
                   "the data sheet of a 700 W card" % HBM_TBS)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--shapes", default="clevr,gqa")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("model_pipeline.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    os.makedirs(a.out_dir, exist_ok=True)
    out = {"device": device_info(), "rounds": a.rounds, "window_s": a.window, "shapes": {}}
    for name in a.shapes.split(","):
        sh = SHAPES[name]
        cfg = MACConfig.args(sh["variant"], netLength=sh["L"])
        batches = host_batches(sh)
        pins = pinned(batches)
        res = {"shape": sh, "models": {}, "ingest": ingest_part(sh, a.rounds)}
        for mname, mkw in MODELS.items():
            net = MACnet(cfg, sh["L"], V, A, wrd_emb_dim=E, image_in_dim=sh["C"], classifier_dims=(512,), seed=7, **mkw)
            arms, pipes = {"runBatch_loop": run_batch_arm(net, batches)}, {}
            for slots in (1, 2, 4):
                for cast in ((True, False) if mname == "bf16" else (False,)):
                    key = "pipeline_%dslot_%s" % (slots, "hostcast" if cast else "fp32copy")
                    pipes[key] = ModelPipeline(net, (sh["B"], sh["S"], sh["H"], sh["W"]), slots=slots, host_cast=cast)
                    arms[key] = pipeline_arm(pipes[key], pins)
            r = compare(arms, a.rounds, a.window)
            for key, v in r.items():
                v["questions_per_s"] = v["batches_per_s"] * sh["B"]
                if key in pipes:
                    v["h2d_bytes_per_batch"], v["d2h_bytes_per_batch"] = pipes[key].h2d_bytes, pipes[key].d2h_bytes
                    v["h2d_gb_per_s"] = pipes[key].h2d_bytes * v["batches_per_s"] / 1e9
                else:
                    v["h2d_bytes_per_batch"] = batches[0]["images"].nbytes + batches[0]["questions"].nbytes + 2 * 4 * sh["B"]
            best = max((k for k in r if k in pipes), key=lambda k: r[k]["batches_per_s"])
            res["models"][mname] = {"arms": r, "best_pipeline": best,
                                    "speedup_over_runBatch_loop": r[best]["batches_per_s"] / r["runBatch_loop"]["batches_per_s"],
                                    "cast_ms": {k: p.cast_ms for k, p in pipes.items() if p.cast_ms is not None}}
            del pipes, arms
            res["models"][mname]["stages"] = stages(net, sh, pins[0], a.rounds)
            print(json.dumps({name: {mname: res["models"][mname]}}), flush=True)
            del net
            torch.cuda.empty_cache()
        out["shapes"][name] = res
    path = os.path.join(a.out_dir, "model_pipeline_h100.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out["device"]))


if __name__ == "__main__":
    main()
