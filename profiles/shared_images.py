"""Several questions per image: serving.ModelPipeline(images=U) against ModelPipeline() fed one image per question, and
mac_kb_gather against mac_cast_bf16.  Usage:  python profiles/shared_images.py OUT_DIR [--rounds 5] [--window 1.0]

  arms:    at the CLEVR shape (B=64, S=40, 1024x14x14, d=512, L=12) and the GQA shape (B=64, S=30, 2048x7x7, d=512, L=6), for
           prec="bf16" and for prec="fp8" + eval_stem_prec="fp8" + eval_enc_prec="bf16", four slots, fp32 copies (no host
           cast): (a) images=None fed the duplicated features (B images per batch); (b) images=16 and (c) images=8, fed
           batches of 16 and 8 distinct images.  Method of profiles/model_pipeline.py (DESIGN.md section 8): one process,
           the arms alternating `--rounds` times, every window at least `--window` seconds of host clock ending in a
           synchronise, the inputs rotating over three pinned host batches.  Outputs of the arms are compared on one batch.
  gather:  mac_kb_gather (bf16 and fp32 out) at the CLEVR shape, U = 8 and 16, against mac_cast_bf16 of the B per-question
           rows, CUDA events around 30 back-to-back launches, with the bytes each has to move over its time beside the
           H100's 3.35 TB/s of HBM bandwidth.
Records the card (name, power limit, max SM clock from nvidia-smi).  Writes OUT_DIR/shared_images_h100.json.  Fails without
a GPU."""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np
import torch

from mac_network_b200 import _lib as L
from mac_network_b200.config import MACConfig
from mac_network_b200.model import MACnet
from mac_network_b200.serving import ModelPipeline
from model_pipeline import A, E, HBM_TBS, MODELS, SHAPES, V, compare, device_info, timed

IMAGES = (16, 8)


def host_batches(sh, k, n=3, seed=0):
    """n batches of B questions over k distinct images each: the shared form (k images + index) and the duplicated one."""
    rng = np.random.RandomState(seed + k)
    B, S = sh["B"], sh["S"]
    out = []
    for _ in range(n):
        lengths = rng.randint(S // 2, S + 1, size=(B,)).astype(np.int32)
        lengths[0] = S
        q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
        q[np.arange(S)[None, :] >= lengths[:, None]] = 0
        img = np.maximum(rng.standard_normal((k, sh["C"], sh["H"], sh["W"])), 0).astype(np.float32)
        index = np.concatenate([np.arange(k), rng.randint(0, k, size=B - k)]).astype(np.int32)
        rng.shuffle(index)
        base = {"questions": torch.from_numpy(q).pin_memory(), "questionLengths": torch.from_numpy(lengths).pin_memory()}
        out.append({"shared": dict(base, images=torch.from_numpy(img).pin_memory(), imageIndex=torch.from_numpy(index)),
                    "dup": dict(base, images=torch.from_numpy(np.ascontiguousarray(img[index])).pin_memory())})
    return out


def pipeline_arm(pipe, batches):
    def go(n):
        for i in range(n):
            pipe.submit(batches[i % len(batches)], next_batch=batches[(i + 1) % len(batches)])
        pipe.drain()
    return go


def gather_part(sh, rounds, iters=30):
    lib = L.load()
    B, N, d = sh["B"], sh["H"] * sh["W"], 512
    s = L.stream_ptr()
    kb = torch.randn(B, N, d, device="cuda")
    kb16 = torch.empty(B, N, d, dtype=torch.bfloat16, device="cuda")
    kb32 = torch.empty(B, N, d, device="cuda")
    fns = {"cast_bf16_B_rows": (lambda: L.check(lib.mac_cast_bf16(L.ptr(kb), L.ptr(kb16), kb.numel(), s)), B * N * d * 6)}
    for U in IMAGES:
        ku = kb[:U].contiguous()
        idx = torch.from_numpy(np.random.RandomState(U).randint(0, U, size=B).astype(np.int32)).cuda()
        idx[:U] = torch.arange(U, dtype=torch.int32, device="cuda")
        fns["gather_bf16_U%d" % U] = ((lambda ku=ku, idx=idx, U=U: L.check(lib.mac_kb_gather(
            L.ptr(ku), L.ptr(idx), L.ptr(kb16), 1, B, U, N, d, s))), U * N * d * 4 + B * N * d * 2)
        fns["gather_fp32_U%d" % U] = ((lambda ku=ku, idx=idx, U=U: L.check(lib.mac_kb_gather(
            L.ptr(ku), L.ptr(idx), L.ptr(kb32), 0, B, U, N, d, s))), U * N * d * 4 + B * N * d * 4)
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
    out["note"] = ("B=%d, N=%d, d=%d.  min_bytes: U*N*d*4 read + B*N*d*{2,4} written for the gather (repeated rows come from "
                   "L2), B*N*d*(4+2) for the cast.  The bound is HBM bandwidth, %.2f TB/s on the data sheet of a 700 W card"
                   % (B, N, d, HBM_TBS))
    return out


def max_rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--shapes", default="clevr,gqa")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("shared_images.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    os.makedirs(a.out_dir, exist_ok=True)
    out = {"device": device_info(), "rounds": a.rounds, "window_s": a.window, "slots": 4, "copies": "fp32, no host cast",
           "gather": gather_part(SHAPES["clevr"], a.rounds), "shapes": {}}
    print(json.dumps({"gather": out["gather"]}), flush=True)
    for name in a.shapes.split(","):
        sh = SHAPES[name]
        cfg = MACConfig.args(sh["variant"], netLength=sh["L"])
        shape = (sh["B"], sh["S"], sh["H"], sh["W"])
        data = {k: host_batches(sh, k) for k in IMAGES}
        res = {"shape": sh, "models": {}}
        for mname, mkw in MODELS.items():
            net = MACnet(cfg, sh["L"], V, A, wrd_emb_dim=E, image_in_dim=sh["C"], classifier_dims=(512,), seed=7, **mkw)
            pipes = {"images_None_duplicated": ModelPipeline(net, shape, slots=4, host_cast=False)}
            arms = {"images_None_duplicated": pipeline_arm(pipes["images_None_duplicated"], [b["dup"] for b in data[8]])}
            for k in IMAGES:
                key = "images_%d" % k
                pipes[key] = ModelPipeline(net, shape, slots=4, host_cast=False, images=k)
                arms[key] = pipeline_arm(pipes[key], [b["shared"] for b in data[k]])
            # the arms' outputs on one batch of 8 images: the dup arm against images=8 and images=16 (k = 8 < U)
            ref = {kk: v.clone() for kk, v in pipes["images_None_duplicated"].result(
                pipes["images_None_duplicated"].submit(data[8][0]["dup"])).items()}
            agree = {}
            for k in IMAGES:
                got = pipes["images_%d" % k].result(pipes["images_%d" % k].submit(data[8][0]["shared"]))
                agree["images_%d" % k] = {kk: ("bit_equal" if torch.equal(got[kk], ref[kk]) else max_rel(got[kk], ref[kk]))
                                          for kk in ("logits", "memory", "att_kb", "att_question")}
            for p in pipes.values():
                p.drain()
            r = compare(arms, a.rounds, a.window)
            base = r["images_None_duplicated"]["batches_per_s"]
            for key, v in r.items():
                v["questions_per_s"] = v["batches_per_s"] * sh["B"]
                v["h2d_bytes_per_batch"] = pipes[key].h2d_bytes
                v["h2d_gb_per_s"] = pipes[key].h2d_bytes * v["batches_per_s"] / 1e9
                v["speedup_over_duplicated"] = v["batches_per_s"] / base
            res["models"][mname] = {"arms": r, "outputs_against_duplicated": agree}
            print(json.dumps({name: {mname: res["models"][mname]}}), flush=True)
            del pipes, arms, net
            torch.cuda.empty_cache()
        out["shapes"][name] = res
    path = os.path.join(a.out_dir, "shared_images_h100.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out["device"]))


if __name__ == "__main__":
    main()
