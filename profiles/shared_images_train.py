"""Several questions per image in training: serving.TrainPipeline(images=U) against the pipeline fed one copy of the image
per question.  Usage:  python profiles/shared_images_train.py OUT_DIR [--rounds 5] [--window 1.0]

  arms:    at the CLEVR training shape (B=64, S=40 with question lengths mixed in 20..40, 1024x14x14, d=512, L=12), for
           "all_tc" (prec="bf16", bwd_tc=True, bf16 stem and encoder) and "tc32" (the parity form, bf16x3 stem):
           images=None over the duplicated features (B images per batch), images=16 and images=8 (16 or 8 distinct images per
           batch and each question's index), each over numpy batches and over batches whose images are pinned tensors.
           One process, the arms alternating `--rounds` times, every window at least `--window` seconds of host clock ending
           in a synchronise, the inputs rotating over three host batches.  Each arm reads a step's result after the next
           submit, as a training loop would.  The arms share one model: every step trains it, which does not change the
           work a step does.
  kernels: CUDA events around 30 back-to-back launches, medians of `--rounds`: mac_kb_gather_bwd at B=64, N=196, d=512 and
           U = 8, 16, with the bytes it has to move over its time beside the H100's 3.35 TB/s of HBM bandwidth; the stem's
           training forward (forward_nchw, keep 0.82, save) plus backward over 8, 16 and 64 images, bf16 and bf16x3.
Records the card (name, power limit, max SM clock from nvidia-smi).  Writes OUT_DIR/shared_images_train_h100.json.  Fails
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
from profiles.train_pipeline import A, CONFIGS, E, KEEP, SHAPE, V, host_batches, pipeline_arm

IMAGES = (16, 8)


def shared_batches(batches, k, seed):
    """The batches with k distinct images: the first k of each batch's images, every one asked about, the others at random."""
    rng = np.random.RandomState(seed)
    out = []
    for b in batches:
        B = b["questions"].shape[0]
        idx = rng.randint(0, k, size=B).astype(np.int32)
        idx[rng.permutation(B)[:k]] = np.arange(k)
        out.append(dict(b, images=np.ascontiguousarray(b["images"][:k]), imageIndex=idx))
    return out


def duplicated(batches):
    """What a caller without an index feeds: each question's image, copied once per question."""
    return [dict({k: v for k, v in b.items() if k != "imageIndex"}, images=np.ascontiguousarray(b["images"][b["imageIndex"]]))
            for b in batches]


def pinned(batches):
    return [dict(b, images=torch.from_numpy(b["images"]).pin_memory()) for b in batches]


def summed(us):
    med = float(np.median(us))
    return {"us": med, "us_min": min(us), "us_max": max(us)}


def kernel_part(sh, rounds, iters=30):
    lib = L.load()
    B, N, d = sh["B"], sh["H"] * sh["W"], 512
    g = torch.randn(B, N, d, device="cuda")
    s = L.stream_ptr()
    out = {}
    for U in sorted(IMAGES):
        rng = np.random.RandomState(U)
        pat = rng.randint(0, U, size=B)
        pat[rng.permutation(B)[:U]] = np.arange(U)
        idx = torch.from_numpy(pat.astype(np.int32)).cuda()
        dst = torch.empty(U, N, d, device="cuda")
        fn = lambda: L.check(lib.mac_kb_gather_bwd(L.ptr(g), L.ptr(idx), L.ptr(dst), B, U, N, d, s), "mac_kb_gather_bwd")
        fn()
        r = summed([timed(fn, iters) for _ in range(rounds)])
        nbytes = B * N * d * 4 + U * N * d * 4 + B * 4
        r.update(min_bytes=nbytes, tb_per_s_of_min_bytes=nbytes / r["us"] / 1e6,
                 share_of_hbm_bound=nbytes / r["us"] / 1e6 / HBM_TBS)
        out["kb_gather_bwd_U%d" % U] = r
    out["note"] = ("B=%d, N=%d, d=%d.  min_bytes: every question row read once, every image row written once, the index.  The "
                   "%.1f MB of question rows fit in the H100's 50 MB L2 and back-to-back launches read the same ones, so the "
                   "operands are largely L2-resident: tb_per_s_of_min_bytes beside HBM's %.2f TB/s (the data sheet of a 700 W "
                   "card) is an upper-bound comparison, not a measured HBM rate" % (B, N, d, B * N * d * 4 / 1e6, HBM_TBS))
    return out


def stem_part(cfg, sh, rounds, iters=30):
    """Forward (training ingest + both layers, saved) plus backward of the stem alone, over n images."""
    from mac_network_b200.stem import Stem, init_stem_params, stem_specs
    p = {k: torch.from_numpy(v).cuda() for k, v in init_stem_params(stem_specs(sh["C"], cfg.memDim), seed=3).items()}
    out = {}
    for prec in ("bf16", "bf16x3"):
        st = Stem(p, relu="ELU", prec=prec, seed=5)
        grads = {k: torch.zeros_like(v) for k, v in p.items()}
        for n in (8, 16, sh["B"]):
            x = torch.relu(torch.randn(n, sh["C"], sh["H"], sh["W"], device="cuda"))
            d_kb = torch.randn(n, sh["H"] * sh["W"], cfg.memDim, device="cuda")

            def fn():
                st.forward_nchw(x, keep=KEEP, step=1, save_for_backward=True)
                st.backward(d_kb, grads)
            fn()
            out["%s_images%d" % (prec, n)] = summed([timed(fn, iters) for _ in range(rounds)])
        del st
        torch.cuda.empty_cache()
    out["note"] = "keep %.2f; 1024 -> 512 -> 512 channels, 3x3, 14x14; no image gradient (as in training)" % KEEP
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("shared_images_train.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    os.makedirs(a.out_dir, exist_ok=True)
    sh = SHAPE
    cfg = MACConfig.args(sh["variant"], netLength=sh["L"])
    out = {"device": device_info(), "rounds": a.rounds, "window_s": a.window, "shape": sh, "stem_dropout": KEEP,
           "kernels": kernel_part(sh, a.rounds), "stem_fwd_bwd": stem_part(cfg, sh, a.rounds), "configs": {}}
    print(json.dumps({"kernels": out["kernels"], "stem_fwd_bwd": out["stem_fwd_bwd"]}), flush=True)
    base = host_batches(sh)
    per_u = {U: shared_batches(base, U, seed=U) for U in IMAGES}
    # the unshared arm trains on the features of the 8-image batches, each question's image copied out
    dup = duplicated(per_u[8])
    for name in a.configs.split(","):
        net = MACnet(cfg, sh["L"], V, A, wrd_emb_dim=E, image_in_dim=sh["C"], classifier_dims=(512,), seed=7, prec="bf16",
                     **CONFIGS[name])
        shape = (sh["B"], sh["S"], sh["H"], sh["W"])
        pipes = {None: TrainPipeline(net, shape, depth=2)}
        pipes.update({U: TrainPipeline(net, shape, depth=2, images=U) for U in IMAGES})
        arms = {"images_None_numpy": pipeline_arm(pipes[None], dup), "images_None_pinned": pipeline_arm(pipes[None], pinned(dup))}
        for U in IMAGES:
            arms["images_%d_numpy" % U] = pipeline_arm(pipes[U], per_u[U])
            arms["images_%d_pinned" % U] = pipeline_arm(pipes[U], pinned(per_u[U]))
        r = compare(arms, a.rounds, a.window)
        for k, v in r.items():
            ref = r["images_None_" + k.rsplit("_", 1)[1]]["ms_per_batch"]
            v["questions_per_s"] = v["batches_per_s"] * sh["B"]
            v["speedup_over_images_None"] = ref / v["ms_per_batch"]
        out["configs"][name] = {"trainer": CONFIGS[name], "arms": r}
        print(json.dumps({name: out["configs"][name]}), flush=True)
        del pipes, arms, net
        torch.cuda.empty_cache()
    path = os.path.join(a.out_dir, "shared_images_train_h100.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out["device"]))


if __name__ == "__main__":
    main()
