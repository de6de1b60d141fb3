"""The image stem at the reference's other geometries (--stemKernelSize(s), --stemStrideSizes, --stemLinear) against the
default 3x3 stride-1 stem.  Usage:  python profiles/stem_geometry.py OUT_DIR [--rounds 5] [--window 0.4]

  stem:      Stem.forward (keep 1) and Stem.forward(save_for_backward=True, keep 0.82) + Stem.backward (no image gradient)
             at B=64, 14x14, 1024 -> 512 -> 512, in bf16 and bf16x3, for 3x3/1 (the 3x3 kernels), 1x1, 3x3 stride 2 on
             layer 0, and the linear stem (one 1024 -> 512 layer).
  patches:   each general patch pass (mac_im2col fp32 / bf16 / split, mac_im2col_t bf16 / split, mac_col2im) on its own at
             the stem's layer-0 shape, with the bytes it must move (every input element read once, every output element
             written once) over its time, as a share of the H100 SXM data-sheet 3.35 TB/s.
  pipeline:  ModelPipeline per-batch time at the CLEVR serving shape (B=64, S=40, L=12, prec="bf16") with the stride-2 stem
             against the default stem.
Arms of a comparison alternate in one process, `--rounds` times each, after a warm-up of every arm; medians are reported,
with the card (name, power limit, max SM clock).  Fails without a GPU.  Writes OUT_DIR/stem_geometry.json."""
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
from mac_network_b200.serving import ModelPipeline
from mac_network_b200.stem import SITE_STEM, Stem, init_stem_params, stem_grid, stem_specs
from profiles import model_pipeline as mp
from profiles.stem_train_tc import B, C_IN, C_OUT, H, KEEP, W, compare, device_info

HBM_TBPS = 3.35
GEOMS = {"3x3_s1": dict(ksizes=[3, 3], strides=[1, 1]), "1x1": dict(ksizes=[1, 1], strides=[1, 1]),
         "3x3_s2": dict(ksizes=[3, 3], strides=[2, 1]), "linear": dict(linear=True, strides=[1])}


def stem_part(rounds, window_s):
    g = torch.Generator(device="cuda").manual_seed(6)
    images = torch.relu(torch.randn(B, H, W, C_IN, device="cuda", generator=g))
    arms = {}
    for gname, gm in GEOMS.items():
        linear = gm.get("linear", False)
        specs = stem_specs(C_IN, C_OUT, ksizes=gm.get("ksizes"), linear=linear)
        params = {k: torch.from_numpy(v).cuda() for k, v in init_stem_params(specs, seed=5).items()}
        for prec in ("bf16", "bf16x3"):
            st = Stem(params, relu="ELU", prec=prec, seed=11, strides=gm["strides"], linear=linear)
            Ho, Wo = st.grid(H, W)
            d_kb = torch.randn(B, Ho * Wo, C_OUT, device="cuda", generator=g) * 1e-3
            grads = {k: torch.zeros_like(v) for k, v in params.items()}

            def train(st=st, d_kb=d_kb, grads=grads):
                st.forward(images, keep=KEEP, step=3, save_for_backward=True)
                st.backward(d_kb, grads)

            arms["%s/%s/forward" % (gname, prec)] = (lambda st=st: st.forward(images))
            arms["%s/%s/forward_backward" % (gname, prec)] = train
    return compare(arms, rounds, window_s)


def patch_part(rounds, window_s):
    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.relu(torch.randn(B, H, W, C_IN, device="cuda", generator=g))
    arms, nbytes = {}, {}
    for (k, s) in ((1, 1), (3, 2), (5, 1)):
        Ho, Wo = stem_grid(H, W, [s])
        M, K = B * Ho * Wo, k * k * C_IN
        Mp = (M + 63) // 64 * 64
        xin = x.numel() * 4
        for form, name, esz, wide in ((0, "f32", 4, 1), (1, "bf16", 2, 1), (2, "split", 2, 2)):
            cols = torch.empty(M * K * wide, dtype=torch.float32 if form == 0 else torch.bfloat16, device="cuda")
            key = "mac_im2col/%s/k%d_s%d" % (name, k, s)
            arms[key] = (lambda cols=cols, form=form, k=k, s=s: L.check(lib.mac_im2col(
                L.ptr(x), L.ptr(cols), form, KEEP, 1, SITE_STEM, 2, B, H, W, C_IN, k, s, L.stream_ptr())))
            nbytes[key] = xin + M * K * wide * esz
        for split in (0, 1):
            colsT = torch.empty(K * Mp * (2 if split else 1), dtype=torch.bfloat16, device="cuda")
            key = "mac_im2col_t/%s/k%d_s%d" % ("split" if split else "bf16", k, s)
            arms[key] = (lambda colsT=colsT, split=split, k=k, s=s: L.check(lib.mac_im2col_t(
                L.ptr(x), L.ptr(colsT), split, KEEP, 1, SITE_STEM, 2, B, H, W, C_IN, k, s, L.stream_ptr())))
            nbytes[key] = xin + K * Mp * (2 if split else 1) * 2
        dcols = torch.randn(M * K, device="cuda", generator=g)
        dx = torch.empty_like(x)
        key = "mac_col2im/k%d_s%d" % (k, s)
        arms[key] = (lambda dcols=dcols, k=k, s=s: L.check(lib.mac_col2im(
            L.ptr(dcols), L.ptr(dx), KEEP, 1, SITE_STEM, 2, B, H, W, C_IN, k, s, L.stream_ptr())))
        nbytes[key] = M * K * 4 + xin
    res = compare(arms, rounds, window_s)
    for key, r in res.items():
        r["bytes"] = nbytes[key]
        r["tb_per_s"] = nbytes[key] / (r["ms"] * 1e-3) / 1e12
        r["share_of_3.35TBps"] = r["tb_per_s"] / HBM_TBPS
    return res


def pipeline_part(rounds, window_s):
    sh = mp.SHAPES["clevr"]
    cfg = MACConfig.args(sh["variant"], netLength=sh["L"])
    batches = mp.host_batches(sh)
    arms = {}
    for name, geom in (("default", {}), ("stride2", dict(stem_kernel_sizes=[3, 3], stem_strides=[2, 1]))):
        net = MACnet(cfg, sh["L"], mp.V, mp.A, wrd_emb_dim=mp.E, image_in_dim=sh["C"], classifier_dims=(512,), seed=7,
                     prec="bf16", **geom)
        pipe = ModelPipeline(net, (sh["B"], sh["S"], sh["H"], sh["W"]), slots=2)
        arms[name] = mp.pipeline_arm(pipe, batches)
    return {"shape": sh, "arms": mp.compare(arms, rounds, window_s)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stem_geometry.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    os.makedirs(a.out_dir, exist_ok=True)
    out = {"device": device_info(), "rounds": a.rounds, "window_s": a.window,
           "shape": {"B": B, "H": H, "W": W, "dims": [C_IN, C_OUT, C_OUT], "keep_train": KEEP},
           "stem": stem_part(a.rounds, a.window), "patches": patch_part(a.rounds, a.window),
           "pipeline": pipeline_part(a.rounds, 1.0)}
    path = os.path.join(a.out_dir, "stem_geometry.json")
    with open(path, "w") as fh:
        json.dump(out, fh, indent=1, sort_keys=True)
    print(json.dumps({k: out[k] for k in ("device",)}))
    for sec in ("stem", "patches"):
        for k, r in sorted(out[sec].items()):
            print("%-40s %8.3f ms%s" % (k, r["ms"], "  %.2f TB/s" % r["tb_per_s"] if "tb_per_s" in r else ""))
    for k, r in out["pipeline"]["arms"].items():
        print("pipeline %-10s %8.3f ms/batch" % (k, r["ms_per_batch"]))


if __name__ == "__main__":
    main()
