"""The location-aware stem (--locationAware, L and PE) against the location-free stem.
Usage:  python profiles/stem_location.py OUT_DIR [--rounds 5] [--window 1.0]

  stem:      Stem.forward (keep 1) and Stem.forward(save_for_backward=True, keep 0.82) + Stem.backward (no image gradient)
             at B=64, 14x14, 1024 -> 512 -> 512, in bf16 and bf16x3, with no location, L (l = 2) and PE (l = 128).
  kernels:   at the same layer-0 shape, each location step alone: the location patches (mac_loc_cols bf16 / split), the
             location GEMM Q W_loc + b (mac_linear_tc_fwd / _tc32_fwd, K = Kq), the image GEMM with the _acc epilogue
             against the same GEMM without it, and the location weight gradient (mac_loc_cols_t + the split-K wgrad, as the
             difference of mac_conv_bwd_loc_tc and mac_conv_bwd_tc).
  pipeline:  ModelPipeline per-batch time at the CLEVR serving shape (B=64, S=40, L=12, prec="bf16") with and without L.
Arms of a comparison alternate in one process, `--rounds` times each, windows of at least `--window` seconds, after a
warm-up of every arm; medians are reported with each round, and the card (name, power limit, max SM clock).  Fails without
a GPU.  Writes OUT_DIR/stem_location.json."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from mac_network_b200 import _lib as L
from mac_network_b200 import packs
from mac_network_b200.config import MACConfig
from mac_network_b200.model import MACnet
from mac_network_b200.serving import ModelPipeline
from mac_network_b200.stem import SITE_LOCATION, SITE_STEM, Stem, init_stem_params, location_width, stem_specs
from profiles import model_pipeline as mp
from profiles.stem_train_tc import B, C_IN, C_OUT, H, KEEP, W, compare, device_info

LOCS = {"none": None, "L": ("L", 1.0, 32), "PE": ("PE", 1.0, 32)}


def stem_part(rounds, window_s):
    g = torch.Generator(device="cuda").manual_seed(6)
    images = torch.relu(torch.randn(B, H, W, C_IN, device="cuda", generator=g))
    d_kb = torch.randn(B, H * W, C_OUT, device="cuda", generator=g) * 1e-3
    arms = {}
    for lname, loc in LOCS.items():
        params = {k: torch.from_numpy(v).cuda() for k, v in init_stem_params(stem_specs(C_IN, C_OUT, location=loc),
                                                                             seed=5).items()}
        for prec in ("bf16", "bf16x3"):
            st = Stem(params, relu="ELU", prec=prec, seed=11, location=loc)
            grads = {k: torch.zeros_like(v) for k, v in params.items()}

            def train(st=st, grads=grads):
                st.forward(images, keep=KEEP, step=3, save_for_backward=True)
                st.backward(d_kb, grads)
            arms["%s/%s/forward" % (lname, prec)] = (lambda st=st: st.forward(images))
            arms["%s/%s/forward_backward" % (lname, prec)] = train
    return compare(arms, rounds, window_s)


def kernel_part(rounds, window_s):
    lib = L.load()
    sp = L.stream_ptr
    g = torch.Generator(device="cuda").manual_seed(7)
    M, K = B * H * W, 9 * C_IN
    x = torch.relu(torch.randn(B, H, W, C_IN, device="cuda", generator=g))
    P16 = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    P3 = torch.randn(M, 2 * K, device="cuda", generator=g).to(torch.bfloat16)
    W_img = torch.randn(K, C_OUT, device="cuda", generator=g) * 0.01
    Wi16, Wi3 = packs.bf16(W_img, sp()), packs.split3(W_img, sp())
    b = torch.zeros(C_OUT, device="cuda")
    y = torch.zeros(M, C_OUT, device="cuda")
    dy = torch.randn(M, C_OUT, device="cuda", generator=g) * 1e-3
    arms = {
        "image_gemm/bf16": lambda: L.check(lib.mac_linear_tc_fwd(L.ptr(P16), L.ptr(Wi16), L.ptr(b), 3, L.ptr(y), 0, M, K,
                                                                 C_OUT, sp())),
        "image_gemm_acc/bf16": lambda: L.check(lib.mac_linear_tc_fwd_acc(L.ptr(P16), L.ptr(Wi16), 3, L.ptr(y), M, K, C_OUT,
                                                                         sp())),
        "image_gemm/bf16x3": lambda: L.check(lib.mac_linear_tc32_fwd(L.ptr(P3), L.ptr(Wi3), L.ptr(b), 3, L.ptr(y), M, K,
                                                                     C_OUT, sp())),
        "image_gemm_acc/bf16x3": lambda: L.check(lib.mac_linear_tc32_fwd_acc(L.ptr(P3), L.ptr(Wi3), 3, L.ptr(y), M, K,
                                                                             C_OUT, sp())),
    }
    for lname, loc in (("L", LOCS["L"]), ("PE", LOCS["PE"])):
        st = Stem({k: torch.from_numpy(v).cuda() for k, v in init_stem_params(stem_specs(C_IN, C_OUT, location=loc),
                                                                               seed=5).items()}, location=loc)
        grid, l = st.location_grid(H, W), st.nloc
        Kq = location_width(l, 3)
        W_loc = torch.randn(Kq, C_OUT, device="cuda", generator=g) * 0.01
        Wl16, Wl3 = packs.bf16(W_loc, sp()), packs.split3(W_loc, sp())
        q16 = torch.empty(M, Kq, dtype=torch.bfloat16, device="cuda")
        q3 = torch.empty(M, 2 * Kq, dtype=torch.bfloat16, device="cuda")
        arms["loc_cols/bf16/" + lname] = (lambda q16=q16, grid=grid, l=l: L.check(lib.mac_loc_cols(
            L.ptr(grid), L.ptr(q16), 1, KEEP, 1, SITE_LOCATION, 2, B, H, W, l, 3, 1, sp())))
        arms["loc_cols/split/" + lname] = (lambda q3=q3, grid=grid, l=l: L.check(lib.mac_loc_cols(
            L.ptr(grid), L.ptr(q3), 2, KEEP, 1, SITE_LOCATION, 2, B, H, W, l, 3, 1, sp())))
        arms["loc_gemm/bf16/" + lname] = (lambda q16=q16, Wl16=Wl16, Kq=Kq: L.check(lib.mac_linear_tc_fwd(
            L.ptr(q16), L.ptr(Wl16), L.ptr(b), 0, L.ptr(y), 0, M, Kq, C_OUT, sp())))
        arms["loc_gemm/bf16x3/" + lname] = (lambda q3=q3, Wl3=Wl3, Kq=Kq: L.check(lib.mac_linear_tc32_fwd(
            L.ptr(q3), L.ptr(Wl3), L.ptr(b), 0, L.ptr(y), M, Kq, C_OUT, sp())))
        for prec, suffix in (("bf16", "tc"), ("bf16x3", "tc32")):
            nb = int(getattr(lib, "mac_conv_bwd_loc_%s_workspace_bytes" % suffix)(B, H, W, C_IN, C_OUT, l, 3, 1, 0))
            ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
            dk = torch.zeros(K, C_OUT, device="cuda")
            dwl = torch.zeros(Kq, C_OUT, device="cuda")
            db = torch.zeros(C_OUT, device="cuda")
            arms["conv_bwd_loc/%s/%s" % (prec, lname)] = (
                lambda f=getattr(lib, "mac_conv_bwd_loc_" + suffix), ws=ws, nb=nb, dk=dk, dwl=dwl, db=db, grid=grid, l=l:
                L.check(f(L.ptr(x), L.ptr(y), L.ptr(dy), L.ptr(W_img), 3, KEEP, 1, SITE_STEM, 2, L.ptr(grid), l, SITE_LOCATION,
                          L.ptr(dk), L.ptr(dwl), L.ptr(db), None, L.ptr(ws), nb, B, H, W, C_IN, C_OUT, 3, 1, sp())))
    for prec, suffix in (("bf16", "tc"), ("bf16x3", "tc32")):
        nb = int(getattr(lib, "mac_conv_bwd_%s_workspace_bytes" % suffix)(B, H, W, C_IN, C_OUT, 3, 1, 0))
        ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
        dk = torch.zeros(K, C_OUT, device="cuda")
        db = torch.zeros(C_OUT, device="cuda")
        arms["conv_bwd/%s" % prec] = (
            lambda f=getattr(lib, "mac_conv_bwd_" + suffix), ws=ws, nb=nb, dk=dk, db=db:
            L.check(f(L.ptr(x), L.ptr(y), L.ptr(dy), L.ptr(W_img), 3, KEEP, 1, SITE_STEM, 2, L.ptr(dk), L.ptr(db), None,
                      L.ptr(ws), nb, B, H, W, C_IN, C_OUT, 3, 1, sp())))
    res = compare(arms, rounds, window_s)
    for lname in ("L", "PE"):
        for prec in ("bf16", "bf16x3"):
            res["loc_wgrad/%s/%s (difference)" % (prec, lname)] = {
                "ms": res["conv_bwd_loc/%s/%s" % (prec, lname)]["ms"] - res["conv_bwd/%s" % prec]["ms"]}
    return res


def pipeline_part(rounds, window_s):
    sh = mp.SHAPES["clevr"]
    cfg = MACConfig.args(sh["variant"], netLength=sh["L"])
    batches = mp.host_batches(sh)
    arms = {}
    for name, kw in (("none", {}), ("L", dict(stem_location="L"))):
        net = MACnet(cfg, sh["L"], mp.V, mp.A, wrd_emb_dim=mp.E, image_in_dim=sh["C"], classifier_dims=(512,), seed=7,
                     prec="bf16", **kw)
        pipe = ModelPipeline(net, (sh["B"], sh["S"], sh["H"], sh["W"]), slots=2)
        arms[name] = mp.pipeline_arm(pipe, batches)
    return {"shape": sh, "arms": mp.compare(arms, rounds, window_s)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=1.0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stem_location.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    os.makedirs(a.out_dir, exist_ok=True)
    out = {"device": device_info(), "rounds": a.rounds, "window_s": a.window,
           "shape": {"B": B, "H": H, "W": W, "dims": [C_IN, C_OUT, C_OUT], "keep_train": KEEP},
           "stem": stem_part(a.rounds, a.window), "kernels": kernel_part(a.rounds, a.window),
           "pipeline": pipeline_part(a.rounds, a.window)}
    path = os.path.join(a.out_dir, "stem_location.json")
    with open(path, "w") as fh:
        json.dump(out, fh, indent=1, sort_keys=True)
    print(json.dumps(out["device"]))
    for sec in ("stem", "kernels"):
        for k, r in sorted(out[sec].items()):
            print("%-44s %8.4f ms %s" % (k, r["ms"], r.get("ms_rounds", "")))
    for k, r in out["pipeline"]["arms"].items():
        print("pipeline %-6s %8.3f ms/batch %s" % (k, r["ms_per_batch"], r.get("ms_rounds", "")))


if __name__ == "__main__":
    main()
