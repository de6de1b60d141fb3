"""The e4m3 inference stem (Stem(prec="fp8"), csrc/tc_gemm_fp8.cuh) against the bf16 one, alone and inside the whole-model
evaluation.  Usage:  python profiles/stem_fp8.py OUT_DIR [--rounds 5] [--window 0.5]

  stem:    Stem.forward at B=64, 14x14, 1024 -> 512 -> 512 (177.6 GFLOP), bf16 and fp8 alternating `--rounds` times, every
           window at least `--window` seconds of CUDA events.
  parts:   each layer's patch matrix (mac_im2col3x3 bf16 / mac_im2col3x3_fp8) and GEMM (mac_linear_tc_fwd /
           mac_linear_fp8_fwd) on their own, CUDA events around 50 back-to-back launches, alternating.
  whole:   MACnet.runBatch(train=False) at the bench shape (B=64, S=40, 14x14, 1024 image channels, d=512, netLength=12),
           prec="fp8" with the bf16 stem against prec="fp8" with eval_stem_prec="fp8", alternating; the images are already
           on the device, so no host copy is timed.
Also records the card (name, power limit, max SM clock from nvidia-smi).  Writes OUT_DIR/stem_fp8_h100.json."""
import argparse
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from mac_network_b200 import _lib as L
from mac_network_b200.stem import Stem, init_stem_params, stem_specs

B, H, W, C_IN, C_OUT = 64, 14, 14, 1024, 512
PRECS = ("bf16", "fp8")


def device_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock, "torch_device": torch.cuda.get_device_name(0)}


def timed(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def compare(arms, rounds, window_s):
    """arms: name -> callable.  Warm up, size each window to >= window_s, alternate the arms `rounds` times (ms per call)."""
    iters = {}
    for name, fn in arms.items():
        for _ in range(2):
            fn()
        iters[name] = max(3, int(math.ceil(1.2 * window_s * 1e3 / timed(fn, 2))))
    rows = {name: [] for name in arms}
    for _ in range(rounds):
        for name, fn in arms.items():
            rows[name].append(timed(fn, iters[name]))
    return {name: {"ms": float(np.median(v)), "ms_min": min(v), "ms_max": max(v), "ms_rounds": [round(x, 4) for x in v],
                   "iters_per_window": iters[name], "window_s": round(iters[name] * min(v) / 1e3, 3)}
            for name, v in rows.items()}


def stem_part(rounds, window_s):
    p = {k: torch.from_numpy(v).cuda() for k, v in init_stem_params(stem_specs(C_IN, C_OUT), seed=5).items()}
    g = torch.Generator(device="cuda").manual_seed(6)
    images = torch.relu(torch.randn(B, H, W, C_IN, device="cuda", generator=g))
    stems = {pr: Stem(p, relu="ELU", prec=pr) for pr in PRECS}
    res = compare({pr: (lambda st=st: st.forward(images)) for pr, st in stems.items()}, rounds, window_s)
    M = B * H * W
    gflop = sum(2.0 * M * 9 * ci * co for ci, co in ((C_IN, C_OUT), (C_OUT, C_OUT))) / 1e9
    for r in res.values():
        r["tflops_algorithmic"] = gflop / r["ms"]
    out = {"shape": {"B": B, "H": H, "W": W, "dims": [C_IN, C_OUT, C_OUT]}, "gflop": gflop, "arms": res,
           "speedup_fp8": res["bf16"]["ms"] / res["fp8"]["ms"]}
    kb = {pr: stems[pr].forward(images) for pr in PRECS}
    torch.cuda.synchronize()
    out["fp8_vs_bf16_max_rel"] = float((kb["fp8"] - kb["bf16"]).abs().max() / kb["bf16"].abs().max())
    out["parts"] = parts(stems, images, rounds)
    return out


def parts(stems, images, rounds, iters=50):
    """Each layer's im2col and GEMM on their own, CUDA events around `iters` launches, the two precisions alternating."""
    lib = L.load()
    M = B * H * W
    s = L.stream_ptr()
    fns = {}
    keep = []
    x = images
    for i, (ci, co) in enumerate(((C_IN, C_OUT), (C_OUT, C_OUT))):
        K = 9 * ci
        b = stems["bf16"].p["stem/cnnLayercnn_%d/biases/bias" % i]
        _, Wt = stems["bf16"]._weights(i)
        _, (W8, sw) = stems["fp8"]._weights(i)
        cols16 = torch.empty((M, K), dtype=torch.bfloat16, device="cuda")
        cols8 = torch.empty((M, K), dtype=torch.uint8, device="cuda")
        sa = torch.empty(M, device="cuda")
        nb = lib.mac_im2col3x3_fp8_workspace_bytes(B, H, W, ci)
        ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
        y = torch.empty((M, co), device="cuda")
        keep += [cols16, cols8, sa, ws, y]
        fns["layer%d_im2col_bf16" % i] = lambda x=x, c=cols16, ci=ci: L.check(lib.mac_im2col3x3(
            L.ptr(x), L.ptr(c), 1, 1.0, 0, 32, 0, B, H, W, ci, s))
        fns["layer%d_im2col_fp8" % i] = lambda x=x, c=cols8, a=sa, w=ws, nb=nb, ci=ci: L.check(lib.mac_im2col3x3_fp8(
            L.ptr(x), L.ptr(c), L.ptr(a), L.ptr(w), nb, B, H, W, ci, s))
        fns["layer%d_gemm_bf16" % i] = lambda c=cols16, Wt=Wt, b=b, y=y, K=K, co=co: L.check(lib.mac_linear_tc_fwd(
            L.ptr(c), L.ptr(Wt), L.ptr(b), L.ACT["ELU"], L.ptr(y), 0, M, K, co, s))
        fns["layer%d_gemm_fp8" % i] = lambda c=cols8, a=sa, W8=W8, sw=sw, b=b, y=y, K=K, co=co: L.check(lib.mac_linear_fp8_fwd(
            L.ptr(c), L.ptr(a), L.ptr(W8), L.ptr(sw), L.ptr(b), L.ACT["ELU"], L.ptr(y), M, K, co, s))
        fns["layer%d_im2col_fp8" % i]()              # the fp8 GEMM's operands hold real data
        x = torch.nn.functional.elu(torch.randn(B, H, W, co, device="cuda"))
        keep.append(x)
    for fn in fns.values():
        fn()
    us = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            us[k].append(timed(fn, iters) * 1e3)
    out = {k: {"us": float(np.median(v)), "us_min": min(v), "us_max": max(v)} for k, v in us.items()}
    for i, (ci, co) in enumerate(((C_IN, C_OUT), (C_OUT, C_OUT))):
        fl = 2.0 * M * 9 * ci * co
        for pr in PRECS:
            out["layer%d_gemm_%s" % (i, pr)]["tflops"] = fl / out["layer%d_gemm_%s" % (i, pr)]["us"] / 1e6
        out["layer%d_patch_matrix_bytes" % i] = {"bf16": M * 9 * ci * 2, "fp8": M * 9 * ci}
    out["note"] = "CUDA events around %d back-to-back launches of one call; median / min / max over rounds" % iters
    return out


def whole_part(rounds, window_s):
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    from mac_network_b200.synthetic import SHAPES
    Bm, S, N, d, Ls = SHAPES["headline"]
    V, E, A = 90, 300, 28
    cfg = MACConfig.args("args", netLength=Ls)
    rng = np.random.RandomState(31)
    lengths = rng.randint(S // 2, S + 1, size=(Bm,)).astype(np.int32)
    lengths[0] = S
    q = rng.randint(1, V + 1, size=(Bm, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    data = {"questions": q, "questionLengths": lengths, "answers": rng.randint(0, A, size=(Bm,)).astype(np.int32)}
    images = {"images": torch.relu(torch.randn(Bm, C_IN, H, W, device="cuda"))}
    kw = dict(wrd_emb_dim=E, image_in_dim=C_IN, classifier_dims=(512,), seed=7, prec="fp8")
    nets = {"fp8_cell_bf16_stem": MACnet(cfg, Ls, V, A, **kw), "fp8_cell_fp8_stem": MACnet(cfg, Ls, V, A, eval_stem_prec="fp8", **kw)}
    res = compare({k: (lambda n=n: n.runBatch(None, data, images, train=False)) for k, n in nets.items()}, rounds, window_s)
    preds = {k: [p["prediction"] for p in n.runBatch(None, data, images, train=False)["preds"]] for k, n in nets.items()}
    agree = float(np.mean(np.array(preds["fp8_cell_bf16_stem"]) == np.array(preds["fp8_cell_fp8_stem"])))
    return {"shape": {"B": Bm, "S": S, "N": N, "d": d, "L": Ls, "image_channels": C_IN}, "arms": res,
            "saved_ms": res["fp8_cell_bf16_stem"]["ms"] - res["fp8_cell_fp8_stem"]["ms"],
            "speedup_fp8_stem": res["fp8_cell_bf16_stem"]["ms"] / res["fp8_cell_fp8_stem"]["ms"],
            "prediction_agreement": agree,
            "note": "MACnet.runBatch(train=False) per call (images resident on the device); median / min / max over rounds"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stem_fp8.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    os.makedirs(a.out_dir, exist_ok=True)
    out = {"device": device_info(), "rounds": a.rounds}
    out["stem"] = stem_part(a.rounds, a.window)
    print(json.dumps({"stem": out["stem"]}), flush=True)
    torch.cuda.empty_cache()
    out["whole_model"] = whole_part(a.rounds, a.window)
    path = os.path.join(a.out_dir, "stem_fp8_h100.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
