"""The split-bf16 image stem (Stem(prec="bf16x3")) against the fp32 and the bf16 stem, on its own and inside the whole-model
training step with the cell in split bf16 too.  Usage:  python profiles/stem_train_bf16x3.py OUT_DIR [--rounds 5] [--window 0.4]

  forward:  Stem.forward at B=64, 14x14, 1024 -> 512 -> 512, keep 0.82 (177.6 GFLOP).
  train:    Stem.forward(save_for_backward=True) + Stem.backward, the image gradient not asked for (414.3 GFLOP).
  parts:    each layer's patch pass (mac_im2col3x3 fp32 / bf16, mac_im2col3x3_split) and GEMM (mac_linear_fwd,
            mac_linear_tc_fwd, mac_linear_tc32_fwd) on their own.
  whole:    DPTrainer.train_step_full at the bench.py train_full shape, the cell at prec="tc32", bwd_tc=True in every arm,
            stem_prec "fp32", "bf16x3" and "bf16": the difference is the stem alone.
The arms of a comparison alternate in one process, `--rounds` times each, after a warm-up of every arm, every window at
least `--window` seconds of CUDA events.  Also reports the max-rel agreement of the bf16x3 and bf16 stem gradients with the
fp32 ones at this size, and the card (name, power limit, max SM clock: nvidia-smi queries).  Fails without a GPU.
Writes OUT_DIR/stem_train_bf16x3.json."""
import argparse
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from mac_network_b200 import _lib as L
from mac_network_b200.config import MACConfig
from mac_network_b200.dp import DPTrainer
from mac_network_b200.stem import SITE_STEM, Stem, init_stem_params, stem_specs
from mac_network_b200.synthetic import SHAPES
from profiles.stem_train_tc import B, C_IN, C_OUT, H, KEEP, W, compare, device_info, stem_gflop

PRECS = ("fp32", "bf16x3", "bf16")


def _rates(res, gflop):
    for r in res.values():
        r["tflops_algorithmic"] = gflop / r["ms"]
    return res


def stem_part(rounds, window_s):
    params = {k: torch.from_numpy(v).cuda() for k, v in init_stem_params(stem_specs(C_IN, C_OUT), seed=5).items()}
    g = torch.Generator(device="cuda").manual_seed(6)
    images = torch.relu(torch.randn(B, H, W, C_IN, device="cuda", generator=g))
    d_kb = torch.randn(B, H * W, C_OUT, device="cuda", generator=g) * 1e-3
    stems = {p: Stem(params, relu="ELU", prec=p, seed=11) for p in PRECS}
    grads = {p: {k: torch.zeros_like(v) for k, v in params.items()} for p in PRECS}

    def step(p):
        stems[p].forward(images, keep=KEEP, step=3, save_for_backward=True)
        stems[p].backward(d_kb, grads[p])

    for p in PRECS:                                  # agreement: from zeroed gradients, the same masks (seed, site, step)
        step(p)
    torch.cuda.synchronize()
    agree = {p: {k: float((grads[p][k] - grads["fp32"][k]).abs().max() / grads["fp32"][k].abs().max()) for k in params}
             for p in PRECS[1:]}
    dims = [C_IN, C_OUT, C_OUT]
    M = B * H * W
    fwd_gf = sum(2.0 * M * 9 * dims[i] * dims[i + 1] for i in range(2)) / 1e9
    out = {"shape": {"B": B, "H": H, "W": W, "dims": dims, "keep": KEEP},
           "forward": {"gflop": fwd_gf, "arms": _rates(compare(
               {p: (lambda p=p: stems[p].forward(images, keep=KEEP, step=3)) for p in PRECS}, rounds, window_s), fwd_gf)},
           "train": {"gflop": stem_gflop(B, H, W, dims), "arms": _rates(compare(
               {p: (lambda p=p: step(p)) for p in PRECS}, rounds, window_s), stem_gflop(B, H, W, dims))},
           "grad_max_rel_vs_fp32": agree}
    del grads
    out["parts"] = parts(stems, images, rounds, window_s / 2)
    return out


def parts(stems, images, rounds, window_s):
    lib, P, st = L.load(), L.ptr, L.stream_ptr
    M = B * H * W
    fns = {}
    x = images
    for i in range(2):
        ci = x.shape[3]
        K = 9 * ci
        b = stems["fp32"].p["stem/cnnLayercnn_%d/biases/bias" % i]
        Wf, _ = stems["fp32"]._weights(i)
        W16, W3 = stems["bf16"]._weights(i)[1], stems["bf16x3"]._weights(i)[1]
        y = torch.empty(M, C_OUT, device="cuda")
        c32 = torch.empty(M, K, device="cuda")
        c16 = torch.empty(M, K, dtype=torch.bfloat16, device="cuda")
        c2 = torch.empty(M, 2 * K, dtype=torch.bfloat16, device="cuda")
        args = (KEEP, 11, SITE_STEM + i, 3, B, H, W, ci)
        fns["layer%d_patch_fp32" % i] = lambda x=x, c=c32, a=args: L.check(lib.mac_im2col3x3(P(x), P(c), 0, *a, st()))
        fns["layer%d_patch_bf16" % i] = lambda x=x, c=c16, a=args: L.check(lib.mac_im2col3x3(P(x), P(c), 1, *a, st()))
        fns["layer%d_patch_bf16x3" % i] = lambda x=x, c=c2, a=args: L.check(lib.mac_im2col3x3_split(P(x), P(c), *a, st()))
        one = lambda v, t=ctypes.c_int: (t * 1)(v)
        fns["layer%d_gemm_fp32" % i] = lambda c=c32, Wf=Wf, b=b, y=y, K=K: L.check(lib.mac_linear_fwd(
            one(c.data_ptr(), ctypes.c_void_p), one(K), one(K), 1, P(Wf), P(b), 0.0, L.ACT["ELU"], P(y), C_OUT, M, C_OUT, None,
            0, st()))
        fns["layer%d_gemm_bf16" % i] = lambda c=c16, w=W16, b=b, y=y, K=K: L.check(lib.mac_linear_tc_fwd(
            P(c), P(w), P(b), L.ACT["ELU"], P(y), 0, M, K, C_OUT, st()))
        fns["layer%d_gemm_bf16x3" % i] = lambda c=c2, w=W3, b=b, y=y, K=K: L.check(lib.mac_linear_tc32_fwd(
            P(c), P(w), P(b), L.ACT["ELU"], P(y), M, K, C_OUT, st()))
        for p in PRECS:                              # the GEMMs read real patches
            fns["layer%d_patch_%s" % (i, p)]()
        x = torch.relu(torch.randn(B, H, W, C_OUT, device="cuda"))
    res = compare(fns, rounds, window_s)
    for name, r in res.items():
        i = int(name[5])
        K = 9 * (C_IN if i == 0 else C_OUT)
        if "_gemm_" in name:
            r["tflops_algorithmic"] = 2.0 * M * K * C_OUT / 1e9 / r["ms"]
        else:
            width = {"fp32": 4, "bf16": 2, "bf16x3": 4}[name.split("_")[-1]]
            r["gb_per_s_written"] = M * K * width / 1e6 / r["ms"]
    return res


def whole_part(rounds, window_s):
    Bm, S, N, d, Ls = SHAPES["headline"]
    V, E, A = 90, 300, 28                         # bench.py train_full: CLEVR question vocabulary, embeddings, answers
    cfg = MACConfig.args("args", netLength=Ls)
    rng = np.random.RandomState(31)
    lengths = rng.randint(S // 2, S + 1, size=(Bm,)).astype(np.int32)
    lengths[0] = S
    q = rng.randint(1, V + 1, size=(Bm, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    data = {"questions": torch.from_numpy(q).cuda(), "questionLengths": torch.from_numpy(lengths).cuda(),
            "images": torch.relu(torch.randn(Bm, H, W, C_IN, device="cuda")),
            "answers": torch.from_numpy(rng.randint(0, A, size=(Bm,)).astype(np.int32)).cuda()}
    trainers = {sp: DPTrainer(cfg, Ls, seed=7, classifier=(A, [512]), encoder=(V, E), stem=(C_IN, 2), prec="tc32",
                              bwd_tc=True, stem_prec=sp) for sp in PRECS}
    res = compare({sp: (lambda tr=tr: tr.train_step_full(0, data, Bm)) for sp, tr in trainers.items()}, rounds, window_s)
    return {"shape": {"B": Bm, "S": S, "N": N, "d": d, "L": Ls, "stem_in": C_IN}, "cell": "prec=tc32, bwd_tc=True",
            "arms": res, "saved_ms_bf16x3": res["fp32"]["ms"] - res["bf16x3"]["ms"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stem_train_bf16x3.py measures on a CUDA device; none is visible")
    os.makedirs(a.out_dir, exist_ok=True)
    out = {"device": device_info(), "rounds": a.rounds}
    out["stem"] = stem_part(a.rounds, a.window)
    print(json.dumps({"stem": out["stem"]}), flush=True)
    torch.cuda.empty_cache()
    out["whole_model"] = whole_part(a.rounds, a.window)
    with open(os.path.join(a.out_dir, "stem_train_bf16x3.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
