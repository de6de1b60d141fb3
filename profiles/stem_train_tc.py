"""Mixed-precision training of the image stem: fp32 against bf16 (tensor-core) stem, on its own and inside the whole-model
training step.  Usage:  python profiles/stem_train_tc.py OUT_DIR [--rounds 3] [--window 0.5]

  stem:   Stem.forward(save_for_backward=True) + Stem.backward at B=64, 14x14, 1024 -> 512 -> 512, keep 0.82, the image
          gradient not asked for (as in training).  414.4 GFLOP per iteration: the forward (177.6), the weight gradients
          (177.6) and layer 1's data gradient (59.2).
  whole:  DPTrainer.train_step_full at the bench.py train_full shape with the cell on tensor cores in both arms
          (prec="bf16", bwd_tc=True), stem_prec="fp32" against "bf16": the difference is the stem alone.
Both arms of a comparison alternate in one process, `--rounds` times each, every window at least `--window` seconds of
CUDA events.  Also reports launches per iteration, the max-rel agreement of the bf16 stem gradients with the fp32 ones at
this size, and the card (name, power limit, max SM clock from nvidia-smi).  Writes OUT_DIR/stem_train_tc.json."""
import argparse
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from mac_network_b200 import _lib
from mac_network_b200.config import MACConfig
from mac_network_b200.dp import DPTrainer
from mac_network_b200.stem import Stem, init_stem_params, stem_specs
from mac_network_b200.synthetic import SHAPES

B, H, W, C_IN, C_OUT, KEEP = 64, 14, 14, 1024, 512, 0.82


def stem_gflop(B, H, W, dims):
    """forward + weight gradients of every layer, data gradients of layers >= 1 (the image gradient is not needed)"""
    M = B * H * W
    f = [2.0 * M * 9 * dims[i] * dims[i + 1] for i in range(len(dims) - 1)]
    return (2 * sum(f) + sum(f[1:])) / 1e9


def device_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock, "torch_device": torch.cuda.get_device_name(0)}


def timed(fn, n):
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.mac_b200_launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, (lib.mac_b200_launch_count() - n0) / n


def compare(arms, rounds, window_s):
    """arms: name -> callable.  Warm up, size each window to >= window_s, alternate the arms `rounds` times."""
    iters = {}
    for name, fn in arms.items():
        for _ in range(2):
            fn()
        ms, _ = timed(fn, 2)
        iters[name] = max(3, int(math.ceil(1.2 * window_s * 1e3 / ms)))      # margin over the 2-iteration estimate
    rows = {name: [] for name in arms}
    launches = {}
    for _ in range(rounds):
        for name, fn in arms.items():
            ms, nl = timed(fn, iters[name])
            rows[name].append(ms)
            launches[name] = nl
    return {name: {"ms": float(np.median(v)), "ms_rounds": [round(x, 4) for x in v], "iters_per_window": iters[name],
                   "window_s": round(iters[name] * min(v) / 1e3, 3), "launches": launches[name]} for name, v in rows.items()}


def stem_part(rounds, window_s):
    specs = stem_specs(C_IN, C_OUT)
    params = {k: torch.from_numpy(v).cuda() for k, v in init_stem_params(specs, seed=5).items()}
    g = torch.Generator(device="cuda").manual_seed(6)
    images = torch.relu(torch.randn(B, H, W, C_IN, device="cuda", generator=g))
    d_kb = torch.randn(B, H * W, C_OUT, device="cuda", generator=g) * 1e-3
    stems = {p: Stem(params, relu="ELU", prec=p, seed=11) for p in ("fp32", "bf16")}
    grads = {p: {k: torch.zeros_like(v) for k, v in params.items()} for p in stems}

    def step(p):
        st = stems[p]
        st.forward(images, keep=KEEP, step=3, save_for_backward=True)
        st.backward(d_kb, grads[p])

    # agreement: one forward(save) + backward of each from zeroed gradients, same masks (seed, site, step)
    for p in stems:
        for t in grads[p].values():
            t.zero_()
        step(p)
    torch.cuda.synchronize()
    agree = {k: float((grads["bf16"][k] - grads["fp32"][k]).abs().max() / grads["fp32"][k].abs().max()) for k in params}
    res = compare({p: (lambda p=p: step(p)) for p in stems}, rounds, window_s)
    gf = stem_gflop(B, H, W, [C_IN, C_OUT, C_OUT])
    for p, r in res.items():
        r["tflops_algorithmic"] = gf / r["ms"]
    return {"shape": {"B": B, "H": H, "W": W, "dims": [C_IN, C_OUT, C_OUT], "keep": KEEP}, "gflop_per_iter": gf,
            "arms": res, "speedup_bf16": res["fp32"]["ms"] / res["bf16"]["ms"],
            "grad_max_rel_bf16_vs_fp32": agree}


def whole_part(rounds, window_s):
    Bm, S, N, d, L = SHAPES["headline"]
    V, E, A = 90, 300, 28                         # bench.py train_full: CLEVR question vocabulary, embeddings, answers
    cfg = MACConfig.args("args", netLength=L)
    rng = np.random.RandomState(31)
    lengths = rng.randint(S // 2, S + 1, size=(Bm,)).astype(np.int32)
    lengths[0] = S
    q = rng.randint(1, V + 1, size=(Bm, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    data = {"questions": torch.from_numpy(q).cuda(), "questionLengths": torch.from_numpy(lengths).cuda(),
            "images": torch.relu(torch.randn(Bm, H, W, C_IN, device="cuda")),
            "answers": torch.from_numpy(rng.randint(0, A, size=(Bm,)).astype(np.int32)).cuda()}
    trainers = {sp: DPTrainer(cfg, L, seed=7, classifier=(A, [512]), encoder=(V, E), stem=(C_IN, 2), prec="bf16",
                              bwd_tc=True, stem_prec=sp) for sp in ("fp32", "bf16")}
    res = compare({sp: (lambda tr=tr: tr.train_step_full(0, data, Bm)) for sp, tr in trainers.items()}, rounds, window_s)
    return {"shape": {"B": Bm, "S": S, "N": N, "d": d, "L": L, "stem_in": C_IN}, "cell": "prec=bf16, bwd_tc=True",
            "arms": res, "saved_ms": res["fp32"]["ms"] - res["bf16"]["ms"],
            "speedup_bf16": res["fp32"]["ms"] / res["bf16"]["ms"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window", type=float, default=0.5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stem_train_tc.py measures on a CUDA device; none is visible")
    os.makedirs(a.out_dir, exist_ok=True)
    out = {"device": device_info(), "rounds": a.rounds}
    out["stem"] = stem_part(a.rounds, a.window)
    print(json.dumps({"stem": out["stem"]}), flush=True)
    torch.cuda.empty_cache()
    out["whole_model"] = whole_part(a.rounds, a.window)
    path = os.path.join(a.out_dir, "stem_train_tc.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
