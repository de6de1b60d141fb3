"""Image features stored in fp16: the `_f16` ingest kernels, ModelPipeline and TrainPipeline with image_dtype=torch.float16,
each against the same path over fp32 features, and what the fp16 rounding of the features costs at the stem's output.
Usage:  python profiles/half_features.py OUT_DIR [--rounds 5] [--window 1.0] [--images 512]

  kernels:   mac_ingest_nchw(_f16) in both modes and mac_ingest_nchw_train(_f16) in both forms (keep 0.82) at the CLEVR
             (64 x 1024 x 14 x 14) and GQA (64 x 2048 x 7 x 7) features, fp16 against fp32 input: CUDA events around 30
             back-to-back launches, the bytes the kernel must move (input read once, outputs written once) over time beside
             3.35 TB/s.
  serving:   ModelPipeline, four slots, fp32 features (host_cast=False) against image_dtype=torch.float16, over three
             pre-built numpy batches and three pinned ones, in bf16 and e4m3 (prec="fp8", e4m3 stem, bf16 encoder) at the
             CLEVR (B=64, S=40, 1024x14x14, L=12) and GQA (B=64, S=30, 2048x7x7, L=6) shapes.  Also: the fp16 pipeline's
             outputs against the fp32 pipeline fed the widened fp16 features (must be bit-equal), and its answers against the
             fp32 pipeline fed the original fp32 features of the same seeded batch (the storage's effect on the answers).
  cache:     ModelPipeline(images=16, cache=I/2) at the CLEVR shape in bf16, on the kb_cache.py stream (I images, 10
             questions each, shuffled into batches of 64: about half of each batch's images hit), with a loader that gathers
             the missing features from a host array of the I images (fp32, or fp16) on 8 threads into pinned memory.  The
             loader's own host seconds are counted.
  training:  TrainPipeline (depth 2) at the CLEVR training shape (B=64, S=40, 1024x14x14, L=12, all tensor cores), fp32
             against fp16 features, over numpy and pinned batches.
  storage:   the max-norm relative error of the stem's output (1024 -> 512 -> 512, B=64, 14x14) from fp16-rounded
             features against fp32 features, ReLU-like features, in each stem precision.
Method of profiles/model_pipeline.py: one process, the arms alternating `--rounds` times, every window at least `--window`
seconds of host clock ending in a synchronise, medians.  Records the card (name, power limit, max SM clock from nvidia-smi).
Writes OUT_DIR/half_features_h100.json.  Fails without a GPU."""
import argparse
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np
import torch

from mac_network_b200 import _lib as L
from mac_network_b200.config import MACConfig
from mac_network_b200.model import MACnet
from mac_network_b200.serving import ModelPipeline, TrainPipeline
from model_pipeline import A, E, HBM_TBS, MODELS, SHAPES, V, compare, device_info, host_batches, timed

U = 16
TRAIN = dict(train_prec="bf16", bwd_tc=True, stem_prec="bf16", enc_prec="bf16")


def kernel_part(rounds, iters=30):
    lib = L.load()
    s = L.stream_ptr()
    out = {}
    for shape_name in ("clevr", "gqa"):
        sh = SHAPES[shape_name]
        B, C, H, W = sh["B"], sh["C"], sh["H"], sh["W"]
        x32 = torch.relu(torch.randn(B, C, H, W, device="cuda"))
        x16 = x32.half()
        nhwc = torch.empty((B, H, W, C), device="cuda")
        cols = torch.empty((B * H * W, 2 * 9 * C), dtype=torch.bfloat16, device="cuda")
        n, nc = x32.numel(), B * H * W * 9 * C
        fns = {}
        for tag, x, esz in (("fp32", x32, 4), ("fp16", x16, 2)):
            if tag == "fp32":
                ing = lambda m, x=x: L.check(lib.mac_ingest_nchw(L.ptr(x), 0, L.ptr(cols if m else nhwc), m, B, C, H, W, s))
                tr = lambda f, x=x: L.check(lib.mac_ingest_nchw_train(L.ptr(x), L.ptr(nhwc), L.ptr(cols), f, 0.82, 7, 32, 1,
                                                                      B, C, H, W, s))
            else:
                ing = lambda m, x=x: L.check(lib.mac_ingest_nchw_f16(L.ptr(x), L.ptr(cols if m else nhwc), m, B, C, H, W, s))
                tr = lambda f, x=x: L.check(lib.mac_ingest_nchw_train_f16(L.ptr(x), L.ptr(nhwc), L.ptr(cols), f, 0.82, 7, 32,
                                                                          1, B, C, H, W, s))
            fns["nhwc_from_" + tag] = (lambda ing=ing: ing(0), n * esz + n * 4)
            fns["patch_bf16_from_" + tag] = (lambda ing=ing: ing(1), n * esz + nc * 2)
            fns["train_cols_bf16_from_" + tag] = (lambda tr=tr: tr(0), n * esz + n * 4 + nc * 2)
            fns["train_cols_split_from_" + tag] = (lambda tr=tr: tr(1), n * esz + n * 4 + nc * 4)
        us = {k: [] for k in fns}
        for fn, _ in fns.values():
            fn()
        for _ in range(rounds):
            for k, (fn, _) in fns.items():
                us[k].append(timed(fn, iters))
        res = {}
        for k, (_, nbytes) in fns.items():
            med = float(np.median(us[k]))
            res[k] = {"us": med, "us_min": min(us[k]), "us_max": max(us[k]), "min_bytes": nbytes,
                      "tb_per_s": nbytes / med / 1e6, "share_of_hbm_bound": nbytes / med / 1e6 / HBM_TBS}
        for k in ("nhwc", "patch_bf16", "train_cols_bf16", "train_cols_split"):
            res[k + "_fp16_over_fp32_time"] = res[k + "_from_fp16"]["us"] / res[k + "_from_fp32"]["us"]
        res["shape"] = [B, C, H, W]
        out[shape_name] = res
    out["note"] = ("min_bytes: the input read once plus every output written once.  share_of_hbm_bound: that over the "
                   "%.2f TB/s of the data sheet of a 700 W H100 SXM" % HBM_TBS)
    return out


def _pipe_arm(pipe, batches):
    def go(n):
        for i in range(n):
            pipe.submit(batches[i % len(batches)])
        pipe.drain()
    return go


def _half(batches):
    return [dict(b, images=b["images"].astype(np.float16)) for b in batches]


def _pinned(batches):
    return [{k: torch.from_numpy(v).pin_memory() for k, v in b.items() if k != "answers"} for b in batches]


def _max_rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def serving_part(rounds, window):
    out = {}
    for shape_name in ("clevr", "gqa"):
        sh = SHAPES[shape_name]
        shape = (sh["B"], sh["S"], sh["H"], sh["W"])
        b32 = [{k: v for k, v in b.items() if k != "answers"} for b in host_batches(sh)]
        b16 = _half(b32)
        wid = [dict(b, images=b["images"].astype(np.float32)) for b in b16]
        p32, p16 = _pinned(b32), _pinned(b16)
        for model in ("bf16", "fp8"):
            cfg = MACConfig.args(sh["variant"], netLength=sh["L"])
            net = MACnet(cfg, sh["L"], V, A, wrd_emb_dim=E, image_in_dim=sh["C"], classifier_dims=(512,), seed=7,
                         **MODELS[model])
            pipe32 = ModelPipeline(net, shape, slots=4, host_cast=False)
            pipe16 = ModelPipeline(net, shape, slots=4, image_dtype=torch.float16)
            # outputs: bit for bit the fp32 pipeline's on the widened features; the answers against the original features
            got = {k: v.clone() for k, v in pipe16.result(pipe16.submit(b16[0])).items()}
            ref = {k: v.clone() for k, v in pipe32.result(pipe32.submit(wid[0])).items()}
            orig = {k: v.clone() for k, v in pipe32.result(pipe32.submit(b32[0])).items()}
            check = {"bit_equal_to_fp32_pipeline_on_widened_features": all(torch.equal(got[k], ref[k]) for k in got),
                     "answers_equal_to_fp32_features": float((got["answers"][:, 0] == orig["answers"][:, 0]).float().mean()),
                     "logits_max_rel_to_fp32_features": _max_rel(got["logits"], orig["logits"]),
                     "memory_max_rel_to_fp32_features": _max_rel(got["memory"], orig["memory"])}
            arms = {"fp32_numpy": _pipe_arm(pipe32, b32), "fp16_numpy": _pipe_arm(pipe16, b16),
                    "fp32_pinned": _pipe_arm(pipe32, p32), "fp16_pinned": _pipe_arm(pipe16, p16)}
            r = compare(arms, rounds, window)
            for src in ("numpy", "pinned"):
                r["fp16_over_fp32_time_" + src] = r["fp16_" + src]["ms_per_batch"] / r["fp32_" + src]["ms_per_batch"]
            r["h2d_bytes"] = {"fp32": pipe32.h2d_bytes, "fp16": pipe16.h2d_bytes}
            out["%s_%s" % (shape_name, model)] = {"shape": sh, "model": MODELS[model], "slots": 4, "arms": r,
                                                  "outputs": check}
            print(json.dumps({"%s_%s" % (shape_name, model): out["%s_%s" % (shape_name, model)]}), flush=True)
            del pipe32, pipe16, arms, net
            torch.cuda.empty_cache()
    return out


def cache_part(rounds, window, I):
    from kb_cache import Stream
    sh = SHAPES["clevr"]
    B = sh["B"]
    shape = (B, sh["S"], sh["H"], sh["W"])
    st = Stream(sh, I)
    feats = {"fp32": st.feats, "fp16": st.feats.astype(np.float16)}
    cfg = MACConfig.args(sh["variant"], netLength=sh["L"])
    net = MACnet(cfg, sh["L"], V, A, wrd_emb_dim=E, image_in_dim=sh["C"], classifier_dims=(512,), seed=7, **MODELS["bf16"])
    pipes = {"fp32": ModelPipeline(net, shape, slots=4, images=U, cache=I // 2),
             "fp16": ModelPipeline(net, shape, slots=4, images=U, cache=I // 2, image_dtype=torch.float16)}
    counters = {k: [0, 0.0, 0.0] for k in pipes}

    def loader(tag):
        f, c = feats[tag], counters[tag]
        dt = torch.from_numpy(f[:1]).dtype

        def load(ids):
            t0 = time.perf_counter()
            out = torch.empty((B,) + f.shape[1:], dtype=dt, pin_memory=True)[:len(ids)]
            dst, cuts = out.numpy(), np.linspace(0, len(ids), 9).astype(int)
            list(st.pool.map(lambda i: np.take(f, ids[cuts[i]:cuts[i + 1]], axis=0, out=dst[cuts[i]:cuts[i + 1]]), range(8)))
            c[2] += time.perf_counter() - t0
            return out
        return load

    def arm(tag):
        pipe, c, load = pipes[tag], counters[tag], loader(tag)

        def go(n):
            for _ in range(n):
                b = dict(st.batches[c[0] % len(st.batches)], images=load)
                t0 = time.perf_counter()
                pipe.submit(b)
                c[1] += time.perf_counter() - t0
                c[0] += 1
            pipe.drain()
        return go
    arms = {k: arm(k) for k in pipes}
    for go in arms.values():
        go(len(st.batches))                 # a pass over the stream: the cache holds its steady half
    before = {k: (dict(p.cache_stats()), list(counters[k])) for k, p in pipes.items()}
    r = compare(arms, rounds, window)
    for k, v in r.items():
        s0, c0 = before[k]
        s1 = pipes[k].cache_stats()
        nb = counters[k][0] - c0[0]
        hits, miss = s1["hits"] - s0["hits"], s1["misses"] - s0["misses"]
        v["hit_rate"] = hits / max(1, hits + miss)
        v["image_mb_per_batch"] = (s1["image_bytes"] - s0["image_bytes"]) / nb / 1e6
        v["host_submit_ms_per_batch"] = 1e3 * (counters[k][1] - c0[1]) / nb
        v["host_loader_ms_per_batch"] = 1e3 * (counters[k][2] - c0[2]) / nb
        v["batches_timed_and_warm"] = nb
    r["fp16_over_fp32_time"] = r["fp16"]["ms_per_batch"] / r["fp32"]["ms_per_batch"]
    res = {"shape": sh, "model": MODELS["bf16"], "slots": 4, "images_per_pass": U, "cache": I // 2, "images_in_stream": I,
           "arms": r}
    print(json.dumps({"cache": res}), flush=True)
    st.pool.shutdown()
    return res


def train_part(rounds, window):
    from train_pipeline import SHAPE, host_batches as train_batches, pipeline_arm
    sh = SHAPE
    shape = (sh["B"], sh["S"], sh["H"], sh["W"])
    cfg = MACConfig.args(sh["variant"], netLength=sh["L"])
    b32 = train_batches(sh)
    b16 = _half(b32)
    pin = lambda bs: [dict(b, images=torch.from_numpy(b["images"]).pin_memory()) for b in bs]
    nets = {k: MACnet(cfg, sh["L"], V, A, wrd_emb_dim=E, image_in_dim=sh["C"], classifier_dims=(512,), seed=7, prec="bf16",
                      **TRAIN) for k in ("fp32", "fp16")}
    p32 = TrainPipeline(nets["fp32"], shape, depth=2)
    p16 = TrainPipeline(nets["fp16"], shape, depth=2, image_dtype=torch.float16)
    arms = {"fp32_numpy": pipeline_arm(p32, b32), "fp16_numpy": pipeline_arm(p16, b16),
            "fp32_pinned": pipeline_arm(p32, pin(b32)), "fp16_pinned": pipeline_arm(p16, pin(b16))}
    r = compare(arms, rounds, window)
    for src in ("numpy", "pinned"):
        r["fp16_over_fp32_time_" + src] = r["fp16_" + src]["ms_per_batch"] / r["fp32_" + src]["ms_per_batch"]
    res = {"shape": sh, "trainer": TRAIN, "depth": 2, "stage_threads": p32.stage_threads, "arms": r,
           "note": "ms_per_batch is ms per training step"}
    print(json.dumps({"training": res}), flush=True)
    return res


def storage_part():
    from mac_network_b200.stem import Stem, init_stem_params, stem_specs
    p = {k: torch.from_numpy(v).cuda() for k, v in init_stem_params(stem_specs(1024, 512), seed=6).items()}
    x = torch.from_numpy(np.maximum(np.random.RandomState(3).standard_normal((64, 1024, 14, 14)), 0).astype(np.float32)).cuda()
    out = {}
    for prec in ("fp32", "bf16x3", "bf16", "fp8"):
        st = Stem(p, relu="ELU", prec=prec, seed=41)
        kb32 = st.forward_nchw(x).double()
        kb16 = st.forward_nchw(x.half()).double()
        out[prec] = float((kb16 - kb32).abs().max() / kb32.abs().max())
    normal = x >= 2.0 ** -14                       # fp16's normal range: below it the rounding is absolute, 2^-25
    out["feature_rounding_max_rel_normal_range"] = float(((x.half().float() - x).abs() / x)[normal].max())
    out["feature_rounding_max_abs"] = float((x.half().float() - x).abs().max())
    out["features_nonzero_below_fp16_normal_range"] = float(((x > 0) & ~normal).float().mean())
    out["note"] = ("max |stem(fp16(x)) - stem(x)| / max |stem(x)| per stem precision, stem 1024 -> 512 -> 512 (ELU), "
                   "x = max(N(0, 1), 0) of shape 64 x 1024 x 14 x 14, seed 3")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--images", type=int, default=512, help="images in the cache arm's stream (10 questions each)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("half_features.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    os.makedirs(a.out_dir, exist_ok=True)
    out = {"device": device_info(), "rounds": a.rounds, "window_s": a.window}
    out["storage_error"] = storage_part()
    print(json.dumps({"storage_error": out["storage_error"]}), flush=True)
    out["kernels"] = kernel_part(a.rounds)
    print(json.dumps({"kernels": out["kernels"]}), flush=True)
    out["serving"] = serving_part(a.rounds, a.window)
    out["cache"] = cache_part(a.rounds, a.window, a.images)
    out["training"] = train_part(a.rounds, a.window)
    path = os.path.join(a.out_dir, "half_features_h100.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out["device"]))


if __name__ == "__main__":
    main()
