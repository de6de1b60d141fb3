"""Knowledge bases kept on the device across batches: serving.ModelPipeline(images=16, cache=C) against the pipeline without a
cache, on a stream whose batches do not group questions by image.  Usage:  python profiles/kb_cache.py OUT_DIR [--rounds 5]
[--window 1.0] [--images 512]

  stream:  I images with 10 questions each, the 10*I questions shuffled (the reference buckets questions by length, not by
           image), cut into batches of B = 64: a batch asks about ~58 distinct images, and each image comes back in ~10
           batches.  Workloads: the CLEVR shape (B=64, S=40, 1024x14x14, d=512, L=12) in bf16 and in e4m3 (prec="fp8" with
           the e4m3 stem and the bf16 encoder), the GQA shape (B=64, S=30, 2048x7x7, d=512, L=6) in bf16.
  arms:    four slots, fp32 copies (no host cast):  (a) images=None fed each question's features;  (b) images=64 without a
           cache, fed each batch's distinct images (within-batch sharing only: images=16 cannot take a batch of ~58
           distinct images);  (c) images=16, cache=I after a warm pass over the stream: every image hits;  (d) images=16,
           cache=I/2, which evicts (least recently used);  (e) as (d) with a loader that returns rows of one pinned buffer
           written once instead of gathering the ids' features (wrong features: it times the pipeline without the host
           gather, and its outputs are not compared).  The loader of (c) and (d) gathers the missing features from a host
           array of the I images on 8 threads into pinned memory, a host cost the other arms do not pay (they rotate over
           three pre-built pinned batches).  Per arm the host seconds inside `submit` and inside the loader are counted.  Method of profiles/model_pipeline.py (DESIGN.md section 8): one process, the arms
           alternating `--rounds` times, every window at least `--window` seconds of host clock ending in a synchronise.
           Reports ms per batch (median, min, max), the hit rate and the image MB copied per batch, and compares the
           outputs of each arm on one batch with arm (a).
  kernels: mac_kb_pool_insert (16 stem rows into the pool, fp32 and bf16) and mac_kb_gather_bf16 (64 rows out of the bf16
           pool) alone, CUDA events around 30 back-to-back launches, bytes moved over time beside 3.35 TB/s.
Records the card (name, power limit, max SM clock from nvidia-smi).  Writes OUT_DIR/kb_cache_h100.json.  Fails without a
GPU."""
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
from mac_network_b200.serving import ModelPipeline
from model_pipeline import A, E, HBM_TBS, SHAPES, V, compare, device_info, timed

U = 16
WORKLOADS = {"clevr_bf16": ("clevr", dict(prec="bf16")),
             "clevr_fp8": ("clevr", dict(prec="fp8", eval_stem_prec="fp8", eval_enc_prec="bf16")),
             "gqa_bf16": ("gqa", dict(prec="bf16"))}


class Stream(object):
    """The shuffled stream of one shape: I images' features in one host array, keyed 0..I-1, 10 questions each."""

    def __init__(self, sh, I, seed=0):
        rng = np.random.RandomState(seed)
        B, S = sh["B"], sh["S"]
        self.B, self.I = B, I
        self.feats = np.empty((I, sh["C"], sh["H"], sh["W"]), dtype=np.float32)
        for i in range(I):
            self.feats[i] = np.maximum(rng.standard_normal(self.feats.shape[1:]), 0)
        ids = np.repeat(np.arange(I), 10)
        rng.shuffle(ids)
        self.batches = []
        for j in range(len(ids) // B):
            lengths = rng.randint(S // 2, S + 1, size=(B,)).astype(np.int32)
            lengths[0] = S
            q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
            q[np.arange(S)[None, :] >= lengths[:, None]] = 0
            self.batches.append({"questions": torch.from_numpy(q).pin_memory(),
                                 "questionLengths": torch.from_numpy(lengths).pin_memory(),
                                 "imageIds": ids[j * B:(j + 1) * B].copy()})
        from concurrent.futures import ThreadPoolExecutor
        self.pool = ThreadPoolExecutor(8)
        self.fixed = torch.from_numpy(self.feats[:B]).pin_memory()

    def load(self, ids):
        """The loader: the features of `ids` gathered from the host array on 8 threads into the front of a pinned buffer of
        B images.  The buffer is freed when the pipeline lets go of it, and torch's caching host allocator hands its block
        out again only once the copy out of it has finished; one size for every call lets it do so."""
        out = torch.empty((self.B,) + self.feats.shape[1:], dtype=torch.float32, pin_memory=True)[:len(ids)]
        dst, cuts = out.numpy(), np.linspace(0, len(ids), 9).astype(int)
        list(self.pool.map(lambda i: np.take(self.feats, ids[cuts[i]:cuts[i + 1]], axis=0, out=dst[cuts[i]:cuts[i + 1]]),
                           range(8)))
        return out

    def cached(self, j, counter=None, gather=True):
        """Batch j of the stream with a loader.  `counter[2]` accumulates the loader's host seconds.  gather=False: a loader
        that returns the first m rows of one pinned buffer written once -- not the features of the ids -- so that the arm
        times the pipeline without the host gather (its outputs are not compared)."""
        def load(ids):
            t0 = time.perf_counter()
            out = self.load(ids) if gather else self.fixed[:len(ids)]
            if counter is not None:
                counter[2] += time.perf_counter() - t0
            return out
        return dict(self.batches[j % len(self.batches)], images=load)

    def duplicated(self, j):
        b = self.batches[j]
        return {"questions": b["questions"], "questionLengths": b["questionLengths"],
                "images": torch.from_numpy(self.feats[b["imageIds"]]).pin_memory()}

    def shared(self, j):
        b = self.batches[j]
        distinct = list(dict.fromkeys(b["imageIds"].tolist()))
        index = np.array([distinct.index(i) for i in b["imageIds"]], dtype=np.int32)
        return {"questions": b["questions"], "questionLengths": b["questionLengths"], "imageIndex": torch.from_numpy(index),
                "images": torch.from_numpy(self.feats[distinct]).pin_memory()}


def arm(pipe, make, counter):
    """counter: [batches submitted, host seconds in submit (the loader included), host seconds in the loader]."""
    def go(n):
        for _ in range(n):
            b = make(counter[0])
            t0 = time.perf_counter()
            pipe.submit(b)
            counter[1] += time.perf_counter() - t0
            counter[0] += 1
        pipe.drain()
    return go


def kernel_part(sh, I, rounds, iters=30):
    lib = L.load()
    B, N, d = sh["B"], sh["H"] * sh["W"], 512
    s = L.stream_ptr()
    rng = np.random.RandomState(1)
    kb_u = torch.randn(U, N, d, device="cuda")
    pool32 = torch.zeros(I, N, d, device="cuda")
    pool16 = torch.zeros(I, N, d, dtype=torch.bfloat16, device="cuda")
    out16 = torch.empty(B, N, d, dtype=torch.bfloat16, device="cuda")
    slot = torch.from_numpy(rng.choice(I, U, replace=False).astype(np.int32)).cuda()
    index = torch.from_numpy(rng.choice(I, B, replace=False).astype(np.int32)).cuda()
    row = N * d
    fns = {"pool_insert_fp32_U16": (lambda: L.check(lib.mac_kb_pool_insert(L.ptr(kb_u), L.ptr(slot), L.ptr(pool32), 0, U, I,
                                                                           N, d, s)), U * row * 8),
           "pool_insert_bf16_U16": (lambda: L.check(lib.mac_kb_pool_insert(L.ptr(kb_u), L.ptr(slot), L.ptr(pool16), 1, U, I,
                                                                           N, d, s)), U * row * 6),
           "gather_bf16_B64": (lambda: L.check(lib.mac_kb_gather_bf16(L.ptr(pool16), L.ptr(index), L.ptr(out16), B, I, N, d,
                                                                      s)), B * row * 4)}
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
    out["note"] = ("N=%d, d=%d, pool of %d rows.  min_bytes: the fp32 rows read plus the rows written (insert), the bf16 rows "
                   "read plus written (gather).  Each launch moves %.1f-%.1f MB, which the 50 MB L2 holds across the 30 "
                   "back-to-back launches with the same operands, so these are L2-resident figures and may pass the HBM "
                   "bound, %.2f TB/s on the data sheet of a 700 W card"
                   % (N, d, I, U * row * 6 / 1e6, B * row * 4 / 1e6, HBM_TBS))
    return out


def max_rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--images", type=int, default=512, help="I: images in the stream (10 questions each)")
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kb_cache.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    os.makedirs(a.out_dir, exist_ok=True)
    I = a.images
    out = {"device": device_info(), "rounds": a.rounds, "window_s": a.window, "slots": 4, "copies": "fp32, no host cast",
           "images_in_stream": I, "questions_per_image": 10, "stem_rows_per_pass": U,
           "kernels": kernel_part(SHAPES["clevr"], I, a.rounds), "workloads": {}}
    print(json.dumps({"kernels": out["kernels"]}), flush=True)
    for wname in a.workloads.split(","):
        shape_name, mkw = WORKLOADS[wname]
        sh = SHAPES[shape_name]
        st = Stream(sh, I)
        B = sh["B"]
        shape = (B, sh["S"], sh["H"], sh["W"])
        cfg = MACConfig.args(sh["variant"], netLength=sh["L"])
        net = MACnet(cfg, sh["L"], V, A, wrd_emb_dim=E, image_in_dim=sh["C"], classifier_dims=(512,), seed=7, **mkw)
        dup = [st.duplicated(j) for j in range(3)]
        shared = [st.shared(j) for j in range(3)]
        pipes = {"images_None": ModelPipeline(net, shape, slots=4, host_cast=False),
                 "images_64_no_cache": ModelPipeline(net, shape, slots=4, host_cast=False, images=B),
                 "images_16_cache_I": ModelPipeline(net, shape, slots=4, images=U, cache=I),
                 "images_16_cache_I_over_2": ModelPipeline(net, shape, slots=4, images=U, cache=I // 2),
                 "images_16_cache_I_over_2_no_gather": ModelPipeline(net, shape, slots=4, images=U, cache=I // 2)}
        counters = {k: [0, 0.0, 0.0] for k in pipes}
        arms = {"images_None": arm(pipes["images_None"], lambda j: dup[j % 3], counters["images_None"]),
                "images_64_no_cache": arm(pipes["images_64_no_cache"], lambda j: shared[j % 3],
                                          counters["images_64_no_cache"]),
                "images_16_cache_I": arm(pipes["images_16_cache_I"], lambda j: st.cached(j, counters["images_16_cache_I"]),
                                         counters["images_16_cache_I"]),
                "images_16_cache_I_over_2": arm(pipes["images_16_cache_I_over_2"],
                                                lambda j: st.cached(j, counters["images_16_cache_I_over_2"]),
                                                counters["images_16_cache_I_over_2"]),
                "images_16_cache_I_over_2_no_gather": arm(
                    pipes["images_16_cache_I_over_2_no_gather"],
                    lambda j: st.cached(j, counters["images_16_cache_I_over_2_no_gather"], gather=False),
                    counters["images_16_cache_I_over_2_no_gather"])}
        arms["images_16_cache_I"](len(st.batches))             # the warm pass: every image of the stream is cached
        assert pipes["images_16_cache_I"].cache_stats()["resident"] == I
        # the arms' outputs on one batch, against images=None
        ref = {k: v.clone() for k, v in pipes["images_None"].result(pipes["images_None"].submit(dup[0])).items()}
        agree = {}
        for key, b in (("images_64_no_cache", shared[0]), ("images_16_cache_I", st.cached(0)),
                       ("images_16_cache_I_over_2", st.cached(0))):
            got = pipes[key].result(pipes[key].submit(b))
            agree[key] = {kk: ("bit_equal" if torch.equal(got[kk], ref[kk]) else max_rel(got[kk], ref[kk]))
                          for kk in ("logits", "memory", "att_kb", "att_question")}
        for p in pipes.values():
            p.drain()
        before = {k: (dict(p.cache_stats()) if p._cache is not None else None, list(counters[k])) for k, p in pipes.items()}
        r = compare(arms, a.rounds, a.window)
        img_bytes = st.feats[0].nbytes
        for key, v in r.items():
            v["questions_per_s"] = v["batches_per_s"] * B
            v["speedup_over_images_None"] = v["batches_per_s"] / r["images_None"]["batches_per_s"]
            stats0, c0 = before[key]
            nb = counters[key][0] - c0[0]
            v["host_submit_ms_per_batch"] = 1e3 * (counters[key][1] - c0[1]) / nb
            if key.startswith("images_16_cache"):
                v["host_loader_ms_per_batch"] = 1e3 * (counters[key][2] - c0[2]) / nb
            if stats0 is None:
                per = B if key == "images_None" else np.mean([len(set(st.batches[j]["imageIds"].tolist())) for j in range(3)])
                v["images_copied_per_batch"] = float(per)
                v["image_mb_per_batch"] = float(per) * img_bytes / 1e6
            else:
                s1 = pipes[key].cache_stats()
                hits, miss = s1["hits"] - stats0["hits"], s1["misses"] - stats0["misses"]
                v["hit_rate"] = hits / max(1, hits + miss)
                v["distinct_images_per_batch"] = (hits + miss) / nb
                v["image_mb_per_batch"] = (s1["image_bytes"] - stats0["image_bytes"]) / nb / 1e6
            v["batches_timed_and_warm"] = nb
        out["workloads"][wname] = {"shape": sh, "model": mkw, "batches_in_stream": len(st.batches), "arms": r,
                                   "outputs_against_images_None": agree}
        print(json.dumps({wname: out["workloads"][wname]}), flush=True)
        st.pool.shutdown()
        del pipes, arms, net, st
        torch.cuda.empty_cache()
    path = os.path.join(a.out_dir, "kb_cache_h100.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out["device"]))


if __name__ == "__main__":
    main()
