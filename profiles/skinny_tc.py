"""The batch-sized split-bf16 projections (mac_linear_tc_small_fwd, csrc/skinny_tc.cuh) of one headline pass (B = 64, d = 512).
Usage:  python profiles/skinny_tc.py OUT_DIR [--base-tree PATH] [--runs 3] [--skip-bench]

  calls:      each batch-sized call of a headline pass alone, CUDA events around 500 launches, median of 5 such blocks:
                projY          [64 x 512]  @ [512 x 512]                       (the first step's memory projection)
                folded_write   [64 x 512 | 64 x 512] @ [1024 x 1024], columns >= 512 to y2   (write unit + next projY)
                last_write     [64 x 512 | 64 x 512] @ [1024 x 512]            (the last step's write unit)
  breakdown:  one headline pass under torch.profiler (profiles/read_setup.py's breakdown): every kernel in launch order with
              its device time, and the totals per kernel name.
  --base-tree the parent commit's tree with its build() done (its Python must match its library).  The call timings and
              `bench.py --gpus 1 --steps 480 --warmup 12 --skip-cpu --skip-train` run `--runs` times per tree, alternating,
              each in its own process; the first bench run of each tree also writes --dump-outputs, and the files are
              compared bit for bit.  The headline, the e2e line, gpu_launches and, after each run, the bf16_gqa sub-line
              (measured as bench.py measures it) are recorded.
Also records the card (name, power limit, clocks from nvidia-smi).  Writes OUT_DIR/skinny_tc_h100.json."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIDES = ("base", "new")
CALLS = (("projY", (512,), 512, 0), ("folded_write", (512, 512), 1024, 512), ("last_write", (512, 512), 512, 0))


def rs():
    if ROOT not in sys.path:
        sys.path.append(ROOT)
    from profiles import read_setup
    return read_setup


def call_times(iters=500, blocks=5):
    """us per launch of each batch-sized call of the headline pass, alone (weights and activations L2-resident, as in the
    pass, where each call's weights were read by the same call one step earlier)."""
    import torch
    from mac_network_b200 import _lib
    from mac_network_b200._lib import check, ptr, segments, stream_ptr
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(11)
    M, out = 64, {}
    for name, segs, n, n_split in CALLS:
        K = sum(segs)
        xs = [torch.randn(M, k, device="cuda", generator=g) for k in segs]
        W = torch.randn(K, n, device="cuda", generator=g) * K ** -0.5
        b = torch.randn(n, device="cuda", generator=g) * 0.1
        hi = torch.empty(n, K, dtype=torch.bfloat16, device="cuda")
        lo = torch.empty_like(hi)
        check(lib.mac_pack_weight_bf16_split(ptr(W), ptr(hi), ptr(lo), K, n, stream_ptr()), "pack")
        ldy = n_split or n
        y, y2 = torch.empty(M, ldy, device="cuda"), (torch.empty(M, ldy, device="cuda") if n_split else None)
        arr_p, arr_k, arr_ld = segments(xs)

        def one():
            check(lib.mac_linear_tc_small_fwd(arr_p, arr_k, arr_ld, len(xs), ptr(hi), ptr(lo), ptr(b), 0.0, 0, ptr(y), ldy,
                                              ptr(y2), n_split, None, None, None, M, n, stream_ptr()), name)
        for _ in range(50):
            one()
        torch.cuda.synchronize()
        per = []
        for _ in range(blocks):
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                one()
            e.record()
            torch.cuda.synchronize()
            per.append(a.elapsed_time(e) * 1e3 / iters)
        out[name] = {"M_K_N": [M, K, n], "ctas": n // (64 if n >= 1024 else 32), "us": float(np.median(per)),
                     "blocks_us": [round(x, 2) for x in per]}
    return out


def worker(tree, what):
    sys.path.insert(0, tree)
    fns = {"calls": call_times} if what == "calls" else {"calls": call_times, "breakdown": rs().breakdown}
    print(json.dumps({k: f() for k, f in fns.items()}))


def run_worker(tree, what):
    out = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", what, "--tree", tree],
                         capture_output=True, text=True, timeout=1800, cwd=tree)
    if out.returncode != 0:
        raise RuntimeError("worker %s: exit %d: %s" % (what, out.returncode, out.stderr[-3000:]))
    return json.loads(out.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir", nargs="?")
    ap.add_argument("--base-tree")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--skip-bench", action="store_true")
    ap.add_argument("--worker")
    ap.add_argument("--tree")
    args = ap.parse_args()
    if args.worker:
        return worker(args.tree, args.worker)
    R = rs()
    out = {"device": R.device_info(), "shape_B_d": [64, 512]}
    out["new"] = run_worker(ROOT, "all")
    if args.base_tree:
        trees = {"base": os.path.abspath(args.base_tree), "new": ROOT}
        out["base"] = run_worker(trees["base"], "all")
        calls = {s: {c[0]: [] for c in CALLS} for s in SIDES}
        for _ in range(args.runs):
            for s in SIDES:
                for k, v in run_worker(trees[s], "calls")["calls"].items():
                    calls[s][k].append(v["us"])
        out["call_us"] = {s: {k: R.spread(v) for k, v in calls[s].items()} for s in SIDES}
        if not args.skip_bench:
            tmp = tempfile.mkdtemp(prefix="skinny_tc_")
            try:
                dumps = {s: os.path.join(tmp, "dump_" + s) for s in SIDES}
                lines = {s: {"headline": [], "bf16_gqa": [], "e2e": []} for s in SIDES}
                launches = {s: [] for s in SIDES}
                for i in range(args.runs):
                    for s in SIDES:
                        extra = ["--gpus", "1", "--steps", "480", "--warmup", "12", "--skip-cpu", "--skip-train"]
                        line = R.bench(trees[s], extra + (["--dump-outputs", dumps[s]] if i == 0 else []))
                        lines[s]["headline"].append(line["value"])
                        lines[s]["e2e"].append(line["e2e"]["value"])
                        launches[s].append(line.get("gpu_launches"))
                        lines[s]["bf16_gqa"].append(R.bench(trees[s], R.GQA)["value"])
                out["reasoning_steps_per_s"] = {s: {k: R.spread(v) for k, v in lines[s].items()} for s in SIDES}
                out["gpu_launches"] = launches
                out["headline_speedup"] = (out["reasoning_steps_per_s"]["new"]["headline"]["median"] /
                                           out["reasoning_steps_per_s"]["base"]["headline"]["median"])
                same = {}
                for name in sorted(os.listdir(dumps["base"])):
                    a, b = np.load(os.path.join(dumps["base"], name)), np.load(os.path.join(dumps["new"], name))
                    same[name] = bool(a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes())
                out["outputs_bit_identical"] = same
            finally:
                shutil.rmtree(tmp, ignore_errors=True)
    out["device_after"] = R.device_info()
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "skinny_tc_h100.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({k: v for k, v in out.items() if k not in ("new", "base")}))
    for s in SIDES:
        if s in out:
            print(s, json.dumps(out[s]["calls"]), json.dumps(out[s]["breakdown"]["per_kernel"][:8]))


if __name__ == "__main__":
    main()
