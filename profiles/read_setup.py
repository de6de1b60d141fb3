"""The read unit's per-pass set-up in the bf16 inference form: the knowledge-base cast to bf16 and the step-invariant
P = KB @ Wx + bx and Q = P @ Wm[d:2d] + bm, at the headline shape (B = 64, N = 196, d = 512).
Usage:  python profiles/read_setup.py OUT_DIR [--base-tree PATH] [--runs 3] [--skip-bench]

  breakdown:  one headline pass as in profiles/one_pass.py (one stream, no CUDA graph) under torch.profiler with CUDA
              activities, after three warm passes: every kernel of the pass in launch order with its device time, and the
              totals per kernel name.
  set-up:     the set-up as MACCell runs it, CUDA events around 200 launches of it rotating over 6 fp32 knowledge bases
              with their bf16 copies and P / Q outputs (6 x 64 MB > 50 MB L2), median of 5 such blocks:
              mac_cast_bf16 + mac_read_invariant; where the library has it, also mac_read_invariant_cast (the cast,
              P and Q in one launch) as `setup_one_launch`.
  --base-tree the parent commit's tree with its build() done (its Python must match its library).  The set-up timing and
              `bench.py --gpus 1 --steps 480 --warmup 12 --skip-cpu --skip-train` run `--runs` times per tree,
              alternating, each in its own process; the first bench run of each tree also writes --dump-outputs, and
              the files are compared bit for bit.  The headline and the e2e line are recorded, and after each run the
              bf16_gqa sub-line, measured as bench.py measures it (`--mode quick --workload gqa`, GQA below).
Also records the card (name, power limit, clocks from nvidia-smi).  Writes OUT_DIR/read_setup_h100.json."""
import argparse
import ctypes
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIDES = ("base", "new")
GQA = ["--mode", "quick", "--workload", "gqa", "--streams", "12", "--steps", "24", "--warmup", "6"]   # bench's bf16_gqa


def device_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm,clocks.mem",
                        "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
    name, power, max_sm, sm, mem = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": max_sm, "sm_clock_idle": sm, "mem_clock": mem}


def spread(xs):
    xs = [float(x) for x in xs]
    return {"median": float(np.median(xs)), "min": min(xs), "max": max(xs), "runs": [round(x, 3) for x in xs]}


def headline_cell(variant="args"):
    import torch
    from mac_network_b200.config import MACConfig
    from mac_network_b200.mac_cell import MACCell, MACParams
    from mac_network_b200.params import init_params, perturb_biases
    from mac_network_b200.synthetic import SHAPES, make_inputs
    B, S, N, d, L = SHAPES["gqa" if variant == "gqa" else "headline"]
    cfg = MACConfig.args(variant, netLength=L)
    params = MACParams(cfg, L, values=perturb_biases(init_params(cfg, L, seed=100), seed=101))
    x = {k: torch.from_numpy(v).cuda() for k, v in make_inputs(B, S, N, d, seed=1234).items()}
    cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], x["knowledgeBase"],
                   1.0, 1.0, 1.0, B, False, config=cfg, params=params, prec="bf16", small_tc=True, fold_y=False)
    return cell, (B, S, N, d, L)


def breakdown():
    """Per-kernel device times of one headline pass (one stream, no graph)."""
    import torch
    from mac_network_b200.mac_cell import mac_network
    cell, (B, S, N, d, L) = headline_cell()
    for _ in range(3):
        mac_network(cell, L)
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        mac_network(cell, L)
        torch.cuda.synchronize()
    kernels = []
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time > 0 and "Memcpy" not in e.name \
                and "Memset" not in e.name:
            kernels.append((e.time_range.start, e.name, e.device_time))
    kernels.sort()
    seq = [{"kernel": n[:80], "us": round(t, 2)} for _, n, t in kernels]
    per = {}
    for _, n, t in kernels:
        k = n[:80]
        c, s = per.get(k, (0, 0.0))
        per[k] = (c + 1, s + t)
    total = sum(t for _, _, t in kernels)
    return {"launches": len(seq), "device_us_sum": round(total, 1), "sequence": seq,
            "per_kernel": sorted(({"kernel": k, "launches": c, "us": round(s, 1)} for k, (c, s) in per.items()),
                                 key=lambda r: -r["us"])}


def setup_time(R=6, iters=200, blocks=5, fused=False):
    """cast + P + Q per pass as MACCell runs them (mac_cast_bf16 + mac_read_invariant), or in one launch
    (mac_read_invariant_cast) with `fused`; CUDA events, inputs rotating over R > L2 sets."""
    import torch
    from mac_network_b200 import _lib
    from mac_network_b200._lib import check, ptr, stream_ptr
    cell, (B, S, N, d, L) = headline_cell()
    lib = _lib.load()
    rw = cell._read_weights("")
    g = torch.Generator(device="cuda").manual_seed(7)
    nb = lib.mac_read_invariant_bytes(B, N, d, 1)
    kbs = [torch.nn.functional.elu(torch.randn(B, N, d, device="cuda", generator=g)) for _ in range(R)]
    k16 = [torch.empty(B, N, d, dtype=torch.bfloat16, device="cuda") for _ in range(R)]
    invs = [torch.empty(nb, dtype=torch.uint8, device="cuda") for _ in range(R)]

    def one(i):
        if fused:
            check(lib.mac_read_invariant_cast(ptr(kbs[i]), ptr(k16[i]), ctypes.byref(rw), 1, ptr(invs[i]), nb, B, N, d,
                                              stream_ptr()), "mac_read_invariant_cast")
        else:
            check(lib.mac_cast_bf16(ptr(kbs[i]), ptr(k16[i]), kbs[i].numel(), stream_ptr()), "mac_cast_bf16")
            check(lib.mac_read_invariant(None, ptr(k16[i]), ctypes.byref(rw), 1, ptr(invs[i]), nb, B, N, d, stream_ptr()),
                  "mac_read_invariant")
    for i in range(2 * R):
        one(i % R)
    torch.cuda.synchronize()
    per = []
    for _ in range(blocks):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(iters):
            one(i % R)
        b.record()
        torch.cuda.synchronize()
        per.append(a.elapsed_time(b) * 1e3 / iters)
    return {"fused": fused, "us_per_pass": float(np.median(per)), "blocks_us": [round(x, 2) for x in per],
            "rotating_sets": R, "set_mb": round((kbs[0].numel() * 4 + k16[0].numel() * 2 + nb) / 1e6, 1)}


def worker(tree, what):
    sys.path.insert(0, tree)
    out = {"setup": setup_time} if what == "setup" else {"breakdown": breakdown, "setup": setup_time}
    if what == "all" and hasattr(__import__("mac_network_b200._lib", fromlist=["load"]).load(), "mac_read_invariant_cast"):
        out["setup_one_launch"] = lambda: setup_time(fused=True)
    print(json.dumps({k: f() for k, f in out.items()}))


def run_worker(tree, what):
    out = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", what, "--tree", tree],
                         capture_output=True, text=True, timeout=1800, cwd=tree)
    if out.returncode != 0:
        raise RuntimeError("worker %s: exit %d: %s" % (what, out.returncode, out.stderr[-3000:]))
    return json.loads(out.stdout.strip().splitlines()[-1])


def bench(tree, extra, timeout_s=1800):
    out = subprocess.run([sys.executable, os.path.join(tree, "bench.py")] + extra, capture_output=True, text=True,
                         timeout=timeout_s, cwd=tree)
    if out.returncode != 0:
        raise RuntimeError("bench.py %s: exit %d: %s" % (" ".join(extra), out.returncode, out.stderr[-2000:]))
    line = json.loads(out.stdout.strip().splitlines()[-1])
    print("%s %s: %s" % (tree, " ".join(extra), line.get("value")), flush=True)
    return line


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
    out = {"device": device_info(), "shape_B_N_d": [64, 196, 512]}
    out["new"] = run_worker(ROOT, "all")
    if args.base_tree:
        trees = {"base": os.path.abspath(args.base_tree), "new": ROOT}
        out["base"] = run_worker(trees["base"], "all")
        setup = {s: [] for s in SIDES}
        for _ in range(args.runs):
            for s in SIDES:
                setup[s].append(run_worker(trees[s], "setup")["setup"]["us_per_pass"])
        out["setup_us_per_pass"] = {s: spread(setup[s]) for s in SIDES}
        if not args.skip_bench:
            tmp = tempfile.mkdtemp(prefix="read_setup_")
            try:
                dumps = {s: os.path.join(tmp, "dump_" + s) for s in SIDES}
                lines = {s: {"headline": [], "bf16_gqa": [], "e2e": []} for s in SIDES}
                for i in range(args.runs):
                    for s in SIDES:
                        extra = ["--gpus", "1", "--steps", "480", "--warmup", "12", "--skip-cpu", "--skip-train"]
                        line = bench(trees[s], extra + (["--dump-outputs", dumps[s]] if i == 0 else []))
                        lines[s]["headline"].append(line["value"])
                        lines[s]["e2e"].append(line["e2e"]["value"])
                        lines[s]["bf16_gqa"].append(bench(trees[s], GQA)["value"])
                out["reasoning_steps_per_s"] = {s: {k: spread(v) for k, v in lines[s].items()} for s in SIDES}
                out["headline_speedup"] = (out["reasoning_steps_per_s"]["new"]["headline"]["median"] /
                                           out["reasoning_steps_per_s"]["base"]["headline"]["median"])
                same = {}
                for name in sorted(os.listdir(dumps["base"])):
                    a, b = np.load(os.path.join(dumps["base"], name)), np.load(os.path.join(dumps["new"], name))
                    same[name] = bool(a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes())
                out["outputs_bit_identical"] = same
            finally:
                shutil.rmtree(tmp, ignore_errors=True)
    out["device_after"] = device_info()
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "read_setup_h100.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({k: v for k, v in out.items() if k not in ("new", "base")}))
    for s in ("base", "new"):
        if s in out:
            print(s, json.dumps(out[s]["setup"]), json.dumps(out[s]["breakdown"]["per_kernel"][:12]))


if __name__ == "__main__":
    main()
