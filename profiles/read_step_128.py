"""The 128-row read step (csrc/read_step.cuh) against the library of the commit before it, alternating in one session.
Usage:  python profiles/read_step_128.py OUT_DIR --base-lib PATH [--part rooflines|headline|both] [--runs 3] [--roof-runs 6]

  --base-lib   the earlier commit's libmac_b200.so (built from that commit's tree); the library this tree's build() made is
               the other side.  Each library runs from its own copy of this tree in a temporary directory.
  headline:    `bench.py --gpus 1 --steps 480 --warmup 12 --skip-cpu`, `--runs` times per library, alternating: the headline
               value, the bf16_gqa sub-line and both info_batched_requests lines (B = 384).
  rooflines:   `bench.py --rooflines-only`, `--roof-runs` times per library, alternating: read_step_fused (read-step kernel +
               kb_attend per reasoning step at the headline shape).
  outputs:     the first headline run of each library also writes --dump-outputs; the files are compared bit for bit.
`--part` runs only one of the two measurements (each takes minutes).  Also records the card (name, power limit, max SM
clock from nvidia-smi).  Writes OUT_DIR/read_step_128_<part>_h100.json."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_REL = os.path.join("mac_network_b200", "csrc", "libmac_b200.so")
SIDES = ("base", "new")


def device_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def spread(xs):
    xs = [float(x) for x in xs]
    return {"median": float(np.median(xs)), "min": min(xs), "max": max(xs), "runs": [round(x, 3) for x in xs]}


def tree_copy(dst, lib):
    shutil.copytree(ROOT, dst, ignore=shutil.ignore_patterns(".git", "*.o", "__pycache__"))
    shutil.copyfile(lib, os.path.join(dst, LIB_REL))
    return dst


def bench(tree, extra, timeout_s=1800):
    out = subprocess.run([sys.executable, os.path.join(tree, "bench.py")] + extra, capture_output=True, text=True,
                         timeout=timeout_s, cwd=tree)
    if out.returncode != 0:
        raise RuntimeError("bench.py %s: exit %d: %s" % (" ".join(extra), out.returncode, out.stderr[-2000:]))
    line = json.loads(out.stdout.strip().splitlines()[-1])
    print("%s %s: %s" % (os.path.basename(tree), " ".join(extra), line.get("value", "done")), flush=True)
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--base-lib", required=True)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--roof-runs", type=int, default=6)
    ap.add_argument("--part", default="both", choices=["rooflines", "headline", "both"])
    args = ap.parse_args()
    out = {"device": device_info(), "runs": args.runs, "roof_runs": args.roof_runs,
           "headline_args": "--gpus 1 --steps 480 --warmup 12 --skip-cpu"}
    tmp = tempfile.mkdtemp(prefix="read_step_128_")
    try:
        trees = {"base": tree_copy(os.path.join(tmp, "base"), os.path.abspath(args.base_lib)),
                 "new": tree_copy(os.path.join(tmp, "new"), os.path.join(ROOT, LIB_REL))}
        dumps = {s: os.path.join(tmp, "dump_" + s) for s in SIDES}

        roof = {s: [] for s in SIDES}
        for _ in range(args.roof_runs if args.part != "headline" else 0):
            for s in SIDES:
                roof[s].append(bench(trees[s], ["--rooflines-only"])["read_step_fused"]["us"])
        if args.part != "headline":
            out["read_step_fused_us"] = {s: spread(roof[s]) for s in SIDES}
            out["read_step_fused_speedup"] = (out["read_step_fused_us"]["base"]["median"] /
                                              out["read_step_fused_us"]["new"]["median"])
        if args.part == "rooflines":
            return finish(args, out)

        lines = {s: {"headline": [], "bf16_gqa": [], "batched_one_stream": [], "batched_two_streams": []} for s in SIDES}
        for i in range(args.runs):
            for s in SIDES:
                extra = ["--gpus", "1", "--steps", "480", "--warmup", "12", "--skip-cpu"]
                line = bench(trees[s], extra + (["--dump-outputs", dumps[s]] if i == 0 else []))
                lines[s]["headline"].append(line["value"])
                lines[s]["bf16_gqa"].append(line["sub_lines"]["bf16_gqa"]["value"])
                lines[s]["batched_one_stream"].append(line["info_batched_requests"]["requests_x6_one_stream"]["value"])
                lines[s]["batched_two_streams"].append(line["info_batched_requests"]["requests_x6_two_streams"]["value"])
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
    finish(args, out)


def finish(args, out):
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "read_step_128_%s_h100.json" % args.part)
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
