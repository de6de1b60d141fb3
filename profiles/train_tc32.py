"""One training step of the cell at fp32, tc32 (split-bf16 tensor cores inside the fp32 parity bar) and bf16, alternating in
one process.  Usage:  python profiles/train_tc32.py OUT_DIR [--rounds 5] [--window 0.5]
  fp32   DPTrainer(prec="fp32")                 the parity configuration: every product on the FMA pipe
  tc32   DPTrainer(prec="tc32", bwd_tc=True)     mac_read_fwd's split-bf16 training form + mac_read_bwd_tc32
  bf16   DPTrainer(prec="bf16", bwd_tc=True)     bf16 operands (~1e-3), for scale
`DPTrainer.train_step` (cell forward with the training dropouts, mac_backward, apply) at two shapes: the bench training shape
(B=64, S=40, N=196, d=512, L=12) and BASELINE.json config (2) (B=32, S=20, N=196, d=512, L=4).  Each arm runs at least
`rounds` timed windows (profiles/stem_train_tc.py's `compare`).
It also times the two forms of a split-bf16 weight gradient dW[in, out] += X^T G over K = B*N at both shapes, for the three
weights of the read unit ([512, 512] twice and [1024, 512]):
  one_launch   tc3_wgrad_splitk: [X_hi^T | X_lo^T] against [G_hi^T | G_hi^T | G_lo^T], ONE split-K launch over 3K (what
               mac_read_bwd_tc32 runs)
  three_calls  three accumulating tc_wgrad_splitk calls (X_hi G_hi, X_lo G_hi, X_hi G_lo) on contiguous hi / lo slabs
Medians and ranges go to OUT_DIR/train_tc32.json with the card's name, power limit and max SM clock, read in the same call."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

from mac_network_b200 import _lib  # noqa: E402
from mac_network_b200.config import MACConfig  # noqa: E402
from mac_network_b200.dp import DPTrainer  # noqa: E402
from mac_network_b200.synthetic import SHAPES, make_inputs  # noqa: E402
from profiles.stem_train_tc import compare, device_info  # noqa: E402

ARMS = {"fp32": dict(prec="fp32"), "tc32": dict(prec="tc32", bwd_tc=True), "bf16": dict(prec="bf16", bwd_tc=True)}


def shape_part(shape, rounds, window_s):
    B, S, N, d, L = shape
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    x = {k: torch.from_numpy(v).cuda() for k, v in make_inputs(B, S, N, d, seed=3).items()}
    g = torch.Generator(device="cuda").manual_seed(5)
    tc_, tm_ = torch.randn(B, d, device="cuda", generator=g), torch.randn(B, d, device="cuda", generator=g)
    trainers = {p: DPTrainer(cfg, L, seed=6, **kw) for p, kw in ARMS.items()}
    r = compare({p: (lambda tr=tr: tr.train_step(0, x, tc_, tm_, B)) for p, tr in trainers.items()}, rounds, window_s)
    del trainers
    torch.cuda.empty_cache()
    for v in r.values():
        v["ms_range"] = [min(v["ms_rounds"]), max(v["ms_rounds"])]
    return {"shape": {"B": B, "S": S, "N": N, "d": d, "L": L},
            "dropouts_train": [cfg.memoryDropout, cfg.readDropout, cfg.writeDropout], "train_step": r,
            "speedup_tc32_over_fp32": r["fp32"]["ms"] / r["tc32"]["ms"],
            "speedup_bf16_over_fp32": r["fp32"]["ms"] / r["bf16"]["ms"]}


def _wgrad_lib():
    """the library's internal split-K weight-gradient exports (units.cu; not part of the ABI header)"""
    lib = _lib.load()
    c_fp, c_int = ctypes.c_void_p, ctypes.c_int
    lib.mac_tc_wgrad_splitk_.restype = lib.mac_tc3_wgrad_splitk_.restype = c_int
    lib.mac_tc_wgrad_splitk_.argtypes = lib.mac_tc3_wgrad_splitk_.argtypes = [c_fp, c_fp, c_fp, c_fp, c_int, c_int, c_int,
                                                                              c_fp]
    lib.mac_tc_wgrad_partial_bytes_.restype = ctypes.c_size_t
    lib.mac_tc_wgrad_partial_bytes_.argtypes = [c_int, c_int]
    return lib


def _time(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def wgrad_forms(M, rounds, iters=50):
    """the two split-bf16 weight-gradient forms for the read unit's three weights at contraction M (ms per backward call of
    all three, median and range over `rounds` alternating windows of `iters` calls), and their largest disagreement"""
    lib = _wgrad_lib()
    P = _lib.ptr
    st = _lib.stream_ptr()
    Mp = (M + 63) // 64 * 64
    g = torch.Generator(device="cuda").manual_seed(7)
    split = lambda t: (t.to(torch.bfloat16), (t - t.to(torch.bfloat16).float()).to(torch.bfloat16))
    padT = lambda t: torch.nn.functional.pad(t.t(), (0, Mp - M)).contiguous()          # [cols, Mp], zero columns M..Mp-1
    cases = []
    for n_in in (512, 1024, 512):
        X, G = torch.randn(M, n_in, device="cuda", generator=g), torch.randn(M, 512, device="cuda", generator=g)
        (xh, xl), (gh, gl) = split(X), split(G)
        xh, xl, gh, gl = padT(xh), padT(xl), padT(gh), padT(gl)
        cases.append(dict(n_in=n_in, xh=xh, xl=xl, gh=gh, gl=gl, xT2=torch.cat([xh, xl], 1).contiguous(),
                          gT3=torch.cat([gh, gh, gl], 1).contiguous(), dW1=torch.zeros(n_in, 512, device="cuda"),
                          dW3=torch.zeros(n_in, 512, device="cuda")))
    part = torch.empty(int(lib.mac_tc_wgrad_partial_bytes_(1024, 512)) // 4, device="cuda")

    def one():
        for c in cases:
            _lib.check(lib.mac_tc3_wgrad_splitk_(P(c["xT2"]), P(c["gT3"]), P(c["dW1"]), P(part), c["n_in"], 512, Mp, st), "tc3")

    def three():
        for c in cases:
            for a, b in ((c["xh"], c["gh"]), (c["xl"], c["gh"]), (c["xh"], c["gl"])):
                _lib.check(lib.mac_tc_wgrad_splitk_(P(a), P(b), P(c["dW3"]), P(part), c["n_in"], 512, Mp, st), "tc")

    for c in cases:
        c["dW1"].zero_(), c["dW3"].zero_()
    one(), three()
    torch.cuda.synchronize()
    diff = max(float((c["dW1"] - c["dW3"]).abs().max() / c["dW3"].abs().max()) for c in cases)
    rows = {"one_launch": [], "three_calls": []}
    for fn in (one, three):
        _time(fn, 5)
    for _ in range(rounds):
        rows["one_launch"].append(_time(one, iters))
        rows["three_calls"].append(_time(three, iters))
    return {"M": M, "Mp": Mp, "max_rel_disagreement": diff,
            **{k: {"ms": float(np.median(v)), "ms_range": [min(v), max(v)], "ms_rounds": [round(x, 4) for x in v]}
               for k, v in rows.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_tc32.py measures on a CUDA device; none is visible")
    os.makedirs(a.out_dir, exist_ok=True)
    out = {"device": device_info(), "rounds": a.rounds, "shapes": {}}
    for name, shape in (("bench_train", SHAPES["headline"]), ("baseline_config_2", SHAPES["cpu_ref"])):
        out["shapes"][name] = r = shape_part(shape, a.rounds, a.window)
        t = r["train_step"]
        print("%s %s: train_step fp32 %.2f ms [%.2f, %.2f], tc32 %.2f ms [%.2f, %.2f], bf16 %.2f ms [%.2f, %.2f]" % (
            name, shape, t["fp32"]["ms"], *t["fp32"]["ms_range"], t["tc32"]["ms"], *t["tc32"]["ms_range"], t["bf16"]["ms"],
            *t["bf16"]["ms_range"]), flush=True)
        with open(os.path.join(a.out_dir, "train_tc32.json"), "w") as f:
            json.dump(out, f, indent=1)
    out["wgrad_forms"] = {}
    for name, shape in (("bench_train", SHAPES["headline"]), ("baseline_config_2", SHAPES["cpu_ref"])):
        out["wgrad_forms"][name] = r = wgrad_forms(shape[0] * shape[2], a.rounds)
        print("%s wgrad (dWx, dWm, dWm2), M = %d: one launch %.3f ms [%.3f, %.3f], three calls %.3f ms [%.3f, %.3f] "
              "(disagree by %.1e)" % (name, r["M"], r["one_launch"]["ms"], *r["one_launch"]["ms_range"],
                                      r["three_calls"]["ms"], *r["three_calls"]["ms_range"], r["max_rel_disagreement"]),
              flush=True)
        with open(os.path.join(a.out_dir, "train_tc32.json"), "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out["device"]), flush=True)


if __name__ == "__main__":
    main()
