"""fp32 against bf16 tensor cores for flag sets outside the shipped flag files (SURVEY section 8(a), "P2") at the headline
shape.  Usage:  python profiles/general_tc.py OUT_DIR [--rounds 5] [--window 0.5] [--cases p2_read_bl,...]
  p2_read_bl, p2_read_add     the composed read unit: [B*N, .] products on mac_linear_tc_seg_fwd / mac_linear_bwd_tc
  p2_unshared, p2_memory_bn   the fused read unit differentiated on the tape: mac_read_bwd_tc
For each flag set (the fixture's flags at B=64, S=40, N=196, d=512, L=12):
  inference:  MACCell(train=False) + mac_network, prec="fp32" against "bf16"
  training:   DPTrainer.train_step (cell forward with the training dropouts, mac_backward, all-reduce-free apply),
              prec="fp32" against prec="bf16", bwd_tc=True
Both arms alternate in one process (profiles/stem_train_tc.py's `compare`).  Writes OUT_DIR/general_tc.json with the card's
name, power limit and max SM clock."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from mac_network_b200.config import MACConfig  # noqa: E402
from mac_network_b200.dp import DPTrainer  # noqa: E402
from mac_network_b200.mac_cell import MACCell, MACParams, mac_network  # noqa: E402
from mac_network_b200.synthetic import SHAPES, make_inputs  # noqa: E402
from profiles.stem_train_tc import compare, device_info  # noqa: E402
from tests._util import load_golden  # noqa: E402

CASES = ["p2_read_bl", "p2_read_add", "p2_unshared", "p2_memory_bn"]


def case_part(case, rounds, window_s):
    B, S, N, d, L = SHAPES["headline"]
    meta, _ = load_golden(case)
    cfg = MACConfig(**dict(meta["cell_flags"], memDim=d, ctrlDim=d, attDim=d, netLength=L)).validate()
    x = {k: torch.from_numpy(v).cuda() for k, v in make_inputs(B, S, N, d, seed=3).items()}
    params = MACParams(cfg, L, seed=4)
    cells = {p: MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"],
                        x["knowledgeBase"], 1.0, 1.0, 1.0, B, False, config=cfg, params=params, prec=p)
             for p in ("fp32", "bf16")}
    inf = compare({p: (lambda c=c: mac_network(c, L)) for p, c in cells.items()}, rounds, window_s)
    del cells
    torch.cuda.empty_cache()
    g = torch.Generator(device="cuda").manual_seed(5)
    tc_, tm_ = torch.randn(B, d, device="cuda", generator=g), torch.randn(B, d, device="cuda", generator=g)
    trainers = {p: DPTrainer(cfg, L, seed=6, prec=p, bwd_tc=p == "bf16") for p in ("fp32", "bf16")}
    train = compare({p: (lambda tr=tr: tr.train_step(0, x, tc_, tm_, B)) for p, tr in trainers.items()}, rounds, window_s)
    del trainers
    torch.cuda.empty_cache()
    return {"flags": meta["argv"][:-8], "fused_read": bool(cfg.is_fast_path),
            "shape": {"B": B, "S": S, "N": N, "d": d, "L": L},
            "dropouts_train": [cfg.memoryDropout, cfg.readDropout, cfg.writeDropout],
            "inference": inf, "train_step": train,
            "speedup_inference": inf["fp32"]["ms"] / inf["bf16"]["ms"],
            "speedup_train_step": train["fp32"]["ms"] / train["bf16"]["ms"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.5)
    ap.add_argument("--cases", default=",".join(CASES))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("general_tc.py measures on a CUDA device; none is visible")
    os.makedirs(a.out_dir, exist_ok=True)
    out = {"device": device_info(), "rounds": a.rounds, "cases": {}}
    for case in a.cases.split(","):
        out["cases"][case] = case_part(case, a.rounds, a.window)
        r = out["cases"][case]
        print("%s: inference %.2f -> %.2f ms, train_step %.2f -> %.2f ms" % (
            case, r["inference"]["fp32"]["ms"], r["inference"]["bf16"]["ms"], r["train_step"]["fp32"]["ms"],
            r["train_step"]["bf16"]["ms"]), flush=True)
        with open(os.path.join(a.out_dir, "general_tc.json"), "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out["device"]), flush=True)


if __name__ == "__main__":
    main()
