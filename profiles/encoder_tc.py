"""The question encoder in fp32 against bf16 on tensor cores (QuestionEncoder(prec="bf16")), on its own and inside the whole
model.  Usage:  python profiles/encoder_tc.py OUT_DIR [--rounds 3] [--window 0.5]
  encoder:   QuestionEncoder.forward, and forward(save_for_backward=True) + backward with the training dropouts (0.85, 0.92),
             at B=64, S=40, E=300, 2 x 256 (profiles/lstm_bench.py's shape)
  train:     DPTrainer.train_step_full at the bench.py train_full shape, cell prec="bf16", bwd_tc=True, stem_prec="bf16",
             enc_prec="fp32" against "bf16"
  eval:      MACnet.runBatch(train=False) at the same shape with prec="fp8" and the e4m3 stem, eval_enc_prec None against "bf16"
Both arms of a comparison alternate in one process (profiles/stem_train_tc.py's `compare`).  Writes OUT_DIR/encoder_tc.json
with the card's name, power limit and max SM clock."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from mac_network_b200.config import MACConfig  # noqa: E402
from mac_network_b200.dp import DPTrainer  # noqa: E402
from mac_network_b200.encoder import QuestionEncoder, encoder_specs, init_encoder_params  # noqa: E402
from mac_network_b200.model import MACnet  # noqa: E402
from mac_network_b200.synthetic import SHAPES  # noqa: E402
from profiles.stem_train_tc import compare, device_info  # noqa: E402

V, E, A, C_IN, HW = 90, 300, 28, 1024, 14


def _questions(B, S, seed):
    rng = np.random.RandomState(seed)
    lengths = rng.randint(S // 2, S + 1, size=(B,)).astype(np.int32)
    lengths[0] = S
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    return q, lengths, rng


def encoder_part(rounds, window_s):
    B, S, D = 64, 40, 512
    pv = init_encoder_params(encoder_specs(V, E, D), seed=1)
    dev = {k: torch.from_numpy(v).cuda() for k, v in pv.items()}
    q, lengths, _ = _questions(B, S, 2)
    qd, ld = torch.from_numpy(q).cuda(), torch.from_numpy(lengths).cuda()
    dc, dq = torch.randn(B, S, D, device="cuda"), torch.randn(B, D, device="cuda")
    grads = {k: torch.zeros_like(v) for k, v in dev.items()}
    encs = {p: QuestionEncoder(dev, prec=p) for p in ("fp32", "bf16")}
    encs_t = {p: QuestionEncoder(dev, keep_input=0.85, keep_question=0.92, prec=p) for p in ("fp32", "bf16")}

    def fb(p):
        encs_t[p].forward(qd, ld, step=1, save_for_backward=True)
        encs_t[p].backward(dc, dq, grads)

    fwd = compare({p: (lambda p=p: encs[p].forward(qd, ld)) for p in encs}, rounds, window_s)
    train = compare({p: (lambda p=p: fb(p)) for p in encs_t}, rounds, window_s)
    return {"shape": {"B": B, "S": S, "E": E, "encDim": D}, "forward": fwd, "forward_backward": train,
            "speedup_forward": fwd["fp32"]["ms"] / fwd["bf16"]["ms"],
            "speedup_forward_backward": train["fp32"]["ms"] / train["bf16"]["ms"]}


def whole_parts(rounds, window_s):
    Bm, S, N, d, L = SHAPES["headline"]
    cfg = MACConfig.args("args", netLength=L)
    q, lengths, rng = _questions(Bm, S, 31)
    answers = rng.randint(0, A, size=(Bm,)).astype(np.int32)
    images = torch.relu(torch.randn(Bm, HW, HW, C_IN, device="cuda"))
    data = {"questions": torch.from_numpy(q).cuda(), "questionLengths": torch.from_numpy(lengths).cuda(),
            "images": images, "answers": torch.from_numpy(answers).cuda()}
    trainers = {ep: DPTrainer(cfg, L, seed=7, classifier=(A, [512]), encoder=(V, E), stem=(C_IN, 2), prec="bf16",
                              bwd_tc=True, stem_prec="bf16", enc_prec=ep) for ep in ("fp32", "bf16")}
    train = compare({ep: (lambda tr=tr: tr.train_step_full(0, data, Bm)) for ep, tr in trainers.items()}, rounds, window_s)
    del trainers
    torch.cuda.empty_cache()
    nets = {ep: MACnet(cfg, L, V, A, wrd_emb_dim=E, image_in_dim=C_IN, classifier_dims=(512,), prec="fp8",
                       eval_stem_prec="fp8", eval_enc_prec=ep) for ep in (None, "bf16")}
    bd = {"questions": q, "questionLengths": lengths, "answers": answers}
    img = {"images": images.permute(0, 3, 1, 2).contiguous()}
    ev = compare({str(ep): (lambda n=n: n.runBatch(None, bd, img, train=False)) for ep, n in nets.items()}, rounds, window_s)
    shape = {"B": Bm, "S": S, "N": N, "d": d, "L": L, "stem_in": C_IN}
    return ({"shape": shape, "cell": "prec=bf16, bwd_tc=True, stem_prec=bf16", "arms": train,
             "saved_ms": train["fp32"]["ms"] - train["bf16"]["ms"]},
            {"shape": shape, "model": "prec=fp8, eval_stem_prec=fp8", "arms": ev,
             "saved_ms": ev["None"]["ms"] - ev["bf16"]["ms"]})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window", type=float, default=0.5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("encoder_tc.py measures on a CUDA device; none is visible")
    os.makedirs(a.out_dir, exist_ok=True)
    out = {"device": device_info(), "rounds": a.rounds}
    out["encoder"] = encoder_part(a.rounds, a.window)
    print(json.dumps({"encoder": out["encoder"]}), flush=True)
    torch.cuda.empty_cache()
    out["train_step_full"], out["run_batch_eval"] = whole_parts(a.rounds, a.window)
    with open(os.path.join(a.out_dir, "encoder_tc.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({k: out[k] for k in ("device", "train_step_full", "run_batch_eval")}), flush=True)


if __name__ == "__main__":
    main()
