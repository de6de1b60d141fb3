"""ORACLE (test infrastructure only): differentiable fp64 PyTorch restatement of the question input unit
(`model.py:208-220, 279-307`, `ops.py:859-905`; TF-1 `BasicLSTMCell` / `bidirectional_dynamic_rnn` semantics as in
`oracle/encoder_oracle.py`), used to check the hand-written BPTT kernels against `torch.autograd` (the reference uses TF
autodiff, `model.py:626-636`).  Its forward is pinned to the numpy oracle in `tests/test_encoder.py`."""
import torch

ENC = "encoder/birnnLayer/bidirectional_rnn/"


def graph(p, qIndices, lengths, keep_input=1.0, keep_question=1.0, uniforms=None, forget_bias=1.0):
    """The encoder as a differentiable graph: `p` maps variable names to fp64 tensors on one device, `qIndices` [B, S]
    and `lengths` [B] are long tensors there.  Returns (questionWords, questionCntxWords, vecQuestions) tensors;
    questionWords is the embedding lookup before the input dropout.  `uniforms`: the draws in the reference's call order
    (an iterator is consumed as far as the dropouts need)."""
    dev = p["qEmbeddings/emb"].device
    t64 = lambda a: torch.as_tensor(a, dtype=torch.float64).to(dev)
    us = iter(uniforms or [])

    def dropout(x, keep):
        if float(keep) == 1.0:
            return x
        return x / keep * torch.floor(keep + t64(next(us)))

    idx, lens = qIndices, lengths
    B, S = idx.shape
    emb = p["qEmbeddings/emb"]
    table = torch.cat([torch.zeros(1, emb.shape[1], dtype=torch.float64, device=dev), emb], 0)
    words = table[idx]
    x = dropout(words, keep_input)
    outs, finals = [], []
    ar = torch.arange(B, device=dev)
    uni = "encoder/rnnLayer/rnn/basic_lstm_cell/kernel" in p
    for name, reverse in ((("", False),) if uni else (("fw", False), ("bw", True))):
        sc = "encoder/rnnLayer/rnn/" if uni else ENC + name + "/"
        K, bias = p[sc + "basic_lstm_cell/kernel"], p[sc + "basic_lstm_cell/bias"]
        hd = K.shape[1] // 4
        c = torch.zeros(B, hd, dtype=torch.float64, device=dev)
        h = torch.zeros(B, hd, dtype=torch.float64, device=dev)
        out = torch.zeros(B, S, hd, dtype=torch.float64, device=dev)
        for s in range(S):
            live = (s < lens)
            t = torch.where(live, (lens - 1 - s) if reverse else torch.full_like(lens, s), torch.zeros_like(lens))
            g = torch.cat([x[ar, t], h], 1) @ K + bias
            i, j, f, o = g.split(hd, dim=1)
            cn = c * torch.sigmoid(f + forget_bias) + torch.sigmoid(i) * torch.tanh(j)
            hn = torch.tanh(cn) * torch.sigmoid(o)
            lv = live.unsqueeze(1)
            c = torch.where(lv, cn, c)
            h = torch.where(lv, hn, h)
            upd = torch.zeros(B, S, hd, dtype=torch.float64, device=dev)
            upd[ar, t] = torch.where(lv, hn, torch.zeros_like(hn))
            out = out + upd
        outs.append(out)
        finals.append(h)
    cntx = torch.cat(outs, -1)
    vecq = dropout(torch.cat(finals, -1), keep_question)
    if "encoder/linearLayerprojCW/weights/weight" in p:
        cntx = cntx @ p["encoder/linearLayerprojCW/weights/weight"] + p["encoder/linearLayerprojCW/biases/bias"]
        vecq = vecq @ p["encoder/linearLayerprojQ/weights/weight"] + p["encoder/linearLayerprojQ/biases/bias"]
    return words, cntx, vecq


def run(params_np, qIndices, lengths, keep_input=1.0, keep_question=1.0, uniforms=None, d_cntx=None, d_vecq=None,
        forget_bias=1.0):
    """Returns (cntx, vecq, grads: name -> d(sum(cntx*d_cntx) + sum(vecq*d_vecq))/d param)."""
    t64 = lambda a: torch.tensor(a, dtype=torch.float64)
    p = {k: t64(v).requires_grad_(True) for k, v in params_np.items()}
    _, cntx, vecq = graph(p, torch.as_tensor(qIndices).long(), torch.as_tensor(lengths).long(), keep_input, keep_question,
                          uniforms, forget_bias)
    grads = {}
    if d_cntx is not None:
        loss = (cntx * t64(d_cntx)).sum() + (vecq * t64(d_vecq)).sum()
        loss.backward()
        grads = {k: v.grad.numpy() for k, v in p.items() if v.grad is not None}
    return cntx.detach().numpy(), vecq.detach().numpy(), grads
