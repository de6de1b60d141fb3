"""ORACLE (test infrastructure only): fp64 restatement of the tensor-core question encoder (`QuestionEncoder(prec="bf16")`,
csrc/encoder_tc.cuh).  Never imported by the product path.

Every matrix-product operand is rounded to bf16 where the kernels round it, everything else is fp64:
  forward    gx = bf16(dropout(X)) @ bf16(kernel[0:E]) + bias;  gates(s) = gx(t) + bf16(h(s)) @ bf16(kernel[E:])
  backward   dh(s) = d_out(t) + bf16(dG(s+1)) @ bf16(kernel[E:])^T  (d_vecq at the last live step instead);
             dKernel = [bf16(dropout(X)) | bf16(h_prev)]^T @ bf16(dG);  dBias = colsum(dG);  dX = sum_dir bf16(dG) @ bf16(kernel[0:E])^T
With `bf16=False` no rounding happens and the functions restate `encoder_oracle.encoder_forward` and the gradients of
`encoder_torch_autograd.run` (tests/test_encoder_tc_host.py checks both)."""
import numpy as np
import torch

from oracle.encoder_oracle import ENC, ENC_UNI, embed


def _sig(x):
    return 1.0 / (1.0 + np.exp(-x))


def _mask(u, keep):
    return np.floor(keep + np.asarray(u, np.float64)) / keep


class EncoderTC(object):
    def __init__(self, params, keep_input=1.0, keep_question=1.0, uniforms=None, forget_bias=1.0, bf16=True):
        """`params`: TF-name -> array; `uniforms`: the kernels' draws in call order (`QuestionEncoder.dropout_uniforms`)."""
        self.p = {k: np.asarray(v, np.float64) for k, v in params.items()}
        self.keep_input, self.keep_question, self.fb, self.bf16 = float(keep_input), float(keep_question), forget_bias, bf16
        us = list(uniforms or [])
        self.u_in = us.pop(0) if self.keep_input < 1.0 else None
        self.u_q = us.pop(0) if self.keep_question < 1.0 else None
        self.scopes = [ENC_UNI] if (ENC_UNI + "basic_lstm_cell/kernel") in self.p else [ENC + "fw/", ENC + "bw/"]

    def r(self, a):
        if not self.bf16:
            return np.asarray(a, np.float64)
        return torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(torch.bfloat16).to(torch.float64).numpy()

    def forward(self, qIndices, lengths):
        """-> dict(questionWords, questionCntxWords, vecQuestions, x16, and per direction gates / c / hprev [B, S, .])."""
        words = embed(self.p["qEmbeddings/emb"], qIndices)
        x = words * _mask(self.u_in, self.keep_input) if self.u_in is not None else words
        B, S, E = x.shape
        lengths = np.asarray(lengths).astype(np.int64)
        self.q, self.lengths, self.x16 = np.asarray(qIndices), lengths, self.r(x)
        outs, finals, self.saved = [], [], []
        for d, sc in enumerate(self.scopes):
            K, b = self.p[sc + "basic_lstm_cell/kernel"], self.p[sc + "basic_lstm_cell/bias"]
            h_dim = K.shape[1] // 4
            gx = self.x16 @ self.r(K[:E]) + b
            Wh = self.r(K[E:])
            out = np.zeros((B, S, h_dim))
            gates = np.zeros((B, S, 4 * h_dim))
            cs = np.zeros((B, S, h_dim))
            hps = np.zeros((B, S, h_dim))
            c, h = np.zeros((B, h_dim)), np.zeros((B, h_dim))
            rows = np.arange(B)
            for s in range(S):
                live = s < lengths
                t = np.where(live, (lengths - 1 - s) if d == 1 else s, 0)
                g = gx[rows, t] + self.r(h) @ Wh
                i, j, f, o = np.split(g, 4, axis=1)
                i, j, f, o = _sig(i), np.tanh(j), _sig(f + self.fb), _sig(o)
                cn = c * f + i * j
                hn = np.tanh(cn) * o
                lr = np.nonzero(live)[0]
                out[lr, t[lr]] = hn[lr]
                gates[lr, t[lr]] = np.concatenate([i, j, f, o], axis=1)[lr]
                cs[lr, t[lr]] = cn[lr]
                hps[lr, t[lr]] = h[lr]
                c = np.where(live[:, None], cn, c)
                h = np.where(live[:, None], hn, h)
            outs.append(out)
            finals.append(h)
            self.saved.append(dict(gates=gates, c=cs, hprev=hps, Wh=Wh, Wx=self.r(K[:E])))
        cntx = np.concatenate(outs, axis=-1)
        vecq = np.concatenate(finals, axis=-1)
        if self.u_q is not None:
            vecq = vecq * _mask(self.u_q, self.keep_question)
        return dict(questionWords=words, questionCntxWords=cntx, vecQuestions=vecq, x16=self.x16,
                    gates=[sv["gates"] for sv in self.saved], c=[sv["c"] for sv in self.saved],
                    hprev=[sv["hprev"] for sv in self.saved])

    def backward(self, d_cntx, d_vecq):
        """Gradients (dict TF-name -> array) of sum(d_cntx * cntx) + sum(d_vecq * vecq) after `forward`."""
        d_cntx, d_vecq = np.asarray(d_cntx, np.float64), np.asarray(d_vecq, np.float64)
        if self.u_q is not None:
            d_vecq = d_vecq * _mask(self.u_q, self.keep_question)
        B, S, E = self.x16.shape
        lengths, rows = self.lengths, np.arange(B)
        grads, dx = {}, np.zeros((B, S, E))
        for d, sc in enumerate(self.scopes):
            sv = self.saved[d]
            h_dim = sv["Wh"].shape[0]
            dG = np.zeros((B, S, 4 * h_dim))
            dcc = np.zeros((B, h_dim))
            dG_next = np.zeros((B, 4 * h_dim))                 # gate gradients of step s+1 by batch row (0 where not live)
            for s in range(S - 1, -1, -1):
                live = s < lengths
                t = np.where(live, (lengths - 1 - s) if d == 1 else s, 0)
                dh = d_cntx[rows, t, d * h_dim:(d + 1) * h_dim]
                rec = self.r(dG_next) @ sv["Wh"].T
                last = (s + 1 >= lengths)[:, None]
                dh = dh + np.where(last, d_vecq[:, d * h_dim:(d + 1) * h_dim], rec)
                g = sv["gates"][rows, t]
                gi, gj, gf, go = np.split(g, 4, axis=1)
                cn = sv["c"][rows, t]
                tp = np.clip(t + 1 if d == 1 else t - 1, 0, S - 1)
                cp = np.where(s > 0, sv["c"][rows, tp], 0.0)
                tc = np.tanh(cn)
                dc = dcc + dh * go * (1 - tc * tc)
                dg = np.concatenate([dc * gj * gi * (1 - gi), dc * gi * (1 - gj * gj), dc * cp * gf * (1 - gf),
                                     dh * tc * go * (1 - go)], axis=1)
                dg = np.where(live[:, None], dg, 0.0)
                dcc = np.where(live[:, None], dc * gf, dcc)
                lr = np.nonzero(live)[0]
                dG[lr, t[lr]] = dg[lr]
                dG_next = dg
            dG16 = self.r(dG.reshape(B * S, -1))
            xh = np.concatenate([self.x16.reshape(B * S, E), self.r(sv["hprev"].reshape(B * S, -1))], axis=1)
            grads[sc + "basic_lstm_cell/kernel"] = xh.T @ dG16
            grads[sc + "basic_lstm_cell/bias"] = dG.reshape(B * S, -1).sum(axis=0)
            dx += (dG16 @ sv["Wx"].T).reshape(B, S, E)
        if self.u_in is not None:
            dx = dx * _mask(self.u_in, self.keep_input)
        demb = np.zeros_like(self.p["qEmbeddings/emb"])
        q = self.q.reshape(-1)
        np.add.at(demb, q[q > 0] - 1, dx.reshape(B * S, E)[q > 0])
        grads["qEmbeddings/emb"] = demb
        return grads
