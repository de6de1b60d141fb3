"""Reverse sweep for the flag combinations outside the hand-scheduled backward of `autograd._Bwd` (the "other working
flags" of /root/reference/config.py:292-387: general read / write / control units, wordsProj, controlWholeQ,
controlContinuous, unsharedCells, ...).

The reference differentiates whatever graph its flags build with TF autodiff (model.py:626-636).  Here every primitive the
cell launches in a training forward (`MACCell._linear`, `_bcast`, `_rowdot`, `_act`, `_dropout`, the attention kernels, the
fused read / write units) appends one node to a tape; `Tape.run` walks the nodes backwards, each node calling the backward
kernel(s) of its primitive (csrc/backward.cu) on the gradient buffers of its inputs.  No host arithmetic: the tape only
decides which kernel runs on which buffers.

Gradient buffers are keyed by (data pointer, element count) of the forward tensor, so a reshaped view shares its
buffer with the tensor it views; the history slots c_0..c_L, m_0..m_L, info_0..info_L map onto rows of three [L+1, B, d]
buffers (the self-attention kernels walk those).  Buffers start at zero and every kernel accumulates.
"""
import collections
import ctypes

import torch

from ._lib import ACT, check, ptr, stream_ptr
from .autograd import read_bwd, read_bwd_workspace_bytes
from .params import PREFIX


class Tape(object):
    def __init__(self, cell):
        self.cell, self.lib, self.p = cell, cell.lib, cell.params
        self.nodes = []
        self.finalizers = []
        self.grads = {}
        self.dev = cell.device
        self._names = {t.data_ptr(): n for n, t in self.p.t.items()}
        self.bucket = None
        self.g = None
        self.lws_bytes = 4096 + 32 * 4 * max(int(t.numel()) for t in self.p.t.values())
        self.lws = None
        self.tc = False              # run(tc=True): the [B*N, .] products of the backward on tensor cores
        self._tcws = None

    # ------------------------------------------------------------------ buffers
    def z(self, *shape):
        return torch.zeros(shape, dtype=torch.float32, device=self.dev)

    def e(self, *shape):
        return torch.empty(shape, dtype=torch.float32, device=self.dev)

    def register_history(self, hist):
        """[L+1, B, d] forward history -> one gradient buffer whose rows are the gradients of the slots."""
        gh = torch.zeros_like(hist)
        for i in range(hist.shape[0]):
            self.grads[(hist[i].data_ptr(), hist[i].numel())] = gh[i]
        return gh

    def grad(self, t):
        """Gradient buffer of forward tensor `t` (zero on first use), shaped like `t`."""
        if not t.is_contiguous():
            raise NotImplementedError("tape gradients need contiguous forward tensors")
        key = (t.data_ptr(), t.numel())
        gbuf = self.grads.get(key)
        if gbuf is None:
            gbuf = self.grads[key] = torch.zeros(t.numel(), dtype=torch.float32, device=self.dev)
        return gbuf.view(t.shape)

    def name_of(self, t):
        return self._names[t.data_ptr()]

    def G(self, full_name):
        return self.g[full_name]

    def add(self, fn):
        self.nodes.append(fn)

    # ------------------------------------------------------------------ small kernels
    def axpy(self, dst, src, alpha=1.0):
        check(self.lib.mac_axpy(ptr(dst), ptr(src), float(alpha), src.numel(), stream_ptr()), "mac_axpy")

    def colsum_B(self, part, out_flat):
        Bp, d = part.shape
        check(self.lib.mac_colsum(ptr(part), ptr(out_flat), 1, Bp, d, 1, stream_ptr()), "mac_colsum")

    def linear_bwd(self, xs, W, wname, bname, dy, dxs):
        n = len(xs)
        Wt = self.p.derived(("T", wname), lambda: W.t().contiguous()) if any(d is not None for d in dxs) else None
        M, n_out = dy.shape
        arr_x = (ctypes.c_void_p * n)(*[x.data_ptr() for x in xs])
        arr_k = (ctypes.c_int * n)(*[x.shape[1] for x in xs])
        arr_ld = (ctypes.c_int * n)(*[x.stride(0) for x in xs])
        arr_dx = (ctypes.c_void_p * n)(*[(d.data_ptr() if d is not None else None) for d in dxs])
        arr_ldd = (ctypes.c_int * n)(*[(d.stride(0) if d is not None else 0) for d in dxs])
        arr_acc = (ctypes.c_int * n)(*[1] * n)
        check(self.lib.mac_linear_bwd(arr_x, arr_k, arr_ld, n, ptr(Wt), ptr(dy), dy.stride(0), arr_dx, arr_ldd, arr_acc,
                                      ptr(self.G(wname)), ptr(self.G(bname)) if bname else None, M, n_out,
                                      ptr(self.lws), self.lws_bytes, stream_ptr()), "mac_linear_bwd")

    def linear_bwd_tc(self, xs, W, wname, bname, dy, dxs):
        """linear_bwd with bf16 operands on tensor cores (mac_linear_bwd_tc): the composed read unit's [B*N, .] products."""
        n = len(xs)
        M, n_out = dy.shape
        arr_x = (ctypes.c_void_p * n)(*[x.data_ptr() for x in xs])
        arr_k = (ctypes.c_int * n)(*[x.shape[1] for x in xs])
        arr_ld = (ctypes.c_int * n)(*[x.stride(0) for x in xs])
        arr_dx = (ctypes.c_void_p * n)(*[d.data_ptr() for d in dxs])
        arr_ldd = (ctypes.c_int * n)(*[d.stride(0) for d in dxs])
        arr_acc = (ctypes.c_int * n)(*[1] * n)
        need = int(self.lib.mac_linear_bwd_tc_workspace_bytes(M, arr_k, n, n_out))
        if self._tcws is None or self._tcws.numel() < need:
            self._tcws = torch.empty(need, dtype=torch.uint8, device=self.dev)
        check(self.lib.mac_linear_bwd_tc(arr_x, arr_k, arr_ld, n, ptr(W), ptr(dy), dy.stride(0), arr_dx, arr_ldd, arr_acc,
                                         ptr(self.G(wname)), ptr(self.G(bname)) if bname else None, M, n_out,
                                         ptr(self._tcws), self._tcws.numel(), stream_ptr()), "mac_linear_bwd_tc")

    # ------------------------------------------------------------------ recorders (called from the forward)
    def linear(self, xs, W, b, out, code, bn_rows=False):
        """y = act(concat(xs) @ W + b)   (ops.py:298-333); bn_rows: a [B*N, .] product of the composed read unit"""
        xs = list(xs)
        wname = self.name_of(W)
        bname = self.name_of(b) if b is not None else None

        def bwd():
            g = self.grad(out)
            dpre = g
            if code != ACT["NON"]:
                dpre = self.e(*out.shape)
                check(self.lib.mac_activation_bwd(ptr(out), ptr(g), code, ptr(dpre), out.numel(), stream_ptr()), "act bwd")
            if bn_rows and self.tc:
                self.linear_bwd_tc(xs, W, wname, bname, dpre, [self.grad(x) for x in xs])
            else:
                self.linear_bwd(xs, W, wname, bname, dpre, [self.grad(x) for x in xs])
        self.add(bwd)

    def act(self, x, out, code):
        def bwd():
            tmp = self.e(*out.shape)
            check(self.lib.mac_activation_bwd(ptr(out), ptr(self.grad(out)), code, ptr(tmp), out.numel(), stream_ptr()),
                  "act bwd")
            self.axpy(self.grad(x), tmp)
        self.add(bwd)

    def bcast(self, x2d, v, mode, mul_bias, bias, out, B, N):
        """ops.mul interaction of x [B*N, d] with v [B, d] (ops.py:694-713)."""
        d = x2d.shape[1]
        bias_name = self.name_of(bias) if bias is not None else None

        def bwd():
            part = self.z(B, d) if bias_name else None
            check(self.lib.mac_bcast_op_bwd(ptr(x2d), ptr(v), ptr(out), ptr(self.grad(out)), mode, float(mul_bias),
                                            ptr(self.grad(x2d)), ptr(self.grad(v)), ptr(part), B, N, d, stream_ptr()),
                  "mac_bcast_op_bwd")
            if bias_name:
                self.colsum_B(part, self.G(bias_name))
        self.add(bwd)

    def rowdot(self, xs, lscope, out):
        """outDim == 1 linear over concatenated segments (ops.py:316-317)."""
        xs = list(xs)
        wname, bname = PREFIX + lscope + "weights/weight", PREFIX + lscope + "biases/bias"
        w = self.p[lscope + "weights/weight"]

        def bwd():
            n, R = len(xs), xs[0].shape[0]
            ktot = sum(x.shape[1] for x in xs)
            nbytes = int(self.lib.mac_rowdot_bwd_workspace_bytes(R, ktot))
            ws = torch.empty(nbytes, dtype=torch.uint8, device=self.dev)
            dxs = [self.grad(x) for x in xs]
            arr_x = (ctypes.c_void_p * n)(*[x.data_ptr() for x in xs])
            arr_k = (ctypes.c_int * n)(*[x.shape[1] for x in xs])
            arr_ld = (ctypes.c_int * n)(*[x.stride(0) for x in xs])
            arr_dx = (ctypes.c_void_p * n)(*[d.data_ptr() for d in dxs])
            arr_ldd = (ctypes.c_int * n)(*[d.stride(0) for d in dxs])
            check(self.lib.mac_rowdot_bwd(arr_x, arr_k, arr_ld, n, ptr(w), ptr(self.grad(out)), arr_dx, arr_ldd,
                                          ptr(self.G(wname)), ptr(self.G(bname)), ptr(ws), nbytes, R, stream_ptr()),
                  "mac_rowdot_bwd")
        self.add(bwd)

    def attend(self, logits, feats, att, out, B, M, dd):
        """att = softmax(logits (masked)); out = sum_m att * feats   (ops.py:143-150, 243-247); feats [B, M, dd] contiguous."""
        def bwd():
            scratch, dl, dbr = self.e(B * M + 4), self.e(B * M + 4), self.z(B)
            check(self.lib.mac_kb_attend_bwd(ptr(feats), ptr(att), ptr(self.grad(out)), ptr(scratch), ptr(dl),
                                             ptr(self.grad(feats)), ptr(dbr), B, M, dd, stream_ptr()), "attend bwd")
            self.axpy(self.grad(logits), dl[:B * M].view(logits.shape))
        self.add(bwd)

    def control_attend(self, cc, in_words, out_words, lscope, att, out, S):
        """The fused control attention (mac_control_attend_fwd with one step): logits = (cc * in_words) . w + b."""
        cell = self.cell
        B, d = cell.B, cell.d
        wname, bname = PREFIX + lscope + "weights/weight", PREFIX + lscope + "biases/bias"
        w = self.p[lscope + "weights/weight"]

        def bwd():
            dcc, part, spart = self.e(B, d), self.z(B, d), self.z(B)
            check(self.lib.mac_control_attend_bwd(ptr(cc), 0, d, ptr(in_words), S * d, d, ptr(out_words), S * d, d, ptr(w),
                                                  ptr(att), ptr(self.grad(out)), 0, d, ptr(self.grad(in_words)),
                                                  ptr(self.grad(out_words)), ptr(dcc), 0, d, 0, ptr(part), ptr(spart), 1, B,
                                                  S, d, stream_ptr()), "control bwd")
            self.axpy(self.grad(cc), dcc)
            self.colsum_B(part, self.G(wname))
            self.colsum_B(spart.view(B, 1), self.G(bname).view(1))
        self.add(bwd)

    def self_attend(self, sc, lscope, att, out, rows, gC, gM):
        """Write-unit self-attention over the first `rows` history slots (mac_cell.py:322-337)."""
        cell = self.cell
        B, d = cell.B, cell.d
        wname, bname = PREFIX + lscope + "weights/weight", PREFIX + lscope + "biases/bias"
        w = self.p[lscope + "weights/weight"]
        hc, hm = cell._hc, cell._hm

        def bwd():
            dsc, part, spart = self.e(B, d), self.z(B, d), self.z(B)
            check(self.lib.mac_control_attend_bwd(ptr(sc), 0, d, ptr(hc), d, B * d, ptr(hm), d, B * d, ptr(w), ptr(att),
                                                  ptr(self.grad(out)), 0, d, ptr(gC), ptr(gM), ptr(dsc), 0, d, 0, ptr(part),
                                                  ptr(spart), 1, B, rows, d, stream_ptr()), "self-att bwd")
            self.axpy(self.grad(sc), dsc)
            self.colsum_B(part, self.G(wname))
            self.colsum_B(spart.view(B, 1), self.G(bname).view(1))
        self.add(bwd)

    def dropout(self, x, out, keep, site, step):
        def bwd():
            g = self.grad(out)
            if out.data_ptr() == x.data_ptr():
                check(self.lib.mac_dropout_fwd(ptr(g), float(keep), self.cell.seed, site, step, ptr(g), g.numel(),
                                               stream_ptr()), "dropout bwd")
                return
            tmp = self.e(*out.shape)
            check(self.lib.mac_dropout_fwd(ptr(g), float(keep), self.cell.seed, site, step, ptr(tmp), g.numel(),
                                           stream_ptr()), "dropout bwd")
            self.axpy(self.grad(x), tmp)
        self.add(bwd)

    def copy(self, dst, src):
        """dst.copy_(src): whatever produced dst before is overwritten, so its gradient stops here."""
        def bwd():
            g = self.grad(dst)
            self.axpy(self.grad(src), g)
            g.zero_()
        self.add(bwd)

    def add_scaled(self, a, b, alpha, out):
        """out = a + alpha * b"""
        def bwd():
            g = self.grad(out)
            self.axpy(self.grad(a), g)
            self.axpy(self.grad(b), g, alpha)
        self.add(bwd)

    def cat(self, segs, out):
        """out = concat(segs, dim=1) (materialised for a flat dropout mask index): split the gradient back."""
        def bwd():
            g = self.grad(out)
            off = 0
            for s in segs:
                k = s.shape[1]
                self.axpy(self.grad(s), g[:, off:off + k].contiguous())
                off += k
        self.add(bwd)

    def batch_norm(self, x, out, gamma, beta, mean, invstd, training):
        """memoryBN (mac_cell.py:369-373); the stored statistics are not trainable: no gradient."""
        B, d = x.shape
        gname = self.name_of(gamma) if gamma is not None else None
        bname = self.name_of(beta) if beta is not None else None

        def bwd():
            check(self.lib.mac_batchnorm_bwd(ptr(x), ptr(gamma), ptr(mean), ptr(invstd), ptr(self.grad(out)), training,
                                             ptr(self.grad(x)), ptr(self.G(gname)) if gname else None,
                                             ptr(self.G(bname)) if bname else None, B, d, stream_ptr()), "mac_batchnorm_bwd")
        self.add(bwd)

    def init_state(self, slot, kind, name):
        def fin():
            if kind == "PRM":
                self.colsum_B(self.grad(slot), self.G(PREFIX + name))
            elif kind == "Q":
                self.axpy(self.grad(self.cell.vecQuestions), self.grad(slot))
        self.finalizers.append(fin)

    def fused_read(self, i, name, knowledgeBase, memory_in, control, info):
        """mac_read_fwd with the activations saved in cell._save[i] -> mac_read_bwd (csrc/backward.cu), or mac_read_bwd_tc
        (its six [B*N, .] products on tensor cores) when the sweep runs with tc=True."""
        cell = self.cell
        B, N, d = cell.B, cell.N, cell.d
        rsc = "MACCell/read" + name + "/"
        lsc = rsc + "inter2att/inter2logits/linearLayerlogits/"

        def lin_names(scope, nm):
            sc = PREFIX + scope + "linearLayer" + nm + "/"
            return sc + "weights/weight", sc + "biases/bias"

        def bwd():
            rw = cell._read_weights(name)
            nWx, nbx = lin_names(rsc + "mulmemInter/", "projX")
            nWy, nby = lin_names(rsc + "mulmemInter/", "projY")
            nWm, nbm = lin_names(rsc, "memKbProj")
            nWm2, nbm2 = lin_names(rsc + "linearLayermemKbProj/", "memKbProj_2")
            wnames = {"Wx": nWx, "Wy": nWy, "Wm": nWm, "Wm2": nWm2}
            Wt = lambda k: self.p.derived(("T", wnames[k]), lambda: self.p.t[wnames[k]].t().contiguous())
            part = {k: self.z(B, d) for k in ("wr", "bx", "bm", "bm2")}
            dbr = self.z(B)
            dmem_in = self.e(B, d)
            form = "tc" if self.tc else "fp32"
            ws_bytes = read_bwd_workspace_bytes(self.lib, form, B, N, d)
            if getattr(self, "_rws", None) is None or self._rws.numel() < ws_bytes:
                self._rws = torch.zeros(ws_bytes, dtype=torch.uint8, device=self.dev)
            read_bwd(self.lib, form, cell, i, knowledgeBase, control, rw, Wt, self.grad(info),
                     [self.grad(knowledgeBase), dmem_in, self.grad(control), self.G(nWx), part["bx"], self.G(nWy),
                      self.G(nby), self.G(nWm), part["bm"], self.G(nWm2), part["bm2"], part["wr"], dbr], self._rws, ws_bytes)
            self.axpy(self.grad(memory_in), dmem_in)
            self.colsum_B(part["wr"], self.G(PREFIX + lsc + "weights/weight"))
            self.colsum_B(part["bx"], self.G(nbx))
            self.colsum_B(part["bm"], self.G(nbm))
            self.colsum_B(part["bm2"], self.G(nbm2))
            self.colsum_B(dbr.view(B, 1), self.G(PREFIX + lsc + "biases/bias").view(1))
        self.add(bwd)

    def fused_write(self, i, name, memory, info, selfSmry, control, out):
        """mac_write_fwd (newMemory over [memory, info, selfSmry], optional gate): mac_cell.py:339-367."""
        cell, c = self.cell, self.cell.cfg
        B, d = cell.B, cell.d
        wsc = "MACCell/write" + name + "/"

        def bwd():
            g_m = self.grad(out)
            dmp = g_m
            if c.writeGate:
                tmp_dm, tmp_dpre = self.e(B, d), self.e(B, d)
                check(self.lib.mac_gate_bwd(ptr(g_m), ptr(cell._gate[i]), ptr(cell._mnew[i]), ptr(memory), ptr(tmp_dm),
                                            ptr(self.grad(memory)), ptr(tmp_dpre), B * d, stream_ptr()), "mac_gate_bwd")
                Wg, bg = self.p.lin(wsc, "gate")
                self.linear_bwd([control], Wg, self.name_of(Wg), self.name_of(bg), tmp_dpre, [self.grad(control)])
                dmp = tmp_dm
            Ww, bw = self.p.lin(wsc, "newMemory")
            xs = [memory, info] + ([selfSmry] if selfSmry is not None else [])
            self.linear_bwd(xs, Ww, self.name_of(Ww), self.name_of(bw), dmp, [self.grad(x) for x in xs])
        self.add(bwd)

    # ------------------------------------------------------------------ the sweep
    def run(self, d_control, d_memory, bucket=None, zero_bucket=True, d_vecq=None, tc=False):
        from .mac_cell import views_of
        cell, c = self.cell, self.cell.cfg
        self.tc = bool(tc)
        self.bucket = bucket if bucket is not None else torch.zeros_like(self.p.flat)
        if bucket is not None and zero_bucket:
            self.bucket.zero_()
        self.g = views_of(self.bucket, self.p.specs, self.p.offsets)
        self.lws = torch.zeros(self.lws_bytes, dtype=torch.uint8, device=self.dev)
        L = cell.L
        if d_control is not None:
            self.axpy(self.grad(cell._hc[L]), d_control.contiguous())
        if d_memory is not None:
            self.axpy(self.grad(cell._hm[L]), d_memory.contiguous())
        if d_vecq is not None:
            self.axpy(self.grad(cell.vecQuestions), d_vecq.contiguous())
        for fn in reversed(self.nodes):
            fn()
        for fn in self.finalizers:
            fn()
        out = collections.OrderedDict(self.g)
        out["knowledgeBase"] = self.grad(cell.knowledgeBase)
        words = cell.questionCntxWords if c.controlContextual else cell.questionWords
        out["questionCntxWords" if c.controlContextual else "questionWords"] = self.grad(words)
        out["vecQuestions"] = self.grad(cell.vecQuestions)
        self.nodes, self.finalizers = [], []          # one sweep per forward: the saved tensors are released here
        return out
