"""CPU checks that the bounds of tests/test_gpu_tc32_training.py separate split-bf16 ("tc32") arithmetic from bf16.

The product chain of mac_read_bwd_tc32 is restated in torch with split-bf16 products (x = hi + lo with hi = bf16(x),
lo = bf16(x - hi); A W ~ A_hi W_hi + A_lo W_hi + A_hi W_lo in fp32) and measured against read_bwd_reference with the GPU
tests' own element-wise bounds `|got - ref| <= TOL_BWD * absref` at B*N = 245 (contraction padded to 256).  The restatement
passes every bound, and each of these planted faults exceeds some bound by more than 100 times:
  * plain bf16 products (the lo terms dropped);
  * garbage instead of zeros in the padding rows of the weight gradients' contraction;
  * the knowledge-base dropout mask drawn one column quad off (a shifted Philox index)."""
import numpy as np
import torch

from tests.test_gpu_backward_kernels import ratio, read_bwd_reference, read_masks
from tests.test_gpu_tc32_training import TOL_BWD
from tests.test_gpu_wgmma import keep_mask

MARGIN = 100


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _split(x):
    hi = x.float().to(torch.bfloat16).float()
    return hi, (x.float() - hi).to(torch.bfloat16).float()


def tc3(a, b):
    """a @ b as the split-bf16 product: three of the four partial products, fp32"""
    ah, al = _split(a)
    bh, bl = _split(b)
    return ah @ bh + al @ bh + ah @ bl


def bf16(a, b):
    """a @ b on plain bf16 operands (the lo terms dropped), fp32"""
    return _split(a)[0] @ _split(b)[0]


def _read_case(B, N, d, keep, seed, step):
    """fp64 read-unit inputs, the forward (P, H, I1, y, att) and read_bwd_reference's gradients"""
    g = _gen(seed)
    r = lambda *s, scale=1.0: torch.randn(*s, generator=g, dtype=torch.float64) * scale
    W = {"Wx": r(d, d, scale=d ** -0.5), "bx": r(d, scale=0.1), "Wy": r(d, d, scale=d ** -0.5), "by": r(d, scale=0.1),
         "Wm": r(2 * d, d, scale=(2 * d) ** -0.5), "bm": r(d, scale=0.1), "Wm2": r(d, d, scale=d ** -0.5),
         "bm2": r(d, scale=0.1), "wr": r(d, scale=4 * d ** -0.5)}
    kb, mem, c, dinfo = torch.nn.functional.elu(r(B, N, d)), r(B, d), r(B, d), r(B, d)
    masks = read_masks(keep, seed, step, B, N, d, "cpu")
    mkb, mmem, mint = masks
    M = B * N
    y = (mem * mmem) @ W["Wy"] + W["by"]
    P = (kb.reshape(M, d) * mkb) @ W["Wx"] + W["bx"]
    yb = y.repeat_interleave(N, 0)
    H = torch.nn.functional.elu(torch.cat([P * yb, P], 1) @ W["Wm"] + W["bm"])
    I1 = H @ W["Wm2"] + W["bm2"]
    I2 = torch.nn.functional.elu(I1 * c.repeat_interleave(N, 0))
    att = torch.softmax(((I2 * mint) @ W["wr"] + 0.25).view(B, N), 1)
    f = lambda t: t.float().double()                  # the kernels see fp32 operands
    P, H, I1, y, att, kb, W = f(P), f(H), f(I1), f(y), f(att), f(kb), {k: f(v) for k, v in W.items()}
    ref = read_bwd_reference(kb, mem, c, W, att, P, H, I1, y, dinfo, keep, seed, step)
    return kb, c, W, att, P, H, I1, y, dinfo, masks, ref


def read_bwd_restated(case, mm, pad_fill=None, mkb=None):
    """mac_read_bwd_tc32's product chain in fp32 with `mm` for each of its six products: the weight gradients contract over
    B*N rounded up to 64 (padding rows zero, or `pad_fill(rows, cols)`); the logits backward is the fp64 reference's"""
    kb, c, W, att, P, H, I1, y, dinfo, masks, ref = case
    B, N, d = kb.shape
    M, Mp = B * N, (B * N + 63) // 64 * 64
    mkb = masks[0] if mkb is None else mkb
    mint = masks[2]
    F = lambda t: t.float()
    bsum = lambda t: t.view(B, N, -1).sum(1)
    pad = lambda x: torch.cat([x, pad_fill(Mp - M, x.shape[1]) if pad_fill else torch.zeros(Mp - M, x.shape[1])], 0)
    wgrad = lambda X, G: mm(pad(X).t(), pad(G))
    cb, yb = c.repeat_interleave(N, 0), y.repeat_interleave(N, 0)
    # dI1 of the fp32 logits backward (shared with mac_read_bwd): from the fp64 softmax backward
    a, di = att, dinfo
    dka = torch.einsum("bnd,bd->bn", kb, di)
    dkl = a * (dka - (a * dka).sum(1, keepdim=True))
    t = I1 * cb
    dI1 = F(dkl.reshape(M, 1) * W["wr"] * mint * torch.where(t > 0, torch.ones_like(t), torch.exp(t)) * cb)
    out = {"dWm2": wgrad(F(H), dI1)}
    eH = F(torch.where(H > 0, torch.ones_like(H), H + 1))
    dZ = mm(dI1, F(W["Wm2"]).t()) * eH
    out["dbm_part"] = bsum(dZ)
    I0 = F(torch.cat([P * yb, P], 1))
    out["dWm"] = wgrad(I0, dZ)
    dI0 = mm(dZ, F(W["Wm"]).t())
    dP = dI0[:, :d] * F(yb) + dI0[:, d:]
    out["dbx_part"] = bsum(dP)
    kbd = F(kb.reshape(M, d) * mkb)
    out["dWx"] = wgrad(kbd, dP)
    out["dkb"] = (mm(dP, F(W["Wx"]).t()) * F(mkb)).view(B, N, d) + F(a[:, :, None] * di[:, None, :])
    return out


def _worst(case, out):
    """the largest ratio / TOL_BWD over the restated outputs, and every ratio"""
    ref = case[-1]
    r = {k: ratio(v, *ref[k]) for k, v in out.items()}
    return max(v / TOL_BWD[k] for k, v in r.items()), r


CASE = (5, 49, 128, 0.85, 7, 3)      # B*N = 245: the weight gradients' contraction is padded to 256


def _check_chain(fault_out, what):
    case = _read_case(*CASE)
    ok, r_ok = _worst(case, read_bwd_restated(case, tc3))
    bad, r_bad = _worst(case, fault_out(case))
    print("%s: tc32 uses %.2f of the bounds %s; the fault %.0f times %s" % (
        what, ok, {k: "%.1e" % v for k, v in r_ok.items()}, bad, {k: "%.1e" % v for k, v in r_bad.items()}))
    assert ok <= 1.0, r_ok
    assert bad > MARGIN, r_bad


def test_backward_bounds_reject_plain_bf16_products():
    _check_chain(lambda case: read_bwd_restated(case, bf16), "lo terms dropped")


def test_backward_bounds_reject_garbage_padding_columns():
    """the padding rows of the contraction hold what an unwritten workspace might: values of the size of the data"""
    g = _gen(8)
    _check_chain(lambda case: read_bwd_restated(case, tc3, pad_fill=lambda r, k: torch.randn(r, k, generator=g)),
                 "garbage padding")


def test_backward_bounds_reject_a_shifted_philox_index():
    """the knowledge-base mask of element (m, c) is draw (m*d + c) / 4 of site READ_KB; the fault takes the next quad's"""
    B, N, d, keep, seed, step = CASE
    M = B * N
    sc = float(np.float32(1.0) / np.float32(keep))
    shifted = keep_mask(seed, 1, step, (M * d + 4,), keep, device="cpu")[4:].view(M, d).double() * sc
    _check_chain(lambda case: read_bwd_restated(case, tc3, mkb=shifted), "Philox index + 4")
