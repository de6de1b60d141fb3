"""The question encoder's kernels (csrc/encoder.cu, csrc/encoder_tc.cuh) and the image stem's patch kernels
(mac_im2col3x3, mac_col2im3x3 in csrc/units.cu) against references of their OWN operation, called through the C ABI.

The LSTM references are per step and are computed from the kernel's own saved state, so rounding does not compound over the
S steps and an error cannot hide where values are small (the backward direction's first step, rows of length 1, late steps
of short questions):

    forward    pre(t) = gx(t) + save_hprev(t) @ Wh (+ forget_bias on f), checked against save_gates through |act'| <= 1;
               save_c(t) = c_prev * f + i * j with the kernel's own gates and c_prev; out_seq(t) = tanh(save_c(t)) * o
    backward   dh(t) = d_out(t) + dG(t') @ Wh^T from the kernel's own dG of the step after it (d_vecq at the last live step),
               the cell-state gradient carried as an fp64 chain

The tensor-core forms use the same references on their bf16 operands (bf16(save_hprev), bf16(dG), bf16(Wh)).  Each
reference has an absolute-value twin and the bound is element-wise, |got - ref| <= tol * absref + tiny, with `tiny` the fp32
evaluation error of tanhf / expf.  The exact relations are checked bit for bit: save_hprev(t) is the previous step's
output, vecq the last live step's output, and rows t >= len are zero although every buffer starts NaN-filled.  The
embedding and the patch kernels are pure data movement (the embedding's backward aside) and must equal their torch
restatement exactly.

Every case also checks the output contracts: "=" outputs start NaN-filled (an unwritten element fails) with a NaN guard
behind them that must survive; "+=" outputs start random and only the increment may change them; two runs from the same
state are bit-identical; lengths outside [0, S] act as the clamped length, bit for bit.  tests/test_encoder_bounds.py
shows on the CPU, with this file's reference and bound code, that planted faults fail these bounds.

Each `tol` is about three times the worst value measured on an H100 80GB HBM3 (SXM, 700 W power limit), written beside
it.  Every reference is computed on the device, so the whole file takes about ten seconds of GPU time.  With fixed seeds
and fixed-order reductions every run gives the same bits, so the ratios do not depend on the clock."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from mac_network_b200 import _lib as L_
from tests.test_gpu_backward_kernels import Report, gen, prefill, randn, run_twice, same_bits
from tests.test_gpu_wgmma import bf16_round, keep_mask

pytestmark = pytest.mark.gpu

MAC_OK, ERR_INVALID, ERR_UNSUPPORTED = 0, -1, -3
SITE = 48                 # the encoder's input-dropout site (any site will do for the kernels)
GUARD = 64                # NaN elements behind every "=" output

# ---- bounds (fraction of absref); measured worst value on the H100 beside each
#                                                                                   measured
TOL_FWD = {"gates": 1e-6, "c": 4e-7, "out": 8e-7}         # mac_lstm_fwd               3.0e-7, 1.2e-7, 2.4e-7
TOL_FWD_TC = {"gates": 4e-7, "c": 4e-7, "out": 8e-7}      # mac_lstm_fwd_tc            1.1e-7, 1.1e-7, 2.3e-7
TOL_BWD = 1.5e-6                                          # mac_lstm_bwd dG            5.1e-7
TOL_BWD_TC = {"dG": 1e-6, "dkernel": 2.5e-6,              # mac_lstm_bwd_tc            3.3e-7, 8.4e-7
              "dbias": 5e-7, "dx": 2e-6}                  #                            1.5e-7, 7.1e-7
TOL_EMBED_BWD = 5e-7                                      # mac_embed_bwd              1.4e-7
# fp32 evaluation of the non-linearities, outside the tol: sigmoid_f / tanhf are within a few ulp relative (the
# activated gates), and 1 - tanhf(c)^2 within 4e-7 absolute (2 ulp of tanhf, two roundings)
EVAL_ACT = 5e-7
EVAL_DTANH = 4e-7


# ------------------------------------------------------------------------------------------------ references
def step_index(lengths, S, reverse):
    """(t, live, L): t[b, s] the time index of step s (len-1-s backward, s forward; s itself past the end, so each row of
    t is a permutation of 0..S-1), live = s < L, L the clamped lengths [B, 1].  `live` is also the time-order mask t < L."""
    L = lengths.long().clamp(0, S)[:, None]
    s = torch.arange(S, device=lengths.device)[None, :]
    live = s < L
    t = torch.where(live, (L - 1 - s) if reverse else s.expand_as(live), s.expand_as(live))
    return t, live, L


def by_step(x, t):
    """[B, S, F] in time order -> step order"""
    return torch.gather(x, 1, t[:, :, None].expand(-1, -1, x.shape[2]))


def by_time(x, t):
    """[B, S, F] in step order -> time order"""
    return torch.empty_like(x).scatter_(1, t[:, :, None].expand(-1, -1, x.shape[2]), x)


def lstm_fwd_reference(gx, Wh, lengths, fb, sg, sc, shp, reverse, bf16=False):
    """One direction, every tensor [B, S, .] by time index as the kernel leaves it.  Returns name -> (ref, absref, tiny) in
    time order (valid where `live`) for the activated gates, the new cell state and the output, and `live`."""
    B, S, G = gx.shape
    h = G // 4
    t, live, _ = step_index(lengths, S, reverse)
    st = lambda x: by_step(x.double(), t)
    hp, W = st(shp), Wh.double()
    if bf16:
        hp, W = bf16_round(hp), bf16_round(W)
    fbv = torch.zeros(G, dtype=torch.float64, device=gx.device)
    fbv[2 * h:3 * h] = fb
    gxs = st(gx)
    pre = gxs + hp @ W + fbv
    apre = gxs.abs() + hp.abs() @ W.abs() + fbv.abs()
    act = torch.cat([torch.sigmoid(pre[..., :h]), torch.tanh(pre[..., h:2 * h]), torch.sigmoid(pre[..., 2 * h:])], -1)
    gi, gj, gf, go = st(sg).split(h, -1)
    c = st(sc)
    cp = torch.cat([torch.zeros_like(c[:, :1]), c[:, :-1]], 1)               # the previous step's cell state, 0 first
    cref, acref = cp * gf + gi * gj, (cp * gf).abs() + (gi * gj).abs()
    out = torch.tanh(c) * go
    bt = lambda x: by_time(x, t)
    return {"gates": (bt(act), bt(apre), bt(EVAL_ACT * act.abs())), "c": (bt(cref), bt(acref), 0.0),
            "out": (bt(out), bt(out.abs()), 0.0)}, live


def lstm_fwd_exact(out, vecq, shp, lengths, reverse):
    """The forward's exact relations for one direction: [(what, holds)].  out / shp [B, S, h] by time index, vecq [B, h]."""
    B, S, h = out.shape
    t, live, L = step_index(lengths, S, reverse)
    o, hp = by_step(out, t), by_step(shp, t)
    prev = torch.cat([torch.zeros_like(o[:, :1]), o[:, :-1]], 1)
    last = torch.gather(o, 1, (L - 1).clamp_min(0)[:, :, None].expand(-1, -1, h))[:, 0]
    want_q = torch.where(L > 0, last, torch.zeros_like(last))
    return [("hprev is the previous output", same_bits(hp[live], prev[live])),
            ("out rows t >= len zero", bool((out[~live] == 0).all())),
            ("hprev rows t >= len zero", bool((shp[~live] == 0).all())),
            ("vecq is the last live output", vecq is None or same_bits(vecq, want_q))]


def lstm_bwd_reference(dG, Wh, lengths, sg, sc, d_out, d_vecq, reverse, bf16=False):
    """One direction: the gate gradients of every live step from the kernel's own dG [B, S, 4h] of the step after it,
    in time order: (ref, absref, tiny, live).  The cell-state gradient is an fp64 chain with its absolute twin and the
    chain of the tanh-derivative evaluation error."""
    B, S, G = dG.shape
    h = G // 4
    t, live, L = step_index(lengths, S, reverse)
    st = lambda x: by_step(x.double(), t)
    g, W = st(dG), Wh.double()
    if bf16:
        g, W = bf16_round(g), bf16_round(W)
    nxt = torch.cat([g[:, 1:], torch.zeros_like(g[:, :1])], 1)              # dG of step s+1 (0 after the last step)
    rec, arec = nxt @ W.t(), nxt.abs() @ W.abs().t()
    do = st(d_out)
    dv = torch.zeros_like(do[:, 0]) if d_vecq is None else d_vecq.double()
    last = (torch.arange(S, device=dG.device)[None, :] + 1 >= L)[:, :, None]  # the last live step: its h is the final state
    dh = torch.where(last, do + dv[:, None], do + rec)
    adh = torch.where(last, do.abs() + dv.abs()[:, None], do.abs() + arec)
    gi, gj, gf, go = st(sg).split(h, -1)
    c = st(sc)
    cp = torch.cat([torch.zeros_like(c[:, :1]), c[:, :-1]], 1)
    tc = torch.tanh(c)
    ref, aref, tiny = (torch.zeros(B, S, G, dtype=torch.float64, device=dG.device) for _ in range(3))
    dcc, adcc, ecc = (torch.zeros(B, h, dtype=torch.float64, device=dG.device) for _ in range(3))
    for s in range(S - 1, -1, -1):
        dt = go[:, s] * (1 - tc[:, s] ** 2)
        dc = dcc + dh[:, s] * dt
        adc = adcc + adh[:, s] * dt.abs()
        edc = ecc + dh[:, s].abs() * go[:, s] * EVAL_DTANH
        fi, fj = gj[:, s] * gi[:, s] * (1 - gi[:, s]), gi[:, s] * (1 - gj[:, s] ** 2)
        ff, fo = cp[:, s] * gf[:, s] * (1 - gf[:, s]), tc[:, s] * go[:, s] * (1 - go[:, s])
        ref[:, s] = torch.cat([dc * fi, dc * fj, dc * ff, dh[:, s] * fo], 1)
        aref[:, s] = torch.cat([adc * fi.abs(), adc * fj.abs(), adc * ff.abs(), adh[:, s] * fo.abs()], 1)
        tiny[:, s] = torch.cat([edc * fi.abs(), edc * fj.abs(), edc * ff.abs(), torch.zeros_like(fo)], 1)
        lv = live[:, s, None]
        dcc, adcc, ecc = (torch.where(lv, x * gf[:, s], y) for x, y in ((dc, dcc), (adc, adcc), (edc, ecc)))
    return by_time(ref, t), by_time(aref, t), by_time(tiny, t), live


def f32_inv(keep):
    """the kernels' scale 1.f / keep, as a float"""
    return float(np.float32(1.0) / np.float32(keep))


def embed_reference(emb, idx, keep, seed, step):
    """(out_raw, out) of mac_embed_fwd: the embedding row (zero for ids outside 1..V), then the keep-mask of the element's
    quad index and the fp32 scale 1/keep"""
    V, E = emb.shape
    idx = idx.reshape(-1).long()
    ok = (idx >= 1) & (idx <= V)
    raw = torch.where(ok[:, None], emb[(idx - 1).clamp(0, V - 1)], torch.zeros((), device=emb.device))
    if keep >= 1.0:
        return raw, raw
    m = keep_mask(seed, SITE, step, raw.shape, keep, device=emb.device)
    return raw, torch.where(m, raw * f32_inv(keep), torch.zeros((), device=emb.device))


def embed_bwd_reference(d_out, idx, V, keep, seed, step):
    """(inc, absinc, referenced rows) of mac_embed_bwd in fp64"""
    E = d_out.shape[-1]
    d = d_out.reshape(-1, E).double()
    if keep < 1.0:
        d = d * keep_mask(seed, SITE, step, d.shape, keep, device=d.device).double() * f32_inv(keep)
    idx = idx.reshape(-1).long()
    ok = (idx >= 1) & (idx <= V)
    inc = torch.zeros(V, E, dtype=torch.float64, device=d.device).index_add_(0, idx[ok] - 1, d[ok])
    ainc = torch.zeros(V, E, dtype=torch.float64, device=d.device).index_add_(0, idx[ok] - 1, d[ok].abs())
    used = torch.zeros(V, dtype=torch.bool, device=d.device)
    used[idx[ok] - 1] = True
    return inc, ainc, used


def patch_mask(x, keep, seed, step):
    """dropout(x) as the patch kernels apply it: the source element's keep-mask, times the fp32 1/keep"""
    if keep >= 1.0:
        return None
    return keep_mask(seed, SITE, step, x.shape, keep, device=x.device)


def im2col_reference(x, keep, seed, step):
    """cols [B*H*W, 9C]: pad, shift each tap (kh*3 + kw), dropout by the source element's mask"""
    B, H, W, C = x.shape
    m = patch_mask(x, keep, seed, step)
    xd = x if m is None else torch.where(m, x * f32_inv(keep), torch.zeros((), device=x.device))
    xp = F.pad(xd, (0, 0, 1, 1, 1, 1))
    cols = torch.stack([xp[:, kh:kh + H, kw:kw + W, :] for kh in range(3) for kw in range(3)], 3)
    return cols.reshape(B * H * W, 9 * C)


def col2im_reference(dcols, shape, keep, seed, step):
    """dx [B, H, W, C]: the fp32 sum over taps 0..8 in the kernel's order of the entries that copied each pixel, then the
    mask and the scale"""
    B, H, W, C = shape
    d = dcols.view(B, H, W, 9, C)
    acc = torch.zeros(B, H, W, C, device=dcols.device)
    for tap in range(9):
        dh, dw = tap // 3 - 1, tap % 3 - 1
        p = F.pad(d[:, :, :, tap], (0, 0, 1, 1, 1, 1))
        acc = acc + p[:, 1 - dh:1 - dh + H, 1 - dw:1 - dw + W, :]
    m = keep_mask(seed, SITE, step, shape, keep, device=dcols.device) if keep < 1.0 else None
    return acc if m is None else torch.where(m, acc * f32_inv(keep), torch.zeros((), device=dcols.device))


# ------------------------------------------------------------------------------------------------ plumbing
def lib():
    return L_.load()


P = L_.ptr


def stream():
    return L_.stream_ptr()


def nan_guarded(n, dtype=torch.float32):
    """(buffer with a NaN guard behind it, its first n elements)"""
    buf = torch.full((n + GUARD,), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[:n]


def guard_intact(buf, n):
    return bool(buf[n:].isnan().all())


def lengths_for(B, S, seed, clamp_cases=True):
    """lengths in 1..S with S and 1 present and, with the clamp, 0, S + 3 and -2"""
    rng = np.random.RandomState(seed)
    lens = rng.randint(1, S + 1, size=B)
    special = [S, 1, 0, S + 3, -2] if clamp_cases else [S, 1]
    if B == 1:
        special = [S + 3] if clamp_cases else [S]
    lens[:len(special[:B])] = special[:B]
    return torch.from_numpy(lens.astype(np.int32)).cuda()


def clamped(lens, S):
    return lens.clamp(0, S).to(torch.int32).contiguous()


def opt(ts, d):
    return P(ts[d]) if d < len(ts) and ts[d] is not None else None


# ================================================================================================ 1. embedding
@pytest.mark.parametrize("form", ["fp32", "fp32_noraw", "tc"])
@pytest.mark.parametrize("keep", [1.0, 0.85])
@pytest.mark.parametrize("E", [4, 300, 516])
def test_embed_fwd_bit_exact(E, keep, form):
    """out_raw is the embedding row or zero (ids 0, V+1, -1, 2^20); out is out_raw * float32(1/keep) where the quad-index
    mask keeps the element; the tc form's x16 is bf16(out) with zero columns E..Ep"""
    lb = lib()
    g = gen(E + int(keep * 100))
    B, S, V, seed, step = 6, 9, 37, 17, 3
    emb = randn(g, V, E)
    idx = torch.randint(0, V + 1, (B, S), device="cuda", generator=g, dtype=torch.int32)
    idx.view(-1)[:5] = torch.tensor([0, V + 1, -1, 1 << 20, V], dtype=torch.int32)
    idx.view(-1)[-1] = 1
    M = B * S
    raw_ref, out_ref = embed_reference(emb, idx, keep, seed, step)
    rbuf, raw = nan_guarded(M * E)
    if form == "tc":
        Ep = (E + 127) // 128 * 128
        xbuf = torch.full((M * Ep + GUARD,), float("nan"), dtype=torch.bfloat16, device="cuda")
        st = lb.mac_embed_fwd_tc(P(emb), P(idx), keep, seed, SITE, step, P(raw), P(xbuf), B, S, V, E, stream())
        torch.cuda.synchronize()
        assert st == MAC_OK
        x16 = xbuf[:M * Ep].view(M, Ep)
        want = torch.zeros(M, Ep, dtype=torch.bfloat16, device="cuda")
        want[:, :E] = out_ref.to(torch.bfloat16)
        assert torch.equal(raw.view(M, E), raw_ref)
        assert torch.equal(x16.view(torch.int16), want.view(torch.int16))
        assert bool(xbuf[M * Ep:].float().isnan().all()) and guard_intact(rbuf, M * E)
        return
    obuf, out = nan_guarded(M * E)
    st = lb.mac_embed_fwd(P(emb), P(idx), keep, seed, SITE, step, P(raw) if form == "fp32" else None, P(out), B, S, V, E,
                          stream())
    torch.cuda.synchronize()
    assert st == MAC_OK
    assert torch.equal(out.view(M, E), out_ref)
    if form == "fp32":
        assert torch.equal(raw.view(M, E), raw_ref) and guard_intact(rbuf, M * E)
    else:
        assert bool(rbuf.isnan().all())
    assert guard_intact(obuf, M * E)


EMBED_BWD_CASES = {"one_id_everywhere": (65, 40, 5, 300), "V1": (6, 9, 1, 300), "E516": (6, 9, 37, 516),
                   "ids_outside": (7, 11, 23, 20)}


@pytest.mark.parametrize("keep", [1.0, 0.85])
@pytest.mark.parametrize("case", list(EMBED_BWD_CASES))
def test_embed_bwd_matches_fp64(case, keep):
    """d_emb += the masked, scaled gradient of every position holding the row's id, in position order; rows no position
    references keep their bits"""
    lb = lib()
    B, S, V, E = EMBED_BWD_CASES[case]
    g = gen(len(case) * 7 + int(keep * 100))
    seed, step = 29, 5
    if case == "one_id_everywhere":
        idx = torch.full((B, S), 3, dtype=torch.int32, device="cuda")
    else:
        idx = torch.randint(0, V + 1, (B, S), device="cuda", generator=g, dtype=torch.int32)
    if case == "ids_outside":
        bad = torch.tensor([0, V + 1, -1, 1 << 20, -(1 << 30)], dtype=torch.int32, device="cuda")
        idx.view(-1)[::2] = bad.repeat(idx.numel())[: (idx.numel() + 1) // 2]
        idx.view(-1)[1] = V
    d_out = randn(g, B, S, E)
    inc, ainc, used = embed_bwd_reference(d_out, idx, V, keep, seed, step)
    pre = prefill(g, ainc)
    demb = pre.clone()
    got, same = run_twice(lambda: lb.mac_embed_bwd(P(d_out), P(idx), keep, seed, SITE, step, P(demb), B, S, V, E, stream()),
                          {"demb": demb})
    rep = Report("embed_bwd %s keep=%g" % (case, keep))
    rep.check(same, "bit-identical rerun")
    rep.add_inc("d_emb", got["demb"][used], pre[used], inc[used], ainc[used], TOL_EMBED_BWD)
    rep.check(same_bits(got["demb"][~used], pre[~used]), "unreferenced rows untouched")
    rep.done()


# ================================================================================================ 2. LSTM, fp32
def run_lstm_fwd(lb, gx, Wh, lens, fb, B, S, h, nd, with_vecq=True, with_save=True):
    """mac_lstm_fwd into NaN-filled, guarded buffers: (status, {name: guarded buffer}, sizes)"""
    M, G = B * S, 4 * h
    n = {"out": M * nd * h, "vecq": B * nd * h, "sg": nd * M * G, "sc": nd * M * h, "shp": nd * M * h}
    bufs = {k: nan_guarded(v)[0] for k, v in n.items()
            if (k != "vecq" or with_vecq) and (k in ("out", "vecq") or with_save)}
    wsb = int(lb.mac_lstm_workspace_bytes(B, h, nd))
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    b = lambda k: P(bufs[k]) if k in bufs else None
    call = lambda: lb.mac_lstm_fwd(P(gx[0]), opt(gx, 1), P(Wh[0]), opt(Wh, 1), P(lens), fb, b("out"), b("vecq"), b("sg"),
                                   b("sc"), b("shp"), P(ws), wsb, B, S, h, nd, stream())
    return call, bufs, n


def fwd_views(bufs, n, B, S, h, nd, d):
    G = 4 * h
    v = lambda k, *shape: bufs[k][:n[k]].view(*shape) if k in bufs else None
    out = v("out", B, S, nd * h)[:, :, d * h:(d + 1) * h]
    vecq = v("vecq", B, nd * h)
    vecq = None if vecq is None else vecq[:, d * h:(d + 1) * h]
    sg, sc, shp = v("sg", nd, B, S, G), v("sc", nd, B, S, h), v("shp", nd, B, S, h)
    return out, vecq, (None if sg is None else sg[d]), (None if sc is None else sc[d]), (None if shp is None else shp[d])


def check_fwd(rep, gx, Wh, lens, fb, bufs, n, B, S, h, nd, tol, bf16=False):
    G = 4 * h
    for k, buf in bufs.items():
        rep.check(guard_intact(buf, n[k]), "%s guard" % k)
    for d in range(nd):
        out, vecq, sg, sc, shp = fwd_views(bufs, n, B, S, h, nd, d)
        refs, live = lstm_fwd_reference(gx[d].view(B, S, G), Wh[d], lens, fb, sg, sc, shp, d == 1, bf16=bf16)
        for name, got in (("gates", sg), ("c", sc), ("out", out)):
            ref, absref, tiny = refs[name]
            rep.add("%s%d" % (name, d), got[live], ref[live], absref[live], tol[name],
                    tiny[live] if torch.is_tensor(tiny) else tiny)
        for what, ok in lstm_fwd_exact(out, vecq, shp, lens, d == 1):
            rep.check(ok, "%s (dir %d)" % (what, d))
        if bf16:                                     # the tensor-core form writes every row of the saved tensors
            rep.check(bool((sg[~live] == 0).all()) and bool((sc[~live] == 0).all()), "saved rows t >= len zero (dir %d)" % d)


FWD_CASES = [  # (h, B, ndir, S): h = 256 is the persistent cluster kernel, every other h the per-step kernel
    (256, 1, 2, 40), (256, 8, 1, 2), (256, 9, 2, 40), (256, 13, 1, 40), (256, 65, 2, 1), (256, 65, 1, 40),
    (8, 1, 1, 40), (8, 130, 2, 2), (72, 64, 2, 40), (72, 65, 1, 1), (72, 130, 2, 40), (600, 1, 2, 2), (600, 65, 2, 40),
    (600, 130, 1, 40), (8, 64, 2, 1)]


def lstm_inputs(g, B, S, h, nd):
    G = 4 * h
    gx = [randn(g, B * S, G, scale=0.7) for _ in range(nd)]
    Wh = [randn(g, h, G, scale=h ** -0.5) for _ in range(nd)]
    return gx, Wh


@pytest.mark.parametrize("h,B,nd,S", FWD_CASES)
def test_lstm_fwd_matches_fp64_per_step(h, B, nd, S):
    lb = lib()
    g = gen(h * 1000 + B * 10 + S + nd)
    gx, Wh = lstm_inputs(g, B, S, h, nd)
    lens, fb = lengths_for(B, S, h + B + S), 1.0
    call, bufs, n = run_lstm_fwd(lb, gx, Wh, lens, fb, B, S, h, nd)
    status = []
    got, same = run_twice(lambda: status.append(call()), bufs)
    assert status == [MAC_OK, MAC_OK]
    rep = Report("lstm_fwd h=%d B=%d ndir=%d S=%d" % (h, B, nd, S))
    rep.check(same, "bit-identical rerun")
    check_fwd(rep, gx, Wh, lens, fb, got, n, B, S, h, nd, TOL_FWD)
    # lengths S + 3, 0, -2 act as S, 0, 0
    call_c, bufs_c, _ = run_lstm_fwd(lb, gx, Wh, clamped(lens, S), fb, B, S, h, nd)
    assert call_c() == MAC_OK
    # vecq NULL; the saved tensors NULL (out_seq unchanged)
    call_q, bufs_q, _ = run_lstm_fwd(lb, gx, Wh, lens, fb, B, S, h, nd, with_vecq=False)
    call_s, bufs_s, _ = run_lstm_fwd(lb, gx, Wh, lens, fb, B, S, h, nd, with_save=False)
    assert call_q() == MAC_OK and call_s() == MAC_OK
    torch.cuda.synchronize()
    rep.check(all(same_bits(got[k], bufs_c[k]) for k in got), "out-of-range lengths act as the clamped ones")
    rep.check(all(same_bits(got[k], bufs_q[k]) for k in bufs_q), "vecq NULL changes nothing else")
    rep.check(all(same_bits(got[k], bufs_s[k]) for k in bufs_s), "saved tensors NULL: same out_seq and vecq")
    rep.done()


@pytest.mark.parametrize("h,status", [(608, ERR_UNSUPPORTED), (12, ERR_INVALID), (4, ERR_INVALID)])
def test_lstm_fwd_refuses_before_any_launch(h, status):
    """h = 608 needs more shared memory than the per-step kernel has (h = 600 is the largest); h % 8 != 0 is invalid"""
    lb = lib()
    B, S, nd = 3, 4, 2
    gx, Wh = lstm_inputs(gen(h), B, S, h, nd)
    call, bufs, _ = run_lstm_fwd(lb, gx, Wh, lengths_for(B, S, 1), 1.0, B, S, h, nd)
    torch.cuda.synchronize()
    before = lb.mac_b200_launch_count()
    assert call() == status
    torch.cuda.synchronize()
    assert lb.mac_b200_launch_count() == before
    assert all(bool(b.isnan().all()) for b in bufs.values())


BWD_CASES = [  # (h, B, ndir, S, d_vecq given): G = 4h = 32, 256 (one full 256-column chunk), 288 (a full and a partial
    # chunk), 768, 1024
    (8, 65, 2, 7, True), (64, 65, 2, 7, True), (64, 1, 1, 7, True), (72, 65, 2, 7, True), (72, 1, 2, 1, True),
    (72, 65, 1, 7, False), (192, 65, 1, 7, True), (256, 65, 2, 7, True), (256, 1, 1, 1, True), (256, 65, 2, 7, False),
    (8, 1, 2, 1, False)]


@pytest.mark.parametrize("h,B,nd,S,with_dv", BWD_CASES)
def test_lstm_bwd_matches_fp64_per_step(h, B, nd, S, with_dv):
    lb = lib()
    g = gen(h * 997 + B * 13 + S * 3 + nd + int(with_dv))
    G, M = 4 * h, B * S
    gx, Wh = lstm_inputs(g, B, S, h, nd)
    lens = lengths_for(B, S, h * B + S)
    call, fb_bufs, n = run_lstm_fwd(lb, gx, Wh, lens, 1.0, B, S, h, nd)
    assert call() == MAC_OK
    sg, sc = fb_bufs["sg"][:n["sg"]], fb_bufs["sc"][:n["sc"]]
    d_out = randn(g, B, S, nd * h)
    d_vecq = randn(g, B, nd * h) if with_dv else None
    wsb = int(lb.mac_lstm_workspace_bytes(B, h, nd))
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")

    def bwd(lengths):
        dg = {"dG%d" % d: nan_guarded(M * G)[0] for d in range(nd)}
        c = lambda: lb.mac_lstm_bwd(P(Wh[0]), opt(Wh, 1), P(lengths), P(sg), P(sc), P(d_out), P(d_vecq), P(dg["dG0"]),
                                    P(dg["dG1"]) if nd == 2 else None, P(ws), wsb, B, S, h, nd, stream())
        return c, dg

    c, dg = bwd(lens)
    status = []
    got, same = run_twice(lambda: status.append(c()), dg)
    assert status == [MAC_OK, MAC_OK]
    rep = Report("lstm_bwd h=%d B=%d ndir=%d S=%d d_vecq=%s" % (h, B, nd, S, with_dv))
    rep.check(same, "bit-identical rerun")
    for d in range(nd):
        dGd = got["dG%d" % d][:M * G].view(B, S, G)
        rep.check(guard_intact(got["dG%d" % d], M * G), "dG%d guard" % d)
        ref, absref, tiny, live = lstm_bwd_reference(
            dGd, Wh[d], lens, sg.view(nd, B, S, G)[d], sc.view(nd, B, S, h)[d], d_out[:, :, d * h:(d + 1) * h],
            None if d_vecq is None else d_vecq[:, d * h:(d + 1) * h], d == 1)
        rep.add("dG%d" % d, dGd[live], ref[live], absref[live], TOL_BWD, tiny[live])
        rep.check(bool((dGd[~live] == 0).all()), "dG%d rows t >= len zero" % d)
    c2, dg2 = bwd(clamped(lens, S))
    assert c2() == MAC_OK
    torch.cuda.synchronize()
    rep.check(all(same_bits(got[k], dg2[k]) for k in got), "out-of-range lengths act as the clamped ones")
    rep.done()


# ================================================================================================ 3. LSTM, tensor cores
TC_CASES = [(1, 1, 128, 1), (1, 11, 300, 2), (63, 11, 300, 2), (64, 11, 128, 1), (65, 11, 300, 2), (65, 1, 128, 2),
            (130, 11, 128, 2), (130, 1, 300, 1), (64, 11, 300, 2)]


@pytest.mark.parametrize("B,S,E,nd", TC_CASES)
def test_lstm_tc_matches_fp64_per_step(B, S, E, nd):
    """mac_lstm_fwd_tc and mac_lstm_bwd_tc (h = 256): the per-step references on the kernels' own bf16 operands; BPTT's dG
    read back from the workspace; dkernel / dbias "+=" and dx from that dG"""
    lb = lib()
    h, G, M = 256, 1024, B * S
    Ep = (E + 127) // 128 * 128
    g = gen(B * 31 + S * 7 + E + nd)
    K = [randn(g, E + h, G, scale=(E + h) ** -0.5) for _ in range(nd)]
    Wh = [k[E:] for k in K]
    gx = [randn(g, M, G, scale=0.7) for _ in range(nd)]
    lens, fb = lengths_for(B, S, B + S + E), 1.0

    def fwd(lengths):
        n = {"out": M * nd * h, "vecq": B * nd * h, "sg": nd * M * G, "sc": nd * M * h, "shp": nd * M * h}
        bufs = {k: nan_guarded(v)[0] for k, v in n.items()}
        c = lambda: lb.mac_lstm_fwd_tc(P(gx[0]), opt(gx, 1), P(Wh[0]), opt(Wh, 1), P(lengths), fb, P(bufs["out"]),
                                       P(bufs["vecq"]), P(bufs["sg"]), P(bufs["sc"]), P(bufs["shp"]), B, S, h, nd, stream())
        return c, bufs, n

    c, bufs, n = fwd(lens)
    status = []
    got, same = run_twice(lambda: status.append(c()), bufs)
    assert status == [MAC_OK, MAC_OK]
    rep = Report("lstm_fwd_tc B=%d S=%d ndir=%d" % (B, S, nd))
    rep.check(same, "bit-identical rerun")
    check_fwd(rep, gx, Wh, lens, fb, got, n, B, S, h, nd, TOL_FWD_TC, bf16=True)
    c2, bufs2, _ = fwd(clamped(lens, S))
    assert c2() == MAC_OK
    torch.cuda.synchronize()
    rep.check(all(same_bits(got[k], bufs2[k]) for k in got), "out-of-range lengths act as the clamped ones")
    rep.done()

    sg, sc, shp = (got[k][:n[k]] for k in ("sg", "sc", "shp"))
    x16 = torch.zeros(M, Ep, dtype=torch.bfloat16, device="cuda")
    x16[:, :E] = randn(g, M, E).to(torch.bfloat16)
    d_out, d_vecq = randn(g, B, S, nd * h), randn(g, B, nd * h)
    wsb = int(lb.mac_lstm_bwd_tc_workspace_bytes(B, S, E, h, nd))
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    dk_pre = [randn(g, E + h, G, scale=0.3) for _ in range(nd)]
    db_pre = [randn(g, G, scale=0.3) for _ in range(nd)]

    def bwd(lengths):
        o = {"dk%d" % d: dk_pre[d].clone() for d in range(nd)}
        o.update({"db%d" % d: db_pre[d].clone() for d in range(nd)})
        o["dx"] = nan_guarded(M * E)[0]
        c = lambda: lb.mac_lstm_bwd_tc(P(x16), P(K[0]), opt(K, 1), P(lengths), P(sg), P(sc), P(shp), P(d_out), P(d_vecq),
                                       P(o["dk0"]), P(o["dk1"]) if nd == 2 else None, P(o["db0"]),
                                       P(o["db1"]) if nd == 2 else None, P(o["dx"]), P(ws), wsb, B, S, E, h, nd, stream())
        return c, o

    c, o = bwd(lens)
    status = []
    gotb, same = run_twice(lambda: status.append(c()), o)
    assert status == [MAC_OK, MAC_OK]
    off = (-ws.data_ptr()) % 1024                     # the workspace's slabs start at its first 1 KB boundary; dG first
    dG = ws[off:off + nd * M * G * 4].view(torch.float32).view(nd, M, G)
    rep = Report("lstm_bwd_tc B=%d S=%d E=%d ndir=%d" % (B, S, E, nd))
    rep.check(same, "bit-identical rerun")
    rep.check(guard_intact(gotb["dx"], M * E), "dx guard")
    dx_ref = torch.zeros(M, E, dtype=torch.float64, device="cuda")
    adx = torch.zeros_like(dx_ref)
    for d in range(nd):
        dGd = dG[d].view(B, S, G)
        ref, absref, tiny, live = lstm_bwd_reference(
            dGd, Wh[d], lens, sg.view(nd, B, S, G)[d], sc.view(nd, B, S, h)[d], d_out[:, :, d * h:(d + 1) * h],
            d_vecq[:, d * h:(d + 1) * h], d == 1, bf16=True)
        rep.add("dG%d" % d, dGd[live], ref[live], absref[live], TOL_BWD_TC["dG"], tiny[live])
        rep.check(bool((dGd[~live] == 0).all()), "dG%d rows t >= len zero" % d)
        g16 = bf16_round(dG[d])
        xh = torch.cat([x16[:, :E].double(), bf16_round(shp.view(nd, M, h)[d])], 1)
        rep.add_inc("dkernel%d" % d, gotb["dk%d" % d], dk_pre[d], xh.t() @ g16, xh.abs().t() @ g16.abs(),
                    TOL_BWD_TC["dkernel"])
        rep.add_inc("dbias%d" % d, gotb["db%d" % d], db_pre[d], dG[d].double().sum(0), dG[d].double().abs().sum(0),
                    TOL_BWD_TC["dbias"])
        wx = bf16_round(K[d][:E])
        dx_ref += g16 @ wx.t()
        adx += g16.abs() @ wx.abs().t()
    rep.add("dx", gotb["dx"][:M * E].view(M, E), dx_ref, adx, TOL_BWD_TC["dx"])
    c2, o2 = bwd(clamped(lens, S))
    assert c2() == MAC_OK
    torch.cuda.synchronize()
    rep.check(all(same_bits(gotb[k], o2[k]) for k in gotb), "out-of-range lengths act as the clamped ones")
    rep.done()


def test_question_encoder_bf16_single_direction_against_fp64():
    """QuestionEncoder(prec="bf16") without encBi (one direction of h = encDim = 256) against the fp64 encoder and its
    torch.autograd gradients"""
    from mac_network_b200.encoder import encoder_specs, init_encoder_params
    from oracle import encoder_torch_autograd
    from oracle.encoder_oracle import encoder_forward
    from tests.test_encoder_tc import TOL_FP64, _batch, _rel, _run
    B, S, V, E, D = 33, 23, 40, 300, 256
    keeps = (0.85, 0.92)
    pv = init_encoder_params(encoder_specs(V, E, D, bi=False), seed=3, dtype=np.float32)
    pv = {k: v.astype(np.float64) for k, v in pv.items()}
    q, lengths = _batch(B, S, V, 4)
    rng = np.random.RandomState(5)
    d_cntx, d_vecq = rng.standard_normal((B, S, D)) / np.sqrt(S), rng.standard_normal((B, D))
    enc, got = _run(pv, q, lengths, keeps, d_cntx, d_vecq)
    assert enc.ndir == 1 and enc.h == 256
    us = enc.dropout_uniforms(B, S, step=1)
    ref = encoder_forward(pv, q, lengths, keeps[0], keeps[1], uniforms=us)
    errs = {"cntx": _rel(got["cntx"], ref["questionCntxWords"]), "vecq": _rel(got["vecq"], ref["vecQuestions"])}
    _, _, gref = encoder_torch_autograd.run(pv, q, lengths, keeps[0], keeps[1], us, d_cntx=d_cntx, d_vecq=d_vecq)
    for k, gr in gref.items():
        errs[k] = _rel(got["grads"][k], gr)
    print("bf16 single direction vs fp64:", {k: "%.1e" % v for k, v in errs.items()})
    bad = {k: v for k, v in errs.items() if not v < TOL_FP64["out" if k in ("cntx", "vecq") else "grad"]}
    assert not bad, bad


# ================================================================================================ 4. stem patch kernels
PATCH_SHAPES = [(1, 1), (1, 5), (5, 1), (14, 14)]


@pytest.mark.parametrize("HW", PATCH_SHAPES)
@pytest.mark.parametrize("C", [4, 8, 12, 128])
def test_im2col3x3_equals_restatement(C, HW):
    lb = lib()
    H, W = HW
    for B in (1, 3):
        for keep in (1.0, 0.82):
            g = gen(C * 100 + H * 10 + W + B)
            x = randn(g, B, H, W, C)
            seed, step = 7, 2
            want = im2col_reference(x, keep, seed, step)
            M = B * H * W
            for bf in (0, 1):
                dt = torch.bfloat16 if bf else torch.float32
                buf = torch.full((M * 9 * C + GUARD,), float("nan"), dtype=dt, device="cuda")
                assert lb.mac_im2col3x3(P(x), P(buf), bf, keep, seed, SITE, step, B, H, W, C, stream()) == MAC_OK
                torch.cuda.synchronize()
                got = buf[:M * 9 * C].view(M, 9 * C)
                w = want.to(dt)
                assert torch.equal(got, w), ("im2col", B, H, W, C, keep, bf, int((got != w).sum()))
                assert bool(buf[M * 9 * C:].float().isnan().all())


@pytest.mark.parametrize("HW", PATCH_SHAPES)
@pytest.mark.parametrize("C", [4, 8, 12, 128])
def test_col2im3x3_equals_restatement(C, HW):
    lb = lib()
    H, W = HW
    for B in (1, 3):
        for keep in (1.0, 0.82):
            g = gen(C * 100 + H * 10 + W + B + 1)
            M = B * H * W
            dcols = randn(g, M, 9 * C)
            seed, step = 9, 4
            want = col2im_reference(dcols, (B, H, W, C), keep, seed, step)
            buf, dx = nan_guarded(M * C)
            assert lb.mac_col2im3x3(P(dcols), P(dx), keep, seed, SITE, step, B, H, W, C, stream()) == MAC_OK
            torch.cuda.synchronize()
            assert torch.equal(dx.view(B, H, W, C), want), ("col2im", B, H, W, C, keep)
            assert guard_intact(buf, M * C)
