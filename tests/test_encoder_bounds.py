"""CPU checks of tests/test_gpu_encoder_kernels.py with that file's own reference and bound code.

1. The references are the operations: on small shapes the per-step LSTM references reproduce the fp64 encoder
   (oracle/encoder_oracle.py, oracle/encoder_tc_oracle.py without rounding) and its torch.autograd gradients
   (oracle/encoder_torch_autograd.py); the embedding and patch references reproduce the oracle's lookup and dropout,
   torch's unfold / fold.
2. The bounds are tight: an fp32 restatement of each kernel passes them, and each planted fault is rejected by a wide
   margin -- forget_bias dropped, the backward direction walking t = S-1-s, one 8-unit chunk reading the wrong Wh column
   block, save_hprev one step stale, BPTT missing its last partial 256-column chunk, d_vecq added one step late, the
   embedding mask taken by element index instead of quad index, and mac_embed_bwd without its mask.
3. The index arithmetic of a question length > S as the LSTM kernels did it before they clamped: the backward direction
   addresses rows of the next sample (past the buffer for the last one) and the forward direction's BPTT never adds
   d_vecq.  With the clamp both are in range."""
import numpy as np
import torch

from mac_network_b200.encoder import encoder_specs, init_encoder_params
from oracle import encoder_torch_autograd
from oracle.encoder_oracle import ENC, embed, encoder_forward
from oracle.encoder_tc_oracle import EncoderTC
from oracle.philox import philox_uniform
from tests.test_gpu_backward_kernels import ratio
from tests.test_gpu_encoder_kernels import (SITE, TOL_BWD, TOL_EMBED_BWD, TOL_FWD, col2im_reference, embed_bwd_reference,
                                            embed_reference, f32_inv, im2col_reference, lstm_bwd_reference,
                                            lstm_fwd_exact, lstm_fwd_reference, step_index)

MARGIN = 100


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _lengths(B, S):
    lens = torch.randint(1, S + 1, (B,), generator=_gen(B * S))
    lens[:2] = torch.tensor([S, 1])
    return lens.to(torch.int32)


def _encoder_case(B=5, S=6, V=9, E=8, D=16, seed=1):
    pv = init_encoder_params(encoder_specs(V, E, D), seed=seed)
    pv = {k: v.astype(np.float64) for k, v in pv.items()}
    rng = np.random.RandomState(seed)
    lengths = rng.randint(1, S + 1, size=B).astype(np.int32)
    lengths[:2] = [S, 1]
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    return pv, q, lengths, rng.standard_normal((B, S, D)), rng.standard_normal((B, D))


# ------------------------------------------------------------------------------------------------ 1. the references
def test_lstm_references_are_the_encoder():
    """From the fp64 encoder's own saved gates, c and h_prev, the forward references reproduce the next step's values and
    the outputs; iterating the backward reference to its fixed point gives autograd's kernel and bias gradients."""
    B, S, E, D = 5, 6, 8, 16
    pv, q, lengths, d_cntx, d_vecq = _encoder_case(B, S, E=E, D=D)
    h = D // 2
    fo = EncoderTC(pv, bf16=False).forward(q, lengths)
    want = encoder_forward(pv, q, lengths)
    assert np.allclose(fo["questionCntxWords"], want["questionCntxWords"], rtol=0, atol=1e-13)
    _, _, gref = encoder_torch_autograd.run(pv, q, lengths, d_cntx=d_cntx, d_vecq=d_vecq)
    lens = torch.from_numpy(lengths)
    x = torch.from_numpy(fo["x16"])
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    for d, name in enumerate(("fw", "bw")):
        K, b = T(pv[ENC + name + "/basic_lstm_cell/kernel"]), T(pv[ENC + name + "/basic_lstm_cell/bias"])
        gx = x @ K[:E] + b
        sg, sc, shp = T(fo["gates"][d]), T(fo["c"][d]), T(fo["hprev"][d])
        out = T(fo["questionCntxWords"][:, :, d * h:(d + 1) * h])
        refs, live = lstm_fwd_reference(gx, K[E:], lens, 1.0, sg, sc, shp, d == 1)
        for key, got in (("gates", sg), ("c", sc), ("out", out)):
            ref, absref, _ = refs[key]
            assert torch.allclose(ref[live], got[live], rtol=0, atol=1e-13), (name, key)
            if key != "gates":                # the gates' absref bounds the pre-activation, |act'| <= 1 carries it over
                assert bool((absref[live] >= ref[live].abs() - 1e-13).all()), (name, key)
        vecq = T(fo["vecQuestions"][:, d * h:(d + 1) * h])
        for what, ok in lstm_fwd_exact(out, vecq, shp, lens, d == 1):
            assert ok, (name, what)
        dG = torch.zeros(B, S, 4 * h, dtype=torch.float64)
        for _ in range(S):                     # step s needs dG of step s+1 only: S rounds reach the fixed point
            ref, absref, _, live = lstm_bwd_reference(dG, K[E:], lens, sg, sc, T(d_cntx[:, :, d * h:(d + 1) * h]),
                                                      T(d_vecq[:, d * h:(d + 1) * h]), d == 1)
            dG = torch.where(live[:, :, None], ref, torch.zeros(()))
        assert bool((absref[live] >= ref[live].abs() - 1e-13).all())
        xh = torch.cat([x, shp], 2).reshape(B * S, -1)
        dK, db = xh.t() @ dG.reshape(B * S, -1), dG.reshape(B * S, -1).sum(0)
        assert np.allclose(dK.numpy(), gref[ENC + name + "/basic_lstm_cell/kernel"], rtol=0, atol=1e-12), name
        assert np.allclose(db.numpy(), gref[ENC + name + "/basic_lstm_cell/bias"], rtol=0, atol=1e-12), name


def test_embedding_references_are_the_lookup_and_dropout():
    V, E, B, S, keep, seed, step = 7, 12, 3, 5, 0.85, 11, 2
    g = _gen(2)
    emb = torch.randn(V, E, generator=g)
    idx = torch.randint(0, V + 1, (B, S), generator=g, dtype=torch.int32)
    idx.view(-1)[:3] = torch.tensor([V + 1, -1, 1 << 20])
    raw, out = embed_reference(emb, idx, keep, seed, step)
    q = idx.clone()
    q[(q < 0) | (q > V)] = 0                   # ids outside 0..V read as the padding row
    want = embed(emb.double().numpy(), q.numpy()).reshape(B * S, E)
    assert np.array_equal(raw.double().numpy(), want)
    u = philox_uniform(seed, SITE, step, B * S * E).reshape(B * S, E)
    assert np.allclose(out.double().numpy(), want / keep * np.floor(keep + u), rtol=1e-6, atol=0)
    d_out = torch.randn(B, S, E, generator=g)
    inc, _, used = embed_bwd_reference(d_out, idx, V, keep, seed, step)
    dx = d_out.double().numpy().reshape(B * S, E) / keep * np.floor(keep + u)
    demb = np.zeros((V, E))
    qq = q.numpy().reshape(-1)
    np.add.at(demb, qq[qq > 0] - 1, dx[qq > 0])
    assert np.allclose(inc.numpy(), demb, rtol=1e-6, atol=1e-12)
    assert np.array_equal(used.numpy(), np.isin(np.arange(V), qq[qq > 0] - 1))


def test_patch_references_are_unfold_and_fold():
    B, H, W, C = 2, 5, 4, 8
    x = torch.randn(B, H, W, C, generator=_gen(3), dtype=torch.float64)
    cols = im2col_reference(x, 1.0, 0, 0)
    u = torch.nn.functional.unfold(x.permute(0, 3, 1, 2), 3, padding=1)           # [B, C*9, H*W], (c, kh, kw)
    want = u.view(B, C, 9, H * W).permute(0, 3, 2, 1).reshape(B * H * W, 9 * C)
    assert torch.equal(cols, want)
    dcols = torch.randn(B * H * W, 9 * C, generator=_gen(4), dtype=torch.float64)
    dx = col2im_reference(dcols, (B, H, W, C), 1.0, 0, 0)
    f = torch.nn.functional.fold(dcols.view(B, H * W, 9, C).permute(0, 3, 2, 1).reshape(B, C * 9, H * W), (H, W), 3,
                                 padding=1)
    assert torch.allclose(dx, f.permute(0, 2, 3, 1), rtol=0, atol=1e-12)


# ------------------------------------------------------------------------------------------------ fp32 restatements
def _fwd_fp32(gx, Wh, lens, fb, reverse, fault=None):
    """one direction of mac_lstm_fwd in fp32 torch ops (time-order [B, S, .] outputs as the kernel leaves them), with the
    planted faults as switches"""
    B, S, G = gx.shape
    h = G // 4
    L = lens.long().clamp(0, S)
    out, shp = torch.zeros(B, S, h), torch.zeros(B, S, h)
    sg, sc = torch.full((B, S, G), float("nan")), torch.full((B, S, h), float("nan"))
    W = Wh.clone()
    if fault == "chunk":                       # units 8..15 read the columns of units 16..23
        for gate in range(4):
            W[:, gate * h + 8:gate * h + 16] = Wh[:, gate * h + 16:gate * h + 24]
    c, hc, hold = torch.zeros(B, h), torch.zeros(B, h), torch.zeros(B, h)
    rows = torch.arange(B)
    for s in range(S):
        live = s < L
        t = torch.where(live, (S - 1 - s if fault == "bw_walks_S" else L - 1 - s) if reverse else torch.full_like(L, s), 0)
        pre = gx[rows, t] + hc @ W
        i, j, f, o = pre.split(h, 1)
        i, j, o = torch.sigmoid(i), torch.tanh(j), torch.sigmoid(o)
        f = torch.sigmoid(f if fault == "no_forget_bias" else f + fb)
        cn = c * f + i * j
        hn = torch.tanh(cn) * o
        lr = rows[live]
        out[lr, t[lr]] = hn[lr]
        sg[lr, t[lr]] = torch.cat([i, j, f, o], 1)[lr]
        sc[lr, t[lr]] = cn[lr]
        shp[lr, t[lr]] = (hold if fault == "stale_hprev" else hc)[lr]
        hold = hc.clone()
        c = torch.where(live[:, None], cn, c)
        hc = torch.where(live[:, None], hn, hc)
    return out, hc, sg, sc, shp


def _bwd_fp32(Wh, lens, sg, sc, d_out, d_vecq, reverse, fault=None):
    """one direction of mac_lstm_bwd in fp32 torch ops: dG [B, S, 4h] by time index"""
    B, S, G = sg.shape
    h = G // 4
    L = lens.long().clamp(0, S)
    dG = torch.zeros(B, S, G)
    dcc = torch.zeros(B, h)
    rows = torch.arange(B)
    kmax = min(G, 256) if fault == "tail_chunk" else G
    for s in range(S - 1, -1, -1):
        live = s < L
        t = torch.where(live, (L - 1 - s) if reverse else torch.full_like(L, s), 0)
        nxt = torch.zeros(B, G)
        has = s + 1 < L
        t1 = torch.where(has, (L - 2 - s) if reverse else torch.full_like(L, s + 1), 0)
        nxt[has] = dG[rows[has], t1[has]]
        rec = nxt[:, :kmax] @ Wh[:, :kmax].t()
        is_last = s + 1 >= L
        late = s + 2 == L                   # the fault adds d_vecq one step late: at the step before the last live one
        dh = d_out[rows, t] + torch.where(is_last[:, None], torch.zeros(()) if fault == "vecq_late" else d_vecq, rec)
        if fault == "vecq_late":
            dh = dh + torch.where(late[:, None], d_vecq, torch.zeros(()))
        gi, gj, gf, go = sg[rows, t].split(h, 1)
        cn = sc[rows, t]
        tp = torch.where(torch.full_like(L, s) > 0, t + 1 if reverse else t - 1, 0).clamp(0, S - 1)
        cp = torch.where(torch.full((B, 1), s > 0), sc[rows, tp], torch.zeros(()))
        tc = torch.tanh(cn)
        dc = dcc + dh * go * (1 - tc * tc)
        dg = torch.cat([dc * gj * gi * (1 - gi), dc * gi * (1 - gj * gj), dc * cp * gf * (1 - gf), dh * tc * go * (1 - go)], 1)
        lr = rows[live]
        dG[lr, t[lr]] = dg[lr]
        dcc = torch.where(live[:, None], dc * gf, dcc)
    return dG


def _fwd_worst(gx, Wh, lens, fb, reverse, res):
    """the worst ratio / tol over the forward's bounds, inf when an exact relation fails"""
    out, vecq, sg, sc, shp = res
    refs, live = lstm_fwd_reference(gx, Wh, lens, fb, sg, sc, shp, reverse)
    worst = 0.0
    for key, got in (("gates", sg), ("c", sc), ("out", out)):
        ref, absref, tiny = refs[key]
        worst = max(worst, ratio(got[live], ref[live], absref[live], tiny[live] if torch.is_tensor(tiny) else tiny)
                    / TOL_FWD[key])
    if not all(ok for _, ok in lstm_fwd_exact(out, vecq, shp, lens, reverse)):
        worst = float("inf")
    return worst


def _check(e_ok, e_bad, what):
    print("%s: fp32 %.2e, fault %.2e (in units of the bound)" % (what, e_ok, e_bad))
    assert e_ok <= 1.0, (what, e_ok)
    assert e_bad > MARGIN, (what, e_bad)


def _lstm_case(B, S, h, seed):
    g = _gen(seed)
    gx = torch.randn(B, S, 4 * h, generator=g) * 0.7
    Wh = torch.randn(h, 4 * h, generator=g) * h ** -0.5
    return gx, Wh, _lengths(B, S)


# ------------------------------------------------------------------------------------------------ 2. planted faults
def test_fwd_bounds_reject_planted_faults():
    B, S, h = 9, 7, 32
    gx, Wh, lens = _lstm_case(B, S, h, 5)
    for reverse, fault in ((False, "no_forget_bias"), (True, "bw_walks_S"), (False, "chunk"), (True, "chunk"),
                           (False, "stale_hprev"), (True, "stale_hprev")):
        ok = _fwd_worst(gx, Wh, lens, 1.0, reverse, _fwd_fp32(gx, Wh, lens, 1.0, reverse))
        bad = _fwd_worst(gx, Wh, lens, 1.0, reverse, _fwd_fp32(gx, Wh, lens, 1.0, reverse, fault))
        _check(ok, bad, "lstm_fwd %s (%s)" % (fault, "bw" if reverse else "fw"))


def test_bwd_bounds_reject_planted_faults():
    """h = 72 (G = 288: a full 256-column chunk and a partial one)"""
    B, S, h = 9, 7, 72
    gx, Wh, lens = _lstm_case(B, S, h, 6)
    g = _gen(7)
    d_out, d_vecq = torch.randn(B, S, h, generator=g), torch.randn(B, h, generator=g)
    for reverse in (False, True):
        _, _, sg, sc, _ = _fwd_fp32(gx, Wh, lens, 1.0, reverse)
        for fault in ("tail_chunk", "vecq_late"):
            e = []
            for f in (None, fault):
                dG = _bwd_fp32(Wh, lens, sg, sc, d_out, d_vecq, reverse, f)
                ref, absref, tiny, live = lstm_bwd_reference(dG, Wh, lens, sg, sc, d_out, d_vecq, reverse)
                e.append(ratio(dG[live], ref[live], absref[live], tiny[live]) / TOL_BWD)
            _check(e[0], e[1], "lstm_bwd %s (%s)" % (fault, "bw" if reverse else "fw"))


def test_embed_fwd_rejects_the_mask_by_element_index():
    """the kernels number the Philox draws by quad (counter i/4, word i%4); a mask drawn with counter i is a different mask"""
    V, E, B, S, keep, seed, step = 11, 300, 4, 6, 0.85, 13, 1
    g = _gen(8)
    emb = torch.randn(V, E, generator=g)
    idx = torch.randint(1, V + 1, (B, S), generator=g, dtype=torch.int32)
    raw, out = embed_reference(emb, idx, keep, seed, step)
    n = raw.numel()
    words = philox_uniform(seed, SITE, step, 4 * n).reshape(n, 4)[np.arange(n), np.arange(n) % 4]
    thr = np.ceil((1.0 - float(np.float32(keep))) * 16777216.0)
    m_bad = torch.from_numpy(words * 16777216.0 >= thr).view_as(raw)
    bad = torch.where(m_bad, raw * f32_inv(keep), torch.zeros(()))
    differ = int((bad != out).sum())
    print("embed mask by element index: %d of %d elements differ" % (differ, n))
    assert differ > n // 10


def test_embed_bwd_bound_rejects_a_missing_mask():
    V, E, B, S, keep, seed, step = 5, 64, 13, 9, 0.85, 3, 4
    g = _gen(9)
    idx = torch.randint(0, V + 1, (B, S), generator=g, dtype=torch.int32)
    d_out = torch.randn(B, S, E, generator=g)
    inc, ainc, used = embed_bwd_reference(d_out, idx, V, keep, seed, step)
    ids = idx.reshape(-1).long()
    ok_pos = (ids >= 1) & (ids <= V)
    d = d_out.reshape(-1, E)
    m = torch.from_numpy(philox_uniform(seed, SITE, step, d.numel()).reshape(d.shape) * 16777216.0 >=
                         np.ceil((1.0 - float(np.float32(keep))) * 16777216.0))
    good = torch.zeros(V, E).index_add_(0, ids[ok_pos] - 1, torch.where(m, d * f32_inv(keep), torch.zeros(()))[ok_pos])
    bad = torch.zeros(V, E).index_add_(0, ids[ok_pos] - 1, (d * f32_inv(keep))[ok_pos])
    _check(ratio(good[used], inc[used], ainc[used]) / TOL_EMBED_BWD, ratio(bad[used], inc[used], ainc[used]) / TOL_EMBED_BWD,
           "embed_bwd without its mask")


# ------------------------------------------------------------------------------------------------ 3. lengths > S
def _unclamped_rows(length, s, S, b):
    """the rows of [B*S] the LSTM kernels addressed at step s for an unclamped length, backward direction: the forward
    kernels' gx read and out_seq / saved stores (t = len-1-s), the BPTT kernel's dG(s+1) read (t1 = len-2-s)"""
    live = s < length
    t = length - 1 - s
    return (b * S + t if live else None), (b * S + length - 2 - s if s + 1 < length else None)


def test_unclamped_length_above_S_addresses_the_next_sample():
    B, S = 4, 6
    length = S + 3
    for b in range(B):
        row, row1 = _unclamped_rows(length, 0, S, b)
        assert row >= (b + 1) * S and row1 >= (b + 1) * S                # rows of sample b + 1
    row, _ = _unclamped_rows(length, 0, S, B - 1)
    assert row >= B * S                                                  # past the end of the buffer
    # forward direction, BPTT: d_vecq is added where s + 1 >= len; at s = S - 1 that never holds for len > S
    assert not any(s + 1 >= length for s in range(S))
    # with the clamp: every live step's row is in the sample, and the forward direction's last live step is S - 1
    t, live, L = step_index(torch.tensor([length, -2, 0], dtype=torch.int32), S, True)
    assert int(L[0]) == S and int(L[1]) == 0 and not bool(live[1:].any())
    assert bool(((t >= 0) & (t < S)).all())
    assert int(t[0, 0]) == S - 1 and int(t[0, S - 1]) == 0
