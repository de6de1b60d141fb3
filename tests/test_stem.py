"""Image stem (SURVEY section 8(f) rank 1): oracle vs fixtures from the reference's own ops.CNNLayer (CPU), product
(fused dropout+im2col kernel + GEMM) vs oracle on the GPU for the fp32 and the wgmma bf16 path."""
import json
import os

import numpy as np
import pytest

from oracle.model_torch_autograd import stem_grads
from oracle.stem_oracle import stem_forward
from mac_network_b200.stem import stem_specs, init_stem_params
from tests._util import GOLDEN_DIR, max_rel


def _load(case):
    z = np.load(os.path.join(GOLDEN_DIR, case + ".npz"))
    meta = json.loads(bytes(z["meta_json"]).decode())
    return meta, {k: z[k] for k in z.files if k != "meta_json"}


@pytest.mark.parametrize("case", ["stem_eval", "stem_train"])
def test_stem_oracle_matches_reference_fixture(case):
    meta, g = _load(case)
    B, H, W, cin, cout = meta["shape"]
    specs = stem_specs(cin, cout, meta["layers"], meta["ksize"])
    assert {k: list(v[0]) for k, v in specs.items()} == meta["variables"]
    params = init_stem_params(specs, seed=meta["param_seed"], dtype=np.float64)
    us = [g["uniform_%03d" % i] for i in range(meta["n_uniform"])]
    kb = stem_forward(meta["relu"], params, g["images"], keep=meta["keep"], uniforms=us)
    assert np.max(np.abs(kb - g["kb"])) < 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("prec,keep,shape", [("fp32", 1.0, (4, 14, 14, 1024, 512)), ("fp32", 0.82, (2, 7, 7, 64, 128)),
                                             ("bf16", 1.0, (8, 14, 14, 1024, 512)), ("bf16", 0.82, (8, 14, 14, 256, 256))])
def test_stem_gpu(prec, keep, shape):
    import torch
    from mac_network_b200 import _lib as L
    from mac_network_b200.stem import Stem, SITE_STEM
    lib = L.load()
    B, H, W, cin, cout = shape
    specs = stem_specs(cin, cout)
    pv = init_stem_params(specs, seed=5, dtype=np.float64)
    images = np.maximum(np.random.RandomState(6).standard_normal((B, H, W, cin)), 0)
    params = {k: torch.from_numpy(v.astype(np.float32)).cuda() for k, v in pv.items()}
    st = Stem(params, relu="ELU", prec=prec, seed=31)
    kb = st.forward(torch.from_numpy(images.astype(np.float32)).cuda(), keep=keep, step=2)
    torch.cuda.synchronize()
    us = []
    if keep < 1.0:
        for layer, c in ((0, cin), (1, cout)):
            u = torch.empty(B * H * W * c, device="cuda")
            L.check(lib.mac_dropout_uniform(31, SITE_STEM + layer, 2, L.ptr(u), u.numel(), L.stream_ptr()))
            us.append(u.cpu().numpy().astype(np.float64).reshape(B, H, W, c))
    ref = stem_forward("ELU", pv, images, keep=keep, uniforms=us)
    err = max_rel(kb.cpu().numpy(), ref)
    print("stem %s keep=%s max-rel error %.2e" % (prec, keep, err))
    assert err < (1e-4 if prec == "fp32" else 2e-2)


def test_torch_stem_restatement_matches_oracle():
    meta, g = _load("stem_train")
    B, H, W, cin, cout = meta["shape"]
    pv = init_stem_params(stem_specs(cin, cout, meta["layers"], meta["ksize"]), seed=meta["param_seed"], dtype=np.float64)
    us = [g["uniform_%03d" % i] for i in range(meta["n_uniform"])]
    kb, _, _ = stem_grads(meta["relu"], pv, g["images"], meta["keep"], us, np.zeros_like(g["kb"]))
    assert np.max(np.abs(kb - g["kb"])) < 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("keep,shape", [(1.0, (3, 14, 14, 64, 128)), (0.82, (2, 7, 7, 32, 64)), (0.82, (1, 5, 4, 8, 8))])
def test_stem_backward_gpu(keep, shape):
    """Stem backward (activation', wgrad/dgrad GEMMs on the re-generated patch matrix, col2im with the dropout mask) against
    torch.autograd on the fp64 restatement."""
    import torch
    from mac_network_b200 import _lib as L
    from mac_network_b200.stem import Stem, SITE_STEM
    lib = L.load()
    B, H, W, cin, cout = shape
    pv = init_stem_params(stem_specs(cin, cout), seed=8, dtype=np.float64)
    images = np.maximum(np.random.RandomState(9).standard_normal((B, H, W, cin)), 0)
    params = {k: torch.from_numpy(v.astype(np.float32)).cuda() for k, v in pv.items()}
    st = Stem(params, relu="ELU", prec="fp32", seed=13)
    kb = st.forward(torch.from_numpy(images.astype(np.float32)).cuda(), keep=keep, step=4, save_for_backward=True)
    d_kb = np.random.RandomState(10).standard_normal(tuple(kb.shape))
    grads = {k: torch.zeros_like(v) for k, v in params.items()}
    d_img = st.backward(torch.from_numpy(d_kb.astype(np.float32)).cuda(), grads, need_d_images=True)
    torch.cuda.synchronize()
    us = []
    if keep < 1.0:
        for layer, c in ((0, cin), (1, cout)):
            u = torch.empty(B * H * W * c, device="cuda")
            L.check(lib.mac_dropout_uniform(13, SITE_STEM + layer, 4, L.ptr(u), u.numel(), L.stream_ptr()))
            us.append(u.cpu().numpy().astype(np.float64).reshape(B, H, W, c))
    kb_ref, gref, dimg_ref = stem_grads("ELU", pv, images, keep, us, d_kb)
    assert max_rel(kb.cpu().numpy(), kb_ref) < 1e-4
    for k in gref:
        err = max_rel(grads[k].cpu().numpy(), gref[k])
        print("stem grad %-40s max-rel %.2e" % (k, err))
        assert err < 2e-4, (k, err)
    assert max_rel(d_img.cpu().numpy(), dimg_ref) < 2e-4
