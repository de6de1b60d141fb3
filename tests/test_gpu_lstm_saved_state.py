"""The LSTM's saved state for the backward (csrc/encoder.cu, mac_lstm_fwd): rows of save_hprev past a question's length are
multiplied by zero gate gradients in the weight-gradient GEMM, so they must be finite whatever the buffer held before.
Every scratch buffer of the encoder is NaN-filled here; the gradients must still match the fp64 oracle in both LSTM forms
(D = 512, h = 256: the persistent cluster kernel; D = 384, h = 192: the per-step kernels)."""
import numpy as np
import pytest

from oracle import encoder_torch_autograd
from mac_network_b200.encoder import encoder_specs, init_encoder_params
from tests._util import max_rel


@pytest.mark.gpu
@pytest.mark.parametrize("D", [512, 384])
def test_lstm_gradients_ignore_stale_buffer_contents(D):
    import torch
    from mac_network_b200.encoder import QuestionEncoder
    B, S, V, E = 13, 11, 90, 300
    pv = init_encoder_params(encoder_specs(V, E, D), seed=61, dtype=np.float64)
    rng = np.random.RandomState(62)
    lengths = rng.randint(1, S + 1, size=(B,)).astype(np.int32)
    lengths[0], lengths[1] = S, 1
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    dev = {k: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)).cuda() for k, v in pv.items()}
    d_cntx = rng.standard_normal((B, S, D)) / np.sqrt(S)
    d_vecq = rng.standard_normal((B, D))
    enc = QuestionEncoder(dev, keep_input=1.0, keep_question=1.0, seed=9)
    enc._new = lambda *shape: torch.full(shape, float("nan"), dtype=torch.float32, device="cuda")
    enc.forward(torch.from_numpy(q).cuda(), torch.from_numpy(lengths).cuda(), step=2, save_for_backward=True)
    grads = {k: torch.zeros_like(v) for k, v in dev.items()}
    enc.backward(torch.from_numpy(d_cntx.astype(np.float32)).cuda(), torch.from_numpy(d_vecq.astype(np.float32)).cuda(), grads)
    torch.cuda.synchronize()
    _, _, gref = encoder_torch_autograd.run(pv, q, lengths, 1.0, 1.0, enc.dropout_uniforms(B, S, step=2), d_cntx=d_cntx,
                                            d_vecq=d_vecq)
    for k, gr in gref.items():
        got = grads[k].cpu().numpy()
        assert np.isfinite(got).all(), k
        assert max_rel(got, gr) < 2e-4, k
