"""Both forms of the LSTM recurrence (csrc/encoder.cu, mac_lstm_fwd) against the fp64 oracle, forward and (through the
tensors they save) backward.  At h == 256 (encDim D = 512, the reference default) the persistent form runs,
`lstm_seq_kernel`: one thread-block cluster of 8 CTAs per (direction, 8 batch rows) keeps the recurrent weights in shared
memory for all S steps and exchanges h over DSMEM.  Every other h runs the per-step kernels (D = 384: h = 192).  Runs
last: the persistent form is the newest kernel in the library."""
import numpy as np
import pytest

from oracle.encoder_oracle import encoder_forward
from oracle import encoder_torch_autograd
from mac_network_b200.encoder import encoder_specs, init_encoder_params
from tests._util import max_rel


@pytest.mark.gpu
@pytest.mark.parametrize("D", [512, 384])
@pytest.mark.parametrize("B,S,keeps", [(64, 40, (1.0, 1.0)), (13, 11, (0.85, 0.92))])
def test_lstm_matches_oracle(B, S, keeps, D):
    import torch
    from mac_network_b200.encoder import QuestionEncoder
    V, E = 90, 300
    pv = init_encoder_params(encoder_specs(V, E, D), seed=51, dtype=np.float64)
    rng = np.random.RandomState(52)
    lengths = rng.randint(max(1, S // 2), S + 1, size=(B,)).astype(np.int32)
    lengths[0], lengths[1] = S, 1
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    dev = {k: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)).cuda() for k, v in pv.items()}
    qd, ld = torch.from_numpy(q).cuda(), torch.from_numpy(lengths).cuda()
    d_cntx = rng.standard_normal((B, S, D)) / np.sqrt(S)
    d_vecq = rng.standard_normal((B, D))
    enc = QuestionEncoder(dev, keep_input=keeps[0], keep_question=keeps[1], seed=9)
    _, cntx, vecq = enc.forward(qd, ld, step=2, save_for_backward=True)
    grads = {k: torch.zeros_like(v) for k, v in dev.items()}
    enc.backward(torch.from_numpy(d_cntx.astype(np.float32)).cuda(), torch.from_numpy(d_vecq.astype(np.float32)).cuda(), grads)
    torch.cuda.synchronize()
    us = enc.dropout_uniforms(B, S, step=2)
    ref = encoder_forward(pv, q, lengths, keeps[0], keeps[1], uniforms=us)
    _, _, gref = encoder_torch_autograd.run(pv, q, lengths, keeps[0], keeps[1], us, d_cntx=d_cntx, d_vecq=d_vecq)
    assert max_rel(cntx.cpu().numpy(), ref["questionCntxWords"]) < 1e-4
    assert max_rel(vecq.cpu().numpy(), ref["vecQuestions"]) < 1e-4
    for k, gr in gref.items():
        assert max_rel(grads[k].cpu().numpy(), gr) < 2e-4, k
