"""Question input unit timing at the headline question shape (B=64, S=40, E=300, 2 x 256, which runs the persistent
cluster kernel of the LSTM): forward only and forward+backward, eager and as a CUDA graph."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from mac_network_b200.encoder import QuestionEncoder, encoder_specs, init_encoder_params  # noqa: E402

torch.cuda.set_device(0)
B, S, V, E, D = 64, 40, 90, 300, 512
pv = init_encoder_params(encoder_specs(V, E, D), seed=1)
dev = {k: torch.from_numpy(v).cuda() for k, v in pv.items()}
rng = np.random.RandomState(2)
lengths = rng.randint(S // 2, S + 1, size=(B,)).astype(np.int32)
lengths[0] = S
q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
q[np.arange(S)[None, :] >= lengths[:, None]] = 0
qd, ld = torch.from_numpy(q).cuda(), torch.from_numpy(lengths).cuda()


def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


enc = QuestionEncoder(dev)
out = {"forward_eager_us": timeit(lambda: enc.forward(qd, ld))}
g = torch.cuda.CUDAGraph()
s = torch.cuda.Stream()
with torch.cuda.stream(s):
    enc.forward(qd, ld)
    s.synchronize()
    with torch.cuda.graph(g, stream=s):
        enc.forward(qd, ld)
out["forward_graph_us"] = timeit(g.replay)
enc_t = QuestionEncoder(dev, keep_input=0.85, keep_question=0.92)
grads = {k: torch.zeros_like(v) for k, v in dev.items()}
dc, dq = torch.randn(B, S, D, device="cuda"), torch.randn(B, D, device="cuda")


def fb():
    enc_t.forward(qd, ld, save_for_backward=True)
    enc_t.backward(dc, dq, grads)


out["train_forward_backward_eager_us"] = timeit(fb, iters=10)
print(json.dumps(out), flush=True)
