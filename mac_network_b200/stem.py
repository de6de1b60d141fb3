"""Image stem -- the producer of the knowledge base (SURVEY.md section 8(f), "next" row 1):
`MACnet.stem` (`model.py:165-204`) = `ops.CNNLayer` (`ops.py:423-438`) of `stemNumLayers` x `ops.cnn` (`ops.py:380-405`):
dropout on the layer input, 3x3 stride-1 SAME convolution (HWIO kernel) + bias, ELU after every layer; then the
`[B,H,W,d] -> [B, H*W, d]` reshape.  177.6 GFLOP per B=64 batch (56 % of the twelve cell steps).

GPU formulation: convolution as GEMM.  `mac_im2col3x3` builds the `[B*H*W, 9*C]` patch matrix (tap-major, channel fastest
-- exactly the row-major reshape of the HWIO kernel to `[9*C, Cout]`) with the input dropout fused (the Philox mask is
indexed by the SOURCE element, so all nine copies of a pixel share its mask), in bf16 for the wgmma GEMM
(`mac_linear_tc_fwd`, ELU epilogue) or fp32 for the parity GEMM (`mac_linear_fwd`)."""
import collections
import ctypes

import numpy as np
import torch

from . import _lib
from ._lib import ACT, check, ptr, stream_ptr

SITE_STEM = 32            # Philox site base for the stem's input dropouts (site + layer index)


def stem_specs(in_dim, out_dim, num_layers=2, ksize=3, stem_dim=None):
    stem_dim = out_dim if stem_dim is None else stem_dim
    dims = [in_dim] + [stem_dim] * (num_layers - 1) + [out_dim]
    s = collections.OrderedDict()
    for i in range(num_layers):
        s["stem/cnnLayercnn_%d/kernels/kernel" % i] = ((ksize, ksize, dims[i], dims[i + 1]), "xavier")
        s["stem/cnnLayercnn_%d/biases/bias" % i] = ((dims[i + 1],), "zeros")
    return s


def init_stem_params(specs, seed=0, dtype=np.float32, bias_scale=0.1):
    rng = np.random.RandomState(seed)
    out = collections.OrderedDict()
    for name, (shape, kind) in specs.items():
        if kind == "zeros":
            v = bias_scale * rng.standard_normal(shape)
        else:       # tf.contrib.layers.xavier_initializer on [kh,kw,cin,cout]: fan_in = kh*kw*cin, fan_out = kh*kw*cout
            rf = shape[0] * shape[1]
            lim = np.sqrt(6.0 / (rf * shape[2] + rf * shape[3]))
            v = rng.uniform(-lim, lim, size=shape)
        out[name] = np.asarray(v, dtype=dtype)
    return out


class Stem(object):
    def __init__(self, params, relu="ELU", prec="fp32", seed=0, version=None):
        """`params`: dict TF-name -> CUDA fp32 tensor (HWIO kernels, biases).  `version`: optional callable returning a counter
        that changes whenever the parameter values do (`MACParams.version`): the packed bf16 kernels are rebuilt when it moves
        (optimizer step, checkpoint restore, EMA swap -- ADVICE r1), whoever changed the values."""
        self.lib = _lib.load()
        self.p = params
        self.relu, self.prec, self.seed = relu, prec, int(seed)
        self.nlayers = len([k for k in params if k.endswith("kernels/kernel")])
        self._packed = {}
        self._version_fn, self._packed_version = version, None
        dev = next(iter(params.values())).device
        self.device = dev

    def _weights(self, i):
        K = self.p["stem/cnnLayercnn_%d/kernels/kernel" % i]
        W = K.reshape(-1, K.shape[3])                       # [9*Cin, Cout], row-major view of the HWIO kernel
        if self.prec == "bf16":
            v = self._version_fn() if self._version_fn is not None else None
            if v != self._packed_version:
                self._packed.clear()
                self._packed_version = v
            if i not in self._packed:
                Wt = torch.empty((W.shape[1], W.shape[0]), dtype=torch.bfloat16, device=W.device)
                check(self.lib.mac_pack_weight_bf16(ptr(W), ptr(Wt), W.shape[0], W.shape[1], stream_ptr()), "pack")
                self._packed[i] = Wt
            return W, self._packed[i]
        return W, None

    def forward(self, images, keep=1.0, step=0, save_for_backward=False):
        """images: [B,H,W,C] fp32 NHWC (the reference transposes the NCHW h5 features first, model.py:~770).
        Returns the knowledge base [B, H*W, outDim] fp32."""
        x = images
        B, H, Wd, C = x.shape
        act = ACT["ELU"] if self.relu == "ELU" else ACT["RELU_STD"]
        if save_for_backward:
            if self.prec != "fp32":
                raise NotImplementedError("stem backward runs on the fp32 path (DESIGN.md section 9)")
            self._saved = {"xs": [], "ys": [], "keep": float(keep), "step": int(step), "act": act}
        for i in range(self.nlayers):
            if save_for_backward:
                self._saved["xs"].append(x)
            W, Wt = self._weights(i)
            b = self.p["stem/cnnLayercnn_%d/biases/bias" % i]
            C = x.shape[3]
            M, K, Nout = B * H * Wd, 9 * C, W.shape[1]
            bf16 = self.prec == "bf16"
            cols = torch.empty((M, K), dtype=torch.bfloat16 if bf16 else torch.float32, device=self.device)
            check(self.lib.mac_im2col3x3(ptr(x), ptr(cols), 1 if bf16 else 0, float(keep), self.seed, SITE_STEM + i, step,
                                         B, H, Wd, C, stream_ptr()), "mac_im2col3x3")
            y = torch.empty((M, Nout), dtype=torch.float32, device=self.device)
            if bf16:
                check(self.lib.mac_linear_tc_fwd(ptr(cols), ptr(Wt), ptr(b), act, ptr(y), 0, M, K, Nout, stream_ptr()),
                      "mac_linear_tc_fwd")
            else:
                arr_p = (ctypes.c_void_p * 1)(cols.data_ptr())
                arr_k = (ctypes.c_int * 1)(K)
                check(self.lib.mac_linear_fwd(arr_p, arr_k, arr_k, 1, ptr(W), ptr(b), 0.0, act, ptr(y), Nout, M, Nout, None,
                                              0, stream_ptr()), "mac_linear_fwd")
            if save_for_backward:
                self._saved["ys"].append(y)
            x = y.view(B, H, Wd, Nout)
        return x.view(B, H * Wd, x.shape[3])

    def backward(self, d_kb, grads, need_d_images=False):
        """Backward of `forward(save_for_backward=True)` (the reference differentiates the graph with TF autodiff,
        model.py:626-636).  d_kb [B, H*W, outDim]; accumulates (+=) into `grads` (dict TF-name -> tensor shaped like the
        parameter).  Per layer, last to first:  dZ = dY * act'(Y);  dKernel += cols^T @ dZ, dBias += colsum(dZ)
        (`mac_linear_bwd` on the re-generated patch matrix);  dcols = dZ @ Kernel^T;  dX = col2im(dcols) * dropout mask.
        The gradient w.r.t. the images (and with it layer 0's largest GEMM) is skipped unless asked for."""
        sv = getattr(self, "_saved", None)
        if sv is None:
            raise RuntimeError("forward(save_for_backward=True) must run first")
        B, H, Wd, _ = sv["xs"][0].shape
        M = B * H * Wd
        dy = d_kb.contiguous().view(M, -1)
        dx = None
        for i in reversed(range(self.nlayers)):
            x, y = sv["xs"][i], sv["ys"][i]
            C, Nout = x.shape[3], y.shape[1]
            K = 9 * C
            W, _ = self._weights(i)
            dz = torch.empty_like(y)
            check(self.lib.mac_activation_bwd(ptr(y), ptr(dy), sv["act"], ptr(dz), dz.numel(), stream_ptr()), "mac_activation_bwd")
            cols = torch.empty((M, K), dtype=torch.float32, device=self.device)
            check(self.lib.mac_im2col3x3(ptr(x), ptr(cols), 0, sv["keep"], self.seed, SITE_STEM + i, sv["step"], B, H, Wd, C,
                                         stream_ptr()), "mac_im2col3x3")
            need_dx = need_d_images or i > 0
            dcols = torch.empty((M, K), dtype=torch.float32, device=self.device) if need_dx else None
            Wt = W.t().contiguous() if need_dx else None
            one = lambda v, t=ctypes.c_int: (t * 1)(v)
            check(self.lib.mac_linear_bwd(one(cols.data_ptr(), ctypes.c_void_p), one(K), one(K), 1, ptr(Wt), ptr(dz), Nout,
                                          one(None if dcols is None else dcols.data_ptr(), ctypes.c_void_p), one(K), one(0),
                                          ptr(grads["stem/cnnLayercnn_%d/kernels/kernel" % i]),
                                          ptr(grads["stem/cnnLayercnn_%d/biases/bias" % i]), M, Nout, None, 0, stream_ptr()),
                  "mac_linear_bwd")
            if need_dx:
                dx = torch.empty_like(x)
                check(self.lib.mac_col2im3x3(ptr(dcols), ptr(dx), sv["keep"], self.seed, SITE_STEM + i, sv["step"], B, H, Wd,
                                             C, stream_ptr()), "mac_col2im3x3")
                dy = dx.view(M, C)
        return dx if need_d_images else None
