"""Image stem -- the producer of the knowledge base (SURVEY.md section 8(f), "next" row 1):
`MACnet.stem` (`model.py:165-204`) = `ops.CNNLayer` (`ops.py:423-438`) of `stemNumLayers` x `ops.cnn` (`ops.py:380-405`):
dropout on the layer input, 3x3 stride-1 SAME convolution (HWIO kernel) + bias, ELU after every layer; then the
`[B,H,W,d] -> [B, H*W, d]` reshape.  177.6 GFLOP per B=64 batch (56 % of the twelve cell steps).

GPU formulation: convolution as GEMM.  `mac_im2col3x3` builds the `[B*H*W, 9*C]` patch matrix (tap-major, channel fastest
-- exactly the row-major reshape of the HWIO kernel to `[9*C, Cout]`) with the input dropout fused (the Philox mask is
indexed by the SOURCE element, so all nine copies of a pixel share its mask), in bf16 for the wgmma GEMM
(`mac_linear_tc_fwd`, ELU epilogue) or fp32 for the parity GEMM (`mac_linear_fwd`).  `prec="fp8"` is an inference-only
forward in e4m3: `mac_im2col3x3_fp8` (per-row scales, no dropout) and `mac_linear_fp8_fwd` (csrc/tc_gemm_fp8.cuh).
`prec="bf16x3"` is the parity arithmetic on tensor cores, for inference and training: every fp32 operand as hi + lo bf16
halves and three bf16 products per fp32 product (`mac_im2col3x3_split`, `mac_linear_tc32_fwd`, `mac_conv3x3_bwd_tc32`;
the split-bf16 scheme the cell calls "tc32", DESIGN.md section 9 item 6)."""
import collections

import numpy as np
import torch

from . import _lib, packs
from ._lib import act_code, check, ptr, segments, stream_ptr

SITE_STEM = 32            # Philox site base for the stem's input dropouts (site + layer index)
INGEST_NHWC_F32, INGEST_PATCH_BF16 = 0, 1       # enum MAC_INGEST_* (include/mac_b200.h)
INGEST_COLS_BF16, INGEST_COLS_SPLIT = 0, 1      # enum MAC_INGEST_COLS_*


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
        that changes whenever the parameter values do (`MACParams.version`): the packed bf16 / e4m3 kernels are rebuilt when it moves
        (optimizer step, checkpoint restore, EMA swap -- ADVICE r1), whoever changed the values."""
        self.lib = _lib.load()
        self.p = params
        self.relu, self.prec, self.seed = relu, prec, int(seed)
        self.nlayers = len([k for k in params if k.endswith("kernels/kernel")])
        self._cache = packs.Cache(version)
        dev = next(iter(params.values())).device
        self.device = dev

    def _weights(self, i):
        """(W, packed): the fp32 [9*Cin, Cout] view and, for bf16, the bf16 [Cout, 9*Cin] pack; for bf16x3, the split pack
        [Cout, 3*9*Cin] = [hi | hi | lo]; for fp8, the e4m3 [Cout, 9*Cin] pack and its per-column scales as a pair."""
        K = self.p["stem/cnnLayercnn_%d/kernels/kernel" % i]
        W = K.reshape(-1, K.shape[3])                       # [9*Cin, Cout], row-major view of the HWIO kernel
        build = {"bf16": packs.bf16, "bf16x3": packs.split3, "fp8": packs.fp8}.get(self.prec)
        return W, None if build is None else self._cache.pack(build, W, stream=stream_ptr())

    def _check_fp8(self, in_dim, keep):
        """The e4m3 stem is the inference forward only (no dropout) with every channel count a multiple of 128 (whole
        128-byte k-blocks and 128-column tiles of mac_linear_fp8_fwd).  Raises before any launch."""
        if float(keep) != 1.0:
            raise NotImplementedError("the fp8 stem is inference only: keep must be 1.0, got %r" % (keep,))
        dims = [in_dim] + [int(self.p["stem/cnnLayercnn_%d/kernels/kernel" % i].shape[3]) for i in range(self.nlayers)]
        if any(c % 128 for c in dims):
            raise NotImplementedError("the fp8 stem needs channel counts that are multiples of 128, got %s" % dims)

    def _forward_fp8(self, x, act):
        B, H, Wd, _ = x.shape
        M = B * H * Wd
        for i in range(self.nlayers):
            _, (W8, sw) = self._weights(i)
            b = self.p["stem/cnnLayercnn_%d/biases/bias" % i]
            C, Nout = x.shape[3], W8.shape[0]
            cols = torch.empty((M, 9 * C), dtype=torch.uint8, device=self.device)
            sa = torch.empty(M, dtype=torch.float32, device=self.device)
            nbytes = int(self.lib.mac_im2col3x3_fp8_workspace_bytes(B, H, Wd, C))
            ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            check(self.lib.mac_im2col3x3_fp8(ptr(x), ptr(cols), ptr(sa), ptr(ws), nbytes, B, H, Wd, C, stream_ptr()),
                  "mac_im2col3x3_fp8")
            y = torch.empty((M, Nout), dtype=torch.float32, device=self.device)
            check(self.lib.mac_linear_fp8_fwd(ptr(cols), ptr(sa), ptr(W8), ptr(sw), ptr(b), act, ptr(y), M, 9 * C, Nout,
                                              stream_ptr()), "mac_linear_fp8_fwd")
            x = y.view(B, H, Wd, Nout)
        return x.view(B, H * Wd, x.shape[3])

    def _check_tiles(self, in_dim, what):
        dims = [in_dim] + [int(self.p["stem/cnnLayercnn_%d/kernels/kernel" % i].shape[3]) for i in range(self.nlayers)]
        if any(c % 128 for c in dims):
            raise NotImplementedError("%s needs channel counts that are multiples of 128 (the wgmma tiles of "
                                      "mac_conv3x3_bwd_tc), got %s; use prec='fp32' (DESIGN.md section 9)" % (what, dims))

    def _check_trainable(self, in_dim):
        """Training (forward with save_for_backward + backward) runs in fp32, or on tensor cores in bf16
        (`mac_conv3x3_bwd_tc`, DESIGN.md section 9 item 2) or split bf16 ("bf16x3", `mac_conv3x3_bwd_tc32`, item 6), whose
        GEMM tiles need every layer's input and output channel counts to be multiples of 128.  Raises before any launch."""
        if self.prec == "fp32":
            return
        if self.prec not in ("bf16", "bf16x3"):
            raise NotImplementedError("stem training runs in fp32, bf16 or bf16x3, not %r (DESIGN.md section 9)" % self.prec)
        self._check_tiles(in_dim, "%s stem training" % self.prec)

    def forward(self, images, keep=1.0, step=0, save_for_backward=False, _cols0=None):
        """images: [B,H,W,C] fp32 NHWC (the reference transposes the NCHW h5 features first, model.py:~770).
        Returns the knowledge base [B, H*W, outDim] fp32.  `_cols0` (`forward_nchw`, bf16 and bf16x3 stems): layer 0's patch
        matrix, already built with this call's keep and step; `images` is then read only by the backward, if at all."""
        x = images
        B, H, Wd, C = x.shape
        act = act_code("RELU", self.relu)
        if save_for_backward:
            self._check_trainable(C)
            self._saved = {"xs": [], "ys": [], "keep": float(keep), "step": int(step), "act": act}
        if self.prec == "fp8":
            self._check_fp8(C, keep)
            return self._forward_fp8(x, act)
        if self.prec == "bf16x3":
            self._check_tiles(C, "the bf16x3 stem")
        for i in range(self.nlayers):
            if save_for_backward:
                self._saved["xs"].append(x)
            W, Wt = self._weights(i)
            b = self.p["stem/cnnLayercnn_%d/biases/bias" % i]
            C = x.shape[3]
            M, K, Nout = B * H * Wd, 9 * C, W.shape[1]
            bf16 = self.prec == "bf16"
            y = torch.empty((M, Nout), dtype=torch.float32, device=self.device)
            if self.prec == "bf16x3":
                if i == 0 and _cols0 is not None:
                    cols = _cols0
                else:
                    cols = torch.empty((M, 2 * K), dtype=torch.bfloat16, device=self.device)          # [hi | lo]
                    check(self.lib.mac_im2col3x3_split(ptr(x), ptr(cols), float(keep), self.seed, SITE_STEM + i, step, B, H,
                                                       Wd, C, stream_ptr()), "mac_im2col3x3_split")
                check(self.lib.mac_linear_tc32_fwd(ptr(cols), ptr(Wt), ptr(b), act, ptr(y), M, K, Nout, stream_ptr()),
                      "mac_linear_tc32_fwd")
                if save_for_backward:
                    self._saved["ys"].append(y)
                x = y.view(B, H, Wd, Nout)
                continue
            if i == 0 and _cols0 is not None:
                cols = _cols0
            else:
                cols = torch.empty((M, K), dtype=torch.bfloat16 if bf16 else torch.float32, device=self.device)
                check(self.lib.mac_im2col3x3(ptr(x), ptr(cols), 1 if bf16 else 0, float(keep), self.seed, SITE_STEM + i, step,
                                             B, H, Wd, C, stream_ptr()), "mac_im2col3x3")
            if bf16:
                check(self.lib.mac_linear_tc_fwd(ptr(cols), ptr(Wt), ptr(b), act, ptr(y), 0, M, K, Nout, stream_ptr()),
                      "mac_linear_tc_fwd")
            else:
                arr_p, arr_k, arr_ld = segments([cols])
                check(self.lib.mac_linear_fwd(arr_p, arr_k, arr_ld, 1, ptr(W), ptr(b), 0.0, act, ptr(y), Nout, M, Nout, None,
                                              0, stream_ptr()), "mac_linear_fwd")
            if save_for_backward:
                self._saved["ys"].append(y)
            x = y.view(B, H, Wd, Nout)
        return x.view(B, H * Wd, x.shape[3])

    def forward_nchw(self, images, keep=1.0, step=0, save_for_backward=False):
        """`forward` from the features in the layout they are stored in: images [B,C,H,W], contiguous, fp32, fp16 or -- `prec="bf16"`
        inference only, whose layer 0 then reads nothing but bf16(x) -- bf16.  The ingest kernels (csrc/ingest.cuh) replace
        the NHWC permute.  Inference (keep = 1, no save_for_backward): `mac_ingest_nchw` writes the bf16 stem's layer-0 patch
        matrix directly, for the other precisions the fp32 NHWC tensor their own patch passes read.  Training (a dropout or
        save_for_backward): the bf16 and bf16x3 stems run `mac_ingest_nchw_train`, which writes the undropped fp32 NHWC tensor
        (saved as layer 0's input) and layer 0's dropped-out bf16 or split patch matrix from one read; the fp32 stem runs the
        NHWC ingest and its usual pass.  Returns -- and saves, and differentiates -- what
        `forward(images.permute(0, 2, 3, 1).contiguous(), keep, step, save_for_backward)` does, bit for bit.  fp16 images
        (every precision, inference and training) run the `_f16` entry points, which widen on the device: the result, the
        saved tensors and the gradients are those of `forward_nchw(images.float(), ...)` bit for bit.  C must be a multiple
        of 64.  Raises before any launch."""
        if images.dim() != 4 or not images.is_contiguous():
            raise ValueError("images must be a contiguous [B, C, H, W] tensor")
        if images.dtype not in (torch.float32, torch.bfloat16, torch.float16):
            raise ValueError("images must be float32, float16 or bfloat16, got %s" % images.dtype)
        x_bf16 = int(images.dtype == torch.bfloat16)
        f16 = images.dtype == torch.float16
        train = save_for_backward or float(keep) != 1.0
        if x_bf16 and (self.prec != "bf16" or train):
            raise ValueError("bf16 images are for the bf16 stem's inference only: prec=%r%s reads the fp32 features"
                             % (self.prec, " in training" if train else ""))
        B, C, H, Wd = images.shape
        if C % 64:
            raise NotImplementedError("forward_nchw needs a channel count that is a multiple of 64, got %d" % C)
        if save_for_backward:
            self._check_trainable(C)
        if self.prec == "fp8":
            self._check_fp8(C, keep)
        if self.prec == "bf16x3":
            self._check_tiles(C, "the bf16x3 stem")
        if train and self.prec in ("bf16", "bf16x3"):
            split = self.prec == "bf16x3"
            x = torch.empty((B, H, Wd, C), dtype=torch.float32, device=self.device)
            cols = torch.empty((B * H * Wd, 9 * C * (2 if split else 1)), dtype=torch.bfloat16, device=self.device)
            name = "mac_ingest_nchw_train_f16" if f16 else "mac_ingest_nchw_train"
            check(getattr(self.lib, name)(ptr(images), ptr(x), ptr(cols), INGEST_COLS_SPLIT if split else INGEST_COLS_BF16,
                                          float(keep), self.seed, SITE_STEM, int(step), B, C, H, Wd, stream_ptr()), name)
            return self.forward(x, keep, step, save_for_backward, _cols0=cols)
        if self.prec != "bf16":
            if self.prec == "fp8":
                self._check_fp8(C, 1.0)
            x = torch.empty((B, H, Wd, C), dtype=torch.float32, device=self.device)
            self._ingest(images, x_bf16, x, INGEST_NHWC_F32)
            return self.forward(x, keep, step, save_for_backward)
        cols = torch.empty((B * H * Wd, 9 * C), dtype=torch.bfloat16, device=self.device)
        self._ingest(images, x_bf16, cols, INGEST_PATCH_BF16)
        return self.forward(images.permute(0, 2, 3, 1), _cols0=cols)     # a view: layer 0 reads `cols`, not the image

    def _ingest(self, images, x_bf16, out, mode):
        """`mac_ingest_nchw` of fp32 or bf16 images, `mac_ingest_nchw_f16` of fp16 ones."""
        B, C, H, Wd = images.shape
        if images.dtype == torch.float16:
            check(self.lib.mac_ingest_nchw_f16(ptr(images), ptr(out), mode, B, C, H, Wd, stream_ptr()), "mac_ingest_nchw_f16")
        else:
            check(self.lib.mac_ingest_nchw(ptr(images), x_bf16, ptr(out), mode, B, C, H, Wd, stream_ptr()), "mac_ingest_nchw")

    def backward(self, d_kb, grads, need_d_images=False):
        """Backward of `forward(save_for_backward=True)` (the reference differentiates the graph with TF autodiff,
        model.py:626-636).  d_kb [B, H*W, outDim]; accumulates (+=) into `grads` (dict TF-name -> tensor shaped like the
        parameter).  Per layer, last to first:  dZ = dY * act'(Y);  dKernel += cols^T @ dZ, dBias += colsum(dZ)
        (`mac_linear_bwd` on the re-generated patch matrix);  dcols = dZ @ Kernel^T;  dX = col2im(dcols) * dropout mask.
        The gradient w.r.t. the images (and with it layer 0's largest GEMM) is skipped unless asked for.
        With prec="bf16" each layer is one `mac_conv3x3_bwd_tc` call: the same steps with both GEMMs on tensor cores; with
        prec="bf16x3" one `mac_conv3x3_bwd_tc32` call: the same again on split-bf16 operands."""
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
            if self.prec in ("bf16", "bf16x3"):
                name = "mac_conv3x3_bwd_tc" if self.prec == "bf16" else "mac_conv3x3_bwd_tc32"
                dx = torch.empty_like(x) if (need_d_images or i > 0) else None
                nbytes = int(getattr(self.lib, name + "_workspace_bytes")(B, H, Wd, C, Nout, int(dx is not None)))
                ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
                check(getattr(self.lib, name)(ptr(x), ptr(y), ptr(dy), ptr(W), sv["act"], sv["keep"], self.seed,
                                              SITE_STEM + i, sv["step"], ptr(grads["stem/cnnLayercnn_%d/kernels/kernel" % i]),
                                              ptr(grads["stem/cnnLayercnn_%d/biases/bias" % i]), ptr(dx), ptr(ws), nbytes,
                                              B, H, Wd, C, Nout, stream_ptr()), name)
                if dx is not None:
                    dy = dx.view(M, C)
                continue
            dz = torch.empty_like(y)
            check(self.lib.mac_activation_bwd(ptr(y), ptr(dy), sv["act"], ptr(dz), dz.numel(), stream_ptr()), "mac_activation_bwd")
            cols = torch.empty((M, K), dtype=torch.float32, device=self.device)
            check(self.lib.mac_im2col3x3(ptr(x), ptr(cols), 0, sv["keep"], self.seed, SITE_STEM + i, sv["step"], B, H, Wd, C,
                                         stream_ptr()), "mac_im2col3x3")
            need_dx = need_d_images or i > 0
            dcols = torch.empty((M, K), dtype=torch.float32, device=self.device) if need_dx else None
            Wt = W.t().contiguous() if need_dx else None
            _lib.linear_bwd([cols], Wt, dz, [dcols], [0], grads["stem/cnnLayercnn_%d/kernels/kernel" % i],
                            grads["stem/cnnLayercnn_%d/biases/bias" % i], None, 0, stream_ptr())
            if need_dx:
                dx = torch.empty_like(x)
                check(self.lib.mac_col2im3x3(ptr(dcols), ptr(dx), sv["keep"], self.seed, SITE_STEM + i, sv["step"], B, H, Wd,
                                             C, stream_ptr()), "mac_col2im3x3")
                dy = dx.view(M, C)
        return dx if need_d_images else None
