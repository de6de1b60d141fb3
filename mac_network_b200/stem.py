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
the split-bf16 scheme the cell calls "tc32", DESIGN.md section 9 item 6).

Other geometries (--stemKernelSize(s), --stemStrideSizes, --stemLinear): a layer is (k, s, act, dropout) with TF SAME
padding (`Ho = ceil(H / s)`, the odd padding row on the bottom / right); the linear stem is the layer (1, 1, NON, no
dropout) on the `[inDim, outDim]` weight viewed as `[1, 1, inDim, outDim]`.  Layers with k = 3, s = 1 run the 3x3 kernels
above; every other layer runs the general patch passes (`mac_im2col`, `mac_col2im`, `mac_conv_bwd_tc` / `_tc32`) with the
same GEMMs.  The e4m3 stem keeps only the 3x3 stride-1 geometry.

Location features (--locationAware, DESIGN.md "Location-aware stem"): layer 0 reads concat(x, g) with the constant grid
g [H, W, l] (`location_grid`), as conv(x, K_img) + conv(g, K_loc).  The image half is the layer-0 path above, unchanged; the
location half is the patch matrix Q [M, Kq] of g (`mac_loc_cols`, its own dropout site SITE_LOCATION) against W_loc, the
kernel's location rows padded with zero rows to Kq = k^2 l rounded up to 128."""
import collections

import numpy as np
import torch

from . import _lib, packs
from ._lib import act_code, check, ptr, segments, stream_ptr

SITE_STEM = 32            # Philox site base for the stem's input dropouts (site + layer index)
INGEST_NHWC_F32, INGEST_PATCH_BF16 = 0, 1       # enum MAC_INGEST_* (include/mac_b200.h)
INGEST_COLS_BF16, INGEST_COLS_SPLIT = 0, 1      # enum MAC_INGEST_COLS_*
COLS_F32, COLS_BF16, COLS_SPLIT = 0, 1, 2       # enum MAC_COLS_*
LINEAR_W, LINEAR_B = "stem/linearLayer/weights/weight", "stem/linearLayer/biases/bias"
SITE_LOCATION = 50        # Philox site of layer 0's location channels' dropout


def location_spec(location):
    """`location`: None, or (type, bias, dim) -- --locationType ("L" or "PE"), --locationBias, --locationDim -- or a bare
    type with the reference's defaults (bias 1.0, dim 32).  Returns None or the checked (type, bias, dim)."""
    if location is None:
        return None
    if isinstance(location, str):
        location = (location, 1.0, 32)
    kind, bias, dim = location
    if kind not in ("L", "PE"):
        raise ValueError("location type must be 'L' or 'PE', got %r" % (kind,))
    if not np.isfinite(float(bias)):
        raise ValueError("location bias must be finite, got %r" % (bias,))
    if int(dim) != dim or int(dim) < 1:
        raise ValueError("location dim must be a positive integer, got %r" % (dim,))
    return kind, float(bias), int(dim)


def location_channels(location):
    """l, the location channels layer 0 reads after the image's: 2 for L, 4 dim for PE (ops.py:448-488)."""
    loc = location_spec(location)
    return 0 if loc is None else (2 if loc[0] == "L" else 4 * loc[2])


def location_grid(location, H, W):
    """The location grid [H, W, l] in fp64 (ops.py:448-488, addLocation's CNCT mode): x = linspace(-bias, bias, W)[w], y =
    linspace(-bias, bias, H)[h] (TF's linspace of one point is [-bias]); L is [x, y]; PE is
    [sin x_i | cos x_i | sin y_i | cos y_i] with x_i = x / 10000^(i / dim), i = 0 .. dim - 1."""
    kind, bias, dim = location_spec(location)
    lin = lambda n: np.linspace(-bias, bias, n) if n > 1 else np.array([-bias])
    x = np.broadcast_to(lin(W)[None, :, None], (H, W, 1))
    y = np.broadcast_to(lin(H)[:, None, None], (H, W, 1))
    if kind == "L":
        return np.concatenate([x, y], axis=-1)
    f = np.power(10000.0, np.arange(dim) / float(dim))
    return np.concatenate([np.sin(x / f), np.cos(x / f), np.sin(y / f), np.cos(y / f)], axis=-1)


def location_width(l, k):
    """Kq: the location patch matrix's width, k^2 l rounded up to the 128-wide wgmma tile (mac_loc_cols_width)."""
    return -(-k * k * l // 128) * 128


def stem_specs(in_dim, out_dim, num_layers=2, ksize=3, stem_dim=None, ksizes=None, linear=False, location=None):
    """The stem's variables as the reference names and shapes them (model.py:165-204): `--stemLinear` one `ops.linear`
    (`stem/linearLayer/weights/weight` [inDim, outDim] and its bias), else `num_layers` HWIO kernels
    `stem/cnnLayercnn_i/kernels/kernel` [k_i, k_i, Cin, Cout] of kernel size `ksizes[i]` (--stemKernelSizes) or `ksize`
    (--stemKernelSize) for every layer.  `location` (--locationAware, `location_spec`) gives layer 0 Cin = inDim + l and
    creates no variable."""
    s = collections.OrderedDict()
    if linear:
        if location is not None:
            raise ValueError("the linear stem takes no location features (the reference adds them in the CNN stem only)")
        if ksizes is not None or stem_dim is not None:
            raise ValueError("the linear stem is one [inDim, outDim] layer: it takes no ksizes or stem_dim")
        s[LINEAR_W] = ((in_dim, out_dim), "xavier")
        s[LINEAR_B] = ((out_dim,), "zeros")
        return s
    stem_dim = out_dim if stem_dim is None else stem_dim
    ks = [ksize] * num_layers if ksizes is None else [int(k) for k in ksizes]
    if len(ks) != num_layers:
        raise ValueError("ksizes has %d entries for %d stem layers" % (len(ks), num_layers))
    dims = [in_dim + location_channels(location)] + [stem_dim] * (num_layers - 1) + [out_dim]
    for i in range(num_layers):
        s["stem/cnnLayercnn_%d/kernels/kernel" % i] = ((ks[i], ks[i], dims[i], dims[i + 1]), "xavier")
        s["stem/cnnLayercnn_%d/biases/bias" % i] = ((dims[i + 1],), "zeros")
    return s


def conv_out(n, s):
    """TF SAME output extent of a stride-`s` convolution over `n` pixels: ceil(n / s) whatever the kernel size."""
    return -(-int(n) // int(s))


def stem_grid(H, W, strides):
    """The knowledge-base grid (Ho, Wo) a stem with per-layer `strides` makes of an H x W feature map."""
    for s in strides:
        H, W = conv_out(H, s), conv_out(W, s)
    return H, W


def init_stem_params(specs, seed=0, dtype=np.float32, bias_scale=0.1):
    rng = np.random.RandomState(seed)
    out = collections.OrderedDict()
    for name, (shape, kind) in specs.items():
        if kind == "zeros":
            v = bias_scale * rng.standard_normal(shape)
        else:       # tf.contrib.layers.xavier_initializer on [kh,kw,cin,cout]: fan_in = kh*kw*cin, fan_out = kh*kw*cout
            rf = shape[0] * shape[1] if len(shape) == 4 else 1
            lim = np.sqrt(6.0 / (rf * shape[-2] + rf * shape[-1]))
            v = rng.uniform(-lim, lim, size=shape)
        out[name] = np.asarray(v, dtype=dtype)
    return out


class Stem(object):
    def __init__(self, params, relu="ELU", prec="fp32", seed=0, version=None, strides=None, linear=False, location=None):
        """`params`: dict TF-name -> CUDA fp32 tensor (HWIO kernels, biases; or with `linear=True` the `stem/linearLayer`
        weight [inDim, outDim] and bias).  Each layer's kernel size is read from its kernel's shape; `strides`
        (--stemStrideSizes) gives one stride per layer, default 1.  `version`: optional callable returning a counter
        that changes whenever the parameter values do (`MACParams.version`): the packed bf16 / e4m3 kernels are rebuilt when it moves
        (optimizer step, checkpoint restore, EMA swap -- ADVICE r1), whoever changed the values.  `location`
        (--locationAware, `location_spec`): layer 0's kernel holds inDim + l input channels, the last l of them the location
        grid's; not with the linear stem (ValueError) or prec="fp8" (NotImplementedError)."""
        self.location = location_spec(location)
        if self.location is not None and linear:
            raise ValueError("the linear stem takes no location features (the reference adds them in the CNN stem only)")
        if self.location is not None and prec == "fp8":
            raise NotImplementedError("the fp8 stem does not run location features; use prec='bf16'")
        self.nloc = location_channels(self.location)
        self._grids = {}
        self.lib = _lib.load()
        self.p = params
        self.relu, self.prec, self.seed = relu, prec, int(seed)
        self.linear = bool(linear)
        if self.linear:
            if set(params) != {LINEAR_W, LINEAR_B}:
                raise ValueError("a linear stem takes %s and %s, got %s" % (LINEAR_W, LINEAR_B, sorted(params)))
            self.nlayers, self.ksizes = 1, [1]
        else:
            self.nlayers = len([k for k in params if k.endswith("kernels/kernel")])
            self.ksizes = [int(params["stem/cnnLayercnn_%d/kernels/kernel" % i].shape[0]) for i in range(self.nlayers)]
        self.strides = [1] * self.nlayers if strides is None else [int(v) for v in strides]
        if len(self.strides) != self.nlayers or any(v < 1 for v in self.strides) or (self.linear and self.strides != [1]):
            raise ValueError("strides %s do not fit a %s stem of %d layer(s)" % (strides, "linear" if self.linear else "CNN",
                                                                                 self.nlayers))
        self._cache = packs.Cache(version)
        dev = next(iter(params.values())).device
        self.device = dev

    @property
    def in_dim(self):
        """The image channels the stem reads (layer 0's Cin)."""
        return int(self.p[self._names(0)[0]].shape[-2]) - self.nloc

    def grid(self, H, W):
        """The knowledge base's grid (Ho, Wo) for H x W features: the knowledge base has Ho * Wo rows."""
        return stem_grid(H, W, self.strides)

    def _names(self, i):
        if self.linear:
            return LINEAR_W, LINEAR_B
        return "stem/cnnLayercnn_%d/kernels/kernel" % i, "stem/cnnLayercnn_%d/biases/bias" % i

    def _bias(self, i):
        return self.p[self._names(i)[1]]

    def _k3s1(self, i):
        return self.ksizes[i] == 3 and self.strides[i] == 1

    def _act(self):
        return act_code("NON", self.relu) if self.linear else act_code("RELU", self.relu)

    def _keep(self, keep):
        return 1.0 if self.linear else float(keep)      # ops.linear runs without dropout in the stem (ops.py:298)

    def _cout(self, i):
        return int(self.p[self._names(i)[0]].shape[-1])

    def _weights(self, i):
        """(W, packed): the fp32 [k*k*Cin, Cout] view and, for bf16, the bf16 [Cout, k*k*Cin] pack; for bf16x3, the split pack
        [Cout, 3*k*k*Cin] = [hi | hi | lo]; for fp8, the e4m3 [Cout, 9*Cin] pack and its per-column scales as a pair."""
        K = self.p[self._names(i)[0]]
        W = K.reshape(-1, K.shape[-1])                      # [k*k*Cin, Cout], row-major view of the HWIO kernel
        build = {"bf16": packs.bf16, "bf16x3": packs.split3, "fp8": packs.fp8}.get(self.prec)
        return W, None if build is None else self._cache.pack(build, W, stream=stream_ptr())

    def location_grid(self, H, W):
        """The fp32 location grid [H, W, l] on the device, built once per (H, W) (a captured graph reads this tensor)."""
        if (H, W) not in self._grids:
            g = np.ascontiguousarray(location_grid(self.location, H, W), dtype=np.float32)
            self._grids[(H, W)] = torch.from_numpy(g).to(self.device)
        return self._grids[(H, W)]

    def _loc_weights(self):
        """(W_img [k^2 C, Cout], W_loc [Kq, Cout]): fp32 contiguous views of one [W_img; W_loc] gathered from layer 0's
        interleaved [k^2 (C + l), Cout] rows (W_loc's rows k^2 l..Kq-1 zero), rebuilt when the parameters move."""
        K = self.p[self._names(0)[0]]
        k, Cout, l = int(K.shape[0]), int(K.shape[-1]), self.nloc
        C = int(K.shape[2]) - l
        n_img = k * k * C

        def build():
            Kv = K.detach().reshape(k * k, C + l, Cout)
            cat = torch.zeros((n_img + location_width(l, k), Cout), dtype=torch.float32, device=K.device)
            cat[:n_img].view(k * k, C, Cout).copy_(Kv[:, :C])
            cat[n_img:n_img + k * k * l].view(k * k, l, Cout).copy_(Kv[:, C:])
            return cat
        cat = self._cache.get(("location", K.data_ptr()), build)
        return cat, cat[:n_img], cat[n_img:]

    def _loc_cols(self, B, H, Wd, form, keep, step):
        """Q [M, Kq] (or [M, 2 Kq] split) of layer 0's location channels on the H x W input grid, dropout fused."""
        k, s = self.ksizes[0], self.strides[0]
        M = B * conv_out(H, s) * conv_out(Wd, s)
        Kq = location_width(self.nloc, k)
        q = torch.empty((M, Kq * (2 if form == COLS_SPLIT else 1)),
                        dtype=torch.float32 if form == COLS_F32 else torch.bfloat16, device=self.device)
        check(self.lib.mac_loc_cols(ptr(self.location_grid(H, Wd)), ptr(q), form, float(keep), self.seed, SITE_LOCATION,
                                    int(step), B, H, Wd, self.nloc, k, s, stream_ptr()), "mac_loc_cols")
        return q

    def _loc_scatter(self, grads, dk_img, dw_loc):
        """Adds dK_img [k^2 C, Cout] and dW_loc[:k^2 l] into layer 0's interleaved kernel gradient [k, k, C + l, Cout]."""
        G = grads[self._names(0)[0]]
        k, l, Cout = int(G.shape[0]), self.nloc, int(G.shape[-1])
        Gv = G.view(k * k, -1, Cout)
        C = Gv.shape[1] - l
        Gv[:, :C] += dk_img.view(k * k, C, Cout)
        Gv[:, C:] += dw_loc[:k * k * l].view(k * k, l, Cout)

    def _backward_loc0_tc(self, x, y, dy, W_img, dx, grads):
        """Layer 0's tensor-core backward with location features (`mac_conv_bwd_loc_tc` / `_tc32`): the image half as
        `mac_conv_bwd_tc`, and dW_loc += Q^T dZ from the same dZ^T; both scattered into the interleaved kernel gradient."""
        sv = self._saved
        B, H, Wd, C = x.shape
        Nout, k, s, l = y.shape[1], self.ksizes[0], self.strides[0], self.nloc
        name = "mac_conv_bwd_loc_tc" if self.prec == "bf16" else "mac_conv_bwd_loc_tc32"
        nbytes = int(getattr(self.lib, name + "_workspace_bytes")(B, H, Wd, C, Nout, l, k, s, int(dx is not None)))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        dk = torch.zeros_like(W_img)
        dwl = torch.zeros((location_width(l, k), Nout), dtype=torch.float32, device=self.device)
        check(getattr(self.lib, name)(ptr(x), ptr(y), ptr(dy), ptr(W_img), sv["act"], sv["keep"], self.seed, SITE_STEM,
                                      sv["step"], ptr(self.location_grid(H, Wd)), l, SITE_LOCATION, ptr(dk), ptr(dwl),
                                      ptr(grads[self._names(0)[1]]), ptr(dx), ptr(ws), nbytes, B, H, Wd, C, Nout, k, s,
                                      stream_ptr()), name)
        self._loc_scatter(grads, dk, dwl)

    def _check_fp8(self, in_dim, keep):
        """The e4m3 stem is the inference forward only (no dropout) of the 3x3 stride-1 geometry with every channel count a
        multiple of 128 (whole 128-byte k-blocks and 128-column tiles of mac_linear_fp8_fwd).  Raises before any launch."""
        if self.linear or not all(self._k3s1(i) for i in range(self.nlayers)):
            raise NotImplementedError("the fp8 stem runs the 3x3 stride-1 geometry only, got %s"
                                      % ("the linear stem" if self.linear else "kernel sizes %s, strides %s"
                                         % (self.ksizes, self.strides)))
        if float(keep) != 1.0:
            raise NotImplementedError("the fp8 stem is inference only: keep must be 1.0, got %r" % (keep,))
        dims = [in_dim] + [self._cout(i) for i in range(self.nlayers)]
        if any(c % 128 for c in dims):
            raise NotImplementedError("the fp8 stem needs channel counts that are multiples of 128, got %s" % dims)

    def _forward_fp8(self, x, act):
        B, H, Wd, _ = x.shape
        M = B * H * Wd
        for i in range(self.nlayers):
            _, (W8, sw) = self._weights(i)
            b = self._bias(i)
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
        dims = [in_dim] + [self._cout(i) for i in range(self.nlayers)]
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

    def _patches(self, x, i, form, keep, step):
        """Layer i's patch matrix of x [B,H,W,C] (form COLS_F32, COLS_BF16 or COLS_SPLIT), dropout fused: the 3x3 stride-1
        passes for that geometry, `mac_im2col` for every other."""
        B, H, Wd, C = x.shape
        k, s = self.ksizes[i], self.strides[i]
        Ho, Wo = conv_out(H, s), conv_out(Wd, s)
        K = k * k * C
        cols = torch.empty((B * Ho * Wo, K * (2 if form == COLS_SPLIT else 1)),
                           dtype=torch.float32 if form == COLS_F32 else torch.bfloat16, device=self.device)
        if not self._k3s1(i):
            check(self.lib.mac_im2col(ptr(x), ptr(cols), form, float(keep), self.seed, SITE_STEM + i, int(step), B, H, Wd, C,
                                      k, s, stream_ptr()), "mac_im2col")
        elif form == COLS_SPLIT:
            check(self.lib.mac_im2col3x3_split(ptr(x), ptr(cols), float(keep), self.seed, SITE_STEM + i, int(step), B, H, Wd,
                                               C, stream_ptr()), "mac_im2col3x3_split")
        else:
            check(self.lib.mac_im2col3x3(ptr(x), ptr(cols), int(form == COLS_BF16), float(keep), self.seed, SITE_STEM + i,
                                         int(step), B, H, Wd, C, stream_ptr()), "mac_im2col3x3")
        return cols

    def forward(self, images, keep=1.0, step=0, save_for_backward=False, _cols0=None):
        """images: [B,H,W,C] fp32 NHWC (the reference transposes the NCHW h5 features first, model.py:~770).
        Returns the knowledge base [B, Ho*Wo, outDim] fp32 (`grid`).  `_cols0` (`forward_nchw`, bf16 and bf16x3 stems): layer
        0's patch matrix, already built with this call's keep and step; `images` is then read only by the backward, if at all."""
        x = images
        B, H, Wd, C = x.shape
        act = self._act()
        keep = self._keep(keep)
        if save_for_backward:
            self._check_trainable(C)
            self._saved = {"xs": [], "ys": [], "keep": keep, "step": int(step), "act": act}
        if self.prec == "fp8":
            self._check_fp8(C, keep)
            return self._forward_fp8(x, act)
        if self.prec == "bf16x3":
            self._check_tiles(C, "the bf16x3 stem")
        form = {"bf16": COLS_BF16, "bf16x3": COLS_SPLIT}.get(self.prec, COLS_F32)
        for i in range(self.nlayers):
            if save_for_backward:
                self._saved["xs"].append(x)
            loc0 = i == 0 and self.location is not None
            W, Wt = (self._loc_weights()[1], None) if loc0 else self._weights(i)
            b = self._bias(i)
            Hin, Win = H, Wd
            H, Wd = conv_out(H, self.strides[i]), conv_out(Wd, self.strides[i])
            M, K, Nout = B * H * Wd, W.shape[0], W.shape[1]
            y = torch.empty((M, Nout), dtype=torch.float32, device=self.device)
            cols = _cols0 if (i == 0 and _cols0 is not None) else self._patches(x, i, form, keep, step)
            if loc0:
                self._forward_loc0(cols, self._loc_cols(B, Hin, Win, form, keep, step), form, b, act, y)
            elif form == COLS_SPLIT:
                check(self.lib.mac_linear_tc32_fwd(ptr(cols), ptr(Wt), ptr(b), act, ptr(y), M, K, Nout, stream_ptr()),
                      "mac_linear_tc32_fwd")
            elif form == COLS_BF16:
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

    def _forward_loc0(self, cols, q, form, b, act, y):
        """Layer 0 with location features: y = act(P W_img + (Q W_loc + b)) -- one fp32 GEMM over the segments [P, Q], or on
        tensor cores Q W_loc + b into y, then the image GEMM adding y before its activation (mac_linear_tc(32)_fwd_acc)."""
        cat, W_img, W_loc = self._loc_weights()
        M, Nout = y.shape
        if form == COLS_F32:
            arr_p, arr_k, arr_ld = segments([cols, q])
            check(self.lib.mac_linear_fwd(arr_p, arr_k, arr_ld, 2, ptr(cat), ptr(b), 0.0, act, ptr(y), Nout, M, Nout, None, 0,
                                          stream_ptr()), "mac_linear_fwd")
            return
        K, Kq = W_img.shape[0], W_loc.shape[0]
        if form == COLS_SPLIT:
            check(self.lib.mac_linear_tc32_fwd(ptr(q), ptr(self._cache.pack(packs.split3, W_loc, stream=stream_ptr())), ptr(b),
                                               _lib.ACT["NON"], ptr(y), M, Kq, Nout, stream_ptr()), "mac_linear_tc32_fwd")
            check(self.lib.mac_linear_tc32_fwd_acc(ptr(cols), ptr(self._cache.pack(packs.split3, W_img, stream=stream_ptr())),
                                                   act, ptr(y), M, K, Nout, stream_ptr()), "mac_linear_tc32_fwd_acc")
        else:
            check(self.lib.mac_linear_tc_fwd(ptr(q), ptr(self._cache.pack(packs.bf16, W_loc, stream=stream_ptr())), ptr(b),
                                             _lib.ACT["NON"], ptr(y), 0, M, Kq, Nout, stream_ptr()), "mac_linear_tc_fwd")
            check(self.lib.mac_linear_tc_fwd_acc(ptr(cols), ptr(self._cache.pack(packs.bf16, W_img, stream=stream_ptr())), act,
                                                 ptr(y), M, K, Nout, stream_ptr()), "mac_linear_tc_fwd_acc")

    def forward_nchw(self, images, keep=1.0, step=0, save_for_backward=False):
        """`forward` from the features in the layout they are stored in: images [B,C,H,W], contiguous, fp32, fp16 or -- `prec="bf16"`
        inference only, whose layer 0 then reads nothing but bf16(x) -- bf16.  The ingest kernels (csrc/ingest.cuh) replace
        the NHWC permute.  Inference (keep = 1, no save_for_backward): `mac_ingest_nchw` writes the bf16 stem's layer-0 patch
        matrix directly, for the other precisions the fp32 NHWC tensor their own patch passes read.  A layer 0 of any other
        geometry than 3x3 stride 1 reads the fp32 NHWC tensor in every precision.  Training (a dropout or
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
        keep = self._keep(keep)
        train = save_for_backward or keep != 1.0
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
        if not self._k3s1(0):         # the fused ingests build 3x3 patches: write the NHWC tensor, then the general pass
            x = torch.empty((B, H, Wd, C), dtype=torch.float32, device=self.device)
            self._ingest(images, x_bf16, x, INGEST_NHWC_F32)
            return self.forward(x, keep, step, save_for_backward)
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
        model.py:626-636).  d_kb [B, Ho*Wo, outDim]; accumulates (+=) into `grads` (dict TF-name -> tensor shaped like the
        parameter).  Per layer, last to first:  dZ = dY * act'(Y);  dKernel += cols^T @ dZ, dBias += colsum(dZ)
        (`mac_linear_bwd` on the re-generated patch matrix);  dcols = dZ @ Kernel^T;  dX = col2im(dcols) * dropout mask.
        The gradient w.r.t. the images (and with it layer 0's largest GEMM) is skipped unless asked for.
        With prec="bf16" each layer is one `mac_conv3x3_bwd_tc` call (`mac_conv_bwd_tc` for other geometries): the same
        steps with both GEMMs on tensor cores; with prec="bf16x3" one `mac_conv3x3_bwd_tc32` (`mac_conv_bwd_tc32`) call: the
        same again on split-bf16 operands."""
        sv = getattr(self, "_saved", None)
        if sv is None:
            raise RuntimeError("forward(save_for_backward=True) must run first")
        dy = d_kb.contiguous().view(-1, d_kb.shape[-1])
        dx = None
        for i in reversed(range(self.nlayers)):
            x, y = sv["xs"][i], sv["ys"][i]
            B, H, Wd, C = x.shape
            Nout = y.shape[1]
            k, s = self.ksizes[i], self.strides[i]
            wname, bname = self._names(i)
            loc0 = i == 0 and self.location is not None
            W = self._loc_weights()[1] if loc0 else self._weights(i)[0]
            need_dx = need_d_images or i > 0
            if self.prec in ("bf16", "bf16x3") and loc0:
                dx = torch.empty_like(x) if need_dx else None
                self._backward_loc0_tc(x, y, dy, W, dx, grads)
                continue
            if self.prec in ("bf16", "bf16x3"):
                dx = torch.empty_like(x) if need_dx else None
                if self._k3s1(i):
                    name = "mac_conv3x3_bwd_tc" if self.prec == "bf16" else "mac_conv3x3_bwd_tc32"
                    geom = ()
                else:
                    name = "mac_conv_bwd_tc" if self.prec == "bf16" else "mac_conv_bwd_tc32"
                    geom = (k, s)
                nbytes = int(getattr(self.lib, name + "_workspace_bytes")(B, H, Wd, C, Nout, *geom, int(dx is not None)))
                ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
                check(getattr(self.lib, name)(ptr(x), ptr(y), ptr(dy), ptr(W), sv["act"], sv["keep"], self.seed,
                                              SITE_STEM + i, sv["step"], ptr(grads[wname].view(W.shape)), ptr(grads[bname]),
                                              ptr(dx), ptr(ws), nbytes, B, H, Wd, C, Nout, *geom, stream_ptr()), name)
                if dx is not None:
                    dy = dx.view(-1, C)
                continue
            dz = torch.empty_like(y)
            check(self.lib.mac_activation_bwd(ptr(y), ptr(dy), sv["act"], ptr(dz), dz.numel(), stream_ptr()), "mac_activation_bwd")
            cols = self._patches(x, i, COLS_F32, sv["keep"], sv["step"])
            dcols = torch.empty_like(cols) if need_dx else None
            if loc0:                    # segments [P, Q] against [W_img; W_loc]; only P takes a data gradient
                cat = self._loc_weights()[0]
                q = self._loc_cols(B, H, Wd, COLS_F32, sv["keep"], sv["step"])
                dcat = torch.zeros_like(cat)
                _lib.linear_bwd([cols, q], cat.t().contiguous() if need_dx else None, dz, [dcols, None], [0, 0], dcat,
                                grads[bname], None, 0, stream_ptr())
                self._loc_scatter(grads, dcat[:W.shape[0]], dcat[W.shape[0]:])
            else:
                Wt = W.t().contiguous() if need_dx else None
                _lib.linear_bwd([cols], Wt, dz, [dcols], [0], grads[wname].view(W.shape), grads[bname], None, 0, stream_ptr())
            if need_dx:
                dx = torch.empty_like(x)
                if self._k3s1(i):
                    check(self.lib.mac_col2im3x3(ptr(dcols), ptr(dx), sv["keep"], self.seed, SITE_STEM + i, sv["step"], B, H,
                                                 Wd, C, stream_ptr()), "mac_col2im3x3")
                else:
                    check(self.lib.mac_col2im(ptr(dcols), ptr(dx), sv["keep"], self.seed, SITE_STEM + i, sv["step"], B, H, Wd,
                                              C, k, s, stream_ptr()), "mac_col2im")
                dy = dx.view(-1, C)
        return dx if need_d_images else None
