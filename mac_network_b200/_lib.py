"""ctypes binding of libmac_b200.so (the C ABI declared in include/mac_b200.h).

The product path has no CPU or PyTorch fallback: if the shared library is missing, or a call
returns a non-zero status, this module raises.  PyTorch is used only for device memory and streams;
every pointer handed to the library is `tensor.data_ptr()`.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libmac_b200.so")

ACT = {"NON": 0, "TANH": 1, "SIGMOID": 2, "ELU": 3, "RELU_STD": 4}
PREC = {"fp32": 0, "bf16": 1, "tc32": 2, "fp8": 3}
SITE_MEM_VAR, SITE_READ_KB, SITE_READ_MEM, SITE_READ_INTER, SITE_WRITE_INFO, SITE_MEM_PLAIN = range(6)

c_fp = ctypes.c_void_p
c_int = ctypes.c_int
c_ll = ctypes.c_longlong
c_f = ctypes.c_float
c_sz = ctypes.c_size_t
c_u64 = ctypes.c_uint64


class ReadWeights(ctypes.Structure):
    """struct mac_read_weights (include/mac_b200.h)."""
    _fields_ = [("Wx", c_fp), ("bx", c_fp), ("Wy", c_fp), ("by", c_fp), ("Wm", c_fp), ("bm", c_fp),
                ("Wm2", c_fp), ("bm2", c_fp), ("wr", c_fp), ("br", c_f),
                ("Wx_bf16", c_fp), ("Wm_bf16", c_fp), ("Wm2_bf16", c_fp),
                ("Wx_s3", c_fp), ("Wma_s3", c_fp), ("Wmb_s3", c_fp), ("Wm2_s3", c_fp),
                ("Wm_fp8", c_fp), ("Wm_fp8_scale", c_fp), ("Wm2_fp8", c_fp), ("Wm2_fp8_scale", c_fp),
                ("Wm_s3", c_fp)]


# name -> (restype, argtypes); every symbol include/mac_b200.h declares
PROTOTYPES = {
    "mac_b200_abi_version": (c_int, []),
    "mac_b200_strerror": (ctypes.c_char_p, [c_int]),
    "mac_b200_device_ok": (c_int, []),
    "mac_b200_launch_count": (c_ll, []),
    "mac_linear_fwd": (c_int, [ctypes.POINTER(c_fp), ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_int, c_fp, c_fp,
                               c_f, c_int, c_fp, c_int, c_int, c_int, c_fp, c_sz, c_fp]),
    "mac_linear_workspace_bytes": (c_sz, [c_int, c_int, c_int]),
    "mac_control_attend_fwd": (c_int, [c_fp, c_ll, c_ll, c_fp, c_ll, c_ll, c_fp, c_ll, c_ll, c_fp, c_fp, c_f, c_fp,
                                       c_fp, c_int, c_int, c_int, c_int, c_fp]),
    "mac_read_fwd": (c_int, [c_fp, c_fp, c_fp, c_fp, ctypes.POINTER(ReadWeights), c_f, c_u64, c_int, c_int, c_fp,
                             c_fp, c_fp, c_fp, c_sz, c_int, c_int, c_int, c_fp]),
    "mac_read_workspace_bytes": (c_sz, [c_int, c_int, c_int, c_int]),
    "mac_read_invariant_bytes": (c_sz, [c_int, c_int, c_int, c_int]),
    "mac_read_invariant": (c_int, [c_fp, c_fp, ctypes.POINTER(ReadWeights), c_int, c_fp, c_sz, c_int, c_int, c_int,
                                   c_fp]),
    "mac_read_invariant_cast": (c_int, [c_fp, c_fp, ctypes.POINTER(ReadWeights), c_int, c_fp, c_sz, c_int, c_int,
                                        c_int, c_fp]),
    "mac_read_fwd_inv": (c_int, [c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, ctypes.POINTER(ReadWeights), c_int, c_fp, c_fp,
                                 c_fp, c_sz, c_int, c_int, c_int, c_fp]),
    "mac_read_step_fused": (c_int, [c_fp, c_fp, c_fp, c_fp, ctypes.POINTER(ReadWeights), c_fp, c_fp, c_int, c_int, c_int,
                                    c_fp]),
    "mac_read_step_fused_supported": (c_int, [c_int, c_int, c_int]),
    "mac_write_fwd_next_y": (c_int, [c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_sz, c_int, c_int, c_fp]),
    "mac_kb_attend_fwd": (c_int, [c_fp, c_int, c_f, c_fp, c_int, c_fp, c_fp, c_int, c_int, c_int, c_fp]),
    "mac_write_fwd": (c_int, [c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_f, c_fp, c_fp, c_fp, c_sz, c_int,
                              c_int, c_fp]),
    "mac_write_workspace_bytes": (c_sz, [c_int, c_int]),
    "mac_bcast_mul": (c_int, [c_fp, c_fp, c_f, c_fp, c_int, c_int, c_int, c_fp]),
    "mac_activation": (c_int, [c_fp, c_int, c_fp, c_ll, c_fp]),
    "mac_dropout_fwd": (c_int, [c_fp, c_f, c_u64, c_int, c_int, c_fp, c_ll, c_fp]),
    "mac_dropout_uniform": (c_int, [c_u64, c_int, c_int, c_fp, c_ll, c_fp]),
    "mac_cast_bf16": (c_int, [c_fp, c_fp, c_ll, c_fp]),
    "mac_host_cast_bf16": (c_int, [c_fp, c_fp, c_ll, c_int]),
    "mac_host_cast_bf16_begin": (c_int, [c_fp, c_fp, c_ll, c_int]),
    "mac_host_cast_bf16_end": (c_int, []),
    "mac_host_crc32c": (ctypes.c_uint32, [c_fp, c_ll, ctypes.c_uint32]),
    "mac_linear_bwd": (c_int, [ctypes.POINTER(c_fp), ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_int, c_fp, c_fp, c_int,
                               ctypes.POINTER(c_fp), ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_fp, c_fp, c_int, c_int,
                               c_fp, c_sz, c_fp]),
    "mac_control_attend_bwd": (c_int, [c_fp, c_ll, c_ll, c_fp, c_ll, c_ll, c_fp, c_ll, c_ll, c_fp, c_fp, c_fp, c_ll, c_ll,
                                       c_fp, c_fp, c_fp, c_ll, c_ll, c_int, c_fp, c_fp, c_int, c_int, c_int, c_int, c_fp]),
    "mac_kb_attend_bwd": (c_int, [c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_int, c_int, c_int, c_fp]),
    "mac_read_bwd": (c_int, [c_fp, c_fp, c_fp, ctypes.POINTER(ReadWeights), c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_f,
                             c_u64, c_int] + [c_fp] * 13 + [c_fp, c_sz, c_int, c_int, c_int, c_fp]),
    "mac_read_bwd_workspace_bytes": (c_sz, [c_int, c_int, c_int]),
    "mac_read_bwd_tc": (c_int, [c_fp, c_fp, c_fp, ctypes.POINTER(ReadWeights), c_fp, c_fp, c_fp, c_fp, c_f, c_u64, c_int]
                        + [c_fp] * 13 + [c_fp, c_sz, c_int, c_int, c_int, c_fp]),
    "mac_read_bwd_tc_workspace_bytes": (c_sz, [c_int, c_int, c_int]),
    "mac_read_bwd_tc32": (c_int, [c_fp, c_fp, c_fp, ctypes.POINTER(ReadWeights), c_fp, c_fp, c_fp, c_fp, c_f, c_u64, c_int]
                          + [c_fp] * 13 + [c_fp, c_sz, c_int, c_int, c_int, c_fp]),
    "mac_read_bwd_tc32_workspace_bytes": (c_sz, [c_int, c_int, c_int]),
    "mac_gate_bwd": (c_int, [c_fp] * 7 + [c_ll, c_fp]),
    "mac_activation_bwd": (c_int, [c_fp, c_fp, c_int, c_fp, c_ll, c_fp]),
    "mac_widen_bf16": (c_int, [ctypes.POINTER(c_fp), ctypes.POINTER(c_fp), c_int, c_ll, c_fp]),
    "mac_batchnorm_fwd": (c_int, [c_fp, c_fp, c_fp, c_fp, c_fp, c_f, c_f, c_int, c_fp, c_fp, c_fp, c_int, c_int, c_fp]),
    "mac_batchnorm_bwd": (c_int, [c_fp, c_fp, c_fp, c_fp, c_fp, c_int, c_fp, c_fp, c_fp, c_int, c_int, c_fp]),
    "mac_bcast_op_bwd": (c_int, [c_fp, c_fp, c_fp, c_fp, c_int, c_f, c_fp, c_fp, c_fp, c_int, c_int, c_int, c_fp]),
    "mac_rowdot_bwd": (c_int, [ctypes.POINTER(c_fp), ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_int, c_fp, c_fp,
                               ctypes.POINTER(c_fp), ctypes.POINTER(c_int), c_fp, c_fp, c_fp, ctypes.c_size_t, c_ll, c_fp]),
    "mac_rowdot_bwd_workspace_bytes": (ctypes.c_size_t, [c_ll, c_int]),
    "mac_colsum": (c_int, [c_fp, c_fp, c_int, c_int, c_int, c_int, c_fp]),
    "mac_axpy": (c_int, [c_fp, c_fp, c_f, c_ll, c_fp]),
    "mac_clip_adam_ema_step": (c_int, [c_fp, c_fp, c_fp, c_fp, c_fp, c_ll, c_f, c_f, c_f, c_f, c_f, c_f, c_int, c_f, c_fp, c_fp,
                                       c_sz, c_fp]),
    "mac_optimizer_workspace_bytes": (c_sz, []),
    "mac_rowdot_fwd": (c_int, [ctypes.POINTER(c_fp), ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_int, c_fp, c_f, c_fp,
                               c_ll, c_fp]),
    "mac_attend_fwd": (c_int, [c_fp, c_fp, c_fp, c_ll, c_ll, c_fp, c_fp, c_int, c_int, c_int, c_fp]),
    "mac_bcast_op": (c_int, [c_fp, c_fp, c_int, c_f, c_fp, c_fp, c_int, c_int, c_int, c_fp]),
    "mac_softmax_xent": (c_int, [c_fp, c_fp, c_fp, c_fp, c_f, c_int, c_int, c_fp]),
    "mac_answer_topk": (c_int, [c_fp, c_int, c_int, c_int, c_fp, c_fp, c_fp]),
    "mac_ingest_nchw": (c_int, [c_fp, c_int, c_fp, c_int, c_int, c_int, c_int, c_int, c_fp]),
    "mac_ingest_nchw_train": (c_int, [c_fp, c_fp, c_fp, c_int, c_f, c_u64, c_int, c_int, c_int, c_int, c_int, c_int, c_fp]),
    "mac_ingest_nchw_f16": (c_int, [c_fp, c_fp, c_int, c_int, c_int, c_int, c_int, c_fp]),
    "mac_ingest_nchw_train_f16": (c_int, [c_fp, c_fp, c_fp, c_int, c_f, c_u64, c_int, c_int, c_int, c_int, c_int, c_int,
                                          c_fp]),
    "mac_kb_gather": (c_int, [c_fp, c_fp, c_fp, c_int, c_int, c_int, c_int, c_int, c_fp]),
    "mac_kb_gather_bwd": (c_int, [c_fp, c_fp, c_fp, c_int, c_int, c_int, c_int, c_fp]),
    "mac_kb_pool_insert": (c_int, [c_fp, c_fp, c_fp, c_int, c_int, c_int, c_int, c_int, c_fp]),
    "mac_kb_gather_bf16": (c_int, [c_fp, c_fp, c_fp, c_int, c_int, c_int, c_int, c_fp]),
    "mac_im2col3x3": (c_int, [c_fp, c_fp, c_int, c_f, c_u64, c_int, c_int, c_int, c_int, c_int, c_int, c_fp]),
    "mac_im2col3x3_fp8": (c_int, [c_fp, c_fp, c_fp, c_fp, c_sz, c_int, c_int, c_int, c_int, c_fp]),
    "mac_im2col3x3_fp8_workspace_bytes": (c_sz, [c_int, c_int, c_int, c_int]),
    "mac_linear_fp8_fwd": (c_int, [c_fp, c_fp, c_fp, c_fp, c_fp, c_int, c_fp, c_int, c_int, c_int, c_fp]),
    "mac_embed_fwd": (c_int, [c_fp, c_fp, c_f, c_u64, c_int, c_int, c_fp, c_fp, c_int, c_int, c_int, c_int, c_fp]),
    "mac_embed_bwd": (c_int, [c_fp, c_fp, c_f, c_u64, c_int, c_int, c_fp, c_int, c_int, c_int, c_int, c_fp]),
    "mac_lstm_workspace_bytes": (c_sz, [c_int, c_int, c_int]),
    "mac_lstm_fwd": (c_int, [c_fp, c_fp, c_fp, c_fp, c_fp, c_f, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_sz, c_int, c_int,
                             c_int, c_int, c_fp]),
    "mac_lstm_bwd": (c_int, [c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_fp, c_sz, c_int, c_int, c_int, c_int,
                             c_fp]),
    "mac_embed_fwd_tc": (c_int, [c_fp, c_fp, c_f, c_u64, c_int, c_int, c_fp, c_fp, c_int, c_int, c_int, c_int, c_fp]),
    "mac_pack_weight_bf16_kpad": (c_int, [c_fp, c_fp, c_int, c_int, c_int, c_fp]),
    "mac_lstm_fwd_tc": (c_int, [c_fp, c_fp, c_fp, c_fp, c_fp, c_f, c_fp, c_fp, c_fp, c_fp, c_fp, c_int, c_int, c_int, c_int,
                                c_fp]),
    "mac_lstm_bwd_tc": (c_int, [c_fp] * 15 + [c_sz, c_int, c_int, c_int, c_int, c_int, c_fp]),
    "mac_lstm_bwd_tc_workspace_bytes": (c_sz, [c_int, c_int, c_int, c_int, c_int]),
    "mac_col2im3x3": (c_int, [c_fp, c_fp, c_f, c_u64, c_int, c_int, c_int, c_int, c_int, c_int, c_fp]),
    "mac_conv3x3_bwd_tc": (c_int, [c_fp, c_fp, c_fp, c_fp, c_int, c_f, c_u64, c_int, c_int, c_fp, c_fp, c_fp, c_fp, c_sz,
                                   c_int, c_int, c_int, c_int, c_int, c_fp]),
    "mac_conv3x3_bwd_tc_workspace_bytes": (c_sz, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "mac_im2col3x3_split": (c_int, [c_fp, c_fp, c_f, c_u64, c_int, c_int, c_int, c_int, c_int, c_int, c_fp]),
    "mac_linear_tc32_fwd": (c_int, [c_fp, c_fp, c_fp, c_int, c_fp, c_int, c_int, c_int, c_fp]),
    "mac_conv3x3_bwd_tc32": (c_int, [c_fp, c_fp, c_fp, c_fp, c_int, c_f, c_u64, c_int, c_int, c_fp, c_fp, c_fp, c_fp, c_sz,
                                     c_int, c_int, c_int, c_int, c_int, c_fp]),
    "mac_conv3x3_bwd_tc32_workspace_bytes": (c_sz, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "mac_im2col": (c_int, [c_fp, c_fp, c_int, c_f, c_u64] + [c_int] * 8 + [c_fp]),
    "mac_col2im": (c_int, [c_fp, c_fp, c_f, c_u64] + [c_int] * 8 + [c_fp]),
    "mac_im2col_t": (c_int, [c_fp, c_fp, c_int, c_f, c_u64] + [c_int] * 8 + [c_fp]),
    "mac_conv_bwd_tc": (c_int, [c_fp, c_fp, c_fp, c_fp, c_int, c_f, c_u64, c_int, c_int, c_fp, c_fp, c_fp, c_fp, c_sz]
                        + [c_int] * 7 + [c_fp]),
    "mac_conv_bwd_tc_workspace_bytes": (c_sz, [c_int] * 8),
    "mac_conv_bwd_tc32": (c_int, [c_fp, c_fp, c_fp, c_fp, c_int, c_f, c_u64, c_int, c_int, c_fp, c_fp, c_fp, c_fp, c_sz]
                          + [c_int] * 7 + [c_fp]),
    "mac_conv_bwd_tc32_workspace_bytes": (c_sz, [c_int] * 8),
    "mac_loc_cols_width": (c_int, [c_int, c_int]),
    "mac_loc_cols": (c_int, [c_fp, c_fp, c_int, c_f, c_u64] + [c_int] * 8 + [c_fp]),
    "mac_loc_cols_t": (c_int, [c_fp, c_fp, c_int, c_f, c_u64] + [c_int] * 8 + [c_fp]),
    "mac_linear_tc_fwd_acc": (c_int, [c_fp, c_fp, c_int, c_fp, c_int, c_int, c_int, c_fp]),
    "mac_linear_tc32_fwd_acc": (c_int, [c_fp, c_fp, c_int, c_fp, c_int, c_int, c_int, c_fp]),
    "mac_conv_bwd_loc_tc": (c_int, [c_fp, c_fp, c_fp, c_fp, c_int, c_f, c_u64, c_int, c_int, c_fp, c_int, c_int, c_fp, c_fp,
                                    c_fp, c_fp, c_fp, c_sz] + [c_int] * 7 + [c_fp]),
    "mac_conv_bwd_loc_tc_workspace_bytes": (c_sz, [c_int] * 9),
    "mac_conv_bwd_loc_tc32": (c_int, [c_fp, c_fp, c_fp, c_fp, c_int, c_f, c_u64, c_int, c_int, c_fp, c_int, c_int, c_fp, c_fp,
                                      c_fp, c_fp, c_fp, c_sz] + [c_int] * 7 + [c_fp]),
    "mac_conv_bwd_loc_tc32_workspace_bytes": (c_sz, [c_int] * 9),
    "mac_pack_weight_bf16": (c_int, [c_fp, c_fp, c_int, c_int, c_fp]),
    "mac_pack_weight_split3": (c_int, [c_fp, c_fp, c_int, c_int, c_fp]),
    "mac_pack_weight_fp8": (c_int, [c_fp, c_fp, c_fp, c_int, c_int, c_fp]),
    "mac_pack_weight_bf16_split": (c_int, [c_fp, c_fp, c_fp, c_int, c_int, c_fp]),
    "mac_linear_tc_small_fwd": (c_int, [ctypes.POINTER(c_fp), ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_int, c_fp, c_fp,
                                        c_fp, c_f, c_int, c_fp, c_int, c_fp, c_int, c_fp, c_fp, c_fp, c_int, c_int, c_fp]),
    "mac_linear_tc_fwd": (c_int, [c_fp, c_fp, c_fp, c_int, c_fp, c_int, c_int, c_int, c_int, c_fp]),
    "mac_linear_tc_seg_fwd": (c_int, [ctypes.POINTER(c_fp), ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_int, c_fp, c_fp,
                                      c_f, c_int, c_fp, c_int, c_int, c_int, c_fp, c_sz, c_fp]),
    "mac_linear_tc_seg_workspace_bytes": (c_sz, [c_int, c_int]),
    "mac_linear_bwd_tc": (c_int, [ctypes.POINTER(c_fp), ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_int, c_fp, c_fp, c_int,
                                  ctypes.POINTER(c_fp), ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_fp, c_fp, c_int, c_int,
                                  c_fp, c_sz, c_fp]),
    "mac_linear_bwd_tc_workspace_bytes": (c_sz, [c_int, ctypes.POINTER(c_int), c_int, c_int]),
}

_lib = None


class MacB200Error(RuntimeError):
    pass


def load():
    """Load the library (once).  Raises if it has not been built -- there is no fallback path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MacB200Error("%s not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(nvcc, sm_90a).  mac_network_b200 has no CPU/PyTorch fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)          # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.mac_b200_abi_version() != 1:
        raise MacB200Error("ABI version mismatch")
    _lib = lib
    return lib


def check(status, what=""):
    if status != 0:
        msg = load().mac_b200_strerror(status).decode()
        raise MacB200Error("%s failed: status %d (%s)" % (what or "mac_b200 call", status, msg))


def ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def segments(ts):
    """(pointers, widths, leading dimensions): the arrays a segmented entry point takes for a list of 2-D row-major tensors.
    A None entry (an output segment nobody asked for) gives a null pointer, width 0 and leading dimension 0."""
    n = len(ts)
    return ((c_fp * n)(*[None if t is None else t.data_ptr() for t in ts]),
            (c_int * n)(*[0 if t is None else t.shape[1] for t in ts]),
            (c_int * n)(*[0 if t is None else t.stride(0) for t in ts]))


def act_code(act, relu):
    """ACT code of an activation name; "RELU" is the configured `relu`: ELU when relu == "ELU", else max(x, 0)."""
    if act == "RELU":
        return ACT["ELU"] if relu == "ELU" else ACT["RELU_STD"]
    return ACT[act]


def linear_bwd(xs, Wt, dy, dxs, accum, dW, db, ws, ws_bytes, stream):
    """Backward of y = concat(xs) @ W + b (mac_linear_bwd): dxs[i] = (or += where accum[i]) dy @ Wt's rows of segment i
    (a None dxs[i] is skipped; Wt = W^T, needed only when some dxs[i] is given), dW += concat(xs)^T @ dy, db += colsum(dy)
    (each skipped when None).  `ws`: the caller's split-K workspace; its size chooses the summation order."""
    n = len(xs)
    x_p, x_k, x_ld = segments(xs)
    dx_p, _, dx_ld = segments(dxs)
    check(load().mac_linear_bwd(x_p, x_k, x_ld, n, ptr(Wt), ptr(dy), dy.stride(0), dx_p, dx_ld,
                                (c_int * n)(*[int(a) for a in accum]), ptr(dW), ptr(db), dy.shape[0], dy.shape[1], ptr(ws),
                                ws_bytes, stream), "mac_linear_bwd")
