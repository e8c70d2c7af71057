"""ctypes binding of the C-ABI CUDA layer (include/lce_b200.h).

PyTorch is used only as plumbing: device memory (torch tensors), streams and
``torch.distributed``. Every function here goes through ``liblce_b200.so``; there
is no eager / CPU fallback -- a missing library or device raises ``LceError``.

The Python names mirror the reference's op surface (LCE/tflite/kernels):
``quantize`` = LceQuantize, ``dequantize`` = LceDequantize, ``BConv2d`` =
LceBconv2d (Init/Prepare/Eval as constructor / set_input_shape / __call__),
``bmaxpool`` = LceBMaxPool2d, ``BGemm`` = core/bgemm.
"""
from __future__ import annotations

import ctypes as C
import math
import os

import torch

from . import build as _build

PADDING_SAME, PADDING_VALID = 0, 1
ACT_NONE, ACT_RELU, ACT_RELU_N1_TO_1, ACT_RELU6 = 0, 1, 2, 3
OUT_FLOAT, OUT_INT8, OUT_BITPACKED, OUT_RAW_ACC = 0, 1, 2, 3
T_FLOAT, T_INT8, T_BOOL = 0, 1, 2


class LceError(RuntimeError):
    pass


class BconvDesc(C.Structure):
    """``lce_bconv2d_desc`` (include/lce_b200_types.h)."""

    _fields_ = [(n, C.c_int32) for n in (
        "batch", "in_h", "in_w", "channels_in", "filter_h", "filter_w",
        "channels_out", "groups", "stride_h", "stride_w", "dilation_h",
        "dilation_w", "padding", "pad_value", "activation", "out_type")] + [
        ("out_scale", C.c_float), ("out_zero_point", C.c_int32)]


class BMaxPoolDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "batch", "in_h", "in_w", "channels_packed", "filter_h", "filter_w",
        "stride_h", "stride_w", "padding")]


class PoolDesc(C.Structure):
    """``lce_f32_pool_desc`` (include/lce_b200_builtins.h)."""
    _fields_ = [(n, C.c_int32) for n in (
        "batch", "in_h", "in_w", "channels", "filter_h", "filter_w", "stride_h", "stride_w",
        "padding", "activation")]


class ChainDesc(C.Structure):
    """lce_chain_desc: device pointers of the per-channel vectors; None = the op is absent."""
    _fields_ = [("shift_in", C.c_void_p), ("alpha", C.c_void_p), ("shift_out", C.c_void_p),
                ("sign_shift", C.c_void_p)]


def _chain_desc(shift_in=None, alpha=None, shift_out=None, sign_shift=None):
    vecs = [None if v is None else _dev(v, torch.float32) for v in (shift_in, alpha, shift_out, sign_shift)]
    return ChainDesc(*[None if v is None else v.data_ptr() for v in vecs]), vecs


class GateDesc(C.Structure):
    """lce_gate_desc: device pointers; gate [batch, C] is required, None = the op is absent."""
    _fields_ = [("gate", C.c_void_p), ("alpha", C.c_void_p), ("sign_scale", C.c_void_p),
                ("sign_shift", C.c_void_p)]


def _gate_desc(gate, alpha=None, sign_scale=None, sign_shift=None):
    vecs = [None if v is None else _dev(v, torch.float32) for v in (gate, alpha, sign_scale, sign_shift)]
    return GateDesc(*[None if v is None else v.data_ptr() for v in vecs]), vecs


class ScaleDesc(C.Structure):
    """lce_scale_desc: device pointers; scale [OH * OW, C] is required, None = the op is absent."""
    _fields_ = [("scale", C.c_void_p), ("sign_scale", C.c_void_p), ("sign_shift", C.c_void_p)]


def _scale_desc(scale, sign_scale=None, sign_shift=None):
    vecs = [None if v is None else _dev(v, torch.float32) for v in (scale, sign_scale, sign_shift)]
    return ScaleDesc(*[None if v is None else v.data_ptr() for v in vecs]), vecs


class BgemmEpilogue(C.Structure):
    _fields_ = [("out_type", C.c_int32), ("clamp_min", C.c_int32),
                ("clamp_max", C.c_int32), ("multiplier", C.c_void_p),
                ("bias", C.c_void_p), ("thresholds", C.c_void_p)]


EXPORTS = [
    "lce_b200_abi_version", "lce_b200_last_error", "lce_b200_device_count",
    "lce_b200_quantize", "lce_b200_dequantize", "lce_b200_bmaxpool_out_shape",
    "lce_b200_bmaxpool", "lce_b200_bconv2d_out_shape", "lce_b200_bconv2d_create",
    "lce_b200_bconv2d_set_input_shape", "lce_b200_bconv2d_get_desc",
    "lce_b200_bconv2d_set_zero_padding_mode", "lce_b200_path_counts", "lce_b200_tc_debug",
    "lce_b200_bconv2d_run", "lce_b200_bconv2d_run_fused", "lce_b200_bconv2d_run_fused_chain",
    "lce_b200_bconv2d_run_fused_pair",
    "lce_b200_bconv2d_run_fused_gate", "lce_b200_bconv2d_run_fused_scale",
    "lce_b200_bconv2d_run_slice", "lce_b200_bconv2d_run_slice_add", "lce_b200_bconv2d_run_fused_shuffle",
    "lce_b200_bconv2d_run_fused_fc", "lce_b200_bconv2d_run_fused_fc_max",
    "lce_b200_f32_chain_sign", "lce_b200_f32_gate_sign", "lce_b200_f32_scale_sign", "lce_b200_f32_logistic",
    "lce_b200_f32_affine_sign", "lce_b200_f32_maxpool_affine_sign",
    "lce_b200_f32_maximum", "lce_b200_f32_minimum", "lce_b200_f32_div", "lce_b200_f32_round",
    "lce_b200_f32_quant2_planes", "lce_b200_f32_grouped_conv2d",
    "lce_b200_bconv2d_bases_create", "lce_b200_bconv2d_bases_set_input_shape",
    "lce_b200_bconv2d_bases_get_desc", "lce_b200_bconv2d_bases_run", "lce_b200_bconv2d_bases_destroy",
    "lce_b200_f32_shift_sign_planes",
    "lce_b200_f32_resize_nearest", "lce_b200_f32_resize_bilinear", "lce_b200_f32_upsample_add_sign",
    "lce_b200_f32_argmax", "lce_b200_f32_reduce_max", "lce_b200_resize_bilinear_argmax_max_row_floats", "lce_b200_f32_resize_bilinear_argmax",
    "lce_b200_f32_depth_to_space", "lce_b200_subpixel_conv_max_out_channels", "lce_b200_f32_subpixel_conv",
    "lce_b200_f32_transpose_conv2d",
    "lce_b200_detection_max_anchors", "lce_b200_detection_workspace_bytes", "lce_b200_f32_detection_postprocess",
    "lce_b200_bconv2d_run_f32", "lce_b200_bconv2d_run_host",
    "lce_b200_bconv2d_destroy", "lce_b200_bgemm_create", "lce_b200_bgemm_run",
    "lce_b200_bgemm_destroy", "lce_b200_launch_count",
]

_lib = None


def lib():
    """Load liblce_b200.so (built in-tree). Fails loudly if it is missing."""
    global _lib
    if _lib is None:
        path = os.environ.get("LCE_B200_LIB") or _build.cuda_lib_path()   # override: A/B experiments
        if not os.path.exists(path):
            raise LceError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; "
                           "g.build()'` (there is no CPU fallback)")
        _lib = C.CDLL(path)
        _lib.lce_b200_last_error.restype = C.c_char_p
        _lib.lce_b200_launch_count.restype = C.c_uint64
        if _lib.lce_b200_abi_version() != 1:
            raise LceError("liblce_b200.so ABI version mismatch")
    return _lib


def _check(rc):
    if rc != 0:
        raise LceError(lib().lce_b200_last_error().decode() or f"error {rc}")


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _dev(t, dtype=None):
    if not t.is_cuda:
        raise LceError("expected a CUDA tensor (no CPU path)")
    if dtype is not None and t.dtype != dtype:
        raise LceError(f"expected dtype {dtype}, got {t.dtype}")
    return t.contiguous()


def path_counts():
    """Launches per binary inner product so far: [wgmma, mma.sync (b1 or int8), XOR + POPC]."""
    a = (C.c_uint64 * 3)()
    lib().lce_b200_path_counts(a)
    return [int(v) for v in a]


def launch_count():
    return int(lib().lce_b200_launch_count())


def cdiv(a, b):
    return (a + b - 1) // b


# ------------------------------------------------------------------------- #
def quantize(x: torch.Tensor, zero_point: int = 0, out: torch.Tensor | None = None):
    """LceQuantize: bitpack the last axis (float32 / int8 / bool) into int32 words."""
    x = _dev(x)
    if x.dtype == torch.float32:
        t = T_FLOAT
    elif x.dtype == torch.int8:
        t = T_INT8
    elif x.dtype == torch.bool:
        t = T_BOOL
    else:
        raise LceError(f"LceQuantize: unsupported input type {x.dtype}")
    cols = x.shape[-1]
    rows = x.numel() // cols if cols else 0
    if out is None:
        out = torch.empty(x.shape[:-1] + (cdiv(cols, 32),), dtype=torch.int32, device=x.device)
    _check(lib().lce_b200_quantize(C.c_int(t), _p(x), C.c_int64(rows), C.c_int64(cols),
                                   C.c_int32(zero_point), _p(out), _stream()))
    return out


def dequantize(packed: torch.Tensor, channels: int, dtype=torch.float32, scale=1.0,
               zero_point=0):
    """LceDequantize: unpack int32 words into +-1 float / int8 / bool."""
    packed = _dev(packed, torch.int32)
    t = {torch.float32: T_FLOAT, torch.int8: T_INT8, torch.bool: T_BOOL}.get(dtype)
    if t is None:
        raise LceError(f"LceDequantize: unsupported output type {dtype}")
    if packed.shape[-1] != cdiv(channels, 32):
        raise LceError("LceDequantize: packed channels do not match")
    rows = packed.numel() // packed.shape[-1] if packed.shape[-1] else 0
    out = torch.empty(packed.shape[:-1] + (channels,), dtype=dtype, device=packed.device)
    _check(lib().lce_b200_dequantize(C.c_int(t), _p(packed), C.c_int64(rows),
                                     C.c_int64(channels), C.c_float(scale),
                                     C.c_int32(zero_point), _p(out), _stream()))
    return out


def bmaxpool(x: torch.Tensor, filter_hw, stride_hw, padding=PADDING_SAME):
    """LceBMaxPool2d on a bitpacked NHWC tensor."""
    x = _dev(x, torch.int32)
    b, h, w, c = x.shape
    d = BMaxPoolDesc(b, h, w, c, filter_hw[0], filter_hw[1], stride_hw[0], stride_hw[1], padding)
    oh, ow = C.c_int(), C.c_int()
    _check(lib().lce_b200_bmaxpool_out_shape(C.byref(d), C.byref(oh), C.byref(ow)))
    out = torch.empty((b, oh.value, ow.value, c), dtype=torch.int32, device=x.device)
    _check(lib().lce_b200_bmaxpool(C.byref(d), _p(x), _p(out), _stream()))
    return out


def chain_sign(x: torch.Tensor, shift_in=None, alpha=None, shift_out=None, sign_shift=None,
               out=True, packed=True, channels=None):
    """ReActNet's per-channel chain (RPReLU, then RSign's signs) over the last axis of x, or over
    `channels` trailing elements (PRELU with a trailing-shape alpha). Returns (out | None,
    packed | None)."""
    x = _dev(x, torch.float32)
    ch = channels or x.shape[-1]
    rows = x.numel() // ch
    desc, _keep = _chain_desc(shift_in, alpha, shift_out, sign_shift)
    o = torch.empty_like(x) if out else None
    pk = torch.empty(x.shape[:-1] + (cdiv(x.shape[-1], 32),), dtype=torch.int32,
                     device=x.device) if packed else None
    _check(lib().lce_b200_f32_chain_sign(_p(x), C.byref(desc), C.c_int64(rows), C.c_int(ch), _p(o),
                                         _p(pk), _stream()))
    return o, pk


def gate_sign(x: torch.Tensor, gate, residual=None, activation=0, alpha=None, sign_scale=None,
              sign_shift=None, out=True, packed=True):
    """Real-to-Binary's gated tail over x [B, H, W, C] with gate [B, C] (or [B, 1, 1, C]):
    act(prelu(x * gate, alpha) + residual), and the signs of that * sign_scale + sign_shift.
    Returns (out | None, packed | None)."""
    x = _dev(x, torch.float32)
    b, ch = x.shape[0], x.shape[-1]
    desc, _keep = _gate_desc(gate, alpha, sign_scale, sign_shift)
    res = None if residual is None else _dev(residual, torch.float32)
    o = torch.empty_like(x) if out else None
    pk = torch.empty(x.shape[:-1] + (cdiv(ch, 32),), dtype=torch.int32,
                     device=x.device) if packed else None
    _check(lib().lce_b200_f32_gate_sign(_p(x), C.byref(desc), _p(res), C.c_int(activation),
                                        C.c_int64(b), C.c_int64(x.numel() // max(b * ch, 1)),
                                        C.c_int(ch), _p(o), _p(pk), _stream()))
    return o, pk


def scale_sign(x: torch.Tensor, scale, residual=None, activation=0, sign_scale=None, sign_shift=None,
               out=True, packed=True):
    """XNOR-Net++'s scaled tail over x [B, H, W, C] with scale [H, W, C] (or [1, H, W, C]):
    act(x * scale + residual), and the signs of that * sign_scale + sign_shift. `out` may also be
    a tensor to write into (x itself, for one in place). Returns (out | None, packed | None)."""
    x = _dev(x, torch.float32)
    b, ch = x.shape[0], x.shape[-1]
    desc, _keep = _scale_desc(scale, sign_scale, sign_shift)
    res = None if residual is None else _dev(residual, torch.float32)
    o = out if isinstance(out, torch.Tensor) else (torch.empty_like(x) if out else None)
    pk = torch.empty(x.shape[:-1] + (cdiv(ch, 32),), dtype=torch.int32,
                     device=x.device) if packed else None
    _check(lib().lce_b200_f32_scale_sign(_p(x), C.byref(desc), _p(res), C.c_int(activation),
                                         C.c_int64(b), C.c_int64(x.numel() // max(b * ch, 1)),
                                         C.c_int(ch), _p(o), _p(pk), _stream()))
    return o, pk


def affine_sign(x: torch.Tensor, channels=None, scale=None, shift=None, copy_to=None):
    """The signs of x[..., :channels] * scale + shift over x's pixels (the last axis is the pixel
    stride, so x may be the leading channels of a wider map). copy_to (optional): a float tensor
    with x's pixels whose leading `channels` receive x's, bit for bit. Returns the packed signs."""
    x = _dev(x, torch.float32)
    ch = channels or x.shape[-1]
    rows = x.numel() // x.shape[-1]
    vecs = [None if v is None else _dev(v, torch.float32) for v in (scale, shift)]
    pk = torch.empty(x.shape[:-1] + (cdiv(ch, 32),), dtype=torch.int32, device=x.device)
    if copy_to is not None and (not copy_to.is_cuda or copy_to.dtype != torch.float32 or
                                not copy_to.is_contiguous()):
        raise LceError("affine_sign: copy_to must be a contiguous CUDA float32 tensor")
    _check(lib().lce_b200_f32_affine_sign(_p(x), C.c_int64(x.shape[-1]), C.c_int64(rows), C.c_int(ch),
                                          _p(vecs[0]), _p(vecs[1]), _p(pk), _p(copy_to),
                                          C.c_int64(0 if copy_to is None else copy_to.shape[-1]),
                                          _stream()))
    return pk


def maxpool_affine_sign(x: torch.Tensor, filter_hw, stride_hw, padding=PADDING_VALID, activation=ACT_NONE,
                        scale=None, shift=None):
    """MAX_POOL_2D (with its fused activation) -> MUL(scale) -> ADD(shift) -> LceQuantize in one
    pass over a float NHWC map: the packed signs [B, OH, OW, ceil(C / 32)]. scale / shift: [C]
    float32 CUDA tensors, or None where that op is absent."""
    x = _dev(x, torch.float32)
    b, h, w, c = x.shape
    vecs = [None if v is None else _dev(v, torch.float32) for v in (scale, shift)]
    d = PoolDesc(b, h, w, c, filter_hw[0], filter_hw[1], stride_hw[0], stride_hw[1], padding, activation)
    oh, ow = C.c_int(), C.c_int()
    _check(lib().lce_b200_f32_pool_out_shape(C.byref(d), C.byref(oh), C.byref(ow)))
    pk = torch.empty((b, max(oh.value, 0), max(ow.value, 0), cdiv(c, 32)), dtype=torch.int32, device=x.device)
    _check(lib().lce_b200_f32_maxpool_affine_sign(_p(x), b, h, w, c, filter_hw[0], filter_hw[1], stride_hw[0],
                                                  stride_hw[1], padding, activation, _p(vecs[0]), _p(vecs[1]),
                                                  _p(pk), _stream()))
    return pk


def quant2_planes(x: torch.Tensor, pool=None):
    """DoReFaNet's 2-bit quantiser q = round(clip(x, 0, 1) * 3) of a float NHWC map, as int32 bit
    planes [B, OH, OW, 3 * C / 32] = [bit 0 | bit 1 | bit 1] (C % 32 == 0). pool: None, or
    (filter_hw, stride_hw, padding, activation) of a MAX_POOL_2D applied first."""
    x = _dev(x, torch.float32)
    b, h, w, c = x.shape
    (fh, fw), (sh, sw), padding, activation = pool if pool is not None else ((0, 0), (1, 1), PADDING_VALID, ACT_NONE)
    oh, ow = C.c_int(h), C.c_int(w)
    if pool is not None:
        d = PoolDesc(b, h, w, c, fh, fw, sh, sw, padding, activation)
        _check(lib().lce_b200_f32_pool_out_shape(C.byref(d), C.byref(oh), C.byref(ow)))
    planes = torch.empty((b, max(oh.value, 0), max(ow.value, 0), 3 * (c // 32)), dtype=torch.int32, device=x.device)
    _check(lib().lce_b200_f32_quant2_planes(_p(x), b, h, w, c, fh, fw, sh, sw, padding, activation, _p(planes),
                                            _stream()))
    return planes


def shift_sign_planes(x: torch.Tensor, shifts):
    """ABC-Net's shifted signs of a float map x [..., C] (C % 32 == 0): one int32 plane
    [..., C / 32] per shift, bit = fl(x + shift) < 0. Returns the list of planes."""
    x = _dev(x, torch.float32)
    c = x.shape[-1]
    n = len(shifts)
    planes = [torch.empty(x.shape[:-1] + (c // 32,), dtype=torch.int32, device=x.device) for _ in range(n)]
    sh = (C.c_float * max(n, 1))(*[float(s) for s in shifts])
    ptrs = (C.c_void_p * max(n, 1))(*[p.data_ptr() for p in planes])
    _check(lib().lce_b200_f32_shift_sign_planes(_p(x), C.c_int64(x.numel() // c if c else 0), C.c_int(c),
                                                C.c_int(n), sh, ptrs, _stream()))
    return planes


def resize(x: torch.Tensor, size, bilinear=False, align_corners=False, half_pixel_centers=False):
    """RESIZE_NEAREST_NEIGHBOR (or with bilinear RESIZE_BILINEAR) of a float NHWC map to
    size = (new_height, new_width), bit for bit TFLite's reference kernel."""
    x = _dev(x, torch.float32)
    b, h, w, c = x.shape
    oh, ow = int(size[0]), int(size[1])
    out = torch.empty((b, oh, ow, c), dtype=torch.float32, device=x.device)
    fn = lib().lce_b200_f32_resize_bilinear if bilinear else lib().lce_b200_f32_resize_nearest
    _check(fn(_p(x), b, h, w, c, oh, ow, int(bool(align_corners)), int(bool(half_pixel_centers)), _p(out),
              _stream()))
    return out


def argmax(x: torch.Tensor, axis=-1, out_dtype=torch.int64):
    """ARG_MAX of a float tensor over `axis`, bit for bit TFLite's reference loop (ties to the lowest
    index, a NaN at index 0 gives 0, a NaN elsewhere is never chosen); int64 or int32 labels."""
    x = _dev(x, torch.float32)
    if out_dtype not in (torch.int64, torch.int32):
        raise LceError("argmax: out_dtype must be torch.int64 or torch.int32")
    a = axis + x.dim() if axis < 0 else axis
    if x.dim() < 1 or not 0 <= a < x.dim():
        raise LceError(f"argmax: axis {axis} is out of range for rank {x.dim()}")
    outer, inner = math.prod(x.shape[:a]), math.prod(x.shape[a + 1:])
    out = torch.empty(x.shape[:a] + x.shape[a + 1:], dtype=out_dtype, device=x.device)
    _check(lib().lce_b200_f32_argmax(_p(x), C.c_int64(outer), C.c_int(x.shape[a]), C.c_int64(inner),
                                     int(out_dtype == torch.int64), _p(out), _stream()))
    return out


def reduce_max(x: torch.Tensor, axes, keep_dims=False):
    """REDUCE_MAX of a float tensor over `axes` (contiguous once normalised; negative and duplicate axes as
    in TFLite), TFLite's reference rule bit for bit: cur = -FLT_MAX, then cur = x > cur ? x : cur in index
    order (a NaN is never chosen, the first of equal values wins, an all-NaN / all--inf / empty slice gives
    -FLT_MAX)."""
    x = _dev(x, torch.float32)
    r = x.dim()
    red = sorted({a + r if a < 0 else a for a in ([axes] if isinstance(axes, int) else axes)})
    if not red or red[0] < 0 or red[-1] >= r or red != list(range(red[0], red[-1] + 1)):
        raise LceError(f"reduce_max: axes {axes} must be non-empty, in range and contiguous for rank {r}")
    a, b = red[0], red[-1] + 1
    outer, n, inner = math.prod(x.shape[:a]), math.prod(x.shape[a:b]), math.prod(x.shape[b:])
    shape = x.shape[:a] + ((1,) * (b - a) if keep_dims else ()) + x.shape[b:]
    out = torch.empty(shape, dtype=torch.float32, device=x.device)
    _check(lib().lce_b200_f32_reduce_max(_p(x), C.c_int64(outer), C.c_int64(n), C.c_int64(inner), _p(out),
                                         _stream()))
    return out


def resize_bilinear_argmax_max_row_floats():
    return int(lib().lce_b200_resize_bilinear_argmax_max_row_floats())


def resize_bilinear_argmax(x: torch.Tensor, size, align_corners=False, half_pixel_centers=False,
                           out_dtype=torch.int64):
    """ARG_MAX over the channels of RESIZE_BILINEAR(x) to size = (new_height, new_width), in one pass
    that never writes the resized map: the labels [B, new_height, new_width], bit for bit the two ops'."""
    x = _dev(x, torch.float32)
    if out_dtype not in (torch.int64, torch.int32):
        raise LceError("resize_bilinear_argmax: out_dtype must be torch.int64 or torch.int32")
    b, h, w, c = x.shape
    oh, ow = int(size[0]), int(size[1])
    out = torch.empty((b, oh, ow), dtype=out_dtype, device=x.device)
    _check(lib().lce_b200_f32_resize_bilinear_argmax(_p(x), b, h, w, c, oh, ow, int(bool(align_corners)),
                                                     int(bool(half_pixel_centers)), int(out_dtype == torch.int64),
                                                     _p(out), _stream()))
    return out


def upsample_add_sign(u: torch.Tensor, skip: torch.Tensor, align_corners=False, half_pixel_centers=False,
                      activation=ACT_NONE, out=True, packed=True):
    """RESIZE_NEAREST_NEIGHBOR(u) to skip's size -> ADD(skip) with its activation [-> LceQuantize] in
    one pass. Returns (sum | None, packed signs | None)."""
    u, skip = _dev(u, torch.float32), _dev(skip, torch.float32)
    b, h, w, c = u.shape
    oh, ow = skip.shape[1], skip.shape[2]
    if skip.shape[0] != b or skip.shape[3] != c:
        raise LceError("upsample_add_sign: skip must be [B, new_height, new_width, C]")
    o = torch.empty_like(skip) if out else None
    pk = torch.empty((b, oh, ow, cdiv(c, 32)), dtype=torch.int32, device=u.device) if packed else None
    _check(lib().lce_b200_f32_upsample_add_sign(_p(u), b, h, w, c, oh, ow, int(bool(align_corners)),
                                                int(bool(half_pixel_centers)), _p(skip), C.c_int(activation),
                                                _p(o), _p(pk), _stream()))
    return o, pk


class DetectionOptions(C.Structure):
    """lce_b200_detection_options (TFLite_Detection_PostProcess's custom_options)."""
    _fields_ = [("max_detections", C.c_int), ("max_classes_per_detection", C.c_int),
                ("detections_per_class", C.c_int), ("num_classes", C.c_int), ("use_regular_nms", C.c_int),
                ("nms_score_threshold", C.c_float), ("nms_iou_threshold", C.c_float), ("y_scale", C.c_float),
                ("x_scale", C.c_float), ("h_scale", C.c_float), ("w_scale", C.c_float)]


def detection_max_anchors():
    return int(lib().lce_b200_detection_max_anchors())


def detection_postprocess(boxes: torch.Tensor, scores: torch.Tensor, anchors: torch.Tensor, **options):
    """TFLite_Detection_PostProcess of float box encodings [B, N, K >= 4], class predictions
    [B, N, C + label_offset] and anchors [N, 4], each image as TFLite's kernel computes it alone.
    options: the DetectionOptions fields. Returns (boxes [B, D, 4], classes [B, D], scores [B, D],
    num_detections [B]) with D = max_detections * max_classes_per_detection."""
    boxes, scores, anchors = (_dev(t, torch.float32) for t in (boxes, scores, anchors))
    o = DetectionOptions(**options)
    b, n, k = boxes.shape
    d = o.max_detections * o.max_classes_per_detection
    f = dict(dtype=torch.float32, device=boxes.device)
    out = (torch.empty((b, d, 4), **f), torch.empty((b, d), **f), torch.empty((b, d), **f), torch.empty((b,), **f))
    L = lib()
    L.lce_b200_detection_workspace_bytes.restype = C.c_size_t
    ws_bytes = L.lce_b200_detection_workspace_bytes(b, n, C.byref(o))
    ws = torch.empty(max(int(ws_bytes), 16), dtype=torch.uint8, device=boxes.device)
    _check(L.lce_b200_f32_detection_postprocess(_p(boxes), _p(scores), b, n, k, scores.shape[2], _p(anchors),
                                                C.byref(o), *(_p(t) for t in out), _p(ws), _stream()))
    return out


class BConv2dBases:
    """ABC-Net layer plan (lce_b200_bconv2d_bases_*): M * N LceBconv2d terms, term n * M + m on input
    plane n with base filter m, summed left to right, then the BatchNorm, an optional shortcut and
    the next layer's shifted signs, in one kernel."""

    def __init__(self, m_bases, n_planes, desc: BconvDesc, filters, post_muls, post_biases):
        import numpy as np
        t = m_bases * n_planes
        if not (len(filters) == len(post_muls) == len(post_biases) == t):
            raise LceError("BConv2dBases: M * N filters, multipliers and biases")
        self._h = C.c_void_p()
        self.desc = desc
        self.m, self.n = m_bases, n_planes
        keep = [np.ascontiguousarray(f, np.int32) for f in filters] + \
            [np.ascontiguousarray(v, np.float32) for v in list(post_muls) + list(post_biases)]
        descs = (BconvDesc * t)(*[desc] * t)
        ptr = [a.ctypes.data_as(C.c_void_p) for a in keep]
        fs, ms, bs = ((C.c_void_p * t)(*ptr[k * t:(k + 1) * t]) for k in range(3))
        _check(lib().lce_b200_bconv2d_bases_create(C.c_int(m_bases), C.c_int(n_planes), descs, fs, ms, bs,
                                                   C.byref(self._h)))

    def out_shape(self):
        d = BconvDesc()
        oh, ow = C.c_int(), C.c_int()
        _check(lib().lce_b200_bconv2d_bases_get_desc(self._h, C.byref(d), C.byref(oh), C.byref(ow)))
        return (d.batch, oh.value, ow.value, d.channels_out)

    def __call__(self, planes, bn_scale, bn_shift, bn_activation=ACT_NONE, residual=None,
                 add_activation=ACT_NONE, next_shifts=(), out=True):
        """planes: N packed inputs. Returns (float out | None, [next planes])."""
        planes = [_dev(p, torch.int32) for p in planes]
        b, h, w = planes[0].shape[:3]
        if (b, h, w) != (self.desc.batch, self.desc.in_h, self.desc.in_w):
            _check(lib().lce_b200_bconv2d_bases_set_input_shape(self._h, b, h, w))
            self.desc.batch, self.desc.in_h, self.desc.in_w = b, h, w
        shape = self.out_shape()
        dev = planes[0].device
        o = torch.empty(shape, dtype=torch.float32, device=dev) if out else None
        nxt = [torch.empty(shape[:3] + (shape[3] // 32,), dtype=torch.int32, device=dev) for _ in next_shifts]
        vecs = [_dev(v, torch.float32) for v in (bn_scale, bn_shift)]
        res = None if residual is None else _dev(residual, torch.float32)
        k = len(next_shifts)
        pin = (C.c_void_p * len(planes))(*[p.data_ptr() for p in planes])
        sh = (C.c_float * max(k, 1))(*[float(s) for s in next_shifts])
        pout = (C.c_void_p * max(k, 1))(*[p.data_ptr() for p in nxt])
        _check(lib().lce_b200_bconv2d_bases_run(self._h, pin, _p(vecs[0]), _p(vecs[1]), C.c_int(bn_activation),
                                                _p(res), C.c_int(add_activation), _p(o), C.c_int(k), sh, pout,
                                                _stream()))
        return o, nxt

    def close(self):
        if self._h:
            lib().lce_b200_bconv2d_bases_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ConvDesc(C.Structure):
    """``lce_f32_conv_desc`` (include/lce_b200_builtins.h)."""
    _fields_ = [(n, C.c_int32) for n in (
        "batch", "in_h", "in_w", "in_c", "filter_h", "filter_w", "out_c", "stride_h", "stride_w",
        "dilation_h", "dilation_w", "padding", "activation")]


def grouped_conv2d(x: torch.Tensor, filt: torch.Tensor, bias=None, stride=(1, 1), dilation=(1, 1),
                   padding=PADDING_SAME, activation=ACT_NONE, scale=None, shift=None,
                   post_activation=ACT_NONE, out: torch.Tensor | None = None):
    """Grouped CONV_2D of a float NHWC map x [B, H, W, C_in] with an OHWI filter [C_out, kh, kw,
    C_in / groups] (groups = C_in / filter_in, as TFLite infers it), then the optional BatchNorm
    epilogue fl(fl(act(y) * scale) + shift) and post_activation. bias / scale / shift: [C_out]
    float32 CUDA tensors or None. `out` may be given (a view at any 4-byte offset)."""
    x = _dev(x, torch.float32)
    filt = _dev(filt, torch.float32)
    b, h, w, cin = x.shape
    cout, kh, kw, fin = filt.shape
    if fin < 1 or cin % fin:
        raise LceError(f"grouped_conv2d: the filter's {fin} input channels do not divide {cin}")
    vecs = [None if v is None else _dev(v, torch.float32) for v in (bias, scale, shift)]
    d = ConvDesc(b, h, w, cin, kh, kw, cout, stride[0], stride[1], dilation[0], dilation[1], padding, activation)
    oh, ow = C.c_int(), C.c_int()
    _check(lib().lce_b200_f32_conv_out_shape(C.byref(d), C.byref(oh), C.byref(ow)))
    if out is None:
        out = torch.empty((b, oh.value, ow.value, cout), dtype=torch.float32, device=x.device)
    _check(lib().lce_b200_f32_grouped_conv2d(C.byref(d), C.c_int(cin // fin), _p(x), _p(filt), _p(vecs[0]),
                                             _p(vecs[1]), _p(vecs[2]), C.c_int(post_activation), _p(out),
                                             _stream()))
    return out


def depth_to_space(x: torch.Tensor, block_size: int):
    """DEPTH_TO_SPACE of a float NHWC map [B, H, W, C] to [B, H * r, W * r, C / r^2]: the values
    moved as TFLite's reference moves them."""
    x = _dev(x, torch.float32)
    b, h, w, c = x.shape
    r = int(block_size)
    if r <= 0 or c % (r * r):
        raise LceError(f"depth_to_space: {c} channels are not a multiple of block_size^2 (block size {r})")
    out = torch.empty((b, h * r, w * r, c // (r * r)), dtype=torch.float32, device=x.device)
    _check(lib().lce_b200_f32_depth_to_space(_p(x), b, h, w, c, r, _p(out), _stream()))
    return out


class TransposeConvDesc(C.Structure):
    """``lce_f32_transpose_conv_desc`` (include/lce_b200_types.h)."""
    _fields_ = [(n, C.c_int32) for n in (
        "batch", "in_h", "in_w", "in_c", "filter_h", "filter_w", "out_c", "out_h", "out_w", "stride_h",
        "stride_w", "pad_h", "pad_w", "activation")]


def transpose_conv2d(x: torch.Tensor, filt: torch.Tensor, bias, out_hw, stride, padding=PADDING_SAME,
                     activation=ACT_NONE):
    """TFLite's float TRANSPOSE_CONV of an NHWC map x [B, H, W, C_in] with weights [C_out, kh, kw, C_in]
    to [B, out_h, out_w, C_out]: TFLite's padding for that output size (the floor half), each output one
    fmaf chain in the reference's order, then the bias (may be None) and the activation."""
    x = _dev(x, torch.float32)
    filt = _dev(filt, torch.float32)
    bias = None if bias is None else _dev(bias, torch.float32)
    b, h, w, cin = x.shape
    cout, kh, kw, _ = filt.shape
    (oh, ow), (sh, sw) = out_hw, stride
    want = [(o + s - 1) // s if padding == PADDING_SAME else (o + s - k) // s
            for o, s, k in ((oh, sh, kh), (ow, sw, kw))]
    if filt.shape[3] != cin or want != [h, w]:
        raise LceError(f"transpose_conv2d: input {tuple(x.shape)} is not what a convolution with filter "
                       f"{tuple(filt.shape)}, stride {stride} gives from output {out_hw}")
    ph, pw = (max((n - 1) * s + k - o, 0) // 2 for n, s, k, o in ((h, sh, kh, oh), (w, sw, kw, ow)))
    d = TransposeConvDesc(b, h, w, cin, kh, kw, cout, oh, ow, sh, sw, ph, pw, activation)
    out = torch.empty((b, oh, ow, cout), dtype=torch.float32, device=x.device)
    _check(lib().lce_b200_f32_transpose_conv2d(C.byref(d), _p(x), _p(filt), _p(bias), _p(out), _stream()))
    return out


def subpixel_conv_max_out_channels():
    return int(lib().lce_b200_subpixel_conv_max_out_channels())


def subpixel_conv(x: torch.Tensor, filt: torch.Tensor, bias, block_size: int, img=None, align_corners=False,
                  half_pixel_centers=False, activation=ACT_NONE, add_activation=ACT_NONE):
    """A super-resolution tail in one pass: CONV_2D(x, filt [C_out, kh, kw, C_in], bias, stride 1, SAME,
    activation) -> DEPTH_TO_SPACE(block_size) [-> ADD(RESIZE_BILINEAR(img) to the output's size, with
    add_activation)], [B, H * r, W * r, C_out / r^2]; bit for bit the ops one by one."""
    x = _dev(x, torch.float32)
    filt = _dev(filt, torch.float32)
    bias = None if bias is None else _dev(bias, torch.float32)
    img = None if img is None else _dev(img, torch.float32)
    b, h, w, cin = x.shape
    cout, kh, kw, _ = filt.shape
    r = int(block_size)
    if r <= 0 or cout % (r * r):
        raise LceError(f"subpixel_conv: {cout} output channels are not a multiple of block_size^2 (block size {r})")
    d = ConvDesc(b, h, w, cin, kh, kw, cout, 1, 1, 1, 1, PADDING_SAME, activation)
    out = torch.empty((b, h * r, w * r, cout // (r * r)), dtype=torch.float32, device=x.device)
    ih, iw = (img.shape[1], img.shape[2]) if img is not None else (0, 0)
    _check(lib().lce_b200_f32_subpixel_conv(C.byref(d), _p(x), _p(filt), _p(bias), r, _p(img), ih, iw,
                                            int(bool(align_corners)), int(bool(half_pixel_centers)),
                                            int(add_activation), _p(out), _stream()))
    return out


class BConv2d:
    """LceBconv2d plan: constructor = Init + Prepare + OneTimeSetup
    (LCE/tflite/kernels/bconv2d.cc:85-392), ``__call__`` = Eval (:551-564)."""

    def __init__(self, desc: BconvDesc, filt, post_mul=None, post_bias=None, thresholds=None):
        self._h = C.c_void_p()
        self.desc = desc
        keep = []

        def ptr(t, dtype):
            if t is None:
                return C.c_void_p(0)
            if isinstance(t, torch.Tensor):
                t = t.to(dtype).contiguous()
                keep.append(t)
                return C.c_void_p(t.data_ptr())
            import numpy as np
            a = np.ascontiguousarray(t, {torch.int32: np.int32, torch.float32: np.float32}[dtype])
            keep.append(a)
            return a.ctypes.data_as(C.c_void_p)

        rc = lib().lce_b200_bconv2d_create(
            C.byref(desc), ptr(filt, torch.int32), ptr(post_mul, torch.float32),
            ptr(post_bias, torch.float32), ptr(thresholds, torch.int32), C.byref(self._h))
        _check(rc)

    def set_input_shape(self, batch, in_h, in_w):
        _check(lib().lce_b200_bconv2d_set_input_shape(self._h, batch, in_h, in_w))
        self.desc.batch, self.desc.in_h, self.desc.in_w = batch, in_h, in_w

    def set_zero_padding_mode(self, mode):
        """0: the reference kernel's integers (reference.h:100-103); 1: the optimised kernels'
        float correction (zero_padding_correction.h) -- see include/lce_b200_types.h."""
        _check(lib().lce_b200_bconv2d_set_zero_padding_mode(self._h, int(mode)))

    def out_shape(self):
        d = BconvDesc()
        oh, ow = C.c_int(), C.c_int()
        _check(lib().lce_b200_bconv2d_get_desc(self._h, C.byref(d), C.byref(oh), C.byref(ow)))
        last = cdiv(d.channels_out, 32) if d.out_type == OUT_BITPACKED else d.channels_out
        return (d.batch, oh.value, ow.value, last)

    def out_dtype(self):
        return {OUT_FLOAT: torch.float32, OUT_INT8: torch.int8,
                OUT_BITPACKED: torch.int32}[self.desc.out_type]

    def _alloc(self, like, out):
        if out is None:
            out = torch.empty(self.out_shape(), dtype=self.out_dtype(), device=like.device)
        return out

    def __call__(self, x: torch.Tensor, out: torch.Tensor | None = None):
        """x: bitpacked NHWC int32, or float32 NHWC (LceQuantize fused in front)."""
        x = _dev(x)
        if tuple(x.shape[:3]) != (self.desc.batch, self.desc.in_h, self.desc.in_w):
            self.set_input_shape(*x.shape[:3])
        out = self._alloc(x, out)
        if x.dtype == torch.float32:
            if x.shape[3] != self.desc.channels_in:
                raise LceError("LceBconv2d: float input channels do not match channels_in")
            _check(lib().lce_b200_bconv2d_run_f32(self._h, _p(x), _p(out), _stream()))
        elif x.dtype == torch.int32:
            if x.shape[3] != cdiv(self.desc.channels_in, 32):
                raise LceError("LceBconv2d: packed input channels do not match channels_in")
            _check(lib().lce_b200_bconv2d_run(self._h, _p(x), _p(out), _stream()))
        else:
            raise LceError(f"LceBconv2d: unsupported input type {x.dtype}")
        return out

    def run_fused_chain(self, x: torch.Tensor, residual=None, add_activation=0, shift_in=None,
                        alpha=None, shift_out=None, sign_shift=None, packed=True):
        """lce_b200_bconv2d_run_fused_chain on bitpacked x: returns (float out, packed signs | None)."""
        x = _dev(x, torch.int32)
        if tuple(x.shape[:3]) != (self.desc.batch, self.desc.in_h, self.desc.in_w):
            self.set_input_shape(*x.shape[:3])
        out = self._alloc(x, None)
        pk = torch.empty(out.shape[:3] + (cdiv(out.shape[3], 32),), dtype=torch.int32,
                         device=x.device) if packed else None
        res = None if residual is None else _dev(residual, torch.float32)
        desc, _keep = _chain_desc(shift_in, alpha, shift_out, sign_shift)
        _check(lib().lce_b200_bconv2d_run_fused_chain(self._h, _p(x), _p(res), C.c_int(add_activation),
                                                      C.byref(desc), _p(out), _p(pk), _stream()))
        return out, pk

    def run_fused_gate(self, x: torch.Tensor, gate, residual=None, add_activation=0, alpha=None,
                       sign_scale=None, sign_shift=None, packed=True, out=None):
        """lce_b200_bconv2d_run_fused_gate on bitpacked x with gate [batch, C] (or [batch, 1, 1, C]):
        returns (float out, packed signs | None). `out` may be given (the C-ABI refuses one that
        overlaps the residual or the gate)."""
        x = _dev(x, torch.int32)
        if tuple(x.shape[:3]) != (self.desc.batch, self.desc.in_h, self.desc.in_w):
            self.set_input_shape(*x.shape[:3])
        out = self._alloc(x, out)
        pk = torch.empty(out.shape[:3] + (cdiv(out.shape[3], 32),), dtype=torch.int32,
                         device=x.device) if packed else None
        res = None if residual is None else _dev(residual, torch.float32)
        desc, _keep = _gate_desc(gate, alpha, sign_scale, sign_shift)
        _check(lib().lce_b200_bconv2d_run_fused_gate(self._h, _p(x), C.byref(desc), _p(res),
                                                     C.c_int(add_activation), _p(out), _p(pk),
                                                     _stream()))
        return out, pk

    def run_fused_scale(self, x: torch.Tensor, scale, residual=None, add_activation=0, sign_scale=None,
                        sign_shift=None, packed=True, out=None):
        """lce_b200_bconv2d_run_fused_scale on bitpacked x with scale [OH, OW, C] (or [1, OH, OW, C]):
        returns (float out, packed signs | None). `out` may be given (the C-ABI refuses one that
        overlaps the residual or the scale)."""
        x = _dev(x, torch.int32)
        if tuple(x.shape[:3]) != (self.desc.batch, self.desc.in_h, self.desc.in_w):
            self.set_input_shape(*x.shape[:3])
        out = self._alloc(x, out)
        pk = torch.empty(out.shape[:3] + (cdiv(out.shape[3], 32),), dtype=torch.int32,
                         device=x.device) if packed else None
        res = None if residual is None else _dev(residual, torch.float32)
        desc, _keep = _scale_desc(scale, sign_scale, sign_shift)
        _check(lib().lce_b200_bconv2d_run_fused_scale(self._h, _p(x), C.byref(desc), _p(res),
                                                      C.c_int(add_activation), _p(out), _p(pk),
                                                      _stream()))
        return out, pk

    def run_fused_fc(self, x: torch.Tensor, alpha=None, bias=None, activation=0, scale=None, shift=None,
                     bn_activation=0, packed=True):
        """lce_b200_bconv2d_run_fused_fc: a binary dense layer on packed x [rows, ceil(K / 32)] (a 1x1 plan
        with in_h = in_w = 1 and channels_in = K; rows re-plans the batch). Per column c of N:
        y = activation(fl(fl(alpha[c] * D) + bias[c])), then bn_activation(fl(fl(y * scale[c]) + shift[c])),
        D the exact +-1 dot product; each vector [N] may be None. Returns (float out [rows, N], packed
        signs [rows, N / 32] | None)."""
        x = _dev(x, torch.int32)
        rows = x.shape[0]
        if x.dim() != 2 or x.shape[1] != cdiv(self.desc.channels_in, 32):
            raise LceError("run_fused_fc: x must be packed rows [rows, ceil(channels_in / 32)]")
        if (rows, self.desc.in_h, self.desc.in_w) != (self.desc.batch, 1, 1):
            self.set_input_shape(rows, 1, 1)
        n = self.desc.channels_out
        vecs = [None if v is None else torch.as_tensor(v, dtype=torch.float32, device=x.device).contiguous()
                for v in (alpha, bias, scale, shift)]
        out = torch.empty((rows, n), dtype=torch.float32, device=x.device)
        pk = torch.empty((rows, cdiv(n, 32)), dtype=torch.int32, device=x.device) if packed else None
        _check(lib().lce_b200_bconv2d_run_fused_fc(self._h, _p(x), _p(vecs[0]), _p(vecs[1]), C.c_int(activation),
                                                   _p(vecs[2]), _p(vecs[3]), C.c_int(bn_activation), _p(out),
                                                   _p(pk), _stream()))
        return out, pk

    def run_fused_fc_max(self, x: torch.Tensor, points: int, alpha=None, bias=None, activation=0, scale=None,
                         shift=None, bn_activation=0, store_max=True, packed=True):
        """lce_b200_bconv2d_run_fused_fc_max: run_fused_fc's layer on packed x [rows, ceil(K / 32)], rows =
        B * points, then each image's column max by TFLite's REDUCE_MAX rule. Returns (float max [B, N] |
        None, packed signs [B, N / 32] | None)."""
        x = _dev(x, torch.int32)
        rows = x.shape[0]
        if x.dim() != 2 or x.shape[1] != cdiv(self.desc.channels_in, 32):
            raise LceError("run_fused_fc_max: x must be packed rows [rows, ceil(channels_in / 32)]")
        if (rows, self.desc.in_h, self.desc.in_w) != (self.desc.batch, 1, 1):
            self.set_input_shape(rows, 1, 1)
        n, b = self.desc.channels_out, rows // max(points, 1)
        vecs = [None if v is None else torch.as_tensor(v, dtype=torch.float32, device=x.device).contiguous()
                for v in (alpha, bias, scale, shift)]
        keys = torch.empty((max(b, 1), n), dtype=torch.int64, device=x.device)
        out = torch.empty((b, n), dtype=torch.float32, device=x.device) if store_max else None
        pk = torch.empty((b, cdiv(n, 32)), dtype=torch.int32, device=x.device) if packed else None
        _check(lib().lce_b200_bconv2d_run_fused_fc_max(self._h, _p(x), _p(vecs[0]), _p(vecs[1]), C.c_int(activation),
                                                       _p(vecs[2]), _p(vecs[3]), C.c_int(bn_activation),
                                                       C.c_int(points), _p(keys), _p(out), _p(pk), _stream()))
        return out, pk

    def run_slice(self, x: torch.Tensor, out: torch.Tensor, offset: int = 0):
        """lce_b200_bconv2d_run_slice on bitpacked x: writes the float output into channels
        [offset, offset + channels_out) of `out`, a contiguous float32 [B, OH, OW, C] map (or any
        tensor whose last axis is the pixel stride), and nothing else. Returns out."""
        x = _dev(x, torch.int32)
        if tuple(x.shape[:3]) != (self.desc.batch, self.desc.in_h, self.desc.in_w):
            self.set_input_shape(*x.shape[:3])
        if not out.is_cuda or out.dtype != torch.float32 or not out.is_contiguous():
            raise LceError("run_slice: out must be a contiguous CUDA float32 tensor")
        ptr = C.c_void_p(out.data_ptr() + 4 * offset)
        _check(lib().lce_b200_bconv2d_run_slice(self._h, _p(x), ptr, C.c_int64(out.shape[-1]),
                                                _stream()))
        return out

    def run_slice_add(self, x: torch.Tensor, out: torch.Tensor, offset: int = 0, scratch=None):
        """lce_b200_bconv2d_run_slice_add on bitpacked x: adds the float output to channels
        [offset, offset + channels_out) of `out`, a contiguous float32 [B, OH, OW, C] map (or any
        tensor whose last axis is the pixel stride), in place, and writes nothing else. scratch: a
        contiguous CUDA float32 tensor of pixels * channels_out elements, required by CORRECTION
        plans (zero padding with the float correction). Returns out."""
        x = _dev(x, torch.int32)
        if tuple(x.shape[:3]) != (self.desc.batch, self.desc.in_h, self.desc.in_w):
            self.set_input_shape(*x.shape[:3])
        for name, t in (("out", out), ("scratch", scratch)):
            if t is not None and (not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous()):
                raise LceError(f"run_slice_add: {name} must be a contiguous CUDA float32 tensor")
        ptr = C.c_void_p(out.data_ptr() + 4 * offset)
        _check(lib().lce_b200_bconv2d_run_slice_add(self._h, _p(x), ptr, C.c_int64(out.shape[-1]),
                                                    _p(scratch), _stream()))
        return out

    def run_fused_pair(self, second, x: torch.Tensor, residual: torch.Tensor, act1=0, act2=0,
                       packed=True):
        """lce_b200_bconv2d_run_fused_pair: this layer, then `second`, as two residual blocks on
        bitpacked x and shortcut residual. Returns (float x2, packed signs of x2 | None)."""
        x = _dev(x, torch.int32)
        for plan in (self, second):
            if tuple(x.shape[:3]) != (plan.desc.batch, plan.desc.in_h, plan.desc.in_w):
                plan.set_input_shape(*x.shape[:3])
        res = _dev(residual, torch.float32)
        out = torch.empty_like(res)
        pk = torch.empty(res.shape[:3] + (cdiv(res.shape[3], 32),), dtype=torch.int32,
                         device=x.device) if packed else None
        _check(lib().lce_b200_bconv2d_run_fused_pair(self._h, second._h, _p(x), _p(res),
                                                     C.c_int(act1), C.c_int(act2), _p(out),
                                                     _p(pk), _stream()))
        return out, pk

    def run_host(self, x_host, out_host):
        """Host-buffer call (numpy arrays): H2D + kernel + D2H, synchronised."""
        _check(lib().lce_b200_bconv2d_run_host(
            self._h, x_host.ctypes.data_as(C.c_void_p), out_host.ctypes.data_as(C.c_void_p)))
        return out_host

    def close(self):
        if self._h:
            lib().lce_b200_bconv2d_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class BGemm:
    """Binary GEMM plan: out[M,N] = epilogue(sum_k popc(A[m,k] ^ W[n,k]))."""

    def __init__(self, W, out_type=OUT_RAW_ACC, clamp=(0, 2**31 - 1), multiplier=None,
                 bias=None, thresholds=None):
        import numpy as np
        self._h = C.c_void_p()
        self.out_type = out_type
        if isinstance(W, torch.Tensor):
            W = W.to(torch.int32).contiguous()
            wp = C.c_void_p(W.data_ptr())
        else:
            W = np.ascontiguousarray(W, np.int32)
            wp = W.ctypes.data_as(C.c_void_p)
        self.N, self.Kw = W.shape
        keep = [W]

        def hp(a, dt):
            if a is None:
                return None
            if isinstance(a, torch.Tensor):
                a = a.detach().cpu().numpy()
            a = np.ascontiguousarray(a, dt)
            keep.append(a)
            return a.ctypes.data_as(C.c_void_p)

        ep = BgemmEpilogue(out_type, clamp[0], clamp[1], hp(multiplier, np.float32),
                           hp(bias, np.float32), hp(thresholds, np.int32))
        _check(lib().lce_b200_bgemm_create(C.c_int(self.N), C.c_int(self.Kw), wp, C.byref(ep),
                                           C.byref(self._h)))

    def __call__(self, A: torch.Tensor, out: torch.Tensor | None = None):
        A = _dev(A, torch.int32)
        M = A.shape[0]
        if A.shape[1] != self.Kw:
            raise LceError("BGemm: K mismatch")
        if out is None:
            if self.out_type == OUT_BITPACKED:
                out = torch.empty((M, cdiv(self.N, 32)), dtype=torch.int32, device=A.device)
            else:
                dt = {OUT_FLOAT: torch.float32, OUT_INT8: torch.int8,
                      OUT_RAW_ACC: torch.int32}[self.out_type]
                out = torch.empty((M, self.N), dtype=dt, device=A.device)
        _check(lib().lce_b200_bgemm_run(self._h, C.c_int64(M), _p(A), _p(out), _stream()))
        return out

    def close(self):
        if self._h:
            lib().lce_b200_bgemm_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
