"""GPU tests of the float builtins' fused / tensor-core kernels through the C-ABI
(include/lce_b200_builtins.h): each must reproduce the plain kernels it replaces.

* lce_b200_f32_stem_conv_dw == DEQUANTIZE -> CONV_2D -> DEPTHWISE_CONV_2D run one after the other,
  bit for bit (same accumulation order), over paddings, odd sizes, several column tiles and the
  unaligned loader.
* the wgmma tf32 pointwise convolution (csrc/lce_b200_pw.cuh) against an fp64 product:
  |err| <= 2e-6 * sum|a||w| (the FMA kernels it replaces measure 2-4e-7, the 3-pass split 2-10e-7),
  and its fused LceQuantize words == the signs of its own float output.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PADDING_SAME, PADDING_VALID = 0, 1
T_FLOAT, T_INT8, T_UINT8 = 0, 1, 2


class ConvDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("batch", "in_h", "in_w", "in_c", "filter_h", "filter_w", "out_c",
                                         "stride_h", "stride_w", "dilation_h", "dilation_w", "padding",
                                         "activation")]


def _env():
    import torch
    from compute_engine_b200 import capi
    return torch, capi.lib()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _out_hw(lib, d):
    oh, ow = C.c_int(), C.c_int()
    assert lib.lce_b200_f32_conv_out_shape(C.byref(d), C.byref(oh), C.byref(ow)) == 0
    return oh.value, ow.value


@pytest.mark.parametrize("in_type", [T_FLOAT, T_INT8, T_UINT8])
@pytest.mark.parametrize("B,H,W,pad1,pad2,act1,act2", [
    (3, 224, 224, PADDING_SAME, PADDING_SAME, 1, 0),      # QuickNet's stem (aligned rows, one column tile)
    (2, 64, 64, PADDING_SAME, PADDING_SAME, 1, 0),
    (2, 100, 100, PADDING_SAME, PADDING_SAME, 0, 1),      # odd maps, unaligned int8 rows
    (1, 37, 53, PADDING_VALID, PADDING_SAME, 3, 0),
    (1, 75, 480, PADDING_SAME, PADDING_VALID, 1, 3),      # three column tiles
    (2, 19, 457, PADDING_VALID, PADDING_VALID, 0, 0),
])
def test_fused_stem_is_bit_identical_to_its_three_kernels(in_type, B, H, W, pad1, pad2, act1, act2):
    torch, lib = _env()
    g = torch.Generator(device="cpu").manual_seed(H * 1000 + W + in_type)
    if in_type == T_FLOAT:
        x = torch.randn(B, H, W, 3, generator=g).cuda()
        scale, zp = 1.0, 0
    elif in_type == T_INT8:
        x = torch.randint(-128, 128, (B, H, W, 3), generator=g, dtype=torch.int16).to(torch.int8).cuda()
        scale, zp = 4.0 / 127, -3
    else:
        x = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.int16).to(torch.uint8).cuda()
        scale, zp = 1.0 / 255, 117
    w1 = (torch.randn(16, 3, 3, 3, generator=g) * 0.4).cuda()
    b1 = torch.randn(16, generator=g).cuda()
    w2 = (torch.randn(1, 3, 3, 16, generator=g) * 0.4).cuda()
    b2 = torch.randn(16, generator=g).cuda()
    d1 = ConvDesc(B, H, W, 3, 3, 3, 16, 2, 2, 1, 1, pad1, act1)
    oh1, ow1 = _out_hw(lib, d1)
    d2 = ConvDesc(B, oh1, ow1, 16, 3, 3, 16, 2, 2, 1, 1, pad2, act2)
    oh2, ow2 = _out_hw(lib, d2)
    if oh2 < 1 or ow2 < 1:
        pytest.skip("empty output")
    st = None
    # the separate kernels
    if in_type == T_FLOAT:
        xf = x
    else:
        xf = torch.empty(B, H, W, 3, device="cuda")
        assert lib.lce_b200_dequantize_affine(in_type, _p(x), _p(xf), C.c_int64(x.numel()), C.c_double(scale),
                                              C.c_int32(zp), st) == 0
    y1 = torch.empty(B, oh1, ow1, 16, device="cuda")
    assert lib.lce_b200_f32_conv2d(C.byref(d1), _p(xf), _p(w1), _p(b1), _p(y1), st) == 0
    want = torch.empty(B, oh2, ow2, 16, device="cuda")
    assert lib.lce_b200_f32_depthwise_conv2d(C.byref(d2), _p(y1), _p(w2), _p(b2), _p(want), st) == 0
    # the fused kernel
    got = torch.full((B, oh2, ow2, 16), float("nan"), device="cuda")
    hw1, hb1, hw2, hb2 = (t.cpu().contiguous() for t in (w1, b1, w2, b2))     # the filters travel by value
    rc = lib.lce_b200_f32_stem_conv_dw(C.byref(d1), C.byref(d2), in_type, _p(x), C.c_double(scale), C.c_int32(zp),
                                       _p(hw1), _p(hb1), _p(hw2), _p(hb2), _p(got), st)
    assert rc == 0, lib.lce_b200_last_error().decode()
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))


def test_fused_stem_refuses_other_shapes():
    torch, lib = _env()
    x = torch.zeros(1, 32, 32, 4, device="cuda")
    w1 = torch.zeros(16, 3, 3, 4)
    w2 = torch.zeros(1, 3, 3, 16)
    out = torch.zeros(1, 8, 8, 16, device="cuda")
    d1 = ConvDesc(1, 32, 32, 4, 3, 3, 16, 2, 2, 1, 1, PADDING_SAME, 0)       # four input channels
    d2 = ConvDesc(1, 16, 16, 16, 3, 3, 16, 2, 2, 1, 1, PADDING_SAME, 0)
    rc = lib.lce_b200_f32_stem_conv_dw(C.byref(d1), C.byref(d2), T_FLOAT, _p(x), C.c_double(1.0), C.c_int32(0), _p(w1),
                                       None, _p(w2), None, _p(out), None)
    assert rc != 0 and b"unsupported shapes" in lib.lce_b200_last_error()


@pytest.mark.parametrize("M,K,N,act,with_packed", [
    (16384, 16, 64, 1, True),          # pixel pairs, W' = diag(W, W)
    (20002, 16, 64, 0, False),
    (8192 + 77, 64, 128, 0, True),     # weights resident, ragged last tile
    (9001, 128, 256, 1, True),         # weight ring, two column tiles
    (4999, 256, 512, 3, True),
    (8192, 96, 128, 2, False),
    (256, 512, 1000, 0, False),        # FULLY_CONNECTED's logits: ragged last column tile, two row tiles
    (1500, 64, 200, 1, False),
])
def test_tf32_pointwise_conv_matches_fp64_product(M, K, N, act, with_packed):
    torch, lib = _env()
    g = torch.Generator(device="cpu").manual_seed(M + K)
    A = (torch.randn(M, K, generator=g) * 1.5).cuda()
    Wt = (torch.randn(N, K, generator=g) * 0.3).cuda()
    b = torch.randn(N, generator=g).cuda()
    out = torch.empty(M, N, device="cuda")
    packed = torch.zeros(M, N // 32, dtype=torch.int32, device="cuda") if with_packed else None
    d = ConvDesc(1, 1, M, K, 1, 1, N, 1, 1, 1, 1, PADDING_VALID, act)
    if with_packed:
        rc = lib.lce_b200_f32_conv2d_packed(C.byref(d), _p(A), _p(Wt), _p(b), _p(out), _p(packed), None)
    else:
        rc = lib.lce_b200_f32_conv2d(C.byref(d), _p(A), _p(Wt), _p(b), _p(out), None)
    assert rc == 0, lib.lce_b200_last_error().decode()
    torch.cuda.synchronize()
    ref = A.double() @ Wt.double().t() + b.double()
    if act == 1:
        ref = ref.clamp(min=0)
    elif act == 2:
        ref = ref.clamp(-1, 1)
    elif act == 3:
        ref = ref.clamp(0, 6)
    mag = A.abs().double() @ Wt.abs().double().t() + b.abs().double()
    rel = ((out.double() - ref).abs() / mag).max().item()
    assert rel < 2e-6, rel
    if with_packed:
        bits = (out < 0).view(M, N // 32, 32).to(torch.int64)
        words = (bits << torch.arange(32, device="cuda")).sum(-1)
        words = torch.where(words >= 2**31, words - 2**32, words).to(torch.int32)
        assert torch.equal(words, packed)


@pytest.mark.parametrize("B,H,W,padding,act", [(8, 224, 224, PADDING_SAME, 0), (3, 101, 77, PADDING_SAME, 1),
                                              (5, 64, 64, PADDING_VALID, 3)])
def test_tf32_7x7_stem_matches_fp64_convolution(B, H, W, padding, act):
    """CONV_2D 7x7 / stride 2 / 3 -> 64 (Bi-RealNet's stem; csrc/lce_b200_pw.cuh stem7_tf32_kernel:
    per-thread im2col gather into the wgmma A registers, 3-pass tf32) against an fp64 convolution, same error bound
    as the pointwise kernel: 2e-6 * sum|a||w|."""
    torch, lib = _env()
    import torch.nn.functional as F
    g = torch.Generator(device="cpu").manual_seed(B * 7 + H)
    x = (torch.randn(B, H, W, 3, generator=g) * 1.5).cuda()
    w = (torch.randn(64, 7, 7, 3, generator=g) * 0.2).cuda()
    b = torch.randn(64, generator=g).cuda()
    d = ConvDesc(B, H, W, 3, 7, 7, 64, 2, 2, 1, 1, padding, act)
    oh, ow = _out_hw(lib, d)
    out = torch.full((B, oh, ow, 64), float("nan"), device="cuda")
    assert lib.lce_b200_f32_conv2d(C.byref(d), _p(x), _p(w), _p(b), _p(out), None) == 0, lib.lce_b200_last_error().decode()
    torch.cuda.synchronize()
    if padding == PADDING_SAME:     # TFLite SAME: total = (o - 1) * s + k - in, before = total // 2
        th, tw = max((oh - 1) * 2 + 7 - H, 0), max((ow - 1) * 2 + 7 - W, 0)
        pad = (tw // 2, tw - tw // 2, th // 2, th - th // 2)
    else:
        pad = (0, 0, 0, 0)

    def conv(xx, ww):
        xp = F.pad(xx.permute(0, 3, 1, 2), pad)
        return F.conv2d(xp, ww.permute(0, 3, 1, 2), stride=2).permute(0, 2, 3, 1)

    ref = conv(x.double(), w.double()) + b.double()
    mag = conv(x.abs().double(), w.abs().double()) + b.abs().double()
    if act == 1:
        ref = ref.clamp(min=0)
    elif act == 3:
        ref = ref.clamp(0, 6)
    assert ref.shape == out.shape
    rel = ((out.double() - ref).abs() / mag).max().item()
    assert rel < 2e-6, rel
