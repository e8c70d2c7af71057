"""Kernel-by-kernel tests of the float builtins (csrc/lce_b200_builtins.cu) through the C-ABI of
include/lce_b200_builtins.h, against exact references of the same arithmetic.

Every FMA convolution kernel (conv_direct16 in its three instances, gemm_small_m, conv_gemm128,
conv_igemm8x8, conv_igemm, conv_gemm) accumulates one fmaf chain from 0 over
k = (fy * KW + fx) * Cin + ci, padding taps contributing fma(0, w, acc), then adds the bias and
applies the activation. `fma32` emulates IEEE fmaf exactly in numpy, so the chain is reproduced bit
for bit; the depthwise kernels run the same chain over (fy, fx) with out-of-bounds taps skipped. Pools,
MEAN, the element-wise ops, DEQUANTIZE and PAD are exact in float32 / on the raw words. SOFTMAX (expf)
is held to a bound derived below.

Each GPU case also asserts, from a torch.profiler trace, that the kernel it is shaped for ran. The
variants chosen by LCE_B200_DIRECT_PX, LCE_B200_IGEMM_8X4 and LCE_B200_DIRECT_MAXK (read once per
process) run in a subprocess and must reproduce the default process's outputs bit for bit.

Not asserted: NaN propagation through the activations (fmaxf drops a NaN where TFLite's std::max
keeps it).
"""
import ctypes as C
import json
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

import lce_testlib as L
import tflite_ref as R
from compute_engine_b200.tflite_writer import TFLiteModel

SAME, VALID = L.PADDING_SAME, L.PADDING_VALID
NONE, RELU, N1, RELU6 = L.ACT_NONE, L.ACT_RELU, L.ACT_RELU_N1_TO_1, L.ACT_RELU6
U = 2.0 ** -24     # unit roundoff of float32


# ------------------------------- exact references ------------------------------- #
def fma32(a, b, c):
    """IEEE single-precision fma(a, b, c), elementwise. a * b is exact in float64 (24 + 24 bits);
    the float64 sum p + c is rounded to odd (TwoSum gives its exact error), which makes the final
    cast to float32 a single correct rounding. float32(p + c) alone would round twice."""
    p = np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32).astype(np.float64)
    c = np.asarray(c, np.float32).astype(np.float64)
    s = p + c
    bv = s - p
    err = (p - (s - bv)) + (c - bv)
    even = (s.view(np.uint64) & np.uint64(1)) == 0
    s = np.where((err != 0) & even, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def _act(x, act):
    x = np.asarray(x, np.float32)
    if act == RELU:
        return np.maximum(x, np.float32(0))
    if act == N1:
        return np.minimum(np.maximum(x, np.float32(-1)), np.float32(1))
    if act == RELU6:
        return np.minimum(np.maximum(x, np.float32(0)), np.float32(6))
    return x


def _geom(size, k, s, d, padding):
    eff = (k - 1) * d + 1
    out = -(-size // s) if padding == SAME else max((size + s - eff) // s, 0)
    return out, max((out - 1) * s + eff - size, 0) // 2


def _taps(x, oy, ox):
    """x[:, oy, ox, :] for index vectors oy [OH], ox [OW], 0 where out of bounds; and the mask."""
    H, W = x.shape[1:3]
    vy, vx = (oy >= 0) & (oy < H), (ox >= 0) & (ox < W)
    v = x[:, np.clip(oy, 0, H - 1)][:, :, np.clip(ox, 0, W - 1)]
    m = (vy[:, None] & vx[None, :])[None, :, :, None]
    return np.where(m, v, np.float32(0)), m


def conv_ref(x, w, bias, stride=(1, 1), dil=(1, 1), padding=SAME, act=NONE):
    """CONV_2D NHWC x [B,H,W,Cin], OHWI w [Cout,KH,KW,Cin]: the kernels' fmaf chain."""
    B, H, W, Cin = x.shape
    Cout, KH, KW, _ = w.shape
    OH, ph = _geom(H, KH, stride[0], dil[0], padding)
    OW, pw = _geom(W, KW, stride[1], dil[1], padding)
    acc = np.zeros((B, OH, OW, Cout), np.float32)
    for fy in range(KH):
        for fx in range(KW):
            v, _ = _taps(x, np.arange(OH) * stride[0] - ph + fy * dil[0], np.arange(OW) * stride[1] - pw + fx * dil[1])
            for ci in range(Cin):
                acc = fma32(v[..., ci:ci + 1], w[:, fy, fx, ci], acc)
    if bias is not None:
        acc = (acc + bias).astype(np.float32)
    return _act(acc, act)


def depthwise_ref(x, w, bias, stride=(1, 1), dil=(1, 1), padding=SAME, act=NONE):
    """DEPTHWISE_CONV_2D, filter [1,KH,KW,C]: one fmaf chain per output over the in-bounds taps."""
    B, H, W, Cc = x.shape
    _, KH, KW, _ = w.shape
    OH, ph = _geom(H, KH, stride[0], dil[0], padding)
    OW, pw = _geom(W, KW, stride[1], dil[1], padding)
    acc = np.zeros((B, OH, OW, Cc), np.float32)
    for fy in range(KH):
        for fx in range(KW):
            v, m = _taps(x, np.arange(OH) * stride[0] - ph + fy * dil[0], np.arange(OW) * stride[1] - pw + fx * dil[1])
            acc = np.where(m, fma32(v, w[0, fy, fx], acc), acc)
    if bias is not None:
        acc = (acc + bias).astype(np.float32)
    return _act(acc, act)


def pool_ref(x, f, stride, padding, act, is_max):
    """MAX: exact. AVERAGE (TFLite pooling.h): float32 sum over the in-bounds window in (y, x) order,
    divided by the float count of in-bounds elements."""
    B, H, W, Cc = x.shape
    OH, ph = _geom(H, f[0], stride[0], 1, padding)
    OW, pw = _geom(W, f[1], stride[1], 1, padding)
    v = np.full((B, OH, OW, Cc), np.float32(-np.finfo(np.float32).max) if is_max else np.float32(0))
    cnt = np.zeros((1, OH, OW, 1), np.float32)
    for fy in range(f[0]):
        for fx in range(f[1]):
            t, m = _taps(x, np.arange(OH) * stride[0] - ph + fy, np.arange(OW) * stride[1] - pw + fx)
            v = np.where(m, np.maximum(v, t) if is_max else (v + t).astype(np.float32), v)
            cnt = cnt + m
    if not is_max:
        v = (v / np.maximum(cnt, 1)).astype(np.float32)
    return _act(v, act)


def mean_ref(x, act=NONE):
    s = np.zeros((x.shape[0], x.shape[3]), np.float32)
    for p in _act(x, act).reshape(x.shape[0], -1, x.shape[3]).transpose(1, 0, 2):
        s = (s + p).astype(np.float32)
    return (s / np.float32(x.shape[1] * x.shape[2])).astype(np.float32)


def _round_f32(q):
    """The float32 nearest to the rational q (ties to even), subnormals included."""
    if q == 0:
        return 0.0
    sign, q = (-1 if q < 0 else 1), abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    while Fraction(2) ** e > q:
        e -= 1
    while Fraction(2) ** (e + 1) <= q:
        e += 1
    ulp = Fraction(2) ** (max(e, -126) - 23)
    m = q / ulp
    n = m.numerator // m.denominator
    r = m - n
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n % 2 == 1):
        n += 1
    return sign * float(n * ulp)


def _eq(got, want):
    """Equal values (+0 == -0); NaN (an unwritten output) never matches."""
    return got.shape == want.shape and bool(np.array_equal(got, want))


# ----------------------------------- CPU ----------------------------------- #
def _double_rounding_cases():
    """a * b + c = 2^E (1 + 2^-24) + 2^(E - 24 - 2k) with k >= 15: just above a float32 midpoint, but
    float64 rounds it onto the midpoint and float32 then ties to even, downwards."""
    out = []
    for E in (-60, -3, 0, 7, 40):
        for k in range(15, 22):
            for sgn in (1, -1):
                a = np.float32(sgn * 2.0 ** (E - 24) * (1 + 2.0 ** -k))
                b = np.float32(-(1 - 2.0 ** -k))
                c = np.float32(sgn * 2.0 ** E * (1 + 2.0 ** -23))
                out.append((a, b, c))
    return out


def test_fma32_is_a_single_rounding():
    rng = np.random.default_rng(0)
    n = 3000
    mant = lambda: rng.integers(1 << 23, 1 << 24, n).astype(np.float64) * rng.choice([-1, 1], n)
    a = (mant() * 2.0 ** rng.integers(-40, 10, n)).astype(np.float32)
    b = (mant() * 2.0 ** rng.integers(-40, 10, n)).astype(np.float32)
    c = (mant() * 2.0 ** rng.integers(-70, 20, n)).astype(np.float32)
    # midpoints: a * b is half an ulp of c, exactly (ties to even) or a few ulp of the product off
    e = rng.integers(-100, 100, n)
    cm = (mant() * 2.0 ** (e - 23)).astype(np.float32)             # |c| in [2^e, 2^(e+1))
    am = rng.choice([1.0, -1.0, 0.5, -0.5], n).astype(np.float32)
    bm = (2.0 ** (e - 24) / np.abs(am) * (1 + rng.integers(-3, 4, n) * 2.0 ** -23)).astype(np.float32)
    dr = np.array(_double_rounding_cases(), np.float32)
    a, b, c = (np.concatenate(v) for v in ((a, am, dr[:, 0]), (b, bm, dr[:, 1]), (c, cm, dr[:, 2])))
    got = fma32(a, b, c)
    want = np.array([_round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z)))
                     for x, y, z in zip(a, b, c)], np.float32)
    assert np.array_equal(got, want)
    naive = (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)
    tail = slice(len(a) - len(dr), None)
    assert not np.any(naive[tail] == want[tail])     # every constructed case defeats double rounding
    assert np.array_equal(got[tail], want[tail])


def test_round_f32_matches_numpy_on_doubles():
    rng = np.random.default_rng(1)
    x = rng.standard_normal(2000) * 2.0 ** rng.integers(-140, 60, 2000)   # subnormals included
    want = x.astype(np.float32)   # one rounding from a double: numpy is correct here
    assert np.array_equal(np.array([_round_f32(Fraction(float(v))) for v in x], np.float32), want)


def test_conv_and_pool_references_agree_with_torch():
    """The references' indexing (pads, strides, dilations, h != w) against tflite_ref's torch
    implementation, to float32 summation accuracy."""
    import torch
    import torch.nn.functional as F
    rng = np.random.default_rng(2)
    x = rng.standard_normal((2, 9, 7, 5)).astype(np.float32)
    w = rng.standard_normal((6, 3, 2, 5)).astype(np.float32)
    b = rng.standard_normal(6).astype(np.float32)
    for padding in (SAME, VALID):
        got = conv_ref(x, w, b, (2, 1), (1, 3), padding)
        OH, ph = _geom(9, 3, 2, 1, padding)
        OW, pw = _geom(7, 2, 1, 3, padding)
        th, tw = max((OH - 1) * 2 + 3 - 9, 0), max((OW - 1) * 1 + 4 - 7, 0)
        xt = F.pad(torch.from_numpy(x).double().permute(0, 3, 1, 2), (pw, tw - pw, ph, th - ph))
        want = F.conv2d(xt, torch.from_numpy(w).double().permute(0, 3, 1, 2), torch.from_numpy(b).double(),
                        (2, 1), 0, (1, 3)).permute(0, 2, 3, 1).numpy()
        assert got.shape == want.shape and np.allclose(got, want, rtol=1e-5, atol=1e-5)
        dw = depthwise_ref(x, w[:1, :, :, :5], None, (1, 2), (2, 1), padding)
        wd = torch.from_numpy(w[0, :, :, :5]).double().permute(2, 0, 1)[:, None]
        OH, ph = _geom(9, 3, 1, 2, padding)
        OW, pw = _geom(7, 2, 2, 1, padding)
        th, tw = max((OH - 1) + 5 - 9, 0), max((OW - 1) * 2 + 2 - 7, 0)
        xt = F.pad(torch.from_numpy(x).double().permute(0, 3, 1, 2), (pw, tw - pw, ph, th - ph))
        want = F.conv2d(xt, wd, None, (1, 2), 0, (2, 1), groups=5).permute(0, 2, 3, 1).numpy()
        assert dw.shape == want.shape and np.allclose(dw, want, rtol=1e-5, atol=1e-5)

    class _O:   # builtin options as tflite_ref reads them: padding, stride_w, stride_h, filter_w, filter_h, act
        def __init__(self, *v):
            self.v = v

        def scalar(self, i, fmt, default=0):
            return self.v[i]

    for is_max in (True, False):
        for f, s, padding in (((3, 2), (2, 1), SAME), ((2, 3), (3, 1), VALID), ((5, 4), (1, 1), SAME)):
            got = pool_ref(x, f, s, padding, NONE, is_max)
            want = R._pool(x, _O(padding, s[1], s[0], f[1], f[0], 0), is_max)
            assert got.shape == want.shape and np.allclose(got, want, rtol=1e-6, atol=1e-6)


# ----------------------------------- GPU ----------------------------------- #
class ConvDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("batch", "in_h", "in_w", "in_c", "filter_h", "filter_w", "out_c",
                                         "stride_h", "stride_w", "dilation_h", "dilation_w", "padding",
                                         "activation")]


class PoolDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("batch", "in_h", "in_w", "channels", "filter_h", "filter_w",
                                         "stride_h", "stride_w", "padding", "activation")]


def _lib():
    from compute_engine_b200 import capi
    return capi.lib()


def _err():
    return _lib().lce_b200_last_error().decode()


def _dev(a, off=0):
    """A device copy of `a` starting `off` elements past a 16-byte boundary."""
    import torch
    a = np.ascontiguousarray(a)
    t = torch.empty(a.size + off + 4, dtype=getattr(torch, a.dtype.name), device="cuda")
    v = t[off:off + a.size]
    v.copy_(torch.from_numpy(a.reshape(-1)))
    return v


def _out(n, off=0, dtype=np.float32):
    return _dev(np.full(n, np.nan, dtype) if dtype == np.float32 else np.zeros(n, dtype), off)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _profiled(fn, trace=True):
    """Run fn() under torch.profiler; returns fn's result and the names of the kernels it launched
    (whitespace removed). fn must be repeatable: on an H100 with torch 2.11 about one session in 40
    records no kernel at all, so an empty trace is retried twice, then it fails the test.
    Once another process has profiled, this process's sessions stay empty: the tests that start a
    profiling subprocess (test_env_selected_conv_variants_*) come last and do not trace here."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not trace:
        return fn(), None
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            r = fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        names |= {k.name for e in prof.events() for k in getattr(e, "kernels", [])}
        names = sorted("".join(n.split()) for n in names if n)
        if names:
            return r, names
    raise AssertionError("the profiler recorded no kernel")


def _assert_ran(names, kernel):
    k = "".join(kernel.split())
    assert any(k in n for n in names), (kernel, names)


# CONV_2D cases: (id, x shape, (Cout, KH, KW), stride, dilation, padding, act, bias, out offset,
# packed, the kernel of the default process, {env id: kernel there}). Comments name the path.
D16 = "conv_direct16_kernel<"
CONV = [
    # stem instance 3x3x3 (PX 2; PX 1 / 4 in the subprocess)
    ("stem_s2", (2, 37, 50, 3), (16, 3, 3), (2, 2), (1, 1), SAME, RELU, True, 0, False, D16 + "3,3,3,2,",
     {"px1": D16 + "3,3,3,1,", "px4": D16 + "3,3,3,4,", "nodirect": "conv_igemm8x8_kernel"}),
    ("stem_c24", (1, 20, 17, 3), (24, 3, 3), (1, 2), (2, 1), VALID, RELU6, True, 0, False, D16 + "3,3,3,2,",
     {"px1": D16 + "3,3,3,1,", "px4": D16 + "3,3,3,4,", "nodirect": "conv_igemm8x8_kernel"}),
    # pointwise-16 instance: tf32 declines K 16 unless Cout 64 with even pixels per image
    ("pw16_c64_odd_packed", (3, 9, 13, 16), (64, 1, 1), (1, 1), (1, 1), VALID, NONE, True, 0, True,
     D16 + "1,1,16,4,true>", {"px1": D16 + "1,1,16,1,", "px4": D16 + "1,1,16,4,true>",
                              "nodirect": "gemm_small_m_kernel"}),
    ("pw16_strided", (2, 15, 22, 16), (40, 1, 1), (2, 3), (1, 1), SAME, N1, True, 0, False, D16 + "1,1,16,4,true>",
     {"px1": D16 + "1,1,16,1,", "nodirect": "conv_igemm8x8_kernel"}),
    # generic instance, Cout not a multiple of 16 / 4, packed in the kernel (32, 64, 128) or after it (96)
    ("gen_5x5_c1", (2, 19, 26, 1), (20, 5, 5), (1, 2), (1, 1), SAME, RELU, True, 0, False, D16 + "0,0,0,4,",
     {"nodirect": "conv_igemm8x8_kernel"}),
    ("gen_1x1_s21", (2, 9, 7, 20), (40, 1, 1), (2, 1), (1, 1), VALID, NONE, False, 0, False, D16 + "0,0,0,4,",
     {"nodirect": "conv_igemm8x8_kernel"}),
    ("gen_c100", (1, 10, 13, 3), (100, 2, 2), (1, 1), (1, 1), SAME, RELU6, True, 0, False, D16 + "0,0,0,4,", {}),
    ("gen_packed32", (2, 11, 8, 5), (32, 3, 2), (1, 1), (2, 3), SAME, NONE, True, 0, True, D16 + "0,0,0,4,",
     {"nodirect": "conv_igemm8x8_kernel"}),
    ("gen_packed64", (1, 14, 9, 4), (64, 2, 3), (2, 1), (1, 1), SAME, NONE, True, 0, True, D16 + "0,0,0,4,", {}),
    ("gen_packed128", (2, 6, 11, 7), (128, 1, 1), (1, 1), (1, 1), VALID, NONE, True, 0, True, D16 + "0,0,0,4,",
     {"nodirect": "conv_igemm8x8_kernel"}),
    ("gen_packed96", (1, 12, 7, 6), (96, 4, 1), (1, 1), (1, 1), SAME, NONE, True, 0, True, D16 + "0,0,0,4,", {}),
    # plain GEMM (1x1, stride 1, K % 4 == 0, tf32 declines): fewer than 74 128x128 tiles -> gemm_small_m
    ("gemm_small", (1, 25, 41, 36), (50, 1, 1), (1, 1), (1, 1), VALID, RELU, True, 0, False, "gemm_small_m_kernel", {}),
    ("gemm_small_packed", (1, 5, 40, 64), (96, 1, 1), (1, 1), (1, 1), VALID, NONE, True, 0, True,
     "gemm_small_m_kernel", {}),
    ("gemm128_packed", (1, 1, 10007, 64), (96, 1, 1), (1, 1), (1, 1), VALID, NONE, True, 0, True,
     "conv_gemm128_kernel", {}),
    ("gemm128_n50", (12, 33, 30, 36), (50, 1, 1), (1, 1), (1, 1), SAME, RELU6, True, 0, False, "conv_gemm128_kernel", {}),
    # implicit GEMM: h != w everywhere, asymmetric SAME pads, images smaller than the dilated filter,
    # Cout % 4 != 0, several column tiles, an output 4 bytes off a 16-byte boundary (scalar stores)
    ("igemm_dil", (2, 13, 10, 8), (20, 3, 3), (2, 1), (1, 2), SAME, RELU, True, 0, False, "conv_igemm8x8_kernel",
     {"px1": "conv_igemm_kernel"}),
    ("igemm_5x3", (1, 9, 16, 4), (70, 5, 3), (1, 3), (1, 1), VALID, NONE, True, 0, False, "conv_igemm8x8_kernel",
     {"px1": "conv_igemm_kernel"}),
    ("igemm_tiny", (2, 4, 3, 6), (33, 3, 3), (1, 1), (3, 2), SAME, N1, True, 0, False, "conv_igemm8x8_kernel",
     {"px1": "conv_igemm_kernel"}),
    ("igemm_off4", (2, 12, 15, 4), (16, 3, 3), (2, 2), (1, 1), SAME, RELU6, True, 1, False, "conv_igemm8x8_kernel",
     {"px1": "conv_igemm_kernel"}),
    ("igemm_1x1_off4", (1, 7, 9, 40), (24, 1, 1), (1, 1), (1, 1), VALID, NONE, False, 1, False,
     "conv_igemm8x8_kernel", {"px1": "conv_igemm_kernel"}),
    ("igemm_wide", (3, 20, 23, 12), (200, 3, 3), (1, 1), (1, 1), SAME, RELU6, True, 0, False, "conv_igemm8x8_kernel",
     {"px1": "conv_igemm_kernel"}),
    # K > 4096
    ("gemm_k4608", (1, 6, 5, 512), (20, 3, 3), (1, 1), (1, 1), SAME, NONE, True, 0, False, "conv_gemm_kernel", {}),
    ("gemm_k4200", (2, 3, 7, 1400), (70, 1, 3), (1, 2), (1, 2), VALID, RELU, True, 0, False, "conv_gemm_kernel", {}),
]
CONV_IDS = [c[0] for c in CONV]
VARIANT_ENV = {"px1": {"LCE_B200_DIRECT_PX": "1", "LCE_B200_IGEMM_8X4": "1"},
               "px4": {"LCE_B200_DIRECT_PX": "4"},
               "nodirect": {"LCE_B200_DIRECT_MAXK": "0"}}


def _conv_inputs(case):
    cid, xs, (co, kh, kw) = case[:3]
    rng = np.random.default_rng(sum(map(ord, cid)))
    x = rng.standard_normal(xs).astype(np.float32)
    w = (rng.standard_normal((co, kh, kw, xs[3])) * 0.5).astype(np.float32)
    b = rng.standard_normal(co).astype(np.float32) if case[7] else None
    return x, w, b


def _run_conv(case, x=None, trace=True):
    """The case through lce_b200_f32_conv2d[_packed]: (float output, packed words or None), kernels."""
    cid, xs, (co, kh, kw), st, dil, pad, act, _, off, packed = case[:10]
    x0, w, b = _conv_inputs(case)
    x = x0 if x is None else x
    d = ConvDesc(x.shape[0], x.shape[1], x.shape[2], x.shape[3], kh, kw, co, st[0], st[1], dil[0], dil[1], pad, act)
    oh, ow = C.c_int(), C.c_int()
    assert _lib().lce_b200_f32_conv_out_shape(C.byref(d), C.byref(oh), C.byref(ow)) == 0
    shape = (x.shape[0], oh.value, ow.value, co)
    xd, wd, bd = _dev(x), _dev(w), (_dev(b) if b is not None else None)
    od = _out(int(np.prod(shape)), off)
    pk = _out(int(np.prod(shape[:3])) * -(-co // 32), 0, np.int32) if packed else None

    def go():
        if packed:
            return _lib().lce_b200_f32_conv2d_packed(C.byref(d), _p(xd), _p(wd), _p(bd), _p(od), _p(pk), None)
        return _lib().lce_b200_f32_conv2d(C.byref(d), _p(xd), _p(wd), _p(bd), _p(od), None)

    rc, names = _profiled(go, trace)
    assert rc == 0, _err()
    return (od.cpu().numpy().reshape(shape), None if pk is None else pk.cpu().numpy().reshape(shape[:3] + (-1,))), names


@pytest.mark.gpu
@pytest.mark.parametrize("case", CONV, ids=CONV_IDS)
def test_conv_kernel_matches_the_fmaf_chain(case):
    (got, packed), names = _run_conv(case)
    _assert_ran(names, case[10])
    x, w, b = _conv_inputs(case)
    want = conv_ref(x, w, b, case[3], case[4], case[5], case[6])
    assert _eq(got, want), (np.abs(got - want).max(), np.argwhere(got != want)[:5])
    if packed is not None:
        assert np.array_equal(packed, L.pack_signs(got))


@pytest.mark.gpu
def test_pointwise16_with_several_tiles_per_block():
    """1x1, 16 -> 48 channels over 400 867 pixels (an odd count): the tf32 kernel declines, and each
    block of conv_direct16<1,1,16,4,true> walks two pixel tiles. A strided sample of rows and the
    last rows are compared with the fmaf chain."""
    case = ("pw16_big", (1, 601, 667, 16), (48, 1, 1), (1, 1), (1, 1), VALID, RELU, True, 0, False)
    (got, _), names = _run_conv(case)
    _assert_ran(names, D16 + "1,1,16,4,true>")
    x, w, b = _conv_inputs(case)
    rows = np.concatenate([np.arange(0, 601 * 667, 257), np.arange(601 * 667 - 300, 601 * 667)])
    want = conv_ref(x.reshape(-1, 16)[rows][None, None], w, b, act=RELU)[0, 0]
    assert _eq(got.reshape(-1, 48)[rows], want)


@pytest.mark.gpu
def test_plain_gemm_image_result_does_not_depend_on_its_batch():
    """The same image alone (8 tiles: gemm_small_m) and in a batch of 80 (619 tiles: conv_gemm128)."""
    case = ("gemm_batch", (80, 33, 30, 36), (40, 1, 1), (1, 1), (1, 1), VALID, RELU, True, 0, False)
    x, w, b = _conv_inputs(case)
    (batch, _), n1 = _run_conv(case, x)
    (alone, _), n2 = _run_conv(case, x[:1])
    _assert_ran(n1, "conv_gemm128_kernel")
    _assert_ran(n2, "gemm_small_m_kernel")
    assert np.array_equal(batch[:1].view(np.uint32), alone.view(np.uint32))
    assert _eq(alone, conv_ref(x[:1], w, b, act=RELU))


# DEPTHWISE_CONV_2D: (id, x shape, (KH, KW), stride, dilation, padding, act, bias, pointer offsets
# (in, filter, bias, out), kernel)
DW = [
    ("v4_3x3", (2, 13, 18, 24), (3, 3), (2, 1), (1, 1), SAME, RELU, True, (0, 0, 0, 0), "depthwise_v4_kernel<3>"),
    ("v4_3x3_dil", (1, 11, 9, 8), (3, 3), (1, 1), (2, 1), VALID, RELU6, False, (0, 0, 0, 0), "depthwise_v4_kernel<3>"),
    ("v4_5x3", (2, 7, 11, 12), (5, 3), (1, 2), (1, 1), SAME, N1, True, (0, 0, 0, 0), "depthwise_v4_kernel<0>"),
    ("v4_2x2_s3", (1, 14, 10, 16), (2, 2), (3, 3), (1, 1), VALID, NONE, True, (0, 0, 0, 0), "depthwise_v4_kernel<0>"),
    ("v4_borders", (2, 3, 2, 4), (5, 4), (1, 1), (1, 1), SAME, RELU, True, (0, 0, 0, 0), "depthwise_v4_kernel<0>"),
    ("c10", (2, 9, 6, 10), (3, 3), (1, 1), (1, 1), SAME, NONE, True, (0, 0, 0, 0), "depthwise_kernel"),
    ("c7_borders", (1, 3, 2, 7), (5, 4), (2, 1), (1, 1), SAME, RELU6, True, (0, 0, 0, 0), "depthwise_kernel"),
    ("out_off4", (2, 10, 12, 16), (3, 3), (2, 2), (1, 1), SAME, RELU, True, (0, 0, 0, 1), "depthwise_kernel"),
    ("in_off4", (1, 8, 5, 8), (2, 3), (1, 2), (1, 1), VALID, N1, True, (1, 0, 0, 0), "depthwise_kernel"),
    ("bias_off4", (1, 6, 7, 12), (3, 1), (1, 1), (2, 1), SAME, NONE, True, (0, 0, 1, 0), "depthwise_kernel"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", DW, ids=[c[0] for c in DW])
def test_depthwise_kernel_matches_the_fmaf_chain(case):
    cid, xs, (kh, kw), st, dil, pad, act, has_b, offs, kernel = case
    rng = np.random.default_rng(sum(map(ord, cid)))
    x = rng.standard_normal(xs).astype(np.float32)
    w = rng.standard_normal((1, kh, kw, xs[3])).astype(np.float32)
    b = rng.standard_normal(xs[3]).astype(np.float32) if has_b else None
    want = depthwise_ref(x, w, b, st, dil, pad, act)
    d = ConvDesc(*xs, kh, kw, xs[3], st[0], st[1], dil[0], dil[1], pad, act)
    xd, wd, bd = _dev(x, offs[0]), _dev(w, offs[1]), (_dev(b, offs[2]) if has_b else None)
    od = _out(want.size, offs[3])
    rc, names = _profiled(lambda: _lib().lce_b200_f32_depthwise_conv2d(C.byref(d), _p(xd), _p(wd), _p(bd), _p(od), None))
    assert rc == 0, _err()
    _assert_ran(names, kernel)
    assert _eq(od.cpu().numpy().reshape(want.shape), want)


# pools: (id, is_max, x shape, filter, stride, padding, act, pointer offset, kernel)
POOL = [
    ("max2", True, (2, 9, 12, 8), (2, 2), (2, 2), VALID, NONE, 0, "pool_v4_kernel<true,2>"),
    ("max2_s3", True, (1, 11, 14, 12), (2, 2), (3, 3), VALID, RELU, 0, "pool_v4_kernel<true,2>"),
    ("max3", True, (2, 13, 10, 16), (3, 3), (2, 2), SAME, RELU, 0, "pool_v4_kernel<true,3>"),
    ("max2x3", True, (1, 7, 9, 4), (2, 3), (1, 2), SAME, N1, 0, "pool_v4_kernel<true,0>"),
    ("max1x2_s3", True, (2, 8, 10, 8), (1, 2), (3, 3), VALID, RELU6, 0, "pool_v4_kernel<true,0>"),
    ("max_borders", True, (1, 3, 2, 4), (5, 4), (1, 1), SAME, NONE, 0, "pool_v4_kernel<true,0>"),
    ("avg2", False, (2, 9, 12, 8), (2, 2), (2, 2), SAME, NONE, 0, "pool_v4_kernel<false,2>"),
    ("avg3", False, (2, 13, 10, 16), (3, 3), (2, 1), SAME, RELU, 0, "pool_v4_kernel<false,3>"),
    ("avg3x2_s4", False, (1, 10, 9, 4), (3, 2), (4, 3), VALID, N1, 0, "pool_v4_kernel<false,0>"),
    ("avg_borders", False, (2, 3, 2, 8), (5, 4), (1, 1), SAME, RELU6, 0, "pool_v4_kernel<false,0>"),
    ("max_c6", True, (2, 7, 8, 6), (3, 2), (2, 1), SAME, RELU, 0, "pool_kernel<true>"),
    ("max_off4", True, (1, 9, 6, 8), (2, 2), (1, 2), SAME, N1, 1, "pool_kernel<true>"),
    ("avg_c5", False, (2, 3, 2, 5), (5, 4), (1, 1), SAME, NONE, 0, "pool_kernel<false>"),
    ("avg_off4", False, (1, 8, 11, 12), (3, 3), (3, 2), SAME, RELU6, 1, "pool_kernel<false>"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", POOL, ids=[c[0] for c in POOL])
def test_pool_kernel_is_exact(case):
    cid, is_max, xs, f, st, pad, act, off, kernel = case
    x = (np.random.default_rng(sum(map(ord, cid))).standard_normal(xs) * 3).astype(np.float32)
    want = pool_ref(x, f, st, pad, act, is_max)
    d = PoolDesc(*xs, f[0], f[1], st[0], st[1], pad, act)
    xd, od = _dev(x, off), _out(want.size, off)
    fn = _lib().lce_b200_f32_max_pool if is_max else _lib().lce_b200_f32_avg_pool
    rc, names = _profiled(lambda: fn(C.byref(d), _p(xd), _p(od), None))
    assert rc == 0, _err()
    _assert_ran(names, kernel)
    assert np.array_equal(od.cpu().numpy().reshape(want.shape).view(np.uint32), want.view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("xs,stride,pad,act", [
    ((2, 4, 4, 8), (1, 1), SAME, RELU),        # pooled 3x3: every window is on a border
    ((1, 3, 9, 4), (2, 2), SAME, NONE),        # PH = 2
    ((2, 9, 4, 12), (1, 1), VALID, RELU6),     # PW = 3
    ((2, 21, 70, 8), (1, 1), SAME, N1),        # warps partly interior, partly border
    ((1, 30, 43, 4), (2, 2), SAME, RELU),
    ((1, 17, 120, 16), (2, 1), VALID, NONE),
])
def test_fused_maxpool_depthwise_is_pool_then_depthwise(xs, stride, pad, act):
    rng = np.random.default_rng(xs[1] * 100 + xs[2])
    x = rng.standard_normal(xs).astype(np.float32)
    w = rng.standard_normal((1, 3, 3, xs[3])).astype(np.float32)
    b = rng.standard_normal(xs[3]).astype(np.float32)
    pooled = pool_ref(x, (2, 2), (1, 1), VALID, NONE, True)
    want = depthwise_ref(pooled, w, b, stride, (1, 1), pad, act)
    pd = PoolDesc(*xs, 2, 2, 1, 1, VALID, NONE)
    dd = ConvDesc(xs[0], pooled.shape[1], pooled.shape[2], xs[3], 3, 3, xs[3], stride[0], stride[1], 1, 1, pad, act)
    xd, wd, bd, od = _dev(x), _dev(w), _dev(b), _out(want.size)
    rc, names = _profiled(lambda: _lib().lce_b200_f32_maxpool2x2_depthwise3x3(
        C.byref(pd), C.byref(dd), _p(xd), _p(wd), _p(bd), _p(od), None))
    assert rc == 0, _err()
    _assert_ran(names, "pool2_dw3_v4_kernel")
    assert _eq(od.cpu().numpy().reshape(want.shape), want)


@pytest.mark.gpu
@pytest.mark.parametrize("xs,act", [((3, 7, 9, 13), NONE), ((2, 1, 1, 1000), NONE), ((4, 5, 6, 64), RELU),
                                    ((1, 14, 3, 7), RELU6)])
def test_mean_is_a_sequential_float_sum(xs, act):
    x = (np.random.default_rng(xs[3]).standard_normal(xs) * 2).astype(np.float32)
    want = mean_ref(x, act)
    xd, od = _dev(x), _out(want.size)
    if act == NONE:
        fn = lambda: _lib().lce_b200_f32_mean_hw(_p(xd), _p(od), *xs, None)
    else:
        fn = lambda: _lib().lce_b200_f32_mean_hw_act(_p(xd), _p(od), *xs, act, None)
    rc, names = _profiled(fn)
    assert rc == 0, _err()
    _assert_ran(names, "mean_hw_kernel")
    assert np.array_equal(od.cpu().numpy().reshape(want.shape).view(np.uint32), want.view(np.uint32))


# element-wise: (op, n, b_len, act, pointer offset of a); vector path = b_len == n, n % 4 == 0, aligned
ELT = [(op, n, bl, act, off) for op in ("add", "mul") for (n, bl, act, off) in (
    (3 * 4096, 3 * 4096, NONE, 0),       # vector
    (2 * 5 * 7 * 24, 24, RELU, 0),       # per channel
    (1001, 1001, N1, 0),                 # n % 4 != 0
    (4096, 4096, RELU6, 1),              # unaligned a
    (6 * 13, 13, RELU6, 0))] + [("act", n, n, act, off) for act in (NONE, RELU, N1, RELU6)
                                for (n, off) in ((8192, 0), (1003, 0), (4096, 1))]


@pytest.mark.gpu
@pytest.mark.parametrize("op,n,b_len,act,off", ELT)
def test_eltwise_is_float32_exact(op, n, b_len, act, off):
    rng = np.random.default_rng(n + act)
    a = (rng.standard_normal(n) * 3).astype(np.float32)
    b = (rng.standard_normal(b_len) * 3).astype(np.float32)
    bb = np.tile(b, n // b_len)
    want = _act(a + bb if op == "add" else a * bb if op == "mul" else a, act)
    ad, bd, od = _dev(a, off), _dev(b), _out(n)
    lib = _lib()
    if op == "act":
        fn = lambda: lib.lce_b200_f32_activation(_p(ad), _p(od), C.c_int64(n), act, None)
    else:
        f = lib.lce_b200_f32_add if op == "add" else lib.lce_b200_f32_mul
        fn = lambda: f(_p(ad), _p(bd), _p(od), C.c_int64(n), C.c_int64(b_len), act, None)
    rc, names = _profiled(fn)
    assert rc == 0, _err()
    _assert_ran(names, "eltwise_kernel<%d>" % {"add": 0, "mul": 1, "act": 2}[op])
    assert _eq(od.cpu().numpy(), want)


@pytest.mark.gpu
@pytest.mark.parametrize("qtype,n,scale,zp", [(L.T_INT8, 16 * 300 + 7, 0.037, -5), (L.T_INT8, 5, 1.0 / 127, 0),
                                              (L.T_BOOL, 9_000_003, 1.0 / 255, 117), (L.T_BOOL, 16 * 64, 0.5, 255)])
def test_dequantize_is_exact(qtype, n, scale, zp):
    rng = np.random.default_rng(n)
    dt = np.int8 if qtype == L.T_INT8 else np.uint8
    q = rng.integers(np.iinfo(dt).min, np.iinfo(dt).max + 1, n).astype(dt)
    want = (np.float64(scale) * (q.astype(np.int64) - zp).astype(np.float64)).astype(np.float32)
    qd, od = _dev(q), _out(n)
    rc, names = _profiled(lambda: _lib().lce_b200_dequantize_affine(qtype, _p(qd), _p(od), C.c_int64(n),
                                                                     C.c_double(scale), C.c_int32(zp), None))
    assert rc == 0, _err()
    _assert_ran(names, "dequantize_affine_kernel")
    assert np.array_equal(od.cpu().numpy().view(np.uint32), want.view(np.uint32))


@pytest.mark.gpu
def test_dequantize_refuses_unaligned_buffers():
    q, od = _dev(np.zeros(64, np.int8), 1), _out(64)
    assert _lib().lce_b200_dequantize_affine(L.T_INT8, _p(q), _p(od), C.c_int64(63), C.c_double(1.0),
                                             C.c_int32(0), None) != 0
    assert "dequantize: buffers must be 16-byte aligned" in _err()


@pytest.mark.gpu
@pytest.mark.parametrize("fill", [0x80000000, 0x7FC01234, 0xFFFFFFFF])
def test_pad4d_copies_words_and_fills(fill):
    dims, before, after = (2, 3, 5, 7), (0, 1, 2, 0), (1, 0, 1, 3)
    x = np.random.default_rng(fill & 0xFFFF).integers(0, 2**32, dims, dtype=np.uint64).astype(np.uint32)
    want = np.pad(x, list(zip(before, after)), constant_values=np.uint32(fill))
    xd, od = _dev(x.view(np.int32)), _out(want.size, 0, np.int32)
    arr = lambda v: (C.c_int32 * 4)(*v)
    rc, names = _profiled(lambda: _lib().lce_b200_pad4d_32(_p(xd), _p(od), arr(dims), arr(before), arr(after),
                                                           C.c_uint32(fill), None))
    assert rc == 0, _err()
    _assert_ran(names, "pad4d32_kernel")
    assert np.array_equal(od.cpu().numpy().view(np.uint32).reshape(want.shape), want)


@pytest.mark.gpu
@pytest.mark.parametrize("beta", [0.5, 2.0])
@pytest.mark.parametrize("cols", [1, 127, 128, 1000, 1024, 1025, 4099])
def test_softmax_within_its_derived_bound(cols, beta):
    """Against an fp64 softmax of the float32 input. The kernel's max m is exact. For element j:
    * t_j = float(x_j - m) * beta (beta a power of two: exact) is off by at most u|t_j|, so
      exp(t_j) by a factor within (1 +- u|t_j|) (first order);
    * expf: at most 2 ulp <= 4u relative (a normal result), 2^-148 absolute below 2^-126;
    * the sum S of positive terms over a depth d = ceil(cols / 128) (per thread, sequential from 0)
      + 5 (warp butterfly) + 2 (four warps) has relative error <= gamma_d = d u / (1 - d u), on top of
      its terms' own errors, which are at most u * sum_i p_i |t_i| + 4u relative in total;
    * the division rounds once: u.
    So |y_j - p_j| <= p_j (u |t_j| + 4u + u sum_i p_i |t_i| + 4u + gamma_d + u)(1 + 1e-3) + 2^-147, the
    last factor covering second-order terms and the absolute term a result below the normal range."""
    rows = 5
    x = np.random.default_rng(cols).uniform(-80, 80, (rows, cols)).astype(np.float32)
    xd, od = _dev(x), _out(x.size)
    rc, names = _profiled(lambda: _lib().lce_b200_f32_softmax(_p(xd), _p(od), C.c_int64(rows), cols,
                                                              C.c_float(beta), None))
    assert rc == 0, _err()
    _assert_ran(names, "softmax_kernel")
    got = od.cpu().numpy().reshape(rows, cols).astype(np.float64)
    t = (x.astype(np.float64) - x.max(1, keepdims=True)) * beta
    p = np.exp(t) / np.exp(t).sum(1, keepdims=True)
    d = -(-cols // 128) + 7
    gamma = d * U / (1 - d * U)
    rel = (U * np.abs(t) + 4 * U + U * (p * np.abs(t)).sum(1, keepdims=True) + 4 * U + gamma + U) * (1 + 1e-3)
    bound = p * rel + 2.0 ** -147
    assert np.all(np.abs(got - p) <= bound), (np.abs(got - p) / bound).max()


# ------------------- builtin options -> descriptors on the graph host ------------------- #
def _single_op(kind, x_shape, consts, out_shape, **opts):
    m = TFLiteModel()
    x = m.add_tensor("x", x_shape)
    ins = [x] + [m.add_tensor(f"c{i}", None, v.dtype, data=v) if v is not None else -1 for i, v in enumerate(consts)]
    y = m.add_tensor("y", out_shape)
    m.add_op(kind, ins, [y], **opts)
    m.inputs, m.outputs = [x], [y]
    return m.serialize()


def _run_graph(blob, x):
    from compute_engine_b200 import host as H
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    out = g.read(g.outputs()[0])
    g.close()
    ref = R.run(R.parse(blob), [x])[0][0]
    assert out.shape == ref.shape
    return out, ref


@pytest.mark.gpu
def test_graph_options_reach_the_kernels():
    """One single-op graph per builtin, every h / w pair different: the device result equals the exact
    reference built from the intended parameters, and tflite_ref's reading of the same flatbuffer."""
    rng = np.random.default_rng(7)
    x = rng.standard_normal((2, 11, 8, 5)).astype(np.float32)
    w = (rng.standard_normal((7, 3, 2, 5)) * 0.5).astype(np.float32)
    b = rng.standard_normal(7).astype(np.float32)
    want = conv_ref(x, w, b, (2, 1), (1, 2), SAME, RELU)
    got, ref = _run_graph(_single_op("CONV_2D", x.shape, [w, b], want.shape, padding="SAME", stride=(2, 1),
                                     dilation=(1, 2), activation="RELU"), x)
    assert _eq(got, want) and np.allclose(got, ref, rtol=1e-5, atol=1e-5)

    x = rng.standard_normal((2, 9, 12, 8)).astype(np.float32)
    w = rng.standard_normal((1, 3, 2, 8)).astype(np.float32)
    want = depthwise_ref(x, w, b[:1].repeat(8), (1, 2), (2, 1), SAME, RELU6)
    got, ref = _run_graph(_single_op("DEPTHWISE_CONV_2D", x.shape, [w, b[:1].repeat(8)], want.shape, padding="SAME",
                                     stride=(1, 2), dilation=(2, 1), activation="RELU6"), x)
    assert _eq(got, want) and np.allclose(got, ref, rtol=1e-5, atol=1e-5)

    x = rng.standard_normal((2, 9, 7, 4)).astype(np.float32)
    for kind, is_max, f, st in (("MAX_POOL_2D", True, (3, 2), (2, 1)), ("AVERAGE_POOL_2D", False, (2, 3), (1, 2))):
        want = pool_ref(x, f, st, SAME, NONE, is_max)
        got, ref = _run_graph(_single_op(kind, x.shape, [], want.shape, padding="SAME", stride=st, filter=f), x)
        assert _eq(got, want) and np.allclose(got, ref, rtol=1e-6, atol=1e-6), kind

    x = rng.standard_normal((2, 5, 7, 6)).astype(np.float32)
    want = mean_ref(x).reshape(2, 1, 1, 6)
    got, ref = _run_graph(_single_op("MEAN", x.shape, [np.array([1, 2], np.int32)], want.shape, keep_dims=True), x)
    assert got.shape == (2, 1, 1, 6) and _eq(got, want) and np.allclose(got, ref, rtol=1e-6, atol=1e-7)

    x = rng.uniform(-8, 8, (3, 37)).astype(np.float32)
    got, ref = _run_graph(_single_op("SOFTMAX", x.shape, [], x.shape, beta=0.5), x)
    want = np.exp(0.5 * (x - x.max(1, keepdims=True)).astype(np.float64))
    assert np.allclose(got, want / want.sum(1, keepdims=True), rtol=1e-5, atol=0) and np.allclose(got, ref, rtol=1e-5)

    x = rng.standard_normal((2, 3, 4, 5)).astype(np.float32)
    w = (rng.standard_normal((10, 60)) * 0.5).astype(np.float32)
    want = conv_ref(x.reshape(2, 1, 1, 60), w.reshape(10, 1, 1, 60), b[:1].repeat(10), act=RELU6).reshape(2, 10)
    got, ref = _run_graph(_single_op("FULLY_CONNECTED", x.shape, [w, b[:1].repeat(10)], (2, 10), activation="RELU6"), x)
    assert _eq(got, want) and np.allclose(got, ref, rtol=1e-5, atol=1e-5)


# ------------- env-selected variants (last: their subprocess ends tracing here) ------------- #
def _variant_outputs(cases, trace):
    outs, ran = {}, {}
    for case in cases:
        (o, pk), names = _run_conv(case, trace=trace)
        outs[case[0]] = o
        if pk is not None:
            outs[case[0] + ":packed"] = pk
        ran[case[0]] = names
    return outs, ran


def _dump_variant(outdir, env_id):
    """Subprocess side of test_env_selected_conv_variants_are_bit_identical."""
    outs, ran = _variant_outputs([c for c in CONV if env_id in c[11]], True)
    np.savez(os.path.join(outdir, "outs.npz"), **outs)
    with open(os.path.join(outdir, "ran.json"), "w") as f:
        json.dump(ran, f)


@pytest.mark.gpu
@pytest.mark.parametrize("env_id", sorted(VARIANT_ENV))
def test_env_selected_conv_variants_are_bit_identical(env_id, tmp_path):
    """The env variables are read once per process: the variant runs in a subprocess, which reports
    its outputs and kernels; this process computes the same cases on the default kernels."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, **VARIANT_ENV[env_id])
    code = (f"import sys; sys.path[:0] = [{here!r}, {os.path.dirname(here)!r}]\n"
            f"import test_gpu_float_kernels as T\nT._dump_variant({str(tmp_path)!r}, {env_id!r})\n")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    cases = [c for c in CONV if env_id in c[11]]
    want, _ = _variant_outputs(cases, False)
    got = dict(np.load(tmp_path / "outs.npz"))
    with open(tmp_path / "ran.json") as f:
        ran = json.load(f)
    assert sorted(got) == sorted(want)
    for case in cases:
        _assert_ran(ran[case[0]], case[11][env_id])
    for k in want:
        assert np.array_equal(got[k].view(np.uint32), want[k].view(np.uint32)), k
