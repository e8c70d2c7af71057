"""pw_tf32_kernel's output goes through shared memory and TMA stores (lce_b200_pw.cuh): each math
warpgroup stages its 64 x 128 results as four 32-column SWIZZLE_128B boxes, and the tensor map
clips rows past M and columns past N. CONV_2D+LceQuantize (lce_b200_f32_conv2d_packed) must give
the bits of CONV_2D (lce_b200_f32_conv2d) followed by LceQuantize (lce_b200_quantize), write
nothing past its outputs, and stay within the tf32 bound of an fp64 product.

Cases: QuickNet's four pointwise layers at batch 256 (the 16 -> 64 layer as pixel pairs; each CTA
runs many items), a 1x1 image (one row: the second warpgroup's rows are all outside the tensor),
pixel counts that leave a partial last row tile, batch 7, and column counts that end inside a
32-column box (100) or before the last box (96) of a 128-column tile, and past one tile (1000).
"""
import ctypes as C

import pytest

from test_gpu_float_kernels import ConvDesc, _err, _lib, _p
from test_gpu_float_scale import (NONE, RELU, RELU6, N1, VALID, assert_fp64_bound, guarded_in, guarded_out,
                                  same_bits)

BAND = 128 * 512      # poison past the end of every buffer: one tile of the widest rows here

# (id, batch, H, W, K, N, act, packed)
CASES = [
    ("quicknet_16-64", 256, 56, 56, 16, 64, NONE, True),
    ("quicknet_64-128", 256, 28, 28, 64, 128, NONE, True),
    ("quicknet_128-256", 256, 14, 14, 128, 256, NONE, True),
    ("quicknet_256-512", 256, 7, 7, 256, 512, NONE, True),
    ("one_pixel_64-128", 1, 1, 1, 64, 128, RELU, True),
    ("one_pixel_pairs_16-64", 1, 1, 2, 16, 64, NONE, True),
    ("batch7_5x5_128-256", 7, 5, 5, 128, 256, N1, True),
    ("batch7_pairs_9x10_16-64", 7, 9, 10, 16, 64, RELU6, True),
    ("partial_tile_13x13_64-128", 3, 13, 13, 64, 128, NONE, True),
    ("cols_100", 5, 11, 11, 64, 100, RELU, False),
    ("cols_96", 2, 9, 9, 32, 96, NONE, False),
    ("cols_1000", 300, 1, 1, 512, 1000, NONE, False),
]


def _run(case):
    import torch
    cid, B, H, W, K, N, act, packed = case
    M = B * H * W
    g = torch.Generator(device="cuda").manual_seed(sum(map(ord, cid)))
    A = torch.randn((M, K), device="cuda", generator=g) * 1.5
    Wt = torch.randn((N, K), device="cuda", generator=g) * 0.3
    b = torch.randn(N, device="cuda", generator=g)
    a, w, bias = (guarded_in(t, BAND) for t in (A, Wt, b))
    d = ConvDesc(B, H, W, K, 1, 1, N, 1, 1, 1, 1, VALID, act)
    plain = guarded_out((M, N), BAND)
    assert _lib().lce_b200_f32_conv2d(C.byref(d), _p(a.t), _p(w.t), _p(bias.t), _p(plain.t), None) == 0, _err()
    outs = [plain]
    if packed:
        fused, pk = guarded_out((M, N), BAND), guarded_out((M, N // 32), BAND, torch.int32)
        assert _lib().lce_b200_f32_conv2d_packed(C.byref(d), _p(a.t), _p(w.t), _p(bias.t), _p(fused.t),
                                                 _p(pk.t), None) == 0, _err()
        outs += [fused, pk]
    torch.cuda.synchronize()
    for gb in [a, w, bias] + outs:
        gb.assert_band(cid)
    plain.assert_written(cid)
    if packed:
        fused.assert_written(cid)
    return A, Wt, b, outs


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv2d_quantize_is_conv2d_then_lce_quantize(case):
    from compute_engine_b200 import capi
    A, Wt, b, outs = _run(case)
    plain = outs[0].t
    assert_fp64_bound(plain, A, Wt, b, case[6], case[0])
    if len(outs) > 1:
        fused, pk = outs[1].t, outs[2].t
        assert same_bits(fused, plain), f"{case[0]}: CONV_2D+LceQuantize's floats differ from CONV_2D's"
        assert pk.equal(capi.quantize(plain)), f"{case[0]}: signs differ from LceQuantize of CONV_2D"
