"""QuickNet-style transitions, MAX_POOL_2D 2x2 s1 VALID then the 3x3 blur depthwise, through
lce_b200_f32_maxpool2x2_depthwise3x3 (pool2_dw3_v4_kernel) at the shapes of every model that has
them and at awkward sizes: the result must be the bits of MAX_POOL_2D (lce_b200_f32_max_pool)
followed by DEPTHWISE_CONV_2D (lce_b200_f32_depthwise_conv2d), nothing may be written past the
output and nothing left unwritten.

Cases: QuickNet's three transitions at batch 256 (QuickNetLarge has the same shapes at batch 128),
QuickNetSmall's three at batch 256, a 2x2 input (one pooled pixel, one output), widths whose
output rows end inside a 256-thread block, batch 7, channel counts that are not a multiple of 16
(12 and 40), a stride-1 and a VALID blur, and a tall image of many output rows.
"""
import ctypes as C

import numpy as np
import pytest

from test_gpu_float_kernels import ConvDesc, PoolDesc, _eq, _err, _lib, _p, depthwise_ref, pool_ref
from test_gpu_float_scale import NONE, RELU, RELU6, N1, SAME, VALID, POS_INF, cdiv, guarded_in, guarded_out, same_bits

BAND = 128 * 64 * 64   # poison past the end of every buffer

# (id, batch, H, W, C, stride, padding, act)
CASES = [
    ("quicknet_56x56x64", 256, 56, 56, 64, 2, SAME, NONE),
    ("quicknet_28x28x128", 256, 28, 28, 128, 2, SAME, NONE),
    ("quicknet_14x14x256", 256, 14, 14, 256, 2, SAME, NONE),
    ("quicknet_small_56x56x32", 256, 56, 56, 32, 2, SAME, NONE),
    ("quicknet_small_28x28x64", 256, 28, 28, 64, 2, SAME, NONE),
    ("quicknet_small_14x14x256", 256, 14, 14, 256, 2, SAME, NONE),
    ("one_output_2x2x64", 3, 2, 2, 64, 2, SAME, RELU),
    ("partial_tiles_37x41x64", 7, 37, 41, 64, 2, SAME, N1),
    ("batch7_19x23x128", 7, 19, 23, 128, 2, SAME, NONE),
    ("c12_30x30", 5, 30, 30, 12, 2, SAME, RELU6),
    ("c40_17x26", 4, 17, 26, 40, 2, SAME, NONE),
    ("stride1_20x33x16", 3, 20, 33, 16, 1, SAME, RELU),
    ("valid_25x18x32", 2, 25, 18, 32, 2, VALID, NONE),
    ("tall_300x9x8", 2, 300, 9, 8, 1, VALID, N1),
]


def _launch(case):
    import torch
    cid, B, H, W, c, s, pad, act = case
    g = torch.Generator(device="cuda").manual_seed(sum(map(ord, cid)))
    x = torch.randn((B, H, W, c), device="cuda", generator=g) * 3
    w = torch.randn((1, 3, 3, c), device="cuda", generator=g)
    bias = torch.randn(c, device="cuda", generator=g)
    ph = H - 1
    pwid = W - 1
    oh, ow = (cdiv(ph, s), cdiv(pwid, s)) if pad == SAME else ((ph - 3) // s + 1, (pwid - 3) // s + 1)
    xg = guarded_in(x, BAND, POS_INF)
    wg, bg = guarded_in(w, BAND), guarded_in(bias, BAND)
    pd = PoolDesc(B, H, W, c, 2, 2, 1, 1, VALID, NONE)
    dd = ConvDesc(B, ph, pwid, c, 3, 3, c, s, s, 1, 1, pad, act)
    got, pooled, want = (guarded_out(sh, BAND) for sh in ((B, oh, ow, c), (B, ph, pwid, c), (B, oh, ow, c)))
    assert _lib().lce_b200_f32_maxpool2x2_depthwise3x3(C.byref(pd), C.byref(dd), _p(xg.t), _p(wg.t), _p(bg.t),
                                                       _p(got.t), None) == 0, _err()
    assert _lib().lce_b200_f32_max_pool(C.byref(pd), _p(xg.t), _p(pooled.t), None) == 0, _err()
    assert _lib().lce_b200_f32_depthwise_conv2d(C.byref(dd), _p(pooled.t), _p(wg.t), _p(bg.t), _p(want.t),
                                                None) == 0, _err()
    torch.cuda.synchronize()
    for gb in (xg, wg, bg, got, pooled, want):
        gb.assert_band(cid)
    for gb in (got, want):
        gb.assert_written(cid)
    return (x, w, bias), got.t, want.t


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fused_transition_is_max_pool_then_depthwise(case):
    cid, B, _, _, _, s, pad, act = case
    (x, w, bias), got, want = _launch(case)
    assert same_bits(got, want), f"{cid}: fused != MAX_POOL_2D then DEPTHWISE_CONV_2D"
    wn, bn = w.cpu().numpy(), bias.cpu().numpy()
    for i in sorted({0, B - 1}):
        p = pool_ref(x[i:i + 1].cpu().numpy(), (2, 2), (1, 1), VALID, NONE, True)
        ref = depthwise_ref(p, wn, bn, (s, s), (1, 1), pad, act)
        assert _eq(got[i:i + 1].cpu().numpy(), ref), f"{cid}: image {i} vs the exact references"
