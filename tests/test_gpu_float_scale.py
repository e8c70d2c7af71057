"""The float kernels of the benchmarked graphs at full launch sizes, through the C-ABI of
include/lce_b200_builtins.h, against exact or fp64 references.

Three of them are persistent, so a CTA carries state from one item to the next:
* pw_tf32_kernel (lce_b200_pw.cuh, launched by pw_tf32_conv in lce_b200.cu) launches
  min(items, SMs) CTAs. It carries the 3-stage A/W ring's slot and mbarrier parity, the resident
  W tile (one column tile, KB <= 3) that is loaded and split only on a CTA's first item, and in
  pairs mode (K = 16, N = 64) W' = diag(W, W), which is also built only on the first item.
* stem_conv_dw_kernel (the fused 3x3 s2 conv + depthwise stem, 16 and 8 channels) launches
  min(tile groups, SMs) CTAs, each running one or two groups of 256 threads over 4-row tiles.
* stem7_tf32_kernel (Bi-RealNet's 7x7 stem) launches up to 2 x SMs CTAs of two warpgroups, each
  warpgroup walking 64-pixel tiles.
`pw_layout`, `stem_layout` and `stem7_layout` restate their launch arithmetic, and a CPU test
checks that every case gives each CTA (each thread group, each warpgroup) at least four items on
a 132-SM H100 and reaches the mode it is named for. pool2_dw3_v4_kernel (QuickNet's transition,
MAX_POOL 2x2 s1 then the blur depthwise 3x3 s2) is not persistent; it runs at its benched channel
counts, where one 256-thread block covers many pixels.

The shapes are those zoo.py builds at the benched batches (QuickNet 256, QuickNetLarge 128,
Bi-RealNet-18 512), raised where a layer would give fewer than four items per CTA. QuickNetLarge
has QuickNet's section widths, so its 1x1 layers and transitions have QuickNet's shapes; only its
batch differs.

Every buffer lives in a larger allocation whose base is 256-byte aligned, as the graph arena's
tensors are, so kernel selection is what the graph gets. Inputs are followed by a band of poison
one tile long (128 rows of the case's widest operand); outputs are poisoned whole and the band
past their end must still hold the poison afterwards, and no output element may be left unwritten.

A torch.profiler trace names the kernel of every launch, checked by the last test of the file.
The traces are taken in a fresh subprocess that makes the same launches on the same seeded inputs
(the `traces` fixture starts it with the first GPU test, so it runs alongside the value checks).
Once another process has profiled, as test_gpu_float_kernels' variant tests do before this file
runs, this process's traces come back empty or with kernels missing. Kernel selection depends only
on shapes, pointer alignment and the environment, which both processes share. No CUDA graphs are
captured.

The tf32 bound is test_gpu_builtins' |err| <= 2e-6 (sum |a||w| + |bias|) up to K = 512, which
covers every model layer here. Above that it grows as sqrt(K / 512). The fp32 accumulator takes
3K / 8 wgmma steps, and its rounding grows with their number times the partial sums, which are
about sum |a||w| / sqrt(K). On an H100 the K = 4096 case measures 4.2e-6.
"""
import ctypes as C
import json
import os
import subprocess
import sys
from dataclasses import dataclass, field

import numpy as np
import pytest

import lce_testlib as L
from test_gpu_float_kernels import (ConvDesc, PoolDesc, _assert_ran, _eq, _err, _lib, _p, _profiled, conv_ref,
                                    depthwise_ref, pool_ref)

SAME, VALID = L.PADDING_SAME, L.PADDING_VALID
NONE, RELU, N1, RELU6 = L.ACT_NONE, L.ACT_RELU, L.ACT_RELU_N1_TO_1, L.ACT_RELU6
T_FLOAT, T_INT8 = L.T_FLOAT, L.T_INT8
H100_SMS = 132
MIN_ITEMS_PER_CTA = 4
BOUND = 2e-6                  # test_gpu_builtins' tf32 bound, K <= 512
BAND_ROWS = 128               # one tile of rows
POISON = 0x7FA5A5A5           # a NaN as float32; as an int32 sentinel it marks unwritten packed words
POISON_BYTE = 0xA5            # int8 -91: not the pad value of any quantised image here
POS_INF = 0x7F800000          # max-pool inputs: fmaxf drops a NaN, so their band is +Inf instead
TRACE_ATTEMPTS = 4

PW_KERNEL = "pw_tf32_kernel"
PW16_KERNEL = "conv_direct16_kernel<1,1,16,4,true>"


# ------------------------------------ launch arithmetic ------------------------------------ #
def cdiv(a, b):
    return -(-a // b)


def pw_layout(M, K, N, packed, pairs_ok, sms=H100_SMS):
    """conv2d_impl (lce_b200_builtins.cu) + pw_tf32_conv (lce_b200.cu) on aligned buffers for a
    1x1 stride-1 CONV_2D of M pixels: whether the tf32 kernel takes it, in which mode, and its grid.
    `pairs_ok`: even pixels per image."""
    packed = packed and N % 32 == 0             # conv2d_impl passes the signs only for whole words
    pairs = K == 16 and N == 64 and pairs_ok and M % 2 == 0
    if not pairs and (K % 32 or K > 4096 or N % 4 or (N % 128 and packed)):
        return dict(eligible=False, pairs=False)
    pM, pN = (M // 2, 128) if pairs else (M, N)
    KB = 1 if pairs else K // 32
    n_tiles, m_tiles = cdiv(pN, 128), cdiv(pM, 128)
    if m_tiles > 1 << 22:
        return dict(eligible=False, pairs=False)
    items = n_tiles * m_tiles
    grid = min(items, sms)
    return dict(eligible=True, pairs=pairs, M=pM, KB=KB, n_tiles=n_tiles, m_tiles=m_tiles,
                w_resident=n_tiles == 1 and KB <= 3, grid=grid, per_cta=items // grid, ring_wraps=KB % 3 != 0)


def stem_layout(B, H, W, c1, in_type, sms=H100_SMS):
    """launch_stem2: 3x3 s2 SAME then depthwise 3x3 s2 SAME; tiles of 4 output rows x 56 columns;
    byte images run two 256-thread groups per CTA, float images one of 512."""
    oh2, ow2 = cdiv(cdiv(H, 2), 2), cdiv(cdiv(W, 2), 2)
    tiles = B * cdiv(oh2, 4) * cdiv(ow2, 56)
    groups = 1 if in_type == T_FLOAT else 2
    grid = min(cdiv(tiles, groups), sms)
    return dict(tiles=tiles, groups=groups, grid=grid, per_group=tiles // (grid * groups))


def stem7_layout(B, H, W, sms=H100_SMS):
    """stem7_tf32_conv: 64-pixel tiles, two warpgroups per CTA, two CTAs per SM."""
    m_tiles = cdiv(B * cdiv(H, 2) * cdiv(W, 2), 64)
    grid = min(cdiv(m_tiles, 2), 2 * sms)
    return dict(m_tiles=m_tiles, grid=grid, per_warpgroup=m_tiles // (2 * grid))


# ------------------------------------------ cases ------------------------------------------ #
@dataclass
class Pw:
    name: str
    b: int
    h: int
    w: int
    k: int
    n: int
    act: int = NONE
    packed: bool = False
    target: dict = field(default_factory=dict)

    @property
    def M(self):
        return self.b * self.h * self.w

    @property
    def pairs_ok(self):
        return self.h * self.w % 2 == 0

    @property
    def layout(self):
        return pw_layout(self.M, self.k, self.n, self.packed, self.pairs_ok)


PW = [
    # QuickNet at batch 256 (the last layer at 384: 256 gives 2.97 items per CTA); the layers feeding
    # a binary block carry its LceQuantize
    Pw("quicknet_stem_16-64", 256, 56, 56, 16, 64, packed=True, target={"pairs": True, "w_resident": True}),
    Pw("quicknet_t1_64-128", 256, 28, 28, 64, 128, packed=True, target={"w_resident": True, "KB": 2}),
    Pw("quicknet_t2_128-256", 256, 14, 14, 128, 256, packed=True,
       target={"w_resident": False, "n_tiles": 2, "KB": 4, "ring_wraps": True}),
    Pw("quicknet_t3_256-512_b384", 384, 7, 7, 256, 512, packed=True, target={"n_tiles": 4, "KB": 8}),
    # QuickNetLarge at batch 128 (its later 1x1 layers are QuickNet's t2 / t3 at a smaller batch)
    Pw("quicknet_large_stem_16-64", 128, 56, 56, 16, 64, packed=True, target={"pairs": True}),
    Pw("quicknet_large_t1_64-128", 128, 28, 28, 64, 128, packed=True, target={"w_resident": True}),
    # Bi-RealNet-18's downsampling shortcuts at batch 512: added to the binary output, no signs
    Pw("birealnet_s1_64-128", 512, 28, 28, 64, 128, target={"w_resident": True, "KB": 2}),
    Pw("birealnet_s2_128-256", 512, 14, 14, 128, 256, target={"n_tiles": 2, "KB": 4}),
    Pw("birealnet_s3_256-512", 512, 7, 7, 256, 512, target={"n_tiles": 4, "KB": 8, "ring_wraps": True}),
    # resident weights at KB = 1 (QuickNetSmall's 32 -> 64 transition: 64 of 128 columns) and KB = 3
    Pw("quicknet_small_t1_32-64", 256, 28, 28, 32, 64, RELU,
       target={"w_resident": True, "KB": 1, "n_tiles": 1, "ring_wraps": True}),
    Pw("resident_kb3_96-128", 200, 20, 20, 96, 128, RELU6, True,
       target={"w_resident": True, "KB": 3, "ring_wraps": False}),
    # weight rings that wrap inside an item: one column tile at KB = 4, two at KB = 5
    Pw("ring_kb4_128-128", 300, 16, 16, 128, 128, N1, True,
       target={"w_resident": False, "n_tiles": 1, "KB": 4, "ring_wraps": True}),
    Pw("ring_kb5_160-256", 160, 15, 17, 160, 256, RELU, True, target={"n_tiles": 2, "KB": 5, "ring_wraps": True}),
    Pw("k4096_4096-256", 64, 23, 23, 4096, 256, packed=True, target={"KB": 128, "n_tiles": 2}),
    # a last row tile of one row (each 1x1 "image" one row)
    Pw("ragged_last_row_64-128", 128 * 600 + 1, 1, 1, 64, 128, RELU, True, target={"m_tiles": 601}),
    # FULLY_CONNECTED's 1000 logits: no signs, a last column tile of 104 columns
    Pw("fully_connected_512-1000", 9000, 1, 1, 512, 1000, target={"n_tiles": 8}),
    # odd pixels per image: the tf32 kernel declines K = 16, conv_direct16's pointwise instance runs
    Pw("odd_pixels_16-64", 256, 55, 55, 16, 64, packed=True, target={"eligible": False}),
]
PW_IDS = [s.name for s in PW]

# (id, first-conv channels, image type, batch): QuickNet's benched int8 stem, QuickNetSmall's
# 8-channel instance, and QuickNet's float-image stem (one 512-thread group per CTA)
STEMS = [("quicknet_int8", 16, T_INT8, 256), ("quicknet_small_int8", 8, T_INT8, 256),
         ("quicknet_float32", 16, T_FLOAT, 256)]
STEM_IDS = [c[0] for c in STEMS]
STEM7_BATCH = 512
# QuickNet's (and QuickNetLarge's) three transitions: (batch, input H = W, channels)
POOLS = [(256, 56, 64), (256, 28, 128), (256, 14, 256)]


def test_launch_layouts_give_every_cta_four_items():
    """Every persistent case gives each CTA at least four items on 132 SMs and reaches the mode it
    is named for; together the pointwise cases cover pairs, resident weights at KB = 1, 2, 3, rings
    that do and do not wrap inside an item, ragged row and column tiles, and a declined shape."""
    assert len(set(PW_IDS)) == len(PW_IDS)
    seen = {"pairs": set(), "w_resident": set(), "ring_wraps": set(), "eligible": set()}
    resident_kb, ring_kb = set(), set()
    for s in PW:
        lay = s.layout
        for k, v in s.target.items():
            assert lay[k] == v, (s.name, k, lay)
        seen["eligible"].add(lay["eligible"])
        if not lay["eligible"]:
            continue
        assert lay["per_cta"] >= MIN_ITEMS_PER_CTA, (s.name, lay)
        for k in ("pairs", "w_resident", "ring_wraps"):
            seen[k].add(lay[k])
        (resident_kb if lay["w_resident"] else ring_kb).add(lay["KB"])
    assert all(v == {True, False} for v in seen.values()), seen
    assert {1, 2, 3} <= resident_kb and {4, 5} <= ring_kb, (resident_kb, ring_kb)
    assert any(s.M % 128 == 1 for s in PW) and any(s.n % 128 for s in PW if s.layout["eligible"])
    for _, c1, in_type, b in STEMS:
        lay = stem_layout(b, 224, 224, c1, in_type)
        assert lay["grid"] == H100_SMS and lay["per_group"] >= MIN_ITEMS_PER_CTA, lay
    lay = stem7_layout(STEM7_BATCH, 224, 224)
    assert lay["grid"] == 2 * H100_SMS and lay["per_warpgroup"] >= MIN_ITEMS_PER_CTA, lay


def test_pw_layout_declines_what_pw_tf32_conv_declines():
    assert not pw_layout(1000, 16, 64, False, False)["eligible"]        # odd pixels per image
    assert pw_layout(1000, 16, 64, False, True)["pairs"]
    assert not pw_layout(1000, 16, 128, False, True)["eligible"]       # K = 16 without pairs
    assert not pw_layout(1000, 4128, 128, False, True)["eligible"]     # K > 4096
    assert not pw_layout(1000, 64, 1056, True, True)["eligible"]       # signs of a partial column tile
    assert pw_layout(1000, 64, 1056, False, True)["eligible"]
    assert pw_layout(1000, 64, 1000, True, True)["eligible"]           # 1000 % 32: no signs asked of it
    assert not pw_layout(1000, 64, 102, False, True)["eligible"]       # N % 4


# ------------------------------------------- GPU -------------------------------------------- #
class Guarded:
    """`shape` elements at the 256-byte aligned base of a buffer `band` elements longer, all set to
    the 32-bit word (or byte) `fill`; `data` (a device tensor) is copied in if given."""

    def __init__(self, shape, dtype, band, fill, data=None):
        import torch
        n = int(np.prod(shape))
        self.buf = torch.empty(n + band, dtype=dtype, device="cuda")
        assert self.buf.data_ptr() % 256 == 0
        self.fill = fill
        self._fill(self.buf)
        self.t = self.buf[:n].view(shape)
        self.band = self.buf[n:]
        if data is not None:
            self.t.copy_(data.reshape(shape))

    def _fill(self, t):
        import torch
        if t.element_size() == 4:
            t.view(torch.int32).fill_(self.fill)
        else:
            t.view(torch.uint8).fill_(self.fill & 0xFF)

    def _words(self, t):
        import torch
        return t.view(torch.int32 if t.element_size() == 4 else torch.uint8)

    def assert_band(self, what):
        want = self._words(self.band.new_empty(self.band.shape))
        self._fill(want)
        assert self._words(self.band).equal(want), f"{what}: the band past the end was written"

    def assert_written(self, what):
        """No element still holds the poison (outputs poisoned with a NaN; never a kernel's result)."""
        import torch
        assert not torch.isnan(self.t).any(), f"{what}: elements left unwritten (or NaN)"


def guarded_in(t, band, fill=POISON):
    return Guarded(tuple(t.shape), t.dtype, band, fill if t.element_size() == 4 else POISON_BYTE, t)


def guarded_out(shape, band, dtype=None):
    import torch
    return Guarded(shape, dtype or torch.float32, band, POISON)


def same_bits(a, b):
    import torch
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    return a.view(torch.int32).equal(b.view(torch.int32)) if a.element_size() == 4 else a.equal(b)


def sign_words(out):
    """LceQuantize of a float [M, N] map: bit = x < 0, LSB first."""
    import torch
    M, N = out.shape
    bits = (out < 0).view(M, N // 32, 32).to(torch.int64)
    words = (bits << torch.arange(32, device=out.device)).sum(-1)
    return torch.where(words >= 2**31, words - 2**32, words).to(torch.int32)


def activation(y, act):
    if act == RELU:
        return y.clamp(min=0)
    if act == RELU6:
        return y.clamp(0, 6)
    if act == N1:
        return y.clamp(-1, 1)
    return y


def pw_bound(K):
    return BOUND * max(1.0, (K / 512) ** 0.5)


def assert_fp64_bound(out, A, W, b, act, what):
    """|out - act(A W^T + b)| <= pw_bound(K) (|A| |W|^T + |b|) on every element, the product in fp64."""
    ref = activation(A.double() @ W.double().t() + b.double(), act)
    mag = A.abs().double() @ W.abs().double().t() + b.abs().double()
    rel = (out.double() - ref).abs() / mag
    worst = rel.max().item()
    assert worst <= pw_bound(A.shape[1]), \
        f"{what}: error {worst:.3g} x sum|a||w| at row {int(rel.max(1).values.argmax())}"


def sms_now():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def untraced(label, fn):
    return fn()


# ------------------------- launches (shared with the tracing subprocess) ------------------------- #
# Each takes `launch(label, fn)`, which calls fn (one or more C-ABI calls, returning the last rc);
# in the subprocess it also records the kernels fn ran under `label`.
def run_pw(s, A, W, b, batch, label, launch):
    """CONV_2D 1x1 of `batch` images through lce_b200_f32_conv2d[_packed], every buffer guarded.
    Returns (float output [M, N], signs [M, N / 32] or None)."""
    import torch
    band = BAND_ROWS * max(s.k, s.n)
    ins = [guarded_in(t, band) for t in (A, W, b)]
    rows = A.shape[0]
    out = guarded_out((rows, s.n), band)
    pk = guarded_out((rows, s.n // 32), band, torch.int32) if s.packed else None
    d = ConvDesc(batch, s.h, s.w, s.k, 1, 1, s.n, 1, 1, 1, 1, VALID, s.act)
    a, w, bias = (g.t for g in ins)

    def go():
        if pk is not None:
            return _lib().lce_b200_f32_conv2d_packed(C.byref(d), _p(a), _p(w), _p(bias), _p(out.t), _p(pk.t), None)
        return _lib().lce_b200_f32_conv2d(C.byref(d), _p(a), _p(w), _p(bias), _p(out.t), None)

    assert launch(label, go) == 0, _err()
    for g, what in zip(ins + [out] + ([pk] if pk else []), ("input", "filter", "bias", "output", "signs")):
        g.assert_band(f"{label} {what}")
    out.assert_written(label)
    return out.t, (pk.t if pk else None)


def pw_launches(s, launch):
    """The full launch, then the first and the last image alone: (A, W, b, [(image, out, signs)])."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(41000 + PW_IDS.index(s.name))
    A = torch.randn((s.M, s.k), device="cuda", generator=g) * 1.5
    W = torch.randn((s.n, s.k), device="cuda", generator=g) * 0.3
    b = torch.randn(s.n, device="cuda", generator=g)
    runs = [(None, *run_pw(s, A, W, b, s.b, s.name, launch))]
    hw = s.h * s.w
    for i in (0, s.b - 1):
        runs.append((i, *run_pw(s, A[i * hw:(i + 1) * hw], W, b, 1, f"{s.name}/image{i}", launch)))
    return A, W, b, runs


def stem_launches(case, launch):
    """The fused stem, then DEQUANTIZE -> CONV_2D -> DEPTHWISE_CONV_2D: (inputs, fused, separate)."""
    import torch
    cid, c1, in_type, B = case
    H = W = 224
    g = torch.Generator(device="cuda").manual_seed(42000 + STEM_IDS.index(cid))
    if in_type == T_INT8:
        x = torch.randint(-128, 128, (B, H, W, 3), device="cuda", generator=g, dtype=torch.int16).to(torch.int8)
        scale, zp = 4.0 / 127, -3
    else:
        x = torch.randn((B, H, W, 3), device="cuda", generator=g)
        scale, zp = 1.0, 0
    rng = np.random.default_rng(42000 + STEM_IDS.index(cid))
    filters = [(rng.standard_normal((c1, 3, 3, 3)) * 0.4).astype(np.float32), rng.standard_normal(c1).astype(np.float32),
               (rng.standard_normal((1, 3, 3, c1)) * 0.4).astype(np.float32), rng.standard_normal(c1).astype(np.float32)]
    d1 = ConvDesc(B, H, W, 3, 3, 3, c1, 2, 2, 1, 1, SAME, RELU)
    d2 = ConvDesc(B, 112, 112, c1, 3, 3, c1, 2, 2, 1, 1, SAME, NONE)
    band = BAND_ROWS * W * 3
    xg = guarded_in(x, band)
    host = [torch.from_numpy(f) for f in filters]          # the fused kernel's filters travel by value
    dev = [guarded_in(t.cuda(), band) for t in host]
    got = guarded_out((B, 56, 56, c1), band)
    assert launch(f"{cid}/fused", lambda: _lib().lce_b200_f32_stem_conv_dw(
        C.byref(d1), C.byref(d2), in_type, _p(xg.t), C.c_double(scale), C.c_int32(zp), *map(_p, host), _p(got.t),
        None)) == 0, _err()
    xf = guarded_out((B, H, W, 3), band) if in_type != T_FLOAT else xg
    y1 = guarded_out((B, 112, 112, c1), band)
    want = guarded_out((B, 56, 56, c1), band)

    def separate():
        if in_type != T_FLOAT:
            assert _lib().lce_b200_dequantize_affine(in_type, _p(xg.t), _p(xf.t), C.c_int64(x.numel()),
                                                     C.c_double(scale), C.c_int32(zp), None) == 0, _err()
        assert _lib().lce_b200_f32_conv2d(C.byref(d1), _p(xf.t), _p(dev[0].t), _p(dev[1].t), _p(y1.t), None) == 0, _err()
        return _lib().lce_b200_f32_depthwise_conv2d(C.byref(d2), _p(y1.t), _p(dev[2].t), _p(dev[3].t), _p(want.t), None)

    assert launch(f"{cid}/separate", separate) == 0, _err()
    for gb, what in zip([xg, got, xf, y1, want] + dev, ("image", "fused output", "dequantised", "conv output",
                                                       "depthwise output", "w1", "b1", "w2", "b2")):
        gb.assert_band(f"{cid} {what}")
    for gb, what in ((got, "fused output"), (y1, "conv output"), (want, "depthwise output")):
        gb.assert_written(f"{cid} {what}")
    return (x, scale, zp, filters), got.t, want.t


def stem7_desc(batch):
    return ConvDesc(batch, 224, 224, 3, 7, 7, 64, 2, 2, 1, 1, SAME, NONE)


def stem7_launches(launch):
    """Bi-RealNet's stem at its batch, then the first and the last image alone, each guarded:
    (x, w, b, guarded filter and bias, full output, [(image, output alone)])."""
    import torch
    B = STEM7_BATCH
    g = torch.Generator(device="cuda").manual_seed(43000)
    x = torch.randn((B, 224, 224, 3), device="cuda", generator=g) * 1.5
    w = torch.randn((64, 7, 7, 3), device="cuda", generator=g) * 0.2
    b = torch.randn(64, device="cuda", generator=g)
    band = BAND_ROWS * 224 * 3
    wg, bg = guarded_in(w, band), guarded_in(b, band)
    runs = []
    for i, xs in ((None, x), (0, x[:1]), (B - 1, x[B - 1:])):
        xg, og = guarded_in(xs, band), guarded_out((xs.shape[0], 112, 112, 64), band)
        d = stem7_desc(xs.shape[0])
        label = "stem7" if i is None else f"stem7/image{i}"
        assert launch(label, lambda: _lib().lce_b200_f32_conv2d(C.byref(d), _p(xg.t), _p(wg.t), _p(bg.t), _p(og.t),
                                                                None)) == 0, _err()
        for gb, what in ((xg, "image"), (og, "output")):
            gb.assert_band(f"{label} {what}")
        og.assert_written(label)
        runs.append((i, og.t))
    wg.assert_band("stem7 filter")
    bg.assert_band("stem7 bias")
    return x, w, b, (wg, bg), runs


def pool_launches(B, hw, c, launch):
    """The fused max-pool + depthwise, then MAX_POOL_2D and DEPTHWISE_CONV_2D: (inputs, fused, separate)."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(44000 + hw)
    x = torch.randn((B, hw, hw, c), device="cuda", generator=g) * 3
    w = torch.randn((1, 3, 3, c), device="cuda", generator=g)
    bias = torch.randn(c, device="cuda", generator=g)
    ph, oh = hw - 1, cdiv(hw - 1, 2)
    band = BAND_ROWS * hw * c
    xg = guarded_in(x, band, POS_INF)
    wg, bg = guarded_in(w, band), guarded_in(bias, band)
    pd = PoolDesc(B, hw, hw, c, 2, 2, 1, 1, VALID, NONE)
    dd = ConvDesc(B, ph, ph, c, 3, 3, c, 2, 2, 1, 1, SAME, NONE)
    got, pooled, want = (guarded_out(s, band) for s in ((B, oh, oh, c), (B, ph, ph, c), (B, oh, oh, c)))
    label = f"pool/{hw}x{hw}x{c}"
    assert launch(label + "/fused", lambda: _lib().lce_b200_f32_maxpool2x2_depthwise3x3(
        C.byref(pd), C.byref(dd), _p(xg.t), _p(wg.t), _p(bg.t), _p(got.t), None)) == 0, _err()

    def separate():
        assert _lib().lce_b200_f32_max_pool(C.byref(pd), _p(xg.t), _p(pooled.t), None) == 0, _err()
        return _lib().lce_b200_f32_depthwise_conv2d(C.byref(dd), _p(pooled.t), _p(wg.t), _p(bg.t), _p(want.t), None)

    assert launch(label + "/separate", separate) == 0, _err()
    for gb, what in ((xg, "input"), (wg, "filter"), (bg, "bias"), (got, "fused output"), (pooled, "pooled"),
                     (want, "depthwise output")):
        gb.assert_band(f"{label} {what}")
    for gb, what in ((got, "fused output"), (pooled, "pooled"), (want, "depthwise output")):
        gb.assert_written(f"{label} {what}")
    return (x, w, bias), got.t, want.t


def _trace_all(path):
    """Subprocess side of the `traces` fixture: every launch of this file under torch.profiler.
    Sessions can come back empty or with kernels missing, so a launch is traced again (it is
    repeatable) until the union of its traces names the kernels it is expected to run, at most
    TRACE_ATTEMPTS times; test_each_launch_ran_its_kernel decides."""
    import torch
    names = {}
    want = dict(expected_kernels())

    def traced(label, fn):
        rc, seen = None, set()
        for _ in range(TRACE_ATTEMPTS):
            try:
                rc, got = _profiled(fn)
            except AssertionError:          # three empty sessions
                continue
            seen.update(got)
            if all(any("".join(k.split()) in n for n in seen) for k in want[label]):
                break
        names[label] = sorted(seen)
        return fn() if rc is None else rc

    for s in PW:
        pw_launches(s, traced)
    for case in STEMS:
        stem_launches(case, traced)
    stem7_launches(traced)
    for B, hw, c in POOLS:
        pool_launches(B, hw, c, traced)
    torch.cuda.synchronize()
    with open(path, "w") as f:
        json.dump(names, f)


class Traces:
    """The tracing subprocess (`_trace_all`) and, once it has finished, its kernels by launch label."""

    def __init__(self, tmp):
        here = os.path.dirname(os.path.abspath(__file__))
        self.path, self.log = tmp / "traces.json", tmp / "stderr.txt"
        code = (f"import sys; sys.path[:0] = [{here!r}, {os.path.dirname(here)!r}]\n"
                f"import test_gpu_float_scale as T\nT._trace_all({str(self.path)!r})\n")
        with open(self.log, "w") as err:
            self.proc = subprocess.Popen([sys.executable, "-c", code], stdout=subprocess.DEVNULL, stderr=err)
        self._names = None

    def wait(self):
        try:
            self.proc.wait(timeout=900)
        except subprocess.TimeoutExpired:
            self.proc.kill()
            self.proc.wait()
            raise

    def names(self):
        if self._names is None:
            self.wait()
            assert self.proc.returncode == 0, self.log.read_text()[-3000:]
            self._names = json.loads(self.path.read_text())
        return self._names


@pytest.fixture(scope="module")
def traces(tmp_path_factory):
    """Every GPU test asks for it, so the first one starts the subprocess; the last test reads it."""
    t = Traces(tmp_path_factory.mktemp("float_scale"))
    yield t
    t.wait()


# -------------------------------------------- tests -------------------------------------------- #
@pytest.mark.gpu
@pytest.mark.parametrize("s", PW, ids=PW_IDS)
def test_pointwise_conv_at_scale(s, traces):
    """All rows within the fp64 bound; the signs equal those of the kernel's own float output; the
    first and the last image launched alone give the bits they have in the full launch. The
    declined odd-pixel shape also equals the fmaf chain on three images."""
    lay = pw_layout(s.M, s.k, s.n, s.packed, s.pairs_ok, sms_now())
    assert not lay["eligible"] or lay["per_cta"] >= MIN_ITEMS_PER_CTA, lay
    A, W, b, runs = pw_launches(s, untraced)
    _, out, pk = runs[0]
    tag = f"{s.name} ({lay.get('per_cta')} items per CTA)"
    assert_fp64_bound(out, A, W, b, s.act, tag)
    if pk is not None:
        assert pk.equal(sign_words(out)), f"{tag}: signs"
    hw = s.h * s.w
    if not lay["eligible"]:
        x, w, bias = A.cpu().numpy(), W.cpu().numpy().reshape(s.n, 1, 1, s.k), b.cpu().numpy()
        for i in (0, s.b // 2, s.b - 1):
            want = conv_ref(x[i * hw:(i + 1) * hw].reshape(1, s.h, s.w, s.k), w, bias, act=s.act)
            assert _eq(out[i * hw:(i + 1) * hw].cpu().numpy(), want.reshape(hw, s.n)), f"{tag}: image {i}"
    for i, o1, p1 in runs[1:]:
        rows = slice(i * hw, (i + 1) * hw)
        assert same_bits(o1, out[rows]), f"{tag}: image {i} alone"
        if pk is not None:
            assert p1.equal(pk[rows]), f"{tag}: image {i}'s signs alone"


@pytest.mark.gpu
@pytest.mark.parametrize("case", STEMS, ids=STEM_IDS)
def test_fused_stem_at_scale(case, traces):
    """stem_conv_dw_kernel at 224 x 224 and batch 256: the whole output equals DEQUANTIZE ->
    CONV_2D -> DEPTHWISE_CONV_2D run as separate kernels, bit for bit; the first, a middle and the
    last image equal the fmaf-chain references of the numpy-dequantised image."""
    cid, c1, in_type, B = case
    lay = stem_layout(B, 224, 224, c1, in_type, sms_now())
    assert lay["per_group"] >= MIN_ITEMS_PER_CTA, lay
    (x, scale, zp, (w1, b1, w2, b2)), got, want = stem_launches(case, untraced)
    assert same_bits(got, want), f"{cid}: fused != separate kernels"
    for i in (0, B // 2, B - 1):
        xi = x[i:i + 1].cpu().numpy()
        if in_type != T_FLOAT:
            xi = (np.float64(scale) * (xi.astype(np.int64) - zp)).astype(np.float32)
        ref = depthwise_ref(conv_ref(xi, w1, b1, (2, 2), act=RELU), w2, b2, (2, 2))
        assert _eq(got[i:i + 1].cpu().numpy(), ref), f"{cid}: image {i} vs the fmaf chain"


@pytest.mark.gpu
def test_stem7_at_scale(traces):
    """stem7_tf32_kernel at Bi-RealNet's batch of 512 (190 tiles per warpgroup): eight images spread
    over the batch within the fp64 bound; the first and the last image alone (traced and guarded),
    and then every image alone, give the bits they have in the full launch, where all but the first
    few images run as a warpgroup's later tiles."""
    import torch
    import torch.nn.functional as F
    B = STEM7_BATCH
    lay = stem7_layout(B, 224, 224, sms_now())
    assert lay["per_warpgroup"] >= MIN_ITEMS_PER_CTA, lay
    x, w, b, (wg, bg), runs = stem7_launches(untraced)
    out = runs[0][1]
    sel = torch.from_numpy(np.linspace(0, B - 1, 8).round().astype(np.int64)).cuda()
    xs = x[sel].double().permute(0, 3, 1, 2)
    pad = (2, 3, 2, 3)                         # TFLite SAME: 5 padded columns / rows, 2 before
    conv = lambda xx, ww: F.conv2d(F.pad(xx, pad), ww.permute(0, 3, 1, 2), stride=2).permute(0, 2, 3, 1)
    ref = conv(xs, w.double()) + b.double()
    mag = conv(xs.abs(), w.abs().double()) + b.abs().double()
    rel = ((out[sel].double() - ref).abs() / mag).max().item()
    assert rel <= pw_bound(147), (rel, sel)
    for i, oi in runs[1:]:
        assert same_bits(oi, out[i:i + 1]), f"image {i} alone"
    band = BAND_ROWS * 224 * 3
    xg, alone = guarded_in(x, band), guarded_out(tuple(out.shape), band)
    d = stem7_desc(1)
    for i in range(B):
        assert _lib().lce_b200_f32_conv2d(C.byref(d), _p(xg.t[i]), _p(wg.t), _p(bg.t), _p(alone.t[i]), None) == 0, _err()
    alone.assert_band("images alone")
    if not same_bits(alone.t, out):
        differ = [i for i in range(B) if not same_bits(alone.t[i], out[i])]
        raise AssertionError(f"images alone differ from the full launch: {differ[:10]} ({len(differ)} images)")


@pytest.mark.gpu
@pytest.mark.parametrize("B,hw,c", POOLS, ids=[f"{hw}x{hw}x{c}" for _, hw, c in POOLS])
def test_fused_maxpool_depthwise_at_scale(B, hw, c, traces):
    """pool2_dw3_v4_kernel at QuickNet's transition shapes and batch 256, random filter and bias
    (the blur filter's powers of two would make every product exact): the whole output equals
    MAX_POOL_2D then DEPTHWISE_CONV_2D run separately, bit for bit; three images equal the exact
    references."""
    (x, w, bias), got, want = pool_launches(B, hw, c, untraced)
    assert same_bits(got, want), "fused != separate kernels"
    wn, bn = w.cpu().numpy(), bias.cpu().numpy()
    for i in (0, B // 2, B - 1):
        p = pool_ref(x[i:i + 1].cpu().numpy(), (2, 2), (1, 1), VALID, NONE, True)
        ref = depthwise_ref(p, wn, bn, (2, 2))
        assert _eq(got[i:i + 1].cpu().numpy(), ref), f"image {i} vs the exact references"


def expected_kernels():
    """(launch label, the kernels its trace must show) for every launch of the file."""
    out = []
    for s in PW:
        kernel = PW_KERNEL if s.layout["eligible"] else PW16_KERNEL
        out += [(label, (kernel,)) for label in (s.name, f"{s.name}/image0", f"{s.name}/image{s.b - 1}")]
    for cid, _, in_type, _ in STEMS:
        out += [(f"{cid}/fused", ("stem_conv_dw_kernel",)),
                (f"{cid}/separate", ("conv_direct16_kernel<3,3,3,2,", "depthwise_v4_kernel<3>") + (
                    ("dequantize_affine_kernel",) if in_type != T_FLOAT else ()))]
    out += [(label, ("stem7_tf32_kernel",)) for label in ("stem7", "stem7/image0", f"stem7/image{STEM7_BATCH - 1}")]
    for _, hw, c in POOLS:
        out += [(f"pool/{hw}x{hw}x{c}/fused", ("pool2_dw3_v4_kernel",)),
                (f"pool/{hw}x{hw}x{c}/separate", ("pool_v4_kernel<true,2>", "depthwise_v4_kernel<3>"))]
    return out


KERNELS = expected_kernels()


@pytest.mark.gpu
@pytest.mark.parametrize("label,kernels", KERNELS, ids=[k[0] for k in KERNELS])
def test_each_launch_ran_its_kernel(label, kernels, traces):
    """Last in the file: the traces of the subprocess, one per launch of the tests above."""
    names = traces.names()
    assert sorted(names) == sorted(k[0] for k in KERNELS)
    for k in kernels:
        _assert_ran(names[label], k)
