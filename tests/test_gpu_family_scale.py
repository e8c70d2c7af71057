"""The newer model families' one-pass kernels and fused binary-convolution tails at the sizes their
benchmarks run, and the one-pass kernels' 64-bit index instances.

The one-pass kernels of ReActNet-A, Real-to-Binary Net, BinaryDenseNet, MeliusNet, BinaryAlexNet /
XNOR-Net, DoReFaNet and XNOR-Net++ are grid-stride loops: grid_for (lce_b200_builtins.cu) caps the
grid at 132 x 32 blocks of 256 threads whatever the device, and zpc_tail_kernel's (lce_b200.cu) at
132 x 16. At batch 256 every thread, or every warp of the warp-per-word kernels, runs many
iterations, and an index taken from its first iteration would be right on toy shapes only. Each
launcher also picks an `int` or a `long long` index instance; `launch` restates its rule, and a CPU
test checks that every case here gives each thread or warp at least four iterations and selects the
instance it is named for.

On the GPU: each one-pass kernel at the families' shapes, through the C-ABI into fully poisoned
outputs with a poison band behind each, on inputs with signed zeros, denormals and exact ties at the
sign threshold, against numpy over the whole output (three images where the reference is a
convolution). The fused mma.sync epilogues (run_fused_chain / _gate, run_slice, run_slice_add) and
their zero-padding CORRECTION fallbacks at batch 256, on b1 and int8, against the oracle convolution
plus the numpy tail. The `long long` instances on one buffer of 2^31 + 16 M floats, and the `int`
instances one stride below their threshold, against numpy on the rows around element 2^31 and the
last rows. No CUDA graphs are captured, so the file's place in the run order does not matter.
"""
import ctypes as C
from dataclasses import dataclass

import numpy as np
import pytest

import lce_testlib as L
from test_dorefanet import np_levels, np_maxpool, np_planes
from test_gpu_bconv_scale import POISON, S, THREADS, make_case, poisoned, same_bits, set_env
from test_gpu_parity import assert_same_bits, dev, gpu_desc, path_counts
from test_grouped_conv import _grouped_ref
from test_pooled_signs import _np_pooled_signs, _special_map
from test_reactnet import _np_chain
from test_realtobinary import _gate_tail_ref
from test_xnornetpp import _act_ref, _scale_tail_ref

F32 = np.float32
SAME, VALID = L.PADDING_SAME, L.PADDING_VALID
NONE, RELU, N1, RELU6 = L.ACT_NONE, L.ACT_RELU, L.ACT_RELU_N1_TO_1, L.ACT_RELU6
ACTS = (NONE, RELU, N1, RELU6)
TWO31 = 1 << 31
BUILTIN_CAP, ZPC_CAP = 132 * 32, 132 * 16     # grid_for's block caps in lce_b200_builtins.cu / lce_b200.cu
MIN_ITERS = 4
BAND = 1024                                   # poisoned words behind every output
POISON2 = 0x5A5A5A5A                          # the second run's poison (section 4; b1 vs int8)
SENTINEL = F32(-1234.5)


def cdiv(a, b):
    return -(-a // b)


def grid_for(n, cap=BUILTIN_CAP):
    return int(min(max(cdiv(n, 256), 1), cap))


def pool_out(size, k, s, padding):
    return cdiv(size, s) if padding == SAME else (size - k) // s + 1


# ------------------------------ launch arithmetic ------------------------------ #
@dataclass
class Tail:
    """One launch of a one-pass kernel. kernel: chain | prelu | gate | scale | affine | maxpool |
    quant2 | zpc | grouped. b, h, w, c: the input map (zpc, scale, gate, chain: the output map).
    want: the index instance the launcher must pick ("int", "long", "edge" = int one stride below
    the threshold, None = the kernel has one instance)."""
    name: str
    kernel: str
    b: int
    h: int
    w: int
    c: int
    packed: bool = True
    out: bool = True
    stride: int = 0          # affine: the input's pixel stride (0: c); grouped: the conv stride
    copy: int = 0            # affine: copy_to's pixel stride (0: no copy)
    pool: tuple = None       # maxpool / quant2: (k, s, padding); grouped: (groups, k, cout)
    act: int = NONE
    residual: bool = False
    alpha: bool = True       # gate: PRELU after the MUL
    prelu_c: int = 0         # prelu: the trailing alpha's element count
    want: str = "int"

    @property
    def rows(self):
        return self.b * self.h * self.w * self.c // self.span_c

    @property
    def span_c(self):
        return self.prelu_c if self.kernel == "prelu" else self.c


def launch(t):
    """The launcher's grid, its iterations per thread (per warp for the warp-per-word kernels,
    fewest over threads), its index bound and stride, and whether it picks the long long instance."""
    if t.kernel in ("chain", "prelu", "gate", "scale", "affine"):
        ch = t.span_c
        cw = cdiv(ch, 32)
        rows = t.rows
        n = rows * cw * 32 if (t.packed or t.kernel == "affine") else rows * ch
        grid = grid_for(n)
        step = 256 * grid
        narrow = n + step < TWO31
        if t.kernel == "gate":
            narrow = narrow and t.b * ch < TWO31
        if t.kernel == "affine":
            narrow = narrow and rows * max(t.stride or ch, t.copy) < TWO31
        return dict(grid=grid, iters=n // step, bound=n, step=step, wide=not narrow)
    if t.kernel in ("maxpool", "quant2"):
        oh, ow = (t.h, t.w) if t.pool is None else (pool_out(t.h, t.pool[0], t.pool[1], t.pool[2]),
                                                    pool_out(t.w, t.pool[0], t.pool[1], t.pool[2]))
        words = t.b * oh * ow * cdiv(t.c, 32)
        grid = grid_for(words * 32)
        bound = 3 * words if t.kernel == "quant2" else words
        narrow = t.b * t.h * t.w * t.c < TWO31 and bound + 8 * grid < TWO31
        return dict(grid=grid, iters=words // (8 * grid), bound=bound, step=8 * grid, wide=not narrow, oh=oh, ow=ow)
    if t.kernel == "zpc":
        warps = t.b * t.h * t.w * cdiv(t.c, 32)
        grid = grid_for(warps * 32, ZPC_CAP)
        return dict(grid=grid, iters=warps // (8 * grid), wide=None)
    if t.kernel == "grouped":
        groups, k, cout = t.pool
        oh, ow = cdiv(t.h, t.stride), cdiv(t.w, t.stride)
        n = t.b * oh * ow * cout
        grid = grid_for(n)
        return dict(grid=grid, iters=n // (256 * grid), wide=None, oh=oh, ow=ow)
    raise ValueError(t.kernel)


def grouped_tiled_takes(t):
    """lce_b200_f32_grouped_conv2d's rule for the tiled 3x3 kernel (16-byte aligned operands)."""
    groups, k, cout = t.pool
    cg, og = t.c // groups, cout // groups
    return k == 3 and t.stride == 1 and t.b <= 65535 and (cg, og, groups) in ((8, 8, 4), (4, 8, 8))


T = Tail
# ReActNet-A: the RPReLU / RSign chain (PRELU builtin: alpha over the trailing [W, C])
CHAIN = [
    T("reactnet_112x112x32", "chain", 256, 112, 112, 32),
    T("reactnet_56x56x128", "chain", 256, 56, 56, 128),
    T("reactnet_7x7x1024", "chain", 256, 7, 7, 1024),
    T("reactnet_7x7x1024_float_only", "chain", 256, 7, 7, 1024, packed=False),
    T("reactnet_7x7x1024_signs_only", "chain", 256, 7, 7, 1024, out=False),
    T("chain_28x28x100", "chain", 256, 28, 28, 100),
    T("prelu_112x112x32_alpha_112x32", "prelu", 256, 112, 112, 32, packed=False, prelu_c=112 * 32),
]
# Real-to-Binary Net's gated tail (and MUL's [B,1,1,C] broadcast), XNOR-Net++'s scaled tail: every
# ADD activation with and without the residual, in place
_R2B = [(56, 64), (28, 128), (14, 256), (7, 512)]
GATE = [T(f"r2b_{hw}x{hw}x{c}_act{a}_res{int(r)}", "gate", 256, hw, hw, c, act=a, residual=r)
        for i, (hw, c) in enumerate(_R2B) for a, r in ((ACTS[i], i % 2 == 0),)]
GATE += [T(f"r2b_7x7x512_act{a}_res{int(i % 2 == 1)}", "gate", 256, 7, 7, 512, act=a, residual=i % 2 == 1)
         for i, a in enumerate(ACTS)]
GATE += [T("mul_broadcast_56x56x64", "gate", 256, 56, 56, 64, packed=False, alpha=False)]
SCALE = [T(f"xnorpp_{hw}x{hw}x{c}_act{a}_res{int(r)}", "scale", 256, hw, hw, c, act=a, residual=r)
         for i, (hw, c) in enumerate(_R2B) for a, r in ((ACTS[3 - i], i % 2 == 1),)]
SCALE += [T(f"xnorpp_7x7x512_act{a}_res{int(i % 2 == 1)}", "scale", 256, 7, 7, 512, act=a, residual=i % 2 == 1)
          for i, a in enumerate(ACTS)]
# BinaryDenseNet: the BatchNorm signs of a dense block's leading channels (and the copy into the next map)
AFFINE = [
    T("dense_56x56_s448_c384", "affine", 256, 56, 56, 384, stride=448),
    T("dense_28x28_s544_c480_copy576", "affine", 256, 28, 28, 480, stride=544, copy=576),
    T("dense_14x14_s576_c512_copy512", "affine", 256, 14, 14, 512, stride=576, copy=512),
    T("dense_7x7_s576_c512", "affine", 256, 7, 7, 512, stride=576),
    T("affine_28x28_s104_c100_copy100", "affine", 256, 28, 28, 100, stride=104, copy=100),
]
# BinaryAlexNet / XNOR-Net: the pooled BatchNorm signs (the 13x13 -> 6x6 layer at batch 512)
MAXPOOL = [
    T("alexnet_56x56x64", "maxpool", 256, 56, 56, 64, pool=(3, 2, VALID)),
    T("alexnet_27x27x192", "maxpool", 256, 27, 27, 192, pool=(3, 2, VALID), act=RELU),
    T("alexnet_13x13x256_b512", "maxpool", 512, 13, 13, 256, pool=(3, 2, VALID)),
    T("xnornet_56x56x96", "maxpool", 256, 56, 56, 96, pool=(3, 2, VALID), act=RELU),
    T("xnornet_27x27x256", "maxpool", 256, 27, 27, 256, pool=(3, 2, VALID)),
    T("maxpool_27x27x100_same", "maxpool", 256, 27, 27, 100, pool=(3, 2, SAME)),
]
# DoReFaNet's six quantisers (the two dense ones at batch 512 and 1280)
QUANT2 = [
    T("dorefa_54x54x96", "quant2", 256, 54, 54, 96),
    T("dorefa_54x54x256_pool", "quant2", 256, 54, 54, 256, pool=(3, 2, SAME)),
    T("dorefa_27x27x384_pool", "quant2", 256, 27, 27, 384, pool=(3, 2, SAME)),
    T("dorefa_14x14x384", "quant2", 256, 14, 14, 384),
    T("dorefa_dense9216_b512", "quant2", 512, 1, 1, 9216),
    T("dorefa_dense4096_b1280", "quant2", 1280, 1, 1, 4096),
]
# MeliusNet's grouped stem at stride 2: the tiled 3x3 kernel declines it
GROUPED = [T("melius_stem_112x112x32_g4_s2", "grouped", 256, 112, 112, 32, stride=2, pool=(4, 3, 32), want=None)]


@dataclass
class Fused:
    """A binary convolution (3x3, stride 1) with a fused tail. kind: chain | gate | scale | slice |
    slice_add; width / offset: the map the slice kinds write into. zp_only: run only the
    zero-padding fallback (the one-padding epilogue has a full-size test elsewhere)."""
    name: str
    kind: str
    b: int
    hw: int
    cin: int
    cout: int
    width: int = 0
    offset: int = 0
    zp_only: bool = False

    def tail(self):
        """The one-pass launch that finishes the zero-padding form on mma.sync."""
        k = {"slice": "zpc", "slice_add": "zpc"}.get(self.kind, self.kind)
        return Tail(self.name + "_zp", k, self.b, self.hw, self.hw, self.cout, want=None if k == "zpc" else "int")


FUSED = [
    Fused("chain_56x56x128", "chain", 256, 56, 128, 128),
    Fused("chain_14x14x512", "chain", 256, 14, 512, 512),
    Fused("gate_56x56x64", "gate", 256, 56, 64, 64),
    Fused("gate_7x7x512", "gate", 256, 7, 512, 512),
    Fused("slice_56x56_384to64_w448", "slice", 256, 56, 384, 64, width=448, offset=384),
    Fused("slice_add_56x56x320", "slice_add", 256, 56, 320, 64, width=320, offset=256),
    Fused("slice_add_7x7x640_b704", "slice_add", 704, 7, 640, 64, width=640, offset=576),
    Fused("scale_56x56x64", "scale", 256, 56, 64, 64, zp_only=True),
    Fused("scale_7x7x512", "scale", 256, 7, 512, 512, zp_only=True),
]

# The 64-bit instances, and the 32-bit ones one stride below their threshold
BIG = [
    T("chain_long_c100", "chain", 1, 21_550_000, 1, 100, want="long"),
    T("gate_long_56x56x64", "gate", 10_720, 56, 56, 64, act=RELU, residual=True, want="long"),
    T("scale_long_14x14x256", "scale", 42_880, 14, 14, 256, act=N1, residual=True, want="long"),
    T("affine_long_stride63200", "affine", 1, 34_000, 1, 100, stride=63_200, copy=100, want="long"),
    T("maxpool_long_13x13x256", "maxpool", 49_700, 13, 13, 256, pool=(3, 2, VALID), want="long"),
    T("quant2_long_14x14x384", "quant2", 28_560, 14, 14, 384, want="long"),
    T("chain_edge_c96", "chain", 1, 22_358_357, 1, 96, want="edge"),
    T("gate_edge_56x56x64", "gate", 10_694, 56, 56, 64, act=RELU6, residual=True, want="edge"),
    T("scale_edge_14x14x256", "scale", 42_777, 14, 14, 256, residual=True, want="edge"),
    T("affine_edge_c64", "affine", 1, 33_537_535, 1, 64, stride=64, want="edge"),
]
BIG_FLOATS = TWO31 + (16 << 20)

FAMILY = CHAIN + GATE + SCALE + AFFINE + MAXPOOL + QUANT2 + GROUPED
TABLE = FAMILY + [f.tail() for f in FUSED] + BIG


def ids(cases):
    return [c.name for c in cases]


def test_every_case_iterates_and_selects_its_instance():
    """Each case gives every thread (warp) at least four grid-stride iterations and picks the index
    instance it is named for; the section-4 cases fit the shared buffer."""
    assert len(set(ids(TABLE))) == len(TABLE)
    for t in TABLE:
        lay = launch(t)
        assert lay["iters"] >= MIN_ITERS, (t.name, lay)
        if t.want is None:
            assert lay["wide"] is None, t.name
        elif t.want == "int":
            assert lay["wide"] is False, (t.name, lay)
        elif t.want == "long":
            assert lay["wide"] is True, (t.name, lay)
        else:   # the int instance, with one more stride of work selecting the long one
            assert lay["wide"] is False and lay["bound"] + 2 * lay["step"] >= TWO31, (t.name, lay)
    for t in BIG:
        floats = t.rows * (t.stride or t.span_c)
        assert floats <= BIG_FLOATS, t.name
        if t.want == "long" and t.kernel not in ("maxpool", "quant2"):
            assert floats > TWO31, t.name          # an element past 2^31 is read and written
    assert {t.kernel for t in BIG if t.want == "long"} == {"chain", "gate", "scale", "affine", "maxpool", "quant2"}
    assert {t.kernel for t in BIG if t.want == "edge"} == {"chain", "gate", "scale", "affine"}
    assert any(t.c % 32 for t in FAMILY if t.kernel in ("chain", "maxpool", "affine"))
    assert not any(grouped_tiled_takes(t) for t in GROUPED)


# ----------------------------------- GPU helpers ----------------------------------- #
@pytest.fixture(scope="module")
def capi():
    from compute_engine_b200 import capi as m
    m.lib()
    return m


def _vp(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ok(capi, rc):
    assert rc == 0, capi.lib().lce_b200_last_error()


def guarded(n, dtype, poison=POISON):
    """(buffer, its first n elements): every element poisoned, BAND more behind the view."""
    import torch
    buf = poisoned((n + BAND,), dtype)
    if poison != POISON:
        buf.view(torch.int32).fill_(poison)
    return buf, buf[:n]


def band_intact(buf, n, poison=POISON):
    import torch
    return bool((buf[n:].view(torch.int32) == poison).all())


def shifts(rng, c):
    """Per-channel shifts with +0, -0 and +-0.5 (exact ties against the maps' +-0.5 entries)."""
    v = rng.uniform(-0.5, 0.5, c).astype(F32)
    v[0::5], v[1::5], v[2::10], v[7::10] = F32(0.0), F32(-0.0), F32(0.5), F32(-0.5)
    return v


def scales(rng, c):
    return (rng.uniform(0.25, 1.5, c) * rng.choice([-1.0, 1.0], c)).astype(F32)


def signs(t, sc, sh):
    """MUL(sign_scale) -> ADD(sign_shift) -> LceQuantize in numpy float32."""
    s = t
    if sc is not None:
        s = (s * sc).astype(F32)
    if sh is not None:
        s = (s + sh).astype(F32)
    return L.quantize(s)


def gate_ref(y, gate, alpha, res, act, sc, sh):
    """_gate_tail_ref's MUL -> PRELU -> ADD, then the ADD's activation (any of the four), then the signs."""
    t, _ = _gate_tail_ref(y, gate, alpha, res)
    t = _act_ref(t, act)
    return t, signs(t, sc, sh)


def d(a):
    return None if a is None else dev(a)


# ------------------------- one-pass kernels at family sizes ------------------------- #
@pytest.mark.gpu
@pytest.mark.parametrize("t", CHAIN, ids=ids(CHAIN))
def test_chain_sign_at_family_size(t, capi):
    """lce_b200_f32_chain_sign over ReActNet's maps: the float output and the packed signs equal the
    op sequence in numpy over the whole output; nothing past either output is written."""
    import torch
    rng = np.random.default_rng(41000 + ids(CHAIN).index(t.name))
    rows, ch = t.rows, t.span_c
    x = _special_map(rng, (rows, ch))
    if t.kernel == "prelu":
        v = [None, rng.uniform(0.05, 0.5, ch).astype(F32), None, None]
    else:
        v = [shifts(rng, ch), rng.uniform(0.05, 0.5, ch).astype(F32), shifts(rng, ch), shifts(rng, ch)]
        v[1][::9] = F32(0.0)
    want, want_bits = _np_chain(x, v, t.packed)
    dv = [d(a) for a in v]
    from compute_engine_b200.capi import ChainDesc
    desc = ChainDesc(*[None if a is None else a.data_ptr() for a in dv])
    cw = cdiv(ch, 32)
    obuf, out = guarded(rows * ch, torch.float32) if t.out else (None, None)
    pbuf, pk = guarded(rows * cw, torch.int32) if t.packed else (None, None)
    xd = dev(x)
    _ok(capi, capi.lib().lce_b200_f32_chain_sign(_vp(xd), C.byref(desc), C.c_int64(rows), C.c_int(ch),
                                                  _vp(out), _vp(pk), _stream()))
    torch.cuda.synchronize()
    lay = launch(t)
    tag = f"{t.name} ({lay['iters']} iterations per thread)"
    if t.out:
        assert_same_bits(out.cpu().numpy().reshape(rows, ch), want, tag)
        assert band_intact(obuf, rows * ch), tag + ": wrote past the float output"
    if t.packed:
        assert_same_bits(pk.cpu().numpy().reshape(rows, cw), want_bits, tag + " signs")
        assert band_intact(pbuf, rows * cw), tag + ": wrote past the packed output"


def _tail_inputs(t, rng):
    ch, P = t.c, t.h * t.w
    y = _special_map(rng, (t.b, t.h, t.w, ch))
    res = rng.standard_normal(y.shape).astype(F32) if t.residual else None
    if res is not None:
        res.reshape(-1)[::13] = F32(-0.0)
    sc, sh = (scales(rng, ch), shifts(rng, ch)) if t.packed else (None, None)
    return y, res, sc, sh, P


def _run_in_place(capi, t, fn, desc, y, res):
    """x == out in a poisoned, banded buffer; the packed output poisoned and banded."""
    import torch
    n = y.size
    xbuf, x = guarded(n, torch.float32)
    x.copy_(torch.from_numpy(y.reshape(-1)).cuda())
    cw = cdiv(t.c, 32)
    pbuf, pk = guarded(t.b * t.h * t.w * cw, torch.int32) if t.packed else (None, None)
    r = d(res)
    _ok(capi, fn(_vp(x), C.byref(desc), _vp(r), C.c_int(t.act), C.c_int64(t.b), C.c_int64(t.h * t.w),
                 C.c_int(t.c), _vp(x), _vp(pk), _stream()))
    torch.cuda.synchronize()
    tag = f"{t.name} ({launch(t)['iters']} iterations per thread)"
    assert band_intact(xbuf, n), tag + ": wrote past the map"
    if t.packed:
        assert band_intact(pbuf, pk.numel()), tag + ": wrote past the packed output"
    return x.cpu().numpy().reshape(y.shape), None if pk is None else pk.cpu().numpy().reshape(y.shape[:3] + (cw,)), tag


@pytest.mark.gpu
@pytest.mark.parametrize("t", GATE, ids=ids(GATE))
def test_gate_sign_in_place_at_family_size(t, capi):
    """lce_b200_f32_gate_sign in place over Real-to-Binary Net's maps: every image takes its own
    gate row on every iteration; whole output and signs against numpy."""
    from compute_engine_b200.capi import GateDesc
    rng = np.random.default_rng(42000 + ids(GATE).index(t.name))
    y, res, sc, sh, _ = _tail_inputs(t, rng)
    gate = rng.uniform(0, 1, (t.b, t.c)).astype(F32)
    gate[:, ::11] = F32(0.0)
    alpha = rng.uniform(0.05, 0.5, t.c).astype(F32) if t.alpha else None
    keep = [d(a) for a in (gate, alpha, sc, sh)]
    desc = GateDesc(*[None if a is None else a.data_ptr() for a in keep])
    got, bits, tag = _run_in_place(capi, t, capi.lib().lce_b200_f32_gate_sign, desc, y, res)
    want, want_bits = gate_ref(y, gate, alpha, res, t.act, sc, sh)
    assert_same_bits(got, want, tag)
    if t.packed:
        assert_same_bits(bits, want_bits, tag + " signs")


@pytest.mark.gpu
@pytest.mark.parametrize("t", SCALE, ids=ids(SCALE))
def test_scale_sign_in_place_at_family_size(t, capi):
    """lce_b200_f32_scale_sign in place over XNOR-Net++'s maps: every row takes its own position's
    scale row on every iteration; whole output and signs against numpy."""
    from compute_engine_b200.capi import ScaleDesc
    rng = np.random.default_rng(43000 + ids(SCALE).index(t.name))
    y, res, sc, sh, _ = _tail_inputs(t, rng)
    scale = rng.uniform(0.5, 1.5, (t.h, t.w, t.c)).astype(F32)
    scale.reshape(-1)[::17] = F32(-0.0)
    keep = [d(a) for a in (scale, sc, sh)]
    desc = ScaleDesc(*[None if a is None else a.data_ptr() for a in keep])
    got, bits, tag = _run_in_place(capi, t, capi.lib().lce_b200_f32_scale_sign, desc, y, res)
    want, want_bits = _scale_tail_ref(y, scale, res, t.act, sc, sh)
    assert_same_bits(got, want, tag)
    assert_same_bits(bits, want_bits, tag + " signs")


@pytest.mark.gpu
@pytest.mark.parametrize("t", AFFINE, ids=ids(AFFINE))
def test_affine_sign_at_family_size(t, capi):
    """lce_b200_f32_affine_sign over a dense block's leading channels: the signs of the whole map
    against numpy; copy_to receives those channels bit for bit and keeps its other channels."""
    import torch
    rng = np.random.default_rng(44000 + ids(AFFINE).index(t.name))
    rows, ch, cw = t.rows, t.c, cdiv(t.c, 32)
    x = _special_map(rng, (rows, t.stride))
    sc, sh = scales(rng, ch), shifts(rng, ch)
    pbuf, pk = guarded(rows * cw, torch.int32)
    cbuf, cp = guarded(rows * t.copy, torch.float32) if t.copy else (None, None)
    vs, vh = d(sc), d(sh)
    xd = dev(x)
    _ok(capi, capi.lib().lce_b200_f32_affine_sign(_vp(xd), C.c_int64(t.stride), C.c_int64(rows), C.c_int(ch),
                                                   _vp(vs), _vp(vh), _vp(pk), _vp(cp), C.c_int64(t.copy),
                                                   _stream()))
    torch.cuda.synchronize()
    tag = f"{t.name} ({launch(t)['iters']} iterations per thread)"
    lead = x[:, :ch]
    assert_same_bits(pk.cpu().numpy().reshape(rows, cw), signs(lead, sc, sh), tag)
    assert band_intact(pbuf, rows * cw), tag + ": wrote past the packed output"
    if t.copy:
        got = cp.cpu().numpy().reshape(rows, t.copy)
        assert_same_bits(got[:, :ch], lead, tag + " copy")
        assert (got[:, ch:].view(np.int32) == POISON).all(), tag + ": the copy wrote past its channels"
        assert band_intact(cbuf, rows * t.copy), tag + ": wrote past the copy"


@pytest.mark.gpu
@pytest.mark.parametrize("t", MAXPOOL, ids=ids(MAXPOOL))
def test_maxpool_affine_sign_at_family_size(t, capi):
    """lce_b200_f32_maxpool_affine_sign over the pooled layers: every warp's later words take their
    own image's window; the whole packed output against numpy."""
    import torch
    rng = np.random.default_rng(45000 + ids(MAXPOOL).index(t.name))
    k, s, padding = t.pool
    x = _special_map(rng, (t.b, t.h, t.w, t.c))
    sc, sh = scales(rng, t.c), shifts(rng, t.c)
    lay = launch(t)
    shape = (t.b, lay["oh"], lay["ow"], cdiv(t.c, 32))
    n = int(np.prod(shape))
    pbuf, pk = guarded(n, torch.int32)
    vs, vh = d(sc), d(sh)
    xd = dev(x)
    _ok(capi, capi.lib().lce_b200_f32_maxpool_affine_sign(_vp(xd), t.b, t.h, t.w, t.c, k, k, s, s, padding,
                                                           t.act, _vp(vs), _vp(vh), _vp(pk), _stream()))
    torch.cuda.synchronize()
    tag = f"{t.name} ({lay['iters']} words per warp)"
    want = _np_pooled_signs(x, (k, k), (s, s), "SAME" if padding == SAME else "VALID",
                            "RELU" if t.act == RELU else "NONE", sc, sh)
    assert_same_bits(pk.cpu().numpy().reshape(shape), want, tag)
    assert band_intact(pbuf, n), tag + ": wrote past the packed output"


@pytest.mark.gpu
@pytest.mark.parametrize("t", QUANT2, ids=ids(QUANT2))
def test_quant2_planes_at_family_size(t, capi):
    """lce_b200_f32_quant2_planes over DoReFaNet's quantiser inputs, with and without the pool: the
    whole plane output against MAXIMUM -> MINIMUM -> MUL -> ROUND in numpy float32."""
    import torch
    rng = np.random.default_rng(46000 + ids(QUANT2).index(t.name))
    x = _special_map(rng, (t.b, t.h, t.w, t.c))
    lay = launch(t)
    shape = (t.b, lay["oh"], lay["ow"], 3 * t.c // 32)
    n = int(np.prod(shape))
    pbuf, planes = guarded(n, torch.int32)
    k, s, padding = t.pool if t.pool is not None else (0, 1, VALID)
    xd = dev(x)
    _ok(capi, capi.lib().lce_b200_f32_quant2_planes(_vp(xd), t.b, t.h, t.w, t.c, k, k, s, s, padding, NONE,
                                                     _vp(planes), _stream()))
    torch.cuda.synchronize()
    tag = f"{t.name} ({lay['iters']} words per warp)"
    v = x if t.pool is None else np_maxpool(x, k, s, "SAME" if padding == SAME else "VALID")
    levels = np_levels(v)
    assert all((levels == F32(q)).any() for q in range(4)), tag
    want = np_planes(levels)
    assert_same_bits(planes.cpu().numpy().reshape(shape), want, tag)
    assert band_intact(pbuf, n), tag + ": wrote past the planes"


@pytest.mark.gpu
@pytest.mark.parametrize("t", GROUPED, ids=ids(GROUPED))
def test_grouped_conv_fallback_at_family_size(t, capi):
    """grouped_conv_any_kernel on a MeliusNet-stem-sized map the tiled kernel declines: the first,
    middle and last image against the per-group convolution in numpy, every output written."""
    import torch
    rng = np.random.default_rng(47000)
    groups, k, cout = t.pool
    x = _special_map(rng, (t.b, t.h, t.w, t.c))
    w = (rng.standard_normal((cout, k, k, t.c // groups)) * 0.5).astype(F32)
    bias, sc, sh = rng.standard_normal(cout).astype(F32), scales(rng, cout), shifts(rng, cout)
    lay = launch(t)
    shape = (t.b, lay["oh"], lay["ow"], cout)
    n = int(np.prod(shape))
    obuf, out = guarded(n, torch.float32)
    xd, wd, bd, sd, hd = dev(x), dev(w), dev(bias), dev(sc), dev(sh)
    capi.grouped_conv2d(xd, wd, bd, (t.stride, t.stride), (1, 1), capi.PADDING_SAME, RELU, sd, hd, RELU6,
                        out=out.view(shape))
    torch.cuda.synchronize()
    tag = f"{t.name} ({lay['iters']} iterations per thread)"
    assert band_intact(obuf, n), tag + ": wrote past the output"
    assert not bool((out.view(torch.int32) == POISON).any()), tag + ": outputs left unwritten"
    sel = [0, t.b // 2, t.b - 1]
    want = _grouped_ref(x[sel], w, bias, groups, (t.stride, t.stride), (1, 1), SAME, RELU, sc, sh, RELU6)
    assert_same_bits(out.view(shape)[torch.tensor(sel, device="cuda")].cpu().numpy(), want, tag)


# ------------------- fused mma.sync epilogues and their fallbacks ------------------- #
FORMS = {"one_padding": 1, "zero_padding": 0}


@pytest.mark.gpu
@pytest.mark.parametrize("f", FUSED, ids=ids(FUSED))
def test_fused_tail_at_family_size(f, capi, monkeypatch):
    """The binary convolution with its fused tail at batch 256 (one-padding: the mma.sync epilogue;
    zero padding, CORRECTION: the convolution on mma.sync, then the one-pass tail or zpc_tail_kernel),
    on b1 and on int8: the launch counters name mma.sync; three images equal the oracle convolution
    followed by the numpy tail; b1 and int8 give the same whole outputs, written into buffers (and,
    for run_slice, a slice) poisoned with different values; run_slice_add changes every element of
    its slice, whose initial values are small enough that no sum rounds back to them; the slice
    kinds leave every other channel of the map at its sentinel and nothing behind the map."""
    import torch
    from compute_engine_b200.capi import ChainDesc, GateDesc, ScaleDesc
    n_case = ids(FUSED).index(f.name)
    rng = np.random.default_rng(48000 + n_case)
    M = f.b * f.hw * f.hw
    cw = cdiv(f.cout, 32)
    act = ACTS[n_case % 4]
    sel = np.array([0, f.b // 2, f.b - 1])
    sel_t = torch.from_numpy(sel).cuda()
    gen = torch.Generator(device="cuda").manual_seed(n_case)
    res = None
    if f.kind in ("chain", "gate", "scale"):
        res = torch.randn((f.b, f.hw, f.hw, f.cout), device="cuda", generator=gen)
        res_sel = res[sel_t].cpu().numpy()
    vecs = {}
    if f.kind == "chain":
        vecs["v"] = [shifts(rng, f.cout), rng.uniform(0.05, 0.5, f.cout).astype(F32), shifts(rng, f.cout),
                     shifts(rng, f.cout)]
    elif f.kind == "gate":
        vecs["gate"] = rng.uniform(0, 1, (f.b, f.cout)).astype(F32)
        vecs["v"] = [rng.uniform(0.05, 0.5, f.cout).astype(F32), scales(rng, f.cout), shifts(rng, f.cout)]
    elif f.kind == "scale":
        vecs["scale"] = rng.uniform(0.5, 1.5, (f.hw, f.hw, f.cout)).astype(F32)
        vecs["v"] = [scales(rng, f.cout), shifts(rng, f.cout)]
    keep = {k: ([d(a) for a in v] if isinstance(v, list) else d(v)) for k, v in vecs.items()}
    init = None
    if f.kind == "slice_add":
        init = torch.randn((M, f.cout), device="cuda", generator=gen) * 2.0**-20
        init_sel = init.view(f.b, f.hw, f.hw, f.cout)[sel_t].cpu().numpy()
    for form, pv in FORMS.items():
        if f.zp_only and form == "one_padding":
            continue
        spec = S(f.name, f.b, f.hw, f.hw, f.cin, 3, 3, f.cout, pv=pv, corr=pv == 0)
        case = make_case(spec, 48100 + 2 * n_case + pv)
        x = dev(case.inp)
        sub = L.BconvDesc.from_buffer_copy(case.desc)
        sub.batch = len(sel)
        y = L.bconv2d(sub, case.inp[sel], case.filt, case.mul, case.bias, None, kind=1 - pv, threads=THREADS)
        if f.kind == "chain":
            s = _act_ref((y + res_sel).astype(F32), act)
            wants = _np_chain(s, vecs["v"], True)
        elif f.kind == "gate":
            wants = gate_ref(y, vecs["gate"][sel], vecs["v"][0], res_sel, act, *vecs["v"][1:])
        elif f.kind == "scale":
            wants = _scale_tail_ref(y, vecs["scale"], res_sel, act, *vecs["v"])
        elif f.kind == "slice":
            wants = (y,)
        else:
            wants = ((init_sel + y).astype(F32),)
        results = {}
        for env, poison in (("b1", POISON), ("int8", POISON2)):
            set_env(monkeypatch, env)
            plan = capi.BConv2d(gpu_desc(capi, case.desc), case.filt, case.mul, case.bias)
            if pv == 0:
                plan.set_zero_padding_mode(1)
            tag = f"{f.name} {form} on {env}"
            before = path_counts(capi)
            lib, h, s_ = capi.lib(), plan._h, _stream()
            if f.kind in ("chain", "gate", "scale"):
                obuf, out = guarded(M * f.cout, torch.float32, poison)
                pbuf, pk = guarded(M * cw, torch.int32, poison)
                v = keep["v"]
                if f.kind == "chain":
                    desc = ChainDesc(*[a.data_ptr() for a in v])
                    rc = lib.lce_b200_bconv2d_run_fused_chain(h, _vp(x), _vp(res), C.c_int(act), C.byref(desc),
                                                              _vp(out), _vp(pk), s_)
                elif f.kind == "gate":
                    desc = GateDesc(keep["gate"].data_ptr(), *[a.data_ptr() for a in v])
                    rc = lib.lce_b200_bconv2d_run_fused_gate(h, _vp(x), C.byref(desc), _vp(res), C.c_int(act),
                                                             _vp(out), _vp(pk), s_)
                else:
                    desc = ScaleDesc(keep["scale"].data_ptr(), *[a.data_ptr() for a in v])
                    rc = lib.lce_b200_bconv2d_run_fused_scale(h, _vp(x), C.byref(desc), _vp(res), C.c_int(act),
                                                              _vp(out), _vp(pk), s_)
                _ok(capi, rc)
                torch.cuda.synchronize()
                assert band_intact(obuf, M * f.cout, poison) and band_intact(pbuf, M * cw, poison), tag
                outs = [out.view(f.b, f.hw, f.hw, f.cout), pk.view(f.b, f.hw, f.hw, cw)]
            else:
                iobuf, io = guarded(M * f.width, torch.float32, poison)
                io = io.view(M, f.width)
                io.fill_(float(SENTINEL))
                if init is not None:
                    io[:, f.offset:f.offset + f.cout] = init
                else:   # run_slice must write every element of its slice
                    io.view(torch.int32)[:, f.offset:f.offset + f.cout].fill_(poison)
                ptr = C.c_void_p(io.data_ptr() + 4 * f.offset)
                if f.kind == "slice":
                    rc = lib.lce_b200_bconv2d_run_slice(h, _vp(x), ptr, C.c_int64(f.width), s_)
                else:
                    sbuf, scratch = guarded(M * f.cout, torch.float32, poison)
                    rc = lib.lce_b200_bconv2d_run_slice_add(h, _vp(x), ptr, C.c_int64(f.width),
                                                            _vp(scratch if pv == 0 else None), s_)
                _ok(capi, rc)
                torch.cuda.synchronize()
                rest = torch.cat([io[:, :f.offset], io[:, f.offset + f.cout:]], 1)
                assert bool((rest == float(SENTINEL)).all()), tag + ": wrote outside its slice"
                assert band_intact(iobuf, M * f.width, poison), tag + ": wrote past the map"
                if init is not None:
                    unchanged = io[:, f.offset:f.offset + f.cout].view(torch.int32) == init.view(torch.int32)
                    assert not bool(unchanged.any()), tag + ": slice elements left unchanged"
                if f.kind == "slice_add":
                    assert band_intact(sbuf, M * f.cout, poison), tag + ": wrote past the scratch"
                outs = [io[:, f.offset:f.offset + f.cout].contiguous().view(f.b, f.hw, f.hw, f.cout)]
                del io, iobuf
            ran = [b - a for a, b in zip(before, path_counts(capi))]
            plan.close()
            assert ran == [0, 1, 0], (tag, ran)
            for what, got, want in zip(("output", "signs"), outs, wants):
                assert_same_bits(got[sel_t].cpu().numpy(), want, f"{tag}: {what} vs the oracle")
            results[env] = outs
        for what, a, b in zip(("output", "signs"), results["b1"], results["int8"]):
            assert same_bits(a, b), f"{f.name} {form}: b1 and int8 {what} differ"
        del results


# ------------------------- 64-bit index instances (2^31 + 16 M floats) ------------------------- #
PEAK_LIMIT = 12 * 10**9       # bytes: the section's peak device allocation, buffer included


@pytest.fixture(scope="module")
def big(pytestconfig):
    """A holder of one device buffer of 2^31 + 16 M floats (8.6 GB) shared by the section's cases.
    pytest keeps the yielded object alive until after teardown, so the tests read holder["buf"] and
    teardown empties the holder, then returns the memory to the device. Teardown reports the
    section's peak device allocation on the terminal, past pytest's output capture."""
    import torch
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    holder = {"buf": torch.empty(BIG_FLOATS, dtype=torch.float32, device="cuda"), "peak": 0}
    yield holder
    peak = holder["peak"]
    holder.clear()
    torch.cuda.empty_cache()
    capman = pytestconfig.pluginmanager.getplugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print(f"\n64-bit index cases: peak device memory {peak / 2**30:.2f} GiB "
              f"(limit {PEAK_LIMIT / 2**30:.2f} GiB); reserved after teardown "
              f"{torch.cuda.memory_reserved() / 2**30:.2f} GiB")


def _check_rows(n_rows, straddles):
    """The first two rows, the rows either side of each straddling index, the last two rows."""
    picks = {0, 1, n_rows - 2, n_rows - 1}
    for r in straddles:
        picks |= {r - 1, r, r + 1}
    return np.array(sorted(p for p in picks if 0 <= p < n_rows), np.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("t", BIG, ids=ids(BIG))
def test_index_instances_past_2_pow_31(t, big, capi):
    """Each one-pass kernel on the long long instance (an element, or an input pixel, past 2^31) and
    the elementwise kernels' int instance one stride below its threshold, in place where the kernel
    allows it: the rows around element 2^31 (and packed word 2^26) and the last rows against numpy.
    Each case runs twice, refilled from the same seed, into packed outputs poisoned with different
    values: equal results mean every packed word was written; neither poison band is touched."""
    import torch
    from compute_engine_b200.capi import ChainDesc, GateDesc, ScaleDesc
    n_case = ids(BIG).index(t.name)
    rng = np.random.default_rng(49000 + n_case)
    lay = launch(t)
    assert lay["wide"] is (t.want == "long"), lay
    buf = big["buf"]
    lib = capi.lib()
    ch = t.c
    cw = cdiv(ch, 32)
    keep = []

    if t.kernel in ("chain", "gate", "scale", "affine"):
        width = t.stride or ch
        rows = t.rows
        x = buf[:rows * width].view(rows, width)
        e_row = TWO31 // width
        p_row = (1 << 26) // cw
        picks = _check_rows(rows, [e_row, p_row] if t.want == "long" else [rows - 1])
        n_pk = rows * cw
    elif t.kernel == "maxpool":
        per = t.h * t.w * t.c
        x = buf[:t.b * per].view(t.b, t.h, t.w, t.c)
        picks = _check_rows(t.b, [TWO31 // per])
        n_pk = t.b * lay["oh"] * lay["ow"] * cw
    else:   # quant2, no pool: one row per pixel
        rows = t.b * t.h * t.w
        x = buf[:rows * ch].view(rows, ch)
        picks = _check_rows(rows, [TWO31 // ch, (1 << 26) // (3 * cw)])
        n_pk = rows * 3 * cw
    picks_t = torch.from_numpy(picks).cuda()
    special = _special_map(rng, (len(picks),) + tuple(x.shape[1:]))

    if t.kernel == "chain":
        v = [shifts(rng, ch), rng.uniform(0.05, 0.5, ch).astype(F32), shifts(rng, ch), shifts(rng, ch)]
        keep = [d(a) for a in v]
        desc = ChainDesc(*[a.data_ptr() for a in keep])

        def call(pk, cp):
            return lib.lce_b200_f32_chain_sign(_vp(x), C.byref(desc), C.c_int64(rows), C.c_int(ch), _vp(x), _vp(pk),
                                               _stream())

        def ref(xs):
            return _np_chain(xs, v, True)
    elif t.kernel in ("gate", "scale"):
        P = t.h * t.w
        sc, sh = scales(rng, ch), shifts(rng, ch)
        if t.kernel == "gate":
            g = rng.uniform(0, 1, (t.b, ch)).astype(F32)
            alpha = rng.uniform(0.05, 0.5, ch).astype(F32)
            keep = [d(a) for a in (g, alpha, sc, sh)]
            desc = GateDesc(*[a.data_ptr() for a in keep])
            fn = lib.lce_b200_f32_gate_sign
        else:
            g = rng.uniform(0.5, 1.5, (P, ch)).astype(F32)
            keep = [d(a) for a in (g, sc, sh)]
            desc = ScaleDesc(*[a.data_ptr() for a in keep])
            fn = lib.lce_b200_f32_scale_sign

        def call(pk, cp):   # x is the input, the residual and the output
            return fn(_vp(x), C.byref(desc), _vp(x), C.c_int(t.act), C.c_int64(t.b), C.c_int64(P), C.c_int(ch),
                      _vp(x), _vp(pk), _stream())

        def ref(xs):
            if t.kernel == "gate":
                t_, bits = gate_ref(xs[:, None, None], g[picks // P], alpha, xs[:, None, None], t.act, sc, sh)
            else:
                t_, bits = _scale_tail_ref(xs[None, :, None], g[picks % P][:, None], xs[None, :, None], t.act, sc, sh)
            return t_.reshape(xs.shape), bits.reshape(len(xs), cw)
    elif t.kernel == "affine":
        sc, sh = scales(rng, ch), shifts(rng, ch)
        keep = [d(sc), d(sh)]

        def call(pk, cp):
            return lib.lce_b200_f32_affine_sign(_vp(x), C.c_int64(t.stride), C.c_int64(rows), C.c_int(ch),
                                                _vp(keep[0]), _vp(keep[1]), _vp(pk), _vp(cp), C.c_int64(t.copy),
                                                _stream())

        def ref(xs):
            return None, signs(xs[:, :ch], sc, sh)
    elif t.kernel == "maxpool":
        k, s, padding = t.pool
        sc, sh = scales(rng, ch), shifts(rng, ch)
        keep = [d(sc), d(sh)]

        def call(pk, cp):
            return lib.lce_b200_f32_maxpool_affine_sign(_vp(x), t.b, t.h, t.w, ch, k, k, s, s, padding, t.act,
                                                        _vp(keep[0]), _vp(keep[1]), _vp(pk), _stream())

        def ref(xs):
            return None, _np_pooled_signs(xs, (k, k), (s, s), "VALID" if padding == VALID else "SAME", "NONE", sc, sh)
    else:
        def call(pk, cp):
            return lib.lce_b200_f32_quant2_planes(_vp(x), t.b, t.h, t.w, ch, 0, 0, 1, 1, VALID, NONE, _vp(pk),
                                                  _stream())

        def ref(xs):
            return None, np_planes(np_levels(xs))

    first = pbuf = pk = cbuf = cp = None
    try:
        for poison in (POISON, POISON2):
            gen = torch.Generator(device="cuda").manual_seed(n_case)
            x.normal_(generator=gen)
            x[picks_t] = torch.from_numpy(special).cuda()
            pbuf, pk = guarded(n_pk, torch.int32, poison)
            cbuf, cp = guarded(rows * t.copy, torch.float32, poison) if t.copy else (None, None)
            _ok(capi, call(pk, cp))
            torch.cuda.synchronize()
            tag = f"{t.name} ({t.want} instance, poison {poison:#x})"
            assert band_intact(pbuf, n_pk, poison), tag + ": wrote past the packed output"
            if cp is not None:
                assert band_intact(cbuf, rows * t.copy, poison), tag + ": wrote past the copy"
            if first is None:
                want_x, want_bits = ref(special)
                if t.kernel == "maxpool":
                    got_bits = pk.view(t.b, lay["oh"], lay["ow"], cw)[picks_t].cpu().numpy()
                else:
                    got_bits = pk.view(-1, pk.numel() // x.shape[0])[picks_t].cpu().numpy()
                assert_same_bits(got_bits, want_bits.reshape(got_bits.shape), tag + ": signs")
                if want_x is not None:
                    assert_same_bits(x[picks_t].cpu().numpy(), want_x, tag + ": float output")
                if cp is not None:
                    got = cp.view(rows, t.copy)[picks_t].cpu().numpy()
                    assert_same_bits(got, special[:, :ch], tag + ": copy")
                first = (pk.clone(), None if cp is None else cp.clone())
            else:
                assert same_bits(pk, first[0]), tag + ": packed words left unwritten"
                if cp is not None:
                    assert same_bits(cp, first[1]), tag + ": copy elements left unwritten"
            del pbuf, pk, cbuf, cp
    finally:   # a failing case must not keep its outputs, or a view of the buffer, alive in its traceback
        first = pbuf = pk = cbuf = cp = x = buf = None
    peak = torch.cuda.max_memory_allocated()
    big["peak"] = max(big["peak"], peak)
    assert peak < PEAK_LIMIT, f"peak device memory {peak / 2**30:.2f} GiB"
