"""The binary convolution's kernels at full launch sizes, through the C-ABI, against the oracle and
against each other.

The wgmma kernel (lce_b200_tc.cuh) is persistent: it launches min(items, ctas x SMs) CTAs and each
CTA walks item += gridDim.x, carrying the halo ring's slot and parity, the weight ring's slot and
parity and the resident-weight state from one item to the next. Every case here gives each CTA at
least four items on a 132-SM H100. `tc_layout` restates tc_launch's arithmetic (lce_b200.cu), and a
CPU test checks that each case reaches the layout it is meant to exercise (channel chunks, flat
halos, resident or ring weights, one or two CTAs per SM).

On the GPU each case runs on every kernel that can take it, chosen by LCE_B200_BCONV_IMMA / _B1 /
_TC (read when a plan is created): the b1 and int8 mma.sync kernels, wgmma, XOR + POPC; zero-padding
CORRECTION plans are finished by zpc_tail_kernel on the kernels other than wgmma. The launch
counters show which kernel ran; the whole outputs of all kernels are equal bit for bit, and the
first, a middle and the last image equal the oracle (the last image is in every CTA's final item).
No CUDA graphs are captured, so the file's place in the run order does not matter.
"""
import ctypes as C
import os
from dataclasses import dataclass, field

import numpy as np
import pytest

import lce_testlib as L
from test_bitpacked_b1 import spread_thresholds
from test_gpu_parity import assert_same_bits, dev, gpu_desc, path_counts

SAME, VALID = L.PADDING_SAME, L.PADDING_VALID
NONE, RELU, N1, RELU6 = L.ACT_NONE, L.ACT_RELU, L.ACT_RELU_N1_TO_1, L.ACT_RELU6
FLOAT, INT8, BITPACKED = L.OUT_FLOAT, L.OUT_INT8, L.OUT_BITPACKED
TC, IMMA, XOR = 0, 1, 2                  # slots of lce_b200_path_counts
H100_SMS = 132
MIN_ITEMS_PER_CTA = 4

# lce::tc constants (lce_b200_tc.cuh) and tc_launch's shared-memory budgets (lce_b200.cu)
KBM, KWS, KNR, KMAXNB, KMAXRING, KBAR = 128, 8, 2, 32, 4, 1024
HALF_BUDGET = (227 * 1024 // 2 - 1024) & ~1023
FULL_BUDGET = 226 * 1024


@dataclass
class Spec:
    name: str
    b: int
    h: int
    w: int
    cin: int
    fh: int
    fw: int
    cout: int
    stride: tuple = (1, 1)
    dil: tuple = (1, 1)
    pad: int = SAME
    pv: int = 1
    out: int = FLOAT
    act: int = NONE
    corr: bool = False          # zero padding with the optimised kernels' float correction
    gemm: bool = False          # a BGEMM: b rows of cin / 32 words, 1 x 1 "images"
    target: dict = field(default_factory=dict)

    @property
    def taps(self):
        return self.fh * self.fw


def geometry(s):
    """(OH, OW, pad_h, pad_w): out_size / pad_before of lce_b200.cu."""
    def one(size, k, st, d):
        eff = (k - 1) * d + 1
        o = (size + st - 1) // st if s.pad == SAME else (size + st - eff) // st
        return o, max((o - 1) * st + eff - size, 0) // 2
    oh, ph = one(s.h, s.fh, s.stride[0], s.dil[0])
    ow, pw = one(s.w, s.fw, s.stride[1], s.dil[1])
    return oh, ow, ph, pw


def max_halo_px(s):
    """tc_max_halo_px: the most input pixels the taps of one 128-pixel tile touch."""
    oh, ow, ph, pw = geometry(s)
    M = s.b * oh * ow
    total = s.b * s.h * s.w
    m0 = np.arange(0, M, KBM, dtype=np.int64)
    m1 = np.minimum(m0 + KBM, M) - 1

    def flat(m, fy, fx):
        b, r = np.divmod(m, oh * ow)
        oy, ox = np.divmod(r, ow)
        return (b * s.h + oy * s.stride[0] - ph + fy * s.dil[0]) * s.w + (ox * s.stride[1] - pw + fx * s.dil[1])
    lo = np.minimum(np.maximum(flat(m0, 0, 0), 0), total - 1)
    hi = np.minimum(flat(m1, s.fh - 1, s.fw - 1) + 1, total)
    return int(max(1, np.maximum(hi - lo, 1).max()))


def tc_layout(s, sms=H100_SMS):
    """build_tc_weights + tc_launch on an aligned fresh buffer: the wgmma kernel's launch, or None
    where that kernel refuses the plan."""
    zero_pad = s.pad == SAME and s.pv == 0
    if s.out == FLOAT and (s.cout % 4 or s.cout < 32):
        return None
    if zero_pad and s.taps > 64:
        return None
    cw = L.cdiv(s.cin, 32)
    bn = 64 if s.cout > 32 else 32
    n_tiles = L.cdiv(s.cout, bn)
    if cw % 4 == 0:
        flat, v, ccb = False, 4, min(cw, 32)
    else:
        flat, v, ccb = True, (2 if cw % 2 == 0 else 1), cw
        if cw > 64:
            return None
    n_chunks = L.cdiv(cw, ccb)
    cc_last = cw - (n_chunks - 1) * ccb
    s_t = (n_chunks - 1) * L.cdiv(s.taps * ccb, KWS) + L.cdiv(s.taps * cc_last, KWS)
    oh, ow, _, _ = geometry(s)
    M = s.b * oh * ow
    if M >= 2**31 or s.b * s.h * s.w * cw >= 2**31:
        return None
    max_px = max_halo_px(s)
    if flat:
        raw = L.cdiv(max_px * cw + 3, 256) * 1024
    else:
        raw = L.cdiv(max_px, 128) * 128 * ccb * 4
    raw = (raw + 1023) & ~1023
    stage = bn * 32 * KWS
    resident = (bn * 32 * s.taps * cw + 1023) & ~1023
    fixed = KNR * raw + KBAR
    ctas = 2 if fixed + 2 * stage <= HALF_BUDGET else 1
    budget = HALF_BUDGET if ctas == 2 else FULL_BUDGET
    if fixed + 2 * stage > budget:
        return None
    room = budget - fixed
    b_resident = n_tiles == 1 and s_t <= KMAXNB and room >= resident
    n_b = s_t if b_resident else min(KMAXRING, room // stage)
    m_tiles = L.cdiv(M, KBM)
    items = n_tiles * m_tiles
    grid = min(items, ctas * sms)
    return dict(BN=bn, n_tiles=n_tiles, m_tiles=m_tiles, flat=flat, V=v, CcB=ccb, chunks=n_chunks,
                cc_last=cc_last, S_t=s_t, max_px=max_px, raw_stage=raw, ctas=ctas,
                resident=b_resident, nB=n_b, items=items, grid=grid, per_cta=items // grid)


def imma_takes(s):
    """The mma.sync kernel's plan rule (build_core_weights) with an aligned output (takes_imma)."""
    return s.out != INT8 and s.cout % 64 == 0


# Which kernel each environment selects: (IMMA, B1, TC)
ENVS = {"default": ("1", "1", "1"), "b1": ("1", "1", "0"), "int8": ("1", "0", "0"),
        "wgmma": ("0", "1", "1"), "xor": ("0", "1", "0")}


def expected_path(s, env):
    imma_on, _, tc_on = ENVS[env]
    tc = tc_on == "1" and tc_layout(s) is not None
    imma = imma_on == "1" and imma_takes(s)
    if s.corr and tc:          # the CORRECTION epilogue is the wgmma kernel's; others need a tail
        return TC
    return IMMA if imma else TC if tc else XOR


def kernels_for(s):
    """(environment, launch-counter slot) of every kernel that can take the plan."""
    runs = [("default", expected_path(s, "default"))]
    if imma_takes(s):
        if s.corr and runs[0][1] != IMMA:
            runs.append(("b1", IMMA))
        runs.append(("int8", IMMA))
    if tc_layout(s) is not None and runs[0][1] != TC:
        runs.append(("wgmma", TC))
    runs.append(("xor", XOR))
    return runs


S = Spec


# the distinct shapes of Bi-RealNet-18's 16 binary 3x3 convolutions: (in hw, cin, cout, stride)
BIREALNET = [(56, 64, 64, 1), (56, 64, 128, 2), (28, 128, 128, 1), (28, 128, 256, 2), (14, 256, 256, 1),
             (14, 256, 512, 2), (7, 512, 512, 1)]
BIREALNET_BATCH = {(56, 1): 64, (56, 2): 128, (28, 1): 128, (28, 2): 256, (14, 1): 256, (14, 2): 512,
                   (7, 1): 512}

CASES = [
    # Bi-RealNet-18, zero padding, CORRECTION (what the model's default registration computes)
    *[S(f"birealnet_{hw}x{hw}x{ci}-{co}s{st}", BIREALNET_BATCH[hw, st], hw, hw, ci, 3, 3, co, (st, st),
        pv=0, corr=True) for hw, ci, co, st in BIREALNET],
    S("corr_5x5", 192, 28, 28, 128, 5, 5, 64, pv=0, corr=True),
    S("corr_odd_s2", 384, 27, 23, 96, 3, 3, 192, (2, 2), pv=0, corr=True),
    S("corr_odd_5x5_s2", 1024, 15, 17, 64, 5, 5, 128, (2, 2), pv=0, corr=True, target={"flat": True}),
    # int8 output (wgmma or XOR + POPC only), multipliers of either sign and zero
    S("int8_28x28x128-128", 128, 28, 28, 128, 3, 3, 128, out=INT8, act=RELU),
    S("int8_cout72", 128, 28, 28, 128, 3, 3, 72, pv=0, out=INT8),
    S("int8_14x14x256-200_s2", 1024, 14, 14, 256, 3, 3, 200, (2, 2), out=INT8, act=N1),
    # bitpacked output with spread thresholds, one- and zero-padding
    S("bp_alexnet_13x13x384", 256, 13, 13, 384, 3, 3, 384, out=BITPACKED),
    S("bp_alexnet_13x13x384_zp", 256, 13, 13, 384, 3, 3, 384, pv=0, out=BITPACKED),
    S("bp_56x56x64", 256, 56, 56, 64, 3, 3, 64, out=BITPACKED),
    S("bp_56x56x64_zp", 256, 56, 56, 64, 3, 3, 64, pv=0, out=BITPACKED),
    S("bp_cout36", 256, 28, 28, 128, 3, 3, 36, out=BITPACKED, target={"BN": 64}),
    # channels_out not a whole number of 64-channel tiles
    S("cout32", 256, 28, 28, 128, 3, 3, 32, act=RELU, target={"BN": 32}),
    S("cout36", 256, 28, 28, 128, 3, 3, 36, pv=0, corr=True),
    S("cout96", 128, 28, 28, 128, 3, 3, 96, act=RELU6),
    S("cout160", 64, 28, 28, 256, 3, 3, 160, pv=0, corr=True),
    # more than one channel chunk in the 2-D halo mode, and the flat mode with odd words
    S("cin1280_14x14", 128, 14, 14, 1280, 3, 3, 512, target={"chunks": 2, "cc_last": 8}),
    S("cin1280_7x7_zp", 384, 7, 7, 1280, 3, 3, 512, pv=0, corr=True, target={"chunks": 2, "cc_last": 8}),
    S("cin2048_7x7", 384, 7, 7, 2048, 3, 3, 512, act=RELU, target={"chunks": 2, "cc_last": 32}),
    S("cin2048_14x14_zp", 256, 14, 14, 2048, 3, 3, 256, pv=0, out=INT8, target={"chunks": 2}),
    S("cin1056_flat", 256, 14, 14, 1056, 3, 3, 256, target={"flat": True, "V": 1}),
    S("bgemm_kw256", 100_000, 1, 1, 256 * 32, 1, 1, 128, pad=VALID, gemm=True, target={"chunks": 8}),
    # resident weights, a ring with one n-tile, a ring with eight
    S("resident_28x28x128-64", 192, 28, 28, 128, 3, 3, 64, target={"resident": True}),
    S("ring1_cin1024_5x5", 704, 14, 14, 1024, 5, 5, 64, target={"resident": False, "n_tiles": 1}),
    S("ring8_512-512", 384, 7, 7, 512, 3, 3, 512, act=RELU, target={"resident": False, "n_tiles": 8}),
    # 128-pixel tiles that span several small images, zero padding
    S("span_7x7_s1", 512, 7, 7, 256, 3, 3, 384, pv=0, corr=True),
    S("span_7x7_s2", 2048, 7, 7, 128, 3, 3, 320, (2, 2), pv=0, out=INT8),
    S("span_5x3_s1", 2048, 5, 3, 128, 3, 3, 320, pv=0, out=BITPACKED),
    S("span_5x3_s2", 8192, 5, 3, 128, 3, 3, 256, (2, 2), pv=0, corr=True),
    # one CTA per SM: two halo stages do not fit half the shared memory
    S("one_cta_dilated", 32, 64, 64, 1024, 3, 3, 64, dil=(2, 2), target={"ctas": 1}),
]
CASE_IDS = [c.name for c in CASES]


def test_case_table_reaches_its_targets():
    """Every case gives each wgmma CTA at least four items on 132 SMs and hits the layout it is
    named for; together the table covers both CTA counts, resident and ring weights, flat and
    multi-chunk halos and both tile widths."""
    assert len(set(CASE_IDS)) == len(CASE_IDS)
    seen = {"ctas": set(), "resident": set(), "flat": set(), "chunks": set(), "BN": set()}
    for s in CASES:
        lay = tc_layout(s)
        assert lay is not None, s.name
        assert lay["per_cta"] >= MIN_ITEMS_PER_CTA, (s.name, lay)
        for k, v in s.target.items():
            assert lay[k] == v, (s.name, k, lay)
        for k in seen:
            seen[k].add(lay[k])
        if s.corr:
            assert s.pad == SAME and s.pv == 0 and s.out == FLOAT and s.act == NONE, s.name
    assert seen["ctas"] == {1, 2} and seen["resident"] == {True, False}
    assert seen["flat"] == {True, False} and seen["BN"] == {32, 64} and max(seen["chunks"]) >= 2


# ----------------------------------- GPU ----------------------------------- #
POISON = 0x7FA5A5A5              # a NaN / a packed word with every tail bit set: no kernel writes it
GEMM_CLAMP = (0, 2**31 - 1)
THREADS = min(os.cpu_count() or 4, 16)


@pytest.fixture(scope="module")
def capi():
    from compute_engine_b200 import capi as m
    m.lib()
    return m


def set_env(monkeypatch, env):
    for k, v in zip(("LCE_B200_BCONV_IMMA", "LCE_B200_BCONV_B1", "LCE_B200_BCONV_TC"), ENVS[env]):
        monkeypatch.setenv(k, v)


def launches(capi, before):
    return [y - x for x, y in zip(before, path_counts(capi))]


def one_hot(slot, n):
    r = [0, 0, 0]
    r[slot] = n
    return r


def poisoned(shape, dtype):
    import torch
    t = torch.empty(shape, dtype=dtype, device="cuda")
    if dtype == torch.int8:
        return t.fill_(-91)
    t.view(torch.int32).fill_(POISON)
    return t


def same_bits(a, b):
    import torch
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if a.dtype == torch.int8:
        return torch.equal(a, b)
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def ptr(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def random_words(rng, lead, channels):
    """Packed signs: uniform random bits, the tail bits of a partial word zero."""
    w = rng.integers(0, 2**32, lead + (L.cdiv(channels, 32),), dtype=np.uint32)
    if channels % 32:
        w[..., -1] &= np.uint32((1 << (channels % 32)) - 1)
    return w.view(np.int32)


def make_case(s, seed):
    rng = np.random.default_rng(seed)
    desc = L.BconvDesc(s.b, s.h, s.w, s.cin, s.fh, s.fw, s.cout, 1, *s.stride, *s.dil, s.pad, s.pv,
                       s.act, s.out, 1.0, 0)
    inp = random_words(rng, (s.b, s.h, s.w), s.cin)
    filt = random_words(rng, (s.cout, s.fh, s.fw), s.cin)
    mul = rng.uniform(0.01, 1.5, s.cout).astype(np.float32)
    bias = rng.uniform(0.01, 1.5, s.cout).astype(np.float32)
    thr = None
    if s.out == INT8:     # multipliers and biases of either sign, every seventh multiplier zero
        desc.out_scale = float(np.float32(1) / np.float32(rng.integers(1, 21)))
        desc.out_zero_point = int(rng.integers(-20, 21))
        mul = rng.uniform(-2, 2, s.cout).astype(np.float32)
        mul[::7] = 0
        bias = rng.uniform(-3, 3, s.cout).astype(np.float32)
    elif s.out == BITPACKED:
        mul = bias = None
        thr = spread_thresholds(rng, s.cout, s.taps * s.cin)
    return L.BconvCase(desc, inp, filt, mul, bias, thr)


def add_activation(y, res, act):
    """ADD of the shortcut with its fused activation, then (the caller) LceQuantize."""
    v = (y + res).astype(np.float32)
    lo, hi = {NONE: (None, None), RELU: (0, None), N1: (-1, 1), RELU6: (0, 6)}[act]
    if lo is not None:
        v = np.maximum(v, np.float32(lo))
    if hi is not None:
        v = np.minimum(v, np.float32(hi))
    return v


def run_conv(capi, s, case, x, res, act):
    """A plain run and, for float plans, run_fused with the shortcut and the next layer's signs,
    each into a fresh poisoned output. Returns [out] or [out, fused sum, fused signs]."""
    import torch
    plan = capi.BConv2d(gpu_desc(capi, case.desc), case.filt, case.mul, case.bias, case.thr)
    if s.corr:
        plan.set_zero_padding_mode(1)
    shape = plan.out_shape()
    outs = [poisoned(shape, plan.out_dtype())]
    plan(x, out=outs[0])
    if s.out == FLOAT:
        outs += [poisoned(shape, torch.float32), poisoned(shape[:3] + (L.cdiv(s.cout, 32),), torch.int32)]
        rc = capi.lib().lce_b200_bconv2d_run_fused(plan._h, ptr(x), ptr(res), C.c_int(act), ptr(outs[1]),
                                                   ptr(outs[2]), stream())
        assert rc == 0, capi.lib().lce_b200_last_error()
    torch.cuda.synchronize()
    plan.close()
    return outs


def run_gemm(capi, s, case, x):
    import torch
    gemm = capi.BGemm(case.filt.reshape(s.cout, -1), capi.OUT_FLOAT, GEMM_CLAMP, case.mul, case.bias)
    out = poisoned((s.b, s.cout), torch.float32)
    gemm(x, out=out)
    torch.cuda.synchronize()
    gemm.close()
    return [out]


@pytest.mark.gpu
@pytest.mark.parametrize("s", CASES, ids=CASE_IDS)
def test_every_kernel_gives_the_oracle_bits_at_scale(s, capi, monkeypatch):
    """One case on every kernel that takes it: the launch counters name the kernel; whole outputs
    (and, for float plans, run_fused's sum and signs with the ADD activation cycling over the
    cases) are equal across kernels; three images (BGEMM: three row blocks) equal the oracle."""
    import torch
    lay = tc_layout(s, torch.cuda.get_device_properties(0).multi_processor_count)
    assert lay is not None and lay["per_cta"] >= MIN_ITEMS_PER_CTA, lay
    n = CASE_IDS.index(s.name)
    case = make_case(s, 31000 + n)
    act = (NONE, RELU, N1, RELU6)[n % 4]
    if s.gemm:
        A = case.inp.reshape(s.b, -1)
        sel = np.r_[0:128, s.b // 2 - 64:s.b // 2 + 64, s.b - 128:s.b]
        wants = [L.bgemm(A[sel], case.filt.reshape(s.cout, -1), FLOAT, GEMM_CLAMP, case.mul, case.bias,
                         threads=THREADS)]
        x, res = dev(A), None
    else:
        sel = np.array([0, s.b // 2, s.b - 1])
        sub = L.BconvDesc.from_buffer_copy(case.desc)
        sub.batch = len(sel)
        y = L.bconv2d(sub, case.inp[sel], case.filt, case.mul, case.bias, case.thr, kind=int(s.corr),
                      threads=THREADS)
        wants = [y]
        x, res = dev(case.inp), None
        if s.out == FLOAT:
            oh, ow, _, _ = geometry(s)
            g = torch.Generator(device="cuda").manual_seed(n)
            res = torch.randn((s.b, oh, ow, s.cout), device="cuda", generator=g)
            ws = add_activation(y, res[torch.from_numpy(sel).cuda()].cpu().numpy(), act)
            wants += [ws, L.quantize(ws)]
    sel_t = torch.from_numpy(sel).cuda()
    first = None
    for env, slot in kernels_for(s):
        set_env(monkeypatch, env)
        before = path_counts(capi)
        outs = run_gemm(capi, s, case, x) if s.gemm else run_conv(capi, s, case, x, res, act)
        ran = launches(capi, before)
        tag = f"{s.name} on {env} ({lay['per_cta']} items per CTA)"
        assert ran == one_hot(slot, 2 if len(outs) == 3 else 1), (tag, ran)
        for what, got, want in zip(("output", "fused sum", "fused signs"), outs, wants):
            assert_same_bits(got[sel_t].cpu().numpy(), want, f"{tag}: {what} vs the oracle")
        if first is None:
            first = (env, outs)
        else:
            for what, got, ref in zip(("output", "fused sum", "fused signs"), outs, first[1]):
                assert same_bits(got, ref), f"{tag}: {what} differs from {first[0]}'s"
        del outs


@pytest.mark.gpu
def test_chain_and_gate_fallbacks_equal_the_mma_sync_epilogue(capi, monkeypatch):
    """run_fused_chain / run_fused_gate on a plan the mma.sync kernel does not take (here because
    the environment keeps it off) run the convolution on wgmma or XOR + POPC and the tail as one
    more pass; both give the bits of the mma.sync kernel's fused epilogue, at every ADD activation."""
    import torch
    s = S("tails", 64, 56, 56, 64, 3, 3, 64)
    case = make_case(s, 32000)
    rng = np.random.default_rng(32)
    x = dev(case.inp)
    res = torch.randn((s.b, 56, 56, 64), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    chain = [dev(rng.uniform(-0.5, 0.5, 64).astype(np.float32)), dev(rng.uniform(0.05, 0.5, 64).astype(np.float32)),
             dev(rng.uniform(-0.5, 0.5, 64).astype(np.float32)), dev(rng.uniform(-0.5, 0.5, 64).astype(np.float32))]
    gate = dev(rng.uniform(0, 1, (s.b, 64)).astype(np.float32))
    gvec = [dev(rng.uniform(0.05, 0.5, 64).astype(np.float32)), dev(rng.uniform(0.5, 1.5, 64).astype(np.float32)),
            dev(rng.uniform(-0.5, 0.5, 64).astype(np.float32))]
    acts = (NONE, RELU, N1, RELU6)
    first = None
    for env, slot in (("default", IMMA), ("wgmma", TC), ("xor", XOR)):
        set_env(monkeypatch, env)
        plan = capi.BConv2d(gpu_desc(capi, case.desc), case.filt, case.mul, case.bias)
        before = path_counts(capi)
        outs = []
        for act in acts:
            outs += plan.run_fused_chain(x, res, act, *chain)
            outs += plan.run_fused_gate(x, gate, res, act, *gvec)
        torch.cuda.synchronize()
        ran = launches(capi, before)
        plan.close()
        assert ran == one_hot(slot, 2 * len(acts)), (env, ran)
        if first is None:
            first = outs
            continue
        for i, (got, ref) in enumerate(zip(outs, first)):
            what = ("chain", "gate")[i // 2 % 2] + (" sum", " signs")[i % 2]
            assert same_bits(got, ref), f"{env}: {what}, ADD activation {acts[i // 4]}"


# (environment, input offset, output offset in bytes, the kernel that takes the placement)
PLACEMENTS = {
    False: [("default", 0, 0, IMMA), ("default", 0, 16, IMMA), ("default", 0, 8, TC), ("default", 0, 4, XOR),
            ("default", 8, 0, IMMA), ("wgmma", 0, 0, TC), ("wgmma", 8, 0, XOR)],
    # CORRECTION: wgmma first; elsewhere the mma.sync or XOR + POPC kernel and zpc_tail_kernel
    True: [("default", 0, 0, TC), ("default", 0, 16, TC), ("default", 0, 8, TC), ("default", 0, 4, XOR),
           ("default", 8, 0, IMMA)],
}


@pytest.mark.gpu
@pytest.mark.parametrize("corr", [False, True], ids=["one_padding", "correction"])
def test_pointer_alignment_selects_the_fallbacks(corr, capi, monkeypatch):
    """The same plan with one pointer moved from a 256-byte boundary: the mma.sync kernel needs a
    16-byte aligned output, wgmma an 8-byte aligned output and a 16-byte aligned input; the 8-byte
    input offset is legal for the 8-byte gathers of 64-channel inputs. Every placement gives the
    aligned run's bits, plain and fused. run_fused refuses a residual that is not 16-byte aligned."""
    import torch
    s = S("align", 64, 56, 56, 64, 3, 3, 64, pv=0 if corr else 1, corr=corr)
    case = make_case(s, 33000 + corr)
    x = dev(case.inp).reshape(-1)
    shape = (s.b, 56, 56, 64)
    n_out = int(np.prod(shape))
    res = torch.randn(shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    xbuf = torch.empty(x.numel() + 128, dtype=torch.int32, device="cuda")
    obuf = torch.empty(n_out + 128, dtype=torch.float32, device="cuda")

    def at(buf, off, count):
        base = (-buf.data_ptr() % 256) // 4
        return buf[base + off // 4:base + off // 4 + count]
    plans = {}
    first = None
    for env, in_off, out_off, slot in PLACEMENTS[corr]:
        if env not in plans:
            set_env(monkeypatch, env)
            plans[env] = capi.BConv2d(gpu_desc(capi, case.desc), case.filt, case.mul, case.bias)
            if corr:
                plans[env].set_zero_padding_mode(1)
        h = plans[env]._h
        xi = at(xbuf, in_off, x.numel())
        xi.copy_(x)
        o = at(obuf, out_off, n_out)
        packed = poisoned((n_out // 32,), torch.int32)
        before = path_counts(capi)
        o.view(torch.int32).fill_(POISON)
        assert capi.lib().lce_b200_bconv2d_run(h, ptr(xi), ptr(o), stream()) == 0, capi.lib().lce_b200_last_error()
        plain = o.clone()
        o.view(torch.int32).fill_(POISON)
        assert capi.lib().lce_b200_bconv2d_run_fused(h, ptr(xi), ptr(res), C.c_int(RELU), ptr(o), ptr(packed),
                                                     stream()) == 0, capi.lib().lce_b200_last_error()
        outs = [plain, o.clone(), packed]
        torch.cuda.synchronize()
        tag = f"{env}, input +{in_off} B, output +{out_off} B"
        assert launches(capi, before) == one_hot(slot, 2), (tag, launches(capi, before))
        if first is None:
            first = outs
        for what, got, ref in zip(("output", "fused sum", "fused signs"), outs, first):
            assert same_bits(got, ref), f"{tag}: {what}"
    o = at(obuf, 0, n_out)
    rbuf = torch.empty(n_out + 128, dtype=torch.float32, device="cuda")
    for off in (4, 8):
        r = at(rbuf, off, n_out)
        rc = capi.lib().lce_b200_bconv2d_run_fused(plans["default"]._h, ptr(x), ptr(r), C.c_int(NONE), ptr(o),
                                                   None, stream())
        assert rc != 0 and b"16-byte aligned" in capi.lib().lce_b200_last_error(), off
    for p in plans.values():
        p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("env", ["default", "wgmma"])
def test_a_resized_plan_equals_a_fresh_plan(env, capi, monkeypatch):
    """One plan called at batch 256, 3, 256, then another image size and back: each result equals a
    plan created for that shape (the wgmma launch caches its halo size per input shape), and its
    last image equals the oracle."""
    import torch
    set_env(monkeypatch, env)
    slot = IMMA if env == "default" else TC
    s = S("resize", 256, 14, 14, 256, 3, 3, 128, act=RELU)
    case = make_case(s, 34000)
    plan = capi.BConv2d(gpu_desc(capi, case.desc), case.filt, case.mul, case.bias)
    rng = np.random.default_rng(34)
    for b, h, w in ((256, 14, 14), (3, 14, 14), (256, 14, 14), (64, 9, 11), (256, 14, 14)):
        x = dev(random_words(rng, (b, h, w), s.cin))
        desc = L.BconvDesc.from_buffer_copy(case.desc)
        desc.batch, desc.in_h, desc.in_w = b, h, w
        fresh = capi.BConv2d(gpu_desc(capi, desc), case.filt, case.mul, case.bias)
        before = path_counts(capi)
        got, want = plan(x), fresh(x)
        torch.cuda.synchronize()
        fresh.close()
        assert launches(capi, before) == one_hot(slot, 2), (b, h, w)
        assert same_bits(got, want), (env, b, h, w)
        desc.batch = 1
        assert_same_bits(got[-1:].cpu().numpy(), L.bconv2d(desc, x[-1:].cpu().numpy(), case.filt, case.mul,
                                                            case.bias, threads=THREADS), f"{env} {(b, h, w)}")
    plan.close()


@pytest.mark.gpu
def test_bgemm_output_beyond_2_pow_31_bytes(capi, monkeypatch):
    """A float BGEMM whose output is 2.7 GB: the rows around the 2^31-byte offset and the last rows
    equal the oracle, on mma.sync and on wgmma, and the two outputs are equal."""
    import torch
    M, N, Kw = 2**21 + 77, 320, 2
    rng = np.random.default_rng(35)
    A = random_words(rng, (M,), 32 * Kw)
    W = random_words(rng, (N,), 32 * Kw)
    mul = rng.uniform(-1.5, 1.5, N).astype(np.float32)
    bias = rng.uniform(-1.5, 1.5, N).astype(np.float32)
    edge = 2**31 // (4 * N)
    rows = np.r_[0:64, edge - 64:edge + 64, M - 256:M]
    want = L.bgemm(A[rows], W, FLOAT, GEMM_CLAMP, mul, bias, threads=THREADS)
    x = dev(A)
    outs = []
    for env, slot in (("default", IMMA), ("wgmma", TC)):
        set_env(monkeypatch, env)
        gemm = capi.BGemm(W, capi.OUT_FLOAT, GEMM_CLAMP, mul, bias)
        out = poisoned((M, N), torch.float32)
        before = path_counts(capi)
        gemm(x, out=out)
        torch.cuda.synchronize()
        gemm.close()
        assert launches(capi, before) == one_hot(slot, 1), env
        assert_same_bits(out[torch.from_numpy(rows).cuda()].cpu().numpy(), want, env)
        outs.append(out)
    assert same_bits(outs[0], outs[1])
