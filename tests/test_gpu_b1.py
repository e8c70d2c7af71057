"""The mma.sync kernel's two inner products -- packed b1 fragments on BMMA (the default) and int8
fragments on IMMA (LCE_B200_BCONV_B1=0) -- give the reference's integers and each other's, bit
for bit, over the case grid of test_gpu_parity's inner-product test."""
import ctypes as C

import numpy as np
import pytest
import torch

import lce_testlib as L
from test_gpu_parity import assert_same_bits, dev, gpu_desc, path_counts

pytestmark = pytest.mark.gpu

GRID = [
    # b, h, w, cin, fh, fw, cout, groups, stride, dilation, padding, pad_value, act
    (2, 14, 14, 64, 3, 3, 64, 1, (1, 1), (1, 1), L.PADDING_SAME, 1, L.ACT_RELU),
    (1, 7, 7, 512, 3, 3, 128, 1, (1, 1), (1, 1), L.PADDING_SAME, 1, L.ACT_NONE),
    (3, 9, 11, 64, 3, 3, 64, 1, (1, 1), (1, 1), L.PADDING_SAME, 0, L.ACT_NONE),
    (2, 13, 9, 128, 3, 3, 192, 1, (2, 2), (1, 1), L.PADDING_SAME, 0, L.ACT_NONE),
    (2, 12, 12, 96, 3, 2, 64, 1, (1, 2), (2, 1), L.PADDING_VALID, 1, L.ACT_RELU6),
    (2, 10, 10, 128, 3, 3, 128, 2, (1, 1), (1, 1), L.PADDING_SAME, 1, L.ACT_RELU),
    (1, 5, 5, 1024, 5, 5, 64, 1, (1, 1), (1, 1), L.PADDING_SAME, 1, L.ACT_NONE),   # K = 800 words
    (5, 6, 6, 32, 1, 1, 64, 1, (1, 1), (1, 1), L.PADDING_VALID, 1, L.ACT_RELU_N1_TO_1),
]


@pytest.fixture(scope="module")
def capi():
    from compute_engine_b200 import capi as m
    m.lib()
    return m


def run_case(capi, case, res, act_add):
    """plain and fused (ADD + LceQuantize) results of one plan"""
    plan = capi.BConv2d(gpu_desc(capi, case.desc), case.filt, case.mul, case.bias, case.thr)
    d_in, d_res = dev(case.inp), dev(res)
    plain = plan(d_in)
    out = torch.empty(res.shape, device="cuda")
    co = res.shape[-1]
    packed = torch.empty(res.shape[:3] + (L.cdiv(co, 32),), dtype=torch.int32, device="cuda")
    grouped = case.desc.groups > 1
    rc = capi.lib().lce_b200_bconv2d_run_fused(
        plan._h, C.c_void_p(d_in.data_ptr()), C.c_void_p(d_res.data_ptr()), C.c_int(act_add),
        C.c_void_p(out.data_ptr()), C.c_void_p(0 if grouped else packed.data_ptr()),
        C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, capi.lib().lce_b200_last_error()
    torch.cuda.synchronize()
    r = (plain.cpu().numpy(), out.cpu().numpy(), None if grouped else packed.cpu().numpy())
    plan.close()
    return r


def test_b1_and_int8_fragments_match_the_oracle_and_each_other(capi, monkeypatch):
    monkeypatch.setenv("LCE_B200_BCONV_TC", "0")
    monkeypatch.setenv("LCE_B200_BCONV_IMMA", "1")
    rng = np.random.default_rng(78)
    for n, (b, h, w, cin, fh, fw, co, g, st, dl, pad, pv, act) in enumerate(GRID):
        case = L.make_bconv_case(9100 + n, b, h, w, cin, fh, fw, co, g, st, dl, pad, pv, act,
                                 L.OUT_FLOAT)
        want = L.bconv2d(case.desc, case.inp, case.filt, case.mul, case.bias, case.thr)
        res = rng.standard_normal(want.shape).astype(np.float32)
        act_add = L.ACT_RELU if n % 2 else L.ACT_NONE
        ws = (want + res).astype(np.float32)
        if act_add == L.ACT_RELU:
            ws = np.maximum(ws, 0)
        got = {}
        for b1 in ("1", "0"):
            monkeypatch.setenv("LCE_B200_BCONV_B1", b1)
            before = path_counts(capi)
            got[b1] = run_case(capi, case, res, act_add)
            ran = [y - x for x, y in zip(before, path_counts(capi))]
            assert ran == [0, 2, 0], (b1, n, ran)   # plain + fused, one launch each
            plain, fused, packed = got[b1]
            assert_same_bits(plain, want, f"B1={b1} case {n}")
            assert_same_bits(fused, ws, f"B1={b1} fused sum {n}")
            if packed is not None:
                assert_same_bits(packed, L.quantize(ws), f"B1={b1} fused signs {n}")
        for x, y in zip(got["1"], got["0"]):
            if x is not None:
                assert_same_bits(x, y, f"b1 vs int8 case {n}")


def test_b1_and_int8_raw_accumulators(capi, monkeypatch):
    """plain BGEMM (raw int32 accumulators), K = 24 and 19 words (a k128 tail)"""
    monkeypatch.setenv("LCE_B200_BCONV_TC", "0")
    monkeypatch.setenv("LCE_B200_BCONV_IMMA", "1")
    rng = np.random.default_rng(79)
    for kw in (24, 19):
        A = rng.integers(-2**31, 2**31 - 1, (333, kw), dtype=np.int64).astype(np.int32)
        W = rng.integers(-2**31, 2**31 - 1, (128, kw), dtype=np.int64).astype(np.int32)
        want = L.bgemm(A, W, threads=4)
        got = {}
        for b1 in ("1", "0"):
            monkeypatch.setenv("LCE_B200_BCONV_B1", b1)
            before = path_counts(capi)
            gemm = capi.BGemm(dev(W))
            got[b1] = gemm(dev(A)).cpu().numpy()
            gemm.close()
            ran = [y - x for x, y in zip(before, path_counts(capi))]
            assert ran == [0, 1, 0], (b1, kw, ran)
            assert np.array_equal(got[b1], want), (b1, kw)
        assert np.array_equal(got["1"], got["0"])
