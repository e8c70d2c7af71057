"""Bitpacked-output LceBconv2d and BGEMM on the mma.sync kernel (lce_b200_imma.cuh): the
BITPACKED epilogue compares each accumulator with its channel's threshold and stores the packed
words, for the b1 inner product and its int8 variant (LCE_B200_BCONV_B1=0).

CPU: the new instances compile for sm_90a without spills. GPU: bit-exact against the oracle over
channel counts, filters, strides, both paddings, groups and ragged M, with the launch counters
showing which kernel ran; the same words as the wgmma / XOR + POPC kernels that take these plans
with LCE_B200_BCONV_IMMA=0; the bitpacked BGEMM."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import lce_testlib as L

# b, h, w, cin, fh, fw, cout, groups, stride, padding, pad_value
GRID = [
    (3, 9, 9, 64, 3, 3, 64, 1, 1, L.PADDING_SAME, 1),
    (2, 14, 14, 128, 3, 3, 128, 1, 2, L.PADDING_SAME, 1),
    (2, 11, 7, 96, 3, 3, 192, 1, 1, L.PADDING_SAME, 0),      # REFERENCE zero padding, 3-word rows
    (1, 13, 13, 256, 3, 3, 256, 1, 2, L.PADDING_SAME, 0),
    (5, 6, 6, 64, 1, 1, 384, 1, 1, L.PADDING_VALID, 1),      # 1x1, M = 180
    (2, 9, 9, 128, 5, 5, 64, 1, 1, L.PADDING_VALID, 1),      # 5x5 VALID
    (1, 7, 7, 1024, 5, 5, 128, 1, 1, L.PADDING_SAME, 1),     # K = 800 words: staged in chunks
    (2, 10, 10, 128, 3, 3, 256, 2, 1, L.PADDING_SAME, 1),    # groups, 128 channels per group
    (3, 8, 8, 96, 3, 3, 192, 3, 2, L.PADDING_SAME, 0),       # groups, 64 channels per group
    (37, 1, 1, 512, 1, 1, 64, 1, 1, L.PADDING_VALID, 1),     # M = 37: one partial tile
]


def spread_thresholds(rng, cout, k):
    """Thresholds around the accumulators' mean k / 2, so both bit values and ties occur, plus
    the extremes and the ends of the attainable range [0, k]."""
    t = np.rint(k / 2 + rng.standard_normal(cout) * np.sqrt(k) * 0.75).astype(np.int64)
    edges = [np.iinfo(np.int32).min, np.iinfo(np.int32).max, -1, 0, k - 1, k]
    t[rng.choice(cout, len(edges), replace=False)] = edges
    return t.astype(np.int32)


def bitpacked_case(n, b, h, w, cin, fh, fw, cout, groups, stride, padding, pad_value):
    case = L.make_bconv_case(7000 + n, b, h, w, cin, fh, fw, cout, groups, (stride, stride),
                             (1, 1), padding, pad_value, L.ACT_NONE, L.OUT_BITPACKED)
    thr = spread_thresholds(np.random.default_rng(n), cout, fh * fw * (cin // groups))
    return case, thr


def run_plan(capi, case, thr):
    import torch
    from test_gpu_parity import dev, gpu_desc
    plan = capi.BConv2d(gpu_desc(capi, case.desc), case.filt, None, None, thr)
    out = plan(dev(case.inp))
    torch.cuda.synchronize()
    plan.close()
    return out.cpu().numpy()


def test_bitpacked_instances_compile_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "bitpacked.cu"
    src.write_text('#include "lce_b200_imma.cuh"\n' + "".join(
        f"template __global__ void lce::bconv_imma_kernel<{v}, LCE_OUT_BITPACKED, {b1}>"
        "(const lce::ConvKParams);\n" for v in (1, 2, 4) for b1 in ("true", "false")))
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xptxas=-v", "-cubin", "-I", os.path.join(repo, "include"),
                        "-I", os.path.join(repo, "compute_engine_b200", "csrc"), str(src),
                        "-o", str(tmp_path / "bitpacked.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S*bconv_imma_kernel\S*)\n\s*(.*)", r.stderr)
    assert len(props) == 6, r.stderr
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)


# ----------------------------------- GPU ----------------------------------- #
@pytest.mark.gpu
@pytest.mark.parametrize("b1", ["1", "0"])
def test_gpu_bitpacked_mma_sync_matches_the_oracle(b1, monkeypatch):
    """Every case runs one mma.sync launch (grouped ones too: whole 64-channel tiles) and gives the
    oracle's words; then the same plans with LCE_B200_BCONV_IMMA=0 give the same words on wgmma
    (ungrouped) or XOR + POPC (grouped)."""
    from compute_engine_b200 import capi
    from test_gpu_parity import assert_same_bits, path_counts
    monkeypatch.setenv("LCE_B200_BCONV_TC", "1")
    for n, spec in enumerate(GRID):
        case, thr = bitpacked_case(n, *spec)
        tag = f"b1={b1} case {n} {spec}"
        want = L.bconv2d(case.desc, case.inp, case.filt, thr=thr, threads=4)
        assert 0 < np.unpackbits(want.view(np.uint8)).mean() < 1, tag + ": all bits equal"
        monkeypatch.setenv("LCE_B200_BCONV_IMMA", "1")
        monkeypatch.setenv("LCE_B200_BCONV_B1", b1)
        before = path_counts(capi)
        got = run_plan(capi, case, thr)
        ran = [y - x for x, y in zip(before, path_counts(capi))]
        assert ran == [0, 1, 0], (tag, ran)
        assert_same_bits(got, want, tag)
        monkeypatch.setenv("LCE_B200_BCONV_IMMA", "0")
        before = path_counts(capi)
        other = run_plan(capi, case, thr)
        ran = [y - x for x, y in zip(before, path_counts(capi))]
        assert ran == ([0, 0, 1] if spec[7] > 1 else [1, 0, 0]), (tag, ran)
        assert_same_bits(other, got, tag + " vs IMMA=0")


@pytest.mark.gpu
@pytest.mark.parametrize("b1", ["1", "0"])
def test_gpu_bitpacked_bgemm_on_mma_sync(b1, monkeypatch):
    from compute_engine_b200 import capi
    from test_gpu_parity import assert_same_bits, dev, path_counts
    monkeypatch.setenv("LCE_B200_BCONV_IMMA", "1")
    monkeypatch.setenv("LCE_B200_BCONV_B1", b1)
    rng = np.random.default_rng(31)
    for M, N, Kw in ((333, 64, 24), (1000, 192, 7), (129, 384, 64)):
        A = rng.integers(-2**31, 2**31 - 1, (M, Kw), dtype=np.int64).astype(np.int32)
        W = rng.integers(-2**31, 2**31 - 1, (N, Kw), dtype=np.int64).astype(np.int32)
        thr = spread_thresholds(rng, N, 32 * Kw)
        before = path_counts(capi)
        gemm = capi.BGemm(dev(W), capi.OUT_BITPACKED, thresholds=thr)
        got = gemm(dev(A)).cpu().numpy()
        gemm.close()
        ran = [y - x for x, y in zip(before, path_counts(capi))]
        assert ran == [0, 1, 0], (M, N, Kw, ran)
        assert_same_bits(got, L.bgemm(A, W, L.OUT_BITPACKED, thr=thr, threads=4), f"{M}x{N}x{Kw}")
