#!/usr/bin/env python
"""Check + time the wgmma tf32 pointwise convolution (csrc/lce_b200_pw.cuh) against an
fp64 product, then run the same cases on the FMA kernels it replaces (child process with
LCE_B200_PW_TF32=0) for the error and time comparison. Usage: pw_check.py [quick]"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compute_engine_b200 import capi  # noqa: E402


class ConvDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("batch", "in_h", "in_w", "in_c", "filter_h", "filter_w", "out_c",
                                         "stride_h", "stride_w", "dilation_h", "dilation_w", "padding",
                                         "activation")]


def run(M, K, N, act, with_packed, seed, reps=int(os.environ.get("PW_REPS", "20"))):
    lib = capi.lib()
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = (torch.randn(M, K, generator=g) * 1.5).cuda()
    W = (torch.randn(N, K, generator=g) * 0.3).cuda()
    b = torch.randn(N, generator=g).cuda()
    out = torch.empty(M, N, device="cuda")
    packed = torch.zeros(M, N // 32, dtype=torch.int32, device="cuda") if with_packed else None
    d = ConvDesc(1, 1, M, K, 1, 1, N, 1, 1, 1, 1, 1, act)   # [1, 1, M, K] image: M pixels
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call():
        if with_packed:
            rc = lib.lce_b200_f32_conv2d_packed(C.byref(d), C.c_void_p(A.data_ptr()), C.c_void_p(W.data_ptr()),
                                                C.c_void_p(b.data_ptr()), C.c_void_p(out.data_ptr()),
                                                C.c_void_p(packed.data_ptr()), st)
        else:
            rc = lib.lce_b200_f32_conv2d(C.byref(d), C.c_void_p(A.data_ptr()), C.c_void_p(W.data_ptr()),
                                         C.c_void_p(b.data_ptr()), C.c_void_p(out.data_ptr()), st)
        assert rc == 0, capi.lib().lce_b200_last_error().decode()

    call()
    torch.cuda.synchronize()
    # fp64 reference on a sample of rows (all rows when small)
    rows = np.unique(np.concatenate([np.arange(min(M, 300)), np.arange(max(0, M - 300), M),
                                     np.random.default_rng(seed).integers(0, M, 2000)]))
    ridx = torch.from_numpy(rows).cuda()
    ref = A[ridx].double() @ W.double().t() + b.double()
    if act == 1:
        ref = ref.clamp(min=0)
    elif act == 3:
        ref = ref.clamp(0, 6)
    got = out[ridx].double()
    mag = (A[ridx].abs().double() @ W.abs().double().t() + b.abs().double())
    rel = ((got - ref).abs() / mag).max().item()
    ok = rel < 2e-6
    msg = f"M={M} K={K} N={N} act={act} packed={int(with_packed)} max|err|/sum|a||w| = {rel:.2e}"
    if with_packed:
        want = (out < 0).view(M, N // 32, 32).to(torch.int64)
        wantw = (want << torch.arange(32, device="cuda")).sum(-1)
        wantw = torch.where(wantw >= 2**31, wantw - 2**32, wantw).to(torch.int32)
        pk_ok = torch.equal(wantw, packed)
        ok = ok and pk_ok
        msg += f" packed_eq={pk_ok}"
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1000 / reps
    gb = (M * K + M * N + N * K) * 4 / 1e9
    msg += f"  {us:8.1f} us  {gb / (us * 1e-6):7.0f} GB/s"
    print(("ok   " if ok else "FAIL ") + msg, flush=True)
    return ok


def main():
    quick = len(sys.argv) > 1 and sys.argv[1] == "quick"
    label = "tf32" if os.environ.get("LCE_B200_PW_TF32") != "0" else "fma "
    print(f"--- pointwise convolution, path = {label}")
    cases = [
        (16384, 16, 64, 1, True), (20002, 16, 64, 0, False),
        (8192, 32, 128, 0, True), (8192 + 77, 64, 128, 0, True), (9001, 128, 256, 1, True),
        (4999, 256, 512, 0, True), (8192, 96, 128, 3, False), (6000, 512, 1024, 0, False),
    ]
    big = [(256 * 56 * 56, 16, 64, 0, True), (256 * 28 * 28, 64, 128, 0, True), (256 * 14 * 14, 128, 256, 0, True),
           (256 * 7 * 7, 256, 512, 0, True)]
    ok = True
    if os.environ.get("PW_ONLY_BIG"):
        cases = []
    for n, c in enumerate(cases + ([] if quick else big)):
        ok &= run(*c, seed=n)
    print("ALL OK" if ok else "FAILURES")
    if label == "tf32" and not quick and not os.environ.get("PW_SKIP_FMA"):
        env = dict(os.environ, LCE_B200_PW_TF32="0")
        subprocess.run([sys.executable, os.path.abspath(__file__)], env=env)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
