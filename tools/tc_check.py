"""Quick parity + timing sweep of the wgmma path against the oracle, one line per case.

Development tool (not collected by pytest): runs from simple to complex so that a failure
localises itself, reads the kernel's deadlock-watchdog record after every case, and compares each
result with the mma.sync / XOR kernels' (which the GPU test-suite already pins to the oracle) and,
for small cases, with the oracle directly.

  python tools/tc_check.py            # all groups
  python tools/tc_check.py bgemm conv # selected groups
"""
from __future__ import annotations

import ctypes as C
import os
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
import lce_testlib as L  # noqa: E402  (checker)
from compute_engine_b200 import capi  # noqa: E402

lib = capi.lib()
lib.lce_b200_path_counts.argtypes = [C.POINTER(C.c_uint64)]
lib.lce_b200_tc_debug.argtypes = [C.POINTER(C.c_int32)]


def paths():
    a = (C.c_uint64 * 3)()
    lib.lce_b200_path_counts(a)
    return list(a)


def watchdog():
    torch.cuda.synchronize()
    a = (C.c_int32 * 8)()
    lib.lce_b200_tc_debug(a)
    return list(a) if a[7] else None


def set_tc(on):
    os.environ["LCE_B200_BCONV_TC"] = "1" if on else "0"


def timeit(fn, n=5):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


FAILS = []


def report(name, ok, extra=""):
    print(("ok   " if ok else "FAIL ") + name + " " + extra, flush=True)
    if not ok:
        FAILS.append(name)


def bgemm_case(M, N, K_bits, out_type=L.OUT_RAW_ACC, seed=0, oracle=True):
    rng = np.random.default_rng(seed)
    Kw = K_bits // 32
    A = rng.integers(-2**31, 2**31, (M, Kw), dtype=np.int64).astype(np.int32)
    W = rng.integers(-2**31, 2**31, (N, Kw), dtype=np.int64).astype(np.int32)
    mul = rng.uniform(0.01, 1.5, N).astype(np.float32)
    bias = rng.uniform(0.01, 1.5, N).astype(np.float32)
    thr = rng.integers(K_bits // 2 - 20, K_bits // 2 + 20, N).astype(np.int32)
    clamp = (0, 2 * K_bits)
    kw = dict(out_type=out_type, clamp=clamp, multiplier=mul, bias=bias, thresholds=thr)
    Ad = torch.from_numpy(A).cuda()
    res = {}
    for on in (False, True):
        set_tc(on)
        plan = capi.BGemm(W, **kw)
        p0 = paths()
        out = plan(Ad)
        wd = watchdog()
        p1 = paths()
        res[on] = (out.cpu().numpy(), [b - a for a, b in zip(p0, p1)], wd, timeit(lambda: plan(Ad)))
        plan.close()
    name = f"bgemm M={M} N={N} K={K_bits} out={out_type}"
    got, path, wd, t_tc = res[True]
    base, _, _, t_old = res[False]
    ok = path[0] == 1 and wd is None and np.array_equal(got.view(np.uint8), base.view(np.uint8))
    extra = f"path={path} wd={wd} t_tc={t_tc*1e3:.1f}us t_old={t_old*1e3:.1f}us"
    if oracle and M * N * Kw <= 3e8:
        want = L.bgemm(A, W, out_type, clamp, mul, bias, thr, threads=32)
        ok_o = np.array_equal(got.view(np.uint8), want.view(np.uint8))
        extra += f" oracle={'eq' if ok_o else 'DIFF'}"
        ok = ok and ok_o
    if not ok and path[0] == 1:
        d = np.argwhere(got != base)
        extra += f" nbad={len(d)} first={d[:4].tolist()}"
        if len(d):
            i = tuple(d[0])
            extra += f" got={got[i]} want={base[i]}"
    tops = 2.0 * M * N * K_bits / (t_tc * 1e-3) / 1e12
    report(name, ok, extra + f" {tops:.0f} TOPS")


def conv_case(seed, b, hw, cin, k, cout, out_type=L.OUT_FLOAT, stride=1, dil=1, padding=L.PADDING_SAME,
              pad_value=1, act=L.ACT_NONE, oracle=True, zp_mode=0):
    case = L.make_bconv_case(seed, b, hw, hw, cin, k, k, cout, stride=(stride, stride), dilation=(dil, dil),
                             padding=padding, pad_value=pad_value, activation=act, out_type=out_type)
    x = torch.from_numpy(case.inp).cuda()
    res = {}
    for on in (False, True):
        set_tc(on)
        d = capi.BconvDesc(*[getattr(case.desc, n) for n, _ in case.desc._fields_])
        plan = capi.BConv2d(d, case.filt, case.mul, case.bias, case.thr)
        plan.set_zero_padding_mode(zp_mode)
        p0 = paths()
        out = plan(x)
        wd = watchdog()
        p1 = paths()
        res[on] = (out.cpu().numpy(), [b_ - a for a, b_ in zip(p0, p1)], wd, timeit(lambda: plan(x)))
        plan.close()
    name = f"conv zp={zp_mode} b={b} hw={hw} cin={cin} k={k} cout={cout} out={out_type} s={stride} d={dil} pad={padding}/{pad_value} act={act}"
    got, path, wd, t_tc = res[True]
    base, _, _, t_old = res[False]
    ok = path[0] == 1 and wd is None and np.array_equal(got.view(np.uint8), base.view(np.uint8))
    extra = f"path={path} wd={wd} t_tc={t_tc*1e3:.1f}us t_old={t_old*1e3:.1f}us"
    if oracle and got.size * k * k * cin <= 4e9:
        want = L.bconv2d(case.desc, case.inp, case.filt, case.mul, case.bias, case.thr, threads=32, kind=zp_mode)
        ok_o = np.array_equal(got.view(np.uint8), want.view(np.uint8))
        extra += f" oracle={'eq' if ok_o else 'DIFF'}"
        ok = ok and ok_o
    if not ok and path[0] == 1:
        d = np.argwhere(got != base)
        extra += f" nbad={len(d)}/{got.size} first={d[:3].tolist()}"
        if len(d):
            i = tuple(d[0])
            extra += f" got={got[i]} want={base[i]}"
    report(name, ok, extra)


def fused_case(seed, b, hw, cin, cout, act_add=L.ACT_NONE):
    """conv + shortcut + next layer's sign bits through lce_b200_bconv2d_run_fused."""
    case = L.make_bconv_case(seed, b, hw, hw, cin, 3, 3, cout, activation=L.ACT_RELU)
    rng = np.random.default_rng(seed + 100)
    x = torch.from_numpy(case.inp).cuda()
    res_t = torch.from_numpy(rng.standard_normal((b, hw, hw, cout)).astype(np.float32)).cuda()
    outs = {}
    for on in (False, True):
        set_tc(on)
        d = capi.BconvDesc(*[getattr(case.desc, n) for n, _ in case.desc._fields_])
        plan = capi.BConv2d(d, case.filt, case.mul, case.bias, None)
        out = torch.empty((b, hw, hw, cout), dtype=torch.float32, device="cuda")
        pk = torch.empty((b, hw, hw, cout // 32), dtype=torch.int32, device="cuda")
        p0 = paths()
        run = lambda: capi._check(lib.lce_b200_bconv2d_run_fused(  # noqa: E731
            plan._h, C.c_void_p(x.data_ptr()), C.c_void_p(res_t.data_ptr()), act_add,
            C.c_void_p(out.data_ptr()), C.c_void_p(pk.data_ptr()), None))
        run()
        wd = watchdog()
        p1 = paths()
        outs[on] = (out.cpu().numpy(), pk.cpu().numpy(), [b_ - a for a, b_ in zip(p0, p1)], wd, timeit(run))
        plan.close()
    got, gpk, path, wd, t_tc = outs[True]
    base, bpk, _, _, t_old = outs[False]
    ok = path[0] == 1 and wd is None and np.array_equal(got.view(np.uint8), base.view(np.uint8)) and np.array_equal(gpk, bpk)
    extra = f"path={path} wd={wd} t_tc={t_tc*1e3:.1f}us t_old={t_old*1e3:.1f}us"
    if not ok and path[0] == 1:
        d = np.argwhere(got != base)
        extra += f" nbad={len(d)}/{got.size} first={d[:3].tolist()} pk_bad={int((gpk != bpk).sum())}"
    report(f"fused b={b} hw={hw} cin={cin} cout={cout} act_add={act_add}", ok, extra)


def main():
    groups = set(sys.argv[1:]) or {"bgemm", "conv", "fused", "big"}
    torch.cuda.set_device(0)
    if "bgemm" in groups:
        bgemm_case(128, 64, 128)
        bgemm_case(128, 64, 256)
        bgemm_case(128, 128, 1024)
        bgemm_case(100, 64, 128)          # M tail
        bgemm_case(1000, 256, 512)
        bgemm_case(256, 64, 2304)         # Kw = 72: two channel chunks (64 + 8)
        bgemm_case(256, 64, 96)           # Kw = 3: flat mode, V = 1
        bgemm_case(256, 64, 192)          # Kw = 6: flat mode, V = 2
        bgemm_case(512, 256, 8192)
        for ot in (L.OUT_FLOAT, L.OUT_INT8, L.OUT_BITPACKED):
            bgemm_case(384, 128, 512, out_type=ot)
        bgemm_case(300, 96, 256, out_type=L.OUT_FLOAT)   # ragged N
        bgemm_case(300, 40, 256, out_type=L.OUT_INT8)
        bgemm_case(300, 40, 256, out_type=L.OUT_BITPACKED)
    if "conv" in groups:
        conv_case(1, 2, 8, 128, 3, 64)
        conv_case(2, 2, 8, 64, 3, 64)                        # Cw = 2: flat mode
        conv_case(3, 3, 14, 256, 3, 256, act=L.ACT_RELU)
        conv_case(4, 5, 7, 512, 3, 512)
        conv_case(5, 2, 16, 128, 3, 128, pad_value=0)        # zero-padding correction
        conv_case(6, 2, 16, 64, 3, 128, stride=2, pad_value=0)
        conv_case(5, 2, 16, 128, 3, 128, pad_value=0, zp_mode=1)   # the optimised kernels' float correction
        conv_case(6, 2, 16, 64, 3, 128, stride=2, pad_value=0, zp_mode=1)
        conv_case(12, 3, 7, 96, 3, 64, pad_value=0, zp_mode=1)
        conv_case(13, 1, 12, 32, 5, 32, dil=2, pad_value=0, zp_mode=1)
        conv_case(7, 2, 12, 32, 5, 64, dil=2)                # Cw = 1
        conv_case(8, 2, 12, 96, 3, 64, padding=L.PADDING_VALID)
        conv_case(9, 2, 9, 128, 1, 128)
        for ot in (L.OUT_INT8, L.OUT_BITPACKED):
            conv_case(10, 2, 10, 128, 3, 128, out_type=ot, act=L.ACT_RELU)
            conv_case(11, 2, 10, 64, 3, 48, out_type=ot)
    if "fused" in groups:
        fused_case(1, 2, 8, 64, 64)
        fused_case(2, 4, 14, 256, 256, L.ACT_RELU)
        fused_case(3, 3, 7, 512, 512)
    if "big" in groups:
        # QuickNet stage shapes at batch 256 (oracle skipped: compared with the mma.sync kernel)
        for hw, c in ((56, 64), (28, 128), (14, 256), (7, 512)):
            conv_case(20, 256, hw, c, 3, c, act=L.ACT_RELU, oracle=False)
            fused_case(21, 256, hw, c, c)
        bgemm_case(4096, 4096, 256, oracle=False)
        bgemm_case(4096, 4096, 8192, oracle=False)
        bgemm_case(4096, 4096, 1024, out_type=L.OUT_FLOAT, oracle=False)
    print("FAILS:", FAILS if FAILS else "none", flush=True)


if __name__ == "__main__":
    main()
