"""Time lce_b200_bconv2d_run_fused_pair against two lce_b200_bconv2d_run_fused calls (the residual
blocks it replaces) per activation shape, with CUDA events, and check that both give the same bits.

    python tools/pair_bench.py [--batch 256] [--iters 50]

Prints one line per shape: H x W x C, both times in ms per pair, and their ratio. Graph::
FuseResidualPairs pairs blocks only on the shapes where the pair kernel wins (images that split
into whole tiles); this is the measurement behind that rule."""
import argparse
import ctypes as C
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compute_engine_b200 import capi  # noqa: E402

SHAPES = [(56, 56, 64), (28, 28, 128), (14, 14, 64), (14, 14, 128), (42, 42, 64),
          (32, 32, 64), (22, 22, 64), (16, 16, 64), (11, 11, 128), (8, 8, 128), (7, 7, 128)]


def plan(rng, b, h, w, c, act):
    d = capi.BconvDesc(b, h, w, c, 3, 3, c, 1, 1, 1, 1, 1, capi.PADDING_SAME, 1, act, capi.OUT_FLOAT, 1.0, 0)
    filt = rng.integers(-2**31, 2**31 - 1, (c, 3, 3, c // 32)).astype(np.int32)
    return capi.BConv2d(d, filt, rng.uniform(0.001, 0.01, c).astype(np.float32),
                        rng.uniform(-1, 1, c).astype(np.float32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    s = torch.cuda.current_stream().cuda_stream
    lib = capi.lib()
    print(f"# {torch.cuda.get_device_name()}, batch {a.batch}, {a.iters} iterations, median of 3")
    for h, w, c in SHAPES:
        b = a.batch
        p1, p2 = plan(rng, b, h, w, c, capi.ACT_RELU), plan(rng, b, h, w, c, capi.ACT_RELU)
        x0 = torch.randn((b, h, w, c), device="cuda")
        xq = capi.quantize(x0)
        x1, x2, y2 = torch.empty_like(x0), torch.empty_like(x0), torch.empty_like(x0)
        p1q = torch.empty(xq.shape, dtype=torch.int32, device="cuda")
        p2q, q2 = torch.empty_like(p1q), torch.empty_like(p1q)
        ptr = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731

        def two():
            assert lib.lce_b200_bconv2d_run_fused(p1._h, ptr(xq), ptr(x0), 0, ptr(x1), ptr(p1q), C.c_void_p(s)) == 0
            assert lib.lce_b200_bconv2d_run_fused(p2._h, ptr(p1q), ptr(x1), 0, ptr(x2), ptr(p2q), C.c_void_p(s)) == 0

        def pair():
            assert lib.lce_b200_bconv2d_run_fused_pair(p1._h, p2._h, ptr(xq), ptr(x0), 0, 0, ptr(y2), ptr(q2),
                                                       C.c_void_p(s)) == 0

        def timed(f):
            for _ in range(5):
                f()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                f()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / a.iters

        t_two, t_pair = [], []
        for _ in range(3):
            t_two.append(timed(two))
            t_pair.append(timed(pair))
        same = torch.equal(x2.view(torch.int32), y2.view(torch.int32)) and torch.equal(p2q, q2)
        m2, mp = float(np.median(t_two)), float(np.median(t_pair))
        print(f"{h:3d} x {w:3d} x {c:3d}: two run_fused {m2:.4f} ms, pair {mp:.4f} ms, "
              f"pair / two {mp / m2:.2f}, same bits {same}")
        p1.close()
        p2.close()


if __name__ == "__main__":
    main()
