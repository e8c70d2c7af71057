"""Time bitpacked-output LceBconv2d layers on the mma.sync b1 kernel against the wgmma kernel that
takes the same plans with LCE_B200_BCONV_IMMA=0, with CUDA events, and check that both give the
same words.

    python tools/bitpacked_bench.py [--batch 256] [--iters 100] [--runs 5]

Prints the card, its power limit and max SM clock, then one line per layer: the median (min-max) of
`runs` alternated runs of `iters` launches per kernel, in microseconds per launch. The layers are
3x3 one-padded: BinaryAlexNet's 13x13 conv3 -> conv4 -> conv5 and QuickNet-sized shapes."""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
import lce_testlib as L  # noqa: E402
from compute_engine_b200 import capi  # noqa: E402

LAYERS = [(13, 384, 384), (13, 384, 256), (56, 64, 64), (28, 128, 128), (14, 256, 256)]  # (H=W, C_in, C_out)
ARMS = (("mma.sync b1", "1"), ("wgmma", "0"))   # LCE_B200_BCONV_IMMA at plan creation


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this tool times the GPU"
    print(f"# {card()}; batch {a.batch}, {a.iters} launches per run, median (min-max) of {a.runs} alternated runs")
    for hw, cin, cout in LAYERS:
        case = L.make_bconv_case(1, a.batch, hw, hw, cin, 3, 3, cout, out_type=L.OUT_BITPACKED)
        x = torch.from_numpy(case.inp).cuda()
        plans, outs = {}, {}
        for arm, imma in ARMS:
            os.environ["LCE_B200_BCONV_IMMA"] = imma
            d = capi.BconvDesc(*[getattr(case.desc, n) for n, _ in case.desc._fields_])
            plans[arm] = capi.BConv2d(d, case.filt, None, None, case.thr)
            outs[arm] = plans[arm](x)
            for _ in range(10):
                plans[arm](x, outs[arm])
        os.environ.pop("LCE_B200_BCONV_IMMA")
        torch.cuda.synchronize()
        before = capi.path_counts()
        plans["mma.sync b1"](x, outs["mma.sync b1"])
        plans["wgmma"](x, outs["wgmma"])
        torch.cuda.synchronize()
        assert [y - b for b, y in zip(before, capi.path_counts())] == [1, 1, 0], "not the two kernels"
        same = torch.equal(outs["mma.sync b1"], outs["wgmma"])
        times = {arm: [] for arm in plans}
        for _ in range(a.runs):
            for arm, p in plans.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.iters):
                    p(x, outs[arm])
                e1.record()
                torch.cuda.synchronize()
                times[arm].append(e0.elapsed_time(e1) / a.iters * 1000)
        cols = "  ".join(f"{arm} {np.median(t):.1f} ({min(t):.1f}-{max(t):.1f}) us" for arm, t in times.items())
        print(f"{hw}x{hw} {cin}->{cout} 3x3: {cols}  same words: {same}")
        for p in plans.values():
            p.close()


if __name__ == "__main__":
    main()
