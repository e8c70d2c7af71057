"""DoReFaNet throughput on one GPU, with and without the quantised-activation fusion.

  python tools/dorefanet_bench.py [--batch 256] [--image 224] [--runs 5] [--steps 20] [--warmup 3]

Two arms on the same int8-input model (synthetic weights, compute_engine_b200/zoo.py):
  base  : fuse_all() without fuse_quantized_activations() -- each 2-bit quantiser runs as MAXIMUM,
          MINIMUM, MUL, ROUND and DIV, five passes over a float map, and each quantised layer as a
          float CONV_2D / FULLY_CONNECTED on the FP32 CUDA-core path
  fused : fuse_all() -- each quantiser (with the MAX_POOL_2D in front of it) is one pass that writes
          three bit planes, and each quantised layer a binary convolution over them on the mma.sync
          b1 kernel
Both graphs replay as CUDA graphs with the images already in HBM (the graph's compute, not the
host link). The arms alternate, `--runs` times each; the JSON line gives each arm's median and
range in images/s, the card's name, power limit and max SM clock (read with nvidia-smi in the same
run), per-node times of one profiled eager step of each arm (a separate run), the 12x12 stem's time
and share and the largest node of each arm, each Quant2 node's time and achieved bandwidth (the
float map it reads plus the planes it writes, from shapes, over its time) beside the data sheet's
3.35 TB/s of HBM3 (a data-sheet figure, not a measurement), and the agreement of the two arms'
outputs on the same seeded input: the largest absolute difference of the softmax and the share of
images whose top-1 class agrees. The fused arm computes each quantised layer in exact integers, the
base arm in float32 with a rounding per term, so the outputs agree closely but not bit for bit.
Needs a GPU; there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compute_engine_b200 import host as H, zoo  # noqa: E402

QUANT2 = ("Quant2", "MAX_POOL_2D+Quant2")
HBM_DATA_SHEET_GB_PER_S = 3350.0   # NVIDIA's H100 SXM data sheet


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def make_graph(blob, arm, x, profile=False):
    """the arm's graph, allocated for x's shape, with x written to its input"""
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    if arm == "fused":
        g.fuse_all()
    else:
        g.fuse_dense_blocks()
        g.fuse_residual_blocks()
        g.fuse_float_glue()
        g.fuse_pooled_signs()
        g.fuse_channel_gates()
        g.fuse_activation_chains()
        g.fuse_residual_pairs()
    g.enable_profiling(profile)
    g.resize_input(g.inputs()[0], x.shape)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    return g


def images_per_s(g, batch, steps):
    g.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        g.invoke()
    g.synchronize()
    return batch * steps / (time.perf_counter() - t0)


def profile(blob, arm, x):
    """one eager step after one warm-up step: [(node name, ms)] in graph order, and each Quant2
    node's time, bytes from shapes and bandwidth"""
    g = make_graph(blob, arm, x, profile=True)
    g.invoke()
    g.reset_profile()
    g.invoke()
    nodes, quant = [], []
    for i, ms in enumerate(g.node_times_ms()):
        name = g.node_name(i)
        nodes.append((name, ms))
        if name in QUANT2:
            ins, outs = g.node_io(i)
            nbytes = g.nbytes(ins[0]) + g.nbytes(outs[0])
            gbs = nbytes / (ms * 1e6) if ms else None
            quant.append({"node": name, "map": list(g.shape(ins[0])), "ms": round(ms, 4), "bytes": nbytes,
                          "gb_per_s": round(gbs, 1) if gbs else None,
                          "share_of_data_sheet_hbm": round(gbs / HBM_DATA_SHEET_GB_PER_S, 3) if gbs else None})
    g.close()
    return nodes, quant


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--image", type=int, default=224)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if H.device_count() < 1:
        print("dorefanet_bench: no CUDA device; nothing is measured without one", file=sys.stderr)
        return 2
    info = gpu_info()
    blob = zoo.dorefanet(batch=1, seed=0, image=a.image, input_type="int8")
    x = np.random.default_rng(0).integers(-128, 128, (a.batch, a.image, a.image, 3)).astype(np.int8)
    arms = ("base", "fused")
    graphs, outputs = {}, {}
    for arm in arms:
        g = make_graph(blob, arm, x)
        g.invoke()                                   # eager: plans are built
        outputs[arm] = g.read(g.outputs()[0])
        g.enable_cuda_graph(True)
        for _ in range(a.warmup + 2):                # the first two replays capture the graph
            g.invoke()
        graphs[arm] = g
    rates = {arm: [] for arm in arms}
    for _ in range(a.runs):
        for arm in arms:
            rates[arm].append(images_per_s(graphs[arm], a.batch, a.steps))
    nodes = {arm: graphs[arm].num_nodes() for arm in arms}
    for g in graphs.values():
        g.close()
    out = dict(info)
    out.update({
        "workload": "dorefanet", "batch": a.batch, "image": a.image, "input_type": "int8", "runs": a.runs,
        "steps": a.steps, "unit": "images/s", "nodes": nodes,
        "softmax_max_abs_diff": float(np.abs(outputs["base"] - outputs["fused"]).max()),
        "top1_agreement": float((outputs["base"].argmax(-1) == outputs["fused"].argmax(-1)).mean()),
        "hbm_data_sheet_gb_per_s": HBM_DATA_SHEET_GB_PER_S,
    })
    for arm in arms:
        r = sorted(rates[arm])
        out[arm] = {"median": round(float(np.median(r)), 1), "min": round(r[0], 1), "max": round(r[-1], 1)}
        prof, quant = profile(blob, arm, x)
        total = sum(ms for _, ms in prof)
        stem = next(ms for name, ms in prof if name == "builtin:3")   # the first CONV_2D is the 12x12 stem
        big = max(range(len(prof)), key=lambda i: prof[i][1])
        out[arm].update({
            "profiled_step_ms": round(total, 4), "stem_ms": round(stem, 4),
            "stem_share": round(stem / total, 3) if total else None,
            "largest_node": {"index": big, "name": prof[big][0], "ms": round(prof[big][1], 4)},
            "nodes_ms": [[name, round(ms, 4)] for name, ms in prof],
        })
        if arm == "fused":
            out["quant2_nodes"] = quant
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
