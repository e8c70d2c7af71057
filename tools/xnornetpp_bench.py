"""XNOR-Net++ throughput on one GPU, with and without the spatial-scale fusion.

  python tools/xnornetpp_bench.py [--batch 256] [--image 224] [--pad-values 0 1] [--runs 5]
                                  [--steps 20] [--warmup 3]

For each padding value, two arms on the same int8-input model (synthetic weights,
compute_engine_b200/zoo.py xnornetpp):
  base   : fuse_all() without fuse_spatial_scales() -- each block's MUL(Gamma) -> ADD(shortcut) and
           the next block's MUL -> ADD -> LceQuantize run as float passes (the ADD -> LceQuantize as
           one)
  scales : fuse_all()
Both graphs replay as CUDA graphs with the images already in HBM (the graph's compute, not the
host link). The arms alternate, `--runs` times each, every run `--steps` steps; one JSON line per
padding value gives each arm's median and range in images/s, the card's name, power limit and max
SM clock (read with nvidia-smi in the same run), per-node-name summed times of one profiled step of
each arm, and whether both arms give identical output bits on the same seeded input: with every
tensor kept (no arena reuse, so both arms lay tensors out alike) and with the arenas the timed
graphs use. Needs a GPU; there is no CPU path.
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compute_engine_b200 import host as H, zoo  # noqa: E402

BASE_PASSES = ("fuse_dense_blocks", "fuse_residual_blocks", "fuse_float_glue", "fuse_grouped_conv_affine",
               "fuse_quantized_activations", "fuse_pooled_signs", "fuse_channel_gates",
               "fuse_activation_chains", "fuse_residual_pairs")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def make_graph(blob, arm, x, profile=False, preserve=False):
    """the arm's graph, allocated for x's shape, with x written to its input"""
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    if arm == "scales":
        g.fuse_all()
    else:
        for p in BASE_PASSES:
            getattr(g, p)()
    g.enable_profiling(profile)
    g.preserve_all_tensors(preserve)
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
    """per-node-name device time (ms) of one eager step, after one warm-up step"""
    g = make_graph(blob, arm, x, profile=True)
    g.invoke()
    g.reset_profile()
    g.invoke()
    by_name = collections.defaultdict(float)
    for i, ms in enumerate(g.node_times_ms()):
        by_name[g.node_name(i)] += ms
    g.close()
    return {k: round(v, 4) for k, v in sorted(by_name.items(), key=lambda kv: -kv[1])}


def bench(a, info, pad_values):
    blob = zoo.xnornetpp(batch=1, seed=0, image=a.image, input_type="int8", pad_values=pad_values)
    x = np.random.default_rng(0).integers(-128, 128, (a.batch, a.image, a.image, 3)).astype(np.int8)
    arms = ("base", "scales")
    kept = {}
    for arm in arms:
        g = make_graph(blob, arm, x, preserve=True)
        g.invoke()
        kept[arm] = g.read(g.outputs()[0])
        g.close()
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
    prof = {arm: profile(blob, arm, x) for arm in arms}
    out = dict(info)
    out.update({
        "workload": "xnornetpp", "batch": a.batch, "image": a.image, "input_type": "int8",
        "pad_values": pad_values, "runs": a.runs, "steps": a.steps, "unit": "images/s",
        "nodes": nodes,
        "identical_outputs": bool(np.array_equal(kept["base"].view(np.uint8), kept["scales"].view(np.uint8))),
        "identical_outputs_reused_arena": bool(np.array_equal(outputs["base"].view(np.uint8),
                                                              outputs["scales"].view(np.uint8))),
    })
    for arm in arms:
        r = sorted(rates[arm])
        out[arm] = {"median": round(float(np.median(r)), 1), "min": round(r[0], 1), "max": round(r[-1], 1)}
    out["profile_ms_per_step"] = prof
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--image", type=int, default=224)
    ap.add_argument("--pad-values", type=int, nargs="+", default=[0, 1], choices=(0, 1))
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    info = gpu_info()
    ok = True
    for pv in a.pad_values:
        out = bench(a, info, pv)
        print(json.dumps(out), flush=True)
        ok = ok and out["identical_outputs"] and out["identical_outputs_reused_arena"]
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
