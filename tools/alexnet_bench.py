"""BinaryAlexNet and XNOR-Net throughput on one GPU, with and without the pooled-sign fusion.

  python tools/alexnet_bench.py [--model binaryalexnet|xnornet] [--batch 256] [--image 224]
                                [--pad-values 0] [--runs 5] [--steps 20] [--warmup 3]

Two arms on the same int8-input model (synthetic weights, compute_engine_b200/zoo.py):
  base   : fuse_all() without fuse_pooled_signs() -- each pooled layer runs as MAX_POOL_2D, MUL and
           ADD+LceQuantize, three passes that each read or write a full float map
  pooled : fuse_all() -- each pooled layer reads the convolution's float map once and writes only
           the signs (MAX_POOL_2D+MUL+ADD+LceQuantize)
Both graphs replay as CUDA graphs with the images already in HBM (the graph's compute, not the
host link). The arms alternate, `--runs` times each; the JSON line gives each arm's median and
range in images/s, the card's name, power limit and max SM clock (read with nvidia-smi in the same
run), per-node-name summed times of one profiled step of each arm, the pooled layers' time and
share of it (the fused nodes, or the nodes they replace), each fused node's time and achieved
bandwidth (its float map plus its packed signs over its time), the 11x11 stem's time and share,
and whether both arms give identical output bits on the same seeded input: with every tensor kept
(no arena reuse, so both arms lay tensors out alike) and with the arenas the timed graphs use.
Exits 1 when the outputs differ. Needs a GPU; there is no CPU path.
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

POOLED = "MAX_POOL_2D+MUL+ADD+LceQuantize"
# the nodes a pooled layer runs as in the base arm (no other MAX_POOL_2D, MUL or ADD is in these models)
POOLED_BASE = ("builtin:17", "builtin:18", "ADD+LceQuantize")
STEM = "builtin:3"


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def make_graph(blob, arm, x, profile=False, preserve=False):
    """the arm's graph, allocated for x's shape, with x written to its input"""
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    if arm == "pooled":
        g.fuse_all()
    else:
        g.fuse_dense_blocks()
        g.fuse_residual_blocks()
        g.fuse_float_glue()
        g.fuse_channel_gates()
        g.fuse_activation_chains()
        g.fuse_residual_pairs()
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
    """per-node-name device time (ms) of one eager step after one warm-up step, and each fused
    pooled node's (time ms, bytes it must move)"""
    g = make_graph(blob, arm, x, profile=True)
    g.invoke()
    g.reset_profile()
    g.invoke()
    by_name = collections.defaultdict(float)
    layers = []
    for i, ms in enumerate(g.node_times_ms()):
        name = g.node_name(i)
        by_name[name] += ms
        if name == POOLED:
            ins, outs = g.node_io(i)
            nbytes = g.nbytes(ins[0]) + g.nbytes(outs[0])
            layers.append({"map": list(g.shape(ins[0])), "ms": round(ms, 4), "bytes": nbytes,
                           "gb_per_s": round(nbytes / (ms * 1e6), 1) if ms else None})
    g.close()
    return {k: round(v, 4) for k, v in sorted(by_name.items(), key=lambda kv: -kv[1])}, layers


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="binaryalexnet", choices=["binaryalexnet", "xnornet"])
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--image", type=int, default=224)
    ap.add_argument("--pad-values", type=int, default=0, choices=(0, 1))
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    info = gpu_info()
    blob = zoo.MODELS[a.model](batch=1, seed=0, image=a.image, input_type="int8", pad_values=a.pad_values)
    x = np.random.default_rng(0).integers(-128, 128, (a.batch, a.image, a.image, 3)).astype(np.int8)
    arms = ("base", "pooled")
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
    prof, layers = {}, {}
    for arm in arms:
        prof[arm], layers[arm] = profile(blob, arm, x)
    out = dict(info)
    out.update({
        "workload": a.model, "batch": a.batch, "image": a.image, "input_type": "int8",
        "pad_values": a.pad_values, "runs": a.runs, "steps": a.steps, "unit": "images/s",
        "nodes": nodes,
        "identical_outputs": bool(np.array_equal(kept["base"].view(np.uint8), kept["pooled"].view(np.uint8))),
        "identical_outputs_reused_arena": bool(np.array_equal(outputs["base"].view(np.uint8),
                                                              outputs["pooled"].view(np.uint8))),
    })
    for arm in arms:
        r = sorted(rates[arm])
        out[arm] = {"median": round(float(np.median(r)), 1), "min": round(r[0], 1), "max": round(r[-1], 1)}
        total = sum(prof[arm].values())
        pooled = sum(v for k, v in prof[arm].items() if k == POOLED or (arm == "base" and k in POOLED_BASE))
        stem = prof[arm].get(STEM, 0.0)
        out[arm]["pooled_layers_ms"] = round(pooled, 4)
        out[arm]["pooled_layers_share"] = round(pooled / total, 3) if total else None
        out[arm]["stem_ms"] = round(stem, 4)
        out[arm]["stem_share"] = round(stem / total, 3) if total else None
    out["profile_ms_per_step"] = prof
    out["pooled_layers"] = layers["pooled"]
    print(json.dumps(out))
    return 0 if out["identical_outputs"] and out["identical_outputs_reused_arena"] else 1


if __name__ == "__main__":
    sys.exit(main())
