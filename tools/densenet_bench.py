"""BinaryDenseNet and MeliusNet throughput on one GPU, with and without the dense-block fusion.

  python tools/densenet_bench.py [--model binarydensenet28|...|meliusnet22] [--batch 256] [--image 224]
                                 [--pad-values 0] [--runs 5] [--steps 20] [--warmup 3]

Two arms on the same int8-input model (synthetic weights, compute_engine_b200/zoo.py):
  base  : fuse_all() without fuse_dense_blocks() -- each dense layer runs as MUL, ADD, LceQuantize,
          LceBconv2d and a CONCATENATION that copies the whole map; each MeliusNet improvement
          layer as MUL, ADD, LceQuantize, two STRIDED_SLICE copies, LceBconv2d + ADD and a
          CONCATENATION
  dense : fuse_all() -- each layer packs its signs in one pass and writes its new channels into
          the block's final map in place (an improvement layer adds them to the map's last ones)
Both graphs replay as CUDA graphs with the images already in HBM (the graph's compute, not the
host link). The arms alternate, `--runs` times each; the JSON line gives each arm's median and
range in images/s, the card's name, power limit and max SM clock (read with nvidia-smi in the same
run), per-node-name summed times of one profiled step of each arm with the dense and improvement
layers' share of it, and whether both arms give
identical output bits on the same seeded input: with every tensor kept (no arena reuse, so both
arms lay tensors out alike) and with the arenas the timed graphs use. Needs a GPU; there is no CPU
path.
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


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def make_graph(blob, arm, x, profile=False, preserve=False):
    """the arm's graph, allocated for x's shape, with x written to its input"""
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    if arm == "dense":
        g.fuse_all()
    else:
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="binarydensenet28",
                    choices=[m for m in zoo.MODELS if m.startswith(("binarydensenet", "meliusnet"))])
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
    arms = ("base", "dense")
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
        "workload": a.model, "batch": a.batch, "image": a.image, "input_type": "int8",
        "pad_values": a.pad_values, "runs": a.runs, "steps": a.steps, "unit": "images/s",
        "nodes": nodes,
        "identical_outputs": bool(np.array_equal(kept["base"].view(np.uint8), kept["dense"].view(np.uint8))),
        "identical_outputs_reused_arena": bool(np.array_equal(outputs["base"].view(np.uint8),
                                                              outputs["dense"].view(np.uint8))),
    })
    for arm in arms:
        r = sorted(rates[arm])
        out[arm] = {"median": round(float(np.median(r)), 1), "min": round(r[0], 1), "max": round(r[-1], 1)}
    out["profile_ms_per_step"] = prof
    # the dense and improvement layers' nodes: the fused ones, or the ops each replaces (in the base
    # arm this also counts the stem's, transitions' and head's BatchNorm MUL and ADD). The
    # improvement layers alone: their fused nodes (dense arm), or the ops only they have (base arm:
    # the slices and the convolution with its ADD).
    dense_node = "MUL+ADD+LceQuantize+LceBconv2d+CONCATENATION"
    improvement_node = "MUL+ADD+LceQuantize+LceBconv2d+STRIDED_SLICE+ADD+CONCATENATION"
    layer_ops = ("builtin:18", "builtin:0", "LceQuantize", "ADD+LceQuantize", "LceBconv2d", "builtin:2",
                 "builtin:45", "LceBconv2d+ADD")
    for arm in arms:
        total = sum(prof[arm].values())
        fused = (dense_node, improvement_node)
        dense = sum(v for k, v in prof[arm].items() if k in fused or (arm == "base" and k in layer_ops))
        impr = sum(v for k, v in prof[arm].items()
                   if k == improvement_node or (arm == "base" and k in ("builtin:45", "LceBconv2d+ADD")))
        out[arm]["dense_layers_ms"] = round(dense, 4)
        out[arm]["dense_layers_share"] = round(dense / total, 3) if total else None
        out[arm]["improvement_layers_ms"] = round(impr, 4)
        out[arm]["improvement_layers_share"] = round(impr / total, 3) if total else None
    print(json.dumps(out))
    return 0 if out["identical_outputs"] else 1


if __name__ == "__main__":
    sys.exit(main())
