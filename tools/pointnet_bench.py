"""Binary PointNet (zoo.binary_pointnet, BiPointNet without T-Nets) on one GPU: the last point-wise layer's max
over points fused into the b1 kernel's store, against the same graph without that fusion and without either
binary dense fusion.

  python tools/pointnet_bench.py [--batch 256] [--points 1024] [--alpha none|lsr] [--runs 5] [--steps 20]
                                 [--warmup 3]

Three arms (synthetic weights, float32 points):
  fused    : fuse_all() -- the last point-wise layer and its REDUCE_MAX one LceBfc+MUL+ADD+REDUCE_MAX+LceQuantize
  fc       : fuse_all() without fuse_binary_fc_max() -- that layer an LceBfc+MUL+ADD storing [B, P, 1024]
             floats, then the REDUCE_MAX builtin
  unfused  : fuse_all() without fuse_binary_fc_max() and fuse_binary_fully_connected() -- every binary layer
             LceDequantize and a float FULLY_CONNECTED
Every graph replays as a CUDA graph with the points already in HBM. The arms alternate, `--runs` times each,
every run `--steps` steps; one JSON line gives each arm's median and range in images/s, the card's name,
power limit and max SM clock (read with nvidia-smi in the same run), whether the fused and fc arms give
identical output bits (and the unfused arm too with +-1 weights), and from one profiled step of each arm (a
separate eager run): every node's time, and the fused node's time against the LceBfc + REDUCE_MAX pair it
replaces, with bytes/s. Bytes come from shapes (the arena tensors a node reads and writes, its temporaries,
plus its constant weights). Needs a GPU; there is no CPU path.
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

ARMS = ("fused", "fc", "unfused")
PASSES = ("fuse_binary_bases", "fuse_dense_blocks", "fuse_binary_transpose_convs", "fuse_binary_fc_max",
          "fuse_binary_fully_connected", "fuse_residual_blocks", "fuse_spatial_scales", "fuse_float_glue",
          "fuse_upsample_merges", "fuse_resize_argmax", "fuse_subpixel_convs", "fuse_grouped_conv_affine",
          "fuse_quantized_activations", "fuse_pooled_signs", "fuse_channel_gates", "fuse_activation_chains",
          "fuse_residual_pairs")
SKIP = {"fused": (), "fc": ("fuse_binary_fc_max",), "unfused": ("fuse_binary_fc_max", "fuse_binary_fully_connected")}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def make_graph(a, arm, x, profile=False):
    alpha = None if a.alpha == "none" else a.alpha
    g = H.HostGraph.from_tflite(zoo.binary_pointnet(batch=x.shape[0], seed=0, points=a.points, alpha=alpha),
                                device_arena=True)
    if arm == "fused":
        g.fuse_all()
    else:
        for p in PASSES:
            if p not in SKIP[arm]:
                getattr(g, p)()
    g.enable_profiling(profile)
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


def node_bytes(g, i):
    ins = g.node_io(i)[0]
    moved = [t for t in ins if t >= 0 and g.in_arena(t)] + [t for t in g.node_outputs(i) if t >= 0]
    weights = ins[1] if len(ins) > 1 and ins[1] >= 0 and not g.in_arena(ins[1]) else None
    return sum(g.nbytes(t) for t in moved) + (g.nbytes(weights) if weights is not None else 0)


def profile(a, arm, x):
    g = make_graph(a, arm, x, profile=True)
    g.invoke()
    g.reset_profile()
    g.invoke()
    times = g.node_times_ms()
    names = [g.node_name(i) for i in range(g.num_nodes())]
    nodes = []
    for i, (n, t) in enumerate(zip(names, times)):
        b = node_bytes(g, i)
        nodes.append({"node": i, "name": n, "ms": round(t, 4), "bytes": b,
                      "GB_per_s": round(b / (t * 1e6), 1) if t else None})
    g.close()
    # the max over points and the layer before it: the fused node, or the REDUCE_MAX and its producer
    if arm == "fused":
        pair = [d for d in nodes if "REDUCE_MAX" in d["name"]]
    else:
        r = next(i for i, n in enumerate(names) if n == "builtin:82")
        pair = nodes[r - 1:r + 1]
    return {"step_ms": round(sum(times), 4), "max_layer": pair,
            "max_layer_ms": round(sum(d["ms"] for d in pair), 4), "nodes": nodes}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--points", type=int, default=1024)
    ap.add_argument("--alpha", choices=("none", "lsr"), default="none")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    info = gpu_info()
    x = np.random.default_rng(0).standard_normal((a.batch, a.points, 3)).astype(np.float32)
    graphs, outputs = {}, {}
    for arm in ARMS:
        g = make_graph(a, arm, x)
        g.invoke()                                   # eager: plans are built
        outputs[arm] = g.read(g.outputs()[0])
        g.enable_cuda_graph(True)
        for _ in range(a.warmup + 2):                # the first two replays capture the graph
            g.invoke()
        graphs[arm] = g
    rates = {arm: [] for arm in ARMS}
    for _ in range(a.runs):
        for arm in ARMS:
            rates[arm].append(images_per_s(graphs[arm], a.batch, a.steps))
    nodes = {arm: graphs[arm].num_nodes() for arm in ARMS}
    for g in graphs.values():
        g.close()
    out = dict(info)
    out.update({"workload": "binary_pointnet", "batch": a.batch, "points": a.points, "alpha": a.alpha,
                "runs": a.runs, "steps": a.steps, "unit": "images/s", "nodes": nodes})

    def same(p, q):
        return bool(np.array_equal(outputs[p].view(np.uint8), outputs[q].view(np.uint8)))

    ok = same("fused", "fc")
    out["identical_outputs_fused_fc"] = ok
    out["identical_outputs_fused_unfused"] = same("fused", "unfused")
    out["max_softmax_diff_unfused"] = float(np.abs(outputs["fused"] - outputs["unfused"]).max())
    for arm in ARMS:
        r = sorted(rates[arm])
        out[arm] = {"median": round(float(np.median(r)), 1), "min": round(r[0], 1), "max": round(r[-1], 1)}
    out["profile"] = {arm: profile(a, arm, x) for arm in ARMS}
    print(json.dumps(out), flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
