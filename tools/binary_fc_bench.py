"""BinaryAlexNet or XNOR-Net with larq's binary dense head on one GPU: the dense layers with and without their
fusion into the b1 convolution, and the head restated as convolutions (the default zoo model) for reference.

  python tools/binary_fc_bench.py --model binaryalexnet|xnornet [--pad-values 0] [--batch 256] [--image 224]
                                  [--runs 5] [--steps 20] [--warmup 3]

Three arms on int8-input models (synthetic weights, compute_engine_b200/zoo.py):
  fused   : dense="fully_connected", fuse_all() -- each 4096-wide layer one LceBfc[+MUL+ADD][+LceQuantize]
  unfused : dense="fully_connected", fuse_all() without fuse_binary_fully_connected() -- each layer
            LceDequantize and a float FULLY_CONNECTED (and its BatchNorm and sign)
  conv    : dense="conv" (the dense layers as LceBconv2d), fuse_all()
Every graph replays as a CUDA graph with the images already in HBM. The arms alternate, `--runs` times each,
every run `--steps` steps; one JSON line gives each arm's median and range in images/s, the card's name,
power limit and max SM clock (read with nvidia-smi in the same run), for BinaryAlexNet whether the fused and
unfused arms give identical output bits, for XNOR-Net the largest softmax difference between them and their
top-1 agreement, and from one profiled step of each arm (a separate eager run): every node's time, the
head's share of the step (from the flattened pooled sign on; the conv arm from its last pooled sign) and
each dense node's time and bytes/s. Bytes come from shapes (the arena tensors a node reads plus those it
writes, plus its constant weights: packed signs for a fused node, float32 for a FULLY_CONNECTED). Needs a
GPU; there is no CPU path.
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

ARMS = ("fused", "unfused", "conv")
UNFUSED_PASSES = ("fuse_binary_bases", "fuse_dense_blocks", "fuse_binary_transpose_convs", "fuse_residual_blocks",
                  "fuse_spatial_scales", "fuse_float_glue", "fuse_upsample_merges", "fuse_resize_argmax",
                  "fuse_subpixel_convs", "fuse_grouped_conv_affine", "fuse_quantized_activations",
                  "fuse_pooled_signs", "fuse_channel_gates", "fuse_activation_chains", "fuse_residual_pairs")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def model(name, arm, batch, image, pad_values):
    """The model at the timed batch: LceDequantize keeps its output's shape (the reference's Prepare checks
    it and does not resize), so a graph with one left cannot be resized to another batch."""
    dense = "conv" if arm == "conv" else "fully_connected"
    return getattr(zoo, name)(batch=batch, seed=0, image=image, input_type="int8", pad_values=pad_values,
                              dense=dense)


def make_graph(a, arm, x, profile=False):
    g = H.HostGraph.from_tflite(model(a.model, arm, x.shape[0], a.image, a.pad_values), device_arena=True)
    if arm == "unfused":
        for p in UNFUSED_PASSES:
            getattr(g, p)()
    else:
        g.fuse_all()
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


def node_bytes(g, i):
    ins = g.node_io(i)[0]
    moved = [t for t in ins if t >= 0 and g.in_arena(t)] + [t for t in g.node_outputs(i) if t >= 0]
    weights = ins[1] if len(ins) > 1 and ins[1] >= 0 and not g.in_arena(ins[1]) else None
    return sum(g.nbytes(t) for t in moved) + (g.nbytes(weights) if weights is not None else 0)


def is_dense(name):
    return name.startswith("LceBfc") or name in ("builtin:9", "LceDequantize")


def profile(a, arm, x):
    g = make_graph(a, arm, x, profile=True)
    g.invoke()
    g.reset_profile()
    g.invoke()
    times = g.node_times_ms()
    names = [g.node_name(i) for i in range(g.num_nodes())]
    head0 = max(i for i, n in enumerate(names) if n.startswith("MAX_POOL_2D"))
    total = sum(times)
    dense = []
    for i, n in enumerate(names):
        if is_dense(n):
            b = node_bytes(g, i)
            dense.append({"node": i, "name": n, "ms": round(times[i], 4), "bytes": b,
                          "GB_per_s": round(b / (times[i] * 1e6), 1) if times[i] else None})
    g.close()
    return {"step_ms": round(total, 4), "head_share": round(sum(times[head0:]) / total, 4),
            "head_ms": round(sum(times[head0:]), 4), "dense_nodes": dense,
            "nodes": [{"node": i, "name": n, "ms": round(t, 4)} for i, (n, t) in enumerate(zip(names, times))]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=("binaryalexnet", "xnornet"), required=True)
    ap.add_argument("--pad-values", type=int, default=0, choices=(0, 1))
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--image", type=int, default=224)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    info = gpu_info()
    x = np.random.default_rng(0).integers(-128, 128, (a.batch, a.image, a.image, 3)).astype(np.int8)
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
    out.update({"workload": f"{a.model} dense head", "batch": a.batch, "image": a.image, "input_type": "int8",
                "pad_values": a.pad_values, "runs": a.runs, "steps": a.steps, "unit": "images/s", "nodes": nodes})
    f, u = outputs["fused"], outputs["unfused"]
    ok = True
    if a.model == "binaryalexnet":
        ok = bool(np.array_equal(f.view(np.uint8), u.view(np.uint8)))
        out["identical_outputs"] = ok
    else:
        out["max_softmax_diff"] = float(np.abs(f - u).max())
        out["top1_agreement"] = float((f.argmax(1) == u.argmax(1)).mean())
    for arm in ARMS:
        r = sorted(rates[arm])
        out[arm] = {"median": round(float(np.median(r)), 1), "min": round(r[0], 1), "max": round(r[-1], 1)}
    out["profile"] = {arm: profile(a, arm, x) for arm in ARMS}
    print(json.dumps(out), flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
