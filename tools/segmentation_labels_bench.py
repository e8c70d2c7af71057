"""QuickNet segmentation throughput on one GPU when the graph ends in a per-pixel label map.

  python tools/segmentation_labels_bench.py [--batch 256] [--image 224] [--runs 5] [--steps 20] [--warmup 3]

Three arms on the same int8-input model (synthetic weights, compute_engine_b200/zoo.py quicknet_seg):
  logits         : quicknet_seg() with fuse_all() -- the [B, image, image, 21] logits
  labels-unfused : quicknet_seg(labels="int64") with fuse_all() without fuse_resize_argmax() -- the head
                   runs RESIZE_BILINEAR, writing the logits map, then ARG_MAX
  labels         : quicknet_seg(labels="int64") with fuse_all() -- RESIZE_BILINEAR+ARG_MAX in one node
Every graph replays as a CUDA graph with the images already in HBM. The arms alternate, `--runs` times
each, every run `--steps` steps; one JSON line gives each arm's median and range in images/s, the
card's name, power limit and max SM clock (read with nvidia-smi in the same run), whether the two label
arms give identical bits and whether they equal TFLite's ARG_MAX rule applied on the host to the logits
arm's output at the timed batch, and from one profiled eager step of each arm (a separate run): each
head node's time and achieved bytes/s (bytes from shapes: the arena sources read plus the results
written) and the head's share of the step. It also times the copy of each arm's graph output to pinned
host memory (read_ptr_async, then synchronize). Needs a GPU; there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compute_engine_b200 import host as H, zoo  # noqa: E402

UNFUSED_PASSES = ("fuse_binary_bases", "fuse_dense_blocks", "fuse_residual_blocks", "fuse_spatial_scales",
                  "fuse_float_glue", "fuse_upsample_merges", "fuse_grouped_conv_affine",
                  "fuse_quantized_activations", "fuse_pooled_signs", "fuse_channel_gates",
                  "fuse_activation_chains", "fuse_residual_pairs")
ARMS = ("logits", "labels-unfused", "labels")
HEAD_NODES = {"logits": 2, "labels-unfused": 3, "labels": 2}   # the final CONV_2D and what follows it


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def argmax_rule(x):
    """TFLite's ARG_MAX over the last axis (reference/arg_min_max.h): v = x[0], idx = 0, then x[i]
    is taken only when x[i] > v."""
    v = x[..., 0].copy()
    idx = np.zeros(v.shape, np.int64)
    with np.errstate(invalid="ignore"):
        for i in range(1, x.shape[-1]):
            take = x[..., i] > v
            v = np.where(take, x[..., i], v)
            idx[take] = i
    return idx


def make_graph(blobs, arm, x, profile=False):
    g = H.HostGraph.from_tflite(blobs[arm], device_arena=True)
    if arm == "labels-unfused":
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


def copy_ms(g, reps=10):
    """Median time to copy the graph's output into pinned host memory."""
    t = g.outputs()[0]
    n = g.nbytes(t)
    buf = torch.empty(n, dtype=torch.uint8, pin_memory=True)
    times = []
    for _ in range(reps + 1):
        g.synchronize()
        t0 = time.perf_counter()
        g.read_ptr_async(t, buf.data_ptr(), n)
        g.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return {"bytes": n, "ms": round(float(np.median(times[1:])), 4)}


def node_bytes(g, i):
    """bytes node i reads from its arena sources plus the results it writes"""
    ins = [t for t in g.node_io(i)[0] if t >= 0 and g.in_arena(t)]
    outs = [t for t in g.node_outputs(i) if t >= 0]
    return sum(g.nbytes(t) for t in ins + outs)


def profile(blobs, arm, x):
    g = make_graph(blobs, arm, x, profile=True)
    g.invoke()
    g.reset_profile()
    g.invoke()
    times = g.node_times_ms()
    total = sum(times)
    head0 = g.num_nodes() - HEAD_NODES[arm]
    nodes = []
    for i in range(head0, g.num_nodes()):
        b = node_bytes(g, i)
        nodes.append({"node": i, "name": g.node_name(i), "ms": round(times[i], 4), "bytes": b,
                      "GB_per_s": round(b / (times[i] * 1e6), 1) if times[i] else None})
    g.close()
    head = sum(times[head0:])
    return {"step_ms": round(total, 4), "head_ms": round(head, 4), "head_share": round(head / total, 4),
            "head_nodes": nodes}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--image", type=int, default=224)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    info = gpu_info()
    logits_blob = zoo.quicknet_seg(batch=1, seed=0, image=a.image, input_type="int8")
    labels_blob = zoo.quicknet_seg(batch=1, seed=0, image=a.image, input_type="int8", labels="int64")
    blobs = {"logits": logits_blob, "labels-unfused": labels_blob, "labels": labels_blob}
    x = np.random.default_rng(0).integers(-128, 128, (a.batch, a.image, a.image, 3)).astype(np.int8)
    graphs, outputs = {}, {}
    for arm in ARMS:
        g = make_graph(blobs, arm, x)
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
    copies = {arm: copy_ms(graphs[arm]) for arm in ARMS}
    for g in graphs.values():
        g.close()
    lab, unf = outputs["labels"], outputs["labels-unfused"]
    same = bool(lab.dtype == unf.dtype and np.array_equal(lab, unf))
    rule = bool(np.array_equal(lab, argmax_rule(outputs["logits"])))
    out = dict(info)
    out.update({"workload": "quicknet_seg", "batch": a.batch, "image": a.image, "input_type": "int8",
                "labels": "int64", "runs": a.runs, "steps": a.steps, "unit": "images/s", "nodes": nodes,
                "identical_labels": same, "labels_equal_argmax_of_logits": rule})
    for arm in ARMS:
        r = sorted(rates[arm])
        out[arm] = {"median": round(float(np.median(r)), 1), "min": round(r[0], 1), "max": round(r[-1], 1)}
    out["copy_to_pinned_host"] = copies
    out["profile"] = {arm: profile(blobs, arm, x) for arm in ARMS}
    print(json.dumps(out), flush=True)
    return 0 if same and rule else 1


if __name__ == "__main__":
    sys.exit(main())
