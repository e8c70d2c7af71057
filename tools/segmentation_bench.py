"""QuickNet segmentation throughput on one GPU, with and without the decoder-merge fusion.

  python tools/segmentation_bench.py [--batch 256] [--image 224] [--runs 5] [--steps 20] [--warmup 3]

Two arms on the same int8-input model (synthetic weights, compute_engine_b200/zoo.py quicknet_seg):
  base   : fuse_all() without fuse_upsample_merges() -- each decoder merge runs as
           RESIZE_NEAREST_NEIGHBOR, ADD and LceQuantize
  merged : fuse_all()
Both graphs replay as CUDA graphs with the images already in HBM. The arms alternate, `--runs`
times each, every run `--steps` steps; one JSON line gives each arm's median and range in images/s,
the card's name, power limit and max SM clock (read with nvidia-smi in the same run), whether both
arms give identical output bits at the timed batch, and from one profiled step of each arm (a
separate eager run): the encoder's, the decoder's and the head's shares of the step, and the time
and achieved bytes/s of each merge node and of the RESIZE_BILINEAR node. Bytes come from shapes:
the sources read plus the results written. Needs a GPU; there is no CPU path.
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

BASE_PASSES = ("fuse_binary_bases", "fuse_dense_blocks", "fuse_residual_blocks", "fuse_spatial_scales",
               "fuse_float_glue", "fuse_grouped_conv_affine", "fuse_quantized_activations",
               "fuse_pooled_signs", "fuse_channel_gates", "fuse_activation_chains", "fuse_residual_pairs")
ARMS = ("base", "merged")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def make_graph(blob, arm, x, profile=False):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    if arm == "merged":
        g.fuse_all()
    else:
        for p in BASE_PASSES:
            getattr(g, p)()
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
    """bytes node i reads from its float / packed sources plus the results it writes (the size
    input is a host constant)"""
    ins = [t for t in g.node_io(i)[0] if t >= 0 and g.in_arena(t)]
    outs = [t for t in g.node_outputs(i) if t >= 0]
    return sum(g.nbytes(t) for t in ins + outs)


def profile(blob, arm, x):
    g = make_graph(blob, arm, x, profile=True)
    g.invoke()
    g.reset_profile()
    g.invoke()
    times = g.node_times_ms()
    names = [g.node_name(i) for i in range(g.num_nodes())]
    # the decoder starts at the first 1x1 CONV_2D after the encoder's last block; the head is the
    # final CONV_2D and the RESIZE_BILINEAR
    first_resize = min(i for i, n in enumerate(names) if n.startswith("RESIZE_NEAREST_NEIGHBOR") or n == "builtin:97")
    dec0 = first_resize - 1
    head0 = len(names) - 2
    total = sum(times)
    parts = {"encoder": sum(times[:dec0]), "decoder": sum(times[dec0:head0]), "head": sum(times[head0:])}
    nodes = []
    for i, n in enumerate(names):
        unfused_merge = arm == "base" and n in ("builtin:0", "LceQuantize") and dec0 <= i < head0
        if n.startswith("RESIZE") or n in ("builtin:97", "builtin:23") or unfused_merge:
            b = node_bytes(g, i)
            nodes.append({"node": i, "name": n, "ms": round(times[i], 4), "bytes": b,
                          "GB_per_s": round(b / (times[i] * 1e6), 1) if times[i] else None})
    g.close()
    return {"step_ms": round(total, 4), "shares": {k: round(v / total, 4) for k, v in parts.items()},
            "nodes": nodes}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--image", type=int, default=224)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    info = gpu_info()
    blob = zoo.quicknet_seg(batch=1, seed=0, image=a.image, input_type="int8")
    x = np.random.default_rng(0).integers(-128, 128, (a.batch, a.image, a.image, 3)).astype(np.int8)
    graphs, outputs = {}, {}
    for arm in ARMS:
        g = make_graph(blob, arm, x)
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
    same = bool(np.array_equal(outputs["base"].view(np.uint8), outputs["merged"].view(np.uint8)))
    out = dict(info)
    out.update({"workload": "quicknet_seg", "batch": a.batch, "image": a.image, "input_type": "int8",
                "runs": a.runs, "steps": a.steps, "unit": "images/s", "nodes": nodes,
                "identical_outputs": same})
    for arm in ARMS:
        r = sorted(rates[arm])
        out[arm] = {"median": round(float(np.median(r)), 1), "min": round(r[0], 1), "max": round(r[-1], 1)}
    out["profile"] = {arm: profile(blob, arm, x) for arm in ARMS}
    print(json.dumps(out), flush=True)
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
