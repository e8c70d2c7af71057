"""Binary super-resolution throughput on one GPU, with and without the sub-pixel tail fusion.

  python tools/superres_bench.py [--batch 16] [--height 180] [--width 320] [--scales 2 4] [--runs 5] [--steps 20]
                                 [--warmup 3]

For each scale, two arms on the same float32-input model (synthetic weights, compute_engine_b200/zoo.py
binary_srnet: 64 channels, 16 binary residual blocks, the tail CONV_2D 3x3 64 -> 3 r^2 -> DEPTH_TO_SPACE(r)
-> ADD(RESIZE_BILINEAR(image))):
  unfused : fuse_all() without fuse_subpixel_convs() -- the tail runs as its four builtins
  fused   : fuse_all() -- the tail is one CONV_2D+DEPTH_TO_SPACE+RESIZE_BILINEAR+ADD node
Every graph replays as a CUDA graph with the images already in HBM. The arms alternate, `--runs` times
each, every run `--steps` steps; one JSON line gives each arm's median and range in images/s, the card's
name, power limit and max SM clock (read with nvidia-smi in the same run), whether the two arms give
identical output bits, and from one profiled eager step of each arm (a separate run): every node's time,
the tail's nodes with their achieved FLOP/s (the tail convolution's 2 * B * H * W * Cout * 9 * Cin, from
shapes) and bytes/s (the arena sources each node reads plus the results it writes, from shapes), and
the tail's and the body's (the binary blocks and the long skip) shares of the step. Needs a GPU; there
is no CPU path.
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

UNFUSED_PASSES = ("fuse_binary_bases", "fuse_dense_blocks", "fuse_residual_blocks", "fuse_spatial_scales",
                  "fuse_float_glue", "fuse_upsample_merges", "fuse_resize_argmax", "fuse_grouped_conv_affine",
                  "fuse_quantized_activations", "fuse_pooled_signs", "fuse_channel_gates",
                  "fuse_activation_chains", "fuse_residual_pairs")
ARMS = ("unfused", "fused")
TAIL_NODES = {"unfused": 4, "fused": 1}   # CONV_2D, DEPTH_TO_SPACE, RESIZE_BILINEAR, ADD; or the fused node
CHANNELS = 64


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def make_graph(blob, arm, x, profile=False):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
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
    """bytes node i reads from its arena sources plus the results it writes"""
    ins = [t for t in g.node_io(i)[0] if t >= 0 and g.in_arena(t)]
    outs = [t for t in g.node_outputs(i) if t >= 0]
    return sum(g.nbytes(t) for t in ins + outs)


def profile(blob, arm, x, scale):
    g = make_graph(blob, arm, x, profile=True)
    g.invoke()
    g.reset_profile()
    g.invoke()
    times = g.node_times_ms()
    total = sum(times)
    tail0 = g.num_nodes() - TAIL_NODES[arm]
    b, h, w, _ = x.shape
    flops = 2.0 * b * h * w * 3 * scale * scale * 9 * CHANNELS
    nodes = []
    for i in range(tail0, g.num_nodes()):
        nb = node_bytes(g, i)
        conv = i == tail0
        nodes.append({"node": i, "name": g.node_name(i), "ms": round(times[i], 4), "bytes": nb,
                      "GB_per_s": round(nb / (times[i] * 1e6), 1) if times[i] else None,
                      "TFLOP_per_s": round(flops / (times[i] * 1e9), 2) if conv and times[i] else None})
    all_nodes = [{"name": g.node_name(i), "ms": round(times[i], 4)} for i in range(g.num_nodes())]
    g.close()
    tail = sum(times[tail0:])
    body = sum(times[1:tail0])   # after the head node, up to the tail
    return {"step_ms": round(total, 4), "tail_ms": round(tail, 4), "tail_share": round(tail / total, 4),
            "body_ms": round(body, 4), "body_share": round(body / total, 4), "tail_flop": flops,
            "tail_nodes": nodes, "nodes": all_nodes}


def run_scale(a, scale):
    blob = zoo.binary_srnet(batch=1, seed=0, image=(a.height, a.width), scale=scale)
    x = np.random.default_rng(0).standard_normal((a.batch, a.height, a.width, 3), dtype=np.float32)
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
    f, u = outputs["fused"], outputs["unfused"]
    same = bool(f.shape == u.shape and np.array_equal(f.view(np.uint32), u.view(np.uint32)))
    out = {"scale": scale, "nodes": nodes, "identical_bits": same}
    for arm in ARMS:
        r = sorted(rates[arm])
        out[arm] = {"median": round(float(np.median(r)), 1), "min": round(r[0], 1), "max": round(r[-1], 1)}
    out["profile"] = {arm: profile(blob, arm, x, scale) for arm in ARMS}
    return out, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--height", type=int, default=180)
    ap.add_argument("--width", type=int, default=320)
    ap.add_argument("--scales", type=int, nargs="+", default=[2, 4])
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    out = gpu_info()
    out.update({"workload": "binary_srnet", "batch": a.batch, "image": [a.height, a.width], "input_type": "float32",
                "channels": CHANNELS, "blocks": 16, "runs": a.runs, "steps": a.steps, "unit": "images/s"})
    ok = True
    out["scales"] = []
    for scale in a.scales:
        res, same = run_scale(a, scale)
        out["scales"].append(res)
        ok = ok and same
    print(json.dumps(out), flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
