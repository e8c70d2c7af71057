"""QuickNetSmall throughput on one GPU, with and without its fused stem and 32-channel pairs.

  python tools/quicknet_small_bench.py [--batch 256] [--image 224] [--runs 5] [--steps 20] [--warmup 3]

Two arms on the same int8-input model (synthetic weights, compute_engine_b200/zoo.py):
  base  : LCE_B200_FUSE_STEM=0 and fuse_all() without fuse_residual_pairs() -- the stem runs as
          DEQUANTIZE, CONV_2D 3x3/s2 3 -> 8 and DEPTHWISE_CONV_2D, and every residual block as its
          own LceBconv2d+ADD[+LceQuantize] node
  fused : fuse_all() -- one stem node, and the 56x56x32 and 28x28x64 sections' blocks in pairs
Both graphs replay as CUDA graphs with the images already in HBM (the graph's compute, not the
host link). The arms alternate, `--runs` times each; the JSON line gives each arm's median and
range in images/s, the card's name, power limit and max SM clock (read with nvidia-smi in the same
run), per-node-name summed times of one profiled step of each arm, the stem's time and share
(the nodes before the first CONV_2D+LceQuantize), the 32-channel section's time and share (its
binary-convolution nodes), and whether both arms give identical output bits on the same seeded
input: with every tensor kept (no arena reuse) and with the arenas the timed graphs use. Exits 1
when the outputs differ. Needs a GPU; there is no CPU path.
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

STEM_END = "CONV_2D+LceQuantize"   # the 1x1 8 -> 32 convolution after the stem


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def make_graph(blob, arm, x, profile=False, preserve=False):
    """the arm's graph, allocated for x's shape, with x written to its input"""
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    if arm == "fused":
        g.fuse_all()
    else:
        os.environ["LCE_B200_FUSE_STEM"] = "0"     # read while fuse_float_glue() runs
        try:
            g.fuse_dense_blocks()
            g.fuse_residual_blocks()
            g.fuse_float_glue()
            g.fuse_pooled_signs()
            g.fuse_channel_gates()
            g.fuse_activation_chains()
        finally:
            del os.environ["LCE_B200_FUSE_STEM"]
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
    """per-node-name device time (ms) of one eager step after one warm-up step, the stem's nodes
    and time, and the 32-channel section's binary-convolution nodes and time"""
    g = make_graph(blob, arm, x, profile=True)
    g.invoke()
    g.reset_profile()
    g.invoke()
    by_name = collections.defaultdict(float)
    stem, stem_ms, sec, sec_ms = [], 0.0, [], 0.0
    in_stem = True
    for i, ms in enumerate(g.node_times_ms()):
        name = g.node_name(i)
        by_name[name] += ms
        if name == STEM_END:
            in_stem = False
        if in_stem:
            stem.append(name)
            stem_ms += ms
        _, outs = g.node_io(i)
        if name.startswith("LceBconv2d") and g.shape(outs[0])[-1] == 32:
            sec.append(name)
            sec_ms += ms
    g.close()
    by_name = {k: round(v, 4) for k, v in sorted(by_name.items(), key=lambda kv: -kv[1])}
    return by_name, {"stem_nodes": stem, "stem_ms": round(stem_ms, 4),
                     "section32_nodes": sec, "section32_ms": round(sec_ms, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--image", type=int, default=224)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    info = gpu_info()
    blob = zoo.quicknet_small(batch=1, seed=0, image=a.image, input_type="int8")
    x = np.random.default_rng(0).integers(-128, 128, (a.batch, a.image, a.image, 3)).astype(np.int8)
    arms = ("base", "fused")
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
    prof, parts = {}, {}
    for arm in arms:
        prof[arm], parts[arm] = profile(blob, arm, x)
    out = dict(info)
    out.update({
        "workload": "quicknet_small", "batch": a.batch, "image": a.image, "input_type": "int8",
        "runs": a.runs, "steps": a.steps, "unit": "images/s", "nodes": nodes,
        "identical_outputs": bool(np.array_equal(kept["base"].view(np.uint8), kept["fused"].view(np.uint8))),
        "identical_outputs_reused_arena": bool(np.array_equal(outputs["base"].view(np.uint8),
                                                              outputs["fused"].view(np.uint8))),
    })
    for arm in arms:
        r = sorted(rates[arm])
        out[arm] = {"median": round(float(np.median(r)), 1), "min": round(r[0], 1), "max": round(r[-1], 1)}
        total = sum(prof[arm].values())
        p = parts[arm]
        out[arm].update(p)
        out[arm]["step_ms"] = round(total, 4)
        out[arm]["stem_share"] = round(p["stem_ms"] / total, 3) if total else None
        out[arm]["section32_share"] = round(p["section32_ms"] / total, 3) if total else None
    out["profile_ms_per_step"] = prof
    print(json.dumps(out))
    return 0 if out["identical_outputs"] and out["identical_outputs_reused_arena"] else 1


if __name__ == "__main__":
    sys.exit(main())
