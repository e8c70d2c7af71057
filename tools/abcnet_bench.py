"""ABC-Net throughput on one GPU, with and without the binary-bases fusion.

  python tools/abcnet_bench.py [--batch 256] [--image 224] [--bases 3,3 5,5] [--runs 5]
                               [--steps 10] [--warmup 3] [--check-batch 4]

For each (M, N), two arms on the same int8-input model (synthetic weights, compute_engine_b200/zoo.py
abcnet, one-padded):
  base   : fuse_all() without fuse_binary_bases() -- each of the M * N binary convolutions, the
           ADD chain, the BatchNorm and the shifted signs run node by node (what the other passes
           make of them)
  bases  : fuse_all()
Both graphs replay as CUDA graphs with the images already in HBM (the graph's compute, not the
host link). The arms alternate, `--runs` times each, every run `--steps` steps; one JSON line per
(M, N) gives each arm's median and range in images/s, the card's name, power limit and max SM
clock (read with nvidia-smi in the same run), per-node-name summed times of one profiled step of
each arm (a separate run), the ABC nodes' share of the bases arm's step, each fused node's
achieved bytes/s from its activation shapes (planes, shortcut and outputs; the weights stay in
L2), and whether both arms give identical output bits: at the timed batch with the arenas the
timed graphs use, and at `--check-batch` with every tensor kept (the unfused arm keeps every term
and partial sum, too large at the timed batch). Needs a GPU; there is no CPU path.
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

BASE_PASSES = ("fuse_dense_blocks", "fuse_residual_blocks", "fuse_spatial_scales", "fuse_float_glue",
               "fuse_grouped_conv_affine",
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
    if arm == "bases":
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


def fused_bytes(g, n_planes):
    """activation bytes each bases / planes node moves per step, from its tensors' shapes"""
    out = {}
    for i in range(g.num_nodes()):
        name = g.node_name(i)
        ins = g.node_io(i)[0]
        if name == "ADD+LceQuantize":
            reads, n_out = [ins[0]], n_planes
        elif name.startswith("LceBconv2dBases"):
            reads = ins[:n_planes] + ([ins[-1]] if ins[-1] >= 0 else [])
            n_out = 1 if name == "LceBconv2dBases" else n_planes + (1 if ins[-1] >= 0 else 0)
        else:
            continue
        writes = [H.lib().lce_host_node_output(g._g, i, k) for k in range(n_out)]
        out[i] = sum(g.nbytes(t) for t in reads + writes)
    return out


def profile(blob, arm, x, n_planes):
    """per-node-name device time (ms) of one eager step after a warm-up step, the ABC nodes' share,
    and each fused node's achieved bytes/s"""
    g = make_graph(blob, arm, x, profile=True)
    g.invoke()
    g.reset_profile()
    g.invoke()
    times = g.node_times_ms()
    by_name = collections.defaultdict(float)
    for i, ms in enumerate(times):
        by_name[g.node_name(i)] += ms
    total = sum(times)
    abc = sum(ms for i, ms in enumerate(times) if g.node_name(i).startswith("LceBconv2dBases")
              or g.node_name(i) == "ADD+LceQuantize")
    rates = [{"node": i, "name": g.node_name(i), "ms": round(times[i], 4), "bytes": b,
              "GB_per_s": round(b / (times[i] * 1e6), 1)} for i, b in fused_bytes(g, n_planes).items()]
    g.close()
    return ({k: round(v, 4) for k, v in sorted(by_name.items(), key=lambda kv: -kv[1])},
            round(abc / total, 4) if total else 0.0, rates)


def same_bits(a, b):
    return bool(np.array_equal(a.view(np.uint8), b.view(np.uint8)))


def bench(a, info, bases):
    blob = zoo.abcnet(batch=1, seed=0, image=a.image, input_type="int8", bases=bases)
    rng = np.random.default_rng(0)
    x = rng.integers(-128, 128, (a.batch, a.image, a.image, 3)).astype(np.int8)
    arms = ("base", "bases")
    kept = {}
    xc = x[:a.check_batch]
    for arm in arms:
        g = make_graph(blob, arm, xc, preserve=True)
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
    out = dict(info)
    out.update({
        "workload": "abcnet", "m_n": list(bases), "batch": a.batch, "image": a.image, "input_type": "int8",
        "runs": a.runs, "steps": a.steps, "unit": "images/s", "nodes": nodes,
        "identical_outputs_reused_arena": same_bits(outputs["base"], outputs["bases"]),
        "identical_outputs_all_kept": same_bits(kept["base"], kept["bases"]), "check_batch": a.check_batch,
    })
    for arm in arms:
        r = sorted(rates[arm])
        out[arm] = {"median": round(float(np.median(r)), 1), "min": round(r[0], 1), "max": round(r[-1], 1)}
    out["profile_ms_per_step"] = {}
    for arm in arms:
        by_name, share, node_rates = profile(blob, arm, x, bases[1])
        out["profile_ms_per_step"][arm] = by_name
        if arm == "bases":
            out["abc_share_of_step"] = share
            out["fused_node_rates"] = node_rates
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--image", type=int, default=224)
    ap.add_argument("--bases", nargs="+", default=["3,3", "5,5"], help="M,N pairs")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--check-batch", type=int, default=4)
    a = ap.parse_args()
    info = gpu_info()
    ok = True
    for mn in a.bases:
        m, n = (int(v) for v in mn.split(","))
        out = bench(a, info, (m, n))
        print(json.dumps(out), flush=True)
        ok = ok and out["identical_outputs_reused_arena"] and out["identical_outputs_all_kept"]
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
