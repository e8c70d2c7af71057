"""Binary MobileNet throughput on one GPU: grouped binary convolutions native vs split, with
ReActNet-A as the ungrouped reference.

  python tools/binary_mobilenet_bench.py [--batch 256] [--image 224] [--group-channels 32]
                                         [--runs 5] [--steps 10] [--warmup 3] [--check-batch 4]

Three arms on int8-input models (synthetic weights, compute_engine_b200/zoo.py), each with
fuse_all():
  native   : binary_mobilenet(group_conv="native"), each grouped 3x3 layer one grouped LceBconv2d
             (the b1 mma.sync kernel with the block tail in its epilogue)
  split    : binary_mobilenet(group_conv="split"), SPLIT -> one LceBconv2d per group -> CONCATENATION
  reactnet : reactnet_a, the same backbone with ungrouped 3x3 layers
All replay as CUDA graphs with the images already in HBM. The arms alternate, `--runs` times
each, every run `--steps` steps. One JSON line gives each arm's median and range in images/s, the
card's name, power limit and max SM clock (read with nvidia-smi in the same run), and, from one
profiled eager step per arm (a separate run): each grouped node's time, its bytes/s (packed input,
shortcut, float and packed outputs, from the tensor shapes; the weights stay in L2) and binary
ops/s (2 * pixels * C_out * taps * C_in / groups). The same grouped layers are also profiled with
LCE_B200_BCONV_IMMA=0 and _TC=0, unfused on the XOR + POPC kernel. Output bits of native and split
are compared at the timed batch with the arenas the timed graphs use, and at `--check-batch` with
every tensor kept. Needs a GPU; there is no CPU path.
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


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def make_graph(blob, x, fuse=True, profile=False, preserve=False):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    if fuse:
        g.fuse_all()
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


def grouped_nodes(g):
    """{node: (bytes, binary ops)} of the grouped LceBconv2d nodes, from their tensors' shapes"""
    out = {}
    for i in range(g.num_nodes()):
        if not g.node_name(i).startswith("LceBconv2d"):
            continue
        ins, outs = g.node_io(i)
        xs, fs = g.shape(ins[0]), g.shape(ins[1])
        if xs[3] == fs[3]:
            continue
        groups = xs[3] // fs[3]
        ys = g.shape(outs[0])
        pixels = ys[0] * ys[1] * ys[2]
        ops = 2 * pixels * fs[0] * fs[1] * fs[2] * fs[3] * 32
        reads = [ins[0]] + ([ins[5]] if len(ins) > 5 and ins[5] >= 0 else [])
        nbytes = sum(g.nbytes(t) for t in reads) + sum(g.nbytes(t) for t in outs if t >= 0)
        out[i] = (nbytes, ops, groups)
    return out


def profile_grouped(blob, x, fuse=True, env=None):
    saved = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        g = make_graph(blob, x, fuse=fuse, profile=True)
        g.invoke()
        g.reset_profile()
        g.invoke()
        times = g.node_times_ms()
        rows = [{"node": i, "name": g.node_name(i), "groups": gr, "ms": round(times[i], 4), "bytes": b,
                 "GB_per_s": round(b / (times[i] * 1e6), 1), "binary_Tops_per_s": round(ops / (times[i] * 1e9), 2)}
                for i, (b, ops, gr) in grouped_nodes(g).items()]
        total = round(sum(times), 4)
        g.close()
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    return {"step_ms": total, "grouped_ms": round(sum(r["ms"] for r in rows), 4), "nodes": rows}


def same_bits(a, b):
    return bool(np.array_equal(a.view(np.uint8), b.view(np.uint8)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--image", type=int, default=224)
    ap.add_argument("--group-channels", type=int, default=32)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--check-batch", type=int, default=4)
    a = ap.parse_args()
    info = gpu_info()
    blobs = {
        "native": zoo.binary_mobilenet(batch=1, image=a.image, input_type="int8",
                                       group_channels=a.group_channels, group_conv="native"),
        "split": zoo.binary_mobilenet(batch=1, image=a.image, input_type="int8",
                                      group_channels=a.group_channels, group_conv="split"),
        "reactnet": zoo.reactnet_a(batch=1, image=a.image, input_type="int8"),
    }
    x = np.random.default_rng(0).integers(-128, 128, (a.batch, a.image, a.image, 3)).astype(np.int8)
    kept = {}
    for arm in ("native", "split"):
        g = make_graph(blobs[arm], x[:a.check_batch], preserve=True)
        g.invoke()
        kept[arm] = g.read(g.outputs()[0])
        g.close()
    graphs, outputs = {}, {}
    for arm, blob in blobs.items():
        g = make_graph(blob, x)
        g.invoke()                                   # eager: plans are built
        outputs[arm] = g.read(g.outputs()[0])
        g.enable_cuda_graph(True)
        for _ in range(a.warmup + 2):                # the first two replays capture the graph
            g.invoke()
        graphs[arm] = g
    rates = {arm: [] for arm in graphs}
    for _ in range(a.runs):
        for arm, g in graphs.items():
            rates[arm].append(images_per_s(g, a.batch, a.steps))
    nodes = {arm: g.num_nodes() for arm, g in graphs.items()}
    for g in graphs.values():
        g.close()
    out = dict(info)
    out.update({
        "workload": "binary_mobilenet", "group_channels": a.group_channels, "batch": a.batch,
        "image": a.image, "input_type": "int8", "runs": a.runs, "steps": a.steps, "unit": "images/s",
        "nodes": nodes,
        "identical_outputs_reused_arena": same_bits(outputs["native"], outputs["split"]),
        "identical_outputs_all_kept": same_bits(kept["native"], kept["split"]), "check_batch": a.check_batch,
    })
    for arm, r in rates.items():
        r = sorted(r)
        out[arm] = {"median": round(float(np.median(r)), 1), "min": round(r[0], 1), "max": round(r[-1], 1)}
    out["grouped_profile"] = {
        "native_fused_mma": profile_grouped(blobs["native"], x),
        "native_unfused_xor_popc": profile_grouped(
            blobs["native"], x, fuse=False, env={"LCE_B200_BCONV_IMMA": "0", "LCE_B200_BCONV_TC": "0"}),
    }
    print(json.dumps(out), flush=True)
    return 0 if out["identical_outputs_reused_arena"] and out["identical_outputs_all_kept"] else 1


if __name__ == "__main__":
    sys.exit(main())
