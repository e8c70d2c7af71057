"""QuickNet segmentation with learned upsamplers on one GPU: the binary transposed convolutions with and
without their fusion into the b1 convolution, and the float and nearest-neighbour decoders for
reference.

  python tools/transpose_conv_bench.py [--batch 256] [--image 224] [--runs 5] [--steps 20] [--warmup 3]

Four arms on int8-input models (synthetic weights, compute_engine_b200/zoo.py quicknet_seg):
  fused     : upsample="binary_transpose", fuse_all() -- each stage one LceBconv2dTranspose+ADD+LceQuantize
  unfused   : upsample="binary_transpose", fuse_all() without fuse_binary_transpose_convs() -- each stage
              LceDequantize, TRANSPOSE_CONV, ADD and LceQuantize
  transpose : upsample="transpose" (a float TRANSPOSE_CONV 2x2 / stride 2 per stage), fuse_all()
  nearest   : the default decoder (CONV_2D 1x1 -> RESIZE_NEAREST_NEIGHBOR per stage), fuse_all()
Every graph replays as a CUDA graph with the images already in HBM. The arms alternate, `--runs` times
each, every run `--steps` steps; one JSON line gives each arm's median and range in images/s, the card's
name, power limit and max SM clock (read with nvidia-smi in the same run), whether the fused and unfused
arms give identical output bits at the timed batch, and from one profiled step of each arm (a separate
eager run): the decoder's share of the step and each upsampling node's time, bytes/s and op/s. Bytes
come from shapes (the arena tensors a node reads plus those it writes); ops are 2 M N K of the node's
GEMM view (a +-1 product counts as a multiply and an add). Needs a GPU; there is no CPU path.
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

ARMS = ("fused", "unfused", "transpose", "nearest")
UNFUSED_PASSES = ("fuse_binary_bases", "fuse_dense_blocks", "fuse_residual_blocks", "fuse_spatial_scales",
                  "fuse_float_glue", "fuse_upsample_merges", "fuse_resize_argmax", "fuse_subpixel_convs",
                  "fuse_grouped_conv_affine", "fuse_quantized_activations", "fuse_pooled_signs",
                  "fuse_channel_gates", "fuse_activation_chains", "fuse_residual_pairs")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def model(arm, batch, image):
    """The model at the timed batch: LceDequantize keeps its output's shape (the reference's Prepare
    checks it and does not resize), so the unfused binary graph cannot be resized to another batch."""
    up = {"fused": "binary_transpose", "unfused": "binary_transpose"}.get(arm, arm)
    return zoo.quicknet_seg(batch=batch, seed=0, image=image, input_type="int8", upsample=up)


def make_graph(arm, image, x, profile=False):
    g = H.HostGraph.from_tflite(model(arm, x.shape[0], image), device_arena=True)
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
    ins = [t for t in g.node_io(i)[0] if t >= 0 and g.in_arena(t)]
    outs = [t for t in g.node_outputs(i) if t >= 0]
    return sum(g.nbytes(t) for t in ins + outs)


def node_ops(g, i, name):
    """2 M N K of the node's GEMM view, or None for a node without one."""
    ins = g.node_io(i)[0]
    if name == "builtin:67":                      # TRANSPOSE_CONV: [shape, weights, x, bias]
        b, h, w, cin = g.shape(ins[2])
        cout, kh, kw, _ = g.shape(ins[1])
        return 2 * b * h * w * cin * cout * kh * kw
    if name.startswith("LceBconv2dTranspose"):    # [q, packed filter [s*s*C, 1, 1, Cin/32], ...]
        b, h, w, cw = g.shape(ins[0])
        return 2 * b * h * w * 32 * cw * g.shape(ins[1])[0]
    if name in ("builtin:3", "CONV_2D"):          # the nearest decoder's 1x1 CONV_2D
        b, h, w, cin = g.shape(ins[0])
        return 2 * b * h * w * cin * g.shape(ins[1])[0]
    return None


def is_upsampling(names, i):
    n = names[i]
    if n in ("builtin:67", "LceDequantize") or n.startswith(("LceBconv2dTranspose", "RESIZE_NEAREST")):
        return True
    # the nearest decoder's 1x1 CONV_2D, and the unfused stage's ADD and signs after its TRANSPOSE_CONV
    nxt = names[i + 1] if i + 1 < len(names) else ""
    prev = [names[k] for k in range(max(0, i - 2), i)]
    return (n == "builtin:3" and nxt.startswith("RESIZE_NEAREST")) or (
        n in ("builtin:0", "ADD+LceQuantize", "LceQuantize") and "builtin:67" in prev)


def profile(arm, image, x):
    g = make_graph(arm, image, x, profile=True)
    g.invoke()
    g.reset_profile()
    g.invoke()
    times = g.node_times_ms()
    names = [g.node_name(i) for i in range(g.num_nodes())]
    ups = [i for i in range(len(names)) if is_upsampling(names, i)]
    dec0, head0 = ups[0], len(names) - 2          # the head: the final CONV_2D and RESIZE_BILINEAR
    total = sum(times)
    nodes = []
    for i in ups:
        b, ops = node_bytes(g, i), node_ops(g, i, names[i])
        nodes.append({"node": i, "name": names[i], "ms": round(times[i], 4), "bytes": b,
                      "GB_per_s": round(b / (times[i] * 1e6), 1) if times[i] else None,
                      "TOP_per_s": round(ops / (times[i] * 1e9), 2) if ops and times[i] else None})
    g.close()
    return {"step_ms": round(total, 4), "decoder_share": round(sum(times[dec0:head0]) / total, 4),
            "upsampling_ms": round(sum(times[i] for i in ups), 4), "nodes": nodes}


def main():
    ap = argparse.ArgumentParser()
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
        g = make_graph(arm, a.image, x)
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
    same = bool(np.array_equal(outputs["fused"].view(np.uint8), outputs["unfused"].view(np.uint8)))
    out = dict(info)
    out.update({"workload": "quicknet_seg upsample", "batch": a.batch, "image": a.image, "input_type": "int8",
                "runs": a.runs, "steps": a.steps, "unit": "images/s", "nodes": nodes,
                "identical_binary_outputs": same})
    for arm in ARMS:
        r = sorted(rates[arm])
        out[arm] = {"median": round(float(np.median(r)), 1), "min": round(r[0], 1), "max": round(r[-1], 1)}
    out["profile"] = {arm: profile(arm, a.image, x) for arm in ARMS}
    print(json.dumps(out), flush=True)
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
