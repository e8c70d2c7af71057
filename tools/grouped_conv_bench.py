"""MeliusNet22 throughput on one GPU, its stem's grouped convolutions as the split form against one
grouped CONV_2D each.

  python tools/grouped_conv_bench.py [--batch 256] [--image 224] [--runs 5] [--steps 20] [--warmup 3]

Two int8-input models from compute_engine_b200/zoo.py with the same weights, both with fuse_all():
  split  : meliusnet(group_conv="split"), larq-zoo's form: SPLIT -> one CONV_2D per group ->
           CONCATENATION -> MUL -> ADD(RELU) for each of the stem's two grouped convolutions
  native : meliusnet(group_conv="native"): one grouped CONV_2D each, which fuse_all() turns into a
           CONV_2D+MUL+ADD node (lce_b200_f32_grouped_conv2d with the BatchNorm in its epilogue)
Both graphs replay as CUDA graphs with the images already in HBM. The arms alternate, `--runs` times
each; the JSON line gives each arm's median and range in images/s, the card's name, power limit and
max SM clock (read with nvidia-smi in the same run), per-node times of one profiled eager step of
each arm (a separate run) for the stem (every node before the first MAX_POOL_2D) and the step, each
CONV_2D+MUL+ADD node's time with its bytes (the map it reads and the map it writes) and FLOPs (2 per
multiply-add) from shapes and the achieved rates, beside the data sheet's 3.35 TB/s of HBM3 and
67 TFLOP/s of FP32 (data-sheet figures, not measurements), and whether the two arms' outputs are
identical bit for bit on the same seeded input. Needs a GPU; there is no CPU path.
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

GROUPED = "CONV_2D+MUL+ADD"
HBM_DATA_SHEET_GB_PER_S = 3350.0      # NVIDIA's H100 SXM data sheet
FP32_DATA_SHEET_TFLOP_S = 67.0


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def make_graph(blob, x, profile=False):
    """the graph with fuse_all(), allocated for x's shape, with x written to its input"""
    g = H.HostGraph.from_tflite(blob, device_arena=True)
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


def profile(blob, x):
    """one eager step after one warm-up step: [(node name, ms)] in graph order, the index of the first
    MAX_POOL_2D, and each grouped node's time, bytes, FLOPs and rates"""
    g = make_graph(blob, x, profile=True)
    g.invoke()
    g.reset_profile()
    g.invoke()
    nodes, grouped = [], []
    for i, ms in enumerate(g.node_times_ms()):
        name = g.node_name(i)
        nodes.append((name, ms))
        if name == GROUPED:
            ins, outs = g.node_io(i)
            b, oh, ow, cout = g.shape(outs[0])
            _, kh, kw, cin_g = g.shape(ins[1])
            nbytes = g.nbytes(ins[0]) + g.nbytes(outs[0])
            flops = 2 * b * oh * ow * cout * kh * kw * cin_g
            grouped.append({"in": list(g.shape(ins[0])), "filter": list(g.shape(ins[1])), "out": [b, oh, ow, cout],
                            "ms": round(ms, 4), "bytes": nbytes, "flops": flops,
                            "gb_per_s": round(nbytes / (ms * 1e6), 1) if ms else None,
                            "tflop_per_s": round(flops / (ms * 1e9), 2) if ms else None})
    g.close()
    pool = next(i for i, (name, _) in enumerate(nodes) if name.startswith("builtin:17"))
    return nodes, pool, grouped


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--image", type=int, default=224)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if H.device_count() < 1:
        print("grouped_conv_bench: no CUDA device; nothing is measured without one", file=sys.stderr)
        return 2
    info = gpu_info()
    arms = ("split", "native")
    blobs = {arm: zoo.meliusnet(batch=1, seed=0, image=a.image, input_type="int8", group_conv=arm) for arm in arms}
    x = np.random.default_rng(0).integers(-128, 128, (a.batch, a.image, a.image, 3)).astype(np.int8)
    graphs, outputs = {}, {}
    for arm in arms:
        g = make_graph(blobs[arm], x)
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
        "workload": "meliusnet22", "batch": a.batch, "image": a.image, "input_type": "int8", "runs": a.runs,
        "steps": a.steps, "unit": "images/s", "nodes": nodes,
        "outputs_bit_identical": bool(np.array_equal(outputs["split"].view(np.uint8), outputs["native"].view(np.uint8))),
        "hbm_data_sheet_gb_per_s": HBM_DATA_SHEET_GB_PER_S, "fp32_data_sheet_tflop_per_s": FP32_DATA_SHEET_TFLOP_S,
    })
    for arm in arms:
        r = sorted(rates[arm])
        out[arm] = {"median": round(float(np.median(r)), 1), "min": round(r[0], 1), "max": round(r[-1], 1)}
        prof, pool, grouped = profile(blobs[arm], x)
        total = sum(ms for _, ms in prof)
        stem = sum(ms for _, ms in prof[:pool])
        out[arm].update({
            "profiled_step_ms": round(total, 4), "stem_ms": round(stem, 4),
            "stem_share": round(stem / total, 3) if total else None,
            "stem_nodes_ms": [[name, round(ms, 4)] for name, ms in prof[:pool]],
        })
        if arm == "native":
            for n in grouped:
                n["share_of_data_sheet_hbm"] = round(n["gb_per_s"] / HBM_DATA_SHEET_GB_PER_S, 3) if n["gb_per_s"] else None
            out["grouped_nodes"] = grouped
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())
