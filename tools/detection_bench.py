"""QuickNet SSD throughput on one GPU, with TFLite_Detection_PostProcess in fast and regular mode against
the graph without post-processing.

  python tools/detection_bench.py [--batch 256] [--image 224] [--runs 5] [--steps 20] [--warmup 3]

Three arms on int8-input models (synthetic weights, compute_engine_b200/zoo.py quicknet_ssd), all
fuse_all()ed:
  raw     : postprocess=False -- the box encodings [B, N, 4] and class scores [B, N, 21] are the outputs,
            what a user without the op copies to the host to run NMS there
  fast    : the op with use_regular_nms=False (the export default)
  regular : the op with use_regular_nms=True
Every graph replays as a CUDA graph with the images already in HBM. The arms alternate, `--runs` times
each, every run `--steps` steps; one JSON line gives each arm's median and range in images/s, the card's
name, power limit and max SM clock (read with nvidia-smi in the same run), and from one profiled step of
each post-processing arm (a separate eager run): the op's time, its share of the step and its bytes/s.
Its bytes come from shapes: box encodings and scores read once, the four outputs written. Needs a GPU;
there is no CPU path.
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

OP = "TFLite_Detection_PostProcess"
ARMS = {"raw": dict(postprocess=False), "fast": dict(use_regular_nms=False), "regular": dict(use_regular_nms=True)}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def make_graph(blob, x, profile=False):
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
    g = make_graph(blob, x, profile=True)
    g.invoke()
    g.reset_profile()
    g.invoke()
    times = g.node_times_ms()
    i = [g.node_name(k) for k in range(g.num_nodes())].index(OP)
    ins = [t for t in g.node_io(i)[0][:2]]
    b = sum(g.nbytes(t) for t in ins + list(g.node_outputs(i)))
    total = sum(times)
    g.close()
    return {"step_ms": round(total, 4), "op_ms": round(times[i], 4), "op_share": round(times[i] / total, 4),
            "op_bytes": b, "op_GB_per_s": round(b / (times[i] * 1e6), 1) if times[i] else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--image", type=int, default=224)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    info = gpu_info()
    blobs = {arm: zoo.quicknet_ssd(batch=1, seed=0, image=a.image, input_type="int8", **kw)
             for arm, kw in ARMS.items()}
    x = np.random.default_rng(0).integers(-128, 128, (a.batch, a.image, a.image, 3)).astype(np.int8)
    graphs, detections = {}, {}
    for arm, blob in blobs.items():
        g = make_graph(blob, x)
        g.invoke()                                   # eager: plans are built
        if arm != "raw":
            detections[arm] = float(g.read(g.outputs()[3]).mean())
        g.enable_cuda_graph(True)
        for _ in range(a.warmup + 2):                # the first two replays capture the graph
            g.invoke()
        graphs[arm] = g
    rates = {arm: [] for arm in ARMS}
    for _ in range(a.runs):
        for arm in ARMS:
            rates[arm].append(images_per_s(graphs[arm], a.batch, a.steps))
    for g in graphs.values():
        g.close()
    out = dict(info)
    out.update({"workload": "quicknet_ssd", "batch": a.batch, "image": a.image, "input_type": "int8",
                "runs": a.runs, "steps": a.steps, "unit": "images/s", "mean_num_detections": detections})
    for arm in ARMS:
        r = sorted(rates[arm])
        out[arm] = {"median": round(float(np.median(r)), 1), "min": round(r[0], 1), "max": round(r[-1], 1)}
    out["profile"] = {arm: profile(blobs[arm], x) for arm in ("fast", "regular")}
    print(json.dumps(out), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
