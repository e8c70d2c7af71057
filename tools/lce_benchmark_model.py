#!/usr/bin/env python
"""lce_benchmark_model -- command-line timing of a `.tflite` graph on the GPU path, with
the flags of the reference's benchmark tool (LCE/tflite/benchmark/lce_benchmark_tflite_model.cc:
41-71 adds --use_reference_bconv / --use_indirect_bgemm to TFLite's benchmark_model flags
--graph, --num_runs, --warmup_runs, --num_threads, --enable_op_profiling;
tensorflow/lite/tools/benchmark/benchmark_model.cc:57-66).

  python tools/lce_benchmark_model.py --graph=model.tflite --num_runs=50 --warmup_runs=5 \
         [--batch=256] [--enable_op_profiling=true] [--use_cuda_graph=true]
  python tools/lce_benchmark_model.py --zoo=quicknet --batch=256      # synthetic model
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _bool(v):
    return str(v).lower() in ("1", "true", "yes")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graph", default="")
    ap.add_argument("--zoo", default="", help="quicknet | quicknet_large | quicknet_small | birealnet18 | reactnet_a | realtobinarynet | "
                    "binarydensenet28 | binarydensenet37 | binarydensenet37_dilated | binarydensenet45 | meliusnet22 | "
                    "binaryalexnet | xnornet | dorefanet")
    ap.add_argument("--num_runs", type=int, default=50)
    ap.add_argument("--warmup_runs", type=int, default=5)
    ap.add_argument("--num_threads", type=int, default=1)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--use_reference_bconv", type=_bool, default=False)
    ap.add_argument("--use_indirect_bgemm", type=_bool, default=False)
    ap.add_argument("--enable_op_profiling", type=_bool, default=False)
    ap.add_argument("--use_cuda_graph", type=_bool, default=True)
    ap.add_argument("--fuse", type=_bool, default=True)
    a = ap.parse_args()
    from compute_engine_b200 import host as H, zoo
    if a.graph:
        blob = open(a.graph, "rb").read()
    elif a.zoo:
        blob = zoo.MODELS[a.zoo](batch=1, seed=0)
    else:
        ap.error("--graph or --zoo is required")
    t0 = time.perf_counter()
    # --use_reference_bconv / --use_indirect_bgemm pick the registration LceBconv2d resolves to,
    # as lce_benchmark_tflite_model.cc:41-71 does through RegisterLCECustomOps; --num_threads is
    # reported back but configures nothing (the device path has no CPU worker threads).
    g = H.HostGraph.from_tflite(blob, device_arena=True, use_reference_bconv=a.use_reference_bconv,
                                use_indirect_bgemm=a.use_indirect_bgemm)
    fused = g.fuse_all() if a.fuse else 0
    for t in g.inputs():
        shape = list(g.shape(t))
        shape[0] = a.batch
        g.resize_input(t, shape)
    g.allocate_tensors()
    init_ms = (time.perf_counter() - t0) * 1e3
    rng = np.random.default_rng(0)
    for t in g.inputs():                     # random inputs, like the reference's tool
        if np.issubdtype(g.dtype(t), np.floating):
            g.write(t, rng.standard_normal(g.shape(t)).astype(g.dtype(t)))
        else:
            g.write(t, rng.integers(-100, 100, g.shape(t)).astype(g.dtype(t)))
    g.enable_cuda_graph(a.use_cuda_graph and not a.enable_op_profiling)
    g.enable_profiling(a.enable_op_profiling)
    for _ in range(max(a.warmup_runs, 2)):
        g.invoke()
    g.synchronize()
    g.reset_profile()
    times = []
    for _ in range(a.num_runs):
        t1 = time.perf_counter()
        g.invoke()
        g.synchronize()
        times.append((time.perf_counter() - t1) * 1e3)
    registration = ("Register_BCONV_2D_REF" if a.use_reference_bconv else
                    "Register_BCONV_2D_OPT_INDIRECT_BGEMM" if a.use_indirect_bgemm else "Register_BCONV_2D")
    out = {"graph": a.graph or f"zoo:{a.zoo}", "batch": a.batch, "nodes": g.num_nodes(),
           "bconv_registration": registration, "num_threads": a.num_threads,
           "fused_nodes_removed": fused, "init_ms": round(init_ms, 2),
           "inference_ms": {"avg": round(float(np.mean(times)), 4),
                            "min": round(float(np.min(times)), 4),
                            "max": round(float(np.max(times)), 4),
                            "std": round(float(np.std(times)), 4)},
           "images_per_s": round(a.batch / (np.mean(times) * 1e-3), 1),
           "arena_MB": round(g.arena_bytes() / 1e6, 1)}
    if a.enable_op_profiling:
        per = {}
        for i, ms in enumerate(g.node_times_ms()):
            per[g.node_name(i)] = per.get(g.node_name(i), 0.0) + ms / a.num_runs
        out["op_profile_ms"] = {k: round(v, 4) for k, v in sorted(per.items(), key=lambda kv: -kv[1])}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
