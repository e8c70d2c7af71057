"""The wiring of every fused graph, pinned node for node.

For each zoo model (and the variants below) and three arms -- the passes in fuse_all()'s order, each
pass alone on a fresh graph, and fuse_all()'s order with the stem and CONV_2D -> LceQuantize fusions
switched off -- tests/golden/fusion_nodes.json holds each pass's return value, the graph's tensor
and node counts and the SHA-256 of the final node list, written as compact JSON of [node name, inputs,
output 0, output 1 where the name says the node writes packed signs as its second output] per node.
The per-model tests check names, counts and a few nodes' tensors; this one fails when any pass
rewrites a node differently, wires one to another tensor, leaves the nodes in another order or
returns another count. To see which node moved, print _nodes() of the graph at both commits.

A pass that returned 0 alone is not recorded: the test then checks that it left the unfused graph's
node list and tensor count.

The passes run on a device-arena graph without touching a device until allocate_tensors(), so none
of this needs a GPU. Regenerate the file, after a change that is meant to alter a fused graph, with
    python tests/test_fusion_snapshot.py
"""
import hashlib
import json
import os
import sys

import pytest

if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from compute_engine_b200 import host as H
from compute_engine_b200 import zoo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fusion_nodes.json")
# HostGraph.fuse_all()'s order
PASSES = ("fuse_dense_blocks", "fuse_residual_blocks", "fuse_float_glue", "fuse_grouped_conv_affine",
          "fuse_quantized_activations", "fuse_pooled_signs", "fuse_channel_gates", "fuse_activation_chains",
          "fuse_residual_pairs")
SWITCHES = ("LCE_B200_FUSE_STEM", "LCE_B200_FUSE_CONV_QUANT")
ONE_PADDED = ("realtobinarynet", "binarydensenet28", "binarydensenet37", "binarydensenet37_dilated",
              "binarydensenet45", "meliusnet22", "binaryalexnet", "xnornet")


def _configs():
    c = {}
    for name, make in zoo.MODELS.items():
        c[f"{name}-224"] = (make, dict(batch=2, image=224))
        c[f"{name}-64-int8"] = (make, dict(batch=2, image=64, input_type="int8"))
    for name in ONE_PADDED:
        c[f"{name}-224-pad1"] = (zoo.MODELS[name], dict(batch=2, image=224, pad_values=1))
    c["meliusnet22-224-native-groups"] = (zoo.meliusnet, dict(batch=2, image=224, group_conv="native"))
    return c


CONFIGS = _configs()


def _nodes(g):
    out = []
    for i in range(g.num_nodes()):
        name = g.node_name(i)
        ins, outs = g.node_io(i)
        rec = [name, ins, outs[0]]
        # a fused node that ends in the sign writes the packed words as output 1, except the pooled
        # sign, whose only output they are
        if name.endswith("+LceQuantize") and name != "MAX_POOL_2D+MUL+ADD+LceQuantize":
            rec.append(H.lib().lce_host_node_output(g._g, i, 1))
        out.append(rec)
    return out


def _digest(nodes):
    return hashlib.sha256(json.dumps(nodes, separators=(",", ":")).encode()).hexdigest()


def _run(blob, passes):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    counts = [getattr(g, p)() for p in passes]
    nodes = _nodes(g)
    rec = {"removed": counts, "tensors": H.lib().lce_host_num_tensors(g._g), "nodes": len(nodes),
           "sha256": _digest(nodes)}
    g.close()
    return rec


def _switches(value):
    for s in SWITCHES:
        if value is None:
            os.environ.pop(s, None)
        else:
            os.environ[s] = value


def snapshot(key):
    make, kw = CONFIGS[key]
    blob = make(seed=1, **kw)
    saved = {s: os.environ.get(s) for s in SWITCHES}
    try:
        _switches(None)
        unfused = _run(blob, ())
        snap = {"all": _run(blob, PASSES), "alone": {}}
        for p in PASSES:
            rec = _run(blob, (p,))
            if rec["removed"] == [0]:
                assert rec == dict(unfused, removed=[0]), (key, p)
            else:
                snap["alone"][p] = rec
        _switches("0")
        snap["switched_off"] = _run(blob, PASSES)
    finally:
        _switches(None)
        os.environ.update({s: v for s, v in saved.items() if v is not None})
    return snap


def _dump(snaps):
    """One arm per line, so that a changed graph is a changed line."""
    parts = []
    for key, s in snaps.items():
        alone = ",\n".join(f'      "{p}": {json.dumps(r)}' for p, r in s["alone"].items())
        parts.append(f'  "{key}": {{\n    "all": {json.dumps(s["all"])},\n    "alone": {{\n{alone}\n    }},\n'
                     f'    "switched_off": {json.dumps(s["switched_off"])}\n  }}')
    return "{\n" + ",\n".join(parts) + "\n}\n"


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_golden_covers_every_configuration():
    assert sorted(_golden()) == sorted(CONFIGS)


@pytest.mark.parametrize("key", sorted(CONFIGS))
def test_fused_graph_matches_snapshot(key):
    want, got = _golden()[key], snapshot(key)
    assert got["all"] == want["all"], (key, "all")
    assert got["switched_off"] == want["switched_off"], (key, "switched_off")
    assert sorted(got["alone"]) == sorted(want["alone"]), key
    for p in got["alone"]:
        assert got["alone"][p] == want["alone"][p], (key, p)


def test_fuse_all_runs_the_passes_in_the_recorded_order():
    blob = zoo.MODELS["quicknet"](batch=2, image=64, seed=1, input_type="int8")
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    want = _golden()["quicknet-64-int8"]["all"]
    assert g.fuse_all() == sum(want["removed"]) and _digest(_nodes(g)) == want["sha256"]
    g.close()


if __name__ == "__main__":
    snaps = {key: snapshot(key) for key in sorted(CONFIGS)}
    text = _dump(snaps)
    assert json.loads(text) == snaps
    with open(GOLDEN, "w") as f:
        f.write(text)
    print(f"wrote {GOLDEN}: {len(text)} bytes, {len(CONFIGS)} configurations")
