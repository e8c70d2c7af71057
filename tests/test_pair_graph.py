"""CPU: Graph::FuseResidualPairs, which merges two consecutive residual blocks into one
"LceBconv2d+ADD+LceBconv2d+ADD[+LceQuantize]" node (lce_b200_bconv2d_run_fused_pair), and the
pair kernel's build: it compiles for sm_90a without register spills."""
import collections
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from compute_engine_b200 import host as H
from compute_engine_b200 import zoo
from compute_engine_b200.tflite_writer import TFLiteModel, bconv2d_options

PAIR = "LceBconv2d+ADD+LceBconv2d+ADD"


def _fused(blob):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.fuse_residual_blocks()
    g.fuse_float_glue()
    g.fuse_activation_chains()
    return g


def _names(g):
    return [g.node_name(i) for i in range(g.num_nodes())]


@pytest.mark.parametrize("make,pairs", [(zoo.quicknet, 4), (zoo.quicknet_large, 7)])
def test_quicknet_pairs_its_64_and_128_channel_stages(make, pairs):
    """Stages 1 and 2 (C = 64, 128) pair up: QuickNet 2 + 2 pairs of its 4 + 4 blocks, QuickNetLarge
    3 + 4 of its 6 + 8. Stages 3 and 4 (C = 256, 512) keep two nodes per pair."""
    g = _fused(make(batch=1, image=224, seed=1))
    before = collections.Counter(_names(g))
    assert g.fuse_residual_pairs() == pairs
    names = collections.Counter(_names(g))
    assert names[PAIR + "+LceQuantize"] + names[PAIR] == pairs
    assert names[PAIR] == 2   # the last pair of each paired stage feeds the transition block
    assert sum(before.values()) - sum(names.values()) == pairs
    g.close()
    g = H.HostGraph.from_tflite(make(batch=1, image=224, seed=1), device_arena=True)
    g.fuse_all()                                    # the pair pass runs last
    assert collections.Counter(_names(g)) == names
    g.close()


@pytest.mark.parametrize("make", [zoo.birealnet18, zoo.reactnet_a])
def test_models_without_pairs_are_not_changed(make):
    g = _fused(make(batch=1, image=64, seed=2))
    before = _names(g)
    assert g.fuse_residual_pairs() == 0
    assert _names(g) == before
    g.close()


def _blocks(n=2, c=64, hw=14, extra_consumer=False, x1_output=False, pad_values=1, stride=(1, 1)):
    """x -> n residual blocks [LceQuantize -> LceBconv2d 3x3 -> ADD(shortcut)] -> out.
    A stride-2 block takes its shortcut from a graph input of its output's shape."""
    rng = np.random.default_rng(3)
    m = TFLiteModel()
    x = m.add_tensor("x", (1, hw, hw, c))
    inputs, outputs, sums = [x], [], []   # sums: (tensor, shape)
    for k in range(n):
        s = stride[k] if k < len(stride) else 1
        ohw = -(-hw // s)
        xq = m.add_tensor(f"xq{k}", (1, hw, hw, c // 32), np.int32)
        f = m.add_tensor(f"f{k}", None, np.int32,
                         data=rng.integers(-2**31, 2**31 - 1, (c, 3, 3, c // 32)).astype(np.int32))
        mul = m.add_tensor(f"mul{k}", None, np.float32, data=rng.uniform(0.1, 1, c))
        bias = m.add_tensor(f"bias{k}", None, np.float32, data=rng.uniform(-1, 1, c))
        y = m.add_tensor(f"y{k}", (1, ohw, ohw, c))
        o = m.add_tensor(f"s{k}", (1, ohw, ohw, c))
        m.add_op("LceQuantize", [x], [xq], custom_options=b"")
        m.add_op("LceBconv2d", [xq, f, mul, bias, -1], [y],
                 custom_options=bconv2d_options(c, (s, s), pad_values=pad_values, activation=1))
        short = x
        if s != 1:
            short = m.add_tensor(f"short{k}", (1, ohw, ohw, c))
            inputs.append(short)
        m.add_op("ADD", [y, short], [o])
        x, hw = o, ohw
        sums.append((o, (1, ohw, ohw, c)))
    if extra_consumer:
        r = m.add_tensor("relu", sums[0][1])
        m.add_op("RELU", [sums[0][0]], [r])
        outputs.append(r)
    if x1_output:
        outputs.append(sums[0][0])
    m.inputs, m.outputs = inputs, [x] + outputs
    return m.serialize()


def test_two_blocks_pair():
    g = _fused(_blocks())
    assert _names(g) == ["LceQuantize", "LceBconv2d+ADD+LceQuantize", "LceBconv2d+ADD"]
    assert g.fuse_residual_pairs() == 1
    assert _names(g) == ["LceQuantize", PAIR]
    ins, _ = g.node_io(1)
    assert len(ins) == 10
    g.close()


@pytest.mark.parametrize("variant", ["x1_has_another_consumer", "x1_is_a_graph_output", "zero_padding",
                                     "stride_2", "channels_not_a_multiple_of_64",
                                     "channels_beyond_the_kernel", "image_mostly_tile_padding"])
def test_pairing_leaves_the_graph_when_a_precondition_fails(variant):
    kw = {"x1_has_another_consumer": dict(extra_consumer=True),
          "x1_is_a_graph_output": dict(x1_output=True),
          "zero_padding": dict(pad_values=0),
          "stride_2": dict(stride=(1, 2, 1)),
          "channels_not_a_multiple_of_64": dict(c=96),
          "channels_beyond_the_kernel": dict(c=256),
          # 8 x 8 fills a third of a 14 x 14 tile: two blocks run faster than the pair kernel
          "image_mostly_tile_padding": dict(hw=8)}[variant]
    g = _fused(_blocks(**kw))
    before = _names(g)
    assert g.fuse_residual_pairs() == 0
    assert _names(g) == before
    g.close()


def test_pairing_follows_how_full_the_tiles_are():
    """Pairs where at least half of the tiles' pixels are the image's: 7 x 7 (one 14 x 14 tile at
    64 channels is a quarter full) stays, 7 x 7 at 128 channels (one 7 x 14 tile, half full) and
    22 x 22 (62 %) pair."""
    for hw, c, pairs in ((7, 64, 0), (7, 128, 1), (22, 64, 1), (16, 64, 0), (28, 128, 1)):
        g = _fused(_blocks(hw=hw, c=c))
        assert g.fuse_residual_pairs() == pairs, (hw, c)
        g.close()


def test_an_odd_run_pairs_all_but_its_last_block():
    g = _fused(_blocks(n=5))
    assert g.fuse_residual_pairs() == 2
    assert _names(g) == ["LceQuantize", PAIR + "+LceQuantize", PAIR + "+LceQuantize",
                         "LceBconv2d+ADD"]
    g.close()
    g = H.HostGraph.from_tflite(_blocks(n=5), device_arena=False)   # the host arena never pairs
    assert g.fuse_residual_pairs() == 0
    g.close()


def test_the_b1_switches_keep_blocks_unpaired(monkeypatch):
    for name in ("LCE_B200_BCONV_IMMA", "LCE_B200_BCONV_B1"):
        monkeypatch.setenv(name, "0")
        g = _fused(_blocks())
        assert g.fuse_residual_pairs() == 0
        g.close()
        monkeypatch.delenv(name)


def test_pair_kernel_compiles_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "pair.cu"
    src.write_text('#include "lce_b200_pair.cuh"\n'
                   "template __global__ void lce::bconv_pair_kernel<2>(const lce::PairParams);\n"
                   "template __global__ void lce::bconv_pair_kernel<4>(const lce::PairParams);\n")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xptxas=-v", "-cubin", "-I", os.path.join(repo, "include"),
                        "-I", os.path.join(repo, "compute_engine_b200", "csrc"), str(src),
                        "-o", str(tmp_path / "pair.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S*bconv_pair_kernel\S*)\n\s*(.*)", r.stderr)
    assert len(props) == 2, r.stderr
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)

