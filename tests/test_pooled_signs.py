"""BinaryAlexNet and XNOR-Net: the zoo models, the pooled BatchNorm and sign in one pass over the
float map (lce_b200_f32_maxpool_affine_sign) and the graph fusion that uses it
(Graph::FusePooledSigns).

CPU: each model's op, channel, shape and threshold counts, a CPU reference run, both readers, host
prepare and resize, the fused node list and each refused precondition, the other models' node lists
and bytes, and the new kernel compiled without spills. GPU: the kernel bit-exact against numpy
float32 and against the device's own MAX_POOL_2D -> MUL -> ADD -> LceQuantize kernels, both models
op by op, fused vs unfused under eager runs and CUDA-graph replay, the bitpacked layers on mma.sync,
and Interpreter.predict across batch resizes."""
import collections
import hashlib
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import lce_testlib as L
import tflite_ref as R
from compute_engine_b200 import host as H
from compute_engine_b200 import zoo
from compute_engine_b200.tflite_writer import TFLiteModel

POOLED = "MAX_POOL_2D+MUL+ADD+LceQuantize"
MODELS = ("binaryalexnet", "xnornet")
# sha256 of the ten earlier models' bytes at the commit before these two were added
OTHER_HASHES = {
    ("quicknet", 224): "80c00a45aea6e3ba794a0ac5a120f32f08384617492d3bc543cef8d83d1af335",
    ("quicknet", 64): "024123bcc04f5e52f563f836878ce7e64bf0e2d1dd31b6841d91d30b0e964b56",
    ("quicknet_large", 224): "ae386c9d6e07d995bc93739c6ecdcf1ab957c83ac8fa07bc5cc66c86d824a6e2",
    ("quicknet_large", 64): "f62eefd6554e1517ce4a3adabd83d8bfa055e7e34c43a5ac9fddd359a3862ac2",
    ("birealnet18", 224): "69b00efc25be1c89fd630ce5bc79d9f55f2076d93aa0014540d88a54bd717e1e",
    ("birealnet18", 64): "d2817ee2a793f1ce2f048e2396023ea2eed7e4dd331b171bceeceb562f4b5376",
    ("reactnet_a", 224): "37dd82f28895b77a623313d33f1ecf6364e53fffc5ab7445d8e848df8fab2085",
    ("reactnet_a", 64): "9f30ae372234f05158fa5fd25836d415dc23b78d412f291837cdc7b6903c90e5",
    ("realtobinarynet", 224): "d867acd75a420cca207684b4a48e71924f8ea98c3ccec5cd0a44016de002048f",
    ("realtobinarynet", 64): "5dbf6262d7d84cd91a1cce3119e1985242c10de65b35c7d2d8959dcb1034dcd4",
    ("binarydensenet28", 224): "fcb1f3e89ef1bd23fc6b751d23f9441f2a73dfe383e58beb7d595e61b5b85762",
    ("binarydensenet28", 64): "7042a35c340ad516c49ef7b9845d7af9ebb9c7f8e9796a52d1d458b8b36c1e28",
    ("binarydensenet37", 224): "f8d5bc67f8d50711afc2ae4fe3eb50b182937a849793927657bb4d15a5e118b9",
    ("binarydensenet37", 64): "b5bedcb32ab2f7f2965f53e597a1b8c31a2c63480f42d2eb228a76b9cba87bb3",
    ("binarydensenet37_dilated", 224): "1feab16cddee572d8fd747be7913765858bde31fc97731180a6cf43ad279ee1d",
    ("binarydensenet37_dilated", 64): "76bde634d67060324c82ae6daae8ac2d2af8c1a0eb6eb3a60411e66df562e156",
    ("binarydensenet45", 224): "f73b99c0b8ea8f7ff1d14feccb2c4cae89022041bd79d676bd08502e0c091e15",
    ("binarydensenet45", 64): "7ac5fdfc1c9253821f8ab3d3128f201aa0b260022b047d114e0a818e7d19d37a",
    ("meliusnet22", 224): "f2fe2d5101d56c090022dc7b0198dfb6f346959ebad5825908d033a18301b176",
    ("meliusnet22", 64): "e788a9d4fc97bbf9db34023f80f6b1a123d1fd1c6fa1e725f8168248bbfa566d",
}
OTHERS = sorted({name for name, _ in OTHER_HASHES})


# ------------------------------ CPU reference ------------------------------ #
def _run_op(model, op, vals):
    """One op on the CPU through tflite_ref. A binary convolution with bitpacked output follows the
    reference kernel's zero padding (the only one bconv2d.cc admits for it), every other one the
    optimised kernels', as the graph host's default registration does."""
    t = model["tensors"]
    act = [i for i in op["inputs"] if i >= 0 and t[i]["data"] is None]
    sub = {"tensors": t, "ops": [op], "inputs": act, "outputs": [op["outputs"][0]]}
    bitpacked = op["custom"] == "LceBconv2d" and t[op["outputs"][0]]["dtype"] == np.int32
    return R.run(sub, [vals[i] for i in act], bconv_kind=0 if bitpacked else 1)[0][0]


def _run_model(model, inputs):
    vals = dict(zip(model["inputs"], inputs))
    for op in model["ops"]:
        vals[op["outputs"][0]] = _run_op(model, op, vals)
    return [vals[i] for i in model["outputs"]]


def _bconvs(m):
    return [o for o in m["ops"] if o["code"] == 32 and o["custom"] == "LceBconv2d"]


# ----------------------------------- CPU ----------------------------------- #
# model: (stem channels, [(LceBconv2d C_in, C_out, filter, bitpacked)], pooled maps (H, C))
SPECS = {
    "binaryalexnet": (64, [(64, 192, 5, False), (192, 384, 3, True), (384, 384, 3, True),
                           (384, 256, 3, False), (256, 4096, 6, True), (4096, 4096, 1, True),
                           (4096, 1000, 1, False)], [(27, 64), (13, 192), (6, 256)]),
    "xnornet": (96, [(96, 256, 5, False), (256, 384, 3, True), (384, 384, 3, True),
                     (384, 256, 3, False), (256, 4096, 6, True), (4096, 4096, 1, False)],
                [(27, 96), (13, 256), (6, 256)]),
}


@pytest.mark.parametrize("name", MODELS)
def test_op_channel_shape_and_threshold_counts(name):
    m = R.parse(zoo.MODELS[name](batch=1, image=224, seed=1))
    t = m["tensors"]
    stem, convs, pooled = SPECS[name]
    kinds = collections.Counter((o["code"], o["custom"]) for o in m["ops"])
    want = {(3, ""): 1, (17, ""): 3, (18, ""): 3, (0, ""): 3, (32, "LceQuantize"): 3,
            (32, "LceBconv2d"): len(convs), (22, ""): 1, (25, ""): 1}
    if name == "xnornet":
        want[(9, "")] = 1
    assert dict(kinds) == want
    assert t[m["ops"][0]["outputs"][0]]["shape"] == (1, 56, 56, stem)
    if name == "binaryalexnet":   # +-1 stem weights, no bias
        w = t[m["ops"][0]["inputs"][1]]["data"]
        assert set(np.unique(w)) == {-1.0, 1.0} and m["ops"][0]["inputs"][2] == -1
    for op, (cin, cout, k, bitpacked) in zip(_bconvs(m), convs):
        a = R._flex_ints(op["custom_options"])
        filt, out = t[op["inputs"][1]]["data"], t[op["outputs"][0]]
        assert a["channels_in"] == cin and filt.shape == (cout, k, k, L.cdiv(cin, 32)), (cin, cout)
        assert a["padding"] == (0 if k in (3, 5) else 1)
        if bitpacked:
            assert out["dtype"] == np.int32 and out["shape"][3] == L.cdiv(cout, 32)
            assert op["inputs"][2] == op["inputs"][3] == -1
            thr = t[op["inputs"][4]]["data"]
            kk = k * k * cin
            assert thr.dtype == np.int32 and thr.shape == (cout,)
            assert abs(thr.mean() - kk / 2) < 0.25 * np.sqrt(kk) and 0 < thr.min() and thr.max() < kk
        else:
            assert out["dtype"] == np.float32 and out["shape"][3] == cout and op["inputs"][4] == -1
    assert sum(t[o["outputs"][0]]["dtype"] == np.int32 for o in _bconvs(m)) == (4 if name == "binaryalexnet" else 3)
    pools = [o for o in m["ops"] if o["code"] == 17]
    assert [t[p["outputs"][0]]["shape"][1:] for p in pools] == [(h, h, c) for h, c in pooled]
    for p in pools:   # each pool feeds only its BatchNorm's MUL, then ADD, then LceQuantize
        y = p["outputs"][0]
        chain = [o for o in m["ops"] if y in o["inputs"]]
        assert [o["code"] for o in chain] == [18]
    assert t[m["outputs"][0]]["shape"] == (1, 1000)


@pytest.mark.parametrize("name", MODELS)
def test_cpu_reference_runs(name):
    m = R.parse(zoo.MODELS[name](batch=1, image=224, seed=2))
    x = np.random.default_rng(0).standard_normal((2, 224, 224, 3)).astype(np.float32)
    out = _run_model(m, [x])[0]
    assert out.shape == (2, 1000) and np.isfinite(out).all() and np.allclose(out.sum(-1), 1.0, atol=1e-4)


@pytest.mark.parametrize("name", MODELS)
def test_readers_agree_host_prepare_and_resize(name):
    blob = zoo.MODELS[name](batch=2, image=224, seed=1)
    m = R.parse(blob)
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    assert g.num_nodes() == len(m["ops"])
    for i, t in enumerate(m["tensors"]):
        assert g.shape(i) == t["shape"], t["name"]
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (2, 1000)
    g.resize_input(g.inputs()[0], (3, 224, 224, 3))
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (3, 1000)
    assert g.fuse_pooled_signs() == 0   # the pass leaves a host-arena graph alone
    g.close()


def _names(g):
    return [g.node_name(i) for i in range(g.num_nodes())]


def _base(g):
    """fuse_all() without the pooled-sign pass"""
    return (g.fuse_dense_blocks() + g.fuse_residual_blocks() + g.fuse_float_glue() + g.fuse_channel_gates()
            + g.fuse_activation_chains() + g.fuse_residual_pairs())


@pytest.mark.parametrize("name", MODELS)
def test_fused_node_list(name):
    blob = zoo.MODELS[name](batch=2, image=224, seed=1)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    before = len(_names(g))
    assert g.fuse_pooled_signs() == 9 and g.fuse_pooled_signs() == 0
    names = _names(g)
    c = collections.Counter(names)
    assert c[POOLED] == 3 and len(names) == before - 9
    assert c["builtin:17"] == 0 and c["builtin:18"] == 0 and c["builtin:0"] == 0 and c["LceQuantize"] == 0
    # each fused node reads the float map before it and writes the signs the next convolution reads
    for i, n in enumerate(names):
        if n == POOLED:
            ins, outs = g.node_io(i)
            assert len(ins) == 3 and names[i + 1] == "LceBconv2d" and g.node_io(i + 1)[0][0] == outs[0]
    g.close()
    # under fuse_all the pass runs before the activation-chain pass, which otherwise takes ADD ->
    # LceQuantize: the base arm keeps MAX_POOL_2D, MUL and ADD+LceQuantize
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    assert g.fuse_all() == 9 and collections.Counter(_names(g))[POOLED] == 3
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    assert _base(g) == 3
    c = collections.Counter(_names(g))
    assert c["builtin:17"] == 3 and c["builtin:18"] == 3 and c["ADD+LceQuantize"] == 3
    g.close()


@pytest.mark.parametrize("name", OTHERS)
def test_other_models_keep_their_node_lists(name):
    blob = zoo.MODELS[name](batch=1, image=224, seed=2)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n = _base(g)
    before = _names(g)
    assert g.fuse_pooled_signs() == 0
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    assert g.fuse_all() == n and _names(g) == before
    g.close()


def test_other_models_bytes_are_unchanged():
    for (name, image), want in OTHER_HASHES.items():
        kw = dict(batch=1, image=224, seed=0) if image == 224 else dict(batch=2, image=64, seed=3,
                                                                          input_type="int8")
        assert hashlib.sha256(zoo.MODELS[name](**kw)).hexdigest() == want, (name, image)


def _pooled_block(x_shape=(2, 9, 9, 40), kind="MAX_POOL_2D", k=3, s=2, padding="VALID", pool_act="NONE",
                  scale_shape=None, mul_act="NONE", add_act="NONE", output=None, extra_reader=None, square=False):
    """x -> pool -> MUL(scale) -> ADD(shift) -> LceQuantize; `output` makes "y" (pool), "u" (MUL) or
    "v" (ADD) a graph output too, `extra_reader` gives that tensor a RELU reader, `square` makes the
    MUL read the pool's output as both operands (one reading node, two reading inputs)."""
    rng = np.random.default_rng(5)
    b, h, w, c = x_shape
    oh = -(-h // s) if padding == "SAME" else (h - k) // s + 1
    ow = -(-w // s) if padding == "SAME" else (w - k) // s + 1
    ys = (b, oh, ow, c)
    m = TFLiteModel()
    x = m.add_tensor("x", x_shape)
    t = {"y": m.add_tensor("y", ys), "u": m.add_tensor("u", ys), "v": m.add_tensor("v", ys)}
    scale = m.add_tensor("scale", None, data=rng.uniform(-1.5, 1.5, scale_shape or (c,)).astype(np.float32))
    shift = m.add_tensor("shift", None, data=rng.uniform(-0.5, 0.5, (c,)).astype(np.float32))
    q = m.add_tensor("q", ys[:3] + (L.cdiv(c, 32),), np.int32)
    m.add_op(kind, [x], [t["y"]], padding=padding, stride=(s, s), filter=(k, k), activation=pool_act)
    m.add_op("MUL", [t["y"], t["y"] if square else scale], [t["u"]], activation=mul_act)
    m.add_op("ADD", [t["u"], shift], [t["v"]], activation=add_act)
    m.add_op("LceQuantize", [t["v"]], [q], custom_options=b"")
    m.inputs, m.outputs = [x], [q]
    if extra_reader:
        r = m.add_tensor("r", ys)
        m.add_op("RELU", [t[extra_reader]], [r])
        m.outputs.append(r)
    if output:
        m.outputs.append(t[output])
    return m.serialize()


def test_pooled_block_fuses():
    g = H.HostGraph.from_tflite(_pooled_block(), device_arena=True)
    assert g.fuse_pooled_signs() == 3 and _names(g) == [POOLED]
    g.close()


@pytest.mark.parametrize("variant", ["pool_read_twice", "scale_not_per_channel", "mul_activation",
                                     "add_activation", "pool_is_a_graph_output", "mul_is_a_graph_output",
                                     "add_is_a_graph_output", "average_pool", "mul_reads_pool_twice"])
def test_pooled_block_refusals(variant):
    kw = {"pool_read_twice": dict(extra_reader="y"),
          "scale_not_per_channel": dict(scale_shape=(2, 4, 4, 40)),
          "mul_activation": dict(mul_act="RELU"),
          "add_activation": dict(add_act="RELU"),
          "pool_is_a_graph_output": dict(output="y"),
          "mul_is_a_graph_output": dict(output="u"),
          "add_is_a_graph_output": dict(output="v"),
          "average_pool": dict(kind="AVERAGE_POOL_2D"),
          "mul_reads_pool_twice": dict(square=True)}[variant]
    blob = _pooled_block(**kw)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    before = _names(g)
    assert g.fuse_pooled_signs() == 0
    assert _names(g) == before
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=False)   # and the graph prepares unfused
    g.allocate_tensors()
    g.close()


def test_kernel_compiles_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas=-v",
                        "-cubin", "-I", os.path.join(repo, "include"),
                        os.path.join(repo, "compute_engine_b200", "csrc", "lce_b200_builtins.cu"),
                        "-o", str(tmp_path / "builtins.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S*maxpool_affine_sign_kernel\S*)\n\s*(.*)", r.stderr)
    assert len(props) == 6, r.stderr
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)


# ----------------------------------- GPU ----------------------------------- #
def _np_pooled_signs(x, k, s, padding, act, scale, shift):
    """numpy float32: max over the in-bounds window, the activation, x * scale then + shift (each
    rounded), then the packed signs."""
    b, h, w, c = x.shape
    if padding == "SAME":
        oh, ow = -(-h // s[0]), -(-w // s[1])
        ph = max(0, (oh - 1) * s[0] + k[0] - h) // 2
        pw = max(0, (ow - 1) * s[1] + k[1] - w) // 2
    else:
        oh, ow, ph, pw = (h - k[0]) // s[0] + 1, (w - k[1]) // s[1] + 1, 0, 0
    y = np.empty((b, oh, ow, c), np.float32)
    for oy in range(oh):
        for ox in range(ow):
            y0, x0 = oy * s[0] - ph, ox * s[1] - pw
            win = x[:, max(0, y0):min(h, y0 + k[0]), max(0, x0):min(w, x0 + k[1])]
            y[:, oy, ox] = win.max(axis=(1, 2))
    if act == "RELU":
        y = np.maximum(y, np.float32(0))
    return L.pack_signs((y * scale).astype(np.float32) + shift)


# (x shape, filter, stride, padding, pool activation)
KERNEL_GRID = [
    ((2, 9, 9, 64), (3, 3), (2, 2), "VALID", "NONE"),
    ((2, 9, 9, 32), (3, 3), (2, 2), "SAME", "RELU"),
    ((3, 11, 7, 96), (3, 3), (2, 2), "SAME", "NONE"),        # h != w, windows crossing two borders
    ((2, 10, 13, 100), (3, 3), (1, 1), "SAME", "NONE"),      # C % 4 != 0: the scalar pool kernel
    ((1, 8, 6, 192), (2, 2), (2, 2), "VALID", "RELU"),
    ((2, 7, 9, 256), (2, 2), (1, 1), "SAME", "NONE"),
    ((2, 13, 13, 100), (3, 3), (2, 2), "VALID", "RELU"),
    ((4, 6, 5, 64), (3, 2), (1, 2), "SAME", "NONE"),         # a non-square window
    ((2, 27, 27, 192), (3, 3), (2, 2), "VALID", "NONE"),     # BinaryAlexNet's second pooled layer
]


def _special_map(rng, shape):
    """N(0, 1) with signed zeros, denormals and exact ties sprinkled in"""
    x = rng.standard_normal(shape).astype(np.float32)
    flat = x.reshape(-1)
    idx = rng.choice(flat.size, flat.size // 8, replace=False)
    specials = np.array([0.0, -0.0, 1e-40, -1e-40, 1e-45, -1e-45, 0.5, -0.5], np.float32)
    flat[idx] = specials[rng.integers(0, len(specials), idx.size)]
    return x


def _pool_graph(x_shape, k, s, padding, act, scale, shift):
    """the unfused MAX_POOL_2D -> MUL -> ADD -> LceQuantize as a graph"""
    b, h, w, c = x_shape
    m = TFLiteModel()
    x = m.add_tensor("x", x_shape)
    oh = -(-h // s[0]) if padding == "SAME" else (h - k[0]) // s[0] + 1
    ow = -(-w // s[1]) if padding == "SAME" else (w - k[1]) // s[1] + 1
    ys = (b, oh, ow, c)
    y, u, v = (m.add_tensor(n, ys) for n in "yuv")
    q = m.add_tensor("q", ys[:3] + (L.cdiv(c, 32),), np.int32)
    m.add_op("MAX_POOL_2D", [x], [y], padding=padding, stride=s, filter=k, activation=act)
    m.add_op("MUL", [y, m.add_tensor("scale", None, data=scale)], [u])
    m.add_op("ADD", [u, m.add_tensor("shift", None, data=shift)], [v])
    m.add_op("LceQuantize", [v], [q], custom_options=b"")
    m.inputs, m.outputs = [x], [q]
    return m.serialize()


@pytest.mark.gpu
def test_gpu_kernel_matches_numpy_and_the_unfused_kernels():
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import assert_same_bits, dev
    rng = np.random.default_rng(11)
    for n, (shape, k, s, padding, act) in enumerate(KERNEL_GRID):
        c = shape[3]
        x = _special_map(rng, shape)
        scale = rng.uniform(0.25, 1.5, c).astype(np.float32) * rng.choice([-1, 1], c).astype(np.float32)
        shift = rng.uniform(-0.5, 0.5, c).astype(np.float32)
        shift[rng.choice(c, c // 4, replace=False)] = np.float32(0.0)
        shift[rng.choice(c, c // 8, replace=False)] = np.float32(-0.0)
        shift[rng.choice(c, c // 8, replace=False)] = np.float32(1e-40)
        tag = f"case {n} {shape} {k} {s} {padding} {act}"
        want = _np_pooled_signs(x, k, s, padding, act, scale, shift)
        assert 0 < np.unpackbits(want.view(np.uint8)).mean() < 1, tag
        code = {"SAME": capi.PADDING_SAME, "VALID": capi.PADDING_VALID}[padding]
        got = capi.maxpool_affine_sign(dev(x), k, s, code, {"NONE": capi.ACT_NONE, "RELU": capi.ACT_RELU}[act],
                                       dev(scale), dev(shift))
        torch.cuda.synchronize()
        assert_same_bits(got.cpu().numpy(), want, tag)
        g = H.HostGraph.from_tflite(_pool_graph(shape, k, s, padding, act, scale, shift), device_arena=True)
        g.allocate_tensors()
        g.write(g.inputs()[0], x)
        g.invoke()
        assert_same_bits(g.read(g.outputs()[0]), want, tag + " (unfused kernels)")
        g.close()


@pytest.mark.gpu
def test_gpu_kernel_refusals():
    import torch
    from compute_engine_b200 import capi
    x = torch.zeros(1, 5, 5, 32, device="cuda")
    with pytest.raises(capi.LceError, match="unknown padding"):
        capi.maxpool_affine_sign(x, (3, 3), (2, 2), 7)
    with pytest.raises(capi.LceError, match="pool: bad parameters"):
        capi.maxpool_affine_sign(x, (3, 3), (0, 2))


def _gpu_step(blob, x, fused, preserve, launches):
    """a warm-up step, one eager step (its launches counted), then a CUDA-graph capture and replay;
    returns the eager and replayed outputs. The input is written before every step: with reused
    arenas a later tensor may take the input's memory."""
    from compute_engine_b200 import capi
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.resize_input(g.inputs()[0], x.shape)
    g.fuse_all() if fused else _base(g)
    g.preserve_all_tensors(preserve)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    g.synchronize()
    g.write(g.inputs()[0], x)
    l0 = capi.launch_count()
    g.invoke()
    g.synchronize()
    launches.append(capi.launch_count() - l0)
    eager = g.read(g.outputs()[0])
    g.enable_cuda_graph(True)
    g.write(g.inputs()[0], x)
    g.invoke()   # capture
    g.write(g.inputs()[0], x)
    g.invoke()   # replay
    replay = g.read(g.outputs()[0])
    g.close()
    return eager, replay


@pytest.mark.gpu
@pytest.mark.parametrize("name", MODELS)
def test_gpu_graph_op_by_op(name):
    """The unfused graph on the device at 224, op by op on the device's own input tensors: every
    LCE op, MAX_POOL_2D, MUL, ADD and RESHAPE bit exact, the float convolution, FULLY_CONNECTED and
    SOFTMAX within the torch fp32 reference's tolerance; then the class probabilities against the
    CPU graph."""
    blob = zoo.MODELS[name](batch=2, image=224, seed=9)
    m = R.parse(blob)
    x = np.random.default_rng(3).standard_normal((2, 224, 224, 3)).astype(np.float32)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.preserve_all_tensors(True)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    exact = collections.Counter()
    for op in m["ops"]:
        vals = {i: g.read(i) for i in op["inputs"] if i >= 0 and m["tensors"][i]["data"] is None}
        want = _run_op(m, op, vals)
        got = g.read(op["outputs"][0])
        key = op["custom"] or op["code"]
        assert got.shape == want.shape, key
        if op["code"] in (32, 17, 18, 0, 22):
            assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), key
            exact[key] += 1
        else:
            scale = max(1.0, float(np.abs(want).max()))
            if op["code"] == 9:   # 4096-term dot products: their rounding error scales with sum |x w|
                w = m["tensors"][op["inputs"][1]]["data"]
                xin = vals[op["inputs"][0]].reshape(-1, w.shape[1])
                scale = max(scale, float((np.abs(xin) @ np.abs(w).T).max()))
            assert np.allclose(got, want, rtol=1e-4, atol=1e-5 * scale), (key, np.abs(got - want).max())
    assert exact["LceBconv2d"] == len(SPECS[name][1]) and exact["LceQuantize"] == 3 and exact[17] == 3
    want_out = _run_model(m, [x])[0]
    assert np.abs(g.read(g.outputs()[0]) - want_out).max() <= 2e-4
    g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", MODELS)
@pytest.mark.parametrize("pad_values", [0, 1])
def test_gpu_fused_equals_unfused(name, pad_values):
    """With every tensor kept and with reused arenas, eager and on CUDA-graph replay. Each pooled
    layer runs one launch where the base arm ran three (MAX_POOL_2D, MUL, ADD+LceQuantize)."""
    blob = zoo.MODELS[name](batch=1, image=224, seed=4, pad_values=pad_values, input_type="int8")
    x = np.random.default_rng(6).integers(-128, 128, (2, 224, 224, 3)).astype(np.int8)
    for preserve in (True, False):
        launches = []
        ref = _gpu_step(blob, x, False, preserve, launches)
        got = _gpu_step(blob, x, True, preserve, launches)
        assert launches[0] - launches[1] == 2 * 3, launches
        assert np.isfinite(got[0]).all()
        for r, o, what in ((ref[0], got[0], "eager"), (ref[1], got[1], "replay"), (got[0], got[1], "fused eager vs replay")):
            assert np.array_equal(r.view(np.uint8), o.view(np.uint8)), (name, pad_values, preserve, what)


@pytest.mark.gpu
@pytest.mark.parametrize("name", MODELS)
def test_gpu_bitpacked_layers_run_on_mma_sync(name):
    """Each bitpacked LceBconv2d of the model as a one-node graph: one mma.sync launch and the
    oracle's words."""
    from compute_engine_b200 import capi
    from test_gpu_parity import assert_same_bits, path_counts
    m = R.parse(zoo.MODELS[name](batch=2, image=224, seed=7))
    t = m["tensors"]
    rng = np.random.default_rng(8)
    n = 0
    for op in _bconvs(m):
        if t[op["outputs"][0]]["dtype"] != np.int32:
            continue
        sub = TFLiteModel()
        xs = t[op["inputs"][0]]["shape"]
        xi = sub.add_tensor("x", xs, np.int32)
        f = sub.add_tensor("f", None, np.int32, data=t[op["inputs"][1]]["data"])
        thr = sub.add_tensor("thr", None, np.int32, data=t[op["inputs"][4]]["data"])
        y = sub.add_tensor("y", t[op["outputs"][0]]["shape"], np.int32)
        sub.add_op("LceBconv2d", [xi, f, -1, -1, thr], [y], custom_options=op["custom_options"])
        sub.inputs, sub.outputs = [xi], [y]
        x = rng.integers(-2**31, 2**31 - 1, xs, dtype=np.int64).astype(np.int32)
        g = H.HostGraph.from_tflite(sub.serialize(), device_arena=True)
        g.allocate_tensors()
        g.write(g.inputs()[0], x)
        before = path_counts(capi)
        g.invoke()
        g.synchronize()
        ran = [b - a for a, b in zip(before, path_counts(capi))]
        assert ran == [0, 1, 0], (xs, ran)
        assert_same_bits(g.read(g.outputs()[0]), _run_op(m, op, {op["inputs"][0]: x}), str(xs))
        g.close()
        n += 1
    assert n == (4 if name == "binaryalexnet" else 3)


@pytest.mark.gpu
@pytest.mark.parametrize("name", MODELS)
def test_gpu_interpreter_predict_resizes_the_fused_graph(name):
    from compute_engine_b200.interpreter import Interpreter
    blob = zoo.MODELS[name](batch=3, image=224, seed=5)
    m = R.parse(blob)
    it = Interpreter(blob)
    try:
        for b in (3, 5, 3):
            x = np.random.default_rng(b).standard_normal((b, 224, 224, 3)).astype(np.float32)
            got = it.predict(x)
            want = _run_model(m, [x])[0]
            assert got.shape == (b, 1000) and np.abs(got - want).max() <= 2e-4, b
    finally:
        it.close()   # its graph, arena and captured CUDA graph go now, not at garbage collection
