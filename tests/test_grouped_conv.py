"""Grouped CONV_2D: the kernel (lce_b200_f32_grouped_conv2d), the builtin's grouped filters, the
graph fusion of a grouped convolution with the BatchNorm after it (Graph::FuseGroupedConvAffine) and
MeliusNet with its two grouped stem convolutions as one op each (zoo.meliusnet(group_conv="native")).

CPU: the native model's op counts and filter shapes, the default model's bytes, its weights against
the split form's, the two forms through the CPU reference (grouped CONV_2D as per-group slices
through tflite_ref), both readers, host prepare and resize, grouped shape inference and each refusal,
the fused node list and each refused precondition, the existing CONV_2D passes on grouped
convolutions, every zoo model's node list, and the new instances compiled without spills. GPU: the
kernel bit for bit against conv_ref per group (test_gpu_float_kernels) with and without the epilogue,
and against per-group lce_b200_f32_conv2d plus a concatenation on the device; the native model bit for
bit against the split one, eager and under CUDA-graph replay, with every tensor kept and with reused
arenas, with the launches the fusion saves; Interpreter.predict across batch sizes."""
import collections
import hashlib
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import tflite_ref as R
from compute_engine_b200 import host as H
from compute_engine_b200 import zoo
from compute_engine_b200.tflite_writer import TFLiteModel
from test_dorefanet import OTHER_HASHES as _OLDER_HASHES

F32 = np.float32
FUSED = "CONV_2D+MUL+ADD"
# sha256 of every zoo model's bytes at the commit before group_conv="native" was added
ALL_HASHES = dict(_OLDER_HASHES)
ALL_HASHES.update({
    ("dorefanet", 224): "5edd486e889b1185d93e29d99175ac95a7e19208c34e656f061acbe111cd85a3",
    ("dorefanet", 64): "145662faee7a756c1d9c7a2a411a9ac725d8993769827175c03ae59395f2685b",
})


def _hash_kw(image):
    return dict(batch=1, image=224, seed=0) if image == 224 else dict(batch=2, image=64, seed=3, input_type="int8")


def _names(g):
    return [g.node_name(i) for i in range(g.num_nodes())]


def _native(**kw):
    return zoo.meliusnet(group_conv="native", **kw)


# ------------------------------ CPU reference ------------------------------ #
def _run_op(model, op, vals):
    """One op on the CPU as a list of its outputs: SPLIT in numpy, a grouped CONV_2D as one
    tflite_ref convolution per group on the channel slices, concatenated, every other op (and
    STRIDED_SLICE through test_meliusnet's numpy slicing) as test_meliusnet runs it."""
    from test_meliusnet import _run_op as melius_op
    t = model["tensors"]
    if op["code"] == 3:
        x, w = vals[op["inputs"][0]], t[op["inputs"][1]]["data"]
        bias = t[op["inputs"][2]]["data"] if len(op["inputs"]) > 2 and op["inputs"][2] >= 0 else None
        groups = x.shape[3] // w.shape[3]
        if groups > 1:
            cg, og = w.shape[3], w.shape[0] // groups
            parts = [R._conv(np.ascontiguousarray(x[..., k * cg:(k + 1) * cg]), w[k * og:(k + 1) * og],
                             None if bias is None else bias[k * og:(k + 1) * og], op["options"], False)
                     for k in range(groups)]
            return [np.concatenate(parts, axis=3)]
    return melius_op(model, op, vals)


def _run_model(model, inputs):
    vals = dict(zip(model["inputs"], inputs))
    for op in model["ops"]:
        vals.update(zip(op["outputs"], _run_op(model, op, vals)))
    return [vals[i] for i in model["outputs"]]


# ----------------------------------- CPU ----------------------------------- #
def test_native_model_op_counts_and_filters():
    split = R.parse(zoo.meliusnet22(batch=1, image=224, seed=1))
    m = R.parse(_native(batch=1, image=224, seed=1))
    t = m["tensors"]
    kinds = collections.Counter((o["code"], o["custom"]) for o in m["ops"])
    want = collections.Counter((o["code"], o["custom"]) for o in split["ops"])
    want[(49, "")] -= 2                       # no SPLIT
    want[(3, "")] -= 12 - 2                   # 12 per-group convolutions become 2
    want[(2, "")] -= 2                        # and their concatenations go
    assert kinds == +want and kinds[(49, "")] == 0 and kinds[(3, "")] == 6
    convs = [o for o in m["ops"] if o["code"] == 3]
    assert [t[c["inputs"][1]]["shape"] for c in convs[1:3]] == [(32, 3, 3, 8), (64, 3, 3, 4)]
    for c, cout in zip(convs[1:3], (32, 64)):
        assert t[c["inputs"][0]]["shape"] == (1, 112, 112, 32) and t[c["outputs"][0]]["shape"] == (1, 112, 112, cout)
        assert c["inputs"][2] == -1 and c["options"].scalar(0, "b") == 0 and c["options"].scalar(3, "b") == 0
        mul = next(o for o in m["ops"] if o["inputs"][0] == c["outputs"][0])
        add = next(o for o in m["ops"] if o["inputs"][0] == mul["outputs"][0])
        assert (mul["code"], add["code"], add["options"].scalar(0, "b")) == (18, 0, 1)   # MUL -> ADD(RELU)
    with pytest.raises(ValueError, match="group_conv"):
        zoo.meliusnet(group_conv="grouped")


def test_default_and_every_other_model_bytes_are_unchanged():
    assert hashlib.sha256(zoo.meliusnet22(**_hash_kw(224))).hexdigest() == ALL_HASHES[("meliusnet22", 224)]
    for (name, image), want in ALL_HASHES.items():
        assert hashlib.sha256(zoo.MODELS[name](**_hash_kw(image))).hexdigest() == want, (name, image)
    assert zoo.meliusnet(**_hash_kw(64)) == zoo.meliusnet22(**_hash_kw(64))


def test_native_weights_equal_the_split_forms():
    split = R.parse(zoo.meliusnet22(batch=1, image=64, seed=4))
    m = R.parse(_native(batch=1, image=64, seed=4))
    convs = [o for o in split["ops"] if o["code"] == 3]
    st, nt = split["tensors"], m["tensors"]
    native_convs = [o for o in m["ops"] if o["code"] == 3]
    for k, groups in ((1, 4), (2, 8)):
        per_group = [st[c["inputs"][1]]["data"] for c in convs[1 + (k - 1) * 4:1 + (k - 1) * 4 + groups]]
        assert np.array_equal(nt[native_convs[k]["inputs"][1]]["data"], np.concatenate(per_group))
    # every other constant, in graph order, bit for bit
    skip_split = {c["inputs"][1] for c in convs[1:13]} | {o["inputs"][0] for o in split["ops"] if o["code"] == 49}
    skip_native = {c["inputs"][1] for c in native_convs[1:3]}
    a = [st[i]["data"] for o in split["ops"] for i in o["inputs"] if i >= 0 and st[i]["data"] is not None
         and i not in skip_split]
    b = [nt[i]["data"] for o in m["ops"] for i in o["inputs"] if i >= 0 and nt[i]["data"] is not None
         and i not in skip_native]
    assert len(a) == len(b) and all(x.dtype == y.dtype and np.array_equal(x.view(np.uint8), y.view(np.uint8))
                                    for x, y in zip(a, b))


def test_cpu_reference_native_equals_split():
    x = np.random.default_rng(0).standard_normal((2, 32, 32, 3)).astype(F32)
    want = _run_model(R.parse(zoo.meliusnet22(batch=1, image=32, seed=2)), [x])[0]
    got = _run_model(R.parse(_native(batch=1, image=32, seed=2)), [x])[0]
    assert got.shape == (2, 1000) and np.allclose(got.sum(-1), 1.0, atol=1e-4)
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8))


def test_readers_agree_host_prepare_and_resize():
    blob = _native(batch=2, image=64, seed=1)
    m = R.parse(blob)
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    assert g.num_nodes() == len(m["ops"])
    assert _names(g) == [f"builtin:{o['code']}" if o["code"] != 32 else o["custom"] for o in m["ops"]]
    for i, t in enumerate(m["tensors"]):
        assert g.shape(i) == t["shape"], t["name"]
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (2, 1000)
    g.resize_input(g.inputs()[0], (3, 64, 64, 3))
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (3, 1000)
    g.close()


def _conv_graph(x_shape, w_shape, stride=1, padding="SAME", dilation=1, act="NONE", bias=False):
    m = TFLiteModel()
    x = m.add_tensor("x", x_shape)
    w = np.random.default_rng(0).standard_normal(w_shape).astype(F32)
    y = m.add_tensor("y", x_shape[:3] + (w_shape[0],))     # the builtin's Prepare sets the shape
    m.add_op("CONV_2D", [x, m.add_tensor("w", None, data=w),
                         m.add_tensor("b", None, data=np.ones(w_shape[0], F32)) if bias else -1], [y],
             padding=padding, stride=(stride, stride), dilation=(dilation, dilation), activation=act)
    m.inputs, m.outputs = [x], [y]
    return m.serialize()


@pytest.mark.parametrize("x_shape,w_shape,stride,padding,dilation,want", [
    ((2, 9, 7, 12), (6, 3, 3, 4), 1, "SAME", 1, (2, 9, 7, 6)),      # 3 groups
    ((2, 9, 7, 12), (8, 3, 3, 3), 2, "SAME", 1, (2, 5, 4, 8)),      # 4 groups
    ((1, 11, 8, 32), (64, 5, 5, 4), 1, "VALID", 1, (1, 7, 4, 64)),  # 8 groups
    ((1, 11, 8, 32), (32, 3, 3, 1), 2, "VALID", 2, (1, 4, 2, 32)),  # 32 groups, dilation 2
    ((3, 6, 5, 6), (4, 1, 1, 3), 1, "SAME", 1, (3, 6, 5, 4)),
])
def test_grouped_shape_inference(x_shape, w_shape, stride, padding, dilation, want):
    g = H.HostGraph.from_tflite(_conv_graph(x_shape, w_shape, stride, padding, dilation), device_arena=False)
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == want
    g.resize_input(g.inputs()[0], (5,) + x_shape[1:])
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (5,) + want[1:]
    g.close()


@pytest.mark.parametrize("x_shape,w_shape,message", [
    ((2, 8, 8, 12), (6, 3, 3, 5), "input's channels must be a multiple of the filter's input channels"),
    ((2, 8, 8, 12), (6, 3, 3, 24), "input's channels must be a multiple of the filter's input channels"),
    ((2, 8, 8, 12), (6, 3, 3, 3), "filter count must be a multiple of the group count"),
])
def test_grouped_refusals(x_shape, w_shape, message):
    g = H.HostGraph.from_tflite(_conv_graph(x_shape, w_shape), device_arena=False)
    with pytest.raises(H.HostError, match=message):
        g.allocate_tensors()
    g.close()


def _block(x_shape=(2, 10, 9, 32), filt=(32, 3, 3, 8), conv_act="NONE", mul_act="NONE", add_act="RELU",
           scale_shape=None, shift_shape=None, bias=False, conv_out_read_twice=False, conv_out_is_output=False,
           mul_out_read_twice=False, mul_out_is_output=False, const_first=False, square=False):
    """x -> CONV_2D -> MUL(scale) -> ADD(shift) [-> extra readers]; `square` makes the MUL read the
    convolution's output as both operands (one reading node, two reading inputs)."""
    rng = np.random.default_rng(3)
    C = filt[0]
    m = TFLiteModel()
    x = m.add_tensor("x", x_shape)
    y = m.add_tensor("y", x_shape[:3] + (C,))
    w = rng.standard_normal(filt).astype(F32) * F32(0.3)
    m.add_op("CONV_2D", [x, m.add_tensor("w", None, data=w),
                         m.add_tensor("b", None, data=rng.uniform(-1, 1, C).astype(F32)) if bias else -1], [y],
             padding="SAME", stride=(1, 1), activation=conv_act)
    scale = rng.uniform(0.5, 1.5, scale_shape or (C,)).astype(F32)
    shift = rng.uniform(-0.5, 0.5, shift_shape or (C,)).astype(F32)
    u = m.add_tensor("u", x_shape[:3] + (C,))
    sc = m.add_tensor("scale", None, data=scale)
    m.add_op("MUL", [y, y] if square else [sc, y] if const_first else [y, sc], [u], activation=mul_act)
    z = m.add_tensor("z", x_shape[:3] + (C,))
    m.add_op("ADD", [u, m.add_tensor("shift", None, data=shift)], [z], activation=add_act)
    m.outputs = [z]
    for read, t in ((conv_out_read_twice, y), (mul_out_read_twice, u)):
        if read:
            r = m.add_tensor("r", x_shape[:3] + (C,))
            m.add_op("RELU", [t], [r])
            m.outputs.append(r)
    if conv_out_is_output:
        m.outputs.append(y)
    if mul_out_is_output:
        m.outputs.append(u)
    m.inputs = [x]
    return m.serialize()


@pytest.mark.parametrize("kw", [dict(), dict(bias=True, add_act="RELU6"), dict(add_act="NONE"),
                                dict(scale_shape=(1, 1, 1, 32), shift_shape=(1, 32)),
                                dict(x_shape=(1, 7, 5, 32), filt=(64, 3, 3, 4)),
                                dict(x_shape=(1, 7, 5, 6), filt=(4, 1, 1, 3))])
def test_block_fuses(kw):
    blob = _block(**kw)
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    assert g.fuse_grouped_conv_affine() == 2 and _names(g) == [FUSED]
    ins, outs = g.node_io(0)
    assert len(ins) == 5 and (ins[2] >= 0) == kw.get("bias", False) and outs == [g.outputs()[0]]
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == kw.get("x_shape", (2, 10, 9, 32))[:3] + (kw.get("filt", (32,))[0],)
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    assert g.fuse_all() == 2 and _names(g) == [FUSED]
    g.close()


@pytest.mark.parametrize("variant", ["ungrouped", "conv_activation", "mul_activation", "scale_not_per_channel",
                                     "shift_not_per_channel", "scale_2d", "conv_out_read_twice", "conv_out_is_output",
                                     "mul_out_read_twice", "mul_out_is_output", "constant_first",
                                     "mul_reads_conv_out_twice"])
def test_block_refusals(variant):
    kw = {"ungrouped": dict(filt=(32, 3, 3, 32)), "conv_activation": dict(conv_act="RELU"),
          "mul_activation": dict(mul_act="RELU"), "scale_not_per_channel": dict(scale_shape=(1,)),
          "shift_not_per_channel": dict(shift_shape=(1,)), "scale_2d": dict(scale_shape=(2, 32)),
          "conv_out_read_twice": dict(conv_out_read_twice=True), "conv_out_is_output": dict(conv_out_is_output=True),
          "mul_out_read_twice": dict(mul_out_read_twice=True), "mul_out_is_output": dict(mul_out_is_output=True),
          "constant_first": dict(const_first=True), "mul_reads_conv_out_twice": dict(square=True)}[variant]
    g = H.HostGraph.from_tflite(_block(**kw), device_arena=False)
    before = _names(g)
    assert g.fuse_grouped_conv_affine() == 0 and _names(g) == before
    g.close()


def test_fused_node_list():
    blob = _native(batch=2, image=64, seed=1)
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    before = _names(g)
    assert g.fuse_grouped_conv_affine() == 4 and g.fuse_grouped_conv_affine() == 0
    names = _names(g)
    assert names.count(FUSED) == 2 and len(names) == len(before) - 4
    i = names.index(FUSED)
    assert names[i - 1:i + 3] == ["builtin:3", FUSED, FUSED, "builtin:17"]
    g.allocate_tensors()
    assert g.shape(g.node_io(i + 1)[1][0]) == (2, 32, 32, 64)
    g.resize_input(g.inputs()[0], (3, 64, 64, 3))
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (3, 1000) and g.shape(g.node_io(i)[1][0]) == (3, 32, 32, 32)
    g.close()
    # with every pass: the split form's fused list with its 20 stem nodes replaced by the two
    split = H.HostGraph.from_tflite(zoo.meliusnet22(batch=2, image=64, seed=1), device_arena=True)
    split.fuse_all()
    want = _names(split)
    split.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.fuse_all()
    got = _names(g)
    g.close()
    k = got.index(FUSED)
    assert got[:k] == want[:k] and got[k + 2:] == want[k + 20:] and len(want) - len(got) == 18
    assert want[k:k + 20].count("builtin:3") == 12 and want[k:k + 20].count("builtin:49") == 2


def _stem_graph(cin):
    """CONV_2D(3x3 s2, filter [16,3,3,3]) -> DEPTHWISE_CONV_2D(3x3 s2): FuseStem's pattern when cin == 3"""
    rng = np.random.default_rng(1)
    m = TFLiteModel()
    x = m.add_tensor("x", (1, 16, 16, cin))
    y = m.add_tensor("y", (1, 8, 8, 16))
    m.add_op("CONV_2D", [x, m.add_tensor("w", None, data=rng.standard_normal((16, 3, 3, 3)).astype(F32)),
                         m.add_tensor("b", None, data=np.zeros(16, F32))], [y], padding="SAME", stride=(2, 2),
             activation="RELU")
    z = m.add_tensor("z", (1, 4, 4, 16))
    m.add_op("DEPTHWISE_CONV_2D", [y, m.add_tensor("dw", None, data=rng.standard_normal((1, 3, 3, 16)).astype(F32)),
                                   m.add_tensor("db", None, data=np.zeros(16, F32))], [z],
             padding="SAME", stride=(2, 2), depth_multiplier=1)
    m.inputs, m.outputs = [x], [z]
    return m.serialize()


def _quantize_graph(cin, cout=32):
    """CONV_2D(3x3, filter [cout,3,3,16]) -> LceQuantize: FuseConvQuantize's pattern when cin == 16"""
    m = TFLiteModel()
    x = m.add_tensor("x", (1, 8, 8, cin))
    y = m.add_tensor("y", (1, 8, 8, cout))
    m.add_op("CONV_2D", [x, m.add_tensor("w", None, data=np.ones((cout, 3, 3, 16), F32)), -1], [y], padding="SAME",
             stride=(1, 1))
    q = m.add_tensor("q", (1, 8, 8, cout // 32), np.int32)
    m.add_op("LceQuantize", [y], [q], custom_options=b"")
    m.inputs, m.outputs = [x], [q]
    return m.serialize()


def test_existing_conv_passes_ignore_a_grouped_convolution():
    from test_dorefanet import _block as quant_block
    # FuseStem: the stem pattern, but the filter's 3 input channels are one of two groups
    for cin, want in ((3, 1), (6, 0)):
        g = H.HostGraph.from_tflite(_stem_graph(cin), device_arena=True)
        assert g.fuse_float_glue() == want, cin
        if want == 0:
            assert _names(g) == ["builtin:3", "builtin:4"]
        g.close()
    g = H.HostGraph.from_tflite(_stem_graph(6), device_arena=False)
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (1, 4, 4, 16)
    g.close()
    # FuseConvQuantize: CONV_2D -> LceQuantize stays two nodes when the conv is grouped
    for cin, want in ((16, 1), (32, 0)):
        g = H.HostGraph.from_tflite(_quantize_graph(cin), device_arena=True)
        assert g.fuse_float_glue() == want, cin
        g.close()
    # FuseQuantizedActivations: the quantiser in front of a grouped +-alpha convolution is left alone
    blob = quant_block(c=64)
    m = R.parse(blob)
    conv = next(o for o in m["ops"] if o["code"] == 3)
    w = m["tensors"][conv["inputs"][1]]["data"]
    assert w.shape == (64, 3, 3, 64)
    mm = TFLiteModel()   # the same block with a 2-group filter [64, 3, 3, 32]
    x = mm.add_tensor("x", (2, 6, 6, 64))
    cur = x
    for kind, v in (("MAXIMUM", 0.0), ("MINIMUM", 1.0), ("MUL", 3.0), ("ROUND", None), ("DIV", 3.0)):
        nxt = mm.add_tensor(kind.lower(), (2, 6, 6, 64))
        mm.add_op(kind, [cur] if v is None else [cur, mm.add_tensor("c", None, data=np.array([v], F32))], [nxt])
        cur = nxt
    y = mm.add_tensor("y", (2, 6, 6, 64))
    mm.add_op("CONV_2D", [cur, mm.add_tensor("w", None, data=np.ascontiguousarray(w[..., :32])), -1], [y],
              padding="SAME", stride=(1, 1))
    mm.inputs, mm.outputs = [x], [y]
    for b, want in ((blob, 4), (mm.serialize(), 0)):
        g = H.HostGraph.from_tflite(b, device_arena=False)
        assert g.fuse_quantized_activations() == want
        g.close()


def _without_grouped(g):
    """fuse_all() without fuse_grouped_conv_affine()"""
    return (g.fuse_dense_blocks() + g.fuse_residual_blocks() + g.fuse_float_glue() + g.fuse_quantized_activations()
            + g.fuse_pooled_signs() + g.fuse_channel_gates() + g.fuse_activation_chains() + g.fuse_residual_pairs())


@pytest.mark.parametrize("name", sorted(zoo.MODELS))
def test_every_zoo_model_keeps_its_node_list(name):
    blob = zoo.MODELS[name](batch=1, image=64, seed=2)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n = _without_grouped(g)
    before = _names(g)
    assert g.fuse_grouped_conv_affine() == 0
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    assert g.fuse_all() == n and _names(g) == before
    g.close()


def test_new_kernels_compile_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas=-v",
                        "-cubin", "-I", os.path.join(repo, "include"),
                        os.path.join(repo, "compute_engine_b200", "csrc", "lce_b200_builtins.cu"),
                        "-o", str(tmp_path / "builtins.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for kernel, count in (("grouped_conv3x3_kernel", 2), ("grouped_conv_any_kernel", 1)):
        props = re.findall(r"Function properties for (\S*%s\S*)\n\s*(.*)" % kernel, r.stderr)
        assert len(props) == count, r.stderr
        for name, line in props:
            assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)


# ----------------------------------- GPU ----------------------------------- #
def _grouped_ref(x, w, bias, groups, stride, dil, padding, act, scale=None, shift=None, post_act=0):
    """conv_ref per group on the channel slices, concatenated, then the epilogue in float32"""
    from test_gpu_float_kernels import _act, conv_ref
    cg, og = x.shape[3] // groups, w.shape[0] // groups
    y = np.concatenate([conv_ref(np.ascontiguousarray(x[..., k * cg:(k + 1) * cg]), w[k * og:(k + 1) * og],
                                 None if bias is None else bias[k * og:(k + 1) * og], stride, dil, padding, act)
                        for k in range(groups)], axis=3)
    if scale is not None:
        y = (y * scale).astype(F32)
    if shift is not None:
        y = (y + shift).astype(F32)
    return _act(y, post_act)


# (groups, in per group, out per group, filter, stride, dilation, padding, act, x (B, H, W), out offset,
# bias): groups 2, 4, 8, 32; 1 to 64 channels in per group, 1 to 16 out; 1x1, 3x3, 5x5; h != w;
# MeliusNet's two instances, also on ragged tiles, with VALID padding and off a 16-byte boundary
GRID = [
    (4, 8, 8, 3, 1, 1, "SAME", 0, (2, 37, 45), 0, False),
    (8, 4, 8, 3, 1, 1, "SAME", 0, (2, 37, 45), 0, False),
    (4, 8, 8, 3, 1, 1, "VALID", 1, (1, 19, 33), 0, True),
    (8, 4, 8, 3, 1, 1, "SAME", 3, (1, 9, 17), 1, True),
    (4, 8, 8, 3, 2, 1, "SAME", 2, (2, 13, 10), 0, True),
    (2, 3, 16, 3, 1, 1, "SAME", 1, (2, 11, 7), 0, True),
    (2, 16, 8, 5, 2, 1, "SAME", 0, (1, 12, 15), 1, False),
    (32, 1, 1, 3, 1, 2, "SAME", 3, (2, 10, 13), 0, True),
    (8, 1, 16, 1, 1, 1, "VALID", 0, (1, 6, 9), 0, True),
    (2, 64, 8, 1, 2, 1, "SAME", 2, (2, 7, 5), 1, False),
    (4, 4, 1, 5, 1, 2, "VALID", 1, (1, 14, 11), 0, True),
    (4, 16, 16, 3, 2, 2, "SAME", 0, (1, 15, 12), 0, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", GRID, ids=[f"g{c[0]}_{c[1]}to{c[2]}_k{c[3]}_s{c[4]}_d{c[5]}_{c[6]}_a{c[7]}_off{c[9]}"
                                            for c in GRID])
def test_gpu_kernel_matches_conv_ref(case):
    import torch
    from compute_engine_b200 import capi
    from test_gpu_float_kernels import _dev
    from test_gpu_parity import assert_same_bits
    groups, cg, og, k, s, d, padding, act, (b, h, w), off, has_bias = case
    rng = np.random.default_rng(groups * 1000 + cg * 100 + og * 10 + k + s + d + act + h)
    x = rng.standard_normal((b, h, w, groups * cg)).astype(F32)
    x.reshape(-1)[::7] = F32(-0.0)
    x.reshape(-1)[3::11] = F32(0.0)
    filt = (rng.standard_normal((groups * og, k, k, cg)) * 0.5).astype(F32)
    bias = rng.standard_normal(groups * og).astype(F32) if has_bias else None
    scale = rng.uniform(-1.5, 1.5, groups * og).astype(F32)
    shift = rng.uniform(-0.5, 0.5, groups * og).astype(F32)
    pad = capi.PADDING_SAME if padding == "SAME" else capi.PADDING_VALID
    for epi in ("none", "scale", "scale_shift"):
        sc = scale if epi != "none" else None
        sh = shift if epi == "scale_shift" else None
        post = {"none": 0, "scale": 0, "scale_shift": 1 + (act % 3)}[epi]
        want = _grouped_ref(x, filt, bias, groups, (s, s), (d, d), pad, act, sc, sh, post)
        out = _dev(np.full(want.size, np.nan, F32), off).view(want.shape)
        got = capi.grouped_conv2d(_dev(x, off).view(x.shape), _dev(filt).view(filt.shape),
                                  None if bias is None else torch.from_numpy(bias).cuda(), (s, s), (d, d), pad, act,
                                  None if sc is None else torch.from_numpy(sc).cuda(),
                                  None if sh is None else torch.from_numpy(sh).cuda(), post, out=out)
        torch.cuda.synchronize()
        assert_same_bits(got.cpu().numpy(), want, f"{case} {epi}")


@pytest.mark.gpu
def test_gpu_kernel_equals_per_group_conv2d_and_concatenation():
    import ctypes as C
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import assert_same_bits
    rng = np.random.default_rng(5)
    for groups, cg, og, shape, bias in ((4, 8, 8, (8, 112, 112), False), (8, 4, 8, (8, 112, 112), False),
                                        (4, 8, 8, (3, 29, 51), True), (2, 3, 16, (2, 21, 14), True)):
        x = torch.from_numpy(rng.standard_normal(shape + (groups * cg,)).astype(F32)).cuda()
        filt = torch.from_numpy((rng.standard_normal((groups * og, 3, 3, cg)) * 0.3).astype(F32)).cuda()
        b = torch.from_numpy(rng.standard_normal(groups * og).astype(F32)).cuda() if bias else None
        got = capi.grouped_conv2d(x, filt, b, activation=capi.ACT_RELU)
        parts = []
        for k in range(groups):
            xs = x[..., k * cg:(k + 1) * cg].contiguous()
            fs = filt[k * og:(k + 1) * og].contiguous()
            bs = None if b is None else b[k * og:(k + 1) * og].contiguous()
            y = torch.empty(shape + (og,), device="cuda")
            d = capi.ConvDesc(*shape, cg, 3, 3, og, 1, 1, 1, 1, capi.PADDING_SAME, capi.ACT_RELU)
            rc = capi.lib().lce_b200_f32_conv2d(C.byref(d), capi._p(xs), capi._p(fs), capi._p(bs), capi._p(y),
                                                capi._stream())
            assert rc == 0, capi.lib().lce_b200_last_error()
            parts.append(y)
        want = torch.cat(parts, dim=3)
        torch.cuda.synchronize()
        assert_same_bits(got.cpu().numpy(), want.cpu().numpy(), f"{groups} x {cg} -> {og} {shape}")


def _gpu_run(blob, x, preserve):
    """an eager step (and its kernel launches) and a CUDA-graph replay with fuse_all()"""
    from compute_engine_b200 import capi
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.resize_input(g.inputs()[0], x.shape)
    g.fuse_all()
    g.preserve_all_tensors(preserve)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()                      # plans are built
    g.write(g.inputs()[0], x)
    g.synchronize()
    before = capi.launch_count()
    g.invoke()
    g.synchronize()
    launches = capi.launch_count() - before
    eager = g.read(g.outputs()[0])
    g.enable_cuda_graph(True)
    g.write(g.inputs()[0], x)
    g.invoke()   # capture
    g.write(g.inputs()[0], x)
    g.invoke()   # replay
    replay = g.read(g.outputs()[0])
    names = _names(g)
    g.close()
    return eager, replay, launches, names


@pytest.mark.gpu
@pytest.mark.parametrize("image", [64, 224])
def test_gpu_native_model_equals_split_bit_for_bit(image):
    x = np.random.default_rng(image).integers(-128, 128, (3, image, image, 3)).astype(np.int8)
    kw = dict(batch=1, image=image, seed=6, input_type="int8")
    for preserve in (True, False):
        want = _gpu_run(zoo.meliusnet22(**kw), x, preserve)
        got = _gpu_run(_native(**kw), x, preserve)
        assert got[3].count(FUSED) == 2 and len(want[3]) - len(got[3]) == 18
        assert np.isfinite(got[0]).all() and np.allclose(got[0].sum(-1), 1.0, atol=1e-4)
        for a, b, what in ((got[0], want[0], "eager"), (got[1], want[1], "replay"), (got[1], got[0], "native replay")):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (image, preserve, what)
        # 12 per-group CONV_2D kernels and two MUL and two ADD passes become two launches; the SPLIT
        # and CONCATENATION nodes are copies, not kernels
        assert want[2] - got[2] == 14, (want[2], got[2])


@pytest.mark.gpu
def test_gpu_interpreter_predict_across_batch_sizes():
    from compute_engine_b200.interpreter import Interpreter
    it, ref = Interpreter(_native(batch=3, image=64, seed=5)), Interpreter(zoo.meliusnet22(batch=3, image=64, seed=5))
    try:
        assert it.fused_nodes_removed - ref.fused_nodes_removed == 4   # two MULs and two ADDs
        for b in (3, 5, 3):
            x = np.random.default_rng(b).standard_normal((b, 64, 64, 3)).astype(F32)
            got, want = it.predict(x), ref.predict(x)
            assert got.shape == (b, 1000) and np.array_equal(got.view(np.uint8), want.view(np.uint8)), b
    finally:
        it.close()
        ref.close()
