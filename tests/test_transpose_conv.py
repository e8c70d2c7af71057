"""Learned-upsampling decoders: the TRANSPOSE_CONV builtin (lce_b200_f32_transpose_conv2d), the binary
upsampler LceDequantize -> TRANSPOSE_CONV (+-1, kernel = stride) [-> ADD] [-> LceQuantize] as one b1
convolution with a pixel-shuffled store (lce_b200_bconv2d_run_fused_shuffle,
Graph::FuseBinaryTransposeConvs) and the zoo's quicknet_seg(upsample=...).

CPU: the writer's and reader's options, the zoo variants' ops, shapes and options (and the default's
bytes), the host's Prepare shapes and refusals, the fused node lists and each fusion precondition, the
other models' node lists, the new kernels' build.
GPU: the float kernel against float64 torch and bit for bit on +-1 data, one launch past 2^31 outputs,
the fused node against the op sequence bit for bit, the whole graph fused vs unfused and op by op,
arena independence and CUDA-graph replay, and Interpreter.predict over mini-batches."""
import collections
import hashlib
import itertools
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import test_segmentation as S
import tflite_ref as R
from compute_engine_b200 import host as H
from compute_engine_b200 import zoo
from compute_engine_b200.tflite_writer import TFLiteModel

F32 = np.float32
ACTS = ["NONE", "RELU", "RELU_N1_TO_1", "RELU6"]
ACT_CODE = {a: i for i, a in enumerate(ACTS)}
FUSED = "LceBconv2dTranspose"
# fuse_all's passes but fuse_binary_transpose_convs, in fuse_all's order
PASSES_BUT_TCONV = ("fuse_binary_bases", "fuse_dense_blocks", "fuse_residual_blocks", "fuse_spatial_scales",
                    "fuse_float_glue", "fuse_upsample_merges", "fuse_resize_argmax", "fuse_subpixel_convs",
                    "fuse_grouped_conv_affine", "fuse_quantized_activations", "fuse_pooled_signs",
                    "fuse_channel_gates", "fuse_activation_chains", "fuse_residual_pairs")


def in_size(out, k, s, padding):
    """The input size a convolution with this filter, stride and padding gives from `out`."""
    return (out + s - 1) // s if padding == "SAME" else (out + s - k) // s


# ---------------------------- small test graphs ---------------------------- #
def _tconv_graph(x_shape, cout, k, s, out_hw, padding="SAME", act="NONE", bias=True, seed=0, dtype=F32,
                 out_shape0=None, shape_dtype=np.int32, shape_len=4, bias_shape=None, w_cin=None, out_c=None):
    rng = np.random.default_rng(seed)
    b, h, w, cin = x_shape
    kh, kw = (k, k) if np.isscalar(k) else k
    sh, sw = (s, s) if np.isscalar(s) else s
    m = TFLiteModel()
    x = m.add_tensor("x", x_shape, dtype)
    shape = [out_shape0 if out_shape0 is not None else b, out_hw[0], out_hw[1], out_c or cout][:shape_len]
    st = m.add_tensor("shape", None, shape_dtype, data=np.array(shape, shape_dtype))
    wt = m.add_tensor("w", None, data=rng.standard_normal((cout, kh, kw, w_cin or cin)).astype(F32))
    ins = [st, wt, x]
    if bias:
        ins.append(m.add_tensor("bias", None, data=rng.uniform(-1, 1, bias_shape or (cout,)).astype(F32)))
    y = m.add_tensor("y", (b, out_hw[0], out_hw[1], cout), dtype)
    m.add_op("TRANSPOSE_CONV", ins, [y], padding=padding, stride=(sh, sw), activation=act)
    m.inputs, m.outputs = [x], [y]
    return m.serialize()


def _binary_graph(shape=(2, 3, 4, 96), cout=64, s=(2, 2), add=True, quant=True, act="NONE", add_act="NONE",
                  bias=True, weights=None, out_extra=(0, 0), skip_first=False, outputs=(), deq_reader=False,
                  broadcast_skip=False, seed=0, bias_values=None):
    """q -> LceDequantize -> TRANSPOSE_CONV [-> ADD(skip)] [-> LceQuantize] with +-1 weights."""
    rng = np.random.default_rng(seed)
    b, h, w, cin = shape
    sh, sw = s
    oh, ow = h * sh + out_extra[0], w * sw + out_extra[1]
    m = TFLiteModel()
    q = m.add_tensor("q", (b, h, w, (cin + 31) // 32), np.int32)
    deq = m.add_tensor("deq", shape)
    m.add_op("LceDequantize", [q], [deq], custom_options=b"")
    if weights is None:
        weights = (rng.integers(0, 2, (cout, sh, sw, cin)) * 2 - 1).astype(F32)
    st = m.add_tensor("shape", None, np.int32, data=np.array([b, oh, ow, cout], np.int32))
    ins = [st, m.add_tensor("w", None, data=weights), deq]
    if bias:
        bv = rng.uniform(-3, 3, cout).astype(F32) if bias_values is None else bias_values
        ins.append(m.add_tensor("bias", None, data=bv))
    y = m.add_tensor("y", (b, oh, ow, cout))
    m.add_op("TRANSPOSE_CONV", ins, [y], padding="SAME", stride=s, activation=act)
    inputs, outs, t = [q], [], {"deq": deq, "y": y}
    last = y
    if add:
        skip = m.add_tensor("skip", (1, 1, 1, cout) if broadcast_skip else (b, oh, ow, cout))
        inputs.append(skip)
        o = m.add_tensor("sum", (b, oh, ow, cout))
        m.add_op("ADD", [skip, y] if skip_first else [y, skip], [o], activation=add_act)
        last = t["sum"] = o
    outs.append(last)
    if quant:
        pk = m.add_tensor("pk", (b, oh, ow, (cout + 31) // 32), np.int32)
        m.add_op("LceQuantize", [last], [pk], custom_options=b"")
        outs.append(pk)
    if deq_reader:
        r = m.add_tensor("relu", shape)
        m.add_op("RELU", [deq], [r])
        outs.append(r)
    outs += [t[n] for n in outputs]
    m.inputs, m.outputs = inputs, outs
    return m.serialize()


def _names(g):
    return [g.node_name(i) for i in range(g.num_nodes())]


# ----------------------------------- CPU ----------------------------------- #
@pytest.mark.parametrize("padding,s,act", [("SAME", (2, 2), "NONE"), ("VALID", (3, 1), "RELU6"),
                                           ("SAME", (1, 3), "RELU_N1_TO_1")])
def test_options_read_back(padding, s, act):
    m = R.parse(_tconv_graph((1, 4, 4, 8), 5, 3, s, (4 * s[0], 4 * s[1]) if padding == "SAME" else
                             ((4 - 1) * s[0] + 3, (4 - 1) * s[1] + 3), padding=padding, act=act))
    op = m["ops"][0]
    assert op["code"] == 67
    o = op["options"]
    assert (o.scalar(0, "b"), o.scalar(1, "i"), o.scalar(2, "i"), o.scalar(3, "b")) == (
        {"SAME": 0, "VALID": 1}[padding], s[1], s[0], ACT_CODE[act])


def test_host_reader_reads_the_options():
    """VALID, stride (3, 1), a 3x3 filter: the host's Prepare gives the output only with these
    options (SAME or other strides would refuse the input's size)."""
    blob = _tconv_graph((2, 4, 6, 8), 5, 3, (3, 1), (12, 8), padding="VALID", act="RELU6")
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (2, 12, 8, 5)
    g.close()


NEAREST_SHA256 = {   # quicknet_seg's bytes before `upsample` existed
    (1, 64, "float32", None): "62f4b814a8c3a5bd2515803540fc8c50bbab6e1c1025847ff0a08331dd83e947",
    (2, 224, "int8", None): "207c45465d2d4151b144c4d54c0732fa697d8c69e02a2c6382b51933af46f4f9",
    (1, 64, "float32", "int64"): "56b8929f63c99782910f3cc85968267db18ab365a7b39c03da574da31275218c",
}


@pytest.mark.parametrize("key", sorted(NEAREST_SHA256, key=str))
def test_nearest_keeps_the_bytes(key):
    batch, image, input_type, labels = key
    kw = dict(batch=batch, image=image, input_type=input_type, labels=labels)
    assert hashlib.sha256(zoo.quicknet_seg(**kw)).hexdigest() == NEAREST_SHA256[key]
    assert zoo.quicknet_seg(upsample="nearest", **kw) == zoo.quicknet_seg(**kw)


@pytest.mark.parametrize("upsample", ["transpose", "binary_transpose"])
def test_zoo_variants_ops_shapes_and_options(upsample):
    m = R.parse(zoo.quicknet_seg(batch=2, image=64, upsample=upsample))
    base = collections.Counter((o["code"], o["custom"]) for o in R.parse(zoo.quicknet_seg(batch=2, image=64))["ops"])
    got = collections.Counter((o["code"], o["custom"]) for o in m["ops"])
    want = base.copy()
    want[(97, "")] -= 3
    want[(3, "")] -= 3
    want[(67, "")] += 3
    if upsample == "binary_transpose":
        want[(32, "LceQuantize")] += 3
        want[(32, "LceDequantize")] += 3
    assert got == +want
    t = m["tensors"]
    stages = [o for o in m["ops"] if o["code"] == 67]
    for op, (cin, cout, hw) in zip(stages, [(512, 256, 4), (256, 128, 8), (128, 64, 16)]):
        shape, wt, x, bias = op["inputs"]
        assert list(t[shape]["data"]) == [2, hw, hw, cout]
        assert t[x]["shape"] == (2, hw // 2, hw // 2, cin)
        assert t[wt]["shape"] == (cout, 2, 2, cin) and t[bias]["shape"] == (cout,)
        o = op["options"]
        assert (o.scalar(0, "b"), o.scalar(1, "i"), o.scalar(2, "i"), o.scalar(3, "b")) == (0, 2, 2, 0)
        assert set(np.unique(t[wt]["data"])) <= ({-1.0, 1.0} if upsample == "binary_transpose" else set(
            np.unique(t[wt]["data"])))
        if upsample == "binary_transpose":
            deq = next(p for p in m["ops"] if p["outputs"] == [x])
            assert deq["custom"] == "LceDequantize"
            qop = next(p for p in m["ops"] if p["outputs"] == deq["inputs"])
            assert qop["custom"] == "LceQuantize"
        add = next(p for p in m["ops"] if op["outputs"][0] in p["inputs"])
        assert add["code"] == 0
    assert t[m["outputs"][0]]["shape"] == (2, 64, 64, 21)
    with pytest.raises(ValueError, match="upsample"):
        zoo.quicknet_seg(upsample="bilinear")


PREPARE_GRID = [(k, s, p) for k in range(1, 6) for s in (1, 2, 3) for p in ("SAME", "VALID")]


def _outputs_for(k, s, padding):
    """Odd and even output sizes, with and without Keras' output_padding, whose input is non-empty."""
    return [o for o in (7, 8, 9, 13) if in_size(o, k, s, padding) >= 1]


@pytest.mark.parametrize("k,s,padding", PREPARE_GRID)
def test_host_prepares_shapes(k, s, padding):
    for oh, ow in itertools.product(_outputs_for(k, s, padding), repeat=2):
        h, w = in_size(oh, k, s, padding), in_size(ow, k, s, padding)
        blob = _tconv_graph((2, h, w, 3), 5, k, s, (oh, ow), padding=padding, out_shape0=7)
        g = H.HostGraph.from_tflite(blob, device_arena=False)
        g.allocate_tensors()
        assert g.shape(g.outputs()[0]) == (2, oh, ow, 5), (oh, ow)
        g.resize_input(g.inputs()[0], (5, h, w, 3))   # the batch follows the input, not output_shape[0]
        g.allocate_tensors()
        assert g.shape(g.outputs()[0]) == (5, oh, ow, 5)
        g.close()


@pytest.mark.parametrize("case,message", [
    ("shape not constant", "output_shape must be a constant int32 tensor of 4 elements"),
    ("shape int64", "output_shape must be a constant int32 tensor of 4 elements"),
    ("shape of 3", "output_shape must be a constant int32 tensor of 4 elements"),
    ("int8", "only float32 is supported"),
    ("rank 3", "the weights and the input must be 4-D"),
    ("cin", "the weights' input channels differ from the input's"),
    ("bias shape", "the bias must have shape [Cout]"),
    ("output channels", "output_shape[3] differs from the weights' output channels"),
    ("stride 0", "strides must be positive"),
    ("stride -1", "strides must be positive"),
    ("activation", "the fused activation must be NONE, RELU, RELU_N1_TO_1 or RELU6"),
    ("input size", "the input's height and width are not what a convolution"),
])
def test_host_refuses(case, message):
    kw = dict(x_shape=(1, 4, 4, 8), cout=6, k=2, s=2, out_hw=(8, 8))
    if case == "shape not constant":
        m = TFLiteModel()
        x = m.add_tensor("x", (1, 4, 4, 8))
        st = m.add_tensor("shape", (4,), np.int32)
        wt = m.add_tensor("w", None, data=np.ones((6, 2, 2, 8), F32))
        y = m.add_tensor("y", (1, 8, 8, 6))
        m.add_op("TRANSPOSE_CONV", [st, wt, x], [y], padding="SAME", stride=(2, 2))
        m.inputs, m.outputs = [x, st], [y]
        blob = m.serialize()
    else:
        if case == "shape int64":
            kw["shape_dtype"] = np.int64
        elif case == "shape of 3":
            kw["shape_len"] = 3
        elif case == "int8":
            kw["dtype"] = np.int8
        elif case == "rank 3":
            kw["x_shape"] = (4, 4, 8)
        elif case == "cin":
            kw["w_cin"] = 7
        elif case == "bias shape":
            kw["bias_shape"] = (1, 6)
        elif case == "output channels":
            kw["out_c"] = 5
        elif case == "stride 0":
            kw["s"] = (0, 2)
        elif case == "stride -1":
            kw["s"] = (2, -1)
        elif case == "input size":
            kw["out_hw"] = (10, 8)
        if case == "rank 3":
            blob = _rank3_graph()
        elif case == "activation":
            blob = _tconv_graph(**kw)
            blob = _patch_activation(blob)
        else:
            blob = _tconv_graph(**kw)
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    with pytest.raises(H.HostError, match=re.escape(message)):
        g.allocate_tensors()
    g.close()


def _rank3_graph():
    m = TFLiteModel()
    x = m.add_tensor("x", (4, 4, 8))
    st = m.add_tensor("shape", None, np.int32, data=np.array([1, 8, 8, 6], np.int32))
    wt = m.add_tensor("w", None, data=np.ones((6, 2, 2, 8), F32))
    y = m.add_tensor("y", (1, 8, 8, 6))
    m.add_op("TRANSPOSE_CONV", [st, wt, x], [y], padding="SAME", stride=(2, 2))
    m.inputs, m.outputs = [x], [y]
    return m.serialize()


def _patch_activation(blob):
    """The writer only writes the four activations TFLite has; a model with code 5 (TANH) is made by
    writing one with a marker activation and patching the byte."""
    import compute_engine_b200.tflite_writer as W
    saved = dict(W.ACT)
    W.ACT["TANH"] = 0x55
    try:
        m = TFLiteModel()
        x = m.add_tensor("x", (1, 4, 4, 8))
        st = m.add_tensor("shape", None, np.int32, data=np.array([1, 8, 8, 6], np.int32))
        wt = m.add_tensor("w", None, data=np.ones((6, 2, 2, 8), F32))
        y = m.add_tensor("y", (1, 8, 8, 6))
        m.add_op("TRANSPOSE_CONV", [st, wt, x], [y], padding="SAME", stride=(2, 2), activation="TANH")
        m.inputs, m.outputs = [x], [y]
        b = bytearray(m.serialize())
    finally:
        W.ACT.clear()
        W.ACT.update(saved)
    assert b.count(0x55) >= 1
    i = bytes(b).index(bytes([0x55]))
    b[i] = 5
    assert R.parse(bytes(b))["ops"][0]["options"].scalar(3, "b") == 5
    return bytes(b)


@pytest.mark.parametrize("add,quant", [(True, True), (True, False), (False, True), (False, False)])
def test_fused_node_lists(add, quant):
    g = H.HostGraph.from_tflite(_binary_graph(add=add, quant=quant, skip_first=add), device_arena=True)
    n0 = g.num_nodes()
    removed = g.fuse_binary_transpose_convs()
    name = FUSED + ("+ADD" if add else "") + ("+LceQuantize" if quant else "")
    assert _names(g) == [name] and removed == n0 - 1
    ins = g.node_io(0)[0]
    assert ins[0] == g.inputs()[0] and (ins[3] == g.inputs()[1] if add else ins[3] == -1)
    assert g.node_outputs(0) == g.outputs()
    g.close()
    g = H.HostGraph.from_tflite(_binary_graph(add=add, quant=quant, bias=False), device_arena=True)
    assert g.fuse_binary_transpose_convs() == n0 - 1 and g.node_io(0)[0][2] == -1
    g.close()


@pytest.mark.parametrize("variant", ["0.5 weight", "-0.0 weight", "cout 32", "output_padding",
                                     "conv output", "sum output unfused", "deq output", "deq second reader",
                                     "broadcast skip", "host arena", "stride 1"])
def test_fusion_preconditions(variant):
    rng = np.random.default_rng(1)
    w = (rng.integers(0, 2, (64, 2, 2, 96)) * 2 - 1).astype(F32)
    kw = {}
    partial = None
    if variant == "0.5 weight":
        w[3, 1, 0, 7] = 0.5
        kw["weights"] = w
    elif variant == "-0.0 weight":
        w[3, 1, 0, 7] = -0.0
        kw["weights"] = w
    elif variant == "cout 32":
        kw["cout"] = 32
    elif variant == "output_padding":
        kw["out_extra"] = (1, 0)
    elif variant == "conv output":
        kw["outputs"] = ("y",)
        partial = FUSED   # y is stored: the ADD and its LceQuantize stay out
    elif variant == "deq output":
        kw["outputs"] = ("deq",)
    elif variant == "deq second reader":
        kw["deq_reader"] = True
    elif variant == "broadcast skip":
        kw["broadcast_skip"] = True
        partial = FUSED   # the ADD (and its LceQuantize) stay out
    elif variant == "stride 1":
        kw["s"] = (1, 1)
    if variant == "sum output unfused":
        kw["outputs"] = ("sum",)   # the sum is stored anyway: the fusion takes it
        partial = FUSED + "+ADD+LceQuantize"
    blob = _binary_graph(**kw)
    g = H.HostGraph.from_tflite(blob, device_arena=variant != "host arena")
    before = _names(g)
    removed = g.fuse_binary_transpose_convs()
    if partial is None:
        assert removed == 0 and _names(g) == before, variant
    else:
        assert _names(g)[0] == partial and removed == len(before) - g.num_nodes(), _names(g)
    g.close()


def _seg_fused(blob):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    removed = g.fuse_all()
    names = _names(g)
    g.close()
    return names, removed


def test_quicknet_seg_binary_transpose_fused_node_list():
    blob = zoo.quicknet_seg(batch=1, image=224, upsample="binary_transpose")
    names, _ = _seg_fused(blob)
    ups = [n for n in names if n.startswith(FUSED)]
    assert ups == [FUSED + "+ADD+LceQuantize"] * 3
    # no other pass takes the TRANSPOSE_CONV, its ADD or its LceQuantize: fuse_all's other passes leave
    # all three of each stage, and the pass alone then fuses them
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    for p in PASSES_BUT_TCONV:
        getattr(g, p)()
    left = _names(g)
    assert left.count("builtin:67") == 3 and left.count("LceDequantize") == 3
    for k, n in enumerate(left):
        if n == "builtin:67":
            y = g.node_io(k)[1][0]
            readers = [j for j in range(g.num_nodes()) if y in g.node_io(j)[0]]
            assert [left[j] for j in readers] == ["builtin:0"]
            s = g.node_io(readers[0])[1][0]
            assert "LceQuantize" in [left[j] for j in range(g.num_nodes()) if s in g.node_io(j)[0]]
    assert g.fuse_binary_transpose_convs() == 9
    g.close()
    # the float variant has nothing to fuse
    g = H.HostGraph.from_tflite(zoo.quicknet_seg(batch=1, image=224, upsample="transpose"), device_arena=True)
    assert g.fuse_binary_transpose_convs() == 0
    g.close()


@pytest.mark.parametrize("case", sorted(S._other_models()))
def test_other_models_keep_their_node_lists(case):
    make, kw = S._other_models()[case]
    blob = make(batch=1, seed=0, image=224, **kw)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n0 = g.num_nodes()
    assert g.fuse_binary_transpose_convs() == 0 and g.num_nodes() == n0
    g.close()
    names, _ = _seg_fused(blob)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    for p in PASSES_BUT_TCONV:
        getattr(g, p)()
    assert _names(g) == names
    g.close()


def _ptxas(src, tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas=-v",
                        "-cubin", "-I", os.path.join(repo, "include"),
                        "-I", os.path.join(repo, "compute_engine_b200", "csrc"),
                        os.path.join(repo, "compute_engine_b200", "csrc", src),
                        "-o", str(tmp_path / "k.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return r.stderr


def test_kernels_compile_without_spills(tmp_path):
    log = _ptxas("lce_b200_builtins.cu", tmp_path)
    props = re.findall(r"Function properties for (\S*transpose_conv_kernel\S*)\n\s*(.*)", log)
    assert len(props) == 2, log   # float and float4 loads
    # the shuffle store: bconv_imma_kernel<V, float, b1, ..., SHUFFLE = true> for V = 1, 2, 4
    log += _ptxas("lce_b200.cu", tmp_path)
    shuffle = re.findall(r"Function properties for (\S*bconv_imma_kernelILi\dELi0ELb1ELb0ELb0ELb0ELb0ELb0ELb1E\S*)"
                         r"\n\s*(.*)", log)
    assert len(shuffle) == 3, log
    for name, line in props + shuffle:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)


# ----------------------------------- GPU ----------------------------------- #
def transpose_conv_ref(x, w, bias, out_hw, stride, act, dtype=torch.float32):
    """TFLite's TRANSPOSE_CONV (reference/transpose_conv.h) of x [B, H, W, Cin] with weights [Cout, kh, kw,
    Cin]: the full transposed convolution cropped at TFLite's padding (ComputePaddingHeightWidth on the
    output's size, the floor half), zeros where the output runs past its end, then the bias and the
    fused activation (a name in ACTS), in `dtype`. The batch follows x. SAME and VALID give the same
    crop once x's size is consistent with the output's."""
    (oh, ow), (sh, sw) = out_hw, stride
    kh, kw = w.shape[1], w.shape[2]
    xt = torch.from_numpy(np.asarray(x)).to(dtype).permute(0, 3, 1, 2)
    wt = torch.from_numpy(np.asarray(w)).to(dtype).permute(3, 0, 1, 2)   # [Cin, Cout, kh, kw]
    y = torch.nn.functional.conv_transpose2d(xt, wt, stride=(sh, sw))
    ph = max((x.shape[1] - 1) * sh + kh - oh, 0) // 2
    pw = max((x.shape[2] - 1) * sw + kw - ow, 0) // 2
    y = torch.nn.functional.pad(y, (0, max(0, pw + ow - y.shape[3]), 0, max(0, ph + oh - y.shape[2])))
    y = y[:, :, ph:ph + oh, pw:pw + ow]
    if bias is not None:
        y = y + torch.from_numpy(np.asarray(bias)).to(dtype).reshape(1, -1, 1, 1)
    return _torch_act(y, act).permute(0, 2, 3, 1).contiguous().numpy()


def _run_op(m, op, vals):
    """One op of a parsed model on the CPU: TRANSPOSE_CONV here (fp32, the order torch picks), every
    other op as test_segmentation runs it."""
    if op["code"] != 67:
        return S._run_op(m, op, vals)
    t, o = m["tensors"], op["options"]
    shape, wt, x = op["inputs"][:3]
    bias = op["inputs"][3] if len(op["inputs"]) > 3 else -1
    return transpose_conv_ref(vals[x], t[wt]["data"], t[bias]["data"] if bias >= 0 else None,
                              tuple(int(v) for v in t[shape]["data"][1:3]), (o.scalar(2, "i"), o.scalar(1, "i")),
                              ACTS[o.scalar(3, "b")])


def _torch_act(y, act):
    return R._act(y, ACT_CODE[act])


def _ref64(x, w, bias, out_hw, s, act):
    return transpose_conv_ref(x, w, bias, out_hw, s, act, dtype=torch.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("k,s,padding", PREPARE_GRID)
def test_gpu_float_kernel_matches_float64(k, s, padding):
    from compute_engine_b200 import capi
    rng = np.random.default_rng(k * 100 + s * 10 + len(padding))
    for (oh, ow), cin, cout, act, bias in zip(
            itertools.product(_outputs_for(k, s, padding), repeat=2),
            itertools.cycle([3, 8, 16, 5]), itertools.cycle([5, 12, 64, 1, 33]), itertools.cycle(ACTS),
            itertools.cycle([True, False, True])):
        h, w = in_size(oh, k, s, padding), in_size(ow, k, s, padding)
        x = rng.standard_normal((2, h, w, cin)).astype(F32)
        wt = rng.standard_normal((cout, k, k, cin)).astype(F32)
        b = rng.uniform(-1, 1, cout).astype(F32) if bias else None
        got = capi.transpose_conv2d(torch.from_numpy(x).cuda(), torch.from_numpy(wt).cuda(),
                                    None if b is None else torch.from_numpy(b).cuda(), (oh, ow), (s, s),
                                    {"SAME": 0, "VALID": 1}[padding], ACT_CODE[act]).cpu().numpy()
        want = _ref64(x, wt, b, (oh, ow), (s, s), act)
        # the sums' magnitude before the activation clamps them sets the rounding error's scale
        scale = max(1.0, float(np.abs(_ref64(x, wt, b, (oh, ow), (s, s), "NONE")).max()))
        assert np.allclose(got, want, rtol=1e-4, atol=1e-5 * scale), (oh, ow, cin, cout, act, bias)
    # the host's node computes the same
    oh = ow = _outputs_for(k, s, padding)[-1]
    h, w = in_size(oh, k, s, padding), in_size(ow, k, s, padding)
    blob = _tconv_graph((2, h, w, 8), 6, k, s, (oh, ow), padding=padding, act="RELU6")
    m = R.parse(blob)
    x = rng.standard_normal((2, h, w, 8)).astype(F32)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    got = g.read(g.outputs()[0])
    g.close()
    t = m["tensors"]
    wt, b = t[m["ops"][0]["inputs"][1]]["data"], t[m["ops"][0]["inputs"][3]]["data"]
    want = _ref64(x, wt, b, (oh, ow), (s, s), "RELU6")
    assert np.allclose(got, want, rtol=1e-4, atol=1e-5 * max(1.0, float(np.abs(want).max())))


def _exact_pm1(x, w, bias, out_hw, s, act):
    """+-1 data: the float64 result is an exact integer; then one float32 rounding for the bias."""
    d = transpose_conv_ref(x, w, None, out_hw, s, "NONE", dtype=torch.float64)
    y = d.astype(F32)
    if bias is not None:
        y = (y + bias).astype(F32)
    return _torch_act(torch.from_numpy(y), act).numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("k,s", [(2, 2), (3, 2), (4, 2), (3, 3), (1, 1), (5, 3)])
def test_gpu_float_kernel_is_exact_on_pm1(k, s):
    from compute_engine_b200 import capi
    rng = np.random.default_rng(k * 10 + s)
    for cin, act in ((96, "NONE"), (512, "RELU"), (7, "RELU6"), (64, "RELU_N1_TO_1")):
        h, w = 5, 6
        x = (rng.integers(0, 2, (2, h, w, cin)) * 2 - 1).astype(F32)
        wt = (rng.integers(0, 2, (64, k, k, cin)) * 2 - 1).astype(F32)
        b = rng.uniform(-3, 3, 64).astype(F32)
        b[::5] = -0.0
        got = capi.transpose_conv2d(torch.from_numpy(x).cuda(), torch.from_numpy(wt).cuda(),
                                    torch.from_numpy(b).cuda(), (h * s, w * s), (s, s), 0, ACT_CODE[act])
        assert S._same_bits(got.cpu().numpy(), _exact_pm1(x, wt, b, (h * s, w * s), (s, s), act))


@pytest.mark.gpu
def test_gpu_float_kernel_past_2_pow_31_outputs():
    """[2, 16384, 16384, 4] outputs (2^31 floats + ...) from a 2x2 / stride 2 layer with 4 channels in."""
    from compute_engine_b200 import capi
    b, h, w, cin, cout = 2, 8192, 8200, 4, 4
    assert b * 2 * h * 2 * w * cout > 2 ** 31
    rng = np.random.default_rng(0)
    x = torch.from_numpy((rng.integers(0, 2, (b, h, w, cin)) * 2 - 1).astype(F32)).cuda()
    wt = (rng.integers(0, 2, (cout, 2, 2, cin)) * 2 - 1).astype(F32)
    bias = rng.uniform(-1, 1, cout).astype(F32)
    out = capi.transpose_conv2d(x, torch.from_numpy(wt).cuda(), torch.from_numpy(bias).cuda(), (2 * h, 2 * w),
                                (2, 2))
    torch.cuda.synchronize()
    for bi, y0 in ((0, 0), (1, h - 3), (1, h // 2)):   # the last rows lie past 2^31 floats
        xs = x[bi:bi + 1, y0:y0 + 3].cpu().numpy()
        want = _exact_pm1(xs, wt, bias, (6, 2 * w), (2, 2), "NONE")
        assert S._same_bits(out[bi:bi + 1, 2 * y0:2 * y0 + 6].cpu().numpy(), want), (bi, y0)
    del out, x
    torch.cuda.empty_cache()


def _run(blob, feeds, fuse):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    removed = g.fuse_binary_transpose_convs() if fuse else 0
    g.allocate_tensors()
    for t, v in zip(g.inputs(), feeds):
        g.write(t, v)
    g.invoke()
    outs = [g.read(t) for t in g.outputs()]
    names = _names(g)
    g.close()
    return outs, removed, names


FUSED_CASES = [dict(add=a, quant=q, act=act, add_act=aa, bias=bi, shape=shp, s=s, cout=c)
               for (a, q), act, aa, bi, shp, s, c in zip(
                   itertools.cycle([(True, True), (True, False), (False, True), (False, False)]),
                   ACTS * 3, ["NONE", "RELU", "RELU6", "RELU_N1_TO_1"] * 3, [True, False, True] * 4,
                   itertools.cycle([(2, 3, 4, 96), (3, 7, 5, 512), (1, 9, 11, 40), (2, 14, 14, 256)]),
                   itertools.cycle([(2, 2), (3, 3), (2, 1), (1, 2)]), itertools.cycle([64, 128, 192]))]


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(FUSED_CASES)))
def test_gpu_fused_node_is_the_op_sequence(case):
    kw = dict(FUSED_CASES[case])
    rng = np.random.default_rng(case)
    b, h, w, cin = kw["shape"]
    sh, sw = kw["s"]
    c = kw["cout"]
    bias = rng.uniform(-3, 3, c).astype(F32)
    bias[::4] = -0.0
    bias[1::4] = 0.0
    kw["bias_values"] = bias
    feeds = [_pack(rng, (b, h, w, cin))]
    if kw["add"]:
        skip = np.round(rng.standard_normal((b, h * sh, w * sw, c)) * 4).astype(F32)
        skip.reshape(-1)[::7] = -0.0
        skip.reshape(-1)[3::7] = 0.0
        feeds.append(skip)
    blob = _binary_graph(**kw)
    want, _, _ = _run(blob, feeds, False)
    got, removed, names = _run(blob, feeds, True)
    assert removed > 0 and names[0].startswith(FUSED), names
    for a, bb in zip(want, got):
        assert S._same_bits(a, bb)


def _pack(rng, shape):
    """LceQuantize of random signs on the host: bit 1 <=> negative, tail bits zero."""
    b, h, w, c = shape
    bits = np.zeros((b, h, w, ((c + 31) // 32) * 32), np.uint64)
    bits[..., :c] = rng.integers(0, 2, (b, h, w, c))
    words = (bits.reshape(b, h, w, -1, 32) << np.arange(32, dtype=np.uint64)).sum(-1)
    return words.astype(np.uint32).view(np.int32)


def _seg_images(batch, image, seed):
    return np.random.default_rng(seed).standard_normal((batch, image, image, 3)).astype(F32)


@pytest.mark.gpu
def test_gpu_quicknet_seg_binary_transpose_fused_equals_unfused():
    # each model at its batch: the unfused graph's LceDequantize keeps its output's shape, as the
    # reference's Prepare does, so that graph cannot be resized to another batch
    for batch in (4, 64):
        blob = zoo.quicknet_seg(batch=batch, image=224, seed=4, upsample="binary_transpose")
        x = _seg_images(batch, 224, batch)
        outs = {}
        for fuse in (False, True):
            g = H.HostGraph.from_tflite(blob, device_arena=True)
            if fuse:
                g.fuse_all()
                assert sum(n.startswith(FUSED) for n in _names(g)) == 3
            g.resize_input(g.inputs()[0], x.shape)
            g.allocate_tensors()
            g.write(g.inputs()[0], x)
            g.invoke()
            outs[fuse] = g.read(g.outputs()[0])
            g.close()
        assert np.isfinite(outs[True]).all()
        assert S._same_bits(outs[False], outs[True]), batch


@pytest.mark.gpu
@pytest.mark.parametrize("upsample", ["transpose", "binary_transpose"])
def test_gpu_quicknet_seg_op_by_op(upsample):
    """The unfused graph on the device, op by op on the device's own inputs: the LCE ops, the ADDs, the
    resize and the binary TRANSPOSE_CONVs (+-1 products: exact) bit for bit, the float builtins within
    the torch fp32 reference's tolerance."""
    blob = zoo.quicknet_seg(batch=3, image=64, seed=9, upsample=upsample)
    m = R.parse(blob)
    x = _seg_images(3, 64, 3)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.preserve_all_tensors(True)
    g.resize_input(g.inputs()[0], x.shape)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    exact = collections.Counter()
    for op in m["ops"]:
        act = [i for i in op["inputs"] if i >= 0 and m["tensors"][i]["data"] is None]
        vals = {i: g.read(i) for i in act}
        got = g.read(op["outputs"][0])
        if op["code"] == 67 and upsample == "binary_transpose":
            shape, wt, xi, bi = op["inputs"]
            t = m["tensors"]
            want = _exact_pm1(vals[xi], t[wt]["data"], t[bi]["data"], tuple(t[shape]["data"][1:3]), (2, 2), "NONE")
        else:
            want = _run_op(m, op, vals)
        assert got.shape == want.shape, (op["code"], op["custom"])
        if op["code"] in (0, 23, 32) or (op["code"] == 67 and upsample == "binary_transpose"):
            assert S._same_bits(got, want.astype(got.dtype)), (op["code"], op["custom"])
            exact[op["custom"] or op["code"]] += 1
        else:
            scale = max(1.0, float(np.abs(want).max()))
            assert np.allclose(got, want, rtol=1e-4, atol=1e-5 * scale), (op["code"], np.abs(got - want).max())
    assert exact[67] == (3 if upsample == "binary_transpose" else 0)
    g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("upsample,fuse", [("binary_transpose", True), ("transpose", True), ("transpose", False)])
def test_gpu_upsamplers_do_not_depend_on_the_arena(upsample, fuse):
    """The checks resize the batch, which the unfused binary graph's LceDequantize does not take."""
    import test_arena_independence as A
    blob = zoo.quicknet_seg(batch=1, seed=0, image=224, upsample=upsample)
    fails = A.check_arena_independence(blob, (A.BATCH, 224, 224, 3), "float32", fuse=fuse)
    assert not fails, f"quicknet_seg({upsample}):\n" + "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("upsample,batch_size", [("binary_transpose", 3), ("transpose", 5)])
def test_gpu_interpreter_predict_over_mini_batches(upsample, batch_size):
    from compute_engine_b200.interpreter import Interpreter
    blob = zoo.quicknet_seg(batch=1, image=64, seed=2, input_type="int8", upsample=upsample)
    x = zoo.quantize_images(_seg_images(11, 64, 1))
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.fuse_all()
    g.resize_input(g.inputs()[0], x.shape)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    want = g.read(g.outputs()[0])
    g.close()
    it = Interpreter(blob, batch_size=batch_size)
    got = it.predict(x)
    it.close()
    assert S._same_bits(np.asarray(got), want)
