"""Super-resolution graphs: the DEPTH_TO_SPACE builtin (lce_b200_f32_depth_to_space), the sub-pixel tail
CONV_2D -> DEPTH_TO_SPACE [-> ADD(RESIZE_BILINEAR(img))] in one pass (lce_b200_f32_subpixel_conv,
Graph::FuseSubpixelConvs) and the zoo's binary_srnet.

CPU: the writer's and reader's block_size, the zoo model's ops, shapes and options, the host's Prepare
shapes and refusals, the fused node list and each fusion precondition, the other models' node lists,
the new kernels' build.
GPU: DEPTH_TO_SPACE bit for bit against a numpy reshape / transpose, the fused kernel against the four
builtins run one by one (signed zeros included), the whole graph fused vs unfused, arena independence
and CUDA-graph replay, and Interpreter.predict over mini-batches."""
import collections
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import test_segmentation as S
import tflite_ref as R
from compute_engine_b200 import host as H
from compute_engine_b200 import zoo
from compute_engine_b200.tflite_writer import TFLiteModel

FUSED = "CONV_2D+DEPTH_TO_SPACE+RESIZE_BILINEAR+ADD"
FUSED_CONV = "CONV_2D+DEPTH_TO_SPACE"
F32 = np.float32

# fuse_all's passes but fuse_subpixel_convs, in fuse_all's order
PASSES_BUT_SUBPIXEL = ("fuse_binary_bases", "fuse_dense_blocks", "fuse_residual_blocks", "fuse_spatial_scales",
                       "fuse_float_glue", "fuse_upsample_merges", "fuse_resize_argmax", "fuse_grouped_conv_affine",
                       "fuse_quantized_activations", "fuse_pooled_signs", "fuse_channel_gates",
                       "fuse_activation_chains", "fuse_residual_pairs")


def depth_to_space_ref(x, r):
    """out[b, y*r + i, x*r + j, c] = in[b, y, x, (i*r + j)*C' + c], as a reshape and a transpose."""
    b, h, w, c = x.shape
    cp = c // (r * r)
    return x.reshape(b, h, w, r, r, cp).transpose(0, 1, 3, 2, 4, 5).reshape(b, h * r, w * r, cp)


# ---------------------------- small test graphs ---------------------------- #
def _d2s_graph(in_shape, r, in_dtype=np.float32, out_dtype=None, out_shape=None):
    m = TFLiteModel()
    x = m.add_tensor("x", in_shape, in_dtype)
    if out_shape is None:
        if len(in_shape) == 4 and r > 0 and in_shape[3] % (r * r) == 0:
            b, h, w, c = in_shape
            out_shape = (b, h * r, w * r, c // (r * r))
        else:
            out_shape = in_shape
    y = m.add_tensor("y", out_shape, out_dtype or in_dtype)
    m.add_op("DEPTH_TO_SPACE", [x], [y], block_size=r)
    m.inputs, m.outputs = [x], [y]
    return m.serialize()


def _tail_graph(shape=(2, 5, 7, 8), r=2, cp=3, img_hw=None, flags=(False, True), residual=True, bias=True,
                conv_act="NONE", add_act="NONE", k=3, stride=1, cout=None, img_first=False, seed=0,
                weights=None, second_reader=None, conv_output=False, shuffled_output=False,
                resized_output=False, dynamic_filter=False, small=False):
    """x -> CONV_2D(k x k, stride) -> y -> DEPTH_TO_SPACE(r) -> s [-> ADD(s, RESIZE_BILINEAR(img))]."""
    rng = np.random.default_rng(seed)
    b, h, w, cin = shape
    cout = cout or cp * r * r
    cp = cout // (r * r)
    oh, ow = -(-h // stride), -(-w // stride)
    m = TFLiteModel()
    x = m.add_tensor("x", shape)
    inputs = [x]
    if weights is None:
        weights = _values(rng, (cout, k, k, cin), small) / np.float32(np.sqrt(k * k * cin))
    if dynamic_filter:
        f = m.add_tensor("f", (cout, k, k, cin))
        inputs.append(f)
    else:
        f = m.add_tensor("f", None, data=weights.astype(F32))
    if bias is True:
        bias = rng.uniform(-0.5, 0.5, cout).astype(F32)
    bt = m.add_tensor("bias", None, data=np.asarray(bias, F32)) if bias is not False else -1
    y = m.add_tensor("y", (b, oh, ow, cout))
    m.add_op("CONV_2D", [x, f, bt], [y], padding="SAME", stride=(stride, stride), activation=conv_act)
    out_shape = (b, oh * r, ow * r, cp)
    s = m.add_tensor("s", out_shape)
    m.add_op("DEPTH_TO_SPACE", [y], [s], block_size=r)
    outs = [s]
    if residual:
        ih, iw = img_hw or (h, w)
        img = m.add_tensor("img", (b, ih, iw, cp))
        inputs.append(img)
        size = m.add_tensor("size", None, np.int32, data=np.array(out_shape[1:3], np.int32))
        up = m.add_tensor("up", out_shape)
        m.add_op("RESIZE_BILINEAR", [img, size], [up], align_corners=flags[0], half_pixel_centers=flags[1])
        o = m.add_tensor("o", out_shape)
        m.add_op("ADD", [up, s] if img_first else [s, up], [o], activation=add_act)
        outs = [o]
        if resized_output:
            outs.append(up)
    if second_reader is not None:
        t = {"conv": y, "shuffled": s, "resized": outs[0] if not residual else up}[second_reader]
        rl = m.add_tensor("relu", tuple(m.tensors[t]["shape"]))
        m.add_op("RELU", [t], [rl])
        outs.append(rl)
    if conv_output:
        outs.append(y)
    if shuffled_output:
        outs.append(s)
    m.inputs, m.outputs = inputs, outs
    return m.serialize()


def _values(rng, shape, small=False):
    """Normal values with exact zeros of both signs; `small` adds +-1e-30 and +-1e-20 too, whose
    products underflow to signed zeros."""
    v = rng.standard_normal(shape).astype(F32)
    levels = np.array([0.0, -0.0] + ([1e-30, -1e-30, 1e-20, -1e-20] if small else []), F32)
    pick = rng.random(shape) < 0.3
    v[pick] = rng.choice(levels, size=int(pick.sum()))
    return v


def _names(g):
    return [g.node_name(i) for i in range(g.num_nodes())]


def _max_cout():
    from compute_engine_b200 import capi
    return capi.subpixel_conv_max_out_channels()


# ----------------------------------- CPU ----------------------------------- #
@pytest.mark.parametrize("r", [1, 2, 3, 4, 7])
def test_block_size_reads_back(r):
    m = R.parse(_d2s_graph((1, 2, 2, r * r * 3), r))
    assert m["ops"][0]["code"] == 5
    assert m["ops"][0]["options"].scalar(0, "i") == r


SR_BODY = {(3, ""): 2, (32, "LceQuantize"): 16, (32, "LceBconv2d"): 16, (0, ""): 17, (5, ""): 1}


@pytest.mark.parametrize("scale", [2, 3, 4])
@pytest.mark.parametrize("image", [64, (18, 32)])
@pytest.mark.parametrize("residual", [True, False])
@pytest.mark.parametrize("input_type", ["float32", "int8"])
def test_binary_srnet_ops_shapes_and_options(scale, image, residual, input_type):
    blob = zoo.binary_srnet(batch=2, image=image, scale=scale, residual=residual, input_type=input_type)
    m = R.parse(blob)
    h, w = (image, image) if isinstance(image, int) else image
    want = dict(SR_BODY)
    if residual:
        want[(0, "")] += 1
        want[(23, "")] = 1
    if input_type == "int8":
        want[(6, "")] = 1
    assert collections.Counter((o["code"], o["custom"]) for o in m["ops"]) == want
    t = m["tensors"]
    assert t[m["outputs"][0]]["shape"] == (2, scale * h, scale * w, 3)
    img = m["inputs"][0]
    if input_type == "int8":
        deq = m["ops"][0]
        assert deq["code"] == 6 and deq["inputs"] == [img] and np.dtype(t[img]["dtype"]) == np.int8
        img = deq["outputs"][0]
    head = next(o for o in m["ops"] if o["code"] == 3)
    assert head["inputs"][0] == img and t[head["inputs"][1]]["shape"] == (64, 3, 3, 3)
    assert t[head["inputs"][2]]["shape"] == (64,)
    tail_i = max(i for i, o in enumerate(m["ops"]) if o["code"] == 3)
    tail = m["ops"][tail_i]
    assert t[tail["inputs"][1]]["shape"] == (3 * scale * scale, 3, 3, 64)
    assert t[tail["inputs"][2]]["shape"] == (3 * scale * scale,)
    assert tail["options"].scalar(0, "b") == 0   # SAME
    ds = m["ops"][tail_i + 1]
    assert ds["code"] == 5 and ds["inputs"] == tail["outputs"] and ds["options"].scalar(0, "i") == scale
    if residual:
        rz, add = m["ops"][tail_i + 2], m["ops"][tail_i + 3]
        assert rz["code"] == 23 and rz["inputs"][0] == img
        assert list(t[rz["inputs"][1]]["data"]) == [scale * h, scale * w]
        assert rz["options"].scalar(3, "b") == 1 and rz["options"].scalar(2, "b") == 0
        assert add["code"] == 0 and sorted(add["inputs"]) == sorted(ds["outputs"] + rz["outputs"])
        assert add["outputs"] == m["outputs"]
    else:
        assert ds["outputs"] == m["outputs"]
    with pytest.raises(ValueError, match="scale"):
        zoo.binary_srnet(scale=5)


def test_binary_srnet_is_not_in_models():
    assert "binary_srnet" not in zoo.MODELS


@pytest.mark.parametrize("r", [1, 2, 3, 4])
@pytest.mark.parametrize("cp", [1, 3, 5])
def test_host_prepares_depth_to_space_shapes(r, cp):
    g = H.HostGraph.from_tflite(_d2s_graph((2, 5, 7, cp * r * r), r), device_arena=False)
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (2, 5 * r, 7 * r, cp)
    g.close()


@pytest.mark.parametrize("case,message", [
    ("rank 3", "input must be a 4-D tensor"),
    ("block_size 0", "block_size must be positive"),
    ("block_size -2", "block_size must be positive"),
    ("channels", "channels must be a multiple of block_size^2"),
    ("int8 input", "only float32 is supported"),
    ("int32 input", "only float32 is supported"),
    ("output type differs", "output's type differs from the input's"),
])
def test_host_refuses_depth_to_space(case, message):
    if case == "rank 3":
        blob = _d2s_graph((5, 7, 12), 2)
    elif case == "block_size 0":
        blob = _d2s_graph((1, 5, 7, 12), 0)
    elif case == "block_size -2":
        blob = _d2s_graph((1, 5, 7, 12), -2)
    elif case == "channels":
        blob = _d2s_graph((1, 5, 7, 12), 3)
    elif case == "int8 input":
        blob = _d2s_graph((1, 5, 7, 12), 2, np.int8)
    elif case == "int32 input":
        blob = _d2s_graph((1, 5, 7, 12), 2, np.int32)
    else:
        blob = _d2s_graph((1, 5, 7, 12), 2, np.float32, np.int32)
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    with pytest.raises(H.HostError, match=re.escape(message)):
        g.allocate_tensors()
    g.close()


def _sr_fused(blocks=16):
    names = ["CONV_2D+LceQuantize"] + ["LceBconv2d+ADD+LceBconv2d+ADD+LceQuantize"] * (blocks // 2 - 1)
    return names + ["LceBconv2d+ADD+LceBconv2d+ADD", "builtin:0"]


@pytest.mark.parametrize("scale", [2, 3, 4])
def test_binary_srnet_fused_node_list(scale):
    blob = zoo.binary_srnet(batch=2, image=64, scale=scale, seed=1)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n0 = g.num_nodes()
    removed = g.fuse_all()
    assert _names(g) == _sr_fused() + [FUSED]
    assert g.num_nodes() == n0 - removed
    g.close()
    # fuse_all's other passes leave the tail as four ops, and the pass alone fuses them
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    for p in PASSES_BUT_SUBPIXEL:
        getattr(g, p)()
    assert _names(g) == _sr_fused() + ["builtin:3", "builtin:5", "builtin:23", "builtin:0"]
    assert g.fuse_subpixel_convs() == 3
    assert _names(g) == _sr_fused() + [FUSED]
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    assert g.fuse_subpixel_convs() == 3 and g.num_nodes() == n0 - 3 and _names(g)[-1] == FUSED
    g.close()
    # without the residual the conv and the shuffle fuse
    g = H.HostGraph.from_tflite(zoo.binary_srnet(image=64, scale=scale, residual=False), device_arena=True)
    assert g.fuse_subpixel_convs() == 1 and _names(g)[-1] == FUSED_CONV
    g.close()


def test_fused_node_inputs():
    g = H.HostGraph.from_tflite(_tail_graph(), device_arena=True)
    assert g.fuse_subpixel_convs() == 3 and _names(g) == [FUSED]
    ins, outs = g.node_io(0)
    assert len(ins) == 5 and ins[0] == g.inputs()[0] and ins[3] == g.inputs()[1] and outs == g.outputs()
    g.close()
    g = H.HostGraph.from_tflite(_tail_graph(bias=False, img_first=True), device_arena=True)
    assert g.fuse_subpixel_convs() == 3 and _names(g) == [FUSED]
    assert g.node_io(0)[0][2] == -1
    g.close()


@pytest.mark.parametrize("variant,want", [
    ("conv second reader", None), ("conv output", None), ("1x1 conv", None), ("strided conv", None),
    ("cout too wide", None), ("dynamic filter", None), ("cin not a multiple of 4", None),
    ("block size 1", None), ("shuffled second reader", "partial"), ("shuffled output", "partial"),
    ("resized second reader", "partial"), ("resized output", "partial"), ("broadcast img", "partial"),
    ("host arena", None),
])
def test_fusion_preconditions(variant, want):
    kw = {}
    if variant == "conv second reader":
        kw["second_reader"] = "conv"
    elif variant == "conv output":
        kw["conv_output"] = True
    elif variant == "1x1 conv":
        kw["k"] = 1
    elif variant == "strided conv":
        kw["stride"] = 2
    elif variant == "cout too wide":   # EDSR's 64 -> 256 upsampler convolution
        kw.update(shape=(1, 6, 6, 64), cout=_max_cout() * 4, r=2)
    elif variant == "dynamic filter":
        kw["dynamic_filter"] = True
    elif variant == "cin not a multiple of 4":
        kw["shape"] = (2, 5, 7, 6)
    elif variant == "block size 1":
        kw.update(r=1, cp=12)
    elif variant == "shuffled second reader":
        kw["second_reader"] = "shuffled"
    elif variant == "shuffled output":
        kw["shuffled_output"] = True
    elif variant == "resized second reader":
        kw["second_reader"] = "resized"
    elif variant == "resized output":
        kw["resized_output"] = True
    elif variant == "broadcast img":
        kw["img_hw"] = (3, 3)
    if variant == "host arena":
        g = H.HostGraph.from_tflite(_tail_graph(), device_arena=False)
        assert g.fuse_subpixel_convs() == 0
        g.close()
        return
    if variant == "broadcast img":
        # an img of another size is resized to s's shape: that is no broadcast, so it fuses; a
        # broadcast ADD ([1, 1, 1, C'] against s) is what must stay
        blob = _broadcast_tail_graph()
    else:
        blob = _tail_graph(**kw)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    before = _names(g)
    removed = g.fuse_subpixel_convs()
    if want is None:
        assert removed == 0 and _names(g) == before
    else:
        assert removed == 1
        assert _names(g) == [FUSED_CONV] + before[2:], _names(g)
    g.close()


def _broadcast_tail_graph():
    """The ADD's other operand is a RESIZE_BILINEAR output [B, 1, 1, C'] that the ADD broadcasts."""
    rng = np.random.default_rng(0)
    m = TFLiteModel()
    x = m.add_tensor("x", (2, 5, 7, 8))
    f = m.add_tensor("f", None, data=rng.standard_normal((12, 3, 3, 8)).astype(F32))
    y = m.add_tensor("y", (2, 5, 7, 12))
    m.add_op("CONV_2D", [x, f, -1], [y], padding="SAME", stride=(1, 1), activation="NONE")
    s = m.add_tensor("s", (2, 10, 14, 3))
    m.add_op("DEPTH_TO_SPACE", [y], [s], block_size=2)
    img = m.add_tensor("img", (2, 3, 3, 3))
    size = m.add_tensor("size", None, np.int32, data=np.array([1, 1], np.int32))
    up = m.add_tensor("up", (2, 1, 1, 3))
    m.add_op("RESIZE_BILINEAR", [img, size], [up])
    o = m.add_tensor("o", (2, 10, 14, 3))
    m.add_op("ADD", [s, up], [o])
    m.inputs, m.outputs = [x, img], [o]
    return m.serialize()


def test_fusion_takes_a_resize_from_another_size():
    g = H.HostGraph.from_tflite(_tail_graph(img_hw=(3, 4)), device_arena=True)
    assert g.fuse_subpixel_convs() == 3 and _names(g) == [FUSED]
    g.close()


@pytest.mark.parametrize("case", sorted(S._other_models()))
def test_other_models_keep_their_node_lists(case):
    make, kw = S._other_models()[case]
    blob = make(batch=1, seed=0, image=224, **kw)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n0 = g.num_nodes()
    assert g.fuse_subpixel_convs() == 0 and g.num_nodes() == n0
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.fuse_all()
    after = _names(g)
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    for p in PASSES_BUT_SUBPIXEL:
        getattr(g, p)()
    assert _names(g) == after
    g.close()


@pytest.mark.parametrize("make", [zoo.quicknet_seg, zoo.quicknet_ssd])
def test_dense_prediction_models_keep_their_node_lists(make):
    g = H.HostGraph.from_tflite(make(batch=1, seed=0, image=224), device_arena=True)
    assert g.fuse_subpixel_convs() == 0
    g.close()


def test_subpixel_kernels_compile_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(repo, "compute_engine_b200", "csrc", "lce_b200_builtins.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas=-v",
                        "-cubin", "-I", os.path.join(repo, "include"),
                        "-I", os.path.join(repo, "compute_engine_b200", "csrc"), src,
                        "-o", str(tmp_path / "builtins.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S*(?:depth_to_space_kernel|subpixel_conv_kernel)\S*)\n\s*(.*)",
                       r.stderr)
    # depth_to_space_kernel by floats and float4s, subpixel_conv_kernel for 16, 32 and 64 channels
    assert len(props) == 5, r.stderr
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)


# ----------------------------------- GPU ----------------------------------- #
@pytest.mark.gpu
@pytest.mark.parametrize("r", [1, 2, 3, 4])
@pytest.mark.parametrize("cp", [1, 3, 4, 5, 16])
def test_gpu_depth_to_space_matches_numpy(r, cp):
    import torch
    from compute_engine_b200 import capi
    rng = np.random.default_rng(r * 100 + cp)
    for b, h, w in ((1, 1, 1), (2, 5, 7), (3, 13, 9)):
        x = _values(rng, (b, h, w, cp * r * r), small=True)
        got = capi.depth_to_space(torch.from_numpy(x).cuda(), r).cpu().numpy()
        assert S._same_bits(got, depth_to_space_ref(x, r)), (b, h, w)
    x = _values(rng, (2, 5, 7, cp * r * r))
    g = H.HostGraph.from_tflite(_d2s_graph(x.shape, r), device_arena=True)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    got = g.read(g.outputs()[0])
    g.close()
    assert S._same_bits(got, depth_to_space_ref(x, r))


@pytest.mark.gpu
def test_gpu_depth_to_space_past_2_pow_31_values():
    """[2, 1024, 1024, 1028] -> [2, 2048, 2048, 257]: 2.16 * 10^9 floats, past 2^31."""
    import torch
    from compute_engine_b200 import capi
    shape, r = (2, 1024, 1024, 1028), 2
    assert np.prod(shape) > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(shape, device="cuda", generator=g)
    got = capi.depth_to_space(x, r)
    want = x.view(2, 1024, 1024, r, r, 257).permute(0, 1, 3, 2, 4, 5).reshape(2, 2048, 2048, 257)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    del x, got, want
    torch.cuda.empty_cache()


def _run(blob, feeds, passes=()):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    for p in passes:
        getattr(g, p)()
    names = _names(g)
    g.allocate_tensors()
    for t, v in zip(g.inputs(), feeds):
        g.write(t, v)
    g.invoke()
    out = g.read(g.outputs()[0])
    g.close()
    return out, names


TAIL_CASES = [(r, cp, cin) for r in (2, 3, 4) for cp in (1, 3) for cin in (4, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("r,cp,cin", TAIL_CASES)
def test_gpu_fused_tail_is_the_four_ops(r, cp, cin):
    rng = np.random.default_rng(r * 1000 + cp * 100 + cin)
    shape = (2, 9, 11, cin)
    combos = [(residual, bias, conv_act, add_act, flags)
              for residual in (True, False) for bias in (False, True)
              for conv_act, add_act in (("NONE", "NONE"), ("RELU", "RELU6"), ("RELU6", "RELU"), ("NONE", "RELU"))
              for flags in (S.FLAGS["bilinear"] if residual else [(False, False)])]
    for residual, bias, conv_act, add_act, flags in combos:
        blob = _tail_graph(shape, r, cp, img_hw=(5, 6), flags=flags, residual=residual, bias=bias,
                           conv_act=conv_act, add_act=add_act, seed=len(combos), small=True)
        feeds = [_values(rng, shape, small=True)]
        if residual:
            feeds.append(_values(rng, (2, 5, 6, cp), small=True))
        fused, names = _run(blob, feeds, ("fuse_subpixel_convs",))
        assert names == [FUSED if residual else FUSED_CONV]
        unfused, _ = _run(blob, feeds)
        assert S._same_bits(fused, unfused), (residual, bias, conv_act, add_act, flags)


@pytest.mark.gpu
def test_gpu_fused_tail_signed_zeros():
    """Inputs and weights whose products underflow to zero, taps past the border and K padding terms,
    without a bias and with a bias of -0.0: every output is a zero, and its bits are the unfused chain's."""
    import torch
    from compute_engine_b200 import capi
    rng = np.random.default_rng(9)
    for cin in (4, 12, 64):
        x = np.where(rng.random((1, 6, 7, cin)) < 0.5, F32(-1e-30), F32(1e-30)).astype(F32)
        w = np.where(rng.random((12, 3, 3, cin)) < 0.5, F32(-1e-20), F32(1e-20)).astype(F32)
        xd, wd = torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda()
        for bias in (None, np.full(12, -0.0, F32)):
            got = capi.subpixel_conv(xd, wd, None if bias is None else torch.from_numpy(bias).cuda(), 2)
            blob = _tail_graph((1, 6, 7, cin), 2, 3, residual=False, bias=False if bias is None else bias,
                               weights=w)
            want, _ = _run(blob, [x])
            assert S._same_bits(got.cpu().numpy(), want), cin
            assert not want.any()


@pytest.mark.gpu
def test_gpu_fused_tail_past_2_pow_31_outputs():
    """[1, 6800, 6800, 4] -> [1, 27200, 27200, 3]: 2.22 * 10^9 output floats, past 2^31, in one launch."""
    rng = np.random.default_rng(31)
    shape = (1, 6800, 6800, 4)
    assert 6800 * 6800 * 48 > 2 ** 31
    blob = _tail_graph(shape, 4, 3, img_hw=(7, 9), flags=(False, True), seed=31)
    feeds = [rng.standard_normal(shape, dtype=F32), rng.standard_normal((1, 7, 9, 3), dtype=F32)]
    fused, names = _run(blob, feeds, ("fuse_subpixel_convs",))
    assert names == [FUSED]
    unfused, _ = _run(blob, feeds)
    assert S._same_bits(fused, unfused)


def _graph_run(blob, x, passes, preserve):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    for p in passes:
        getattr(g, p)()
    names = _names(g)
    g.preserve_all_tensors(preserve)
    g.resize_input(g.inputs()[0], x.shape)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    out = g.read(g.outputs()[0])
    g.close()
    return out, names


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [2, 3, 4])
def test_gpu_binary_srnet_fused_equals_unfused(scale):
    for batch, image, preserve, input_type in ((4, (36, 52), True, "float32"), (16, (180, 320), False, "int8")):
        blob = zoo.binary_srnet(batch=1, image=image, scale=scale, seed=scale, input_type=input_type)
        x = np.random.default_rng(batch).standard_normal((batch,) + image + (3,), dtype=F32)
        if input_type == "int8":
            x = zoo.quantize_images(x)
        fused, names = _graph_run(blob, x, ("fuse_all",), preserve)
        assert names[-1] == FUSED
        unfused, names = _graph_run(blob, x, PASSES_BUT_SUBPIXEL, preserve)
        assert names[-4:] == ["builtin:3", "builtin:5", "builtin:23", "builtin:0"]
        assert fused.shape == (batch, scale * image[0], scale * image[1], 3)
        assert S._same_bits(fused, unfused), (batch, image)
        assert np.isfinite(fused).all() and fused.std() > 0


@pytest.mark.gpu
@pytest.mark.parametrize("fuse", [True, False])
def test_gpu_binary_srnet_does_not_depend_on_the_arena(fuse):
    import test_arena_independence as A
    blob = zoo.binary_srnet(batch=1, seed=0, image=(24, 40), scale=3)
    fails = A.check_arena_independence(blob, (A.BATCH, 24, 40, 3), "float32", fuse=fuse)
    assert not fails, "binary_srnet:\n" + "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("batch_size", [3, 5])
def test_gpu_interpreter_predict_over_mini_batches(batch_size):
    from compute_engine_b200.interpreter import Interpreter
    blob = zoo.binary_srnet(batch=1, image=(20, 28), seed=2, input_type="int8", scale=2)
    x = zoo.quantize_images(np.random.default_rng(1).standard_normal((11, 20, 28, 3), dtype=F32))
    want, _ = _graph_run(blob, x, ("fuse_all",), False)
    it = Interpreter(blob, batch_size=batch_size)
    got = it.predict(x)
    it.close()
    assert S._same_bits(np.asarray(got), want)
