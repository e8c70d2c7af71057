"""Binary segmentation graphs: the RESIZE_NEAREST_NEIGHBOR and RESIZE_BILINEAR builtins
(lce_b200_f32_resize_nearest / _bilinear), the decoder merge RESIZE_NEAREST_NEIGHBOR -> ADD [->
LceQuantize] in one pass (lce_b200_f32_upsample_add_sign, Graph::FuseUpsampleMerges) and the zoo's
quicknet_seg.

CPU: the zoo model and its option fields, the CPU reference, the host's Prepare and refusals, the
fused node list and each fusion precondition, the other models' node lists, the new kernels' build.
GPU: both builtins bit for bit against a numpy float32 restatement of TFLite's reference kernels, the
merge kernel against the op sequence, the whole graph fused vs unfused and op by op against the CPU,
arena independence and CUDA-graph replay, and Interpreter.predict over mini-batches."""
import collections
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

MERGE = "RESIZE_NEAREST_NEIGHBOR+ADD"
F32 = np.float32


# ----------------------- CPU reference of the new ops ----------------------- #
def _scale(n_in, n_out, align_corners):
    if align_corners and n_out > 1:
        return F32(n_in - 1) / F32(n_out - 1)
    return F32(n_in) / F32(n_out)


def nearest_index(n_in, n_out, align_corners, half_pixel_centers):
    """GetNearestNeighbor (reference/resize_nearest_neighbor.h) for every output index."""
    v = (np.arange(n_out, dtype=F32) + F32(0.5 if half_pixel_centers else 0.0)) * _scale(n_in, n_out, align_corners)
    v = v.astype(F32)
    if align_corners:   # TfLiteRound: halves away from zero
        s = (np.sign(v) * np.floor(np.abs(v.astype(np.float64)) + 0.5)).astype(np.int64)
    else:
        s = np.floor(v).astype(np.int64)
    s = np.minimum(s, n_in - 1)
    return np.maximum(s, 0) if half_pixel_centers else s


def resize_nearest_ref(x, size, align_corners=False, half_pixel_centers=False):
    iy = nearest_index(x.shape[1], size[0], align_corners, half_pixel_centers)
    ix = nearest_index(x.shape[2], size[1], align_corners, half_pixel_centers)
    return np.ascontiguousarray(x[:, iy][:, :, ix])


def _bilinear_axis(n_in, n_out, align_corners, half_pixel_centers):
    """ComputeInterpolationValues (reference/resize_bilinear.h): v, lo, hi per output index."""
    o, sc = np.arange(n_out, dtype=F32), _scale(n_in, n_out, align_corners)
    v = ((o + F32(0.5)).astype(F32) * sc).astype(F32) - F32(0.5) if half_pixel_centers else o * sc
    v = v.astype(F32)
    lo = np.maximum(np.floor(v).astype(np.int64), 0)
    hi = np.minimum(np.ceil(v).astype(np.int64), n_in - 1)
    return v, lo, hi


def resize_bilinear_ref(x, size, align_corners=False, half_pixel_centers=False):
    vy, y0, y1 = _bilinear_axis(x.shape[1], size[0], align_corners, half_pixel_centers)
    vx, x0, x1 = _bilinear_axis(x.shape[2], size[1], align_corners, half_pixel_centers)
    dy = (vy - y0.astype(F32)).astype(F32)[None, :, None, None]
    dx = (vx - x0.astype(F32)).astype(F32)[None, None, :, None]
    ey, ex = (F32(1) - dy).astype(F32), (F32(1) - dx).astype(F32)

    def at(iy, ix):
        return x[:, iy][:, :, ix]

    with np.errstate(all="ignore"):
        s = ((at(y0, x0) * ey).astype(F32) * ex).astype(F32)
        s = (s + ((at(y1, x0) * dy).astype(F32) * ex).astype(F32)).astype(F32)
        s = (s + ((at(y0, x1) * ey).astype(F32) * dx).astype(F32)).astype(F32)
        s = (s + ((at(y1, x1) * dy).astype(F32) * dx).astype(F32)).astype(F32)
    return s


def _resize_flags(model, op):
    o = op["options"]
    if op["code"] == 23:
        return bool(o.scalar(2, "b")), bool(o.scalar(3, "b"))
    return bool(o.scalar(0, "b")), bool(o.scalar(1, "b"))


def _run_op(model, op, vals):
    """One op of a parsed model on the CPU: the resizes here, every other op through tflite_ref."""
    if op["code"] in (23, 97):
        size = model["tensors"][op["inputs"][1]]["data"]
        fn = resize_bilinear_ref if op["code"] == 23 else resize_nearest_ref
        return fn(vals[op["inputs"][0]], (int(size[0]), int(size[1])), *_resize_flags(model, op))
    act = [i for i in op["inputs"] if i >= 0 and model["tensors"][i]["data"] is None]
    sub = {"tensors": model["tensors"], "ops": [op], "inputs": act, "outputs": [op["outputs"][0]]}
    return R.run(sub, [vals[i] for i in act])[0][0]


def _run_model(model, inputs):
    vals = dict(zip(model["inputs"], inputs))
    for op in model["ops"]:
        vals[op["outputs"][0]] = _run_op(model, op, vals)
    return [vals[i] for i in model["outputs"]]


# ---------------------------- small test graphs ---------------------------- #
def _resize_graph(kind, in_shape, size, align_corners=False, half_pixel_centers=False, size_const=True,
                  size_dtype=np.int32, in_dtype=np.float32):
    m = TFLiteModel()
    x = m.add_tensor("x", in_shape, in_dtype)
    if size_const:
        s = m.add_tensor("size", None, size_dtype, data=np.array(size, size_dtype))
        inputs = [x]
    else:
        s = m.add_tensor("size", (2,), np.int32)
        inputs = [x, s]
    y = m.add_tensor("y", (in_shape[0], max(size[0], 1), max(size[1], 1), in_shape[3]), in_dtype)
    m.add_op(kind, [x, s], [y], align_corners=align_corners, half_pixel_centers=half_pixel_centers)
    m.inputs, m.outputs = inputs, [y]
    return m.serialize()


def _merge_graph(shape=(2, 4, 4, 64), factor=2, act="NONE", v_first=True, sign=True, sum_readers=0,
                 skip_shape=None, resized_output=False, sum_output=False, align_corners=False,
                 half_pixel_centers=True, second_reader=False):
    """u [B,h,w,C] -> RESIZE_NEAREST_NEIGHBOR -> ADD(skip) [-> LceQuantize], with optional extra
    readers of the sum (RELUs), a second reader of the resized map, a broadcast skip."""
    b, h, w, c = shape
    oh, ow = h * factor, w * factor
    m = TFLiteModel()
    u = m.add_tensor("u", shape)
    skip = m.add_tensor("skip", skip_shape or (b, oh, ow, c))
    size = m.add_tensor("size", None, np.int32, data=np.array([oh, ow], np.int32))
    v = m.add_tensor("v", (b, oh, ow, c))
    m.add_op("RESIZE_NEAREST_NEIGHBOR", [u, size], [v], align_corners=align_corners,
             half_pixel_centers=half_pixel_centers)
    s = m.add_tensor("s", (b, oh, ow, c))
    m.add_op("ADD", [v, skip] if v_first else [skip, v], [s], activation=act)
    outs = []
    if sign:
        q = m.add_tensor("q", (b, oh, ow, (c + 31) // 32), np.int32)
        m.add_op("LceQuantize", [s], [q], custom_options=b"")
        outs.append(q)
    for k in range(sum_readers):
        r = m.add_tensor(f"r{k}", (b, oh, ow, c))
        m.add_op("RELU", [s], [r])
        outs.append(r)
    if second_reader:
        r = m.add_tensor("rv", (b, oh, ow, c))
        m.add_op("RELU", [v], [r])
        outs.append(r)
    if resized_output:
        outs.append(v)
    if sum_output:
        outs.append(s)
    m.inputs, m.outputs = [u, skip], outs
    return m.serialize()


def _node_names(blob, fuse="fuse_upsample_merges"):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n = getattr(g, fuse)()
    names = [g.node_name(i) for i in range(g.num_nodes())]
    g.close()
    return n, names


# ----------------------------------- CPU ----------------------------------- #
SEG_COUNTS = {(3, ""): 9, (4, ""): 4, (17, ""): 3, (32, "LceQuantize"): 22, (32, "LceBconv2d"): 22,
              (0, ""): 25, (97, ""): 3, (23, ""): 1}


@pytest.mark.parametrize("image", [224, 64])
@pytest.mark.parametrize("input_type", ["float32", "int8"])
def test_quicknet_seg_op_counts_and_options(image, input_type):
    m = R.parse(zoo.quicknet_seg(batch=1, image=image, input_type=input_type))
    kinds = collections.Counter((o["code"], o["custom"]) for o in m["ops"])
    want = dict(SEG_COUNTS)
    if input_type == "int8":
        want[(6, "")] = 1
    assert kinds == want
    assert m["tensors"][m["outputs"][0]]["shape"] == (1, image, image, 21)
    sizes = []
    for op in m["ops"]:
        if op["code"] in (23, 97):
            assert _resize_flags(m, op) == (False, True)
            sizes.append(tuple(m["tensors"][op["inputs"][1]]["data"]))
            assert m["tensors"][op["inputs"][1]]["dtype"] == np.int32
    s = image // 32
    assert sizes == [(2 * s, 2 * s), (4 * s, 4 * s), (8 * s, 8 * s), (image, image)]


def test_quicknet_seg_is_not_registered_and_refuses_odd_images():
    assert "quicknet_seg" not in zoo.MODELS and zoo.quicknet_seg not in zoo.MODELS.values()
    with pytest.raises(ValueError, match="multiple of 32"):
        zoo.quicknet_seg(image=100)
    m = R.parse(zoo.quicknet_seg(image=64, classes=5, decoder_blocks=1))
    assert m["tensors"][m["outputs"][0]]["shape"] == (1, 64, 64, 5)
    assert sum(o["custom"] == "LceBconv2d" for o in m["ops"]) == 16 + 3


def test_resize_option_fields_read_back():
    for kind, (fa, fh) in (("RESIZE_BILINEAR", (2, 3)), ("RESIZE_NEAREST_NEIGHBOR", (0, 1))):
        for ac, hp in ((False, False), (True, False), (False, True), (True, True)):
            m = R.parse(_resize_graph(kind, (1, 3, 3, 2), (5, 6), ac, hp))
            o = m["ops"][0]["options"]
            assert (bool(o.scalar(fa, "b")), bool(o.scalar(fh, "b"))) == (ac, hp)
            assert m["ops"][0]["code"] == {"RESIZE_BILINEAR": 23, "RESIZE_NEAREST_NEIGHBOR": 97}[kind]


# sha256 prefixes of every registered model's bytes (batch 1, seed 0), as the writer and the zoo
# produced them before the resize ops and quicknet_seg's shared encoder were added
MODEL_HASHES = {
    "binaryalexnet": "150d60007c51b339", "binarydensenet28": "fcb1f3e89ef1bd23",
    "binarydensenet37": "f8d5bc67f8d50711", "binarydensenet37_dilated": "1feab16cddee572d",
    "binarydensenet45": "f73b99c0b8ea8f7f", "birealnet18": "69b00efc25be1c89", "dorefanet": "5edd486e889b1185",
    "meliusnet22": "f2fe2d5101d56c09", "quicknet": "80c00a45aea6e3ba", "quicknet_large": "ae386c9d6e07d995",
    "quicknet_small": "cf5f288f7f182222", "reactnet_a": "37dd82f28895b77a", "realtobinarynet": "d867acd75a420cca",
    "xnornet": "1320cd7cfb60937f",
}


def test_writer_leaves_existing_models_unchanged():
    import hashlib
    assert set(MODEL_HASHES) == set(zoo.MODELS)
    for name, make in zoo.MODELS.items():
        assert hashlib.sha256(make(batch=1, seed=0)).hexdigest()[:16] == MODEL_HASHES[name], name


def test_cpu_reference_runs_quicknet_seg():
    m = R.parse(zoo.quicknet_seg(batch=1, image=64, seed=2))
    x = np.random.default_rng(0).standard_normal((2, 64, 64, 3)).astype(np.float32)
    out = _run_model(m, [x])[0]
    assert out.shape == (2, 64, 64, 21) and np.isfinite(out).all() and out.std() > 0


def test_resize_refs_on_known_values():
    x = np.arange(2 * 3 * 3, dtype=F32).reshape(1, 3, 3, 2)
    assert np.array_equal(resize_nearest_ref(x, (6, 6), False, True), x.repeat(2, 1).repeat(2, 2))
    assert np.array_equal(resize_bilinear_ref(x, (3, 3)), x)
    # align_corners maps the corners onto each other
    y = resize_bilinear_ref(x, (5, 5), True, False)
    assert np.array_equal(y[:, ::2, ::2], x)
    # half_pixel_centers upscaling extrapolates at the border from the clamped lower neighbour:
    # vy = -0.25 gives the weights 1.25 and -0.25 on row 0
    a = F32(0.1)
    z = resize_bilinear_ref(np.array([a, 4], F32).reshape(1, 2, 1, 1), (4, 1), False, True)
    assert z[0, 0, 0, 0] == (a * F32(1.25)) + (a * F32(-0.25)) and z[0, 3, 0, 0] == F32(4.0)


@pytest.mark.parametrize("kind", ["RESIZE_BILINEAR", "RESIZE_NEAREST_NEIGHBOR"])
@pytest.mark.parametrize("in_hw,size", [((7, 7), (14, 14)), ((7, 7), (3, 2)), ((1, 1), (1, 1)),
                                        ((13, 17), (30, 11)), ((4, 6), (1, 1))])
def test_host_prepares_resize_shapes(kind, in_hw, size):
    blob = _resize_graph(kind, (2,) + in_hw + (5,), size, half_pixel_centers=True)
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (2,) + size + (5,)
    g.resize_input(g.inputs()[0], (3,) + in_hw + (5,))   # the batch follows the input's
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (3,) + size + (5,)
    g.close()


@pytest.mark.parametrize("kind", ["RESIZE_BILINEAR", "RESIZE_NEAREST_NEIGHBOR"])
@pytest.mark.parametrize("case,message", [
    ("dynamic size", "size must be a constant int32"),
    ("zero size", "size must be positive"),
    ("negative size", "size must be positive"),
    ("3-D input", "input must be a 4-D float32"),
    ("int32 input", "input must be a 4-D float32"),
    ("both flags", "align_corners and half_pixel_centers"),
])
def test_host_refuses_resize(kind, case, message):
    shape, size, kw = (1, 4, 4, 3), (8, 8), {}
    if case == "dynamic size":
        kw["size_const"] = False
    elif case == "zero size":
        size = (0, 8)
    elif case == "negative size":
        size = (8, -2)
    elif case == "3-D input":
        shape = (4, 4, 3)
    elif case == "int32 input":
        kw["in_dtype"] = np.int32
    else:
        kw.update(align_corners=True, half_pixel_centers=True)
    if case == "3-D input":
        m = TFLiteModel()
        x = m.add_tensor("x", shape)
        s = m.add_tensor("size", None, np.int32, data=np.array(size, np.int32))
        y = m.add_tensor("y", (8, 8, 3))
        m.add_op(kind, [x, s], [y])
        m.inputs, m.outputs = [x], [y]
        blob = m.serialize()
    else:
        blob = _resize_graph(kind, shape, size, **kw)
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    if case == "both flags" and kind == "RESIZE_NEAREST_NEIGHBOR":
        g.allocate_tensors()   # TFLite's nearest-neighbour Prepare takes both flags
    else:
        with pytest.raises(H.HostError, match=message):
            g.allocate_tensors()
    g.close()


def test_quicknet_seg_prepares_on_the_host():
    blob = zoo.quicknet_seg(batch=2, image=64, seed=1)
    m = R.parse(blob)
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    assert g.num_nodes() == len(m["ops"])
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (2, 64, 64, 21)
    g.close()


SEG_FUSED = [
    "DEQUANTIZE+CONV_2D+DEPTHWISE_CONV_2D", "CONV_2D+LceQuantize",
    "LceBconv2d+ADD+LceBconv2d+ADD+LceQuantize", "LceBconv2d+ADD+LceBconv2d+ADD",
    "MAX_POOL_2D+DEPTHWISE_CONV_2D", "CONV_2D+LceQuantize",
    "LceBconv2d+ADD+LceBconv2d+ADD+LceQuantize", "LceBconv2d+ADD+LceBconv2d+ADD",
    "MAX_POOL_2D+DEPTHWISE_CONV_2D", "CONV_2D+LceQuantize",
    "LceBconv2d+ADD+LceQuantize", "LceBconv2d+ADD+LceQuantize", "LceBconv2d+ADD+LceQuantize", "LceBconv2d+ADD",
    "MAX_POOL_2D+DEPTHWISE_CONV_2D", "CONV_2D+LceQuantize",
    "LceBconv2d+ADD+LceQuantize", "LceBconv2d+ADD+LceQuantize", "LceBconv2d+ADD+LceQuantize", "LceBconv2d+ADD",
    # decoder: 14x14x256 (no pair), 28x28x128 and 56x56x64 (paired), then the head
    "builtin:3", MERGE + "+LceQuantize", "LceBconv2d+ADD+LceQuantize", "LceBconv2d+ADD",
    "builtin:3", MERGE + "+LceQuantize", "LceBconv2d+ADD+LceBconv2d+ADD",
    "builtin:3", MERGE + "+LceQuantize", "LceBconv2d+ADD+LceBconv2d+ADD",
    "builtin:3", "builtin:23",
]


def test_quicknet_seg_fused_node_list():
    g = H.HostGraph.from_tflite(zoo.quicknet_seg(batch=2, image=224, seed=1, input_type="int8"),
                                device_arena=True)
    n0 = g.num_nodes()
    removed = g.fuse_all()
    assert [g.node_name(i) for i in range(g.num_nodes())] == SEG_FUSED
    assert g.num_nodes() == n0 - removed
    # each merge stores the sum, the first decoder block's shortcut
    for i in range(g.num_nodes()):
        if g.node_name(i).startswith(MERGE):
            outs = g.node_outputs(i)
            assert len(outs) == 2 and outs[0] >= 0
    g.close()
    # without the pass the merges stay three ops each
    g = H.HostGraph.from_tflite(zoo.quicknet_seg(batch=2, image=224, seed=1, input_type="int8"),
                                device_arena=True)
    assert g.fuse_upsample_merges() == 6
    g.close()


def test_merge_fuses_with_and_without_the_sign_tail():
    assert _node_names(_merge_graph()) == (2, [MERGE + "+LceQuantize"])
    assert _node_names(_merge_graph(sign=False, sum_readers=1)) == (1, [MERGE, "builtin:19"])
    assert _node_names(_merge_graph(v_first=False, act="RELU")) == (2, [MERGE + "+LceQuantize"])
    # the sum is stored only when something else reads it or it is a graph output
    for kw, stored in (({}, False), ({"sum_readers": 1}, True), ({"sum_output": True}, True)):
        g = H.HostGraph.from_tflite(_merge_graph(**kw), device_arena=True)
        g.fuse_upsample_merges()
        assert (g.node_outputs(0)[0] >= 0) == stored, kw
        g.close()


@pytest.mark.parametrize("variant", ["second reader", "broadcast skip", "C % 32", "resized map output",
                                     "host arena"])
def test_merge_fusion_leaves_the_graph_when_a_precondition_fails(variant):
    if variant == "second reader":
        blob = _merge_graph(second_reader=True)
    elif variant == "broadcast skip":
        blob = _merge_graph(skip_shape=(64,))
    elif variant == "C % 32":   # the fusion stops at the ADD
        blob = _merge_graph(shape=(2, 4, 4, 48))
        assert _node_names(blob) == (1, [MERGE, "LceQuantize"])
        return
    elif variant == "resized map output":
        blob = _merge_graph(resized_output=True)
    else:
        g = H.HostGraph.from_tflite(_merge_graph(), device_arena=False)
        assert g.fuse_upsample_merges() == 0
        g.close()
        return
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    before = [g.node_name(i) for i in range(g.num_nodes())]
    assert g.fuse_upsample_merges() == 0
    assert [g.node_name(i) for i in range(g.num_nodes())] == before
    g.close()


def _other_models():
    import test_arena_independence as A
    cases = {name: (zoo.MODELS[name], {}) for name in zoo.MODELS}
    cases.update(A.FAMILIES)
    return cases


@pytest.mark.parametrize("case", sorted(_other_models()))
def test_other_models_keep_their_node_lists(case):
    make, kw = _other_models()[case]
    blob = make(batch=1, seed=0, image=224, **kw)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.fuse_all()
    after = [g.node_name(i) for i in range(g.num_nodes())]
    assert g.fuse_upsample_merges() == 0
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n0 = g.num_nodes()
    assert g.fuse_upsample_merges() == 0 and g.num_nodes() == n0
    g.close()
    assert not any("RESIZE" in n for n in after)


def test_resize_kernels_compile_without_spills(tmp_path):
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
    props = re.findall(r"Function properties for (\S*(?:resize_nearest|resize_bilinear|upsample_add_sign)\S*)\n"
                       r"\s*(.*)", r.stderr)
    assert len(props) == 5, r.stderr   # float and float4 rows per resize, and the merge
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)


# ----------------------------------- GPU ----------------------------------- #
def _same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


FLAGS = {"bilinear": [(False, False), (True, False), (False, True)],
         "nearest": [(False, False), (True, False), (False, True), (True, True)]}
RESIZE_CASES = [(op, ac, hp, c) for op in FLAGS for ac, hp in FLAGS[op] for c in (1, 3, 21, 64, 256)]


def _sizes(h, w):
    return [(2 * h, 2 * w), (4 * h, 4 * w), (h * 5 // 2 + 1, w * 7 // 3 + 2), (max(1, h // 2), max(1, w // 3)),
            (1, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("op,align_corners,half_pixel_centers,c", RESIZE_CASES)
def test_gpu_resize_matches_the_reference(op, align_corners, half_pixel_centers, c):
    import torch
    from compute_engine_b200 import capi
    rng = np.random.default_rng(c * 7 + align_corners * 2 + half_pixel_centers)
    ref = resize_bilinear_ref if op == "bilinear" else resize_nearest_ref
    border = 0
    for b in (1, 3):
        for h, w in ((1, 1), (7, 7), (13, 17)):
            x = rng.standard_normal((b, h, w, c)).astype(F32)
            xd = torch.from_numpy(x).cuda()
            for size in _sizes(h, w):
                got = capi.resize(xd, size, op == "bilinear", align_corners, half_pixel_centers).cpu().numpy()
                want = ref(x, size, align_corners, half_pixel_centers)
                assert _same_bits(got, want), (b, h, w, size, np.abs(got - want).max())
                if op == "bilinear" and half_pixel_centers:
                    v, _, _ = _bilinear_axis(h, size[0], False, True)
                    border += int((v < 0).any())
    if op == "bilinear" and half_pixel_centers:
        assert border > 0   # the extrapolation at vy < 0 was exercised


@pytest.mark.gpu
@pytest.mark.parametrize("op", ["nearest", "bilinear"])
def test_gpu_resize_past_2_pow_31_output_elements(op):
    """[1, 8, 8, 3] -> [1, 27000, 27000, 3]: 2.19 * 10^9 floats, past 2^31. Three row ranges, the
    first, the middle and the last, are checked against the numpy reference of those rows."""
    import torch
    from compute_engine_b200 import capi
    x = torch.randn((1, 8, 8, 3), device="cuda")
    oh, ow = 27000, 27000
    assert oh * ow * 3 > 2 ** 31
    out = capi.resize(x, (oh, ow), op == "bilinear", False, True)
    xn = x.cpu().numpy()
    iy, ix = nearest_index(8, oh, False, True), nearest_index(8, ow, False, True)
    vy, y0, y1 = _bilinear_axis(8, oh, False, True)
    vx, x0, x1 = _bilinear_axis(8, ow, False, True)
    for rows in (slice(0, 3), slice(oh - 3, oh), slice(13499, 13502)):
        got = out[:, rows].cpu().numpy()
        if op == "nearest":
            want = xn[:, iy[rows]][:, :, ix]
        else:   # resize_bilinear_ref on the selected output rows only
            r = np.arange(oh)[rows]
            dy = (vy[r] - y0[r].astype(F32)).astype(F32)[None, :, None, None]
            dx = (vx - x0.astype(F32)).astype(F32)[None, None, :, None]
            ey, ex = (F32(1) - dy).astype(F32), (F32(1) - dx).astype(F32)

            def at(ry, rx):
                return xn[:, ry][:, :, rx]
            s = ((at(y0[r], x0) * ey).astype(F32) * ex).astype(F32)
            s = (s + ((at(y1[r], x0) * dy).astype(F32) * ex).astype(F32)).astype(F32)
            s = (s + ((at(y0[r], x1) * ey).astype(F32) * dx).astype(F32)).astype(F32)
            want = (s + ((at(y1[r], x1) * dy).astype(F32) * dx).astype(F32)).astype(F32)
        assert _same_bits(got, want), rows
    del out
    torch.cuda.empty_cache()


def _run_graph(blob, feeds, fuse, preserve=True):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    removed = g.fuse_upsample_merges() if fuse else 0
    g.preserve_all_tensors(preserve)
    g.allocate_tensors()
    for t, x in zip(g.inputs(), feeds):
        g.write(t, x)
    g.invoke()
    outs = [g.read(t) for t in g.outputs()]
    names = [g.node_name(i) for i in range(g.num_nodes())]
    g.close()
    return outs, removed, names


MERGE_CASES = [
    dict(act="NONE"), dict(act="RELU"), dict(act="RELU_N1_TO_1"), dict(act="RELU6"),
    dict(act="RELU", v_first=False), dict(v_first=False, sign=False, sum_readers=1),
    dict(sign=False, sum_output=True, act="RELU6"), dict(sum_readers=1), dict(shape=(3, 5, 7, 96)),
    dict(shape=(2, 5, 3, 21), sign=False, sum_readers=1), dict(shape=(2, 4, 4, 48)),
    dict(align_corners=True, half_pixel_centers=False, shape=(1, 5, 6, 32), factor=3),
    dict(align_corners=False, half_pixel_centers=False, shape=(1, 5, 6, 64)),
    dict(align_corners=True, half_pixel_centers=True, shape=(1, 3, 3, 32)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(MERGE_CASES)))
def test_gpu_merge_is_the_op_sequence(case):
    kw = MERGE_CASES[case]
    b, h, w, c = kw.get("shape", (2, 4, 4, 64))
    f = kw.get("factor", 2)
    rng = np.random.default_rng(case)
    u = rng.standard_normal((b, h, w, c)).astype(F32)
    skip = rng.standard_normal((b, h * f, w * f, c)).astype(F32)
    u.reshape(-1)[::7] = -0.0
    skip.reshape(-1)[::11] = 0.0
    blob = _merge_graph(**kw)
    want, _, _ = _run_graph(blob, [u, skip], False)
    got, removed, names = _run_graph(blob, [u, skip], True)
    assert removed >= 1 and names[0].startswith(MERGE)
    for a, bb in zip(want, got):
        assert _same_bits(a, bb)


@pytest.mark.gpu
@pytest.mark.parametrize("stored", [True, False])
def test_gpu_merge_at_the_full_decoder_shape(stored):
    """The 56 x 56 x 64 merge at batch 256, against the unfused ops; the sum stored or not."""
    shape = (256, 28, 28, 64)
    rng = np.random.default_rng(5)
    u = rng.standard_normal(shape).astype(F32)
    skip = rng.standard_normal((256, 56, 56, 64)).astype(F32)
    blob = _merge_graph(shape=shape, sum_readers=1 if stored else 0)
    want, _, _ = _run_graph(blob, [u, skip], False, preserve=False)
    got, removed, _ = _run_graph(blob, [u, skip], True, preserve=False)
    assert removed == 2
    for a, bb in zip(want, got):
        assert _same_bits(a, bb)


@pytest.mark.gpu
def test_gpu_quicknet_seg_fused_equals_unfused():
    blob = zoo.quicknet_seg(batch=1, image=224, seed=4, input_type="int8")
    outs = {}
    for batch, preserve in ((4, True), (256, False)):
        x = zoo.quantize_images(np.random.default_rng(batch).standard_normal((batch, 224, 224, 3), dtype=F32))
        for fuse in (False, True):
            g = H.HostGraph.from_tflite(blob, device_arena=True)
            if fuse:
                assert g.fuse_all() > 0
                assert sum(g.node_name(i).startswith(MERGE) for i in range(g.num_nodes())) == 3
            g.preserve_all_tensors(preserve)
            g.resize_input(g.inputs()[0], x.shape)
            g.allocate_tensors()
            g.write(g.inputs()[0], x)
            g.invoke()
            outs[(batch, fuse)] = g.read(g.outputs()[0])
            g.close()
        assert outs[(batch, True)].shape == (batch, 224, 224, 21)
        assert np.isfinite(outs[(batch, True)]).all()
        assert _same_bits(outs[(batch, False)], outs[(batch, True)]), batch


@pytest.mark.gpu
def test_gpu_quicknet_seg_op_by_op():
    """The unfused graph on the device, op by op on the device's own inputs: the resizes, the ADDs
    that merge, and every LCE op bit exact; the other float builtins within the torch fp32
    reference's tolerance; then the logits against the CPU graph."""
    blob = zoo.quicknet_seg(batch=1, image=64, seed=9)
    m = R.parse(blob)
    x = np.random.default_rng(3).standard_normal((3, 64, 64, 3)).astype(F32)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.preserve_all_tensors(True)
    g.resize_input(g.inputs()[0], x.shape)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    exact = collections.Counter()
    for op in m["ops"]:
        act = [i for i in op["inputs"] if i >= 0 and m["tensors"][i]["data"] is None]
        want = _run_op(m, op, {i: g.read(i) for i in act})
        got = g.read(op["outputs"][0])
        assert got.shape == want.shape, (op["code"], op["custom"])
        if op["code"] in (0, 23, 32, 97):
            assert _same_bits(got, want.astype(got.dtype)), (op["code"], op["custom"])
            exact[op["custom"] or op["code"]] += 1
        else:
            scale = max(1.0, float(np.abs(want).max()))
            assert np.allclose(got, want, rtol=1e-4, atol=1e-5 * scale), (op["code"], np.abs(got - want).max())
    assert exact == {"LceBconv2d": 22, "LceQuantize": 22, 0: 25, 97: 3, 23: 1}
    got_out = g.read(g.outputs()[0])
    want_out = _run_model(m, [x])[0]
    assert np.abs(got_out - want_out).max() <= 1e-3 * max(1.0, float(np.abs(want_out).max()))
    g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fuse", [True, False])
def test_gpu_quicknet_seg_does_not_depend_on_the_arena(fuse):
    import test_arena_independence as A
    blob = zoo.quicknet_seg(batch=1, seed=0, image=224)
    fails = A.check_arena_independence(blob, (A.BATCH, 224, 224, 3), "float32", fuse=fuse)
    assert not fails, "quicknet_seg:\n" + "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("batch_size", [3, 5])
def test_gpu_interpreter_predict_over_mini_batches(batch_size):
    from compute_engine_b200.interpreter import Interpreter
    blob = zoo.quicknet_seg(batch=1, image=64, seed=2, input_type="int8")
    x = zoo.quantize_images(np.random.default_rng(1).standard_normal((11, 64, 64, 3), dtype=F32))
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
    assert _same_bits(np.asarray(got), want)
