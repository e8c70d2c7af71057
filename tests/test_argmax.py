"""Segmentation graphs that end in ARG_MAX: the ARG_MAX builtin (lce_b200_f32_argmax), the head's
RESIZE_BILINEAR -> ARG_MAX in one pass (lce_b200_f32_resize_bilinear_argmax, Graph::FuseResizeArgmax)
and the zoo's quicknet_seg(labels=...).

CPU: the writer's and reader's output_type, the zoo model's ops and unchanged default bytes, the host's
Prepare shapes and refusals, the fused node list and each fusion precondition, the other models' node
lists, the new kernels' build.
GPU: ARG_MAX bit for bit against a numpy restatement of TFLite's sequential loop (not np.argmax, which
treats NaN differently), the fused kernel against RESIZE_BILINEAR then ARG_MAX, the whole graph fused
vs unfused and against TFLite's rule on the logits, arena independence and CUDA-graph replay, and
Interpreter.predict over mini-batches."""
import collections
import hashlib
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

FUSED = "RESIZE_BILINEAR+ARG_MAX"
F32 = np.float32

# fuse_all's passes but fuse_resize_argmax, in fuse_all's order
PASSES_BUT_ARGMAX = ("fuse_binary_bases", "fuse_dense_blocks", "fuse_residual_blocks", "fuse_spatial_scales",
                     "fuse_float_glue", "fuse_upsample_merges", "fuse_grouped_conv_affine",
                     "fuse_quantized_activations", "fuse_pooled_signs", "fuse_channel_gates",
                     "fuse_activation_chains", "fuse_residual_pairs")


def argmax_ref(x, axis):
    """TFLite's ArgMinMax with std::greater (reference/arg_min_max.h), restated: v = x[0], idx = 0,
    then x[i] is taken only when x[i] > v, for every position at once."""
    x = np.moveaxis(np.asarray(x), axis, -1)
    v = x[..., 0].copy()
    idx = np.zeros(v.shape, np.int64)
    with np.errstate(invalid="ignore"):
        for i in range(1, x.shape[-1]):
            take = x[..., i] > v
            v = np.where(take, x[..., i], v)
            idx = np.where(take, i, idx)
    return idx


# ---------------------------- small test graphs ---------------------------- #
def _argmax_graph(in_shape, axis, axis_dtype=np.int32, axis_shape=(), output_type=np.int64, out_dtype=None,
                  axis_const=True, in_dtype=np.float32):
    m = TFLiteModel()
    x = m.add_tensor("x", in_shape, in_dtype)
    inputs = [x]
    if axis_const:
        a = m.add_tensor("axis", None, axis_dtype, data=np.array(axis, axis_dtype).reshape(axis_shape))
        m.tensors[a]["shape"] = tuple(axis_shape)   # the writer keeps data at least 1-D
    else:
        a = m.add_tensor("axis", (1,), axis_dtype)
        inputs.append(a)
    r = len(in_shape)
    k = axis + r if isinstance(axis, int) and -r <= axis < 0 else axis
    out_shape = tuple(d for j, d in enumerate(in_shape) if j != k)
    y = m.add_tensor("y", out_shape, out_dtype or output_type)
    m.add_op("ARG_MAX", [x, a], [y], output_type=output_type)
    m.inputs, m.outputs = inputs, [y]
    return m.serialize()


def _head_graph(shape=(2, 7, 7, 21), size=(28, 28), axis=-1, flags=(False, True), output_type=np.int64,
                second_reader=False, resized_output=False, nearest=False):
    """x -> RESIZE_BILINEAR (or RESIZE_NEAREST_NEIGHBOR) -> v -> ARG_MAX(axis) -> labels."""
    b, h, w, c = shape
    m = TFLiteModel()
    x = m.add_tensor("x", shape)
    s = m.add_tensor("size", None, np.int32, data=np.array(size, np.int32))
    v = m.add_tensor("v", (b,) + tuple(size) + (c,))
    m.add_op("RESIZE_NEAREST_NEIGHBOR" if nearest else "RESIZE_BILINEAR", [x, s], [v],
             align_corners=flags[0], half_pixel_centers=flags[1])
    a = m.add_tensor("axis", None, np.int32, data=np.array(axis, np.int32))
    k = axis % 4
    labels = m.add_tensor("labels", tuple(d for j, d in enumerate((b,) + tuple(size) + (c,)) if j != k),
                          output_type)
    m.add_op("ARG_MAX", [v, a], [labels], output_type=output_type)
    outs = [labels]
    if second_reader:
        r = m.add_tensor("r", (b,) + tuple(size) + (c,))
        m.add_op("RELU", [v], [r])
        outs.append(r)
    if resized_output:
        outs.append(v)
    m.inputs, m.outputs = [x], outs
    return m.serialize()


def _names(g):
    return [g.node_name(i) for i in range(g.num_nodes())]


# ----------------------------------- CPU ----------------------------------- #
@pytest.mark.parametrize("output_type,code", [(np.int32, 2), (np.int64, 4), (np.float32, 0)])
def test_output_type_reads_back(output_type, code):
    m = R.parse(_argmax_graph((3, 5), -1, output_type=output_type))
    assert m["ops"][0]["code"] == 56
    assert m["ops"][0]["options"].scalar(0, "b") == code


@pytest.mark.parametrize("labels", ["int64", "int32"])
@pytest.mark.parametrize("image", [224, 64])
def test_quicknet_seg_labels_op_counts_and_output(labels, image):
    m = R.parse(zoo.quicknet_seg(batch=2, image=image, labels=labels))
    kinds = collections.Counter((o["code"], o["custom"]) for o in m["ops"])
    assert kinds == {**S.SEG_COUNTS, (56, ""): 1}
    out = m["tensors"][m["outputs"][0]]
    assert out["shape"] == (2, image, image) and np.dtype(out["dtype"]) == np.dtype(labels)
    op = m["ops"][-1]
    assert op["code"] == 56 and op["options"].scalar(0, "b") == {"int32": 2, "int64": 4}[labels]
    axis = m["tensors"][op["inputs"][1]]
    assert np.dtype(axis["dtype"]) == np.int32 and axis["shape"] == (1,) and int(axis["data"][0]) == -1
    assert m["ops"][-2]["code"] == 23 and m["ops"][-2]["outputs"][0] == op["inputs"][0]
    with pytest.raises(ValueError, match="labels"):
        zoo.quicknet_seg(image=64, labels="float32")


# sha256 prefixes of quicknet_seg's bytes before the labels option was added
SEG_HASHES = [
    (dict(), "78928c3a80260d6f"),
    (dict(batch=1, seed=0, image=224, input_type="int8"), "8a2bf21b7bb0f0cb"),
    (dict(batch=2, seed=1, image=64), "63c2b6b956b15300"),
    (dict(image=64, classes=5, decoder_blocks=1, seed=3), "74d39132392ffa51"),
]


def test_quicknet_seg_default_bytes_are_unchanged():
    for kw, digest in SEG_HASHES:
        assert hashlib.sha256(zoo.quicknet_seg(**kw)).hexdigest()[:16] == digest, kw
        assert zoo.quicknet_seg(**kw, labels=None) == zoo.quicknet_seg(**kw)


@pytest.mark.parametrize("in_shape,axis,axis_dtype,axis_shape,out_shape", [
    ((2, 5, 6, 21), -1, np.int32, (), (2, 5, 6)),
    ((2, 5, 6, 21), 3, np.int64, (1,), (2, 5, 6)),
    ((2, 5, 6, 21), 0, np.int32, (1,), (5, 6, 21)),
    ((2, 5, 6, 21), -3, np.int64, (), (2, 6, 21)),
    ((2, 5, 6, 21), 2, np.int32, (), (2, 5, 21)),
    ((4, 1000), 1, np.int32, (), (4,)),
    ((4, 1000), -2, np.int64, (1,), (1000,)),
    ((3, 7, 9), 1, np.int32, (), (3, 9)),
    ((17,), 0, np.int32, (), ()),
    ((17,), 0, np.int64, (), ()),
    ((17,), -1, np.int64, (1,), ()),
])
@pytest.mark.parametrize("output_type", [np.int32, np.int64])
def test_host_prepares_argmax_shapes(in_shape, axis, axis_dtype, axis_shape, out_shape, output_type):
    blob = _argmax_graph(in_shape, axis, axis_dtype, axis_shape, output_type)
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    g.allocate_tensors()
    out = g.outputs()[0]
    assert g.shape(out) == out_shape
    assert np.dtype(g.dtype(out)) == np.dtype(output_type)
    g.close()


@pytest.mark.parametrize("case,message", [
    ("int32 input", "input must be a float32 tensor"),
    ("int8 input", "input must be a float32 tensor"),
    ("dynamic axis", "axis must be a constant tensor"),
    ("float axis", "axis must be int32 or int64"),
    ("two-element axis", "axis must have exactly one element"),
    ("[1, 1] axis", "axis must have exactly one element"),
    ("axis too large", "axis is out of range"),
    ("axis too small", "axis is out of range"),
    ("empty axis", "reduced axis is empty"),
    ("float32 output_type", "output_type must be int32 or int64"),
    ("output type differs", "output tensor's type differs from output_type"),
])
def test_host_refuses_argmax(case, message):
    kw = {}
    shape, axis = (2, 5, 21), -1
    if case == "int32 input":
        kw["in_dtype"] = np.int32
    elif case == "int8 input":
        kw["in_dtype"] = np.int8
    elif case == "dynamic axis":
        kw["axis_const"] = False
    elif case == "float axis":
        kw["axis_dtype"] = np.float32
    elif case == "two-element axis":
        axis, kw["axis_shape"] = [2, 2], (2,)
    elif case == "[1, 1] axis":
        kw["axis_shape"] = (1, 1)
    elif case == "axis too large":
        axis = 3
    elif case == "axis too small":
        axis = -4
    elif case == "empty axis":
        shape, axis = (2, 0, 21), 1
    elif case == "float32 output_type":
        kw.update(output_type=np.float32, out_dtype=np.int64)
    else:
        kw.update(output_type=np.int64, out_dtype=np.int32)
    blob = _argmax_graph(shape, axis, **kw)
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    with pytest.raises(H.HostError, match=re.escape(message)):
        g.allocate_tensors()
    g.close()


def test_quicknet_seg_labels_loads_and_prepares_on_the_host():
    blob = zoo.quicknet_seg(batch=2, image=64, seed=1, labels="int64")
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    assert g.num_nodes() == len(R.parse(blob)["ops"])
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (2, 64, 64)
    g.close()


@pytest.mark.parametrize("labels", ["int64", "int32"])
def test_quicknet_seg_labels_fused_node_list(labels):
    blob = zoo.quicknet_seg(batch=2, image=224, seed=1, input_type="int8", labels=labels)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n0 = g.num_nodes()
    removed = g.fuse_all()
    assert _names(g) == S.SEG_FUSED[:-1] + [FUSED]
    assert g.num_nodes() == n0 - removed
    g.close()
    # fuse_all's other passes leave the head as two ops, and the pass alone removes the resize
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    for p in PASSES_BUT_ARGMAX:
        getattr(g, p)()
    assert _names(g) == S.SEG_FUSED + ["builtin:56"]
    assert g.fuse_resize_argmax() == 1
    assert _names(g) == S.SEG_FUSED[:-1] + [FUSED]
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    assert g.fuse_resize_argmax() == 1 and g.num_nodes() == n0 - 1
    assert _names(g)[-1] == FUSED
    g.close()


def test_head_fuses_for_every_flag_combination():
    for flags in S.FLAGS["bilinear"]:
        g = H.HostGraph.from_tflite(_head_graph(flags=flags), device_arena=True)
        assert g.fuse_resize_argmax() == 1 and _names(g) == [FUSED]
        ins, outs = g.node_io(0)
        assert len(ins) == 3 and ins[0] == g.inputs()[0] and outs == g.outputs()
        g.close()
    # the widest source row the kernel stages still fuses
    c = 21
    w = _max_row_floats() // c
    g = H.HostGraph.from_tflite(_head_graph(shape=(1, 2, w, c), size=(4, 2 * w)), device_arena=True)
    assert g.fuse_resize_argmax() == 1
    g.close()


def _max_row_floats():
    from compute_engine_b200 import capi
    return capi.resize_bilinear_argmax_max_row_floats()


@pytest.mark.parametrize("variant", ["second reader", "resized map output", "axis not channels", "rows too wide",
                                     "nearest", "host arena"])
def test_fusion_leaves_the_graph_when_a_precondition_fails(variant):
    if variant == "second reader":
        blob = _head_graph(second_reader=True)
    elif variant == "resized map output":
        blob = _head_graph(resized_output=True)
    elif variant == "axis not channels":
        blob = _head_graph(axis=2)
    elif variant == "rows too wide":
        c = 21
        w = _max_row_floats() // c + 1
        blob = _head_graph(shape=(1, 2, w, c), size=(4, 2 * w))
    elif variant == "nearest":
        blob = _head_graph(nearest=True)
    else:
        g = H.HostGraph.from_tflite(_head_graph(), device_arena=False)
        assert g.fuse_resize_argmax() == 0
        g.close()
        return
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    before = _names(g)
    assert g.fuse_resize_argmax() == 0
    assert _names(g) == before
    g.close()


@pytest.mark.parametrize("case", sorted(S._other_models()))
def test_other_models_keep_their_node_lists(case):
    make, kw = S._other_models()[case]
    blob = make(batch=1, seed=0, image=224, **kw)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n0 = g.num_nodes()
    assert g.fuse_resize_argmax() == 0 and g.num_nodes() == n0
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.fuse_all()
    after = _names(g)
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    for p in PASSES_BUT_ARGMAX:
        getattr(g, p)()
    assert _names(g) == after
    g.close()


def test_quicknet_seg_logits_keep_their_node_list():
    g = H.HostGraph.from_tflite(zoo.quicknet_seg(batch=2, image=224, seed=1, input_type="int8"),
                                device_arena=True)
    g.fuse_all()
    assert _names(g) == S.SEG_FUSED
    g.close()


def test_argmax_kernels_compile_without_spills(tmp_path):
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
    props = re.findall(r"Function properties for (\S*argmax\S*)\n\s*(.*)", r.stderr)
    # argmax_kernel, argmax_warp_kernel and bilinear_argmax_kernel, each for int32 and int64 labels
    assert len(props) == 6, r.stderr
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)


# ----------------------------------- GPU ----------------------------------- #
def _adversarial(rng, shape):
    """Values drawn from a few exact levels, ±0.0, ±inf and NaN, so rows hold ties, signed zeros,
    infinities, NaN at index 0 and NaN elsewhere."""
    levels = np.array([-np.inf, -1.5, -0.0, 0.0, 0.5, 1.5, np.inf, np.nan], F32)
    p = np.array([0.05, 0.2, 0.1, 0.1, 0.2, 0.2, 0.05, 0.1])
    x = rng.choice(levels, size=shape, p=p).astype(F32)
    x.flat[0] = np.nan   # index 0 along every axis
    return x


ARGMAX_SHAPES = [(7,), (1000,), (5, 21), (3, 1000), (6, 63), (6, 64), (4, 6, 5), (2, 3, 4, 21), (3, 2, 5, 64),
                 (2, 2, 1000, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ARGMAX_SHAPES)
@pytest.mark.parametrize("dtype", ["int64", "int32"])
def test_gpu_argmax_matches_tflites_loop(shape, dtype):
    import torch
    from compute_engine_b200 import capi
    rng = np.random.default_rng(len(shape) * 1000 + shape[-1])
    tdt = getattr(torch, dtype)
    nan_first = 0
    for x in (rng.standard_normal(shape).astype(F32), _adversarial(rng, shape)):
        xd = torch.from_numpy(x).cuda()
        for axis in range(-len(shape), len(shape)):
            got = capi.argmax(xd, axis, tdt).cpu().numpy()
            want = argmax_ref(x, axis).astype(dtype)
            assert S._same_bits(got, want), (axis, np.argwhere(got != want)[:3])
            nan_first += int(np.isnan(np.moveaxis(x, axis, -1)[..., 0]).any())
    assert nan_first > 0


@pytest.mark.gpu
def test_gpu_argmax_rules_on_known_rows():
    import torch
    from compute_engine_b200 import capi
    nan, inf = np.nan, np.inf
    rows = [([1, 3, 3, 2], 1), ([-0.0, 0.0], 0), ([0.0, -0.0], 0), ([nan, 5, 7], 0), ([1, nan, 7, nan], 2),
            ([-inf, -inf], 0), ([-inf, nan, -inf], 0), ([2, inf, inf], 1), ([nan, nan], 0), ([-1, nan], 0)]
    for wide in (False, True):   # a thread per row, and a warp per row
        for row, want in rows:
            x = np.array(row, F32)
            if wide:   # the same row followed by values below all of it
                x = np.concatenate([x, np.full(200, -np.inf, F32)])
            got = capi.argmax(torch.from_numpy(x[None]).cuda(), -1).item()
            assert got == want == argmax_ref(x, 0), (row, wide)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,axis,axis_dtype,axis_shape", [
    ((7,), 0, np.int32, ()), ((3, 1000), -1, np.int64, (1,)), ((5, 21), 0, np.int32, (1,)),
    ((2, 5, 6, 21), 3, np.int64, ()), ((2, 5, 6, 21), 1, np.int32, ()), ((4, 6, 5), -2, np.int32, ()),
])
@pytest.mark.parametrize("output_type", [np.int32, np.int64])
def test_gpu_argmax_builtin_in_a_graph(shape, axis, axis_dtype, axis_shape, output_type):
    x = _adversarial(np.random.default_rng(sum(shape)), shape)
    g = H.HostGraph.from_tflite(_argmax_graph(shape, axis, axis_dtype, axis_shape, output_type), device_arena=True)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    got = g.read(g.outputs()[0])
    g.close()
    assert S._same_bits(got, argmax_ref(x, axis).astype(output_type))


def _tied_logits(rng, shape):
    """Logits on a grid of a few levels: resized neighbours and channels meet in exact ties."""
    return (rng.integers(-2, 3, shape) * 0.5).astype(F32)


FUSED_CASES = [(ac, hp, c) for ac, hp in S.FLAGS["bilinear"] for c in (1, 3, 21, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("align_corners,half_pixel_centers,c", FUSED_CASES)
def test_gpu_fused_kernel_is_resize_then_argmax(align_corners, half_pixel_centers, c):
    import torch
    from compute_engine_b200 import capi
    rng = np.random.default_rng(c * 7 + align_corners * 2 + half_pixel_centers)
    flags = (align_corners, half_pixel_centers)
    for b in (1, 3):
        for h, w in ((1, 1), (7, 7), (13, 17)):
            for x in (rng.standard_normal((b, h, w, c)).astype(F32), _tied_logits(rng, (b, h, w, c))):
                xd = torch.from_numpy(x).cuda()
                for size in S._sizes(h, w):
                    for dtype in (torch.int64, torch.int32):
                        got = capi.resize_bilinear_argmax(xd, size, *flags, out_dtype=dtype)
                        unfused = capi.argmax(capi.resize(xd, size, True, *flags), -1, dtype)
                        assert torch.equal(got, unfused), (b, h, w, size, dtype)
                    want = argmax_ref(S.resize_bilinear_ref(x, size, *flags), -1)
                    assert S._same_bits(got.cpu().numpy(), want.astype(np.int32)), (b, h, w, size)


@pytest.mark.gpu
def test_gpu_fused_kernel_refuses_rows_too_wide():
    import torch
    from compute_engine_b200 import capi
    c = 21
    w = capi.resize_bilinear_argmax_max_row_floats() // c + 1
    with pytest.raises(capi.LceError, match="does not fit shared memory"):
        capi.resize_bilinear_argmax(torch.zeros((1, 2, w, c), device="cuda"), (4, 2 * w))


@pytest.mark.gpu
def test_gpu_fused_past_2_pow_31_resized_values():
    """[1, 8, 8, 3] -> 27000 x 27000 labels: the resized map they stand for has 2.19 * 10^9 values,
    past 2^31. The first, middle and last rows are checked against the reference of those rows."""
    import torch
    from compute_engine_b200 import capi
    x = torch.from_numpy(_tied_logits(np.random.default_rng(4), (1, 8, 8, 3))).cuda()
    oh, ow = 27000, 27000
    assert oh * ow * 3 > 2 ** 31
    out = capi.resize_bilinear_argmax(x, (oh, ow), False, True)
    xn = x.cpu().numpy()
    vy, y0, y1 = S._bilinear_axis(8, oh, False, True)
    vx, x0, x1 = S._bilinear_axis(8, ow, False, True)
    for rows in (slice(0, 3), slice(oh - 3, oh), slice(13499, 13502)):
        r = np.arange(oh)[rows]
        dy = (vy[r] - y0[r].astype(F32)).astype(F32)[None, :, None, None]
        dx = (vx - x0.astype(F32)).astype(F32)[None, None, :, None]
        ey, ex = (F32(1) - dy).astype(F32), (F32(1) - dx).astype(F32)

        def at(ry, rx):
            return xn[:, ry][:, :, rx]
        s = ((at(y0[r], x0) * ey).astype(F32) * ex).astype(F32)
        s = (s + ((at(y1[r], x0) * dy).astype(F32) * ex).astype(F32)).astype(F32)
        s = (s + ((at(y0[r], x1) * ey).astype(F32) * dx).astype(F32)).astype(F32)
        s = (s + ((at(y1[r], x1) * dy).astype(F32) * dx).astype(F32)).astype(F32)
        assert S._same_bits(out[:, rows].cpu().numpy(), argmax_ref(s, -1)), rows
    del out
    torch.cuda.empty_cache()


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
def test_gpu_quicknet_seg_labels_fused_equals_unfused_and_tflites_rule():
    logits_blob = zoo.quicknet_seg(batch=1, image=224, seed=4, input_type="int8")
    blob = zoo.quicknet_seg(batch=1, image=224, seed=4, input_type="int8", labels="int64")
    for batch, preserve in ((4, True), (256, False)):
        x = zoo.quantize_images(np.random.default_rng(batch).standard_normal((batch, 224, 224, 3), dtype=F32))
        fused, names = _graph_run(blob, x, ("fuse_all",), preserve)
        assert names[-1] == FUSED
        unfused, names = _graph_run(blob, x, PASSES_BUT_ARGMAX, preserve)
        assert names[-2:] == ["builtin:23", "builtin:56"]
        assert fused.shape == (batch, 224, 224) and fused.dtype == np.int64
        assert S._same_bits(fused, unfused), batch
        logits, _ = _graph_run(logits_blob, x, ("fuse_all",), preserve)
        assert S._same_bits(fused, argmax_ref(logits, -1)), batch
        assert len(np.unique(fused)) > 1


@pytest.mark.gpu
@pytest.mark.parametrize("fuse", [True, False])
def test_gpu_quicknet_seg_labels_do_not_depend_on_the_arena(fuse):
    import test_arena_independence as A
    blob = zoo.quicknet_seg(batch=1, seed=0, image=224, labels="int64")
    fails = A.check_arena_independence(blob, (A.BATCH, 224, 224, 3), "float32", fuse=fuse)
    assert not fails, "quicknet_seg(labels='int64'):\n" + "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("batch_size", [3, 5])
@pytest.mark.parametrize("labels", ["int64", "int32"])
def test_gpu_interpreter_predict_over_mini_batches(batch_size, labels):
    from compute_engine_b200.interpreter import Interpreter
    blob = zoo.quicknet_seg(batch=1, image=64, seed=2, input_type="int8", labels=labels)
    x = zoo.quantize_images(np.random.default_rng(1).standard_normal((11, 64, 64, 3), dtype=F32))
    want, _ = _graph_run(blob, x, ("fuse_all",), False)
    it = Interpreter(blob, batch_size=batch_size)
    assert it.output_types == [np.dtype(labels).type]
    got = it.predict(x)
    it.close()
    assert S._same_bits(np.asarray(got), want)
