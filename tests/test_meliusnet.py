"""MeliusNet: the STRIDED_SLICE and SPLIT builtins, the improvement layer's binary convolution added
into a channel slice of the block's map in place (lce_b200_bconv2d_run_slice_add) and the graph
fusion that uses it (Graph::FuseDenseBlocks, now run first in fuse_all()).

CPU: the zoo model through the numpy reference and both readers, its op and channel counts, host
prepare, STRIDED_SLICE / SPLIT shape inference and refusals, the fused node list, each improvement
precondition, the pass order, the other models' node lists and bytes. GPU: bit-exact against run
plus numpy float32 and numpy slicing, the model op by op, and fused vs unfused under CUDA-graph
replay."""
import collections
import hashlib
import itertools

import numpy as np
import pytest

import lce_testlib as L
import tflite_ref as R
from compute_engine_b200 import host as H
from compute_engine_b200 import zoo
from compute_engine_b200.tflite_writer import TFLiteModel, bconv2d_options

DENSE = "MUL+ADD+LceQuantize+LceBconv2d+CONCATENATION"
IMPROVE = "MUL+ADD+LceQuantize+LceBconv2d+STRIDED_SLICE+ADD+CONCATENATION"
BLOCKS, C0 = (4, 5, 4, 6), (64, 160, 224, 256)
OTHERS = ("quicknet", "quicknet_large", "birealnet18", "reactnet_a", "realtobinarynet", "binarydensenet28",
          "binarydensenet37", "binarydensenet37_dilated", "binarydensenet45")
# sha256 of the other models' bytes at the commit before MeliusNet was added
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
}


# ----------------------- CPU reference of the new ops ----------------------- #
def _strided_slice_ref(x, begin, end, strides, o):
    """TFLite's STRIDED_SLICE as numpy basic slicing: a mask bit leaves that side open, and
    Python's slice bounds normalise negative and out-of-range indices as TFLite does."""
    bm, em = o.scalar(0, "i"), o.scalar(1, "i")
    idx = tuple(slice(None if bm >> k & 1 else int(begin[k]), None if em >> k & 1 else int(end[k]), int(strides[k]))
                for k in range(len(begin)))
    return np.ascontiguousarray(x[idx])


def _run_op(model, op, vals):
    """One op of a parsed model on the CPU, as a list of its outputs: STRIDED_SLICE and SPLIT
    here, every other op through tflite_ref."""
    t = model["tensors"]
    if op["code"] == 45:
        x, b, e, s = (vals[i] if t[i]["data"] is None else t[i]["data"] for i in op["inputs"])
        return [_strided_slice_ref(x, b, e, s, op["options"])]
    if op["code"] == 49:
        axis, x = t[op["inputs"][0]]["data"].item(), vals[op["inputs"][1]]
        return [np.ascontiguousarray(p) for p in np.split(x, op["options"].scalar(0, "i"), axis)]
    act = [i for i in op["inputs"] if i >= 0 and t[i]["data"] is None]
    sub = {"tensors": t, "ops": [op], "inputs": act, "outputs": [op["outputs"][0]]}
    return [R.run(sub, [vals[i] for i in act])[0][0]]


def _run_model(model, inputs):
    vals = dict(zip(model["inputs"], inputs))
    for op in model["ops"]:
        vals.update(zip(op["outputs"], _run_op(model, op, vals)))
    return [vals[i] for i in model["outputs"]]


def _bconv_ops(m):
    return [o for o in m["ops"] if o["code"] == 32 and o["custom"] == "LceBconv2d"]


# ----------------------------------- CPU ----------------------------------- #
def test_cpu_reference_runs_meliusnet22():
    m = R.parse(zoo.meliusnet22(batch=1, image=32, seed=2))
    x = np.random.default_rng(0).standard_normal((2, 32, 32, 3)).astype(np.float32)
    out = _run_model(m, [x])[0]
    assert out.shape == (2, 1000) and np.isfinite(out).all() and np.allclose(out.sum(-1), 1.0, atol=1e-4)


def test_meliusnet22_op_and_channel_counts():
    m = R.parse(zoo.meliusnet22(batch=1, image=224, seed=1))
    kinds = collections.Counter((o["code"], o["custom"]) for o in m["ops"])
    assert kinds[(32, "LceBconv2d")] == 38 and kinds[(45, "")] == 38 and kinds[(49, "")] == 2
    assert kinds[(3, "")] == 16 and kinds[(2, "")] == 40
    convs = iter(_bconv_ops(m))
    for sec, n in enumerate(BLOCKS):
        for k in range(n):
            dense, impr = next(convs), next(convs)
            assert R._flex_ints(dense["custom_options"])["channels_in"] == C0[sec] + 64 * k, (sec, k)
            c = C0[sec] + 64 * (k + 1)
            assert R._flex_ints(impr["custom_options"])["channels_in"] == c, (sec, k)
            # the improvement adds into [C0 + 64k, C0 + 64(k+1)): its ADD reads the slice b of x
            add = next(o for o in m["ops"] if o["code"] == 0 and impr["outputs"][0] in o["inputs"])
            b = next(i for i in add["inputs"] if i != impr["outputs"][0])
            sl = next(o for o in m["ops"] if o["outputs"] == [b])
            x = np.arange(c, dtype=np.float32).reshape(1, 1, 1, c)
            got = _strided_slice_ref(x, *(m["tensors"][i]["data"] for i in sl["inputs"][1:]), sl["options"])
            assert got.ravel().tolist() == list(range(c - 64, c)), (sec, k)
    splits = [o for o in m["ops"] if o["code"] == 49]
    assert [len(o["outputs"]) for o in splits] == [4, 8]
    assert m["tensors"][m["ops"][-4]["outputs"][0]]["shape"][3] == 640   # the head's RELU


def test_meliusnet22_readers_agree_and_it_prepares_on_the_host():
    blob = zoo.meliusnet22(batch=2, image=64, seed=1)
    m = R.parse(blob)
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    assert g.num_nodes() == len(m["ops"])
    for i, t in enumerate(m["tensors"]):
        assert g.shape(i) == t["shape"], t["name"]
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (2, 1000)
    g.resize_input(g.inputs()[0], (3, 64, 64, 3))
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (3, 1000)
    g.close()


def _one_op(kind, x_shape, consts, out_shapes, dtype=np.float32, **opts):
    """x -> one STRIDED_SLICE ([x, begin, end, strides]) or SPLIT ([axis, x]) op -> outputs."""
    m = TFLiteModel()
    x = m.add_tensor("x", x_shape, dtype)
    cs = [m.add_tensor(f"c{k}", None, np.int32, data=np.asarray(v, np.int32)) for k, v in enumerate(consts)]
    outs = [m.add_tensor(f"o{k}", s, dtype) for k, s in enumerate(out_shapes)]
    m.add_op(kind, [x] + cs if kind == "STRIDED_SLICE" else cs + [x], outs, **opts)
    m.inputs, m.outputs = [x], outs
    return m.serialize()


# (x shape, dtype, [begin, end, strides], options, output shape)
SLICES = [
    ((2, 5, 6, 12), np.float32, [[0, 0, 0, -4], [0, 0, 0, 0], [1, 1, 1, 1]],
     dict(begin_mask=0b0111, end_mask=0b1111), (2, 5, 6, 4)),
    ((2, 5, 6, 12), np.float32, [[0, 0, 0, 0], [0, 0, 0, -4], [1, 1, 1, 1]],
     dict(begin_mask=0b1111, end_mask=0b0111), (2, 5, 6, 8)),
    ((2, 5, 6, 12), np.float32, [[0, 1, 0, 0], [0, -1, 0, 0], [1, 1, 1, 1]],
     dict(begin_mask=0b1101, end_mask=0b1101), (2, 3, 6, 12)),
    ((7, 9), np.int32, [[0, 2], [0, 100], [1, 1]], dict(begin_mask=1, end_mask=1), (7, 7)),
    ((10,), np.float32, [[-100], [3], [1]], {}, (3,)),
    ((4, 6), np.int32, [[1], [3], [1]], {}, (2, 6)),
    ((3, 4, 5), np.float32, [[0, 0, 0], [3, 4, 5], [1, 1, 1]], {}, (3, 4, 5)),
]
# (x shape, axis, num_splits, output shape)
SPLITS = [((2, 4, 4, 12), 3, 3, (2, 4, 4, 4)), ((2, 4, 4, 12), -1, 4, (2, 4, 4, 3)),
          ((2, 4, 4, 12), 0, 2, (1, 4, 4, 12)), ((6, 5), 1, 5, (6, 1))]


@pytest.mark.parametrize("case", range(len(SLICES)))
def test_strided_slice_shape_inference(case):
    shape, dtype, consts, opts, want = SLICES[case]
    g = H.HostGraph.from_tflite(_one_op("STRIDED_SLICE", shape, consts, [want], dtype, **opts),
                                device_arena=False)
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == want
    g.close()


@pytest.mark.parametrize("case", range(len(SPLITS)))
def test_split_shape_inference(case):
    shape, axis, n, want = SPLITS[case]
    g = H.HostGraph.from_tflite(_one_op("SPLIT", shape, [axis], [want] * n, num_splits=n), device_arena=False)
    g.allocate_tensors()
    assert [g.shape(t) for t in g.outputs()] == [want] * n
    g.close()


@pytest.mark.parametrize("consts,opts,msg", [
    ([[0, 0, 0, 0], [0, 0, 0, 6], [1, 1, 1, 2]], dict(begin_mask=7, end_mask=7), "only unit strides"),
    ([[0, 0, 0, 0], [0, 0, 0, 6], [1, 1, 1, 1]], dict(ellipsis_mask=1), "ellipsis_mask"),
    ([[0, 0, 0, 0], [0, 0, 0, 6], [1, 1, 1, 1]], dict(new_axis_mask=2), "new_axis_mask"),
    ([[0, 0, 0, 0], [0, 0, 0, 6], [1, 1, 1, 1]], dict(shrink_axis_mask=8), "shrink_axis_mask"),
    ([[0, 0, 0, 0], [0, 0, 0, 6], [1, 1, 1, 1]], dict(begin_mask=7, end_mask=7, offset=True), "offset"),
    ([[0, 1, 0, 0], [0, 3, 0, 6], [1, 1, 1, 1]], dict(begin_mask=5, end_mask=5), "at most one axis"),
])
def test_strided_slice_refusals(consts, opts, msg):
    g = H.HostGraph.from_tflite(_one_op("STRIDED_SLICE", (2, 5, 6, 12), consts, [(2, 5, 6, 6)], **opts),
                                device_arena=False)
    with pytest.raises(H.HostError, match=msg):
        g.allocate_tensors()
    g.close()


def test_split_refuses_an_axis_it_does_not_divide():
    g = H.HostGraph.from_tflite(_one_op("SPLIT", (2, 4, 4, 12), [3], [(2, 4, 4, 2)] * 5, num_splits=5),
                                device_arena=False)
    with pytest.raises(H.HostError, match="must divide the axis"):
        g.allocate_tensors()
    g.close()


def _fused_names(blob, use_reference_bconv=False):
    g = H.HostGraph.from_tflite(blob, device_arena=True, use_reference_bconv=use_reference_bconv)
    n = g.fuse_dense_blocks()
    names = [g.node_name(i) for i in range(g.num_nodes())]
    outs = [g.node_io(i)[1][0] for i in range(g.num_nodes()) if names[i] in (DENSE, IMPROVE)]
    again = g.fuse_dense_blocks()
    g.close()
    return n, names, outs, again


def test_meliusnet22_fused_node_list():
    n, names, outs, again = _fused_names(zoo.meliusnet22(batch=2, image=224, seed=1))
    assert n == 19 * 4 + 19 * 7 and again == 0
    c = collections.Counter(names)
    assert c[DENSE] == 19 and c[IMPROVE] == 19
    assert c["LceBconv2d"] == 0 and c["LceQuantize"] == 0 and c["builtin:45"] == 0
    assert c["builtin:2"] == 2 and c["builtin:49"] == 2   # the stem's grouped convolutions
    # dense and improvement layers alternate; each section's layers write one tensor
    assert [x for x in names if x in (DENSE, IMPROVE)] == [DENSE, IMPROVE] * 19
    assert [len(list(v)) for _, v in itertools.groupby(outs)] == [2 * b for b in BLOCKS]
    # under fuse_all the dense pass runs first, and the layers stay as it left them
    g = H.HostGraph.from_tflite(zoo.meliusnet22(batch=2, image=224, seed=1), device_arena=True)
    total = g.fuse_all()
    c = collections.Counter(g.node_name(i) for i in range(g.num_nodes()))
    assert c[DENSE] == 19 and c[IMPROVE] == 19 and total >= n
    g.close()


def test_meliusnet22_unfused_without_the_mma_sync_kernel(monkeypatch):
    monkeypatch.setenv("LCE_B200_BCONV_IMMA", "0")
    g = H.HostGraph.from_tflite(zoo.meliusnet22(batch=1, image=64, seed=1), device_arena=True)
    assert g.fuse_dense_blocks() == 0
    g.close()


@pytest.mark.parametrize("name", OTHERS)
def test_other_models_keep_their_node_lists(name):
    """fuse_all() with the dense pass first gives the node list of the previous pass order."""
    blob = zoo.MODELS[name](batch=1, image=224, seed=2)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n = (g.fuse_residual_blocks() + g.fuse_float_glue() + g.fuse_dense_blocks() + g.fuse_channel_gates()
         + g.fuse_activation_chains() + g.fuse_residual_pairs())
    before = [g.node_name(i) for i in range(g.num_nodes())]
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    assert g.fuse_all() == n
    assert [g.node_name(i) for i in range(g.num_nodes())] == before
    g.close()


def test_other_models_bytes_are_unchanged():
    for (name, image), want in OTHER_HASHES.items():
        kw = dict(batch=1, image=224, seed=0) if image == 224 else dict(batch=2, image=64, seed=3,
                                                                          input_type="int8")
        assert hashlib.sha256(zoo.MODELS[name](**kw)).hexdigest() == want, (name, image)


def _melius_block(layers="di", c0=64, hw=6, pad_values=1, slices_at="conv", sum_order="by",
                  scale_shape=None, mul_act="NONE", sum_act="NONE", cat_order="as", cat_act="NONE",
                  cat_axis=3, b_bounds=None, output=None, extra_reader=None, cout=64):
    """x_0 [2, hw, hw, c0] -> layers ("d" dense, "i" improvement) -> RELU of the map (the graph
    output). The improvement options apply to every "i" layer: its slices go before its MUL
    ("mul"), before its LceBconv2d ("conv") or after it ("end"); sum_order "by" is ADD(b, y);
    b_bounds replaces b's channel bounds; `output` / `extra_reader` give that named tensor of the
    first improvement layer ("a", "b", "y" or "s") a place among the outputs / a second reader."""
    rng = np.random.default_rng(11)
    m = TFLiteModel()
    x0 = x = m.add_tensor("x0", (2, hw, hw, c0))
    c, inter, j = c0, None, 0
    f32 = lambda name, shape, lo=-0.5, hi=0.5: m.add_tensor(f"{name}{j}", None, np.float32,
                                                            data=rng.uniform(lo, hi, shape))
    i32 = lambda v: m.add_tensor(f"ss{j}_{len(m.tensors)}", None, np.int32, data=np.asarray(v, np.int32))

    def slices():
        lo, hi = b_bounds or (-cout, 0)
        a = m.add_tensor(f"a{j}", (2, hw, hw, c - cout))
        b = m.add_tensor(f"b{j}", (2, hw, hw, (hi % c if hi else c) - lo % c))
        m.add_op("STRIDED_SLICE", [x, i32([0, 0, 0, 0]), i32([0, 0, 0, -cout]), i32([1, 1, 1, 1])], [a],
                 begin_mask=0b1111, end_mask=0b0111)
        m.add_op("STRIDED_SLICE", [x, i32([0, 0, 0, lo]), i32([0, 0, 0, hi]), i32([1, 1, 1, 1])], [b],
                 begin_mask=0b0111, end_mask=0b0111 if hi else 0b1111)
        return a, b

    for j, kind in enumerate(layers):
        cw = (c + 31) // 32
        if kind == "i" and slices_at == "mul":
            a, b = slices()
        t, u = m.add_tensor(f"t{j}", (2, hw, hw, c)), m.add_tensor(f"u{j}", (2, hw, hw, c))
        q = m.add_tensor(f"q{j}", (2, hw, hw, cw), np.int32)
        y = m.add_tensor(f"y{j}", (2, hw, hw, cout))
        m.add_op("MUL", [x, f32("scale", (scale_shape or (c,)) if kind == "i" else (c,), 0.5, 1.5)], [t],
                 activation=mul_act if kind == "i" else "NONE")
        m.add_op("ADD", [t, f32("shift", (c,))], [u])
        m.add_op("LceQuantize", [u], [q], custom_options=b"")
        if kind == "i" and slices_at == "conv":
            a, b = slices()
        filt = m.add_tensor(f"f{j}", None, np.int32,
                            data=rng.integers(-2**31, 2**31 - 1, (cout, 3, 3, cw)).astype(np.int32))
        m.add_op("LceBconv2d", [q, filt, f32("mul", cout, 0.1, 1), f32("bias", cout), -1], [y],
                 custom_options=bconv2d_options(c, pad_values=pad_values))
        if kind == "d":
            z = m.add_tensor(f"x{j + 1}", (2, hw, hw, c + cout))
            m.add_op("CONCATENATION", [x, y], [z], axis=3)
            x, c = z, c + cout
            continue
        if slices_at == "end":
            a, b = slices()
        s = m.add_tensor(f"s{j}", (2, hw, hw, cout))
        m.add_op("ADD", [b, y] if sum_order == "by" else [y, b], [s], activation=sum_act)
        z = m.add_tensor(f"x{j + 1}", (2, hw, hw, c))
        m.add_op("CONCATENATION", [a, s] if cat_order == "as" else [s, a], [z], axis=cat_axis, activation=cat_act)
        if inter is None:
            inter = {"a": a, "b": b, "y": y, "s": s}
        x = z
    r = m.add_tensor("r", m.tensors[x]["shape"])
    m.add_op("RELU", [x], [r])
    outs = [r]
    if output:
        outs.append(inter[output])
    if extra_reader:
        e = m.add_tensor("e", m.tensors[inter[extra_reader]]["shape"])
        m.add_op("RELU", [inter[extra_reader]], [e])
        outs.append(e)
    m.inputs, m.outputs = [x0], outs
    return m.serialize()


@pytest.mark.parametrize("kw,names", [
    (dict(layers="i"), [IMPROVE]),
    (dict(layers="i", slices_at="mul"), [IMPROVE]),
    (dict(layers="i", slices_at="end"), [IMPROVE]),
    (dict(layers="i", sum_order="yb"), [IMPROVE]),
    (dict(layers="i", cat_axis=-1), [IMPROVE]),
    (dict(layers="i", pad_values=0), [IMPROVE]),
    (dict(layers="i", scale_shape=(1, 1, 1, 64)), [IMPROVE]),
    (dict(layers="di"), [DENSE, IMPROVE]),
    (dict(layers="didi", slices_at="mul"), [DENSE, IMPROVE, DENSE, IMPROVE]),
    (dict(layers="iid", c0=128), [IMPROVE, IMPROVE, DENSE]),
])
def test_improvement_layer_fuses(kw, names):
    blob = _melius_block(**kw)
    n, got, outs, again = _fused_names(blob)
    assert got == names + ["builtin:19"], kw
    assert n == 4 * names.count(DENSE) + 7 * names.count(IMPROVE) and again == 0
    assert len(set(outs)) == 1, kw   # one block, one map
    g = H.HostGraph.from_tflite(blob, device_arena=False)   # and the graph prepares unfused
    g.allocate_tensors()
    g.close()


def test_improvement_layer_with_slices_before_the_convolution_fuses_under_fuse_all():
    """fuse_residual_blocks would take LceBconv2d -> ADD(b) once b exists before the convolution:
    the dense pass runs first."""
    g = H.HostGraph.from_tflite(_melius_block(layers="i", slices_at="conv"), device_arena=True)
    g.fuse_all()
    assert [g.node_name(i) for i in range(g.num_nodes())] == [IMPROVE, "builtin:19"]
    g.close()
    g = H.HostGraph.from_tflite(_melius_block(layers="i", slices_at="conv"), device_arena=True)
    assert g.fuse_residual_blocks() == 1 and g.fuse_dense_blocks() == 0   # the old order
    g.close()


@pytest.mark.parametrize("variant", ["scale_not_per_channel", "mul_has_activation", "sum_has_activation",
                                     "concat_order", "b_not_the_last_channels", "cout_not_64",
                                     "slice_is_a_graph_output", "sum_is_a_graph_output",
                                     "slice_read_twice", "y_read_twice"])
def test_improvement_fusion_leaves_the_layer_when_a_precondition_fails(variant):
    kw = {"scale_not_per_channel": dict(scale_shape=(2, 6, 6, 64)),
          "mul_has_activation": dict(mul_act="RELU"),
          "sum_has_activation": dict(sum_act="RELU"),
          "concat_order": dict(cat_order="sa"),
          "b_not_the_last_channels": dict(b_bounds=(-64 - 32, -32), c0=128),
          "cout_not_64": dict(cout=32),
          "slice_is_a_graph_output": dict(output="a"),
          "sum_is_a_graph_output": dict(output="s"),
          "slice_read_twice": dict(extra_reader="b"),
          "y_read_twice": dict(extra_reader="y")}[variant]
    blob = _melius_block(layers="i", **kw)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    before = [g.node_name(i) for i in range(g.num_nodes())]
    assert g.fuse_dense_blocks() == 0
    assert [g.node_name(i) for i in range(g.num_nodes())] == before
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=False)   # and the graph prepares unfused
    g.allocate_tensors()
    g.close()


def test_fused_node_lists_differ_from_the_base_arm_by_the_absorbed_nodes():
    """The GPU comparison below runs fuse_all() against the same passes without the dense one; the
    base arm runs each dense layer as MUL, ADD+LceQuantize, LceBconv2d, CONCATENATION and each
    improvement layer as MUL, ADD+LceQuantize, two STRIDED_SLICEs, LceBconv2d+ADD, CONCATENATION."""
    blob = zoo.meliusnet22(batch=1, image=64, seed=4, input_type="int8")
    n_ref, n_got = _arm_names(blob, False), _arm_names(blob, True)
    c = collections.Counter(n_ref)
    assert c["ADD+LceQuantize"] == 38 and c["LceBconv2d+ADD"] == 19 and c["builtin:45"] == 38
    assert len(n_ref) - len(n_got) == 19 * 3 + 19 * 5


def _arm_names(blob, dense):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    _fuse(g, dense)
    names = [g.node_name(i) for i in range(g.num_nodes())]
    g.close()
    return names


def _fuse(g, dense):
    if dense:
        g.fuse_all()
    else:
        g.fuse_residual_blocks() + g.fuse_float_glue() + g.fuse_channel_gates() + g.fuse_activation_chains()
        g.fuse_residual_pairs()


# ----------------------------------- GPU ----------------------------------- #
SENTINEL = np.float32(-1234.5)


@pytest.mark.gpu
@pytest.mark.parametrize("b1", ["1", "0"])
def test_gpu_run_slice_add_is_run_then_add(b1, monkeypatch):
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import assert_same_bits, dev, gpu_desc, path_counts
    monkeypatch.setenv("LCE_B200_BCONV_IMMA", "1")
    monkeypatch.setenv("LCE_B200_BCONV_B1", b1)
    rng = np.random.default_rng(31)
    # filter x C_in x image; pad values 1 / 0 REFERENCE / 0 CORRECTION cycled
    cases = [(fh, cin, hw) for fh in (3, 1) for cin in (128, 320, 640) for hw in (7, 1)]
    for n, (fh, cin, hw) in enumerate(cases * 2):
        pv, corr = ((1, 0), (0, 0), (0, 1))[n % 3]
        cout = 64
        batch = 5 if hw == 7 else 37          # M = 245 or 37: not a multiple of the 128-row tile
        case = L.make_bconv_case(700 + n, batch, hw, hw, cin, fh, fh, cout, pad_value=pv)
        plan = capi.BConv2d(gpu_desc(capi, case.desc), case.filt, case.mul, case.bias, case.thr)
        if pv == 0:
            plan.set_zero_padding_mode(corr)
        y = plan(dev(case.inp))
        torch.cuda.synchronize()
        y = y.cpu().numpy()
        off = cin - cout   # the improvement layer's slice: the map's last channels
        wide = np.full((batch, hw, hw, cin + 8 * (n % 2)), SENTINEL, np.float32)
        wide[..., off:off + cout] = rng.standard_normal((batch, hw, hw, cout)).astype(np.float32)
        want = wide.copy()
        want[..., off:off + cout] = wide[..., off:off + cout] + y    # TFLite's ADD(b, y) in float32
        io = torch.from_numpy(wide).cuda()
        scratch = torch.empty(batch * hw * hw * cout, device="cuda") if corr or n % 2 else None
        before = path_counts(capi)
        plan.run_slice_add(dev(case.inp), io, off, scratch)
        torch.cuda.synchronize()
        ran = [b - a for a, b in zip(before, path_counts(capi))]
        tag = f"b1={b1} case {n} ({fh}x{fh} {cin}->{cout} {hw}x{hw} pad{pv} corr{corr})"
        assert ran == [0, 1, 0], (tag, ran)
        got = io.cpu().numpy()
        assert_same_bits(got[..., off:off + cout], want[..., off:off + cout], tag)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), tag + ": wrote outside its slice"
        plan.close()


@pytest.mark.gpu
def test_gpu_run_slice_add_refusals(monkeypatch):
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import dev, gpu_desc
    case = L.make_bconv_case(5, 2, 7, 7, 64, 3, 3, 64)
    plan = capi.BConv2d(gpu_desc(capi, case.desc), case.filt, case.mul, case.bias, case.thr)
    x = dev(case.inp)
    with pytest.raises(capi.LceError, match="at least channels_out"):
        plan.run_slice_add(x, torch.zeros(2, 7, 7, 60, device="cuda"))
    with pytest.raises(capi.LceError, match="must be a multiple of 4"):
        plan.run_slice_add(x, torch.zeros(2, 7, 7, 66, device="cuda"))
    with pytest.raises(capi.LceError, match="16-byte aligned"):
        plan.run_slice_add(x, torch.zeros(2, 7, 7, 72, device="cuda"), offset=2)
    buf = torch.zeros(2 * 7 * 7 * 128 + 64, device="cuda")
    xin = buf.view(torch.int32)[:x.numel()].view(x.shape)
    xin.copy_(x)
    with pytest.raises(capi.LceError, match="must not overlap the input"):
        plan.run_slice_add(xin, buf[:2 * 7 * 7 * 128].view(2, 7, 7, 128), offset=64)
    plan.close()
    # a CORRECTION plan and its scratch
    c = L.make_bconv_case(7, 2, 7, 7, 128, 3, 3, 64, pad_value=0)
    plan = capi.BConv2d(gpu_desc(capi, c.desc), c.filt, c.mul, c.bias, c.thr)
    plan.set_zero_padding_mode(1)
    x = dev(c.inp)
    io = torch.zeros(2, 7, 7, 128, device="cuda")
    with pytest.raises(capi.LceError, match="needs the scratch"):
        plan.run_slice_add(x, io, 64)
    with pytest.raises(capi.LceError, match="scratch must be 16-byte aligned"):
        plan.run_slice_add(x, io, 64, torch.zeros(2 * 49 * 64 + 1, device="cuda")[1:])
    with pytest.raises(capi.LceError, match="scratch must not overlap io or the input"):
        plan.run_slice_add(x, io, 64, io.view(-1)[:2 * 49 * 64])
    big = torch.zeros(2 * 49 * 64 + 2 * 49 * 4, device="cuda")
    xin = big.view(torch.int32)[:x.numel()].view(x.shape)
    xin.copy_(x)
    with pytest.raises(capi.LceError, match="scratch must not overlap io or the input"):
        plan.run_slice_add(xin, io, 64, big[:2 * 49 * 64])
    plan.close()
    for kw, env, msg in ((dict(cout=32), {}, "mma.sync weight fragments"),
                         (dict(cout=64), {"LCE_B200_BCONV_IMMA": "0"}, "mma.sync weight fragments"),
                         (dict(cout=64, out_type=L.OUT_BITPACKED), {}, "float output")):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        c = L.make_bconv_case(6, 2, 7, 7, 64, 3, 3, kw["cout"], out_type=kw.get("out_type", L.OUT_FLOAT))
        plan = capi.BConv2d(gpu_desc(capi, c.desc), c.filt, c.mul, c.bias, c.thr)
        with pytest.raises(capi.LceError, match=msg):
            plan.run_slice_add(dev(c.inp), torch.zeros(2, 7, 7, 128, device="cuda"))
        plan.close()
        for k in env:
            monkeypatch.delenv(k)


@pytest.mark.gpu
def test_gpu_strided_slice_and_split_match_numpy():
    rng = np.random.default_rng(17)
    runs = [(_one_op("STRIDED_SLICE", s, cs, [w], dt, **o), s, dt) for s, dt, cs, o, w in SLICES]
    runs += [(_one_op("SPLIT", s, [a], [w] * n, num_splits=n), s, np.float32) for s, a, n, w in SPLITS]
    for blob, shape, dtype in runs:
        m = R.parse(blob)
        x = (rng.standard_normal(shape).astype(np.float32) if dtype == np.float32
             else rng.integers(-2**31, 2**31 - 1, shape).astype(np.int32))
        want = _run_model(m, [x])
        g = H.HostGraph.from_tflite(blob, device_arena=True)
        g.allocate_tensors()
        g.write(g.inputs()[0], x)
        g.invoke()
        for t, w in zip(g.outputs(), want):
            assert np.array_equal(g.read(t).view(np.uint8), w.view(np.uint8)), (shape, m["ops"][0]["code"])
        g.close()


@pytest.mark.gpu
def test_gpu_meliusnet22_graph_op_by_op():
    """The unfused graph on the device, op by op on the device's own input tensors: every LCE op,
    MUL, ADD, CONCATENATION, STRIDED_SLICE and SPLIT bit exact, the other float builtins within the
    torch fp32 reference's tolerance; then the class probabilities against the CPU graph."""
    blob = zoo.meliusnet22(batch=1, image=64, seed=9)
    m = R.parse(blob)
    x = np.random.default_rng(3).standard_normal((3, 64, 64, 3)).astype(np.float32)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.preserve_all_tensors(True)
    g.resize_input(g.inputs()[0], x.shape)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    exact = collections.Counter()
    for op in m["ops"]:
        vals = {i: g.read(i) for i in op["inputs"] if i >= 0 and m["tensors"][i]["data"] is None}
        for t, want in zip(op["outputs"], _run_op(m, op, vals)):
            got = g.read(t)
            assert got.shape == want.shape, (op["code"], op["custom"])
            if op["code"] in (32, 0, 18, 2, 45, 49):
                assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (op["code"], op["custom"])
                exact[op["custom"] or op["code"]] += 1
            else:
                scale = max(1.0, float(np.abs(want).max()))
                assert np.allclose(got, want, rtol=1e-4, atol=1e-5 * scale), (op["code"], np.abs(got - want).max())
    assert exact["LceBconv2d"] == 38 and exact[45] == 38 and exact[49] == 12 and exact[2] == 40
    want_out = _run_model(m, [x])[0]
    assert np.abs(g.read(g.outputs()[0]) - want_out).max() <= 2e-4
    g.close()


def _run_graph(blob, x, dense, preserve, launches, use_reference_bconv=False):
    """fuse_all with or without the dense pass; one eager step (its launches counted), then a
    CUDA-graph capture and replay. Returns the output and the node names."""
    from compute_engine_b200 import capi
    g = H.HostGraph.from_tflite(blob, device_arena=True, use_reference_bconv=use_reference_bconv)
    g.resize_input(g.inputs()[0], x.shape)
    _fuse(g, dense)
    names = [g.node_name(i) for i in range(g.num_nodes())]
    g.preserve_all_tensors(preserve)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    g.synchronize()
    l0 = capi.launch_count()
    g.invoke()
    g.synchronize()
    launches.append(capi.launch_count() - l0)
    g.enable_cuda_graph(True)
    g.invoke()   # capture
    g.write(g.inputs()[0], x)
    g.invoke()   # replay
    out = g.read(g.outputs()[0])
    g.close()
    return out, names


@pytest.mark.gpu
@pytest.mark.parametrize("pad_values,reference", [(0, False), (0, True), (1, False)])
def test_gpu_meliusnet22_fused_equals_unfused(pad_values, reference):
    """Default registration (CORRECTION zero padding), use_reference_bconv (REFERENCE) and one-
    padding; with every tensor kept, then with reused arenas. Each fused layer runs two launches (the
    signs, then the convolution) where the unfused one ran three kernels (MUL, ADD + LceQuantize,
    LceBconv2d [+ ADD]) and its copies; zero padding adds correction passes, so the count is checked
    at one-padding."""
    blob = zoo.meliusnet22(batch=1, image=64, seed=4, pad_values=pad_values, input_type="int8")
    x = np.random.default_rng(6).integers(-128, 128, (2, 64, 64, 3)).astype(np.int8)
    for preserve in (True, False):
        launches = []
        ref, n_ref = _run_graph(blob, x, False, preserve, launches, reference)
        got, n_got = _run_graph(blob, x, True, preserve, launches, reference)
        c = collections.Counter(n_got)
        assert c[DENSE] == 19 and c[IMPROVE] == 19
        if pad_values == 1:
            assert launches[0] - launches[1] == 38, launches
        assert np.isfinite(got).all()
        assert np.array_equal(ref.view(np.uint8), got.view(np.uint8)), (pad_values, reference, preserve)


@pytest.mark.gpu
def test_gpu_interpreter_predict_resizes_the_fused_graph():
    from compute_engine_b200.interpreter import Interpreter
    blob = zoo.meliusnet22(batch=3, image=64, seed=5)
    m = R.parse(blob)
    it = Interpreter(blob)
    for b in (3, 5, 3):
        x = np.random.default_rng(b).standard_normal((b, 64, 64, 3)).astype(np.float32)
        got = it.predict(x)
        want = _run_model(m, [x])[0]
        assert got.shape == (b, 1000) and np.abs(got - want).max() <= 2e-4, b
