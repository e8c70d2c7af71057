"""Binary dense layers: LceDequantize -> FULLY_CONNECTED (+-alpha_o weights) [-> MUL -> ADD] [-> LceQuantize]
as one b1 convolution of the layer's rows (lce_b200_bconv2d_run_fused_fc, Graph::FuseBinaryFullyConnected),
the pooled sign through larq's flattening RESHAPE, and the zoo's binaryalexnet / xnornet(dense=...).

CPU: the default zoo bytes, the dense variants' ops, the fused node lists, each fusion precondition, the other
models' node lists.
GPU: the fused node against the unfused graph and a numpy restatement of TFLite's FULLY_CONNECTED loop bit for
bit (+-1 weights) or fl(fl(alpha * D) + b) bit for bit and within the documented bound of the unfused graph
(other alpha), the C entry directly, which kernel ran, and both dense zoo graphs fused against unfused, on
poisoned arenas and on CUDA-graph replays of new inputs."""
import hashlib

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
FUSED = "LceBfc"
# fuse_all's passes but fuse_binary_fully_connected, in fuse_all's order
PASSES_BUT_FC = ("fuse_binary_bases", "fuse_dense_blocks", "fuse_binary_transpose_convs", "fuse_residual_blocks",
                 "fuse_spatial_scales", "fuse_float_glue", "fuse_upsample_merges", "fuse_resize_argmax",
                 "fuse_subpixel_convs", "fuse_grouped_conv_affine", "fuse_quantized_activations",
                 "fuse_pooled_signs", "fuse_channel_gates", "fuse_activation_chains", "fuse_residual_pairs")
# sha256 of the default models (dense="conv"), as the parent revision writes them
DEFAULT_SHA256 = {
    ("binaryalexnet", ()): "150d60007c51b3398d51c6728d6ccb08693609ff0cd7d1b34ad41f01e2218dac",
    ("binaryalexnet", (("batch", 4), ("pad_values", 1))):
        "072d91ba00d13c5468c61b519313b96ea8089e4bff5787c5168ca347612745b1",
    ("binaryalexnet", (("batch", 2), ("image", 128), ("input_type", "int8"))):
        "b130a2f96476aaa72006e3e8808b04edc82d17df977bb419bcbc26098355359d",
    ("xnornet", ()): "1320cd7cfb60937fccfccefd5cdc8d4925628d2f4d363bc3a2a4e1e25732b586",
    ("xnornet", (("batch", 4), ("pad_values", 1))):
        "c8e8da0ef27bf47a300b6317d7877eb124252f7a045f0f8bee95983c796dc29d",
    ("xnornet", (("batch", 2), ("image", 128), ("input_type", "int8"))):
        "6bca86c7fffd326dc6f5a64d2b5e12b28a0351941a3a6fdfbf961414dc71471d",
}


# ---------------------------- small test graphs ---------------------------- #
def _weights(rng, n, k, alpha=None):
    signs = (rng.integers(0, 2, (n, k)) * 2 - 1).astype(F32)
    return signs if alpha is None else signs * np.asarray(alpha, F32)[:, None]


def _fc_graph(x_shape=(4, 100), n=64, weights=None, alpha=None, bias=True, act="NONE", bn=False,
              bn_act="NONE", quant=False, outputs=(), deq_reader=False, mul_shape=None, seed=0):
    """q -> LceDequantize -> FULLY_CONNECTED [-> MUL(scale) -> ADD(shift)] [-> LceQuantize]. Returns the model
    and its constants."""
    rng = np.random.default_rng(seed)
    k = x_shape[-1] if len(x_shape) == 2 else int(np.prod(x_shape[1:]))
    rows = int(np.prod(x_shape)) // k
    m = TFLiteModel()
    q = m.add_tensor("q", tuple(x_shape[:-1]) + ((x_shape[-1] + 31) // 32,), np.int32)
    deq = m.add_tensor("deq", tuple(x_shape))
    m.add_op("LceDequantize", [q], [deq], custom_options=b"")
    if weights is None:
        weights = _weights(rng, n, k, alpha)
    c = {"w": weights, "b": rng.uniform(-3, 3, n).astype(F32) if bias else None}
    y = m.add_tensor("y", (rows, n))
    m.add_op("FULLY_CONNECTED", [deq, m.add_tensor("w", None, data=weights),
                                 m.add_tensor("b", None, data=c["b"]) if bias else -1], [y], activation=act)
    t = {"deq": deq, "y": y}
    last = y
    if bn:
        c["scale"] = rng.uniform(0.5, 1.5, mul_shape or (n,)).astype(F32)
        c["shift"] = rng.uniform(-0.5, 0.5, n).astype(F32)
        u = m.add_tensor("u", (rows, n))
        m.add_op("MUL", [y, m.add_tensor("scale", None, data=c["scale"])], [u])
        last = t["bn"] = m.add_tensor("bn", (rows, n))
        m.add_op("ADD", [u, m.add_tensor("shift", None, data=c["shift"])], [last], activation=bn_act)
    outs = [last]
    if quant:
        pk = m.add_tensor("pk", (rows, (n + 31) // 32), np.int32)
        m.add_op("LceQuantize", [last], [pk], custom_options=b"")
        outs.append(pk)
    if deq_reader:
        r = m.add_tensor("relu", tuple(x_shape))
        m.add_op("RELU", [deq], [r])
        outs.append(r)
    outs += [t[name] for name in outputs]
    m.inputs, m.outputs = [q], outs
    return m.serialize(), c


def _names(g):
    return [g.node_name(i) for i in range(g.num_nodes())]


def _tail(names, start):
    """The node names from the last one named `start` on."""
    return names[len(names) - 1 - names[::-1].index(start):]


# ----------------------------------- CPU ----------------------------------- #
@pytest.mark.parametrize("key", sorted(DEFAULT_SHA256, key=str))
def test_default_models_keep_their_bytes(key):
    name, kw = key
    assert hashlib.sha256(getattr(zoo, name)(**dict(kw))).hexdigest() == DEFAULT_SHA256[key]
    assert getattr(zoo, name)(**dict(kw), dense="conv") == getattr(zoo, name)(**dict(kw))


def test_unknown_dense_is_refused():
    for make in (zoo.binaryalexnet, zoo.xnornet):
        with pytest.raises(ValueError):
            make(dense="dense")


def _ops_after_last_pool(blob):
    m = R.parse(blob)
    ops = m["ops"]
    last = max(i for i, o in enumerate(ops) if o["code"] == 17)   # MAX_POOL_2D
    return m, ops[last + 1:]


def _op_name(o):
    return o["custom"] or {0: "ADD", 9: "FULLY_CONNECTED", 18: "MUL", 22: "RESHAPE", 25: "SOFTMAX"}[o["code"]]


def test_binaryalexnet_dense_ops():
    m, ops = _ops_after_last_pool(zoo.binaryalexnet(batch=2, dense="fully_connected"))
    layer = ["LceQuantize", "LceDequantize", "FULLY_CONNECTED", "MUL", "ADD"]
    assert [_op_name(o) for o in ops] == ["MUL", "ADD", "RESHAPE"] + layer * 3 + ["SOFTMAX"]
    t = m["tensors"]
    assert t[ops[2]["outputs"][0]]["shape"] == (2, 9216)
    fcs = [o for o in ops if o["code"] == 9]
    for o, (n, k) in zip(fcs, ((4096, 9216), (4096, 4096), (1000, 4096))):
        w = t[o["inputs"][1]]["data"]
        assert w.shape == (n, k) and set(np.unique(w)) == {-1.0, 1.0}
        assert len(o["inputs"]) < 3 or o["inputs"][2] == -1    # no bias
        assert t[o["outputs"][0]]["shape"] == (2, n)
    assert len([o for o in R.parse(zoo.binaryalexnet(dense="fully_connected"))["ops"]
                if o["custom"] == "LceBconv2d"]) == 4


def test_xnornet_dense_ops():
    m, ops = _ops_after_last_pool(zoo.xnornet(batch=2, dense="fully_connected"))
    layer = ["LceQuantize", "LceDequantize", "FULLY_CONNECTED"]
    assert [_op_name(o) for o in ops] == ["MUL", "ADD", "RESHAPE"] + layer * 2 + ["FULLY_CONNECTED", "SOFTMAX"]
    t = m["tensors"]
    fcs = [o for o in ops if o["code"] == 9]
    for o, (n, k) in zip(fcs[:2], ((4096, 9216), (4096, 4096))):
        w = t[o["inputs"][1]]["data"]
        assert w.shape == (n, k) and t[o["inputs"][2]]["data"].shape == (n,)
        a = np.abs(w)
        assert (a == a[:, :1]).all() and (a > 0).all()
        mant = np.frexp(a[:, 0])[0]
        assert (mant != 0.5).mean() > 0.99   # not powers of two
    assert [o["options"].scalar(0, "b") for o in fcs[:2]] == [0, 1]   # NONE, RELU


def _fused(blob, passes=None):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    if passes is None:
        g.fuse_all()
    else:
        for p in passes:
            getattr(g, p)()
    names = _names(g)
    g.close()
    return names


def test_binaryalexnet_dense_fused_node_list():
    names = _fused(zoo.binaryalexnet(batch=1, dense="fully_connected"))
    assert _tail(names, "MAX_POOL_2D+MUL+ADD+RESHAPE+LceQuantize") == [
        "MAX_POOL_2D+MUL+ADD+RESHAPE+LceQuantize", FUSED + "+MUL+ADD+LceQuantize", FUSED + "+MUL+ADD+LceQuantize",
        "LceDequantize", "builtin:9", "builtin:18", "builtin:0", "builtin:25"]   # 1000 classes: N % 64 != 0
    assert names.count("MAX_POOL_2D+MUL+ADD+LceQuantize") == 2


def test_xnornet_dense_fused_node_list():
    names = _fused(zoo.xnornet(batch=1, dense="fully_connected"))
    assert _tail(names, "MAX_POOL_2D+MUL+ADD+RESHAPE+LceQuantize") == [
        "MAX_POOL_2D+MUL+ADD+RESHAPE+LceQuantize", FUSED + "+LceQuantize", FUSED, "builtin:9", "builtin:25"]


def test_passes_before_it_leave_the_dense_layers():
    """fuse_all runs the pass right after fuse_binary_transpose_convs: the passes before it leave every dense
    layer's LceDequantize, FULLY_CONNECTED, MUL, ADD and LceQuantize (a later pass would take ADD ->
    LceQuantize)."""
    before = PASSES_BUT_FC[:PASSES_BUT_FC.index("fuse_binary_transpose_convs") + 1]
    for blob, removed in ((zoo.binaryalexnet(batch=1, dense="fully_connected"), 2 * 4),
                          (zoo.xnornet(batch=1, dense="fully_connected"), 2 + 1)):
        g = H.HostGraph.from_tflite(blob, device_arena=True)
        n0 = g.num_nodes()
        for p in before:
            getattr(g, p)()
        assert g.num_nodes() == n0
        assert g.fuse_binary_fully_connected() == removed
        g.close()


@pytest.mark.parametrize("bias,bn,quant", [(True, True, True), (False, True, False), (True, False, True),
                                           (False, False, False)])
def test_fused_node_lists(bias, bn, quant):
    blob, _ = _fc_graph(bias=bias, bn=bn, quant=quant)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n0 = g.num_nodes()
    removed = g.fuse_binary_fully_connected()
    assert _names(g) == [FUSED + ("+MUL+ADD" if bn else "") + ("+LceQuantize" if quant else "")]
    assert removed == n0 - 1
    ins = g.node_io(0)[0]
    assert len(ins) == 6 and ins[0] == g.inputs()[0]
    assert ins[2] == -1                                  # +-1.0 weights: no alpha vector
    assert (ins[3] >= 0) == bias and (ins[4] >= 0) == bn and (ins[5] >= 0) == bn
    assert g.node_outputs(0) == g.outputs()
    g.close()
    blob, _ = _fc_graph(bias=bias, bn=bn, quant=quant, alpha=np.full(64, 0.3, F32))
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    assert g.fuse_binary_fully_connected() == n0 - 1 and g.node_io(0)[0][2] >= 0
    g.close()


def test_rank4_input_with_whole_words_fuses():
    blob, _ = _fc_graph(x_shape=(3, 2, 2, 64), n=128)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    assert g.fuse_binary_fully_connected() == 1 and _names(g) == [FUSED]
    g.close()


@pytest.mark.parametrize("variant", ["0.5 weight", "-0.0 weight", "0.0 weight", "magnitudes differ",
                                     "negative alpha", "n 96", "n 1000", "k % 32 under rank-4 q",
                                     "deq second reader", "deq output", "host arena", "mul operand not [N]"])
def test_fusion_preconditions(variant):
    rng = np.random.default_rng(1)
    kw = {}
    w = _weights(rng, 64, 100)
    partial = None
    if variant == "0.5 weight":
        w[3, 7] = 0.5
        kw["weights"] = w
    elif variant == "-0.0 weight":
        w[3, 7] = -0.0
        kw["weights"] = w
    elif variant == "0.0 weight":
        w[5, 0] = 0.0
        kw["weights"] = w
    elif variant == "magnitudes differ":
        w = _weights(rng, 64, 100, np.full(64, 0.75, F32))
        w[9, 50] = np.nextafter(w[9, 50], np.float32(np.inf), dtype=F32)
        kw["weights"] = w
    elif variant == "negative alpha":   # every weight of a row negative is still +-alpha; a NaN row is not
        w[2, :] = np.nan
        kw["weights"] = w
    elif variant == "n 96":
        kw["n"] = 96
    elif variant == "n 1000":
        kw["n"] = 1000
    elif variant == "k % 32 under rank-4 q":
        kw["x_shape"] = (2, 2, 2, 25)           # K = 100, each pixel's 25 signs padded to a word
    elif variant == "deq second reader":
        kw["deq_reader"] = True
    elif variant == "deq output":
        kw["outputs"] = ("deq",)
    elif variant == "mul operand not [N]":
        kw.update(bn=True, mul_shape=(1,))
        partial = [FUSED, "builtin:18", "builtin:0"]   # the layer alone; its MUL and ADD stay
    blob, _ = _fc_graph(**kw)
    g = H.HostGraph.from_tflite(blob, device_arena=variant != "host arena")
    before = _names(g)
    removed = g.fuse_binary_fully_connected()
    if partial is None:
        assert removed == 0 and _names(g) == before, variant
    else:
        assert _names(g) == partial and removed == 1, _names(g)
    g.close()


@pytest.mark.parametrize("case", sorted(S._other_models()))
def test_other_models_keep_their_node_lists(case):
    make, kw = S._other_models()[case]
    blob = make(batch=1, seed=0, image=224, **kw)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n0 = g.num_nodes()
    assert g.fuse_binary_fully_connected() == 0 and g.num_nodes() == n0
    g.close()
    assert _fused(blob) == _fused(blob, PASSES_BUT_FC)
    assert not any(n.startswith(FUSED) or "RESHAPE+" in n for n in _fused(blob))


# ----------------------------------- GPU ----------------------------------- #
def _pack(rng, shape):
    """LceQuantize of random signs on the host: bit 1 <=> negative, tail bits zero."""
    c = shape[-1]
    lead = tuple(shape[:-1])
    bits = np.zeros(lead + (((c + 31) // 32) * 32,), np.uint64)
    bits[..., :c] = rng.integers(0, 2, lead + (c,))
    words = (bits.reshape(lead + (-1, 32)) << np.arange(32, dtype=np.uint64)).sum(-1)
    return words.astype(np.uint32).view(np.int32)


def _unpack(q, x_shape):
    """q's signs as +-1.0 rows [rows, K] of the FULLY_CONNECTED's flattened input."""
    c = x_shape[-1]
    bits = (q.view(np.uint32)[..., None] >> np.arange(32, dtype=np.uint32)) & 1
    bits = bits.reshape(q.shape[:-1] + (-1,))[..., :c]
    x = (1 - 2 * bits.astype(np.int64)).reshape(x_shape)
    k = c if len(x_shape) == 2 else int(np.prod(x_shape[1:]))
    return x.reshape(-1, k)


def _act(y, act):
    lo, hi = {"NONE": (-np.inf, np.inf), "RELU": (0, np.inf), "RELU_N1_TO_1": (-1, 1), "RELU6": (0, 6)}[act]
    return np.minimum(np.maximum(y, F32(lo)), F32(hi)).astype(F32) if act != "NONE" else y


def _sign_words(y):
    n = y.shape[1]
    bits = (y < 0).astype(np.uint64).reshape(y.shape[0], n // 32, 32)
    return (bits << np.arange(32, dtype=np.uint64)).sum(-1).astype(np.uint32).view(np.int32)


def _tflite_loop(x, w):
    """TFLite's float FULLY_CONNECTED inner loop: acc = fl(acc + x_k * w_k) for k = 0 .. K-1, from 0."""
    acc = np.zeros((x.shape[0], w.shape[0]), F32)
    xf, wf = x.astype(F32), w.astype(F32)
    for k in range(x.shape[1]):
        acc = (acc + xf[:, k:k + 1] * wf[None, :, k]).astype(F32)
    return acc


def _fused_ref(q, x_shape, c, act, bn_act, loop=False):
    """The fused node's result: y = act(fl(fl(alpha * D) + b)) [-> bn_act(fl(fl(y * scale) + shift))], D exact.
    loop: D through _tflite_loop instead (+-1 weights only, where every partial sum is exact)."""
    x = _unpack(q, x_shape)
    w = c["w"]
    alpha = np.abs(w[:, 0]).astype(F32)
    if loop:
        y = _tflite_loop(x, w)
    else:
        d = x @ np.sign(w).astype(np.int64).T
        y = (d.astype(F32) * alpha[None, :]).astype(F32)
    if c["b"] is not None:
        y = (y + c["b"][None, :]).astype(F32)
    y = _act(y, act)
    if "scale" in c:
        y = _act(((y * c["scale"][None, :]).astype(F32) + c["shift"][None, :]).astype(F32), bn_act)
    return y


def _run(blob, feeds, fuse):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    removed = g.fuse_binary_fully_connected() if fuse else 0
    g.allocate_tensors()
    for t, v in zip(g.inputs(), feeds):
        g.write(t, v)
    g.invoke()
    outs = [g.read(t) for t in g.outputs()]
    names = _names(g)
    g.close()
    return outs, removed, names


# rows 1, 3, 130, 256 (below, across and at 128-row tiles); K 100, 4096, 9216 and 1000 (K % 256 != 0)
PM1_CASES = [
    dict(x_shape=(1, 100), n=64, bias=True, act="NONE", bn=False, quant=False),
    dict(x_shape=(3, 4096), n=128, bias=False, act="RELU", bn=True, bn_act="NONE", quant=True),
    dict(x_shape=(130, 9216), n=64, bias=True, act="NONE", bn=True, bn_act="RELU6", quant=True),
    dict(x_shape=(256, 100), n=192, bias=True, act="RELU_N1_TO_1", bn=False, quant=True),
    dict(x_shape=(256, 9216), n=4096, bias=False, act="NONE", bn=True, bn_act="NONE", quant=True),
    dict(x_shape=(130, 4096), n=4096, bias=True, act="RELU", bn=False, quant=False),
    dict(x_shape=(1, 9216), n=128, bias=False, act="NONE", bn=True, bn_act="RELU", quant=True),
    dict(x_shape=(3, 1000), n=64, bias=True, act="RELU6", bn=True, bn_act="RELU_N1_TO_1", quant=True),
    dict(x_shape=(256, 4096), n=128, bias=True, act="NONE", bn=False, quant=True),
    dict(x_shape=(130, 2, 2, 64), n=64, bias=True, act="NONE", bn=True, quant=True),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(PM1_CASES)))
def test_gpu_pm1_fused_equals_unfused_and_tflite(case):
    from compute_engine_b200 import capi
    kw = dict(PM1_CASES[case])
    rng = np.random.default_rng(case)
    blob, c = _fc_graph(seed=case, **kw)
    feeds = [_pack(rng, kw["x_shape"])]
    want, _, _ = _run(blob, feeds, False)
    paths = capi.path_counts()
    got, removed, names = _run(blob, feeds, True)
    assert capi.path_counts()[1] > paths[1]            # the mma.sync kernel ran (on the b1 plan)
    assert removed > 0 and names == [FUSED + ("+MUL+ADD" if kw["bn"] else "") +
                                     ("+LceQuantize" if kw["quant"] else "")], names
    for a, b in zip(want, got):
        assert S._same_bits(a, b)
    ref = _fused_ref(feeds[0], kw["x_shape"], c, kw["act"], kw.get("bn_act", "NONE"),
                     loop=kw["n"] * kw["x_shape"][0] <= 256 * 192)
    assert S._same_bits(got[0], ref)
    if kw["quant"]:
        assert S._same_bits(got[1], _sign_words(ref))


ALPHA_CASES = [dict(x_shape=(256, 9216), n=4096, act="NONE", quant=True),
               dict(x_shape=(130, 4096), n=128, act="RELU", quant=False),
               dict(x_shape=(3, 100), n=64, act="NONE", quant=True, bn=True)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(ALPHA_CASES)))
def test_gpu_alpha_fused_is_rounded_twice_and_within_the_bound(case):
    kw = dict(ALPHA_CASES[case])
    rng = np.random.default_rng(100 + case)
    n, k = kw["n"], kw["x_shape"][-1]
    alpha = (rng.uniform(0.5, 1.5, n) / np.sqrt(k)).astype(F32)
    assert (np.frexp(alpha)[0] != 0.5).all()
    blob, c = _fc_graph(seed=case, alpha=alpha, **kw)
    feeds = [_pack(rng, kw["x_shape"])]
    want, _, _ = _run(blob, feeds, False)
    got, removed, _ = _run(blob, feeds, True)
    assert removed > 0
    ref = _fused_ref(feeds[0], kw["x_shape"], c, kw["act"], "NONE")
    assert S._same_bits(got[0], ref)
    # documented bound: K * 2^-24 * sum |a| |w| = K * 2^-24 * K * alpha_o, times the BatchNorm's scale
    scale = np.abs(c["scale"]) if "scale" in c else np.ones(n, F32)
    bound = (k * 2.0 ** -24 * k * alpha.astype(np.float64) * scale)[None, :] + 2.0 ** -22 * np.abs(ref)
    diff = np.abs(got[0].astype(np.float64) - want[0].astype(np.float64))
    assert (diff <= bound).all(), float((diff / bound).max())
    if kw["quant"]:
        flips = got[1] != want[1]
        near = _sign_words(np.where(np.abs(ref) <= bound, F32(-1), F32(1)).astype(F32))
        assert not (flips & ~near).any()   # a sign differs only at a near-tie


@pytest.mark.gpu
def test_gpu_c_entry_and_refusals():
    from compute_engine_b200 import capi
    rng = np.random.default_rng(7)
    rows, k, n = 130, 300, 128
    w = _weights(rng, n, k)
    words = (k + 31) // 32
    filt = np.zeros((n, 1, 1, words), np.uint32)
    for o in range(n):
        for i in range(k):
            if w[o, i] < 0:
                filt[o, 0, 0, i >> 5] |= np.uint32(1 << (i & 31))
    d = capi.BconvDesc(rows, 1, 1, k, 1, 1, n, 1, 1, 1, 1, 1, capi.PADDING_VALID, 1, capi.ACT_NONE,
                       capi.OUT_FLOAT, 1.0, 0)
    plan = capi.BConv2d(d, filt.view(np.int32), np.ones(n, F32), np.zeros(n, F32))
    q = _pack(rng, (rows, k))
    alpha = rng.uniform(0.1, 2, n).astype(F32)
    bias, scale, shift = (rng.uniform(-2, 2, n).astype(F32) for _ in range(3))
    out, pk = plan.run_fused_fc(torch.from_numpy(q).cuda(), alpha, bias, 1, scale, shift, 3)
    c = {"w": w * alpha[:, None], "b": bias, "scale": scale, "shift": shift}
    ref = _fused_ref(q, (rows, k), c, "RELU", "RELU6")
    assert S._same_bits(out.cpu().numpy(), ref) and S._same_bits(pk.cpu().numpy(), _sign_words(ref))
    # a batch of another size re-plans the rows
    out, _ = plan.run_fused_fc(torch.from_numpy(q[:3]).cuda(), packed=False)
    assert S._same_bits(out.cpu().numpy(), _fused_ref(q[:3], (3, k), {"w": w, "b": None}, "NONE", "NONE"))
    with pytest.raises(capi.LceError, match="unknown activation"):
        plan.run_fused_fc(torch.from_numpy(q).cuda(), activation=9)
    d96 = capi.BconvDesc(rows, 1, 1, k, 1, 1, 96, 1, 1, 1, 1, 1, capi.PADDING_VALID, 1, capi.ACT_NONE,
                         capi.OUT_FLOAT, 1.0, 0)
    p96 = capi.BConv2d(d96, filt[:96].view(np.int32), np.ones(96, F32), np.zeros(96, F32))
    with pytest.raises(capi.LceError, match="multiple of 64"):
        p96.run_fused_fc(torch.from_numpy(q).cuda())


def _images(batch, seed, image=224):
    return np.random.default_rng(seed).standard_normal((batch, image, image, 3)).astype(F32)


def _zoo_run(blob, x, passes):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    for p in passes:
        getattr(g, p)()
    names = _names(g)
    g.resize_input(g.inputs()[0], x.shape)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    out = g.read(g.outputs()[0])
    g.close()
    return out, names


@pytest.mark.gpu
def test_gpu_binaryalexnet_dense_fused_equals_unfused():
    """Each graph at its own batch: the unfused graph's LceDequantize keeps its output's shape."""
    blob = zoo.binaryalexnet(batch=256, seed=3, dense="fully_connected")
    x = _images(256, 5)
    want, _ = _zoo_run(blob, x, PASSES_BUT_FC)
    got, names = _zoo_run(blob, x, ("fuse_all",))
    assert names.count(FUSED + "+MUL+ADD+LceQuantize") == 2
    assert np.isfinite(got).all() and S._same_bits(want, got)


@pytest.mark.gpu
def test_gpu_xnornet_dense_fused_is_close_to_unfused():
    blob = zoo.xnornet(batch=256, seed=3, dense="fully_connected")
    x = _images(256, 6)
    want, _ = _zoo_run(blob, x, PASSES_BUT_FC)
    got, names = _zoo_run(blob, x, ("fuse_all",))
    assert FUSED + "+LceQuantize" in names and FUSED in names
    assert np.isfinite(got).all()
    assert np.abs(got - want).max() < 0.05
    assert (got.argmax(1) == want.argmax(1)).mean() >= 0.95


def _arena_fails(blob, batch, preserve):
    """The fused graph at its own batch on arenas poisoned with 0xFF and 0x7F, then captured as a CUDA graph
    and replayed on new inputs, as test_arena_independence does (without its batch resize, which the
    1000-class layer's LceDequantize does not take)."""
    import test_arena_independence as A
    shape = (batch, 224, 224, 3)
    xs = [A.images(shape, "float32", 200 + k) for k in range(3)]
    fails = []
    g = A.graph(blob, shape, True, preserve=preserve)
    want = [A.run(g, x, 0) for x in xs]
    if A.same(want[1], want[2]):
        fails.append("the anchors of x1 and x2 are equal")
    anchor_snap = A.snapshot(g) if preserve else None
    if preserve:
        A.run(g, xs[0], 0)
        anchor_snap = A.snapshot(g)
    for tag, byte in A.POISON:
        out = A.run(g, xs[0], byte)
        if preserve:
            snap = A.snapshot(g)
            d = A.first_difference(g, anchor_snap, snap)
            if d is not None:
                fails.append(f"P-{tag}: {d}")
            d = A.stray_write(g, snap, byte)
            if d is not None:
                fails.append(f"P-{tag}: {d}")
            del snap
        if not A.same(out, want[0]):
            fails.append(f"P-{tag}: {A.describe(want[0], out)}")
    g.enable_cuda_graph(True)
    A.put(g, xs[0])
    out = A.put(g, xs[0])
    if not A.same(out, want[0]):
        fails.append(f"capture on x0: {A.describe(want[0], out)}")
    for (tag, byte), k in zip(A.POISON, (1, 2)):
        out = A.run(g, xs[k], byte)
        if not A.same(out, want[k]):
            fails.append(f"replay of x{k} on arena {tag}: {A.describe(want[k], out)}")
    g.close()
    return fails


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["binaryalexnet", "xnornet"])
@pytest.mark.parametrize("batch,preserve", [(4, True), (256, False)])
def test_gpu_dense_graphs_do_not_depend_on_the_arena(model, batch, preserve):
    blob = getattr(zoo, model)(batch=batch, seed=0, dense="fully_connected")
    fails = _arena_fails(blob, batch, preserve)
    assert not fails, f"{model}(dense='fully_connected') at batch {batch}:\n" + "\n".join(fails)
