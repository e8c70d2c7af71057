"""DoReFaNet: the zoo model, the MAXIMUM / MINIMUM / ROUND / DIV builtins, the 2-bit quantiser written
as bit planes (lce_b200_f32_quant2_planes) and the graph fusion that runs each 2-bit-activation layer
as a binary convolution over three planes (Graph::FuseQuantizedActivations).

CPU: the model's op, shape and channel counts, one weight magnitude per output channel, both
readers, the other models' bytes and node lists, the bit-plane identity in numpy against a float64
convolution (and a float32 sequential one within the accumulation bound), the pass's node list and
synthesised constants on a host-arena graph, each refused precondition, and the new kernels
compiled without spills. GPU: the four builtins bit for bit against numpy float32, the planes
against numpy and against packing the device's own unfused ops, each fused layer bit-exact against
the integer reference on the mma.sync kernel, the whole graph fused against unfused (first levels
identical, later near-tie flips counted, softmax within 1e-4) eager and under CUDA-graph replay,
and Interpreter.predict across batch sizes."""
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
from test_pooled_signs import OTHER_HASHES as _TEN_HASHES

F32 = np.float32
QUANT, POOL_QUANT = "Quant2", "MAX_POOL_2D+Quant2"
# sha256 of every older model's bytes at the commit before dorefanet was added
OTHER_HASHES = dict(_TEN_HASHES)
OTHER_HASHES.update({
    ("binaryalexnet", 224): "150d60007c51b3398d51c6728d6ccb08693609ff0cd7d1b34ad41f01e2218dac",
    ("binaryalexnet", 64): "5ae6682d3e5fb5e0eed5e38afbdb0e3c8372af6fafd97f9196c7fdb9ee6f9ed0",
    ("xnornet", 224): "1320cd7cfb60937fccfccefd5cdc8d4925628d2f4d363bc3a2a4e1e25732b586",
    ("xnornet", 64): "da1e02290afbbecd8cc170b3fcca5a01c9d88e3e280e8f77ae37df56554db133",
    ("quicknet_small", 224): "cf5f288f7f18222243c282a17af72c6a88e9349fc502c32347f8b83a07aab1b5",
    ("quicknet_small", 64): "19982f8c3c33c9176dd7168775ec7bd2ac246dd28ea363c3b7c84be6e98a6fd8",
})
OTHERS = sorted({name for name, _ in OTHER_HASHES})
# (C_in, C_out, filter) of the quantised convolutions, then (K, N) of the quantised dense layers
QCONVS = [(96, 256, 5), (256, 384, 3), (384, 384, 3), (384, 256, 3)]


# ------------------------------ numpy references ------------------------------ #
def np_levels(x):
    """q = ROUND(MUL(MINIMUM(MAXIMUM(x, 0), 1), 3)), each op in float32 as the builtins compute it"""
    x = np.asarray(x, F32)
    x = np.where(x > 0, x, F32(0))
    x = np.where(x < 1, x, F32(1))
    return np.rint(x * F32(3)).astype(F32)


def np_planes(q):
    """levels [..., C] -> int32 words [..., 3 * C / 32] = [bit 0 | bit 1 | bit 1]"""
    q = np.asarray(q).astype(np.int64)
    p0, p1 = L.pack_signs(-(q & 1).astype(F32)), L.pack_signs(-((q >> 1) & 1).astype(F32))
    return np.concatenate([p0, p1, p1], axis=-1)


def np_maxpool(x, k, s, padding):
    b, h, w, c = x.shape
    if padding == "SAME":
        oh, ow = -(-h // s), -(-w // s)
        ph, pw = max(0, (oh - 1) * s + k - h) // 2, max(0, (ow - 1) * s + k - w) // 2
    else:
        oh, ow, ph, pw = (h - k) // s + 1, (w - k) // s + 1, 0, 0
    y = np.empty((b, oh, ow, c), F32)
    for oy in range(oh):
        for ox in range(ow):
            y0, x0 = oy * s - ph, ox * s - pw
            y[:, oy, ox] = x[:, max(0, y0):min(h, y0 + k), max(0, x0):min(w, x0 + k)].max(axis=(1, 2))
    return y


def synthesise(w, bias):
    """what the pass makes of +-alpha weights [N, kh, kw, C] and a bias: the filter words repeated three
    times per tap, post_mul = fl(-alpha / 6), post_bias = fl(alpha * W / 2 + bias) computed in double"""
    words = L.pack_signs(w)
    alpha = np.abs(w.reshape(w.shape[0], -1)[:, 0]).astype(np.float64)
    wsum = np.sign(w).reshape(w.shape[0], -1).sum(1).astype(np.float64)
    return (np.concatenate([words, words, words], axis=-1), (-alpha / 6.0).astype(F32),
            (alpha * wsum / 2.0 + bias.astype(np.float64)).astype(F32))


def integer_reference(planes, filt, mul, bias, stride, padding):
    """the CPU oracle's plain one-padded LceBconv2d over the three planes"""
    b, h, w, pw = planes.shape
    n, kh, kw, _ = filt.shape
    d = L.BconvDesc(b, h, w, pw * 32, kh, kw, n, 1, stride, stride, 1, 1, {"SAME": 0, "VALID": 1}[padding], 1, 0,
                    L.OUT_FLOAT, 1.0, 0)
    return L.bconv2d(d, planes, filt, mul, bias, None, kind=1)


def conv64(a, w, bias, stride, padding, dtype=np.float64):
    """zero-padded convolution of a [B,H,W,C] with w [N,kh,kw,C], accumulated term by term in `dtype`"""
    b, h, wd, c = a.shape
    n, kh, kw, _ = w.shape
    if padding == "SAME":
        oh, ow = -(-h // stride), -(-wd // stride)
        ph, pw = max(0, (oh - 1) * stride + kh - h) // 2, max(0, (ow - 1) * stride + kw - wd) // 2
    else:
        oh, ow, ph, pw = (h - kh) // stride + 1, (wd - kw) // stride + 1, 0, 0
    ap = np.zeros((b, (oh - 1) * stride + kh, (ow - 1) * stride + kw, c), dtype)
    ap[:, ph:ph + h, pw:pw + wd] = a[:, :ap.shape[1] - ph, :ap.shape[2] - pw]
    out = np.zeros((b, oh, ow, n), dtype)
    wt = w.astype(dtype)
    for fy in range(kh):
        for fx in range(kw):
            win = ap[:, fy:fy + (oh - 1) * stride + 1:stride, fx:fx + (ow - 1) * stride + 1:stride]
            if dtype == np.float64:
                out += win @ wt[:, fy, fx].T
            else:
                for ch in range(c):   # one rounding per term, as a sequential float32 loop
                    out += win[..., ch:ch + 1] * wt[None, None, None, :, fy, fx, ch]
    return out + bias.astype(dtype)


def pm_alpha(rng, shape):
    alpha = rng.uniform(0.02, 0.2, shape[0]).astype(F32)
    sign = (rng.integers(0, 2, shape) * 2 - 1).astype(F32)
    return sign * alpha.reshape((-1,) + (1,) * (len(shape) - 1))


# ----------------------------------- CPU ----------------------------------- #
@pytest.mark.parametrize("image,maps", [(224, [54, 27, 14, 14, 6]), (64, [14, 7, 4, 4, 1])])
def test_op_shape_and_channel_counts(image, maps):
    m = R.parse(zoo.dorefanet(batch=1, image=image, seed=1))
    t = m["tensors"]
    kinds = collections.Counter(o["code"] for o in m["ops"])
    assert dict(kinds) == {3: 5, 17: 3, 22: 1, 9: 3, 25: 1, 55: 7, 57: 7, 18: 6, 116: 6, 42: 6}
    convs = [o for o in m["ops"] if o["code"] == 3]
    assert t[convs[0]["inputs"][1]]["shape"] == (96, 12, 12, 3) and t[convs[0]["outputs"][0]]["shape"] == (1, maps[0], maps[0], 96)
    for op, (cin, cout, k) in zip(convs[1:], QCONVS):
        assert t[op["inputs"][1]]["shape"] == (cout, k, k, cin)
        assert op["options"].scalar(0, "b") == 0 and op["options"].scalar(3, "b") == 0   # SAME, no activation
    pools = [o for o in m["ops"] if o["code"] == 17]
    assert [t[p["outputs"][0]]["shape"][1] for p in pools] == [maps[1], maps[2], maps[4]]
    flat = maps[4] * maps[4] * 256
    fcs = [o for o in m["ops"] if o["code"] == 9]
    assert [t[o["inputs"][1]]["shape"] for o in fcs] == [(4096, flat), (4096, 4096), (1000, 4096)]
    # each quantiser: MAXIMUM(0) -> MINIMUM(1) -> MUL(3) -> ROUND -> DIV(3), one-element constants
    for op in m["ops"]:
        if op["code"] == 116:
            i = m["ops"].index(op)
            chain = m["ops"][i - 3:i + 2]
            assert [o["code"] for o in chain] == [55, 57, 18, 116, 42]
            assert [float(t[o["inputs"][1]]["data"].reshape(-1)[0]) for o in chain if o["code"] != 116] == [0, 1, 3, 3]
            assert all(t[o["inputs"][1]]["data"].size == 1 for o in chain if o["code"] != 116)
            assert m["ops"][i + 2]["code"] in (3, 9)
    assert t[m["outputs"][0]]["shape"] == (1, 1000)


def test_one_weight_magnitude_per_output_channel():
    m = R.parse(zoo.dorefanet(batch=1, image=64, seed=3))
    t = m["tensors"]
    layers = [o for o in m["ops"] if o["code"] in (3, 9)]
    for op in layers[1:-1]:
        w = t[op["inputs"][1]]["data"]
        mag = np.abs(w).reshape(w.shape[0], -1).view(np.uint32)
        assert (mag == mag[:, :1]).all() and (mag[:, 0] != 0).all()
        assert len(np.unique(mag[:, 0])) > w.shape[0] // 2          # alpha differs between channels
        assert 0.4 < (w < 0).mean() < 0.6 and t[op["inputs"][2]]["data"].shape == (w.shape[0],)
    for op in (layers[0], layers[-1]):                               # the stem and the classifier are float
        w = np.abs(t[op["inputs"][1]]["data"]).reshape(-1)
        assert len(np.unique(w[:64])) > 32


def test_readers_agree_host_prepare_and_resize():
    blob = zoo.dorefanet(batch=2, image=64, seed=1)
    m = R.parse(blob)
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    assert g.num_nodes() == len(m["ops"])
    assert _names(g) == [f"builtin:{o['code']}" for o in m["ops"]]
    for i, t in enumerate(m["tensors"]):
        assert g.shape(i) == t["shape"], t["name"]
        if t["data"] is not None and t["data"].size == 1:
            assert g.read(i).reshape(-1)[0] == t["data"].reshape(-1)[0]
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (2, 1000)
    g.resize_input(g.inputs()[0], (3, 64, 64, 3))
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (3, 1000)
    g.close()


def _run_model(model, inputs):
    """The model on the CPU, op by op: MAXIMUM, MINIMUM, ROUND and DIV in numpy float32 as TFLite
    defines them (a > b ? a : b, a < b ? a : b, halves to even, one division and the fused
    activation), every other op through tflite_ref. Returns the outputs and every tensor's value."""
    t = model["tensors"]
    vals = {i: v["data"] for i, v in enumerate(t) if v["data"] is not None}
    vals.update(zip(model["inputs"], inputs))
    for op in model["ops"]:
        code, ins = op["code"], [vals[i] if i >= 0 else None for i in op["inputs"]]
        if code in (55, 57):
            a, b = ins[0], np.asarray(ins[1], F32)
            out = np.array(np.broadcast_to(np.where(a > b if code == 55 else a < b, a, b), a.shape), F32)
        elif code == 116:
            out = np.rint(ins[0])
        elif code == 42:
            out = (ins[0] / np.asarray(ins[1], F32)).astype(F32)
            if op["options"].scalar(0, "b") == 1:
                out = np.maximum(out, F32(0))
        else:
            act = [i for i in op["inputs"] if i >= 0 and t[i]["data"] is None]
            sub = {"tensors": t, "ops": [op], "inputs": act, "outputs": [op["outputs"][0]]}
            out = R.run(sub, [vals[i] for i in act])[0][0]
        vals[op["outputs"][0]] = out
    return [vals[i] for i in model["outputs"]], vals


def test_cpu_reference_runs_and_uses_every_level():
    m = R.parse(zoo.dorefanet(batch=1, image=64, seed=2))
    x = np.random.default_rng(0).standard_normal((2, 64, 64, 3)).astype(F32)
    outs, vals = _run_model(m, [x])
    assert outs[0].shape == (2, 1000) and np.allclose(outs[0].sum(-1), 1.0, atol=1e-4)
    for op in m["ops"]:
        if op["code"] == 42:
            q = np.rint(vals[op["outputs"][0]] * 3)
            assert sorted(np.unique(q)) == [0, 1, 2, 3] and np.array_equal(q, np_levels(vals[m["ops"][m["ops"].index(op) - 4]["inputs"][0]]))


def test_other_models_bytes_are_unchanged():
    for (name, image), want in OTHER_HASHES.items():
        kw = dict(batch=1, image=224, seed=0) if image == 224 else dict(batch=2, image=64, seed=3,
                                                                          input_type="int8")
        assert hashlib.sha256(zoo.MODELS[name](**kw)).hexdigest() == want, (name, image)


# (x shape, C_out, filter, stride, padding): each stride / padding the pass maps, and the dense case
IDENTITY_CASES = [((2, 9, 9, 32), 64, 5, 1, "SAME"), ((2, 8, 7, 64), 64, 3, 1, "SAME"), ((1, 9, 9, 32), 64, 3, 2, "SAME"),
                  ((2, 7, 7, 32), 64, 3, 1, "VALID"), ((5, 1, 1, 512), 128, 1, 1, "VALID")]


@pytest.mark.parametrize("shape,cout,k,stride,padding", IDENTITY_CASES)
def test_bit_plane_identity_in_numpy(shape, cout, k, stride, padding):
    rng = np.random.default_rng(k * 10 + stride)
    x = rng.uniform(-0.3, 1.3, shape).astype(F32)
    w = pm_alpha(rng, (cout, k, k, shape[3]))
    bias = rng.uniform(-0.5, 0.5, cout).astype(F32)
    q = np_levels(x)
    assert sorted(np.unique(q)) == [0, 1, 2, 3]
    filt, mul, pbias = synthesise(w, bias)
    got = integer_reference(np_planes(q), filt, mul, pbias, stride, padding)
    # exact: the levels' integer sum times alpha / 3 in double; q / 3 itself is the float the DIV op gives
    exact = conv64(q.astype(np.float64), w.astype(np.float64), np.zeros(cout), stride, padding) / 3.0 + bias
    ulp = np.spacing(np.maximum(np.abs(exact), np.abs(bias.astype(np.float64))).astype(F32))
    assert got.shape == exact.shape and (np.abs(got - exact) <= 2 * ulp + 2 * np.spacing(np.abs(mul) * 3 * k * k * shape[3])).all()
    # a float32 convolution of the DIV op's output that rounds after every term stays within the
    # accumulation bound K * 2^-24 * sum |a| |w| of the fused result
    a = (q / F32(3)).astype(F32)
    seq = conv64(a, w, bias, stride, padding, dtype=F32)
    kk = k * k * shape[3]
    bound = (kk + 2) * 2.0 ** -24 * (conv64(a.astype(np.float64), np.abs(w).astype(np.float64), np.abs(bias), stride, padding))
    assert (np.abs(seq - got) <= bound + 2 * ulp).all()


def _names(g):
    return [g.node_name(i) for i in range(g.num_nodes())]


def _base(g):
    """fuse_all() without the quantised-activation pass"""
    return (g.fuse_dense_blocks() + g.fuse_residual_blocks() + g.fuse_float_glue() + g.fuse_pooled_signs()
            + g.fuse_channel_gates() + g.fuse_activation_chains() + g.fuse_residual_pairs())


def test_fused_node_list_and_pass_order():
    blob = zoo.dorefanet(batch=2, image=64, seed=1)
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    before = _names(g)
    assert g.fuse_quantized_activations() == 26 and g.fuse_quantized_activations() == 0
    names = _names(g)
    assert len(names) == len(before) - 26
    assert names == ["builtin:3", QUANT, "LceBconv2d", POOL_QUANT, "LceBconv2d", POOL_QUANT, "LceBconv2d", QUANT,
                     "LceBconv2d", "builtin:17", "builtin:22", QUANT, "LceBconv2d", QUANT, "LceBconv2d", "builtin:55",
                     "builtin:57", "builtin:9", "builtin:25"]
    for i, n in enumerate(names):
        if n in (QUANT, POOL_QUANT):
            (ins, outs), (cins, _) = g.node_io(i), g.node_io(i + 1)
            assert len(ins) == 1 and cins[0] == outs[0] and cins[4] == -1 and g.dtype(outs[0]) == np.int32
            assert g.shape(cins[1])[3] == 3 * g.shape(ins[0])[-1] // 32
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (2, 1000)
    g.resize_input(g.inputs()[0], (5, 64, 64, 3))
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (5, 1000) and g.shape(g.node_io(1)[1][0]) == (5, 14, 14, 9)
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    assert g.fuse_all() == 26 and _names(g) == names
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    assert _base(g) == 0 and _names(g) == before
    g.close()


def test_synthesised_constants():
    blob = zoo.dorefanet(batch=1, image=64, seed=5)
    m = R.parse(blob)
    t = m["tensors"]
    layers = [o for o in m["ops"] if o["code"] in (3, 9)][1:-1]
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    g.fuse_all()
    nodes = [i for i, n in enumerate(_names(g)) if n == "LceBconv2d"]
    assert len(nodes) == len(layers) == 6
    for i, op in zip(nodes, layers):
        w, bias = t[op["inputs"][1]]["data"], t[op["inputs"][2]]["data"]
        if w.ndim == 2:
            w = w.reshape(w.shape[0], 1, 1, w.shape[1])
        filt, mul, pbias = synthesise(w, bias)
        ins, _ = g.node_io(i)
        for got, want in zip((g.read(ins[1]), g.read(ins[2]), g.read(ins[3])), (filt, mul, pbias)):
            assert got.dtype == want.dtype and got.shape == want.shape
            assert np.array_equal(got.view(np.uint8), want.view(np.uint8))
    g.close()


def _block(c=64, cout=64, k=3, mixed=False, conv_act="NONE", three=3.0, quant_is_output=False, zero_weight=False,
           pool=False, two_layers=False, dense=False, x_shape=None):
    """x [-> MAX_POOL_2D] -> the quantiser -> CONV_2D (or FULLY_CONNECTED, or two CONV_2D)"""
    rng = np.random.default_rng(7)
    m = TFLiteModel()
    xs = x_shape or ((2, c) if dense else (2, 6, 6, c))
    x = m.add_tensor("x", xs)
    m.inputs = [x]
    cur = x
    if pool:
        cur = m.add_tensor("p", xs)
        m.add_op("MAX_POOL_2D", [x], [cur], padding="SAME", stride=(1, 1), filter=(3, 3))
    for kind, v in (("MAXIMUM", 0.0), ("MINIMUM", 1.0), ("MUL", three), ("ROUND", None), ("DIV", 3.0)):
        nxt = m.add_tensor(kind.lower(), xs)
        ins = [cur] if v is None else [cur, m.add_tensor("c", None, data=np.array([v], F32))]
        m.add_op(kind, ins, [nxt])
        cur = nxt
    m.outputs = []
    for j in range(2 if two_layers else 1):
        w = pm_alpha(rng, (cout, c) if dense else (cout, k, k, c))
        if mixed:
            w.reshape(-1)[5] *= F32(1.5)
        if zero_weight:
            w[3] = 0
        y = m.add_tensor(f"y{j}", (xs[0], cout) if dense else xs[:3] + (cout,))
        ins = [cur, m.add_tensor("w", None, data=w), m.add_tensor("b", None, data=rng.uniform(-1, 1, cout).astype(F32))]
        if dense:
            r = m.add_tensor(f"r{j}", (xs[0], cout))
            m.add_op("FULLY_CONNECTED", ins, [y], activation=conv_act)
            m.add_op("RELU", [y], [r])
            m.outputs.append(r)
        else:
            m.add_op("CONV_2D", ins, [y], padding="SAME", stride=(1, 1), activation=conv_act)
            m.outputs.append(y)
    if quant_is_output:
        m.outputs.append(cur)
    return m.serialize()


def test_block_fuses():
    for kw, want in ((dict(), [QUANT, "LceBconv2d"]), (dict(pool=True), [POOL_QUANT, "LceBconv2d"]),
                     (dict(two_layers=True), [QUANT, "LceBconv2d", "LceBconv2d"]),
                     (dict(dense=True, c=96), [QUANT, "LceBconv2d", "builtin:19"])):
        g = H.HostGraph.from_tflite(_block(**kw), device_arena=False)
        assert g.fuse_quantized_activations() == (5 if kw.get("pool") else 4) and _names(g) == want, kw
        g.allocate_tensors()
        g.close()


@pytest.mark.parametrize("variant", ["mixed_magnitudes", "zero_weight", "conv_activation", "channels_48", "scalar_2",
                                     "quantiser_is_a_graph_output", "too_many_terms", "dense_is_a_graph_output"])
def test_block_refusals(variant):
    kw = {"mixed_magnitudes": dict(mixed=True), "zero_weight": dict(zero_weight=True),
          "conv_activation": dict(conv_act="RELU"), "channels_48": dict(c=48), "scalar_2": dict(three=2.0),
          "quantiser_is_a_graph_output": dict(quant_is_output=True),
          "too_many_terms": dict(c=2 ** 18, k=5, cout=1, x_shape=(1, 1, 1, 2 ** 18)),    # 3 * 25 * 2^18 >= 2^24
          "dense_is_a_graph_output": dict(dense=True)}[variant]
    blob = _block(**kw)
    if variant == "dense_is_a_graph_output":   # drop the RELU reader: the FULLY_CONNECTED output is the graph's
        m = R.parse(blob)
        assert m["ops"][-1]["code"] == 19
        blob = _dense_output_block()
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    before = _names(g)
    assert g.fuse_quantized_activations() == 0 and g.fuse_all() == 0
    assert _names(g) == before
    g.allocate_tensors()   # and the graph prepares unfused
    g.close()


def _dense_output_block():
    m = TFLiteModel()
    x = m.add_tensor("x", (2, 64))
    cur = x
    for kind, v in (("MAXIMUM", 0.0), ("MINIMUM", 1.0), ("MUL", 3.0), ("ROUND", None), ("DIV", 3.0)):
        nxt = m.add_tensor(kind.lower(), (2, 64))
        m.add_op(kind, [cur] if v is None else [cur, m.add_tensor("c", None, data=np.array([v], F32))], [nxt])
        cur = nxt
    y = m.add_tensor("y", (2, 64))
    w = pm_alpha(np.random.default_rng(1), (64, 64))
    m.add_op("FULLY_CONNECTED", [cur, m.add_tensor("w", None, data=w), -1], [y])
    m.inputs, m.outputs = [x], [y]
    return m.serialize()


@pytest.mark.parametrize("name", OTHERS)
def test_other_models_keep_their_node_lists(name):
    blob = zoo.MODELS[name](batch=1, image=64, seed=2)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n = _base(g)
    before = _names(g)
    assert g.fuse_quantized_activations() == 0
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    assert g.fuse_all() == n and _names(g) == before
    g.close()


def test_minmax_div_round_shape_rules():
    for op in ("MAXIMUM", "MINIMUM", "DIV"):
        for b_shape in ((2, 4, 4, 8), (8,), (1, 1, 1, 8), (1,), ()):
            g = H.HostGraph.from_tflite(_binary_graph(op, (2, 4, 4, 8), b_shape), device_arena=False)
            g.allocate_tensors()
            assert g.shape(g.outputs()[0]) == (2, 4, 4, 8)
            g.close()
        for b_shape in ((2, 1, 1, 8), (1, 4, 1, 1), (1, 1, 1, 1, 1), (4, 8)):
            g = H.HostGraph.from_tflite(_binary_graph(op, (2, 4, 4, 8), b_shape), device_arena=False)
            with pytest.raises(H.HostError, match="only same-shape, last-dimension or single-element broadcast"):
                g.allocate_tensors()
            g.close()


def _binary_graph(op, a_shape, b_shape, act="NONE"):
    m = TFLiteModel()
    a = m.add_tensor("a", a_shape)
    y = m.add_tensor("y", a_shape)
    if op == "ROUND":
        m.add_op(op, [a], [y])
        m.inputs, m.outputs = [a], [y]
    else:
        b = m.add_tensor("b", b_shape)
        m.add_op(op, [a, b], [y], **({"activation": act} if op == "DIV" else {}))
        m.inputs, m.outputs = [a, b], [y]
    return m.serialize()


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
    for kernel, count in (("quant2_planes_kernel", 6), ("eltwise_kernel", 7)):
        props = re.findall(r"Function properties for (\S*%s\S*)\n\s*(.*)" % kernel, r.stderr)
        assert len(props) == count, r.stderr
        for name, line in props:
            assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)


# ----------------------------------- GPU ----------------------------------- #
def _special_values(rng, shape):
    """values around the quantiser's thresholds: exact k/6 ties after the MUL, 0 and 1 and their
    neighbours, signed zeros, halves for ROUND, out-of-range values"""
    x = rng.uniform(-0.5, 1.5, shape).astype(F32)
    flat = x.reshape(-1)
    idx = rng.choice(flat.size, flat.size // 4, replace=False)
    base = np.array([0.0, -0.0, 1.0, 0.5, 1 / 6, 0.5 - 1 / 3, 5 / 6, 2.5, -2.5, 0.5 / 3, 1.5 / 3, 2.5 / 3, 1e-40, -1e-40], F32)
    near = np.concatenate([base, np.nextafter(base, F32(2)), np.nextafter(base, F32(-2))])
    flat[idx] = near[rng.integers(0, len(near), idx.size)]
    return x


@pytest.mark.gpu
def test_gpu_builtins_match_numpy_bit_for_bit():
    from test_gpu_parity import assert_same_bits
    rng = np.random.default_rng(2)
    halves = np.arange(-8.5, 9.0, 0.5, dtype=F32)
    for a_shape, b_shape in (((2, 5, 7, 8), (2, 5, 7, 8)), ((2, 5, 7, 12), (12,)), ((3, 5, 7, 6), (1,)), ((2, 9, 4), ())):
        a = _special_values(rng, a_shape) * F32(3)
        a.reshape(-1)[:halves.size] = halves
        b = _special_values(rng, b_shape if b_shape else (1,)).reshape(b_shape)
        b[b == 0] = F32(3)
        for op in ("MAXIMUM", "MINIMUM", "DIV", "ROUND"):
            acts = ("NONE", "RELU") if op == "DIV" else ("NONE",)
            for act in acts:
                with np.errstate(all="ignore"):
                    want = {"MAXIMUM": lambda: np.where(a > b, a, b), "MINIMUM": lambda: np.where(a < b, a, b),
                            "DIV": lambda: a / b, "ROUND": lambda: np.rint(a)}[op]().astype(F32)
                if act == "RELU":
                    want = np.maximum(want, F32(0))
                g = H.HostGraph.from_tflite(_binary_graph(op, a_shape, b_shape, act), device_arena=True)
                g.allocate_tensors()
                g.write(g.inputs()[0], a)
                if op != "ROUND":
                    g.write(g.inputs()[1], b)
                g.invoke()
                assert_same_bits(g.read(g.outputs()[0]), np.ascontiguousarray(np.broadcast_to(want, a_shape)),
                                 f"{op} {a_shape} {b_shape} {act}")
                g.close()
    # MAXIMUM(-0, +0) and MINIMUM(+0, -0) are the second operand, as a > b ? a : b
    for op, a0, b0 in (("MAXIMUM", -0.0, 0.0), ("MINIMUM", 0.0, -0.0), ("MAXIMUM", np.nan, 0.0)):
        g = H.HostGraph.from_tflite(_binary_graph(op, (4,), (4,)), device_arena=True)
        g.allocate_tensors()
        g.write(g.inputs()[0], np.full(4, a0, F32))
        g.write(g.inputs()[1], np.full(4, b0, F32))
        g.invoke()
        assert_same_bits(g.read(g.outputs()[0]), np.full(4, b0, F32), op)
        g.close()


def _quantiser_graph(shape, pool):
    """the unfused [MAX_POOL_2D ->] MAXIMUM -> MINIMUM -> MUL -> ROUND as a graph"""
    m = TFLiteModel()
    x = m.add_tensor("x", shape)
    cur, ys = x, shape
    if pool:
        k, s, padding = pool
        oh = -(-shape[1] // s) if padding == "SAME" else (shape[1] - k) // s + 1
        ow = -(-shape[2] // s) if padding == "SAME" else (shape[2] - k) // s + 1
        ys = (shape[0], oh, ow, shape[3])
        cur = m.add_tensor("p", ys)
        m.add_op("MAX_POOL_2D", [x], [cur], padding=padding, stride=(s, s), filter=(k, k))
    for kind, v in (("MAXIMUM", 0.0), ("MINIMUM", 1.0), ("MUL", 3.0), ("ROUND", None)):
        nxt = m.add_tensor(kind.lower(), ys)
        m.add_op(kind, [cur] if v is None else [cur, m.add_tensor("c", None, data=np.array([v], F32))], [nxt])
        cur = nxt
    m.inputs, m.outputs = [x], [cur]
    return m.serialize()


# the model's four map shapes (batch 2) with the pool in front of each quantiser, and a ragged one
PLANE_GRID = [((2, 54, 54, 96), None), ((2, 54, 54, 256), (3, 2, "SAME")), ((2, 27, 27, 384), (3, 2, "SAME")),
              ((2, 14, 14, 384), None), ((2, 14, 14, 256), (3, 2, "VALID")), ((3, 11, 7, 160), (3, 2, "SAME")),
              ((3, 11, 7, 32), (2, 1, "VALID")), ((5, 1, 1, 9216), None)]


@pytest.mark.gpu
def test_gpu_planes_match_numpy_and_the_unfused_ops():
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import assert_same_bits, dev
    rng = np.random.default_rng(4)
    for shape, pool in PLANE_GRID:
        x = _special_values(rng, shape)
        pooled = np_maxpool(x, *pool) if pool else x
        want = np_planes(np_levels(pooled))
        code = None if pool is None else ((pool[0], pool[0]), (pool[1], pool[1]),
                                          {"SAME": capi.PADDING_SAME, "VALID": capi.PADDING_VALID}[pool[2]], capi.ACT_NONE)
        got = capi.quant2_planes(dev(x), code)
        torch.cuda.synchronize()
        assert_same_bits(got.cpu().numpy(), want, f"{shape} {pool}")
        g = H.HostGraph.from_tflite(_quantiser_graph(shape, pool), device_arena=True)
        g.allocate_tensors()
        g.write(g.inputs()[0], x)
        g.invoke()
        assert_same_bits(np_planes(g.read(g.outputs()[0])), want, f"{shape} {pool} (unfused ops)")
        g.close()
    with pytest.raises(capi.LceError, match="multiple of 32"):
        capi.quant2_planes(torch.zeros(1, 4, 4, 48, device="cuda"))


@pytest.mark.gpu
def test_gpu_fused_layers_are_bit_exact_on_mma_sync():
    """Each quantised layer of the model as its own fused graph: the device's planes and binary
    convolution against the CPU oracle's integer reference on the same input, one mma.sync launch."""
    from compute_engine_b200 import capi
    from test_gpu_parity import assert_same_bits, path_counts
    rng = np.random.default_rng(9)
    cases = [((2, 27, 27, 96), 256, 5, False), ((2, 14, 14, 256), 384, 3, False), ((2, 14, 14, 384), 384, 3, False),
             ((2, 14, 14, 384), 256, 3, False), ((3, 9216), 4096, 1, True), ((3, 4096), 4096, 1, True)]
    for xs, cout, k, dense in cases:
        c = xs[-1]
        blob = _block(c=c, cout=cout, k=k, dense=dense, x_shape=xs)
        m = R.parse(blob)
        op = [o for o in m["ops"] if o["code"] in (3, 9)][0]
        w, bias = m["tensors"][op["inputs"][1]]["data"], m["tensors"][op["inputs"][2]]["data"]
        x = _special_values(rng, xs)
        g = H.HostGraph.from_tflite(blob, device_arena=True)
        assert g.fuse_all() == 4
        g.preserve_all_tensors(True)
        g.allocate_tensors()
        g.write(g.inputs()[0], x)
        before = path_counts(capi)
        g.invoke()
        g.synchronize()
        ran = [b - a for a, b in zip(before, path_counts(capi))]
        assert ran == [0, 1, 0], (xs, ran)
        planes = np_planes(np_levels(x)).reshape((xs[0], 1, 1, -1) if dense else xs[:3] + (-1,))
        assert_same_bits(g.read(g.node_io(0)[1][0]), planes, str(xs))
        filt, mul, pbias = synthesise(w.reshape(cout, 1, 1, c) if dense else w, bias)
        want = integer_reference(planes, filt, mul, pbias, 1, "VALID" if dense else "SAME")
        assert_same_bits(g.read(g.node_io(1)[1][0]), want, f"{xs} -> {cout}")
        g.close()


def _gpu_run(blob, x, fused, preserve):
    """an eager step and a CUDA-graph replay; returns both outputs and, from the eager step with
    every tensor kept, each quantiser's levels (from the DIV output or the planes)"""
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.resize_input(g.inputs()[0], x.shape)
    g.fuse_all() if fused else _base(g)
    g.preserve_all_tensors(preserve)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    eager = g.read(g.outputs()[0])
    levels = []
    if preserve:
        for i, n in enumerate(_names(g)):
            if n in (QUANT, POOL_QUANT):
                p = g.read(g.node_io(i)[1][0]).view(np.uint32)
                cw = p.shape[-1] // 3
                bits = lambda words: ((words[..., None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(words.shape[:-1] + (-1,))
                levels.append((bits(p[..., :cw]) + 2 * bits(p[..., cw:2 * cw])).reshape(x.shape[0], -1).astype(np.int8))
            elif n == "builtin:116":
                levels.append(g.read(g.node_io(i)[1][0]).reshape(x.shape[0], -1).astype(np.int8))
    g.enable_cuda_graph(True)
    g.write(g.inputs()[0], x)
    g.invoke()   # capture
    g.write(g.inputs()[0], x)
    g.invoke()   # replay
    replay = g.read(g.outputs()[0])
    g.close()
    return eager, replay, levels


@pytest.mark.gpu
def test_gpu_whole_graph_fused_against_unfused():
    blob = zoo.dorefanet(batch=1, image=224, seed=4, input_type="int8")
    x = np.random.default_rng(6).integers(-128, 128, (4, 224, 224, 3)).astype(np.int8)
    flips = None
    for preserve in (True, False):
        ref = _gpu_run(blob, x, False, preserve)
        got = _gpu_run(blob, x, True, preserve)
        assert np.isfinite(got[0]).all() and np.allclose(got[0].sum(-1), 1.0, atol=1e-4)
        # each arm is deterministic: replay equals eager, bit for bit
        assert np.array_equal(got[0].view(np.uint8), got[1].view(np.uint8)), preserve
        assert np.array_equal(ref[0].view(np.uint8), ref[1].view(np.uint8)), preserve
        assert np.abs(got[0] - ref[0]).max() <= 1e-4, (preserve, np.abs(got[0] - ref[0]).max())
        if preserve:
            assert len(ref[2]) == len(got[2]) == 6
            # the levels entering the first quantised layer come from the same float stem: identical
            assert np.array_equal(ref[2][0], got[2][0])
            flips = [int((a != b).sum()) for a, b in zip(ref[2], got[2])]
            sizes = [a.size for a in ref[2]]
            print("near-tie level flips per quantiser:", flips, "of", sizes)
            # later layers: a float-accumulation difference moves a level only at a near-tie
            for f, n, a, b in zip(flips, sizes, ref[2], got[2]):
                assert f <= max(8, n // 2000), (flips, sizes)
                assert np.abs(a.astype(np.int16) - b).max() <= 1
    assert flips is not None


@pytest.mark.gpu
def test_gpu_interpreter_predict_across_batch_sizes():
    from compute_engine_b200.interpreter import Interpreter
    blob = zoo.dorefanet(batch=3, image=224, seed=5)
    it, ref = Interpreter(blob), Interpreter(blob, fuse=False)
    try:
        assert it.fused_nodes_removed == 26 and ref.fused_nodes_removed == 0
        for b in (3, 5, 3):
            x = np.random.default_rng(b).standard_normal((b, 224, 224, 3)).astype(F32)
            got, want = it.predict(x), ref.predict(x)
            assert got.shape == (b, 1000) and np.abs(got - want).max() <= 1e-4, b
    finally:
        it.close()
        ref.close()
