"""ReActNet-A: the PRELU builtin, the RPReLU / RSign chain in the binary convolution's epilogue
(lce_b200_bconv2d_run_fused_chain), the stand-alone chain pass (lce_b200_f32_chain_sign) and the
graph fusion that selects between them (Graph::FuseActivationChains).

CPU: the zoo model through both readers, its fused node list, each fusion precondition, PRELU's
broadcast rule. GPU: bit-exact against the oracle convolution plus numpy float32 op by op, on
every binary-convolution kernel, and the whole graph fused vs unfused."""
import collections
import ctypes as C

import numpy as np
import pytest

import lce_testlib as L
import tflite_ref as R
from compute_engine_b200 import host as H
from compute_engine_b200 import zoo
from compute_engine_b200.tflite_writer import TFLiteModel, bconv2d_options


# ----------------------------------- CPU ----------------------------------- #
def test_reactnet_a_readers_agree_and_it_prepares_on_the_host():
    blob = zoo.reactnet_a(batch=2, image=64, seed=1)
    m = R.parse(blob)
    kinds = collections.Counter((o["code"], o["custom"]) for o in m["ops"])
    assert kinds[(32, "LceBconv2d")] == 31 and kinds[(54, "")] == 26
    assert kinds[(32, "LceQuantize")] == 26 and kinds[(2, "")] == 5 and kinds[(1, "")] == 4
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    assert g.num_nodes() == len(m["ops"])
    for i, t in enumerate(m["tensors"]):
        assert g.shape(i) == t["shape"], t["name"]
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (2, 1000)
    g.close()


def test_reactnet_a_fused_node_list():
    g = H.HostGraph.from_tflite(zoo.reactnet_a(batch=2, image=64, seed=1), device_arena=True)
    assert g.fuse_all() == 205 - 50
    names = collections.Counter(g.node_name(i) for i in range(g.num_nodes()))
    assert names == {
        "builtin:3": 1,                                    # stem
        "ADD+LceQuantize": 1,                              # the first block's RSign
        "LceBconv2d+ADD+RPReLU+ADD+LceQuantize": 20,       # 13 x 3x3, 7 same-width 1x1
        "LceBconv2d+ADD+RPReLU": 1,                        # the last 1x1 (the head reads it)
        "LceBconv2d+ADD": 10,                              # the halves of the widening 1x1s
        "builtin:2": 5,                                    # their CONCATENATION
        "RPReLU+ADD+LceQuantize": 5,                       # the chain after each concatenation
        "builtin:1": 4,                                    # stride-2 shortcuts
        "builtin:40": 1, "builtin:9": 1, "builtin:25": 1,  # head
    }
    g.close()


def test_models_without_chains_are_not_changed():
    for make in (zoo.quicknet, zoo.birealnet18):
        g = H.HostGraph.from_tflite(make(batch=1, image=64, seed=2), device_arena=True)
        g.fuse_residual_blocks()
        g.fuse_float_glue()
        before = [g.node_name(i) for i in range(g.num_nodes())]
        assert g.fuse_activation_chains() == 0
        assert [g.node_name(i) for i in range(g.num_nodes())] == before
        g.close()


def _bconv_then(step, shift_shape=(64,), act="NONE", extra_output=False, shift_is_input=False):
    """LceQuantize -> LceBconv2d -> ADD(shortcut) -> `step` (ADD(shift) or PRELU(alpha))."""
    rng = np.random.default_rng(4)
    m = TFLiteModel()
    x = m.add_tensor("x", (1, 6, 6, 64))
    xq = m.add_tensor("xq", (1, 6, 6, 2), np.int32)
    f = m.add_tensor("f", None, np.int32, data=rng.integers(-2**31, 2**31 - 1, (64, 3, 3, 2)).astype(np.int32))
    mul = m.add_tensor("mul", None, np.float32, data=rng.uniform(0.1, 1, 64))
    bias = m.add_tensor("bias", None, np.float32, data=rng.uniform(0.1, 1, 64))
    y = m.add_tensor("y", (1, 6, 6, 64))
    s = m.add_tensor("s", (1, 6, 6, 64))
    o = m.add_tensor("o", (1, 6, 6, 64))
    if shift_is_input:
        v = m.add_tensor("v", shift_shape)
    else:
        v = m.add_tensor("v", None, np.float32, data=rng.uniform(-0.5, 0.5, shift_shape))
    m.add_op("LceQuantize", [x], [xq], custom_options=b"")
    m.add_op("LceBconv2d", [xq, f, mul, bias, -1], [y], custom_options=bconv2d_options(64))
    m.add_op("ADD", [y, x], [s])
    m.add_op(step, [s, v], [o], **({"activation": act} if step == "ADD" else {}))
    m.inputs = [x, v] if shift_is_input else [x]
    m.outputs = [o, s] if extra_output else [o]
    return m.serialize()


@pytest.mark.parametrize("variant", ["shift_not_constant", "shift_not_per_channel", "alpha_not_per_channel",
                                     "add_has_activation", "sum_is_a_graph_output"])
def test_chain_fusion_leaves_the_graph_when_a_precondition_fails(variant):
    step = "PRELU" if variant == "alpha_not_per_channel" else "ADD"
    kw = {"shift_not_constant": dict(shift_is_input=True),
          "shift_not_per_channel": dict(shift_shape=(1, 6, 6, 64)),
          "alpha_not_per_channel": dict(shift_shape=(6, 6, 64)),
          "add_has_activation": dict(act="RELU"),
          "sum_is_a_graph_output": dict(extra_output=True)}[variant]
    blob = _bconv_then(step, **kw)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    assert g.fuse_residual_blocks() == 1
    assert g.fuse_activation_chains() == 0
    assert [g.node_name(i) for i in range(g.num_nodes())] == \
        ["LceQuantize", "LceBconv2d+ADD", "builtin:" + ("54" if step == "PRELU" else "0")]
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=False)   # and the graph prepares unfused
    g.allocate_tensors()
    g.close()
    # the same graph with the precondition met does fuse
    good = _bconv_then(step, shift_shape=(1, 1, 64) if step == "PRELU" else (64,))
    g = H.HostGraph.from_tflite(good, device_arena=True)
    assert g.fuse_residual_blocks() == 1 and g.fuse_activation_chains() == 1
    assert g.node_name(1) == "LceBconv2d+ADD+" + ("PRELU" if step == "PRELU" else "ADD")
    g.close()


def _prelu_graph(x_shape, alpha):
    m = TFLiteModel()
    x = m.add_tensor("x", x_shape)
    a = m.add_tensor("alpha", None, np.float32, data=alpha)
    y = m.add_tensor("y", x_shape)
    m.add_op("PRELU", [x, a], [y])
    m.inputs, m.outputs = [x], [y]
    return m.serialize()


def test_prelu_broadcast_rule():
    for shape in ((1, 1, 8), (4, 8), (1, 4, 4, 8), (1,)):
        g = H.HostGraph.from_tflite(_prelu_graph((2, 4, 4, 8), np.full(shape, 0.25, np.float32)),
                                    device_arena=False)
        g.allocate_tensors()
        g.close()
    for shape in ((4, 1, 8), (8, 1), (2, 2, 4, 4, 8)):
        g = H.HostGraph.from_tflite(_prelu_graph((2, 4, 4, 8), np.full(shape, 0.25, np.float32)),
                                    device_arena=False)
        with pytest.raises(H.HostError, match="PRELU: alpha must have the shape of the input's trailing"):
            g.allocate_tensors()
        g.close()


# --------------------------- CPU reference of PRELU --------------------------- #
def _prelu_ref(x, alpha):
    """TFLite's PRELU (reference/prelu.h) in numpy float32: x >= 0 ? x : x * alpha."""
    return np.where(x >= 0, x, (x * alpha).astype(np.float32)).astype(np.float32)


def _run_op(model, op, vals):
    """One op of a parsed model on the CPU: PRELU here, every other op through tflite_ref."""
    if op["code"] == 54:
        return _prelu_ref(vals[op["inputs"][0]], model["tensors"][op["inputs"][1]]["data"])
    act = [i for i in op["inputs"] if i >= 0 and model["tensors"][i]["data"] is None]
    sub = {"tensors": model["tensors"], "ops": [op], "inputs": act, "outputs": [op["outputs"][0]]}
    return R.run(sub, [vals[i] for i in act])[0][0]


def _run_model(model, inputs):
    vals = dict(zip(model["inputs"], inputs))
    for op in model["ops"]:
        vals[op["outputs"][0]] = _run_op(model, op, vals)
    return [vals[i] for i in model["outputs"]]


def test_cpu_reference_runs_reactnet_a():
    m = R.parse(zoo.reactnet_a(batch=1, image=32, seed=2))
    x = np.random.default_rng(0).standard_normal((1, 32, 32, 3)).astype(np.float32)
    out = _run_model(m, [x])[0]
    assert out.shape == (1, 1000) and np.isfinite(out).all() and np.allclose(out.sum(-1), 1.0, atol=1e-4)


# ----------------------------------- GPU ----------------------------------- #
def _np_chain(s, v, packed):
    """The op sequence in numpy float32: ADD, PRELU, ADD, then ADD + LceQuantize."""
    si, a, so, ss = v
    if si is not None:
        s = (s + si).astype(np.float32)
    if a is not None:
        s = np.where(s >= 0, s, (s * a).astype(np.float32)).astype(np.float32)
    if so is not None:
        s = (s + so).astype(np.float32)
    bits = None
    if packed:
        bits = L.quantize((s + ss).astype(np.float32) if ss is not None else s)
    return s, bits


MASKS = [(1, 1, 1, 1), (0, 1, 1, 1), (1, 0, 1, 1), (1, 1, 0, 1), (1, 1, 1, 0), (0, 0, 0, 1), (0, 0, 0, 0)]
PATHS = {  # environment at plan creation -> the path-counter slot that must run
    "b1": ({"LCE_B200_BCONV_B1": "1"}, 1),
    "int8": ({"LCE_B200_BCONV_B1": "0"}, 1),
    "wgmma": ({"LCE_B200_BCONV_IMMA": "0"}, 0),
    "xor": ({"LCE_B200_BCONV_IMMA": "0", "LCE_B200_BCONV_TC": "0"}, 2),
}


@pytest.mark.gpu
@pytest.mark.parametrize("path", list(PATHS))
def test_gpu_run_fused_chain_is_the_op_sequence(path, monkeypatch):
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import assert_same_bits, dev, gpu_desc, path_counts
    env, slot = PATHS[path]
    for k in ("LCE_B200_BCONV_B1", "LCE_B200_BCONV_IMMA", "LCE_B200_BCONV_TC"):
        monkeypatch.setenv(k, env.get(k, "1"))
    rng = np.random.default_rng(31)
    n = 0
    # 3x3 s1, 3x3 s2, 1x1; M = 162 / 50 / 162 (not multiples of 128); and a zero-padding plan
    # finished by the float correction (CORRECTION mode)
    plans = [(fh, st, c, 1) for fh, st in ((3, 1), (3, 2), (1, 1)) for c in (64, 256, 1024)]
    plans.append((3, 1, 64, 0))
    for fh, st, c, pv in plans:
        case = L.make_bconv_case(500 + n, 2, 9, 9, c, fh, fh, c, stride=(st, st), pad_value=pv)
        kind = 1 if pv == 0 else 0
        conv = L.bconv2d(case.desc, case.inp, case.filt, case.mul, case.bias, case.thr, kind=kind)
        res = rng.standard_normal(conv.shape).astype(np.float32)
        act = L.ACT_RELU if n % 3 == 1 else L.ACT_NONE
        s = (conv + res).astype(np.float32)
        if act == L.ACT_RELU:
            s = np.maximum(s, 0)
        mask = MASKS[n % len(MASKS)]
        vals = [rng.uniform(-0.5, 0.5, c).astype(np.float32), rng.uniform(0.05, 0.5, c).astype(np.float32),
                rng.uniform(-0.5, 0.5, c).astype(np.float32), rng.uniform(-0.5, 0.5, c).astype(np.float32)]
        v = [x if on else None for x, on in zip(vals, mask)]
        packed = n % 2 == 0
        want, want_bits = _np_chain(s, v, packed)
        plan = capi.BConv2d(gpu_desc(capi, case.desc), case.filt, case.mul, case.bias, case.thr)
        if pv == 0:
            plan.set_zero_padding_mode(1)   # LCE_ZERO_PADDING_CORRECTION
        before = path_counts(capi)
        got, bits = plan.run_fused_chain(dev(case.inp), dev(res), act, *[None if x is None else dev(x) for x in v],
                                         packed=packed)
        torch.cuda.synchronize()
        ran = [y - x for x, y in zip(before, path_counts(capi))]
        tag = f"{path} plan {n} ({fh}x{fh} s{st} C{c} pad{pv} mask {mask} packed {packed})"
        if pv == 1:   # the CORRECTION plan may leave the mma.sync kernel for the correction pass
            assert ran[slot] == 1 and sum(ran) == 1, (tag, ran)
        assert_same_bits(got.cpu().numpy(), want, tag)
        if packed:
            assert_same_bits(bits.cpu().numpy(), want_bits, tag + " signs")
        plan.close()
        n += 1


@pytest.mark.gpu
def test_gpu_chain_sign_and_prelu_builtin():
    import torch
    from compute_engine_b200 import capi
    rng = np.random.default_rng(8)
    for shape, alpha_shape in (((2, 5, 7, 96), (1, 1, 96)), ((2, 5, 7, 96), (7, 96)), ((3, 4, 4, 40), (4, 4, 40))):
        x = rng.standard_normal(shape).astype(np.float32)
        alpha = rng.uniform(0.05, 0.5, alpha_shape).astype(np.float32)
        want = _prelu_ref(x, alpha)
        # the builtin through the graph host
        blob = _prelu_graph(shape, alpha)
        g = H.HostGraph.from_tflite(blob, device_arena=True)
        g.allocate_tensors()
        g.write(g.inputs()[0], x)
        g.invoke()
        got = g.read(g.outputs()[0])
        g.close()
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), alpha_shape
    # the stand-alone chain with packing, channels not a multiple of 32, no float output
    x = rng.standard_normal((3, 5, 5, 40)).astype(np.float32)
    v = [rng.uniform(-0.5, 0.5, 40).astype(np.float32) for _ in range(4)]
    v[1] = np.abs(v[1])
    want, bits = _np_chain(x, v, True)
    dv = [torch.from_numpy(a).cuda() for a in v]
    o, pk = capi.chain_sign(torch.from_numpy(x).cuda(), *dv)
    _, pk_only = capi.chain_sign(torch.from_numpy(x).cuda(), None, None, None, dv[3], out=False)
    torch.cuda.synchronize()
    assert np.array_equal(o.cpu().numpy().view(np.uint32), want.view(np.uint32))
    assert np.array_equal(pk.cpu().numpy(), bits)
    assert np.array_equal(pk_only.cpu().numpy(), L.quantize((x + v[3]).astype(np.float32)))


def _check_reactnet_on_gpu(blob, batch, image, seed, final_atol):
    """The unfused graph on the device, op by op on the device's own input tensors: every LCE op
    and PRELU bit exact, the other float builtins within the torch fp32 reference's tolerance;
    then the class probabilities against the CPU graph. Returns the number of LCE ops checked."""
    m = R.parse(blob)
    x = np.random.default_rng(seed).standard_normal((batch, image, image, 3)).astype(np.float32)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.preserve_all_tensors(True)
    g.resize_input(g.inputs()[0], x.shape)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    n_lce = 0
    for op in m["ops"]:
        act = [i for i in op["inputs"] if i >= 0 and m["tensors"][i]["data"] is None]
        want = _run_op(m, op, {i: g.read(i) for i in act})
        got = g.read(op["outputs"][0])
        assert got.shape == want.shape, (op["code"], op["custom"])
        if op["code"] in (32, 54):
            assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (op["code"], op["custom"])
            n_lce += op["code"] == 32
        else:
            scale = max(1.0, float(np.abs(want).max()))
            assert np.allclose(got, want, rtol=1e-4, atol=1e-5 * scale), (op["code"], np.abs(got - want).max())
    got_out = g.read(g.outputs()[0])
    want_out = _run_model(m, [x])[0]
    assert got_out.shape == want_out.shape
    assert np.abs(got_out - want_out).max() <= final_atol
    assert np.allclose(got_out.sum(-1), 1.0, atol=1e-4)
    g.close()
    return n_lce


@pytest.mark.gpu
def test_gpu_reactnet_a_graph():
    blob = zoo.reactnet_a(batch=1, image=64, seed=9)
    assert _check_reactnet_on_gpu(blob, 2, 64, 3, 2e-4) == 31 + 26
    x = np.random.default_rng(5).standard_normal((2, 64, 64, 3)).astype(np.float32)
    outs, names = [], None
    for fuse in (False, True):
        g = H.HostGraph.from_tflite(blob, device_arena=True)
        g.resize_input(g.inputs()[0], x.shape)
        if fuse:
            assert g.fuse_all() > 0
            names = [g.node_name(i) for i in range(g.num_nodes())]
        g.allocate_tensors()
        g.write(g.inputs()[0], x)
        g.invoke()
        outs.append(g.read(g.outputs()[0]))
        g.close()
    assert "LceBconv2d+ADD+RPReLU+ADD+LceQuantize" in names
    assert np.array_equal(outs[0].view(np.uint8), outs[1].view(np.uint8))
