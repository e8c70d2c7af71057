"""XNOR-Net++: ADD / MUL by a per-position [1,H,W,C] operand, the scaled block tail in the binary
convolution's epilogue (lce_b200_bconv2d_run_fused_scale), the one-pass tail
(lce_b200_f32_scale_sign) and the graph fusion that selects it (Graph::FuseSpatialScales).

CPU: the zoo model's ops and Gamma shapes, the CPU reference, the broadcast rule, the fused node
list, each fusion precondition, every registered model untouched by the pass, the new kernel
instances' build. GPU: bit-exact against `run` plus numpy float32 on every binary-convolution path
and at full launch sizes, the one-pass tail, and the whole graph fused vs unfused, against the CPU
graph and through Interpreter.predict."""
import collections
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
from compute_engine_b200.tflite_writer import TFLiteModel, bconv2d_options

SCALED = "LceBconv2d+MUL+ADD"
SIGN_TAIL = "+MUL+ADD+LceQuantize"
# every pass of fuse_all() but fuse_spatial_scales, in fuse_all()'s order
OTHER_PASSES = ("fuse_dense_blocks", "fuse_residual_blocks", "fuse_float_glue", "fuse_grouped_conv_affine",
                "fuse_quantized_activations", "fuse_pooled_signs", "fuse_channel_gates",
                "fuse_activation_chains", "fuse_residual_pairs")


def _names(g):
    return [g.node_name(i) for i in range(g.num_nodes())]


def _act_ref(t, act):
    if act == L.ACT_RELU:
        return np.maximum(t, np.float32(0))
    if act == L.ACT_RELU6:
        return np.minimum(np.maximum(t, np.float32(0)), np.float32(6))
    if act == L.ACT_RELU_N1_TO_1:
        return np.minimum(np.maximum(t, np.float32(-1)), np.float32(1))
    return t


def _scale_tail_ref(y, scale, residual=None, act=L.ACT_NONE, sign_scale=None, sign_shift=None):
    """MUL(scale [OH, OW, C]) -> ADD(residual) with its activation, then the signs of
    MUL(sign_scale) -> ADD(sign_shift): the op sequence in numpy float32."""
    t = (y * scale.reshape((1,) + scale.shape[-3:])).astype(np.float32)
    if residual is not None:
        t = (t + residual).astype(np.float32)
    t = _act_ref(t, act)
    s = t
    if sign_scale is not None:
        s = (s * sign_scale).astype(np.float32)
    if sign_shift is not None:
        s = (s + sign_shift).astype(np.float32)
    return t, L.quantize(s)


# ----------------------------------- CPU ----------------------------------- #
@pytest.mark.parametrize("image", [224, 64])
def test_xnornetpp_ops_and_gamma_shapes(image):
    m = R.parse(zoo.xnornetpp(batch=2, image=image, seed=1))
    kinds = collections.Counter((o["code"], o["custom"]) for o in m["ops"])
    assert kinds == {(32, "LceBconv2d"): 16, (32, "LceQuantize"): 16, (18, ""): 32, (0, ""): 32,
                     (3, ""): 4, (1, ""): 3, (17, ""): 1, (40, ""): 1, (9, ""): 1, (25, ""): 1}
    t = m["tensors"]
    side = image // 4
    shapes = []
    for k, op in enumerate(m["ops"]):
        if op["custom"] != "LceBconv2d":
            continue
        assert np.all(t[op["inputs"][2]]["data"] == 1) and np.all(t[op["inputs"][3]]["data"] == 0)
        nxt = m["ops"][k + 1]
        assert nxt["code"] == 18 and nxt["inputs"][0] == op["outputs"][0]
        gamma = t[nxt["inputs"][1]]
        assert gamma["data"] is not None and np.all(gamma["data"] > 0)
        assert gamma["shape"] == (1,) + t[op["outputs"][0]]["shape"][1:]
        shapes.append(gamma["shape"])
        # Gamma = alpha[C] x beta[OH] x gamma[OW]: rank 1 in every pair of axes
        g3 = gamma["data"][0].astype(np.float64)
        ratio = g3 / g3[:1, :1, :]
        assert np.allclose(ratio, ratio[:, :, :1], rtol=1e-5)
        assert m["ops"][k + 2]["code"] == 0
    want = [(1, side >> s, side >> s, 64 << s) for s in range(4) for _ in range(4)]
    assert shapes == want
    assert "xnornetpp" not in zoo.MODELS


def test_cpu_reference_runs_xnornetpp():
    m = R.parse(zoo.xnornetpp(batch=1, image=32, seed=2))
    x = np.random.default_rng(0).standard_normal((2, 32, 32, 3)).astype(np.float32)
    out = R.run(m, [x])[0][0]
    assert out.shape == (2, 1000) and np.isfinite(out).all() and np.allclose(out.sum(-1), 1.0, atol=1e-4)


def _binary_graph(op, a_shape, b_shape, act="NONE"):
    m = TFLiteModel()
    a, b, y = m.add_tensor("a", a_shape), m.add_tensor("b", b_shape), m.add_tensor("y", a_shape)
    m.add_op(op, [a, b], [y], activation=act)
    m.inputs, m.outputs = [a, b], [y]
    return m.serialize()


# b shapes that are a's trailing dimensions after leading 1s, newly accepted
TRAILING = [((2, 8, 8, 8), (1, 8, 8, 8)), ((2, 8, 8, 8), (8, 8, 8)), ((2, 8, 8, 8), (8, 8)),
            ((2, 8, 8, 8), (1, 1, 8, 8)), ((3, 5, 7, 4), (1, 5, 7, 4)), ((2, 6, 40), (6, 40))]


@pytest.mark.parametrize("op", ["ADD", "MUL"])
def test_trailing_broadcasts_are_accepted(op):
    for a_shape, b_shape in TRAILING:
        g = H.HostGraph.from_tflite(_binary_graph(op, a_shape, b_shape), device_arena=False)
        g.allocate_tensors()
        assert g.shape(g.outputs()[0]) == a_shape
        g.close()


@pytest.mark.parametrize("op", ["MAXIMUM", "MINIMUM", "DIV"])
def test_other_binary_builtins_keep_their_rule(op):
    for a_shape, b_shape in TRAILING:
        g = H.HostGraph.from_tflite(_binary_graph(op, a_shape, b_shape), device_arena=False)
        with pytest.raises(H.HostError, match="only same-shape, last-dimension or single-element broadcast"):
            g.allocate_tensors()
        g.close()


@pytest.mark.parametrize("pad_values", [0, 1])
def test_xnornetpp_fused_node_list(pad_values):
    g = H.HostGraph.from_tflite(zoo.xnornetpp(batch=2, image=224, seed=1, pad_values=pad_values),
                                device_arena=True)
    n0 = g.num_nodes()
    assert g.fuse_all() == 15 * 5 + 2 + 1
    names = collections.Counter(_names(g))
    assert g.num_nodes() == n0 - 78
    assert names == {
        SCALED + SIGN_TAIL: 15,                    # each block with the next block's sign
        SCALED: 1,                                 # the last block (the head reads it)
        "builtin:18": 1, "ADD+LceQuantize": 1,     # the first block's BatchNorm and sign
        "builtin:3": 4, "builtin:1": 3, "builtin:17": 1,   # stem, downsampling shortcuts
        "builtin:40": 1, "builtin:9": 1, "builtin:25": 1,  # head
    }
    g.close()
    g = H.HostGraph.from_tflite(zoo.xnornetpp(batch=2, image=224, seed=1, pad_values=pad_values),
                                device_arena=True)
    assert g.fuse_spatial_scales() == 15 * 5 + 2
    g.close()


def _model_configs():
    one_padded = ("realtobinarynet", "binarydensenet28", "binarydensenet37", "binarydensenet37_dilated",
                  "binarydensenet45", "meliusnet22", "binaryalexnet", "xnornet")
    for name, make in zoo.MODELS.items():
        for image in (224, 64):
            yield name, make, dict(image=image)
            if name in one_padded:
                yield name, make, dict(image=image, pad_values=1)


@pytest.mark.parametrize("name,make,kw", list(_model_configs()),
                         ids=[f"{n}-{'-'.join(str(v) for v in kw.values())}" for n, _, kw in _model_configs()])
def test_registered_models_are_not_matched(name, make, kw):
    blob = make(batch=2, seed=2, **kw)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    before = _names(g)
    assert g.fuse_spatial_scales() == 0
    assert _names(g) == before
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n = sum(getattr(g, p)() for p in OTHER_PASSES)
    want = _names(g)
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    assert g.fuse_all() == n
    assert _names(g) == want
    g.close()


def _scaled_block(gamma="const", gamma_shape=(1, 6, 6, 64), mul_act="NONE", add_act="NONE",
                  bn_act="NONE", output_t=False, other_reader=None, shortcut_later=False,
                  sign_tail=True):
    """LceQuantize -> LceBconv2d -> MUL(gamma) -> ADD(shortcut) [-> MUL -> ADD -> LceQuantize] on x
    [2, 6, 6, 64]; gamma a constant unless `gamma` == "input". other_reader: "y", "t" or "o", a
    tensor that a RELU also reads (its output a graph output)."""
    rng = np.random.default_rng(5)
    m = TFLiteModel()
    x = m.add_tensor("x", (2, 6, 6, 64))
    f32 = lambda name, shape, lo=-0.5, hi=0.5: m.add_tensor(name, None, np.float32,
                                                            data=rng.uniform(lo, hi, shape))
    xq = m.add_tensor("xq", (2, 6, 6, 2), np.int32)
    filt = m.add_tensor("f", None, np.int32, data=rng.integers(-2**31, 2**31 - 1, (64, 3, 3, 2)).astype(np.int32))
    y = m.add_tensor("y", (2, 6, 6, 64))
    g = m.add_tensor("g", gamma_shape) if gamma == "input" else f32("g", gamma_shape, 0.5, 1.5)
    t, o = m.add_tensor("t", (2, 6, 6, 64)), m.add_tensor("o", (2, 6, 6, 64))
    m.add_op("LceQuantize", [x], [xq], custom_options=b"")
    sc = x
    if shortcut_later:   # the shortcut is computed after the convolution
        sc = m.add_tensor("sc", (2, 6, 6, 64))
    m.add_op("LceBconv2d", [xq, filt, f32("mul", 64, 1, 1), f32("bias", 64, 0, 0), -1], [y],
             custom_options=bconv2d_options(64))
    if shortcut_later:
        m.add_op("RELU", [x], [sc])
    m.add_op("MUL", [y, g], [t], activation=mul_act)
    m.add_op("ADD", [t, sc], [o], activation=add_act)
    outs = [o]
    if sign_tail:
        s1, s2 = m.add_tensor("s1", (2, 6, 6, 64)), m.add_tensor("s2", (2, 6, 6, 64))
        q = m.add_tensor("q", (2, 6, 6, 2), np.int32)
        m.add_op("MUL", [o, f32("scale", 64, 0.5, 1.5)], [s1])
        m.add_op("ADD", [s1, f32("shift", 64)], [s2], activation=bn_act)
        m.add_op("LceQuantize", [s2], [q], custom_options=b"")
        outs.append(q)
    if other_reader is not None:
        r = m.add_tensor("r", (2, 6, 6, 64))
        m.add_op("RELU", [{"y": y, "t": t, "o": o}[other_reader]], [r])
        outs.append(r)
    if output_t:
        outs.append(t)
    m.inputs = [x, g] if gamma == "input" else [x]
    m.outputs = outs
    return m.serialize()


def test_scaled_block_fuses():
    for kw, name, removed in ((dict(), SCALED + SIGN_TAIL, 5), (dict(sign_tail=False), SCALED, 2),
                              (dict(add_act="RELU"), SCALED + SIGN_TAIL, 5),
                              (dict(gamma_shape=(6, 6, 64)), SCALED + SIGN_TAIL, 5),
                              (dict(other_reader="o"), SCALED + SIGN_TAIL, 5),   # the sum is the stream
                              (dict(bn_act="RELU"), SCALED, 2)):   # the sign tail stays apart
        g = H.HostGraph.from_tflite(_scaled_block(**kw), device_arena=True)
        assert g.fuse_spatial_scales() == removed, kw
        assert g.node_name(1) == name, kw
        g.close()


@pytest.mark.parametrize("variant", ["gamma_not_constant", "gamma_per_channel", "gamma_one_row",
                                     "mul_has_activation", "conv_output_has_another_reader",
                                     "product_has_another_reader", "product_is_a_graph_output",
                                     "shortcut_computed_later"])
def test_scale_fusion_leaves_the_graph_when_a_precondition_fails(variant):
    kw = {"gamma_not_constant": dict(gamma="input"),
          "gamma_per_channel": dict(gamma_shape=(1, 1, 1, 64)),
          "gamma_one_row": dict(gamma_shape=(6, 64)),
          "mul_has_activation": dict(mul_act="RELU"),
          "conv_output_has_another_reader": dict(other_reader="y"),
          "product_has_another_reader": dict(other_reader="t"),
          "product_is_a_graph_output": dict(output_t=True),
          "shortcut_computed_later": dict(shortcut_later=True)}[variant]
    blob = _scaled_block(**kw)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    before = _names(g)
    assert g.fuse_spatial_scales() == 0
    assert _names(g) == before
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=False)   # and the graph prepares unfused
    g.allocate_tensors()
    g.close()


def test_scale_instances_compile_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "scale.cu"
    src.write_text('#include "lce_b200_imma.cuh"\n' + "".join(
        f"template __global__ void lce::bconv_imma_kernel<{v}, LCE_OUT_FLOAT, {b1}, false, true, false, true>"
        "(const lce::ConvKParams);\n" for v in (1, 2, 4) for b1 in ("true", "false")))
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xptxas=-v", "-cubin", "-I", os.path.join(repo, "include"),
                        "-I", os.path.join(repo, "compute_engine_b200", "csrc"), str(src),
                        "-o", str(tmp_path / "scale.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S*bconv_imma_kernel\S*)\n\s*(.*)", r.stderr)
    assert len(props) == 6, r.stderr
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)


# ----------------------------------- GPU ----------------------------------- #
@pytest.mark.gpu
def test_gpu_scale_sign_matches_numpy_at_4_byte_offsets():
    import torch
    from compute_engine_b200 import capi
    rng = np.random.default_rng(21)
    acts = (L.ACT_NONE, L.ACT_RELU, L.ACT_RELU6, L.ACT_RELU_N1_TO_1)
    for n, (shape, has_res, has_sc, has_sh, packed) in enumerate((
            ((3, 5, 7, 96), 1, 1, 1, 1), ((2, 4, 4, 40), 0, 1, 1, 1), ((4, 1, 1, 64), 1, 0, 1, 1),
            ((2, 7, 7, 512), 1, 1, 0, 1), ((1, 3, 9, 33), 0, 0, 0, 0), ((5, 6, 6, 64), 1, 0, 0, 1),
            ((2, 3, 3, 8), 0, 1, 1, 0))):
        act = acts[n % 4]
        x = rng.standard_normal(shape).astype(np.float32)
        scale = rng.uniform(-1.5, 1.5, shape[1:]).astype(np.float32)
        res = rng.standard_normal(shape).astype(np.float32) if has_res else None
        sc = rng.uniform(0.5, 1.5, shape[-1]).astype(np.float32) if has_sc else None
        sh = rng.uniform(-0.5, 0.5, shape[-1]).astype(np.float32) if has_sh else None
        want, bits = _scale_tail_ref(x, scale, res, act, sc, sh)

        def at4(a):   # the array one float into a device buffer: a 4-byte aligned view
            if a is None:
                return None
            buf = torch.empty(a.size + 1, dtype=torch.float32, device="cuda")
            v = buf[1:].view(a.shape)
            v.copy_(torch.from_numpy(a))
            return v
        out = at4(np.zeros(shape, np.float32))
        o, pk = capi.scale_sign(at4(x), at4(scale), at4(res), act, at4(sc), at4(sh), out=out, packed=bool(packed))
        torch.cuda.synchronize()
        tag = (shape, has_res, has_sc, has_sh, packed, act)
        assert np.array_equal(o.cpu().numpy().view(np.uint32), want.view(np.uint32)), tag
        if packed:
            assert np.array_equal(pk.cpu().numpy(), bits), tag
    # the signs alone, and in place
    x = rng.standard_normal((2, 5, 5, 64)).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, (5, 5, 64)).astype(np.float32)
    sh = rng.uniform(-0.5, 0.5, 64).astype(np.float32)
    d = lambda v: torch.from_numpy(v).cuda()
    _, pk = capi.scale_sign(d(x), d(scale), sign_shift=d(sh), out=False)
    xd = d(x)
    o, _ = capi.scale_sign(xd, d(scale), out=xd, packed=False)
    torch.cuda.synchronize()
    want, bits = _scale_tail_ref(x, scale, sign_shift=sh)
    assert np.array_equal(pk.cpu().numpy(), bits)
    assert np.array_equal(xd.cpu().numpy().view(np.uint32), want.view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("op", ["ADD", "MUL"])
@pytest.mark.parametrize("a_shape,b_shape", TRAILING)
def test_gpu_trailing_broadcast_matches_numpy(op, a_shape, b_shape):
    rng = np.random.default_rng(len(b_shape) * 10 + b_shape[-1])
    for act in ("NONE", "RELU"):
        a = rng.standard_normal(a_shape).astype(np.float32)
        b = rng.standard_normal(b_shape).astype(np.float32)
        want = (a + b if op == "ADD" else a * b).astype(np.float32)
        if act == "RELU":
            want = np.maximum(want, np.float32(0))
        g = H.HostGraph.from_tflite(_binary_graph(op, a_shape, b_shape, act), device_arena=True)
        g.allocate_tensors()
        g.write(g.inputs()[0], a)
        g.write(g.inputs()[1], b)
        g.invoke()
        got = g.read(g.outputs()[0])
        g.close()
        assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32)), act


# (filter, stride, C_in, C_out, image, pad value, zero-padding mode or None, batch): 7x7 and 14x14
# images so 128-row tiles span several images and M is not a multiple of the tile; 96 channels run
# on another kernel than mma.sync
RUN_CASES = [(3, 1, 64, 64, 7, 1, None, 5), (3, 2, 64, 128, 14, 1, None, 3), (3, 1, 256, 256, 7, 1, None, 3),
             (3, 2, 256, 512, 14, 1, None, 2), (1, 1, 512, 512, 7, 1, None, 3), (3, 1, 128, 128, 9, 1, None, 4),
             (3, 1, 64, 64, 7, 0, 0, 5), (3, 2, 128, 256, 14, 0, 0, 3), (3, 1, 64, 64, 7, 0, 1, 5),
             (3, 2, 128, 256, 14, 0, 1, 3), (3, 1, 96, 96, 7, 1, None, 3), (3, 1, 96, 96, 7, 0, 1, 3)]
MASKS = [(1, 1, 1), (0, 1, 1), (1, 0, 1), (1, 1, 0), (0, 0, 0), (1, 0, 0)]   # residual, sign_scale, sign_shift


@pytest.mark.gpu
@pytest.mark.parametrize("inner", ["b1", "int8"])
def test_gpu_run_fused_scale_is_run_plus_the_tail(inner, monkeypatch):
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import assert_same_bits, dev, gpu_desc, path_counts
    monkeypatch.setenv("LCE_B200_BCONV_B1", "1" if inner == "b1" else "0")
    rng = np.random.default_rng(51)
    for n, (fh, st, cin, cout, hw, pv, mode, batch) in enumerate(RUN_CASES):
        case = L.make_bconv_case(900 + n, batch, hw, hw, cin, fh, fh, cout, stride=(st, st), pad_value=pv)
        plan = capi.BConv2d(gpu_desc(capi, case.desc), case.filt, case.mul, case.bias, case.thr)
        if mode is not None:
            plan.set_zero_padding_mode(mode)   # 0 REFERENCE, 1 CORRECTION (the default registration's)
        x = dev(case.inp)
        y = plan(x).cpu().numpy()              # run
        oh, ow = y.shape[1:3]
        has_res, has_sc, has_sh = MASKS[n % len(MASKS)]
        scale = rng.uniform(0.5, 1.5, (oh, ow, cout)).astype(np.float32)
        res = rng.standard_normal(y.shape).astype(np.float32) if has_res else None
        sc = rng.uniform(0.5, 1.5, cout).astype(np.float32) if has_sc else None
        sh = rng.uniform(-0.5, 0.5, cout).astype(np.float32) if has_sh else None
        act = (L.ACT_NONE, L.ACT_RELU, L.ACT_RELU6)[n % 3]
        packed = n % 5 != 4
        want, want_bits = _scale_tail_ref(y, scale, res, act, sc, sh)
        d = lambda v: None if v is None else dev(v)
        before = path_counts(capi)
        got, bits = plan.run_fused_scale(x, dev(scale[None] if n % 2 else scale), d(res), act, d(sc), d(sh),
                                         packed=packed)
        torch.cuda.synchronize()
        ran = [b - a for a, b in zip(before, path_counts(capi))]
        tag = f"{inner} case {n} ({fh}x{fh} s{st} {cin}->{cout} {hw}x{hw} pad{pv} mode {mode} act {act} packed {packed})"
        if cout % 64 == 0 and mode != 1:   # the epilogue cases: one mma.sync launch
            assert ran == [0, 1, 0], (tag, ran)
        assert_same_bits(got.cpu().numpy(), want, tag)
        if packed:
            assert_same_bits(bits.cpu().numpy(), want_bits, tag + " signs")
        plan.close()


@pytest.mark.gpu
def test_gpu_run_fused_scale_refusals():
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import dev, gpu_desc
    case = L.make_bconv_case(3, 2, 7, 7, 64, 3, 3, 64)
    plan = capi.BConv2d(gpu_desc(capi, case.desc), case.filt, case.mul, case.bias, case.thr)
    x, scale = dev(case.inp), torch.rand(7, 7, 64, device="cuda")
    res = torch.randn(2, 7, 7, 64, device="cuda")
    with pytest.raises(capi.LceError, match="must not overlap the residual"):
        plan.run_fused_scale(x, scale, res, out=res)
    big = torch.zeros(2 * 7 * 7 * 64 + 7 * 7 * 64, device="cuda")
    with pytest.raises(capi.LceError, match="must not overlap the scale"):
        plan.run_fused_scale(x, big[64:64 + 7 * 7 * 64], res, out=big[:2 * 7 * 7 * 64].view(2, 7, 7, 64))
    plan.close()
    gc = L.make_bconv_case(3, 2, 7, 7, 64, 3, 3, 64, groups=2)
    plan = capi.BConv2d(gpu_desc(capi, gc.desc), gc.filt, gc.mul, gc.bias, gc.thr)
    with pytest.raises(capi.LceError, match="packed output needs groups == 1"):
        plan.run_fused_scale(dev(gc.inp), scale)
    plan.close()


@pytest.mark.gpu
@pytest.mark.parametrize("hw,c", [(56, 64), (7, 512)])
def test_gpu_run_fused_scale_at_full_launch_size(hw, c):
    """Batch 256: each persistent mma.sync CTA runs many tiles, and every tile's rows take their
    own positions' scale rows."""
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import assert_same_bits, gpu_desc, path_counts
    rng = np.random.default_rng(hw + c)
    batch = 256
    desc = L.BconvDesc(batch, hw, hw, c, 3, 3, c, 1, 1, 1, 1, 1, L.PADDING_SAME, 1, L.ACT_NONE, L.OUT_FLOAT, 1.0, 0)
    filt = rng.integers(-2**31, 2**31 - 1, (c, 3, 3, c // 32)).astype(np.int32)
    mul = rng.uniform(0.01, 1.5, c).astype(np.float32)
    bias = rng.uniform(-1, 1, c).astype(np.float32)
    plan = capi.BConv2d(gpu_desc(capi, desc), filt, mul, bias)
    x = torch.randint(-2**31, 2**31 - 1, (batch, hw, hw, c // 32), dtype=torch.int32, device="cuda")
    y = plan(x).cpu().numpy()
    scale = rng.uniform(0.5, 1.5, (hw, hw, c)).astype(np.float32)
    res = rng.standard_normal(y.shape).astype(np.float32)
    sc = rng.uniform(0.5, 1.5, c).astype(np.float32)
    sh = rng.uniform(-0.5, 0.5, c).astype(np.float32)
    d = lambda v: torch.from_numpy(v).cuda()
    before = path_counts(capi)
    got, bits = plan.run_fused_scale(x, d(scale), d(res), L.ACT_RELU, d(sc), d(sh))
    torch.cuda.synchronize()
    assert [b - a for a, b in zip(before, path_counts(capi))] == [0, 1, 0]
    want, want_bits = _scale_tail_ref(y, scale, res, L.ACT_RELU, sc, sh)
    assert_same_bits(got.cpu().numpy(), want, f"{hw}x{hw}x{c}")
    assert_same_bits(bits.cpu().numpy(), want_bits, f"{hw}x{hw}x{c} signs")
    plan.close()


def _run_graph(blob, x, fuse, preserve, reference=False):
    g = H.HostGraph.from_tflite(blob, device_arena=True, use_reference_bconv=reference)
    g.resize_input(g.inputs()[0], x.shape)
    removed = g.fuse_all() if fuse else sum(getattr(g, p)() for p in OTHER_PASSES)
    g.preserve_all_tensors(preserve)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    g.enable_cuda_graph(True)
    g.invoke()   # capture
    g.write(g.inputs()[0], x)
    g.invoke()   # replay
    return g, removed


@pytest.mark.gpu
@pytest.mark.parametrize("pad_values,reference", [(0, False), (0, True), (1, False)])
def test_gpu_xnornetpp_fused_equals_unfused(pad_values, reference):
    """With every tensor kept, each fused node's outputs (the block's sum and the next block's
    signs) equal the unfused ops' bit for bit; with reused arenas, so do the class probabilities."""
    blob = zoo.xnornetpp(batch=1, image=224, seed=4, pad_values=pad_values, input_type="int8")
    x = np.random.default_rng(6).integers(-128, 128, (2, 224, 224, 3)).astype(np.int8)
    for preserve in (True, False):
        g0, _ = _run_graph(blob, x, False, preserve, reference)
        g1, removed = _run_graph(blob, x, True, preserve, reference)
        names = collections.Counter(_names(g1))
        assert names[SCALED + SIGN_TAIL] == 15 and names[SCALED] == 1
        out0, out1 = g0.read(g0.outputs()[0]), g1.read(g1.outputs()[0])
        assert np.isfinite(out1).all()
        assert np.array_equal(out0.view(np.uint8), out1.view(np.uint8)), preserve
        if preserve:
            checked = 0
            for i in range(g1.num_nodes()):
                if not g1.node_name(i).startswith(SCALED):
                    continue
                outs = g1.node_io(i)[1]   # output 0; the packed signs are output 1
                if g1.node_name(i).endswith("+LceQuantize"):
                    outs.append(H.lib().lce_host_node_output(g1._g, i, 1))
                for t in outs:
                    a, b = g0.read(t), g1.read(t)
                    assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (i, g1.node_name(i), t)
                    checked += 1
            assert checked == 31
        g0.close()
        g1.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pad_values", [0, 1])
def test_gpu_xnornetpp_against_the_cpu_graph(pad_values):
    blob = zoo.xnornetpp(batch=1, image=64, seed=9, pad_values=pad_values)
    x = np.random.default_rng(3).standard_normal((3, 64, 64, 3)).astype(np.float32)
    want = R.run(R.parse(blob), [x])[0][0]
    g, _ = _run_graph(blob, x, True, False)
    got = g.read(g.outputs()[0])
    g.close()
    assert np.abs(got - want).max() <= 2e-4
    assert np.allclose(got.sum(-1), 1.0, atol=1e-4)


@pytest.mark.gpu
def test_gpu_interpreter_predicts_xnornetpp_in_mini_batches():
    """The converter pins the batch to 1, where [1,OH,OW,C] is the map's own shape; predict resizes
    to each mini-batch, so the scale broadcasts over images (fused and unfused)."""
    from compute_engine_b200.interpreter import Interpreter
    blob = zoo.xnornetpp(batch=1, image=64, seed=11)
    x = np.random.default_rng(8).standard_normal((7, 64, 64, 3)).astype(np.float32)
    want = R.run(R.parse(blob), [x])[0][0]
    outs = []
    for fuse in (True, False):
        it = Interpreter(blob, batch_size=3, fuse=fuse)
        assert (it.fused_nodes_removed > 0) == fuse
        outs.append(it.predict(x))
        it.close()
    assert outs[0].shape == (7, 1000)
    assert np.array_equal(outs[0].view(np.uint8), outs[1].view(np.uint8))
    assert np.abs(outs[0] - want).max() <= 2e-4
