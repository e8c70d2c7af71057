"""Real-to-Binary Net: the LOGISTIC builtin, MUL of a [B,H,W,C] tensor by a [B,1,1,C] one, the gated
block tail in the binary convolution's epilogue (lce_b200_bconv2d_run_fused_gate), the one-pass
tail (lce_b200_f32_gate_sign) and the graph fusion that selects it (Graph::FuseChannelGates).

CPU: the zoo model through both readers and the numpy reference, its fused node list, each fusion
precondition, the MUL broadcast rule, the other models' node lists, the new kernel instances'
build. GPU: bit-exact against the oracle convolution plus numpy float32 on every binary-convolution
kernel, LOGISTIC within an ulp bound, and the whole graph op by op and fused vs unfused."""
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

GATED = "LceBconv2d+MUL+PRELU+ADD"
SIGN_TAIL = "+MUL+ADD+LceQuantize"


# ----------------------- CPU reference of the new ops ----------------------- #
def _logistic_ref(x):
    """TFLite's LOGISTIC (reference/logistic.h) in numpy float32."""
    x = np.asarray(x, np.float32)
    with np.errstate(over="ignore"):
        mid = (np.float32(1) / (np.float32(1) + np.exp(-x))).astype(np.float32)
    return np.where(x > np.float32(16.619047164916992188), np.float32(1),
                    np.where(x < np.float32(-9), np.exp(x), mid)).astype(np.float32)


def _logistic_f64(x):
    """The same formula in float64, for the ulp bound of the device's expf."""
    x = np.asarray(x, np.float32).astype(np.float64)
    with np.errstate(over="ignore"):
        mid = 1.0 / (1.0 + np.exp(-x))
    return np.where(x > np.float64(np.float32(16.619047164916992188)), 1.0, np.where(x < -9.0, np.exp(x), mid))


def _gate_tail_ref(y, gate, alpha=None, residual=None, act=L.ACT_NONE, sign_scale=None, sign_shift=None):
    """MUL(gate [B, C]) -> PRELU -> ADD(residual) with its activation, then the signs of
    MUL(sign_scale) -> ADD(sign_shift): the op sequence in numpy float32."""
    t = (y * gate.reshape(gate.shape[0], 1, 1, -1)).astype(np.float32)
    if alpha is not None:
        t = np.where(t >= 0, t, (t * alpha).astype(np.float32)).astype(np.float32)
    if residual is not None:
        t = (t + residual).astype(np.float32)
    if act == L.ACT_RELU:
        t = np.maximum(t, np.float32(0))
    elif act == L.ACT_RELU6:
        t = np.minimum(np.maximum(t, np.float32(0)), np.float32(6))
    s = t
    if sign_scale is not None:
        s = (s * sign_scale).astype(np.float32)
    if sign_shift is not None:
        s = (s + sign_shift).astype(np.float32)
    return t, L.quantize(s)


def _run_op(model, op, vals):
    """One op of a parsed model on the CPU: PRELU and LOGISTIC here, every other op through
    tflite_ref (torch broadcasts the [B,1,1,C] MUL)."""
    if op["code"] == 54:
        x, a = vals[op["inputs"][0]], model["tensors"][op["inputs"][1]]["data"]
        return np.where(x >= 0, x, (x * a).astype(np.float32)).astype(np.float32)
    if op["code"] == 14:
        return _logistic_ref(vals[op["inputs"][0]])
    act = [i for i in op["inputs"] if i >= 0 and model["tensors"][i]["data"] is None]
    sub = {"tensors": model["tensors"], "ops": [op], "inputs": act, "outputs": [op["outputs"][0]]}
    return R.run(sub, [vals[i] for i in act])[0][0]


def _run_model(model, inputs):
    vals = dict(zip(model["inputs"], inputs))
    for op in model["ops"]:
        vals[op["outputs"][0]] = _run_op(model, op, vals)
    return [vals[i] for i in model["outputs"]]


# ----------------------------------- CPU ----------------------------------- #
def test_cpu_reference_runs_realtobinarynet():
    m = R.parse(zoo.realtobinarynet(batch=1, image=32, seed=2))
    x = np.random.default_rng(0).standard_normal((2, 32, 32, 3)).astype(np.float32)
    out = _run_model(m, [x])[0]
    assert out.shape == (2, 1000) and np.isfinite(out).all() and np.allclose(out.sum(-1), 1.0, atol=1e-4)


def test_realtobinarynet_readers_agree_and_it_prepares_on_the_host():
    blob = zoo.realtobinarynet(batch=2, image=64, seed=1)
    m = R.parse(blob)
    kinds = collections.Counter((o["code"], o["custom"]) for o in m["ops"])
    assert kinds[(32, "LceBconv2d")] == 16 and kinds[(32, "LceQuantize")] == 16
    assert kinds[(14, "")] == 16 and kinds[(22, "")] == 16 and kinds[(54, "")] == 18
    assert kinds[(18, "")] == 32 and kinds[(9, "")] == 33 and kinds[(1, "")] == 3
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    assert g.num_nodes() == len(m["ops"])
    for i, t in enumerate(m["tensors"]):
        assert g.shape(i) == t["shape"], t["name"]
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (2, 1000)
    g.resize_input(g.inputs()[0], (3, 64, 64, 3))   # the RESHAPE's -1 follows the batch
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (3, 1000)
    g.close()


@pytest.mark.parametrize("pad_values", [0, 1])
def test_realtobinarynet_fused_node_list(pad_values):
    g = H.HostGraph.from_tflite(zoo.realtobinarynet(batch=2, image=224, seed=1, pad_values=pad_values),
                                device_arena=True)
    n0 = g.num_nodes()
    assert g.fuse_all() == 15 * 6 + 3 + 1
    names = collections.Counter(g.node_name(i) for i in range(g.num_nodes()))
    assert g.num_nodes() == n0 - 94
    assert names == {
        GATED + SIGN_TAIL: 15,                     # each block with the next block's sign
        GATED: 1,                                  # the last block (the head reads it)
        "builtin:18": 1, "ADD+LceQuantize": 1,     # the first block's BatchNorm and sign
        "builtin:40": 17, "builtin:9": 33, "builtin:14": 16, "builtin:22": 16,   # gates, head
        "builtin:3": 4, "builtin:1": 3,            # stem, downsampling shortcuts
        "builtin:54": 2, "builtin:17": 1, "builtin:25": 1,
    }
    g.close()


@pytest.mark.parametrize("make", [zoo.quicknet, zoo.quicknet_large, zoo.birealnet18, zoo.reactnet_a])
def test_other_models_keep_their_node_lists(make):
    blob = make(batch=1, image=224, seed=2)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n = g.fuse_residual_blocks() + g.fuse_float_glue() + g.fuse_activation_chains() + g.fuse_residual_pairs()
    before = [g.node_name(i) for i in range(g.num_nodes())]
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    assert g.fuse_all() == n
    assert [g.node_name(i) for i in range(g.num_nodes())] == before
    assert g.fuse_channel_gates() == 0
    g.close()


def _gated_block(gate="input", gate_shape=(2, 1, 1, 64), alpha_shape=(1, 1, 64), mul_act="NONE",
                 add_act="NONE", bn_act="NONE", output_t=False, shortcut_later=False, sign_tail=True):
    """LceQuantize -> LceBconv2d -> MUL(gate) -> PRELU -> ADD(shortcut) [-> MUL -> ADD ->
    LceQuantize] on x [2, 6, 6, 64]; the gate a graph input unless `gate` == "const"."""
    rng = np.random.default_rng(4)
    m = TFLiteModel()
    x = m.add_tensor("x", (2, 6, 6, 64))
    f32 = lambda name, shape, lo=-0.5, hi=0.5: m.add_tensor(name, None, np.float32,
                                                            data=rng.uniform(lo, hi, shape))
    xq = m.add_tensor("xq", (2, 6, 6, 2), np.int32)
    filt = m.add_tensor("f", None, np.int32, data=rng.integers(-2**31, 2**31 - 1, (64, 3, 3, 2)).astype(np.int32))
    y = m.add_tensor("y", (2, 6, 6, 64))
    g = f32("g", gate_shape, 0, 1) if gate == "const" else m.add_tensor("g", gate_shape)
    u, v, o = (m.add_tensor(n, (2, 6, 6, 64)) for n in ("u", "v", "o"))
    m.add_op("LceQuantize", [x], [xq], custom_options=b"")
    sc = x
    if shortcut_later:   # the shortcut is computed after the convolution
        sc = m.add_tensor("sc", (2, 6, 6, 64))
    m.add_op("LceBconv2d", [xq, filt, f32("mul", 64, 0.1, 1), f32("bias", 64), -1], [y],
             custom_options=bconv2d_options(64))
    if shortcut_later:
        m.add_op("RELU", [x], [sc])
    m.add_op("MUL", [y, g], [u], activation=mul_act)
    m.add_op("PRELU", [u, f32("alpha", alpha_shape, 0.05, 0.5)], [v])
    m.add_op("ADD", [v, sc], [o], activation=add_act)
    outs = [o]
    if sign_tail:
        s1, s2 = m.add_tensor("s1", (2, 6, 6, 64)), m.add_tensor("s2", (2, 6, 6, 64))
        q = m.add_tensor("q", (2, 6, 6, 2), np.int32)
        m.add_op("MUL", [o, f32("scale", 64, 0.5, 1.5)], [s1])
        m.add_op("ADD", [s1, f32("shift", 64)], [s2], activation=bn_act)
        m.add_op("LceQuantize", [s2], [q], custom_options=b"")
        outs.append(q)
    if output_t:
        outs.append(u)
    m.inputs = [x] if gate == "const" else [x, g]
    m.outputs = outs
    return m.serialize()


def test_gated_block_fuses():
    for kw, name, removed in ((dict(), GATED + SIGN_TAIL, 6), (dict(sign_tail=False), GATED, 3),
                              (dict(add_act="RELU"), GATED + SIGN_TAIL, 6),
                              (dict(bn_act="RELU"), GATED, 3)):   # the sign tail stays apart
        g = H.HostGraph.from_tflite(_gated_block(**kw), device_arena=True)
        assert g.fuse_channel_gates() == removed, kw
        assert g.node_name(1) == name, kw
        g.close()


@pytest.mark.parametrize("variant", ["gate_constant", "gate_not_per_image", "alpha_not_per_channel",
                                     "mul_has_activation", "intermediate_is_a_graph_output",
                                     "shortcut_computed_later"])
def test_gate_fusion_leaves_the_graph_when_a_precondition_fails(variant):
    kw = {"gate_constant": dict(gate="const"),
          "gate_not_per_image": dict(gate_shape=(2, 6, 6, 64)),
          "alpha_not_per_channel": dict(alpha_shape=(6, 6, 64)),
          "mul_has_activation": dict(mul_act="RELU"),
          "intermediate_is_a_graph_output": dict(output_t=True),
          "shortcut_computed_later": dict(shortcut_later=True)}[variant]
    blob = _gated_block(**kw)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    before = [g.node_name(i) for i in range(g.num_nodes())]
    assert g.fuse_channel_gates() == 0
    assert [g.node_name(i) for i in range(g.num_nodes())] == before
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=False)   # and the graph prepares unfused
    g.allocate_tensors()
    g.close()


def _binary_graph(op, a_shape, b_shape, act="NONE"):
    m = TFLiteModel()
    a, b, y = m.add_tensor("a", a_shape), m.add_tensor("b", b_shape), m.add_tensor("y", a_shape)
    m.add_op(op, [a, b], [y], activation=act)
    m.inputs, m.outputs = [a, b], [y]
    return m.serialize()


def test_mul_image_channel_broadcast_rule():
    for shape in ((2, 1, 1, 8), (8,), (2, 4, 4, 8), (1, 1, 1, 8)):
        g = H.HostGraph.from_tflite(_binary_graph("MUL", (2, 4, 4, 8), shape), device_arena=False)
        g.allocate_tensors()
        g.close()
    for shape in ((2, 1, 4, 8), (2, 4, 1, 8), (3, 1, 1, 8), (1, 4, 4, 1), (2, 1, 1, 1, 8)):
        g = H.HostGraph.from_tflite(_binary_graph("MUL", (2, 4, 4, 8), shape), device_arena=False)
        with pytest.raises(H.HostError, match=re.escape("MUL: only same-shape, last-dimension or "
                                                        "[B,H,W,C] x [B,1,1,C] broadcast is supported")):
            g.allocate_tensors()
        g.close()
    g = H.HostGraph.from_tflite(_binary_graph("ADD", (2, 4, 4, 8), (2, 1, 1, 8)), device_arena=False)
    with pytest.raises(H.HostError, match="ADD/MUL: only same-shape or last-dimension broadcast"):
        g.allocate_tensors()
    g.close()


# b shapes the ADD / MUL kernels (out[i] = a[i] op b[i % Count(b)]) compute as TFLite broadcasts
ELT_BROADCASTS = [((2, 8, 8, 8), (8,)), ((2, 8, 8, 8), (1, 1, 1, 8)), ((2, 8, 8, 8), (1, 8)),
                  ((2, 8, 8, 8), (2, 8, 8, 8)), ((1, 8, 8, 8), (8, 8, 8)), ((3, 5, 7, 1), (1,))]
# b's element count is C or a's, but TFLite broadcasts it over other axes, or to a 5-D output, or
# not at all: a kernel reading b[i % Count(b)] would return a wrong result or shape
ELT_WRONG_BROADCASTS = [((2, 8, 8, 8), (1, 8, 1, 1)), ((2, 8, 8, 8), (1, 1, 8, 1)), ((2, 8, 8, 8), (8, 1, 1, 1)),
                        ((2, 4, 4, 2), (2, 1, 1, 1)), ((2, 8, 8, 8), (1, 1, 1, 1, 8)), ((2, 8, 8, 8), (8, 8, 8, 2)),
                        ((1, 8, 8, 8), (1, 1, 8, 8, 8))]


@pytest.mark.parametrize("op", ["ADD", "MUL"])
def test_eltwise_broadcast_rule_looks_at_dimensions(op):
    for a_shape, b_shape in ELT_BROADCASTS:
        g = H.HostGraph.from_tflite(_binary_graph(op, a_shape, b_shape), device_arena=False)
        g.allocate_tensors()
        assert g.shape(g.outputs()[0]) == a_shape
        g.close()
    msg = ("MUL: only same-shape, last-dimension or [B,H,W,C] x [B,1,1,C] broadcast is supported" if op == "MUL"
           else "ADD/MUL: only same-shape or last-dimension broadcast is supported")
    for a_shape, b_shape in ELT_WRONG_BROADCASTS:
        g = H.HostGraph.from_tflite(_binary_graph(op, a_shape, b_shape), device_arena=False)
        with pytest.raises(H.HostError, match=re.escape(msg)):
            g.allocate_tensors()
        g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("op", ["ADD", "MUL"])
@pytest.mark.parametrize("a_shape,b_shape", ELT_BROADCASTS)
def test_gpu_eltwise_broadcast_matches_numpy(op, a_shape, b_shape):
    """One IEEE operation per element: bit-exact against numpy's broadcast in float32."""
    rng = np.random.default_rng(len(b_shape) * 10 + b_shape[-1])
    a = rng.standard_normal(a_shape).astype(np.float32)
    b = rng.standard_normal(b_shape).astype(np.float32)
    want = (a + b if op == "ADD" else a * b).astype(np.float32)
    g = H.HostGraph.from_tflite(_binary_graph(op, a_shape, b_shape), device_arena=True)
    g.allocate_tensors()
    g.write(g.inputs()[0], a)
    g.write(g.inputs()[1], b)
    g.invoke()
    got = g.read(g.outputs()[0])
    g.close()
    assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_gate_instances_compile_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "gate.cu"
    src.write_text('#include "lce_b200_imma.cuh"\n' + "".join(
        f"template __global__ void lce::bconv_imma_kernel<{v}, LCE_OUT_FLOAT, {b1}, false, true>"
        "(const lce::ConvKParams);\n" for v in (1, 2, 4) for b1 in ("true", "false")))
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xptxas=-v", "-cubin", "-I", os.path.join(repo, "include"),
                        "-I", os.path.join(repo, "compute_engine_b200", "csrc"), str(src),
                        "-o", str(tmp_path / "gate.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S*bconv_imma_kernel\S*)\n\s*(.*)", r.stderr)
    assert len(props) == 6, r.stderr
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)


# ----------------------------------- GPU ----------------------------------- #
PATHS = {  # environment at plan creation -> the path-counter slot that must run
    "b1": ({"LCE_B200_BCONV_B1": "1"}, 1),
    "int8": ({"LCE_B200_BCONV_B1": "0"}, 1),
    "wgmma": ({"LCE_B200_BCONV_IMMA": "0"}, 0),
    "xor": ({"LCE_B200_BCONV_IMMA": "0", "LCE_B200_BCONV_TC": "0"}, 2),
}
# which of (alpha, sign_scale, sign_shift, residual) are present, cycled over the cases
MASKS = [(1, 1, 1, 1), (0, 1, 1, 1), (1, 0, 1, 1), (1, 1, 0, 1), (1, 1, 1, 0), (0, 0, 0, 0), (1, 0, 0, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("path", list(PATHS))
def test_gpu_run_fused_gate_is_the_op_sequence(path, monkeypatch):
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import assert_same_bits, dev, gpu_desc, path_counts
    env, slot = PATHS[path]
    for k in ("LCE_B200_BCONV_B1", "LCE_B200_BCONV_IMMA", "LCE_B200_BCONV_TC"):
        monkeypatch.setenv(k, env.get(k, "1"))
    rng = np.random.default_rng(41)
    # 3x3 s1, 3x3 s2, 1x1 on 7x7 images (5 of them: 245 / 80 pixels, so 128-row tiles span
    # several images and M is not a multiple of the tile) and on 1x1 images (37 of them); pad
    # values 1 and 0 alternate (0: in-kernel REFERENCE zero padding); last, a CORRECTION plan
    cases = [(fh, st, c, hw, n % 2, 0) for n, (fh, st, c, hw) in enumerate(
        (fh, st, c, hw) for fh, st in ((3, 1), (3, 2), (1, 1)) for c in (64, 128, 512) for hw in (7, 1))]
    cases.append((3, 1, 64, 7, 0, 1))
    for n, (fh, st, c, hw, pv, corr) in enumerate(cases):
        batch = 5 if hw == 7 else 37
        case = L.make_bconv_case(700 + n, batch, hw, hw, c, fh, fh, c, stride=(st, st), pad_value=pv)
        conv = L.bconv2d(case.desc, case.inp, case.filt, case.mul, case.bias, case.thr, kind=corr)
        mask = MASKS[n % len(MASKS)]
        gate = rng.uniform(0, 1, (batch, c)).astype(np.float32)
        vals = [rng.uniform(0.05, 0.5, c).astype(np.float32), rng.uniform(0.5, 1.5, c).astype(np.float32),
                rng.uniform(-0.5, 0.5, c).astype(np.float32), rng.standard_normal(conv.shape).astype(np.float32)]
        alpha, scale, shift, res = [v if on else None for v, on in zip(vals, mask)]
        act = (L.ACT_NONE, L.ACT_RELU, L.ACT_RELU6)[n % 3]
        packed = n % 4 != 3
        want, want_bits = _gate_tail_ref(conv, gate, alpha, res, act, scale, shift)
        plan = capi.BConv2d(gpu_desc(capi, case.desc), case.filt, case.mul, case.bias, case.thr)
        if pv == 0:
            plan.set_zero_padding_mode(corr)   # 0 REFERENCE, 1 CORRECTION
        before = path_counts(capi)
        d = lambda v: None if v is None else dev(v)
        got, bits = plan.run_fused_gate(dev(case.inp), dev(gate), d(res), act, d(alpha), d(scale), d(shift),
                                        packed=packed)
        torch.cuda.synchronize()
        ran = [y - x for x, y in zip(before, path_counts(capi))]
        tag = f"{path} case {n} ({fh}x{fh} s{st} C{c} {hw}x{hw} pad{pv} corr{corr} mask {mask} act {act} packed {packed})"
        # the CORRECTION plan may leave the mma.sync kernel for the correction pass; mma.sync takes
        # REFERENCE zero padding in-kernel
        if not corr and (pv == 1 or slot == 1):
            assert ran[slot] == 1 and sum(ran) == 1, (tag, ran)
        assert_same_bits(got.cpu().numpy(), want, tag)
        if packed:
            assert_same_bits(bits.cpu().numpy(), want_bits, tag + " signs")
        plan.close()


@pytest.mark.gpu
def test_gpu_run_fused_gate_refusals():
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import dev, gpu_desc
    case = L.make_bconv_case(3, 2, 7, 7, 64, 3, 3, 64)
    plan = capi.BConv2d(gpu_desc(capi, case.desc), case.filt, case.mul, case.bias, case.thr)
    x, gate = dev(case.inp), torch.rand(2, 64, device="cuda")
    res = torch.randn(2, 7, 7, 64, device="cuda")
    with pytest.raises(capi.LceError, match="must not overlap the residual"):
        plan.run_fused_gate(x, gate, res, out=res)
    big = torch.zeros(2 * 7 * 7 * 64 + 256, device="cuda")
    with pytest.raises(capi.LceError, match="must not overlap the gate"):
        plan.run_fused_gate(x, big[128:128 + 128], res, out=big[:2 * 7 * 7 * 64].view(2, 7, 7, 64))
    plan.close()
    bp = L.make_bconv_case(3, 2, 7, 7, 64, 3, 3, 64, out_type=L.OUT_BITPACKED)
    plan = capi.BConv2d(gpu_desc(capi, bp.desc), bp.filt, bp.mul, bp.bias, bp.thr)
    with pytest.raises(capi.LceError, match="only float-output plans can take a gate"):
        plan.run_fused_gate(dev(bp.inp), gate, packed=False, out=torch.empty(2, 7, 7, 64, device="cuda"))
    plan.close()
    gc = L.make_bconv_case(3, 2, 7, 7, 64, 3, 3, 64, groups=2)
    plan = capi.BConv2d(gpu_desc(capi, gc.desc), gc.filt, gc.mul, gc.bias, gc.thr)
    with pytest.raises(capi.LceError, match="packed output needs groups == 1"):
        plan.run_fused_gate(dev(gc.inp), gate)
    plan.close()


@pytest.mark.gpu
def test_gpu_logistic_within_4_ulp_across_the_cutoffs():
    """CUDA's expf is within 2 ulp; with the add and the division rounded once each, the device
    result stays within 4 ulp of the formula evaluated in float64."""
    hi, lo = np.float32(16.619047164916992188), np.float32(-9)
    near = [np.nextafter(v, d, dtype=np.float32) for v in (hi, lo) for d in (-np.inf, np.inf)]
    x = np.concatenate([np.linspace(-30, 30, 200001, dtype=np.float32), [hi, lo, 0, -0.0, -87, -103, 88],
                        np.array(near, np.float32),
                        np.random.default_rng(3).standard_normal(4096).astype(np.float32) * 8]).astype(np.float32)
    m = TFLiteModel()
    t, y = m.add_tensor("x", x.shape), m.add_tensor("y", x.shape)
    m.add_op("LOGISTIC", [t], [y])
    m.inputs, m.outputs = [t], [y]
    g = H.HostGraph.from_tflite(m.serialize(), device_arena=True)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    got = g.read(g.outputs()[0])
    g.close()
    want = _logistic_f64(x).astype(np.float32)
    assert np.all(got[x > hi] == 1.0)
    ulp = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    assert ulp.max() <= 4, (x[ulp.argmax()], got[ulp.argmax()], want[ulp.argmax()])


@pytest.mark.gpu
def test_gpu_broadcast_mul_and_gate_sign():
    import torch
    from compute_engine_b200 import capi
    rng = np.random.default_rng(12)
    for shape, act in (((3, 5, 7, 96), "NONE"), ((2, 4, 4, 40), "RELU"), ((4, 1, 1, 64), "NONE")):
        a = rng.standard_normal(shape).astype(np.float32)
        b = rng.uniform(-1, 1, (shape[0], 1, 1, shape[3])).astype(np.float32)
        want = (a * b).astype(np.float32)
        if act == "RELU":
            want = np.maximum(want, np.float32(0))
        g = H.HostGraph.from_tflite(_binary_graph("MUL", shape, b.shape, act), device_arena=True)
        g.allocate_tensors()
        g.write(g.inputs()[0], a)
        g.write(g.inputs()[1], b)
        g.invoke()
        got = g.read(g.outputs()[0])
        g.close()
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (shape, act)
    # the whole tail in one pass, channels not a multiple of 32, and the signs alone
    x = rng.standard_normal((3, 5, 5, 40)).astype(np.float32)
    gate = rng.uniform(0, 1, (3, 40)).astype(np.float32)
    alpha, scale, shift = (rng.uniform(lo, hi, 40).astype(np.float32) for lo, hi in ((0.05, 0.5), (0.5, 1.5), (-0.5, 0.5)))
    res = rng.standard_normal(x.shape).astype(np.float32)
    want, bits = _gate_tail_ref(x, gate, alpha, res, L.ACT_RELU, scale, shift)
    d = lambda v: torch.from_numpy(v).cuda()
    o, pk = capi.gate_sign(d(x), d(gate), d(res), L.ACT_RELU, d(alpha), d(scale), d(shift))
    _, pk_only = capi.gate_sign(d(x), d(gate), None, 0, None, None, d(shift), out=False)
    torch.cuda.synchronize()
    assert np.array_equal(o.cpu().numpy().view(np.uint32), want.view(np.uint32))
    assert np.array_equal(pk.cpu().numpy(), bits)
    assert np.array_equal(pk_only.cpu().numpy(), _gate_tail_ref(x, gate, sign_shift=shift)[1])


@pytest.mark.gpu
def test_gpu_realtobinarynet_graph_op_by_op():
    """The unfused graph on the device, op by op on the device's own input tensors: every LCE op,
    PRELU and the broadcast MUL bit exact, LOGISTIC within 4 ulp, the other float builtins within
    the torch fp32 reference's tolerance; then the class probabilities against the CPU graph."""
    blob = zoo.realtobinarynet(batch=1, image=64, seed=9)
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
        act = [i for i in op["inputs"] if i >= 0 and m["tensors"][i]["data"] is None]
        want = _run_op(m, op, {i: g.read(i) for i in act})
        got = g.read(op["outputs"][0])
        assert got.shape == want.shape, (op["code"], op["custom"])
        gate_mul = op["code"] == 18 and len(act) == 2
        if op["code"] in (32, 54) or gate_mul:
            assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (op["code"], op["custom"])
            exact[op["custom"] or op["code"]] += 1
        elif op["code"] == 14:
            ulp = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
            assert ulp.max() <= 4
        else:
            scale = max(1.0, float(np.abs(want).max()))
            assert np.allclose(got, want, rtol=1e-4, atol=1e-5 * scale), (op["code"], np.abs(got - want).max())
    assert exact == {"LceBconv2d": 16, "LceQuantize": 16, 54: 18, 18: 16}
    got_out = g.read(g.outputs()[0])
    want_out = _run_model(m, [x])[0]
    assert np.abs(got_out - want_out).max() <= 2e-4
    assert np.allclose(got_out.sum(-1), 1.0, atol=1e-4)
    g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pad_values", [0, 1])
def test_gpu_realtobinarynet_fused_equals_unfused(pad_values):
    """Both arms keep every tensor (no arena reuse), as the QuickNet pair test does: fusing frees
    intermediates, which would move the other tensors in the arena. Each removed op is one launch
    fewer, except that a zero-padding (pad_values 0) layer's CORRECTION plan finishes its gated
    node with one extra pass (run_fused, then lce_b200_f32_gate_sign)."""
    from compute_engine_b200 import capi
    blob = zoo.realtobinarynet(batch=1, image=224, seed=4, pad_values=pad_values, input_type="int8")
    x = np.random.default_rng(6).integers(-128, 128, (2, 224, 224, 3)).astype(np.int8)
    outs, launches, removed, names = [], [], [], None
    for gates in (False, True):
        g = H.HostGraph.from_tflite(blob, device_arena=True)
        g.resize_input(g.inputs()[0], x.shape)
        if gates:
            removed.append(g.fuse_all())
            names = collections.Counter(g.node_name(i) for i in range(g.num_nodes()))
        else:
            removed.append(g.fuse_residual_blocks() + g.fuse_float_glue() + g.fuse_activation_chains()
                           + g.fuse_residual_pairs())
        g.preserve_all_tensors(True)
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
        outs.append(g.read(g.outputs()[0]))
        g.close()
    assert names[GATED + SIGN_TAIL] == 15 and names[GATED] == 1
    extra = 16 if pad_values == 0 else 0
    assert launches[0] - launches[1] == removed[1] - removed[0] - extra
    assert np.isfinite(outs[1]).all()
    assert np.array_equal(outs[0].view(np.uint8), outs[1].view(np.uint8))
