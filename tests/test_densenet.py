"""BinaryDenseNet: the dense layer's binary convolution written into the block's map in place
(lce_b200_bconv2d_run_slice), the one-pass BatchNorm signs over a strided map
(lce_b200_f32_affine_sign) and the graph fusion that uses both (Graph::FuseDenseBlocks).

CPU: the four zoo models through the numpy reference and both readers, their op and channel
counts, host prepare, the fused node lists, each fusion precondition, the other models' node lists
and bytes, the new kernel instances' build. GPU: bit-exact against run + copy and numpy float32,
each model op by op, and fused vs unfused under CUDA-graph replay."""
import collections
import hashlib
import itertools
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

DENSE = "MUL+ADD+LceQuantize+LceBconv2d+CONCATENATION"
# model -> (dense layers per block, block inputs C_0, final C, dilations)
SPEC = {
    "binarydensenet28": ((6, 6, 6, 5), (64, 160, 192, 256), 576, (1, 1, 1, 1)),
    "binarydensenet37": ((6, 8, 12, 6), (64, 128, 192, 256), 640, (1, 1, 1, 1)),
    "binarydensenet37_dilated": ((6, 8, 12, 6), (64, 128, 192, 256), 640, (1, 1, 2, 4)),
    "binarydensenet45": ((6, 12, 14, 8), (64, 160, 288, 288), 800, (1, 1, 1, 1)),
}
OTHERS = ("quicknet", "quicknet_large", "birealnet18", "reactnet_a", "realtobinarynet")
# sha256 of the other models' bytes at the commit before BinaryDenseNet was added
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
}


def _bconv_ops(m):
    return [o for o in m["ops"] if o["code"] == 32 and o["custom"] == "LceBconv2d"]


# ----------------------------------- CPU ----------------------------------- #
@pytest.mark.parametrize("name", list(SPEC))
def test_cpu_reference_runs_binarydensenet(name):
    m = R.parse(zoo.MODELS[name](batch=1, image=32, seed=2))
    x = np.random.default_rng(0).standard_normal((2, 32, 32, 3)).astype(np.float32)
    out = R.run(m, [x])[0][0]
    assert out.shape == (2, 1000) and np.isfinite(out).all() and np.allclose(out.sum(-1), 1.0, atol=1e-4)


@pytest.mark.parametrize("name", list(SPEC))
def test_binarydensenet_op_and_channel_counts(name):
    layers, c0, c_final, dil = SPEC[name]
    m = R.parse(zoo.MODELS[name](batch=1, image=224, seed=1))
    convs = _bconv_ops(m)
    assert len(convs) == sum(layers)
    kinds = collections.Counter((o["code"], o["custom"]) for o in m["ops"])
    assert kinds[(2, "")] == sum(layers) and kinds[(32, "LceQuantize")] == sum(layers)
    assert kinds[(3, "")] == 1 + len(layers) - 1   # the stem and one per transition
    k = 0
    for blk, n in enumerate(layers):
        for j in range(n):
            op = convs[k]
            packed, filt = m["tensors"][op["inputs"][0]], m["tensors"][op["inputs"][1]]
            opts = R._flex_ints(op["custom_options"])
            assert opts["channels_in"] == c0[blk] + 64 * j, (name, blk, j)
            assert filt["shape"][0] == 64 and filt["shape"][1:3] == (3, 3)
            assert opts["dilation_height_factor"] == opts["dilation_width_factor"] == dil[blk]
            assert packed["shape"][3] == (c0[blk] + 64 * j + 31) // 32
            k += 1
    assert m["tensors"][m["ops"][-4]["outputs"][0]]["shape"][3] == c_final   # the head's RELU
    if name == "binarydensenet37_dilated":
        assert {R._flex_ints(o["custom_options"])["dilation_height_factor"] for o in convs} == {1, 2, 4}
        # no pooling before the dilated blocks: blocks 2-4 keep 28x28
        assert m["tensors"][convs[-1]["outputs"][0]]["shape"][1:3] == (28, 28)
    else:
        assert m["tensors"][convs[-1]["outputs"][0]]["shape"][1:3] == (7, 7)


@pytest.mark.parametrize("name", list(SPEC))
def test_binarydensenet_readers_agree_and_it_prepares_on_the_host(name):
    blob = zoo.MODELS[name](batch=2, image=64, seed=1)
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


@pytest.mark.parametrize("name", list(SPEC))
def test_binarydensenet_fused_node_list(name):
    layers = SPEC[name][0]
    g = H.HostGraph.from_tflite(zoo.MODELS[name](batch=2, image=224, seed=1), device_arena=True)
    n0 = g.num_nodes()
    before = collections.Counter(g.node_name(i) for i in range(n0))
    glue = g.fuse_float_glue()   # the stem convolution's RELU
    assert g.fuse_dense_blocks() == 4 * sum(layers)
    assert g.num_nodes() == n0 - glue - 4 * sum(layers)
    names = collections.Counter(g.node_name(i) for i in range(g.num_nodes()))
    assert names[DENSE] == sum(layers)
    assert names["LceBconv2d"] == 0 and names["LceQuantize"] == 0 and names["builtin:2"] == 0
    assert names["builtin:18"] == before["builtin:18"] - sum(layers)   # the transitions' and head's BN
    assert g.fuse_dense_blocks() == 0   # idempotent
    # each block's layers write one tensor, its final map, and read x_0 once
    outs = [g.node_io(i)[1][0] for i in range(g.num_nodes()) if g.node_name(i) == DENSE]
    assert [len(list(v)) for _, v in itertools.groupby(outs)] == list(layers)
    g.close()
    # fuse_all on top: the dense nodes stay as they are
    g = H.HostGraph.from_tflite(zoo.MODELS[name](batch=2, image=224, seed=1), device_arena=True)
    assert g.fuse_all() == glue + 4 * sum(layers)
    assert collections.Counter(g.node_name(i) for i in range(g.num_nodes()))[DENSE] == sum(layers)
    g.close()


def test_binarydensenet_unfused_without_the_mma_sync_kernel(monkeypatch):
    monkeypatch.setenv("LCE_B200_BCONV_IMMA", "0")
    g = H.HostGraph.from_tflite(zoo.binarydensenet28(batch=1, image=64, seed=1), device_arena=True)
    assert g.fuse_dense_blocks() == 0
    g.close()


@pytest.mark.parametrize("make", [getattr(zoo, n) for n in OTHERS])
def test_other_models_keep_their_node_lists(make):
    blob = make(batch=1, image=224, seed=2)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n = (g.fuse_residual_blocks() + g.fuse_float_glue() + g.fuse_channel_gates() + g.fuse_activation_chains()
         + g.fuse_residual_pairs())
    before = [g.node_name(i) for i in range(g.num_nodes())]
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    assert g.fuse_all() == n
    assert [g.node_name(i) for i in range(g.num_nodes())] == before
    assert g.fuse_dense_blocks() == 0
    g.close()


def test_other_models_bytes_are_unchanged():
    for (name, image), want in OTHER_HASHES.items():
        kw = dict(batch=1, image=224, seed=0) if image == 224 else dict(batch=2, image=64, seed=3,
                                                                          input_type="int8")
        assert hashlib.sha256(zoo.MODELS[name](**kw)).hexdigest() == want, (name, image)


def _dense_block(n_layers=2, c0=64, scale_shape=None, shift_shape=None, mul_act="NONE",
                 add_act="NONE", cat_order="xy", cat_act="NONE", cat_axis=3, output=None,
                 extra_reader=None, pad_values=1, cout=64, conv_act="NONE", dilation=1, hw=6):
    """x_0 [2, hw, hw, c0] -> n_layers dense layers -> RELU of the block's map (the graph output).
    `output` adds that layer's named intermediate ("t", "u", "q", "y" or "x") to the outputs;
    `extra_reader` gives that tensor of layer 1 a second reader (a RELU, also an output)."""
    rng = np.random.default_rng(7)
    m = TFLiteModel()
    x0 = x = m.add_tensor("x0", (2, hw, hw, c0))
    outs, c = [], c0
    inter = {}
    for j in range(n_layers):
        cw = (c + 31) // 32
        f32 = lambda name, shape, lo=-0.5, hi=0.5: m.add_tensor(f"{name}{j}", None, np.float32,
                                                                data=rng.uniform(lo, hi, shape))
        t, u = m.add_tensor(f"t{j}", (2, hw, hw, c)), m.add_tensor(f"u{j}", (2, hw, hw, c))
        q = m.add_tensor(f"q{j}", (2, hw, hw, cw), np.int32)
        y = m.add_tensor(f"y{j}", (2, hw, hw, cout))
        z = m.add_tensor(f"x{j + 1}", (2, hw, hw, c + cout))
        m.add_op("MUL", [x, f32("scale", scale_shape or (c,), 0.5, 1.5)], [t], activation=mul_act)
        m.add_op("ADD", [t, f32("shift", shift_shape or (c,))], [u], activation=add_act)
        m.add_op("LceQuantize", [u], [q], custom_options=b"")
        filt = m.add_tensor(f"f{j}", None, np.int32,
                            data=rng.integers(-2**31, 2**31 - 1, (cout, 3, 3, cw)).astype(np.int32))
        m.add_op("LceBconv2d", [q, filt, f32("mul", cout, 0.1, 1), f32("bias", cout), -1], [y],
                 custom_options=bconv2d_options(c, dilation=(dilation, dilation), pad_values=pad_values,
                                                activation={"NONE": 0, "RELU": 1}[conv_act]))
        m.add_op("CONCATENATION", [x, y] if cat_order == "xy" else [y, x], [z], axis=cat_axis,
                 activation=cat_act)
        inter[j] = {"t": t, "u": u, "q": q, "y": y, "x": z}
        x, c = z, c + cout
    r = m.add_tensor("r", (2, hw, hw, c))
    m.add_op("RELU", [x], [r])
    outs.append(r)
    if output:
        outs.append(inter[0][output])
    if extra_reader:
        e = m.add_tensor("e", m.tensors[inter[0][extra_reader]]["shape"])
        m.add_op("RELU", [inter[0][extra_reader]], [e])
        outs.append(e)
    m.inputs, m.outputs = [x0], outs
    return m.serialize()


def test_dense_block_fuses():
    for kw, removed in ((dict(), 8), (dict(n_layers=3), 12), (dict(n_layers=1, scale_shape=(1, 1, 1, 64)), 4),
                        (dict(cat_axis=-1), 8), (dict(pad_values=0), 8), (dict(dilation=2), 8),
                        (dict(c0=36), 8), (dict(output="x"), 8), (dict(conv_act="RELU"), 8)):
        g = H.HostGraph.from_tflite(_dense_block(**kw), device_arena=True)
        assert g.fuse_dense_blocks() == removed, kw
        assert [g.node_name(i) for i in range(g.num_nodes())] == [DENSE] * (removed // 4) + ["builtin:19"], kw
        g.close()
    # x_1 read by something else ends the block after the first layer: two blocks of one layer
    g = H.HostGraph.from_tflite(_dense_block(extra_reader="x"), device_arena=True)
    assert g.fuse_dense_blocks() == 8
    ins = [g.node_io(i)[0][0] for i in range(2)]
    outs = [g.node_io(i)[1][0] for i in range(2)]
    assert outs[0] != outs[1] and ins[1] == outs[0]
    g.close()


@pytest.mark.parametrize("variant", ["scale_not_per_channel", "shift_not_per_channel", "mul_has_activation",
                                     "add_has_activation", "concat_order", "concat_activation",
                                     "cout_not_64", "channels_not_multiple_of_4",
                                     "intermediate_is_a_graph_output", "intermediate_read_twice"])
def test_dense_fusion_leaves_the_layer_when_a_precondition_fails(variant):
    kw = {"scale_not_per_channel": dict(scale_shape=(2, 6, 6, 64)),
          "shift_not_per_channel": dict(shift_shape=(2, 6, 6, 64)),
          "mul_has_activation": dict(mul_act="RELU"),
          "add_has_activation": dict(add_act="RELU"),
          "concat_order": dict(cat_order="yx"),
          "concat_activation": dict(cat_act="RELU"),
          "cout_not_64": dict(cout=32),
          "channels_not_multiple_of_4": dict(c0=34),
          "intermediate_is_a_graph_output": dict(output="u"),
          "intermediate_read_twice": dict(extra_reader="y")}[variant]
    blob = _dense_block(n_layers=1, **kw)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    before = [g.node_name(i) for i in range(g.num_nodes())]
    assert g.fuse_dense_blocks() == 0
    assert [g.node_name(i) for i in range(g.num_nodes())] == before
    g.close()
    if variant != "concat_activation":   # the host's CONCATENATION has no fused activation
        g = H.HostGraph.from_tflite(blob, device_arena=False)   # and the graph prepares unfused
        g.allocate_tensors()
        g.close()


def test_slice_instances_compile_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "slice.cu"
    src.write_text('#include "lce_b200_imma.cuh"\n' + "".join(
        f"template __global__ void lce::bconv_imma_kernel<{v}, LCE_OUT_FLOAT, {b1}, false, false, true>"
        "(const lce::ConvKParams);\n" for v in (1, 2, 4) for b1 in ("true", "false")))
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xptxas=-v", "-cubin", "-I", os.path.join(repo, "include"),
                        "-I", os.path.join(repo, "compute_engine_b200", "csrc"), str(src),
                        "-o", str(tmp_path / "slice.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S*bconv_imma_kernel\S*)\n\s*(.*)", r.stderr)
    assert len(props) == 6, r.stderr
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)


# ----------------------------------- GPU ----------------------------------- #
SENTINEL = np.float32(-1234.5)


@pytest.mark.gpu
@pytest.mark.parametrize("b1", ["1", "0"])
def test_gpu_run_slice_is_run_then_copy(b1, monkeypatch):
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import assert_same_bits, dev, gpu_desc, path_counts
    monkeypatch.setenv("LCE_B200_BCONV_IMMA", "1")
    monkeypatch.setenv("LCE_B200_BCONV_B1", b1)
    # (filter, dilation) x C_in x C_out x image, pad values 1 / 0 REFERENCE / 0 CORRECTION cycled
    cases = [(fh, dl, cin, cout, hw) for fh, dl in ((3, 1), (3, 2), (3, 4), (1, 1))
             for cin in (64, 160, 576) for cout in (64, 128) for hw in (7, 1)]
    for n, (fh, dl, cin, cout, hw) in enumerate(cases):
        pv, corr = ((1, 0), (0, 0), (0, 1))[n % 3]
        batch = 5 if hw == 7 else 37          # M = 245 or 37: not a multiple of the 128-row tile
        case = L.make_bconv_case(900 + n, batch, hw, hw, cin, fh, fh, cout, dilation=(dl, dl), pad_value=pv)
        plan = capi.BConv2d(gpu_desc(capi, case.desc), case.filt, case.mul, case.bias, case.thr)
        if pv == 0:
            plan.set_zero_padding_mode(corr)
        want = plan(dev(case.inp))
        torch.cuda.synchronize()
        want = want.cpu().numpy()
        off = 36 + 4 * (n % 3)
        wide = np.full((batch, hw, hw, off + cout + 12), SENTINEL, np.float32)
        out = torch.from_numpy(wide).cuda()
        before = path_counts(capi)
        plan.run_slice(dev(case.inp), out, off)
        torch.cuda.synchronize()
        ran = [y - x for x, y in zip(before, path_counts(capi))]
        tag = f"b1={b1} case {n} ({fh}x{fh} d{dl} {cin}->{cout} {hw}x{hw} pad{pv} corr{corr})"
        assert ran == [0, 1, 0], (tag, ran)
        got = out.cpu().numpy()
        assert_same_bits(got[..., off:off + cout], want, tag)
        wide[..., off:off + cout] = got[..., off:off + cout]
        assert np.array_equal(got.view(np.uint32), wide.view(np.uint32)), tag + ": wrote outside its slice"
        plan.close()


@pytest.mark.gpu
def test_gpu_run_slice_refusals(monkeypatch):
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import dev, gpu_desc
    case = L.make_bconv_case(5, 2, 7, 7, 64, 3, 3, 64)
    plan = capi.BConv2d(gpu_desc(capi, case.desc), case.filt, case.mul, case.bias, case.thr)
    x = dev(case.inp)
    with pytest.raises(capi.LceError, match="at least channels_out"):
        plan.run_slice(x, torch.zeros(2, 7, 7, 60, device="cuda"))
    with pytest.raises(capi.LceError, match="must be a multiple of 4"):
        plan.run_slice(x, torch.zeros(2, 7, 7, 66, device="cuda"))
    with pytest.raises(capi.LceError, match="16-byte aligned"):
        plan.run_slice(x, torch.zeros(2, 7, 7, 72, device="cuda"), offset=2)
    # the output span over the packed input
    buf = torch.zeros(2 * 7 * 7 * 128 + 64, device="cuda")
    xin = buf.view(torch.int32)[:x.numel()].view(x.shape)
    xin.copy_(x)
    with pytest.raises(capi.LceError, match="must not overlap the input"):
        plan.run_slice(xin, buf[:2 * 7 * 7 * 128].view(2, 7, 7, 128), offset=64)
    plan.close()
    for kw, env, msg in ((dict(cout=32), {}, "mma.sync weight fragments"),
                         (dict(cout=64), {"LCE_B200_BCONV_IMMA": "0"}, "mma.sync weight fragments"),
                         (dict(cout=64, out_type=L.OUT_BITPACKED), {}, "float output")):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        c = L.make_bconv_case(6, 2, 7, 7, 64, 3, 3, kw["cout"], out_type=kw.get("out_type", L.OUT_FLOAT))
        plan = capi.BConv2d(gpu_desc(capi, c.desc), c.filt, c.mul, c.bias, c.thr)
        with pytest.raises(capi.LceError, match=msg):
            plan.run_slice(dev(c.inp), torch.zeros(2, 7, 7, 128, device="cuda"))
        plan.close()
        for k in env:
            monkeypatch.delenv(k)


@pytest.mark.gpu
def test_gpu_affine_sign_is_mul_add_quantize():
    import torch
    from compute_engine_b200 import capi
    rng = np.random.default_rng(13)
    d = lambda v: torch.from_numpy(np.ascontiguousarray(v)).cuda()
    for (b, hw, ch, width) in ((3, 5, 48, 100), (2, 7, 64, 64), (37, 1, 160, 200), (1, 3, 36, 36)):
        x = rng.standard_normal((b, hw, hw, width)).astype(np.float32)
        x[0, 0, 0, :4] = [0.0, -0.0, 1e-40, -1e-40]     # signed zeros and denormals
        scale = rng.uniform(0.5, 1.5, ch).astype(np.float32)
        shift = rng.uniform(-0.5, 0.5, ch).astype(np.float32)
        lead = x[..., :ch]
        for sc, sh in ((scale, shift), (None, shift), (scale, None), (None, None)):
            v = lead
            if sc is not None:
                v = (v * sc).astype(np.float32)
            if sh is not None:
                v = (v + sh).astype(np.float32)
            copy = np.full((b, hw, hw, ch + 28), SENTINEL, np.float32)
            dst = d(copy)
            pk = capi.affine_sign(d(x), ch, None if sc is None else d(sc), None if sh is None else d(sh),
                                  copy_to=dst)
            torch.cuda.synchronize()
            tag = (b, hw, ch, width, sc is None, sh is None)
            assert np.array_equal(pk.cpu().numpy(), L.pack_signs(v)), tag
            copy[..., :ch] = lead
            assert np.array_equal(dst.cpu().numpy().view(np.uint32), copy.view(np.uint32)), tag
        pk = capi.affine_sign(d(x), ch, d(scale), d(shift))   # without the copy
        torch.cuda.synchronize()
        v = ((lead * scale).astype(np.float32) + shift).astype(np.float32)
        assert np.array_equal(pk.cpu().numpy(), L.pack_signs(v))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SPEC))
def test_gpu_binarydensenet_graph_op_by_op(name):
    """The unfused graph on the device, op by op on the device's own input tensors: every LCE op,
    MUL, ADD and CONCATENATION bit exact, the other float builtins within the torch fp32
    reference's tolerance; then the class probabilities against the CPU graph."""
    blob = zoo.MODELS[name](batch=1, image=64, seed=9)
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
        sub = {"tensors": m["tensors"], "ops": [op], "inputs": act, "outputs": [op["outputs"][0]]}
        want = R.run(sub, [g.read(i) for i in act])[0][0]
        got = g.read(op["outputs"][0])
        assert got.shape == want.shape, (op["code"], op["custom"])
        if op["code"] in (32, 0, 18, 2):
            assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (op["code"], op["custom"])
            exact[op["custom"] or op["code"]] += 1
        else:
            scale = max(1.0, float(np.abs(want).max()))
            assert np.allclose(got, want, rtol=1e-4, atol=1e-5 * scale), (op["code"], np.abs(got - want).max())
    n = sum(SPEC[name][0])
    assert exact["LceBconv2d"] == n and exact["LceQuantize"] == n and exact[2] == n
    got_out = g.read(g.outputs()[0])
    want_out = R.run(m, [x])[0][0]
    assert np.abs(got_out - want_out).max() <= 2e-4
    g.close()


def _run_graph(blob, x, dense, preserve, launches=None):
    """fuse_all with or without the dense pass; one eager step (its launches counted), then a
    CUDA-graph capture and replay. Returns (output, node names, every tensor when preserved)."""
    from compute_engine_b200 import capi
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.resize_input(g.inputs()[0], x.shape)
    if dense:
        g.fuse_all()
    else:
        g.fuse_residual_blocks() + g.fuse_float_glue() + g.fuse_channel_gates() + g.fuse_activation_chains()
        g.fuse_residual_pairs()
    names = [g.node_name(i) for i in range(g.num_nodes())]
    g.preserve_all_tensors(preserve)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    g.synchronize()
    l0 = capi.launch_count()
    g.invoke()
    g.synchronize()
    if launches is not None:
        launches.append(capi.launch_count() - l0)
    g.enable_cuda_graph(True)
    g.invoke()   # capture
    g.write(g.inputs()[0], x)
    g.invoke()   # replay
    out = g.read(g.outputs()[0])
    g.close()
    return out, names


@pytest.mark.gpu
@pytest.mark.parametrize("name,pad_values", [(n, 0) for n in SPEC] + [("binarydensenet28", 1)])
def test_gpu_binarydensenet_fused_equals_unfused(name, pad_values):
    """With every tensor kept, then with reused arenas. Each fused layer runs two launches (the
    signs, then the convolution) where the unfused one ran three kernels (MUL, ADD + LceQuantize,
    LceBconv2d) and two copies; a
    zero-padding (pad_values 0) CORRECTION plan adds its correction pass to both arms' counts
    unless the unfused convolution ran on the wgmma kernel, so the count is checked at one-padding."""
    blob = zoo.MODELS[name](batch=1, image=64, seed=4, pad_values=pad_values, input_type="int8")
    x = np.random.default_rng(6).integers(-128, 128, (2, 64, 64, 3)).astype(np.int8)
    for preserve in (True, False):
        launches = []
        ref, n_ref = _run_graph(blob, x, False, preserve, launches)
        got, n_got = _run_graph(blob, x, True, preserve, launches)
        layers = sum(SPEC[name][0])
        # unfused, the activation-chain pass runs each layer's ADD -> LceQuantize as one node
        assert collections.Counter(n_ref)["ADD+LceQuantize"] == layers
        assert collections.Counter(n_got)[DENSE] == layers and len(n_ref) - len(n_got) == 3 * layers
        if pad_values == 1:
            assert launches[0] - launches[1] == layers, launches
        assert np.isfinite(got).all()
        assert np.array_equal(ref.view(np.uint8), got.view(np.uint8)), (name, pad_values, preserve)


@pytest.mark.gpu
def test_gpu_interpreter_predict_resizes_the_fused_graph():
    from compute_engine_b200.interpreter import Interpreter
    blob = zoo.binarydensenet28(batch=3, image=64, seed=5)
    m = R.parse(blob)
    it = Interpreter(blob)
    for b in (3, 5, 3):
        x = np.random.default_rng(b).standard_normal((b, 64, 64, 3)).astype(np.float32)
        got = it.predict(x)
        want = R.run(m, [x])[0][0]
        assert got.shape == (b, 1000) and np.abs(got - want).max() <= 2e-4, b
