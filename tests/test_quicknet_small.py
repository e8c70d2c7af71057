"""QuickNetSmall (zoo.quicknet_small): its topology, what fuse_all() makes of it, and the two kernel
instances its hot spots run on -- the fused stem at 8 first-conv channels and the residual-pair
kernel at 32 channels (bconv_pair_kernel<1>). CPU: the graph rewrites and the sm_90a builds. GPU:
both kernels bit-identical to the op sequences they replace, and the whole graph fused == unfused
and against the CPU checkers."""
import collections
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import tflite_ref as R
from compute_engine_b200 import host as H
from compute_engine_b200 import zoo
from compute_engine_b200.tflite_writer import TFLiteModel, bconv2d_options

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAIR = "LceBconv2d+ADD+LceBconv2d+ADD"
STEM = "DEQUANTIZE+CONV_2D+DEPTHWISE_CONV_2D"


def _names(g):
    return [g.node_name(i) for i in range(g.num_nodes())]


def _fused(blob):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.fuse_residual_blocks()
    g.fuse_float_glue()
    g.fuse_activation_chains()
    return g


# ---------------------------------------------------------------- CPU: topology and fusion

def test_topology():
    m = R.parse(zoo.quicknet_small(batch=1, image=224, seed=0))
    t = m["tensors"]
    shape = lambda i: tuple(t[i]["shape"])
    bconvs = [o for o in m["ops"] if o["code"] == 32 and o["custom"] == "LceBconv2d"]
    assert len(bconvs) == 16
    # [input shape, filter shape] of each binary convolution: 3x3 C -> C, four per section
    want = []
    for hw, c in ((56, 32), (28, 64), (14, 256), (7, 512)):
        want += [((1, hw, hw, c // 32), (c, 3, 3, c // 32))] * 4
    assert [(shape(o["inputs"][0]), shape(o["inputs"][1])) for o in bconvs] == want
    # the stem: CONV_2D 3x3/s2 3 -> 8, DEPTHWISE 3x3/s2 on 8 channels, CONV_2D 1x1 8 -> 32
    conv, dw = [o for o in m["ops"] if o["code"] == 3], [o for o in m["ops"] if o["code"] == 4]
    assert shape(conv[0]["inputs"][1]) == (8, 3, 3, 3) and shape(conv[0]["outputs"][0]) == (1, 112, 112, 8)
    assert shape(dw[0]["inputs"][1]) == (1, 3, 3, 8) and shape(dw[0]["outputs"][0]) == (1, 56, 56, 8)
    assert shape(conv[1]["inputs"][1]) == (32, 1, 1, 8) and shape(conv[1]["outputs"][0]) == (1, 56, 56, 32)
    assert conv[1]["inputs"][0] == dw[0]["outputs"][0] and dw[0]["inputs"][0] == conv[0]["outputs"][0]
    assert zoo.MODELS["quicknet_small"] is zoo.quicknet_small


@pytest.mark.parametrize("input_type,stem", [("int8", STEM), ("float32", "CONV_2D+DEPTHWISE_CONV_2D")])
def test_fuse_all_fuses_the_stem_and_pairs_the_32_and_64_channel_sections(input_type, stem):
    g = H.HostGraph.from_tflite(zoo.quicknet_small(batch=1, image=224, seed=1, input_type=input_type),
                                device_arena=True)
    g.fuse_all()
    names = _names(g)
    assert names.count(stem) == 1 and names[0] == stem and "builtin:6" not in names
    # the 8 -> 32 pointwise convolution emits the first block's signs (the direct kernel, with or
    # without them), as do the 64 -> 256 and 256 -> 512 transitions (the tensor-core kernel). The
    # 32 -> 64 transition keeps its LceQuantize: with the signs it would leave the tensor-core kernel.
    assert names[1] == "CONV_2D+LceQuantize" and names.count("CONV_2D+LceQuantize") == 3
    k = names.index("builtin:3")
    assert names[k + 1] == "LceQuantize" and g.shape(g.node_io(k)[1][0])[-1] == 64
    by_c = collections.defaultdict(list)
    for i, n in enumerate(names):
        if n.startswith("LceBconv2d"):
            by_c[g.shape(g.node_io(i)[1][0])[-1]].append(n)
    assert by_c[32] == [PAIR + "+LceQuantize", PAIR]
    assert by_c[64] == [PAIR + "+LceQuantize", PAIR]
    for c in (256, 512):
        assert len(by_c[c]) == 4 and not any(n.startswith(PAIR) for n in by_c[c])
    g.close()


def test_fuse_stem_switch_keeps_the_8_channel_stem_unfused(monkeypatch):
    monkeypatch.setenv("LCE_B200_FUSE_STEM", "0")
    g = H.HostGraph.from_tflite(zoo.quicknet_small(batch=1, image=224, seed=1, input_type="int8"),
                                device_arena=True)
    g.fuse_all()
    assert _names(g)[:3] == ["builtin:6", "builtin:3", "builtin:4"]
    g.close()


def _blocks(n=2, c=32, hw=14, extra_consumer=False, x1_output=False, pad_values=1, stride=(1, 1)):
    """x -> n residual blocks [LceQuantize -> LceBconv2d 3x3 -> ADD(shortcut)] -> out, as in
    test_pair_graph.py. A stride-2 block takes its shortcut from a graph input of its output's
    shape."""
    rng = np.random.default_rng(3)
    m = TFLiteModel()
    x = m.add_tensor("x", (1, hw, hw, c))
    inputs, outputs, sums = [x], [], []
    for k in range(n):
        s = stride[k] if k < len(stride) else 1
        ohw = -(-hw // s)
        xq = m.add_tensor(f"xq{k}", (1, hw, hw, c // 32), np.int32)
        f = m.add_tensor(f"f{k}", None, np.int32,
                         data=rng.integers(-2**31, 2**31 - 1, (c, 3, 3, c // 32)).astype(np.int32))
        mul = m.add_tensor(f"mul{k}", None, np.float32, data=rng.uniform(0.1, 1, c))
        bias = m.add_tensor(f"bias{k}", None, np.float32, data=rng.uniform(-1, 1, c))
        y = m.add_tensor(f"y{k}", (1, ohw, ohw, c))
        o = m.add_tensor(f"s{k}", (1, ohw, ohw, c))
        m.add_op("LceQuantize", [x], [xq], custom_options=b"")
        m.add_op("LceBconv2d", [xq, f, mul, bias, -1], [y],
                 custom_options=bconv2d_options(c, (s, s), pad_values=pad_values, activation=1))
        short = x
        if s != 1:
            short = m.add_tensor(f"short{k}", (1, ohw, ohw, c))
            inputs.append(short)
        m.add_op("ADD", [y, short], [o])
        x, hw = o, ohw
        sums.append((o, (1, ohw, ohw, c)))
    if extra_consumer:
        r = m.add_tensor("relu", sums[0][1])
        m.add_op("RELU", [sums[0][0]], [r])
        outputs.append(r)
    if x1_output:
        outputs.append(sums[0][0])
    m.inputs, m.outputs = inputs, [x] + outputs
    return m.serialize()


@pytest.mark.parametrize("hw", [14, 56, 22])
def test_two_32_channel_blocks_pair(hw):
    g = _fused(_blocks(hw=hw))
    assert _names(g) == ["LceQuantize", "LceBconv2d+ADD+LceQuantize", "LceBconv2d+ADD"]
    assert g.fuse_residual_pairs() == 1
    assert _names(g) == ["LceQuantize", PAIR]
    g.close()


@pytest.mark.parametrize("variant", ["x1_has_another_consumer", "x1_is_a_graph_output", "zero_padding",
                                     "stride_2", "image_mostly_tile_padding", "b1_switched_off"])
def test_32_channel_pairing_leaves_the_graph_when_a_precondition_fails(variant, monkeypatch):
    kw = {"x1_has_another_consumer": dict(extra_consumer=True),
          "x1_is_a_graph_output": dict(x1_output=True),
          "zero_padding": dict(pad_values=0),
          "stride_2": dict(stride=(1, 2, 1)),
          # 8 x 8 fills a third of a 14 x 14 tile
          "image_mostly_tile_padding": dict(hw=8),
          "b1_switched_off": {}}[variant]
    if variant == "b1_switched_off":
        monkeypatch.setenv("LCE_B200_BCONV_B1", "0")
    g = _fused(_blocks(**kw))
    before = _names(g)
    assert g.fuse_residual_pairs() == 0
    assert _names(g) == before
    g.close()


def _ptxas_spills(src_text, pattern, tmp_path, name):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = tmp_path / f"{name}.cu"
    src.write_text(src_text)
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xptxas=-v", "-cubin", "-I", os.path.join(REPO, "include"),
                        "-I", os.path.join(REPO, "compute_engine_b200", "csrc"), str(src),
                        "-o", str(tmp_path / f"{name}.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return re.findall(r"Function properties for (\S*" + pattern + r"\S*)\n\s*(.*)", r.stderr)


def test_pair_kernel_at_32_channels_compiles_without_spills(tmp_path):
    props = _ptxas_spills('#include "lce_b200_pair.cuh"\n'
                          "template __global__ void lce::bconv_pair_kernel<1>(const lce::PairParams);\n",
                          "bconv_pair_kernel", tmp_path, "pair1")
    assert len(props) == 1
    assert "0 bytes spill stores, 0 bytes spill loads" in props[0][1], props[0]


def test_both_stem_instances_compile_without_spills(tmp_path):
    src = open(os.path.join(REPO, "compute_engine_b200", "csrc", "lce_b200_builtins.cu")).read()
    props = _ptxas_spills(src, "stem_conv_dw_kernel", tmp_path, "builtins")
    # float, int8 and uint8 images, each with 8 and 16 first-conv channels
    assert len(props) == 6, props
    assert sorted(re.search(r"Li(8|16)E", n).group(1) for n, _ in props) == ["16"] * 3 + ["8"] * 3
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)


# ---------------------------------------------------------------- GPU

def _run_fused(capi, torch, plan, x, res, act, packed):
    out = torch.empty_like(res)
    pk = torch.empty(res.shape[:3] + (res.shape[3] // 32,), dtype=torch.int32, device="cuda")
    rc = capi.lib().lce_b200_bconv2d_run_fused(
        plan._h, C.c_void_p(x.data_ptr()), C.c_void_p(res.data_ptr()), C.c_int(act),
        C.c_void_p(out.data_ptr()), C.c_void_p(pk.data_ptr() if packed else 0),
        C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, capi.lib().lce_b200_last_error()
    return out, pk


@pytest.mark.gpu
@pytest.mark.parametrize("b,h,w", [(256, 56, 56), (1, 13, 9), (3, 15, 15), (3, 29, 7), (1, 1, 1),
                                   (3, 56, 56)])
def test_gpu_pair_at_32_channels_equals_two_fused_blocks(b, h, w):
    """At 56 x 56 batch 256 each launch has 4096 CTAs, so every SM runs many tiles; the other
    sizes leave ragged tiles. The stand-alone plans stay on the wgmma kernel; only the pair
    launches the b1 one."""
    import torch
    import lce_testlib as L
    from compute_engine_b200 import capi
    from test_gpu_parity import assert_same_bits, dev, gpu_desc, path_counts
    acts = (L.ACT_NONE, L.ACT_RELU, L.ACT_RELU6, L.ACT_RELU_N1_TO_1)
    n = h * 7 + w + b
    cases = [L.make_bconv_case(500 + n + k, b, h, w, 32, 3, 3, 32, activation=acts[(n + k) % 4])
             for k in range(2)]
    plans = [capi.BConv2d(gpu_desc(capi, cs.desc), cs.filt, cs.mul, cs.bias) for cs in cases]
    rng = np.random.default_rng(n)
    x0 = (rng.standard_normal((b, h, w, 32)) * 2).astype(np.float32)
    x0[0, 0, 0, :5] = [0.0, -0.0, 1.0, -1.0, 6.5]
    xq = dev(L.quantize(x0))
    res = dev(x0)
    act1, act2 = acts[n % 4], acts[(n + 2) % 4]
    before = path_counts(capi)
    x1, p1 = _run_fused(capi, torch, plans[0], xq, res, act1, True)
    want, want_pk = _run_fused(capi, torch, plans[1], p1, x1, act2, True)
    torch.cuda.synchronize()
    assert path_counts(capi)[1] == before[1]    # not the b1 mma.sync kernel
    for packed in (True, False):
        before = path_counts(capi)
        launches = capi.launch_count()
        got, pk = plans[0].run_fused_pair(plans[1], xq, res, act1, act2, packed=packed)
        torch.cuda.synchronize()
        assert capi.launch_count() - launches == 1
        assert [y - x for x, y in zip(before, path_counts(capi))] == [0, 1, 0]
        tag = f"{b}x{h}x{w}x32 acts {act1},{act2} packed {packed}"
        assert_same_bits(got.cpu().numpy(), want.cpu().numpy(), tag)
        if packed:
            assert_same_bits(pk.cpu().numpy(), want_pk.cpu().numpy(), tag + " signs")
        else:
            assert pk is None
    for p in plans:
        p.close()


class ConvDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("batch", "in_h", "in_w", "in_c", "filter_h", "filter_w", "out_c",
                                         "stride_h", "stride_w", "dilation_h", "dilation_w", "padding",
                                         "activation")]


@pytest.mark.gpu
@pytest.mark.parametrize("in_type", [0, 1, 2])   # float32, int8, uint8
@pytest.mark.parametrize("B,H,W,act1,act2", [(3, 224, 224, 1, 0), (2, 101, 75, 3, 1)])
def test_gpu_stem_at_8_channels_is_bit_identical_to_its_kernels(in_type, B, H, W, act1, act2):
    import torch
    from compute_engine_b200 import capi
    lib = capi.lib()
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    g = torch.Generator(device="cpu").manual_seed(H * 1000 + W + in_type)
    if in_type == 0:
        x = torch.randn(B, H, W, 3, generator=g).cuda()
        scale, zp = 1.0, 0
    elif in_type == 1:
        x = torch.randint(-128, 128, (B, H, W, 3), generator=g, dtype=torch.int16).to(torch.int8).cuda()
        scale, zp = 4.0 / 127, -3
    else:
        x = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.int16).to(torch.uint8).cuda()
        scale, zp = 1.0 / 255, 117
    w1 = (torch.randn(8, 3, 3, 3, generator=g) * 0.4).cuda()
    b1 = torch.randn(8, generator=g).cuda()
    w2 = (torch.randn(1, 3, 3, 8, generator=g) * 0.4).cuda()
    b2 = torch.randn(8, generator=g).cuda()
    d1 = ConvDesc(B, H, W, 3, 3, 3, 8, 2, 2, 1, 1, 0, act1)
    oh1, ow1 = C.c_int(), C.c_int()
    assert lib.lce_b200_f32_conv_out_shape(C.byref(d1), C.byref(oh1), C.byref(ow1)) == 0
    d2 = ConvDesc(B, oh1.value, ow1.value, 8, 3, 3, 8, 2, 2, 1, 1, 0, act2)
    oh2, ow2 = C.c_int(), C.c_int()
    assert lib.lce_b200_f32_conv_out_shape(C.byref(d2), C.byref(oh2), C.byref(ow2)) == 0
    oh1, ow1, oh2, ow2 = oh1.value, ow1.value, oh2.value, ow2.value
    if in_type == 0:
        xf = x
    else:
        xf = torch.empty(B, H, W, 3, device="cuda")
        assert lib.lce_b200_dequantize_affine(in_type, p(x), p(xf), C.c_int64(x.numel()), C.c_double(scale),
                                              C.c_int32(zp), None) == 0
    y1 = torch.empty(B, oh1, ow1, 8, device="cuda")
    assert lib.lce_b200_f32_conv2d(C.byref(d1), p(xf), p(w1), p(b1), p(y1), None) == 0
    want = torch.empty(B, oh2, ow2, 8, device="cuda")
    assert lib.lce_b200_f32_depthwise_conv2d(C.byref(d2), p(y1), p(w2), p(b2), p(want), None) == 0
    got = torch.full((B, oh2, ow2, 8), float("nan"), device="cuda")
    hw1, hb1, hw2, hb2 = (t.cpu().contiguous() for t in (w1, b1, w2, b2))
    rc = lib.lce_b200_f32_stem_conv_dw(C.byref(d1), C.byref(d2), in_type, p(x), C.c_double(scale), C.c_int32(zp),
                                       p(hw1), p(hb1), p(hw2), p(hb2), p(got), None)
    assert rc == 0, lib.lce_b200_last_error().decode()
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))


def _graph_out(blob, x, fuse, preserve):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    n = g.fuse_all() if fuse else 0
    g.preserve_all_tensors(preserve)
    g.resize_input(g.inputs()[0], x.shape)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    out = g.read(g.outputs()[0])
    names = _names(g)
    g.close()
    return out, n, names


@pytest.mark.gpu
@pytest.mark.parametrize("input_type", ["int8", "float32"])
def test_gpu_quicknet_small_fused_equals_unfused(input_type):
    blob = zoo.quicknet_small(batch=1, image=224, seed=4, input_type=input_type)
    rng = np.random.default_rng(6)
    x = (rng.integers(-128, 128, (3, 224, 224, 3)).astype(np.int8) if input_type == "int8"
         else rng.standard_normal((3, 224, 224, 3)).astype(np.float32))
    for preserve in (True, False):
        unfused, _, _ = _graph_out(blob, x, False, preserve)
        fused, n, names = _graph_out(blob, x, True, preserve)
        assert n > 0 and names.count(PAIR) + names.count(PAIR + "+LceQuantize") == 4
        assert np.isfinite(fused).all()
        assert np.array_equal(fused.view(np.uint8), unfused.view(np.uint8)), f"preserve {preserve}"


@pytest.mark.gpu
def test_gpu_quicknet_small_against_the_cpu_graph():
    """As bench.py's parity check: on 4 images every LCE op of the unfused graph, fed with the
    device's own input, equals the CPU checker bit for bit, and the fused graph's probabilities are
    within 2e-4 of the CPU graph's."""
    import lce_testlib as L
    impl = "ref" if L.load_ref() is not None else "oracle"
    blob = zoo.quicknet_small(batch=1, image=224, seed=0, input_type="int8")
    m = R.parse(blob)
    x = np.random.default_rng(7).integers(-128, 128, (4, 224, 224, 3)).astype(np.int8)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.preserve_all_tensors(True)
    g.resize_input(g.inputs()[0], x.shape)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    n_lce = 0
    for op in m["ops"]:
        if op["code"] != 32:
            continue
        sub = {"tensors": m["tensors"], "ops": [op], "inputs": [op["inputs"][0]],
               "outputs": [op["outputs"][0]]}
        want, _ = R.run(sub, [g.read(op["inputs"][0])], lce_impl=impl, bconv_kind=1)
        got = g.read(op["outputs"][0])
        assert got.shape == want[0].shape and np.array_equal(got.view(np.uint8), want[0].view(np.uint8)), \
            f"LCE op {n_lce} ({op['custom']})"
        n_lce += 1
    g.close()
    assert n_lce == 32   # 16 LceQuantize + 16 LceBconv2d
    fused, _, _ = _graph_out(blob, x, True, False)
    want_out, _ = R.run(m, [x], lce_impl=impl, bconv_kind=1)
    assert float(np.abs(fused - want_out[0]).max()) <= 2e-4
