"""Binary PointNet graphs: the REDUCE_MAX builtin (lce_b200_f32_reduce_max), FULLY_CONNECTED's keep_num_dims,
the last point-wise binary layer's max over points in the b1 kernel's store (lce_b200_bconv2d_run_fused_fc_max,
Graph::FuseBinaryFcMax) and zoo.binary_pointnet.

CPU: the other zoo models' bytes, binary_pointnet's ops, REDUCE_MAX and keep_num_dims shapes, each REDUCE_MAX
refusal, the fused node lists, each fusion precondition, the other models' node lists, and the new kernel
instances' registers.
GPU: REDUCE_MAX against a numpy statement of TFLite's sequential rule bit for bit (NaN, +-0.0, -inf, empty
slices, three axis forms, past 2^31 elements); the fused node against the unfused graph bit for bit with +-1
weights and with LSR scales against fl(fl(alpha * D) + b) -> BN -> max; binary_pointnet fused against unfused,
on poisoned arenas and CUDA-graph replays; Interpreter.predict at several batches."""
import hashlib
import os
import re

import numpy as np
import pytest

import test_segmentation as S
import tflite_ref as R
from compute_engine_b200 import host as H
from compute_engine_b200 import zoo
from compute_engine_b200.tflite_writer import TFLiteModel

F32 = np.float32
FLT_MAX = np.finfo(F32).max
MAXF = "+REDUCE_MAX"
# sha256 of the zoo models at batch 1, as the parent revision writes them
PARENT_SHA256 = {
    ("binaryalexnet", ()): "150d60007c51b3398d51c6728d6ccb08693609ff0cd7d1b34ad41f01e2218dac",
    ("binarydensenet28", ()): "fcb1f3e89ef1bd23fc6b751d23f9441f2a73dfe383e58beb7d595e61b5b85762",
    ("binarydensenet37", ()): "f8d5bc67f8d50711afc2ae4fe3eb50b182937a849793927657bb4d15a5e118b9",
    ("binarydensenet37_dilated", ()): "1feab16cddee572d8fd747be7913765858bde31fc97731180a6cf43ad279ee1d",
    ("binarydensenet45", ()): "f73b99c0b8ea8f7ff1d14feccb2c4cae89022041bd79d676bd08502e0c091e15",
    ("birealnet18", ()): "69b00efc25be1c89fd630ce5bc79d9f55f2076d93aa0014540d88a54bd717e1e",
    ("dorefanet", ()): "5edd486e889b1185d93e29d99175ac95a7e19208c34e656f061acbe111cd85a3",
    ("meliusnet22", ()): "f2fe2d5101d56c090022dc7b0198dfb6f346959ebad5825908d033a18301b176",
    ("quicknet", ()): "80c00a45aea6e3ba794a0ac5a120f32f08384617492d3bc543cef8d83d1af335",
    ("quicknet_large", ()): "ae386c9d6e07d995bc93739c6ecdcf1ab957c83ac8fa07bc5cc66c86d824a6e2",
    ("quicknet_small", ()): "cf5f288f7f18222243c282a17af72c6a88e9349fc502c32347f8b83a07aab1b5",
    ("reactnet_a", ()): "37dd82f28895b77a623313d33f1ecf6364e53fffc5ab7445d8e848df8fab2085",
    ("realtobinarynet", ()): "d867acd75a420cca207684b4a48e71924f8ea98c3ccec5cd0a44016de002048f",
    ("xnornet", ()): "1320cd7cfb60937fccfccefd5cdc8d4925628d2f4d363bc3a2a4e1e25732b586",
    ("quicknet_seg", ()): "78928c3a80260d6f65554011833f75e3ab757530d7ccfa4cd094ca7fe5229a0d",
    ("binary_srnet", ()): "7f1fe862249154e1d4c5eec81fc55d7a7d88b47fd3ae6dabbef0eb8851544a09",
    ("quicknet_ssd", ()): "ea58fa4048c7d3559d0494ab157b30d8e07abdce76c2853ad727aff1dc480e8e",
    ("binaryalexnet", (("dense", "fully_connected"),)):
        "bb44f567efc46065940a1c0c0930805dfc68169588fb6f624168eb1a768e9a7f",
    ("xnornet", (("dense", "fully_connected"),)): "df94fee8fd039446e1d7b79eaf8efb8ad0373162a1099c721cbb2abe877883d7",
}


def _names(g):
    return [g.node_name(i) for i in range(g.num_nodes())]


def _same_bits(a, b):
    return S._same_bits(a, b)


# ---------------------------- small test graphs ---------------------------- #
def _reduce_graph(shape, axes, keep_dims=False, axes_dtype=np.int32, axes_const=True, in_dtype=np.float32,
                  out_dtype=np.float32, out_shape=None):
    m = TFLiteModel()
    x = m.add_tensor("x", shape, in_dtype)
    a = (m.add_tensor("axes", None, axes_dtype, data=np.asarray(axes, axes_dtype)) if axes_const
         else m.add_tensor("axes", np.shape(axes), axes_dtype))
    red = {k % len(shape) for k in np.atleast_1d(axes)} if len(shape) else set()
    if out_shape is None:
        out_shape = tuple(1 if k in red else d for k, d in enumerate(shape) if keep_dims or k not in red)
    y = m.add_tensor("y", out_shape, out_dtype)
    m.add_op("REDUCE_MAX", [x, a], [y], keep_dims=keep_dims)
    m.inputs, m.outputs = [x] + ([] if axes_const else [a]), [y]
    return m.serialize()


def _weights(rng, n, k, alpha=None):
    w = (rng.integers(0, 2, (n, k)) * 2 - 1).astype(F32)
    return w if alpha is None else w * F32(alpha)


def _fc_max_graph(b=3, p=100, k=64, n=64, alpha=None, bias=True, act="NONE", bn=True, bn_act="NONE", quant=True,
                  store=False, axes=(1,), keep_dims=False, y_output=False, y_reader=False, seed=0):
    """q [B, P, ceil(K/32)] -> LceDequantize -> FULLY_CONNECTED(keep_num_dims) [B, P, N] [-> MUL -> ADD] ->
    REDUCE_MAX(axes) [-> LceQuantize]. store: the max is a graph output too. Returns the model and constants."""
    rng = np.random.default_rng(seed)
    m = TFLiteModel()
    q = m.add_tensor("q", (b, p, (k + 31) // 32), np.int32)
    deq = m.add_tensor("deq", (b, p, k))
    m.add_op("LceDequantize", [q], [deq], custom_options=b"")
    c = {"w": _weights(rng, n, k, alpha), "b": rng.uniform(-3, 3, n).astype(F32) if bias else None}
    y = m.add_tensor("y", (b, p, n))
    m.add_op("FULLY_CONNECTED", [deq, m.add_tensor("w", None, data=c["w"]),
                                 m.add_tensor("b", None, data=c["b"]) if bias else -1], [y], activation=act,
             keep_num_dims=True)
    last = y
    if bn:
        c["scale"] = rng.uniform(0.5, 1.5, n).astype(F32)
        c["shift"] = rng.uniform(-0.5, 0.5, n).astype(F32)
        u = m.add_tensor("u", (b, p, n))
        m.add_op("MUL", [y, m.add_tensor("scale", None, data=c["scale"])], [u])
        last = m.add_tensor("bn", (b, p, n))
        m.add_op("ADD", [u, m.add_tensor("shift", None, data=c["shift"])], [last], activation=bn_act)
    mx = m.add_tensor("max", (b, 1, n) if keep_dims else (b, n))
    m.add_op("REDUCE_MAX", [last, m.add_tensor("axes", None, np.int32, data=np.asarray(axes, np.int32))], [mx],
             keep_dims=keep_dims)
    outs = []
    if quant:
        pk = m.add_tensor("pk", ((b, 1, n // 32) if keep_dims else (b, n // 32)), np.int32)
        m.add_op("LceQuantize", [mx], [pk], custom_options=b"")
        outs.append(pk)
    if store or not quant:
        outs.insert(0, mx)
    if y_reader:
        r = m.add_tensor("relu", (b, p, n))
        m.add_op("RELU", [last], [r])
        outs.append(r)
    if y_output:
        outs.append(last)
    m.inputs, m.outputs = [q], outs
    return m.serialize(), c


def _fused_name(bn, quant):
    return "LceBfc" + ("+MUL+ADD" if bn else "") + MAXF + ("+LceQuantize" if quant else "")


# ----------------------------------- CPU ----------------------------------- #
@pytest.mark.parametrize("key", sorted(PARENT_SHA256, key=str))
def test_other_zoo_models_keep_their_bytes(key):
    name, kw = key
    assert hashlib.sha256(getattr(zoo, name)(batch=1, **dict(kw))).hexdigest() == PARENT_SHA256[key]


def test_binary_pointnet_is_not_in_models():
    assert "binary_pointnet" not in zoo.MODELS
    with pytest.raises(ValueError):
        zoo.binary_pointnet(alpha="per_channel")


def _op_name(o):
    return o["custom"] or {0: "ADD", 9: "FULLY_CONNECTED", 18: "MUL", 25: "SOFTMAX", 82: "REDUCE_MAX"}[o["code"]]


@pytest.mark.parametrize("alpha", [None, "lsr"])
def test_binary_pointnet_ops(alpha):
    m = R.parse(zoo.binary_pointnet(batch=2, points=100, alpha=alpha))
    ops, t = m["ops"], m["tensors"]
    layer = ["LceQuantize", "LceDequantize", "FULLY_CONNECTED", "MUL", "ADD"]
    assert [_op_name(o) for o in ops] == (["FULLY_CONNECTED", "MUL", "ADD"] + layer * 4 + ["REDUCE_MAX"] +
                                          layer * 2 + ["FULLY_CONNECTED", "SOFTMAX"])
    assert t[m["inputs"][0]]["shape"] == (2, 100, 3)
    fcs = [o for o in ops if o["code"] == 9]
    dims = [(64, 3), (64, 64), (64, 64), (128, 64), (1024, 128), (512, 1024), (256, 512), (40, 256)]
    scales = set()
    for i, (o, (n, k)) in enumerate(zip(fcs, dims)):
        w = t[o["inputs"][1]]["data"]
        assert w.shape == (n, k)
        assert o["options"].scalar(2, "b") == (1 if i < 5 else 0)   # keep_num_dims on the point-wise layers
        assert t[o["outputs"][0]]["shape"] == ((2, 100, n) if i < 5 else (2, n))
        if 0 < i < 7:
            a = np.abs(w)
            assert (a == a.flat[0]).all() and len(o["inputs"]) < 3 or o["inputs"][2] == -1
            if alpha is None:
                assert a.flat[0] == 1.0
            else:
                assert np.frexp(a.flat[0])[0] != 0.5
                scales.add(float(a.flat[0]))
    assert alpha is None or len(scales) == 6
    rm = ops[[_op_name(o) for o in ops].index("REDUCE_MAX")]
    assert list(t[rm["inputs"][1]]["data"]) == [1] and t[rm["outputs"][0]]["shape"] == (2, 1024)
    assert t[ops[-1]["outputs"][0]]["shape"] == (2, 40)


def _shapes(blob):
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    g.allocate_tensors()
    shapes = [tuple(g.shape(t)) for t in g.outputs()]
    g.close()
    return shapes


@pytest.mark.parametrize("shape,axes,keep,want", [
    ((2, 5, 8), [1], False, (2, 8)), ((2, 5, 8), [1], True, (2, 1, 8)), ((2, 3, 4, 8), [1, 2], False, (2, 8)),
    ((2, 3, 4, 8), [2, -3, 1], True, (2, 1, 1, 8)), ((7, 9), -1, False, (7,)), ((7,), [0], False, ()),
    ((2, 3, 4, 5, 6), [1, 2, 3], False, (2, 6)), ((3, 0, 4), [1], False, (3, 4))])
def test_reduce_max_shapes(shape, axes, keep, want):
    assert _shapes(_reduce_graph(shape, axes, keep)) == [want]


def test_keep_num_dims_shapes():
    for keep, want in ((True, (2, 5, 16)), (False, (10, 16))):
        m = TFLiteModel()
        x = m.add_tensor("x", (2, 5, 8))
        y = m.add_tensor("y", want)
        m.add_op("FULLY_CONNECTED", [x, m.add_tensor("w", None, data=np.ones((16, 8), F32)), -1], [y],
                 keep_num_dims=keep)
        m.inputs, m.outputs = [x], [y]
        assert _shapes(m.serialize()) == [want]


@pytest.mark.parametrize("kw,msg", [
    (dict(in_dtype=np.int32), "the input must be float32"),
    (dict(out_dtype=np.int32), "the output must be float32"),
    (dict(axes_const=False), "the axes must be a constant tensor"),
    (dict(axes_dtype=np.int64), "int32"),
    (dict(axes=[3]), "an axis is out of range"),
    (dict(axes=[-4]), "an axis is out of range"),
    (dict(axes=[0, 2]), "the reduced axes must be contiguous"),
    (dict(shape=(1, 2, 1, 2, 1, 2), axes=[1]), "rank must be 1 to 5")])
def test_reduce_max_refusals(kw, msg):
    kw = dict(kw)
    shape, axes = kw.pop("shape", (2, 5, 8)), kw.pop("axes", [1])
    if "out_dtype" in kw or "in_dtype" in kw or "axes_const" in kw or "axes_dtype" in kw:
        kw["out_shape"] = (2, 8)
    elif axes != [1]:
        kw["out_shape"] = (2, 8)   # shapes TFLite would not write; the refusal comes first
    g = H.HostGraph.from_tflite(_reduce_graph(shape, axes, **kw), device_arena=False)
    with pytest.raises(Exception, match=re.escape(msg)):
        g.allocate_tensors()
    g.close()


def _fused(blob, passes=("fuse_all",)):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    removed = sum(getattr(g, p)() for p in passes)
    names = _names(g)
    g.close()
    return names, removed


@pytest.mark.parametrize("alpha", [None, "lsr"])
def test_binary_pointnet_fused_node_list(alpha):
    names, _ = _fused(zoo.binary_pointnet(batch=1, points=100, alpha=alpha))
    fc = "LceBfc+MUL+ADD+LceQuantize"
    assert names == ["builtin:9", "builtin:18", "ADD+LceQuantize", fc, fc, fc,
                     "LceBfc+MUL+ADD+REDUCE_MAX+LceQuantize", fc, "LceBfc+MUL+ADD", "builtin:9", "builtin:25"], names
    # without the pass the last point-wise layer runs as LceBfc and a REDUCE_MAX
    g = H.HostGraph.from_tflite(zoo.binary_pointnet(batch=1, points=100, alpha=alpha), device_arena=True)
    g.fuse_binary_fully_connected()
    assert "builtin:82" in _names(g) and not any(MAXF in n for n in _names(g))
    g.close()


@pytest.mark.parametrize("bn,quant,store", [(True, True, False), (True, True, True), (False, False, True),
                                            (False, True, False)])
def test_fused_node_lists(bn, quant, store):
    blob, _ = _fc_max_graph(bn=bn, quant=quant, store=store)
    names, removed = _fused(blob, ("fuse_binary_fc_max",))
    assert names == [_fused_name(bn, quant)] and removed == (5 if bn else 3) + quant - 1
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.fuse_binary_fc_max()
    assert len(g.node_outputs(0)) == int(store or not quant) + int(quant)
    assert g.node_outputs(0) == g.outputs()
    g.close()


@pytest.mark.parametrize("variant", ["axis 2", "axes 1 and 2", "y graph output", "y second reader", "n 96",
                                     "0.5 weight", "host arena"])
def test_fusion_preconditions(variant):
    kw = {"axis 2": {"axes": (2,)}, "axes 1 and 2": {"axes": (1, 2)}, "y graph output": {"y_output": True},
          "y second reader": {"y_reader": True}, "n 96": {"n": 96}}.get(variant, {})
    blob, c = _fc_max_graph(**kw)
    if variant == "0.5 weight":
        w = c["w"].copy()
        w[3, 7] = 0.5
        assert blob.count(c["w"].tobytes()) == 1
        blob = blob.replace(c["w"].tobytes(), w.tobytes())
    g = H.HostGraph.from_tflite(blob, device_arena=variant != "host arena")
    before = _names(g)
    assert g.fuse_binary_fc_max() == 0 and _names(g) == before, variant
    g.close()


@pytest.mark.parametrize("case", sorted(S._other_models()))
def test_other_models_keep_their_node_lists(case):
    make, kw = S._other_models()[case]
    g = H.HostGraph.from_tflite(make(batch=1, seed=0, image=224, **kw), device_arena=True)
    n0 = g.num_nodes()
    assert g.fuse_binary_fc_max() == 0 and g.num_nodes() == n0
    g.close()


def test_fc_max_instances_compile_without_spills(tmp_path):
    import shutil
    import subprocess
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "fcmax.cu"
    src.write_text('#include "lce_b200_imma.cuh"\n' + "".join(
        f"template __global__ void lce::bconv_imma_kernel<{v}, LCE_OUT_FLOAT, true, false, false, false, false, "
        f"false, {shuffle}, {fcmax}>(const lce::ConvKParams);\n"
        for v in (1, 2, 4) for shuffle, fcmax in (("false", "true"), ("true", "false"))))
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas=-v",
                        "-cubin", "-I", os.path.join(repo, "include"),
                        "-I", os.path.join(repo, "compute_engine_b200", "csrc"), str(src),
                        "-o", str(tmp_path / "fcmax.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S*bconv_imma_kernel\S*)\n\s*(.*)", r.stderr)
    assert len(props) == 6, r.stderr
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)


# ----------------------------------- GPU ----------------------------------- #
def reduce_max_ref(x, axes):
    """TFLite's reference reduction, sequentially: cur = -FLT_MAX, then cur = x > cur ? x : cur over the
    reduced axes' elements in index order."""
    x = np.asarray(x, F32)
    r = x.ndim
    red = sorted({a % r for a in np.atleast_1d(axes)})
    a, b = red[0], red[-1] + 1
    v = x.reshape(x.shape[:a] + (-1,) + x.shape[b:])
    cur = np.full(v.shape[:a] + v.shape[a + 1:], -FLT_MAX, F32)
    for i in range(v.shape[a]):
        xi = np.take(v, i, axis=a)
        cur = np.where(xi > cur, xi, cur)
    return cur


def _special(rng, shape):
    """Random values with NaNs, +-0.0 in both orders, -inf and -FLT_MAX sprinkled in."""
    x = rng.standard_normal(shape).astype(F32)
    pick = rng.random(shape)
    x[pick < 0.05] = np.nan
    x[(pick >= 0.05) & (pick < 0.1)] = -np.inf
    x[(pick >= 0.1) & (pick < 0.2)] = 0.0
    x[(pick >= 0.2) & (pick < 0.3)] = -0.0
    x[(pick >= 0.3) & (pick < 0.32)] = -FLT_MAX
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("shape,axes", [((4, 300, 64), 1), ((3, 7, 5, 64), (1, 2)), ((9, 200), -1),
                                        ((5, 40), 1), ((2, 3, 70), (1, -1)), ((6,), 0)])
def test_gpu_reduce_max_equals_the_sequential_rule(shape, axes):
    import torch
    from compute_engine_b200 import capi
    rng = np.random.default_rng(len(shape) * 10 + shape[-1])
    x = _special(rng, shape)
    got = capi.reduce_max(torch.from_numpy(x).cuda(), axes).cpu().numpy()
    assert _same_bits(got, reduce_max_ref(x, axes))
    # the host op: the same through a graph
    g = H.HostGraph.from_tflite(_reduce_graph(shape, list(np.atleast_1d(axes))), device_arena=True)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    assert _same_bits(g.read(g.outputs()[0]), got)
    g.close()


@pytest.mark.gpu
def test_gpu_reduce_max_special_slices():
    import torch
    from compute_engine_b200 import capi
    n = 100   # warp rows (n >= 64) and thread rows
    for length in (n, 5):
        rows = np.zeros((8, length), F32)
        rows[0] = -np.inf
        rows[1] = np.nan
        rows[2, :] = -0.0
        rows[2, 3] = 0.0                  # -0.0 first: stays -0.0
        rows[3, :] = 0.0
        rows[3, 1] = -0.0                 # +0.0 first: stays +0.0
        rows[4, :] = -np.inf
        rows[4, 2] = np.nan
        rows[5, :] = -FLT_MAX
        rows[6, :] = np.nan
        rows[6, length - 1] = -7.0        # a NaN is never chosen
        rows[7] = np.linspace(-1, 1, length, dtype=F32)[::-1]
        got = capi.reduce_max(torch.from_numpy(rows).cuda(), 1).cpu().numpy()
        assert _same_bits(got, reduce_max_ref(rows, 1))
        bits = got.view(np.uint32)
        assert got[0] == -FLT_MAX and got[1] == -FLT_MAX and got[4] == -FLT_MAX and got[6] == -7.0
        assert bits[2] == 0x80000000 and bits[3] == 0
        # the same slices along axis 1 of [B, P, C]
        cube = np.repeat(rows[:, :, None], 3, axis=2)
        assert _same_bits(capi.reduce_max(torch.from_numpy(cube).cuda(), 1).cpu().numpy(), reduce_max_ref(cube, 1))
    empty = torch.empty((3, 0, 4), device="cuda")
    assert (capi.reduce_max(empty, 1).cpu().numpy() == -FLT_MAX).all()


@pytest.mark.gpu
def test_gpu_reduce_max_past_2_31_elements():
    import torch
    from compute_engine_b200 import capi
    b, p, c = 2, (1 << 30) // 64 + 3, 64        # 2 * 16,777,219 * 64 > 2^31 floats
    x = torch.randn((b, p, c), device="cuda")
    assert x.numel() > 2 ** 31
    x[1, p - 1, 5] = 1e9                        # the last image's last point
    x[1, p - 2, 6] = float("nan")
    got = capi.reduce_max(x, 1)
    want = torch.amax(torch.nan_to_num(x, nan=-3e38), 1)
    assert torch.equal(got, want) and got[1, 5].item() == 1e9
    del x
    y = torch.randn((3, (1 << 31) // 3 + 64), device="cuda")   # warp rows past 2^31 elements in all
    y[2, -1] = 5e8
    got = capi.reduce_max(y, -1)
    assert torch.equal(got, torch.amax(y, -1)) and got[2].item() == 5e8


def _pack(rng, shape):
    c = shape[-1]
    lead = tuple(shape[:-1])
    bits = np.zeros(lead + (((c + 31) // 32) * 32,), np.uint64)
    bits[..., :c] = rng.integers(0, 2, lead + (c,))
    words = (bits.reshape(lead + (-1, 32)) << np.arange(32, dtype=np.uint64)).sum(-1)
    return words.astype(np.uint32).view(np.int32)


def _unpack(q, k):
    bits = (q.view(np.uint32)[..., None] >> np.arange(32, dtype=np.uint32)) & 1
    return (1 - 2 * bits.reshape(q.shape[:-1] + (-1,))[..., :k].astype(np.int64))


def _act(y, act):
    lo, hi = {"NONE": (-np.inf, np.inf), "RELU": (0, np.inf), "RELU_N1_TO_1": (-1, 1), "RELU6": (0, 6)}[act]
    return np.minimum(np.maximum(y, F32(lo)), F32(hi)).astype(F32) if act != "NONE" else y


def _sign_words(y):
    n = y.shape[-1]
    bits = (y < 0).astype(np.uint64).reshape(y.shape[:-1] + (n // 32, 32))
    return (bits << np.arange(32, dtype=np.uint64)).sum(-1).astype(np.uint32).view(np.int32)


def _layer_ref(q, c, k, act, bn_act):
    """fl(fl(alpha * D) + b) -> act -> BN (two roundings) -> bn_act, D the exact +-1 dot product: [B, P, N]."""
    x = _unpack(q, k)
    w = c["w"]
    alpha = np.abs(w[:, 0]).astype(F32)
    y = ((x @ np.sign(w).astype(np.int64).T).astype(F32) * alpha).astype(F32)
    if c["b"] is not None:
        y = (y + c["b"]).astype(F32)
    y = _act(y, act)
    if "scale" in c:
        y = _act(((y * c["scale"]).astype(F32) + c["shift"]).astype(F32), bn_act)
    return y


def _run(blob, feeds, passes):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    for p in passes:
        getattr(g, p)()
    g.allocate_tensors()
    for t, v in zip(g.inputs(), feeds):
        g.write(t, v)
    g.invoke()
    outs = [g.read(t) for t in g.outputs()]
    names = _names(g)
    g.close()
    return outs, names


# P 1, 100, 1024 and 2048 (tiles straddling images at 1 and 100); RELU, BatchNorm and signs on and off
FC_MAX_CASES = [
    dict(b=300, p=1, k=64, n=64, act="NONE", bn=True, quant=True, store=False),
    dict(b=5, p=100, k=100, n=128, act="RELU", bn=False, quant=True, store=True),
    dict(b=3, p=1024, k=128, n=1024, act="NONE", bn=True, bn_act="NONE", quant=True, store=False),
    dict(b=2, p=2048, k=64, n=64, act="NONE", bn=True, bn_act="RELU", quant=False, store=True),
    dict(b=7, p=100, k=64, n=192, act="RELU6", bn=True, bn_act="RELU_N1_TO_1", quant=True, store=True),
    dict(b=4, p=1024, k=1024, n=128, act="NONE", bn=False, quant=False, store=True, keep_dims=True),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(FC_MAX_CASES)))
def test_gpu_fused_equals_unfused(case):
    kw = dict(FC_MAX_CASES[case])
    rng = np.random.default_rng(case)
    blob, c = _fc_max_graph(seed=case, **kw)
    feeds = [_pack(rng, (kw["b"], kw["p"], kw["k"]))]
    want, _ = _run(blob, feeds, ())
    mid, _ = _run(blob, feeds, ("fuse_binary_fully_connected",))
    got, names = _run(blob, feeds, ("fuse_binary_fc_max",))
    assert names == [_fused_name(kw["bn"], kw["quant"])], names
    again, _ = _run(blob, feeds, ("fuse_binary_fc_max",))
    for a, m, b, d in zip(want, mid, got, again):
        assert _same_bits(a, b) and _same_bits(m, b) and _same_bits(b, d)
    y = _layer_ref(feeds[0], c, kw["k"], kw["act"], kw.get("bn_act", "NONE"))
    ref = reduce_max_ref(y, 1)
    if kw.get("keep_dims"):
        ref = ref[:, None, :]
    if kw["store"] or not kw["quant"]:
        assert _same_bits(got[0], ref)
    if kw["quant"]:
        assert _same_bits(got[-1], _sign_words(ref))


@pytest.mark.gpu
def test_gpu_c_entry_and_refusals():
    import torch
    from compute_engine_b200 import capi
    rng = np.random.default_rng(7)
    b, p, k, n = 3, 300, 96, 128
    w = _weights(rng, n, k)
    filt = np.zeros((n, 1, 1, (k + 31) // 32), np.uint32)
    for o in range(n):
        for i in range(k):
            if w[o, i] < 0:
                filt[o, 0, 0, i >> 5] |= np.uint32(1 << (i & 31))
    d = capi.BconvDesc(b * p, 1, 1, k, 1, 1, n, 1, 1, 1, 1, 1, capi.PADDING_VALID, 1, capi.ACT_NONE,
                       capi.OUT_FLOAT, 1.0, 0)
    plan = capi.BConv2d(d, filt.view(np.int32), np.ones(n, F32), np.zeros(n, F32))
    q = _pack(rng, (b * p, k))
    alpha = rng.uniform(0.1, 2, n).astype(F32)
    bias, scale, shift = (rng.uniform(-2, 2, n).astype(F32) for _ in range(3))
    out, pk = plan.run_fused_fc_max(torch.from_numpy(q).cuda(), p, alpha, bias, 1, scale, shift, 3)
    c = {"w": w * alpha[:, None], "b": bias, "scale": scale, "shift": shift}
    ref = reduce_max_ref(_layer_ref(q.reshape(b, p, -1), c, k, "RELU", "RELU6"), 1)
    assert _same_bits(out.cpu().numpy(), ref) and _same_bits(pk.cpu().numpy(), _sign_words(ref))
    with pytest.raises(capi.LceError, match="whole number of images"):
        plan.run_fused_fc_max(torch.from_numpy(q).cuda(), 7)
    with pytest.raises(capi.LceError, match="both null"):
        plan.run_fused_fc_max(torch.from_numpy(q).cuda(), p, store_max=False, packed=False)
    with pytest.raises(capi.LceError, match="unknown activation"):
        plan.run_fused_fc_max(torch.from_numpy(q).cuda(), p, activation=9)


@pytest.mark.gpu
@pytest.mark.parametrize("p", [100, 1024])
def test_gpu_lsr_fused_is_rounded_twice_and_within_the_bound(p):
    b, k, n = 4, 128, 1024
    rng = np.random.default_rng(p)
    a = F32(0.3711)
    blob, c = _fc_max_graph(b=b, p=p, k=k, n=n, alpha=a, bn=True, quant=True, store=True, seed=p)
    feeds = [_pack(rng, (b, p, k))]
    want, _ = _run(blob, feeds, ())
    mid, _ = _run(blob, feeds, ("fuse_binary_fully_connected",))
    got, _ = _run(blob, feeds, ("fuse_binary_fc_max",))
    ref = reduce_max_ref(_layer_ref(feeds[0], c, k, "NONE", "NONE"), 1)
    assert _same_bits(got[0], ref) and _same_bits(got[0], mid[0]) and _same_bits(got[1], mid[1])
    # Graph::FuseBinaryFullyConnected's bound, K * 2^-24 * K * alpha_o times the BatchNorm's scale, on each
    # value; the max of values within a bound is within it
    bound = (k * 2.0 ** -24 * k * float(a) * np.abs(c["scale"]))[None, :] + 2.0 ** -22 * np.abs(ref)
    assert (np.abs(got[0].astype(np.float64) - want[0]) <= bound).all()


def _points(batch, seed, p=1024):
    return np.random.default_rng(seed).standard_normal((batch, p, 3)).astype(F32)


def _arena_fails(blob, batch, preserve, p=1024):
    """As test_binary_fc's: the fused graph on arenas poisoned with 0xFF and 0x7F, then captured as a CUDA
    graph and replayed on new inputs."""
    import test_arena_independence as A
    shape = (batch, p, 3)
    xs = [_points(batch, 200 + k, p) for k in range(3)]
    fails = []
    g = A.graph(blob, shape, True, preserve=preserve)
    want = [A.run(g, x, 0) for x in xs]
    if A.same(want[1], want[2]):
        fails.append("the anchors of x1 and x2 are equal")
    if preserve:
        A.run(g, xs[0], 0)
        anchor_snap = A.snapshot(g)
    for tag, byte in A.POISON:
        out = A.run(g, xs[0], byte)
        if preserve:
            snap = A.snapshot(g)
            for d in (A.first_difference(g, anchor_snap, snap), A.stray_write(g, snap, byte)):
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
    return fails, want


@pytest.mark.gpu
@pytest.mark.parametrize("batch,preserve", [(4, True), (256, False)])
def test_gpu_binary_pointnet_fused_equals_unfused(batch, preserve):
    import test_arena_independence as A
    blob = zoo.binary_pointnet(batch=batch, seed=1)
    fails, fused = _arena_fails(blob, batch, preserve)
    assert not fails, f"binary_pointnet at batch {batch}:\n" + "\n".join(fails)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.fuse_binary_fully_connected()   # everything but the max's fusion
    g.preserve_all_tensors(preserve)
    g.allocate_tensors()
    for k in range(3):
        out = A.put(g, _points(batch, 200 + k))
        assert A.same(out, fused[k]), A.describe(fused[k], out)
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=True)   # no fusion at all: +-1 weights, the same bits
    g.allocate_tensors()
    assert A.same(A.put(g, _points(batch, 200)), fused[0])
    g.close()


@pytest.mark.gpu
def test_gpu_interpreter_batches():
    from compute_engine_b200.interpreter import Interpreter
    blob = zoo.binary_pointnet(batch=1, seed=2, points=1024)
    x = _points(256, 9)
    single = zoo.binary_pointnet(batch=256, seed=2, points=1024)
    g = H.HostGraph.from_tflite(single, device_arena=True)
    g.fuse_all()
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    want = g.read(g.outputs()[0])
    g.close()
    for bs in (1, 3, 256):
        got = Interpreter(blob, batch_size=bs, fuse=True).predict(x)
        assert _same_bits(np.asarray(got), want), bs
