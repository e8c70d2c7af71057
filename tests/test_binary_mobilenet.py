"""Binary MobileNet: grouped binary convolutions on the b1 mma.sync kernel (group windows,
bconv_imma_kernel's GW), their block tails in its epilogue, and the zoo family that uses them.

CPU: the zoo model's op counts and grouped filters, its fused node list against ReActNet-A's, and
the fusion refusals for grouped layers the kernel does not take. GPU: grouped plans on the new path
against the XOR + POPC kernel and the oracle, and the whole graph native (fused and unfused)
against its split form, bit for bit."""
import collections
import ctypes as C

import numpy as np
import pytest

import lce_testlib as L
import tflite_ref as R
from compute_engine_b200 import host as H
from compute_engine_b200 import zoo

WIDTHS = [32, 64, 128, 128, 256, 256] + [512] * 6 + [1024, 1024]


# ----------------------------------- CPU ----------------------------------- #
@pytest.mark.parametrize("image", [224, 64])
def test_binary_mobilenet_ops_and_grouped_filters(image):
    m = R.parse(zoo.binary_mobilenet(batch=2, image=image))
    kinds = collections.Counter((o["code"], o["custom"]) for o in m["ops"])
    ref = collections.Counter((o["code"], o["custom"]) for o in R.parse(zoo.reactnet_a(batch=2, image=image))["ops"])
    assert kinds == ref
    bconvs = [o for o in m["ops"] if o["custom"] == "LceBconv2d"]
    three = [o for o in bconvs if m["tensors"][o["inputs"][1]]["shape"][1] == 3]
    assert len(three) == 13
    for o, c in zip(three, WIDTHS[:-1]):
        f = m["tensors"][o["inputs"][1]]["shape"]
        assert tuple(f) == (c, 3, 3, 1), (c, f)              # C / 32 groups of one word
        assert m["tensors"][o["inputs"][0]]["shape"][3] == c // 32
        assert H.flex_get_int(bytes(o["custom_options"]), "channels_in") == c

    s = R.parse(zoo.binary_mobilenet(batch=2, image=image, group_conv="split"))
    sk = collections.Counter((o["code"], o["custom"]) for o in s["ops"])
    groups = sum(c // 32 for c in WIDTHS[1:-1])             # the 12 grouped layers
    assert sk[(32, "LceBconv2d")] == 31 - 12 + groups
    assert sk[(49, "")] == 12 and sk[(2, "")] == 5 + 12       # SPLIT; CONCATENATION
    # per grouped layer the same binary output channels: C / 32 convolutions of 32 channels
    split_convs = [o for o in s["ops"] if o["custom"] == "LceBconv2d"
                   and s["tensors"][o["inputs"][1]]["shape"][1] == 3]
    per_width = collections.Counter(tuple(s["tensors"][o["outputs"][0]]["shape"])[3] for o in split_convs)
    assert per_width == {32: 1 + groups}


def test_binary_mobilenet_fuses_like_reactnet_a():
    names = []
    for blob in (zoo.binary_mobilenet(batch=2, image=64, seed=1), zoo.reactnet_a(batch=2, image=64, seed=1)):
        g = H.HostGraph.from_tflite(blob, device_arena=True)
        assert g.fuse_all() == 205 - 50
        names.append([g.node_name(i) for i in range(g.num_nodes())])
        g.close()
    assert names[0] == names[1]
    assert names[0].count("LceBconv2d+ADD+RPReLU+ADD+LceQuantize") == 20


def _grouped_block(cin, cout, groups, tail):
    """LceQuantize -> grouped LceBconv2d -> `tail`: "add" = ADD(x) -> LceQuantize, "gate" =
    MUL(gate) -> PRELU -> ADD(x) -> MUL -> ADD -> LceQuantize."""
    g = zoo._Builder(3, 1, "grouped_block")
    xs = (1, 8, 8, cin)
    x = g.m.add_tensor("input", xs, np.float32)
    ins = [x]
    q = g.quantize(x, xs)
    y, ys = g.bconv(q, xs, cout, pad_values=1, activation="NONE", groups=groups)
    if tail == "add":
        o = g.add(y, x, ys)
    else:
        gate = g.m.add_tensor("gate", (1, 1, 1, cout), np.float32)
        ins.append(gate)
        t = g.act(ys)
        g.m.add_op("MUL", [y, gate], [t])
        u = g.act(ys)
        g.m.add_op("PRELU", [t, g.const(np.full((1, 1, cout), 0.25, np.float32), name="alpha")], [u])
        o = g.batchnorm(g.add(u, x, ys), ys)
    p = g.quantize(o, ys)
    g.m.inputs, g.m.outputs = ins, [p]
    return g.m.serialize()


def test_fusion_refuses_grouped_layers_the_kernel_does_not_take():
    # 32 * odd output channels per group: fused, the packed signs included
    g = H.HostGraph.from_tflite(_grouped_block(64, 64, 2, "add"), device_arena=True)
    assert g.fuse_residual_blocks() == 2
    assert "LceBconv2d+ADD+LceQuantize" in [g.node_name(i) for i in range(g.num_nodes())]
    g.close()
    # 16 output channels per group: left as it was
    g = H.HostGraph.from_tflite(_grouped_block(64, 32, 2, "add"), device_arena=True)
    before = [g.node_name(i) for i in range(g.num_nodes())]
    assert g.fuse_residual_blocks() == 0
    assert [g.node_name(i) for i in range(g.num_nodes())] == before
    g.close()
    # a gated tail: the gate is fused, its sign-pack is not, as before
    for groups, packs in ((1, True), (2, False)):
        g = H.HostGraph.from_tflite(_grouped_block(64, 64, groups, "gate"), device_arena=True)
        g.fuse_channel_gates()
        names = [g.node_name(i) for i in range(g.num_nodes())]
        assert any(n.startswith("LceBconv2d+") for n in names), names
        assert any(n.startswith("LceBconv2d+") and n.endswith("LceQuantize") for n in names) == packs, names
        g.close()


def test_grouped_prepare_on_the_host_without_fusion():
    g = H.HostGraph.from_tflite(zoo.binary_mobilenet(batch=2, image=64), device_arena=False)
    g.allocate_tensors()
    assert g.shape(g.outputs()[0]) == (2, 1000)
    g.close()


# ----------------------------------- GPU ----------------------------------- #
KERNEL_ENV = {"xor": {"LCE_B200_BCONV_TC": "0", "LCE_B200_BCONV_IMMA": "0"},
              "mma": {"LCE_B200_BCONV_TC": "1", "LCE_B200_BCONV_IMMA": "1", "LCE_B200_BCONV_B1": "1"}}

# (cin_pg, cout_pg, groups, filter, stride, dilation, padding, pad_value, zp_mode)
PLANS = [
    (32, 32, 2, 3, 1, 1, L.PADDING_SAME, 1, None),
    (32, 32, 3, 3, 2, 1, L.PADDING_SAME, 1, None),            # 96 channels: a half tile
    (32, 32, 8, 1, 1, 1, L.PADDING_VALID, 1, None),
    (32, 32, 32, 3, 1, 1, L.PADDING_SAME, 1, None),
    (64, 32, 8, 3, 1, 2, L.PADDING_SAME, 1, None),
    (96, 32, 3, 5, 1, 1, L.PADDING_SAME, 0, 0),               # REFERENCE zero padding
    (32, 96, 2, 3, 2, 1, L.PADDING_SAME, 0, 1),               # CORRECTION zero padding
    (64, 96, 3, 5, 2, 1, L.PADDING_VALID, 1, None),           # 288 channels: a half tile
    (96, 96, 8, 3, 1, 2, L.PADDING_SAME, 0, 0),
    (32, 96, 32, 1, 2, 1, L.PADDING_SAME, 1, None),
    (96, 32, 2, 1, 1, 1, L.PADDING_SAME, 1, None),
    (64, 64, 3, 3, 1, 1, L.PADDING_SAME, 1, None),            # 64-channel groups, as before
    (32, 64, 8, 3, 1, 1, L.PADDING_SAME, 0, 1),
    (96, 64, 2, 5, 1, 2, L.PADDING_VALID, 1, None),
]


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _run_all(capi, case, res, chain, packed):
    """plain float, bitpacked (thresholds), fused residual and fused chain with their signs: packed
    by the kernel, or (packed=False: grouped plans off the b1 kernel take no packed output) by
    LceQuantize's rule on the host from the float result"""
    import torch
    d = capi.BconvDesc(*[getattr(case.desc, n) for n, _ in case.desc._fields_])
    out = {}
    plan = capi.BConv2d(d, case.filt, case.mul, case.bias)
    if case.meta.get("zp") is not None:
        plan.set_zero_padding_mode(case.meta["zp"])
    x = _dev(case.inp)
    out["float"] = plan(x).cpu().numpy()
    y = torch.empty(out["float"].shape, device="cuda")
    pk = torch.empty(y.shape[:3] + (L.cdiv(y.shape[3], 32),), dtype=torch.int32, device="cuda")
    r = _dev(res)
    rc = capi.lib().lce_b200_bconv2d_run_fused(plan._h, C.c_void_p(x.data_ptr()), C.c_void_p(r.data_ptr()),
                                               C.c_int(L.ACT_RELU), C.c_void_p(y.data_ptr()),
                                               C.c_void_p(pk.data_ptr() if packed else 0),
                                               C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, capi.lib().lce_b200_last_error()
    out["fused"] = y.cpu().numpy()
    out["fused_packed"] = pk.cpu().numpy() if packed else L.quantize(out["fused"])
    o, p = plan.run_fused_chain(x, residual=r, packed=packed, **{k: _dev(v) for k, v in chain.items()})
    out["chain"] = o.cpu().numpy()
    out["chain_packed"] = (p.cpu().numpy() if packed else
                           L.quantize((out["chain"] + chain["sign_shift"]).astype(np.float32)))
    plan.close()
    if case.meta.get("zp") is None or case.meta["zp"] == 0:
        db = L.BconvDesc(*[getattr(case.desc, n) for n, _ in case.desc._fields_])
        db.out_type = L.OUT_BITPACKED
        thr = L.compute_thresholds(db.channels_in // db.groups, db.filter_h, db.filter_w, case.mul, case.bias,
                                   db.activation)
        bplan = capi.BConv2d(capi.BconvDesc(*[getattr(db, n) for n, _ in db._fields_]), case.filt, None, None, thr)
        out["bitpacked"] = bplan(x).cpu().numpy()
        bplan.close()
    torch.cuda.synchronize()
    return out


def _cases(batch, hw, seed0):
    for n, (ci, co, g, k, st, dl, pad, pv, zp) in enumerate(PLANS):
        case = L.make_bconv_case(seed0 + n, batch, hw, hw + 1, ci * g, k, k, co * g, g, (st, st), (dl, dl), pad, pv,
                                 L.ACT_NONE, L.OUT_FLOAT)
        case.meta["zp"] = zp
        yield n, case


@pytest.mark.gpu
@pytest.mark.parametrize("size", ["small", "full"])
def test_gpu_grouped_plans_match_xor_popc(size, monkeypatch):
    """Every plan of the matrix on the b1 mma.sync kernel against the same plan on XOR + POPC:
    float, bitpacked and fused residual / chain outputs with packed signs, identical bits; at
    small sizes also the oracle. "full": M = 32 * 28 * 29 = 25984 pixels (not a multiple of 128),
    so each CTA column runs many tiles. The path counters show which kernel ran."""
    from compute_engine_b200 import capi
    batch, hw = (2, 9) if size == "small" else (32, 28)
    rng = np.random.default_rng(5)
    for n, case in _cases(batch, hw, 700 if size == "small" else 800):
        cout = case.desc.channels_out
        want_shape = None
        results = {}
        for kernel in ("xor", "mma"):
            for k, v in KERNEL_ENV[kernel].items():
                monkeypatch.setenv(k, v)
            if want_shape is None:
                d = capi.BconvDesc(*[getattr(case.desc, f) for f, _ in case.desc._fields_])
                probe = capi.BConv2d(d, case.filt, case.mul, case.bias)
                want_shape = probe.out_shape()
                probe.close()
                res = rng.standard_normal(want_shape).astype(np.float32)
                chain = {"shift_in": rng.uniform(-0.3, 0.3, cout).astype(np.float32),
                         "alpha": rng.uniform(0.05, 0.5, cout).astype(np.float32),
                         "shift_out": rng.uniform(-0.3, 0.3, cout).astype(np.float32),
                         "sign_shift": rng.uniform(-0.3, 0.3, cout).astype(np.float32)}
            before = capi.path_counts()
            results[kernel] = _run_all(capi, case, res, chain, packed=kernel == "mma")
            ran = [b - a for a, b in zip(before, capi.path_counts())]
            if kernel == "mma":
                assert ran[2] == 0 and ran[1] >= 3, (n, ran)   # no XOR + POPC launch
            else:
                assert ran[0] == 0 and ran[1] == 0, (n, ran)
        for key, v in results["xor"].items():
            assert np.array_equal(v.view(np.uint8), results["mma"][key].view(np.uint8)), (n, key)
        if size == "small" and case.meta["zp"] != 1:
            want = L.bconv2d(case.desc, case.inp, case.filt, case.mul, case.bias, case.thr)
            assert np.array_equal(results["mma"]["float"].view(np.uint8), want.view(np.uint8)), n


def _graph_output(blob, x, fuse, preserve):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    if fuse:
        assert g.fuse_all() > 0
    g.preserve_all_tensors(preserve)
    g.resize_input(g.inputs()[0], x.shape)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    out = g.read(g.outputs()[0])
    names = [g.node_name(i) for i in range(g.num_nodes())]
    g.close()
    return out, names


@pytest.mark.gpu
@pytest.mark.parametrize("batch,image,input_type,preserve", [(4, 64, "float32", True), (256, 224, "int8", False)])
def test_gpu_binary_mobilenet_native_split_and_fused_agree(batch, image, input_type, preserve):
    native = zoo.binary_mobilenet(batch=1, image=image, seed=4, input_type=input_type)
    split = zoo.binary_mobilenet(batch=1, image=image, seed=4, input_type=input_type, group_conv="split")
    rng = np.random.default_rng(6)
    if input_type == "int8":
        x = rng.integers(-128, 128, (batch, image, image, 3)).astype(np.int8)
    else:
        x = rng.standard_normal((batch, image, image, 3)).astype(np.float32)
    fused, names = _graph_output(native, x, True, preserve)
    assert names.count("LceBconv2d+ADD+RPReLU+ADD+LceQuantize") == 20
    unfused, _ = _graph_output(native, x, False, preserve)
    ref, _ = _graph_output(split, x, True, preserve)
    assert np.array_equal(fused.view(np.uint8), unfused.view(np.uint8))
    assert np.array_equal(fused.view(np.uint8), ref.view(np.uint8))
    assert np.allclose(fused.sum(-1), 1.0, atol=1e-4)
