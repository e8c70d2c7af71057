"""ABC-Net: the zoo graph with M weight bases and N shifted activation signs per layer, the bases
kernel that runs a whole layer with its BatchNorm, shortcut and the next layer's planes
(lce_b200_bconv2d_bases_run), the one-pass planes kernel (lce_b200_f32_shift_sign_planes) and the
graph fusion that selects them (Graph::FuseBinaryBases).

CPU: the zoo model's op counts, the CPU reference, the fused node lists, one refusal per
precondition, every registered model untouched by the pass. GPU: the bases plan against M * N
single plans plus the float32 chain, at small and full launch sizes, the planes kernel against
numpy, and the whole graph fused vs unfused, bit for bit."""
import collections

import numpy as np
import pytest

import lce_testlib as L
import tflite_ref as R
from compute_engine_b200 import host as H
from compute_engine_b200 import zoo
from compute_engine_b200.tflite_writer import TFLiteModel, bconv2d_options

BASES = "LceBconv2dBases"
PLANES = "ADD+LceQuantize"


def _names(g):
    return [g.node_name(i) for i in range(g.num_nodes())]


def _ops(blob):
    return collections.Counter(op["code"] if op["code"] != 32 else op["custom"] for op in R.parse(blob)["ops"])


@pytest.mark.parametrize("bases", [(1, 1), (2, 1), (1, 2), (3, 3)])
def test_abcnet_op_counts(bases):
    m, n = bases
    ops = _ops(zoo.abcnet(batch=1, image=64, bases=bases))
    assert ops["LceBconv2d"] == 16 * m * n
    assert ops["LceQuantize"] == 16 * n
    # ADD: 16 N shifts, 16 (M N - 1) chain ADDs, 16 BatchNorm shifts, 8 shortcuts
    assert ops[0] == 16 * n + 16 * (m * n - 1) + 16 + 8
    assert ops[18] == 16                         # the BatchNorm MULs
    assert ops[3] == 1 + 3 and ops[17] == 1      # stem and the three 1x1 shortcuts, the max pool
    assert ops[40] == 1 and ops[9] == 1 and ops[25] == 1
    assert "abcnet" not in zoo.MODELS


def test_cpu_reference_runs_abcnet():
    m = R.parse(zoo.abcnet(batch=1, image=32, seed=2, bases=(2, 2)))
    x = np.random.default_rng(0).standard_normal((2, 32, 32, 3)).astype(np.float32)
    out = R.run(m, [x])[0][0]
    assert out.shape == (2, 1000) and np.isfinite(out).all() and np.allclose(out.sum(-1), 1.0, atol=1e-4)


@pytest.mark.parametrize("bases", [(1, 2), (2, 1), (3, 3), (5, 5)])
def test_abcnet_fused_node_list(bases):
    g = H.HostGraph.from_tflite(zoo.abcnet(batch=2, image=224, seed=1, bases=bases), device_arena=True)
    n0 = g.num_nodes()
    removed = g.fuse_binary_bases()
    names = collections.Counter(_names(g))
    assert g.num_nodes() == n0 - removed
    assert names[BASES + "+LceQuantize"] == 15 and names[BASES] == 1 and names[PLANES] == 1
    assert names["LceBconv2d"] == 0 and names["LceQuantize"] == 0
    assert names["builtin:0"] == 0 and names["builtin:18"] == 0   # every ADD and MUL absorbed
    g.close()
    g = H.HostGraph.from_tflite(zoo.abcnet(batch=2, image=224, seed=1, bases=bases), device_arena=True)
    assert g.fuse_all() >= removed
    assert collections.Counter(_names(g))[BASES + "+LceQuantize"] == 15
    g.close()


def test_single_base_and_plane_is_not_matched():
    blob = zoo.abcnet(batch=2, image=64, seed=1, bases=(1, 1))
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    before = _names(g)
    assert g.fuse_binary_bases() == 0
    assert _names(g) == before
    g.close()


def test_zero_padded_abcnet_is_not_matched():
    g = H.HostGraph.from_tflite(zoo.abcnet(batch=2, image=64, seed=1, bases=(2, 2), pad_values=0),
                                device_arena=True)
    before = _names(g)
    assert g.fuse_binary_bases() == 0
    assert _names(g) == before
    g.close()


def _model_configs():
    for name, make in zoo.MODELS.items():
        for image in (224, 64):
            yield name, make, dict(image=image)
    for pad_values in (0, 1):
        yield "xnornetpp", zoo.xnornetpp, dict(image=224, pad_values=pad_values)


@pytest.mark.parametrize("name,make,kw", list(_model_configs()),
                         ids=[f"{n}-{'-'.join(str(v) for v in kw.values())}" for n, _, kw in _model_configs()])
def test_registered_models_are_not_matched(name, make, kw):
    blob = make(batch=2, seed=2, **kw)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    before = _names(g)
    assert g.fuse_binary_bases() == 0
    assert _names(g) == before
    g.close()


def _filter(rng, cout, k, cin):
    return rng.integers(-2**31, 2**31 - 1, (cout, k, k, cin // 32)).astype(np.int32)


def _abc_layer(M=2, N=2, C=64, hw=6, variant=None):
    """x [2, hw, hw, C] -> N x (ADD(x, u_n) -> LceQuantize) -> M N LceBconv2d 3x3 -> ADD chain ->
    MUL -> ADD(RELU): one ABC layer, fused into a planes node and a bases node unless `variant`
    breaks a precondition."""
    rng = np.random.default_rng(5)
    m = TFLiteModel()
    xs, ys = (2, hw, hw, C), (2, hw, hw, C)
    ps = (2, hw, hw, C // 32)
    x = m.add_tensor("x", xs)
    const = lambda name, a, dt=np.float32: m.add_tensor(name, None, dt, data=a)
    planes = []
    for n in range(N):
        u = np.full((C,), 0.1 * n, np.float32) if variant == "shift_per_channel" and n == 1 else \
            np.array(0.1 * n - 0.05, np.float32)
        s, q = m.add_tensor(f"s{n}", xs), m.add_tensor(f"q{n}", ps, np.int32)
        m.add_op("ADD", [x, const(f"u{n}", u)], [s])
        m.add_op("LceQuantize", [s], [q], custom_options=b"")
        planes.append(q)
    filts = [const(f"f{j}", _filter(rng, C, 3, C), np.int32) for j in range(M)]
    terms = [(n, j) for n in range(N) for j in range(M)]
    if variant == "chain_order":
        terms[0], terms[1] = terms[1], terms[0]
    y, outs = None, []
    for k, (n, j) in enumerate(terms):
        f = filts[j]
        if variant == "filters" and n == N - 1 and j == 0:
            f = const("fx", _filter(rng, C, 3, C), np.int32)
        act = 1 if variant == "term_activation" and k == 1 else 0
        pad = 0 if variant == "zero_padded" else 1
        dil = 2 if variant == "geometry" and k == 1 else 1   # same output shape, other taps
        opts = bconv2d_options(C, (1, 1), (dil, dil), 0, pad, act)
        t = m.add_tensor(f"t{k}", ys)
        m.add_op("LceBconv2d", [planes[n], f, const(f"pm{k}", rng.uniform(0.01, 0.1, C).astype(np.float32)),
                                const(f"pb{k}", np.zeros(C, np.float32)), -1], [t], custom_options=opts)
        if y is None:
            y = t
        else:
            s = m.add_tensor(f"y{k}", ys)
            m.add_op("ADD", [y, t], [s])
            if variant == "other_reader" and k == 1:
                outs.append(s)
            y = s
    u = m.add_tensor("bn_u", ys)
    m.add_op("MUL", [y, const("bn_s", rng.uniform(0.5, 1.5, C).astype(np.float32))], [u])
    o = m.add_tensor("o", ys)
    m.add_op("ADD", [u, const("bn_t", rng.uniform(-0.5, 0.5, C).astype(np.float32))], [o], activation="RELU")
    m.inputs, m.outputs = [x], [o] + outs
    return m.serialize()


def test_abc_layer_fuses():
    g = H.HostGraph.from_tflite(_abc_layer(), device_arena=True)
    n0 = g.num_nodes()
    assert g.fuse_binary_bases() == n0 - 2
    assert _names(g) == [PLANES, BASES]
    g.close()


def test_bases_over_the_shared_memory_budget_are_refused():
    """8 bases of 3x3x512 filters are 288 KB of b1 fragments per 64-channel tile."""
    for M, fused in ((5, True), (8, False)):
        g = H.HostGraph.from_tflite(_abc_layer(M=M, N=1, C=512, hw=4), device_arena=True)
        assert (g.fuse_binary_bases() > 0) == fused, M
        g.close()


@pytest.mark.parametrize("variant", ["shift_per_channel", "term_activation", "zero_padded", "geometry",
                                     "filters", "chain_order", "other_reader"])
def test_bases_fusion_leaves_the_graph_when_a_precondition_fails(variant):
    blob = _abc_layer(variant=variant)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    before = _names(g)
    assert g.fuse_binary_bases() == 0
    assert _names(g) == before
    g.close()
    g = H.HostGraph.from_tflite(blob, device_arena=False)   # and the graph prepares unfused
    g.allocate_tensors()
    g.close()


# ----------------------------------- GPU ----------------------------------- #
def _bases_ref(capi, desc, M, N, planes, filts, muls, biases, bn_s, bn_t, bn_act, residual, add_act, shifts):
    """M N single plans, then the chain of float32 adds, the BatchNorm, shortcut and next planes,
    op by op on torch float32 (element-wise, IEEE round to nearest)."""
    import torch
    from test_gpu_parity import gpu_desc
    y = None
    for n in range(N):
        for m in range(M):
            plan = capi.BConv2d(gpu_desc(capi, desc), filts[m], muls[n * M + m], biases[n * M + m])
            t = plan(planes[n])
            plan.close()
            y = t if y is None else y + t
    act = {L.ACT_NONE: lambda v: v, L.ACT_RELU: lambda v: torch.clamp_min(v, 0.0)}
    o = act[bn_act]((y * bn_s) + bn_t)
    if residual is not None:
        o = act[add_act](o + residual)
    return o, [capi.quantize(o + torch.tensor(s, dtype=torch.float32, device=o.device)) for s in shifts]


def _bases_case(rng, batch, hw, cin, cout, stride, M, N, zeros=False):
    desc = L.BconvDesc(batch, hw, hw, cin, 3, 3, cout, 1, stride, stride, 1, 1, L.PADDING_SAME, 1, L.ACT_NONE,
                       L.OUT_FLOAT, 1.0, 0)
    filts = [_filter(rng, cout, 3, cin) for _ in range(M)]
    muls = [rng.uniform(0.001, 0.1, cout).astype(np.float32) for _ in range(M * N)]
    biases = [rng.uniform(-1, 1, cout).astype(np.float32) for _ in range(M * N)]
    bn_s = rng.uniform(0.5, 1.5, cout).astype(np.float32)
    bn_t = rng.uniform(-0.5, 0.5, cout).astype(np.float32)
    if zeros:
        # channels 0..7: every term is +0.0 (multiplier 0, bias -0.0: the folded bias is +0.0, so the
        # float output transform never yields -0.0), and the BatchNorm turns the zero sum into
        # fl(fl(+0 * -1) + -0) = -0.0, which the next planes must read as not negative
        for t in range(M * N):
            muls[t][:8] = 0.0
            biases[t][:8] = -0.0
        bn_s[:8] = -1.0
        bn_t[:8] = -0.0
    return desc, filts, muls, biases, bn_s, bn_t


def _check_bases(M, N, batch, hw, cin, cout, stride, residual, zeros=False, seed=0):
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import assert_same_bits, gpu_desc, path_counts
    rng = np.random.default_rng(seed)
    desc, filts, muls, biases, bn_s, bn_t = _bases_case(rng, batch, hw, cin, cout, stride, M, N, zeros)
    planes = [torch.randint(-2**31, 2**31 - 1, (batch, hw, hw, cin // 32), dtype=torch.int32, device="cuda")
              for _ in range(N)]
    oh = -(-hw // stride)
    d = lambda v: torch.from_numpy(v).cuda()
    res = torch.randn((batch, oh, oh, cout), device="cuda") if residual else None
    shifts = [-0.25, 0.0, 0.5][:N]
    plan = capi.BConv2dBases(M, N, gpu_desc(capi, desc), filts * N, muls, biases)
    before = path_counts(capi)
    bn_act = L.ACT_NONE if residual or zeros else L.ACT_RELU
    got, got_planes = plan(planes, d(bn_s), d(bn_t), bn_act, res, L.ACT_RELU, shifts)
    torch.cuda.synchronize()
    assert [b - a for a, b in zip(before, path_counts(capi))] == [0, 1, 0]
    want, want_planes = _bases_ref(capi, desc, M, N, planes, filts, muls, biases, d(bn_s), d(bn_t), bn_act,
                                   res, L.ACT_RELU, shifts)
    tag = f"M={M} N={N} {batch}x{hw}x{hw}x{cin}->{cout}/s{stride}"
    assert_same_bits(got.cpu().numpy(), want.cpu().numpy(), tag)
    for k, (a, b) in enumerate(zip(got_planes, want_planes)):
        assert_same_bits(a.cpu().numpy(), b.cpu().numpy(), f"{tag} plane {k}")
    if zeros:
        assert np.signbit(got.cpu().numpy()[..., :8]).all() and (got.cpu().numpy()[..., :8] == 0).all()
    plan.close()


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,hw,cin,cout,stride,residual", [
    (2, 2, 9, 64, 64, 1, True), (3, 1, 6, 128, 64, 1, False), (1, 3, 7, 64, 128, 2, True),
    (5, 5, 5, 512, 512, 1, True), (3, 3, 8, 256, 128, 2, False)])
def test_gpu_bases_plan_is_single_plans_plus_the_chain(M, N, hw, cin, cout, stride, residual):
    _check_bases(M, N, 3, hw, cin, cout, stride, residual, seed=M * 10 + N)


@pytest.mark.gpu
def test_gpu_bases_plan_keeps_negative_zero():
    """The tail's -0.0 outputs, bit for bit, and their next-layer signs (fl(-0 + 0) = +0)."""
    _check_bases(2, 3, 2, 5, 64, 64, 1, False, zeros=True)


@pytest.mark.gpu
@pytest.mark.parametrize("hw,cin,cout,stride", [(56, 64, 64, 1), (7, 512, 512, 1), (56, 64, 128, 2),
                                                 (14, 256, 512, 2)])
@pytest.mark.parametrize("bases", [(3, 3), (5, 5)])
def test_gpu_bases_plan_at_full_launch_size(hw, cin, cout, stride, bases):
    """Batch 256: many CTAs per SM wave, whole-plane staging (64 channels) and the chunked ring
    (512 channels)."""
    _check_bases(bases[0], bases[1], 256, hw, cin, cout, stride, True, seed=hw + cin)


@pytest.mark.gpu
def test_gpu_bases_plan_refusals():
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import gpu_desc
    rng = np.random.default_rng(1)
    desc, filts, muls, biases, bn_s, bn_t = _bases_case(rng, 2, 6, 64, 64, 1, 2, 2)
    for field, value, msg in (("pad_value", 0, "one-padded"), ("activation", L.ACT_RELU, "fused activation"),
                              ("channels_out", 96, "channels_out % 64")):
        d = L.BconvDesc(*[getattr(desc, n) for n, _ in desc._fields_])
        setattr(d, field, value)
        f = filts if field != "channels_out" else [_filter(rng, 96, 3, 64)] * 2
        mb = (muls, biases) if field != "channels_out" else ([np.ones(96, np.float32)] * 4,) * 2
        with pytest.raises(capi.LceError, match=msg):
            capi.BConv2dBases(2, 2, gpu_desc(capi, d), f * 2, *mb)
    with pytest.raises(capi.LceError, match="share base"):
        capi.BConv2dBases(2, 2, gpu_desc(capi, desc), filts + filts[::-1], muls, biases)
    d512 = L.BconvDesc(2, 4, 4, 512, 3, 3, 64, 1, 1, 1, 1, 1, L.PADDING_SAME, 1, L.ACT_NONE, L.OUT_FLOAT, 1.0, 0)
    with pytest.raises(capi.LceError, match="shared memory"):
        capi.BConv2dBases(8, 1, gpu_desc(capi, d512), [_filter(rng, 64, 3, 512)] * 8,
                          [np.ones(64, np.float32)] * 8, [np.zeros(64, np.float32)] * 8)
    import ctypes as C
    plan = capi.BConv2dBases(2, 2, gpu_desc(capi, desc), filts * 2, muls, biases)
    x = torch.zeros((2, 6, 6, 2), dtype=torch.int32, device="cuda")
    o = torch.empty((2, 6, 6, 64), device="cuda")
    s, t = torch.from_numpy(bn_s).cuda(), torch.from_numpy(bn_t).cuda()
    pin = (C.c_void_p * 2)(x.data_ptr(), x.data_ptr())
    with pytest.raises(capi.LceError, match="overlap the residual"):
        capi._check(capi.lib().lce_b200_bconv2d_bases_run(plan._h, pin, capi._p(s), capi._p(t), 0, capi._p(o), 0,
                                                          capi._p(o), 0, None, None, capi._stream()))
    plan.close()


@pytest.mark.gpu
@pytest.mark.parametrize("shape,shifts", [((3, 5, 7, 96), [-0.5, 0.0, 0.25]), ((1, 1, 1, 32), [0.0]),
                                          ((2, 13, 13, 64), [0.1 * k - 0.35 for k in range(8)])])
def test_gpu_shift_sign_planes_match_numpy(shape, shifts):
    """Pixel counts that are not whole warps per CTA; x = -shift gives +0.0, not negative."""
    import torch
    from compute_engine_b200 import capi
    rng = np.random.default_rng(len(shifts))
    x = rng.standard_normal(shape).astype(np.float32)
    x.reshape(-1)[: len(shifts)] = -np.array(shifts, np.float32)
    x.reshape(-1)[len(shifts): 2 * len(shifts)] = -0.0
    planes = capi.shift_sign_planes(torch.from_numpy(x).cuda(), shifts)
    torch.cuda.synchronize()
    for s, p in zip(shifts, planes):
        assert np.array_equal(p.cpu().numpy(), L.quantize((x + np.float32(s)).astype(np.float32))), s


def _run_graph(blob, x, fuse, preserve):
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.resize_input(g.inputs()[0], x.shape)
    removed = g.fuse_all() if fuse else g.fuse_dense_blocks() + g.fuse_residual_blocks()
    g.preserve_all_tensors(preserve)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    g.enable_cuda_graph(True)
    g.invoke()   # capture
    g.write(g.inputs()[0], x)
    g.invoke()   # replay
    return g, removed


def _fused_outputs(g, n_planes):
    """Every tensor the bases and planes nodes write: N planes; a layer with the next planes writes
    them, after its sum when it has a shortcut (the next block also reads the sum); the last layer
    writes its sum alone."""
    outs = []
    for i in range(g.num_nodes()):
        name = g.node_name(i)
        if name == PLANES:
            n = n_planes
        elif name == BASES + "+LceQuantize":
            n = n_planes + (1 if g.node_io(i)[0][-1] >= 0 else 0)
        elif name == BASES:
            n = 1
        else:
            continue
        outs += [H.lib().lce_host_node_output(g._g, i, k) for k in range(n)]
    return outs


@pytest.mark.gpu
@pytest.mark.parametrize("bases", [(2, 2), (3, 3)])
def test_gpu_abcnet_fused_equals_unfused(bases):
    """With every tensor kept, each fused node's outputs equal the unfused ops' bit for bit; with
    reused arenas, so do the class probabilities. Zero-padded graphs stay unfused and equal."""
    x = np.random.default_rng(6).integers(-128, 128, (2, 64, 64, 3)).astype(np.int8)
    for pad_values in (1, 0):
        blob = zoo.abcnet(batch=1, image=64, seed=4, bases=bases, pad_values=pad_values, input_type="int8")
        for preserve in (True, False):
            g0, _ = _run_graph(blob, x, False, preserve)
            g1, _ = _run_graph(blob, x, True, preserve)
            names = collections.Counter(_names(g1))
            assert names[BASES + "+LceQuantize"] == (15 if pad_values else 0), names
            out0, out1 = g0.read(g0.outputs()[0]), g1.read(g1.outputs()[0])
            assert np.isfinite(out1).all()
            assert np.array_equal(out0.view(np.uint8), out1.view(np.uint8)), (pad_values, preserve)
            if preserve and pad_values:
                checked = 0
                for t in _fused_outputs(g1, bases[1]):
                    a, b = g0.read(t), g1.read(t)
                    assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), t
                    checked += 1
                n = bases[1]
                assert checked == n + 8 * n + 7 * (n + 1) + 1
            g0.close()
            g1.close()


@pytest.mark.gpu
def test_gpu_abcnet_against_the_cpu_graph():
    blob = zoo.abcnet(batch=1, image=32, seed=9, bases=(2, 2))
    x = np.random.default_rng(3).standard_normal((2, 32, 32, 3)).astype(np.float32)
    want = R.run(R.parse(blob), [x])[0][0]
    g, _ = _run_graph(blob, x, True, False)
    got = g.read(g.outputs()[0])
    g.close()
    assert np.abs(got - want).max() <= 2e-4
