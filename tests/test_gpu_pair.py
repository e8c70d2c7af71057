"""GPU: lce_b200_bconv2d_run_fused_pair equals two lce_b200_bconv2d_run_fused calls bit for bit, and
a QuickNet graph with its residual blocks paired equals the graph without pairing."""
import ctypes as C

import numpy as np
import pytest

import lce_testlib as L
from compute_engine_b200 import host as H
from compute_engine_b200 import zoo

ACTS = (L.ACT_NONE, L.ACT_RELU, L.ACT_RELU6, L.ACT_RELU_N1_TO_1)


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
def test_gpu_pair_equals_two_fused_blocks():
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import assert_same_bits, dev, gpu_desc, path_counts
    rng = np.random.default_rng(12)
    # QuickNet's stage shapes at small batch, sizes that are not multiples of the tile, 1 x 1
    shapes = [(2, 56, 56, 64), (2, 28, 28, 128), (3, 13, 9, 64), (2, 1, 1, 128), (2, 2, 17, 64),
              (1, 15, 15, 128), (2, 14, 14, 64), (1, 7, 7, 128), (1, 30, 5, 64)]
    for n, (b, h, w, c) in enumerate(shapes):
        cases = [L.make_bconv_case(900 + 2 * n + k, b, h, w, c, 3, 3, c, activation=ACTS[(n + k) % 4])
                 for k in range(2)]
        plans = [capi.BConv2d(gpu_desc(capi, cs.desc), cs.filt, cs.mul, cs.bias) for cs in cases]
        x0 = (rng.standard_normal((b, h, w, c)) * 2).astype(np.float32)
        x0[0, 0, 0, :5] = [0.0, -0.0, 1.0, -1.0, 6.5]
        xq = dev(L.quantize(x0))
        res = dev(x0)
        act1, act2 = ACTS[n % 4], ACTS[(n + 2) % 4]
        x1, p1 = _run_fused(capi, torch, plans[0], xq, res, act1, True)
        want, want_pk = _run_fused(capi, torch, plans[1], p1, x1, act2, True)
        for packed in (True, False):
            before = path_counts(capi)
            launches = capi.launch_count()
            got, pk = plans[0].run_fused_pair(plans[1], xq, res, act1, act2, packed=packed)
            torch.cuda.synchronize()
            assert capi.launch_count() - launches == 1
            assert [y - x for x, y in zip(before, path_counts(capi))] == [0, 1, 0]
            tag = f"{b}x{h}x{w}x{c} acts {act1},{act2} packed {packed}"
            assert_same_bits(got.cpu().numpy(), want.cpu().numpy(), tag)
            if packed:
                assert_same_bits(pk.cpu().numpy(), want_pk.cpu().numpy(), tag + " signs")
            else:
                assert pk is None
        for p in plans:
            p.close()


@pytest.mark.gpu
def test_gpu_pair_refuses_other_layers():
    import torch
    from compute_engine_b200 import capi
    from test_gpu_parity import dev, gpu_desc
    for kw, msg in ((dict(c=256), "64 or 128"), (dict(pad_value=0), "pad_values = 1"),
                    (dict(stride=(2, 2)), "stride 1")):
        c = kw.pop("c", 64)
        cs = L.make_bconv_case(7, 1, 8, 8, c, 3, 3, c, **kw)
        plan = capi.BConv2d(gpu_desc(capi, cs.desc), cs.filt, cs.mul, cs.bias)
        x = dev(cs.inp)
        res = torch.zeros((1, 8, 8, c), device="cuda")
        with pytest.raises(capi.LceError, match=msg):
            plan.run_fused_pair(plan, x, res)
        plan.close()
    cs = L.make_bconv_case(8, 1, 8, 8, 64, 3, 3, 64)
    plan = capi.BConv2d(gpu_desc(capi, cs.desc), cs.filt, cs.mul, cs.bias)
    res = torch.zeros((1, 8, 8, 64), device="cuda")
    out = torch.empty_like(res)
    rc = capi.lib().lce_b200_bconv2d_run_fused_pair(
        plan._h, plan._h, C.c_void_p(dev(cs.inp).data_ptr()), C.c_void_p(res.data_ptr()), 0, 0,
        C.c_void_p(res.data_ptr()), None, None)
    assert rc != 0 and b"overlap" in capi.lib().lce_b200_last_error()
    plan.close()


@pytest.mark.gpu
@pytest.mark.parametrize("make,input_type", [(zoo.quicknet, "int8"), (zoo.quicknet_large, "int8"),
                                             (zoo.quicknet, "float32")])
def test_gpu_quicknet_paired_equals_unpaired(make, input_type):
    """Both arms keep every tensor (no arena reuse): pairing frees x1 and its signs, which moves the
    other tensors in the arena, and the unpaired graph's result already depends on that layout."""
    from compute_engine_b200 import capi
    blob = make(batch=1, image=224, seed=4, input_type=input_type)
    rng = np.random.default_rng(6)
    x = (rng.integers(-128, 128, (2, 224, 224, 3)).astype(np.int8) if input_type == "int8"
         else rng.standard_normal((2, 224, 224, 3)).astype(np.float32))
    outs, launches = [], []
    for pair in (False, True):
        g = H.HostGraph.from_tflite(blob, device_arena=True)
        g.resize_input(g.inputs()[0], x.shape)
        g.fuse_residual_blocks()
        g.fuse_float_glue()
        g.fuse_activation_chains()
        n_pairs = g.fuse_residual_pairs() if pair else 0
        g.preserve_all_tensors(True)
        g.allocate_tensors()
        g.write(g.inputs()[0], x)
        g.invoke()
        g.synchronize()
        l0 = capi.launch_count()
        g.invoke()
        g.synchronize()
        launches.append(capi.launch_count() - l0)
        outs.append(g.read(g.outputs()[0]))
        g.close()
    assert n_pairs == (4 if make is zoo.quicknet else 7)
    assert launches[0] - launches[1] == n_pairs   # one launch per pair where there were two
    assert np.array_equal(outs[0].view(np.uint8), outs[1].view(np.uint8))
