"""Graph-host / custom-op shell tests.

CPU part (no GPU): flexbuffer attribute decoding pinned on the byte blobs the
reference's own tests hold; a single LceBconv2d
56x56x256->256 k3 s1 driven init -> prepare -> invoke through the host with the
oracle-backed registration (bit-exact plumbing); the error behaviour of the CUDA
registrations' Init / Prepare (which need no device).
GPU part: the same single-op models with the CUDA registrations, device arena,
CUDA-graph replay and the host-arena (stock TFLite) staging path.
"""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

import lce_testlib as L
from compute_engine_b200 import host as H

GOLD_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# LCE/mlir/tests/legalize-lce.mlir:9 and :21 -- bytes written by the real flatbuffers library
BCONV_BLOB = bytes.fromhex(
    "6368616E6E656C735F696E0064696C6174696F6E5F6865696768745F666163746F720064696C6174696F6E5F"
    "77696474685F666163746F720066757365645F61637469766174696F6E5F66756E6374696F6E007061645F76"
    "616C7565730070616464696E67007374726964655F686569676874007374726964655F776964746800088277"
    "614C3329221508010803010100000101010404040404040404102401")
BMAXPOOL_BLOB = bytes.fromhex(
    "70616464696E67007374726964655F7769647468007374726964655F6865696768740066696C7465725F7769"
    "6474680066696C7465725F68656967687400050F1D412D3B050105020200020204040404040A2401")
# tensorflow/lite/testdata/custom_sinh.bin custom_options: {"T": 0}
SINH_BLOB = bytes.fromhex("540001030101010004022401")


@pytest.fixture(scope="module", autouse=True)
def oracle_ops():
    """Register the oracle-backed test doubles under 'Oracle*' names."""
    L.build_oracle()
    H.lib()
    ops = C.CDLL(os.path.join(L.ORACLE_DIR, "liblce_oracle_ops.so"))
    for op, fn in (("OracleBconv2d", "lce_oracle_Register_BCONV_2D"),
                   ("OracleQuantize", "lce_oracle_Register_QUANTIZE"),
                   ("OracleDequantize", "lce_oracle_Register_DEQUANTIZE"),
                   ("OracleBMaxPool2d", "lce_oracle_Register_BMAXPOOL_2D")):
        f = getattr(ops, fn)
        f.restype = C.c_void_p
        H.register_custom(op, f())
    return ops


def test_flexbuffer_known_answers():
    assert H.flex_map_size(BCONV_BLOB) == 8
    want = {"channels_in": 3, "dilation_height_factor": 1, "dilation_width_factor": 1,
            "fused_activation_function": 0, "pad_values": 0, "padding": 1, "stride_height": 1,
            "stride_width": 1}
    for k, v in want.items():
        assert H.flex_get_int(BCONV_BLOB, k) == v
    assert H.flex_get_int(BCONV_BLOB, "nonexistent") is None
    assert H.flex_map_size(BMAXPOOL_BLOB) == 5
    for k, v in {"filter_height": 2, "filter_width": 2, "padding": 0, "stride_height": 2,
                 "stride_width": 2}.items():
        assert H.flex_get_int(BMAXPOOL_BLOB, k) == v
    assert H.flex_map_size(SINH_BLOB) == 1 and H.flex_get_int(SINH_BLOB, "T") == 0
    assert H.flex_map_size(b"") == -1            # LceQuantize / LceDequantize: empty options
    assert H.flex_map_size(b"\x01\x02\x03") == -1


def test_flexbuffer_writer_reproduces_the_library_bytes():
    blob = H.flex_int_map({"channels_in": 3, "dilation_height_factor": 1,
                           "dilation_width_factor": 1, "fused_activation_function": 0,
                           "pad_values": 0, "padding": 1, "stride_height": 1, "stride_width": 1})
    assert blob == BCONV_BLOB
    assert H.bmaxpool_options((2, 2), (2, 2), 0) == BMAXPOOL_BLOB
    big = H.flex_int_map({"a": 70000, "b": -5, "channels_in": 3072})
    assert (H.flex_get_int(big, "a"), H.flex_get_int(big, "b"),
            H.flex_get_int(big, "channels_in")) == (70000, -5, 3072)


def build_bconv_graph(case, op_name, device_arena):
    d = case.desc
    g = H.HostGraph(device_arena=device_arena)
    cw = L.cdiv(d.channels_in, 32)
    t_in = g.add_tensor(np.int32, (d.batch, d.in_h, d.in_w, cw), name="input")
    t_f = g.add_tensor(np.int32, case.filt.shape, const=case.filt, name="filter")
    if d.out_type == L.OUT_BITPACKED:
        t_m = t_b = -1
        t_t = g.add_tensor(np.int32, (d.channels_out,), const=case.thr, name="thresholds")
        t_out = g.add_tensor(np.int32, (1, 1, 1, 1), name="output")
    else:
        t_m = g.add_tensor(np.float32, (d.channels_out,), const=case.mul, name="post_mul")
        t_b = g.add_tensor(np.float32, (d.channels_out,), const=case.bias, name="post_bias")
        t_t = -1
        if d.out_type == L.OUT_INT8:
            t_out = g.add_tensor(np.int8, (1, 1, 1, 1), scale=d.out_scale,
                                 zero_point=d.out_zero_point, quant=True, name="output")
        else:
            t_out = g.add_tensor(np.float32, (1, 1, 1, 1), name="output")
    opts = H.bconv2d_options(d.channels_in, (d.stride_h, d.stride_w), (d.dilation_h, d.dilation_w),
                             d.padding, d.pad_value, d.activation)
    g.add_custom_node(op_name, [t_in, t_f, t_m, t_b, t_t], [t_out], opts)
    g.set_io([t_in], [t_out])
    return g, t_in, t_out


# ---------------------------- CPU: plumbing ------------------------------- #
def test_config1_single_bconv_on_cpu_host_is_bit_exact():
    """A single LceBconv2d 56x56x256 -> 256, k3 s1 SAME."""
    with open(os.path.join(GOLD_DIR, "lce_golden.json")) as f:
        index = json.load(f)["index"]
    for e in index["bconv_full"][:6]:
        case = L.make_bconv_case(e["seed"], 1, 56, 56, 256, 3, 3, 256, 1, (1, 1), (1, 1),
                                 L.PADDING_SAME, e["pad_value"], e["activation"], e["out_type"])
        g, t_in, t_out = build_bconv_graph(case, "OracleBconv2d", device_arena=False)
        g.allocate_tensors()
        want_c = 8 if e["out_type"] == L.OUT_BITPACKED else 256
        assert g.shape(t_out) == (1, 56, 56, want_c)
        g.write(t_in, case.inp)
        g.invoke()
        out = g.read(t_out)
        assert hashlib.sha256(out.tobytes()).hexdigest() == e["sha256_reference_kernel"], e
        g.close()


def test_cpu_host_resize_reprepares():
    case = L.make_bconv_case(3, 1, 6, 6, 64, 3, 3, 16)
    g, t_in, t_out = build_bconv_graph(case, "OracleBconv2d", device_arena=False)
    g.allocate_tensors()
    g.write(t_in, case.inp)
    g.invoke()
    assert np.array_equal(g.read(t_out), L.bconv2d(case.desc, case.inp, case.filt, case.mul, case.bias))
    big = L.make_bconv_case(4, 5, 9, 7, 64, 3, 3, 16)
    big.filt, big.mul, big.bias = case.filt, case.mul, case.bias
    g.resize_input(t_in, (5, 9, 7, 2))     # batch is forced to 1 by the converter: resize + re-prepare
    g.allocate_tensors()
    assert g.shape(t_out) == (5, 9, 7, 16)
    g.write(t_in, big.inp)
    g.invoke()
    assert np.array_equal(g.read(t_out), L.bconv2d(big.desc, big.inp, big.filt, big.mul, big.bias))
    g.close()


def test_cpu_host_chain_quantize_bconv_bmaxpool_dequantize():
    rng = np.random.default_rng(0)
    x = rng.standard_normal((2, 8, 8, 64)).astype(np.float32)
    case = L.make_bconv_case(5, 2, 8, 8, 64, 3, 3, 64, out_type=L.OUT_BITPACKED)
    g = H.HostGraph(device_arena=False)
    t_x = g.add_tensor(np.float32, x.shape, name="x")
    t_q = g.add_tensor(np.int32, (1,) * 4, name="q")
    t_f = g.add_tensor(np.int32, case.filt.shape, const=case.filt)
    t_t = g.add_tensor(np.int32, (64,), const=case.thr)
    t_c = g.add_tensor(np.int32, (1,) * 4, name="conv")
    t_p = g.add_tensor(np.int32, (1,) * 4, name="pool")
    t_o = g.add_tensor(np.float32, (2, 4, 4, 64), name="out")
    g.add_custom_node("OracleQuantize", [t_x], [t_q])
    g.add_custom_node("OracleBconv2d", [t_q, t_f, -1, -1, t_t], [t_c], H.bconv2d_options(64))
    g.add_custom_node("OracleBMaxPool2d", [t_c], [t_p], H.bmaxpool_options((2, 2), (2, 2), 1))
    g.add_custom_node("OracleDequantize", [t_p], [t_o])
    g.set_io([t_x], [t_o])
    g.allocate_tensors()
    g.write(t_x, x)
    g.invoke()
    q = L.quantize(x)
    conv = L.bconv2d(case.desc, q, case.filt, thr=case.thr)
    pool = L.bmaxpool(L.BMaxPoolDesc(2, 8, 8, 2, 2, 2, 2, 2, L.PADDING_VALID), conv)
    assert np.array_equal(g.read(t_o), L.dequantize(pool, 64))
    assert g.arena_bytes() > 0
    g.close()


def _prepare_error(case, op_name, options=None, mutate=None):
    g, t_in, t_out = build_bconv_graph(case, op_name, device_arena=False)
    if options is not None:
        g.close()
        g = H.HostGraph(device_arena=False)
        d = case.desc
        t_in = g.add_tensor(np.int32, (d.batch, d.in_h, d.in_w, L.cdiv(d.channels_in, 32)))
        t_f = g.add_tensor(np.int32, case.filt.shape, const=case.filt)
        t_m = g.add_tensor(np.float32, (d.channels_out,), const=case.mul)
        t_b = g.add_tensor(np.float32, (d.channels_out,), const=case.bias)
        t_out = g.add_tensor(np.float32, (1, 1, 1, 1))
        g.add_custom_node(op_name, [t_in, t_f, t_m, t_b, -1], [t_out], options)
    with pytest.raises(H.HostError) as ei:
        g.allocate_tensors()
    g.close()
    return str(ei.value)


def test_cuda_registration_error_behaviour_matches_reference():
    """Init / Prepare of the CUDA ops need no device; their refusals and messages
    follow LCE/tflite/kernels/bconv2d.cc:94-116,143,169-200 and bconv2d_test.cc:858-917."""
    case = L.make_bconv_case(1, 1, 16, 16, 64, 3, 3, 128)
    # missing attribute -> Init records failure, Prepare returns an error
    bad = H.flex_int_map({"stride_height": 1, "stride_width": 1})
    assert "was not true" in _prepare_error(case, "LceBconv2d", options=bad)
    # pad_values outside {0,1}
    bad = H.bconv2d_options(64, pad_values=2)
    assert "pad_values must be 0 or 1" in _prepare_error(case, "LceBconv2d", options=bad)
    # zero padding + fused ReLU with the optimised registrations (ReluErrorDeathTest)
    zp = L.make_bconv_case(1, 1, 16, 16, 64, 3, 3, 128, pad_value=0, activation=L.ACT_RELU)
    for op in ("LceBconv2d:OPT_BGEMM", "LceBconv2d:OPT_INDIRECT_BGEMM"):
        assert "Zero-padding is only supported by" in _prepare_error(zp, op)
    # ... bitpacked and int8 output too (Int8ErrorDeathTest)
    for ot in (L.OUT_BITPACKED, L.OUT_INT8):
        zp = L.make_bconv_case(1, 1, 16, 16, 64, 3, 3, 128, pad_value=0, out_type=ot)
        assert "Zero-padding is only supported by" in _prepare_error(zp, "LceBconv2d:OPT_BGEMM")
    # the reference registration accepts zero padding only for even channels_in
    odd = L.make_bconv_case(1, 1, 8, 8, 33, 3, 3, 8, pad_value=1)
    odd.desc.pad_value = 0
    assert "Zero-padding is only supported by" in _prepare_error(odd, "LceBconv2d:REF")
    # grouped convolution with the OPT_BGEMM registration
    grp = L.make_bconv_case(1, 1, 8, 8, 64, 3, 3, 8, groups=2)
    assert "Grouped binary convolutions are not supported" in _prepare_error(grp, "LceBconv2d:OPT_BGEMM")
    # and Prepare succeeds (output resized) on the default CUDA registration without a device
    g, t_in, t_out = build_bconv_graph(case, "LceBconv2d", device_arena=False)
    g.allocate_tensors()
    assert g.shape(t_out) == (1, 16, 16, 128)
    g.close()


# ------------------------------ GPU --------------------------------------- #
@pytest.mark.gpu
@pytest.mark.parametrize("op", ["LceBconv2d", "LceBconv2d:REF", "LceBconv2d:OPT_INDIRECT_BGEMM"])
def test_gpu_single_op_models_through_registration(op):
    specs = [(2, 9, 7, 64, 3, 3, 64, 1, (1, 1), (1, 1), L.PADDING_SAME, 1, L.ACT_RELU, L.OUT_FLOAT),
             (1, 8, 8, 96, 3, 3, 40, 1, (2, 2), (1, 1), L.PADDING_VALID, 1, L.ACT_NONE, L.OUT_INT8),
             (3, 6, 6, 128, 2, 3, 70, 2, (1, 1), (1, 2), L.PADDING_SAME, 1, L.ACT_NONE, L.OUT_BITPACKED),
             (1, 12, 12, 64, 3, 3, 32, 1, (1, 1), (1, 1), L.PADDING_SAME, 0, L.ACT_NONE, L.OUT_FLOAT)]
    for n, s in enumerate(specs):
        (b, h, w, c, fh, fw, co, g_, st, dl, pad, pv, act, ot) = s
        case = L.make_bconv_case(40 + n, b, h, w, c, fh, fw, co, g_, st, dl, pad, pv, act, ot)
        g, t_in, t_out = build_bconv_graph(case, op, device_arena=True)
        g.allocate_tensors()
        g.write(t_in, case.inp)
        g.invoke()
        # zero padding: the reference registration computes it in the integers, the optimised ones
        # (and so the default CUDA registration) add the float correction afterwards
        kind = 0 if op.endswith(":REF") else 1
        want = L.bconv2d(case.desc, case.inp, case.filt, case.mul, case.bias, case.thr, kind=kind)
        got = g.read(t_out)
        assert got.shape == want.shape and np.array_equal(got.view(np.uint8), want.view(np.uint8)), s
        g.close()


@pytest.mark.gpu
def test_gpu_chain_with_cuda_graph_replay_and_resize():
    rng = np.random.default_rng(1)
    case = L.make_bconv_case(6, 4, 14, 14, 64, 3, 3, 64, out_type=L.OUT_BITPACKED)
    g = H.HostGraph(device_arena=True)
    t_x = g.add_tensor(np.float32, (4, 14, 14, 64), name="x")
    t_q = g.add_tensor(np.int32, (1,) * 4)
    t_f = g.add_tensor(np.int32, case.filt.shape, const=case.filt)
    t_t = g.add_tensor(np.int32, (64,), const=case.thr)
    t_c = g.add_tensor(np.int32, (1,) * 4)
    t_p = g.add_tensor(np.int32, (1,) * 4)
    t_o = g.add_tensor(np.float32, (4, 7, 7, 64), name="out")
    g.add_custom_node("LceQuantize", [t_x], [t_q])
    g.add_custom_node("LceBconv2d", [t_q, t_f, -1, -1, t_t], [t_c], H.bconv2d_options(64))
    g.add_custom_node("LceBMaxPool2d", [t_c], [t_p], H.bmaxpool_options((2, 2), (2, 2), 1))
    g.add_custom_node("LceDequantize", [t_p], [t_o])
    g.set_io([t_x], [t_o])
    g.allocate_tensors()
    g.enable_cuda_graph(True)

    def expect(x):
        d = L.BconvDesc(*[getattr(case.desc, n) for n, _ in case.desc._fields_])
        d.batch = x.shape[0]
        conv = L.bconv2d(d, L.quantize(x), case.filt, thr=case.thr)
        pool = L.bmaxpool(L.BMaxPoolDesc(x.shape[0], 14, 14, 2, 2, 2, 2, 2, L.PADDING_VALID), conv)
        return L.dequantize(pool, 64)

    for it in range(4):   # eager, capture, replay, replay -- fresh data every time
        x = rng.standard_normal((4, 14, 14, 64)).astype(np.float32)
        g.write(t_x, x)
        g.invoke()
        assert np.array_equal(g.read(t_o), expect(x)), it
    # resize the batch: Prepare runs again, the captured graph is rebuilt
    g.resize_input(t_x, (7, 14, 14, 64))
    g.resize_input(t_o, (7, 7, 7, 64))
    g.allocate_tensors()
    for it in range(3):
        x = rng.standard_normal((7, 14, 14, 64)).astype(np.float32)
        g.write(t_x, x)
        g.invoke()
        assert np.array_equal(g.read(t_o), expect(x)), it
    g.close()


@pytest.mark.gpu
def test_gpu_ops_under_a_host_arena_like_stock_tflite():
    """A stock TFLite interpreter hands the ops HOST pointers: invoke stages through HBM."""
    case = L.make_bconv_case(9, 2, 10, 10, 64, 3, 3, 32, activation=L.ACT_RELU)
    g, t_in, t_out = build_bconv_graph(case, "LceBconv2d", device_arena=False)
    g.allocate_tensors()
    g.write(t_in, case.inp)
    g.invoke()
    want = L.bconv2d(case.desc, case.inp, case.filt, case.mul, case.bias)
    assert np.array_equal(g.read(t_out).view(np.uint8), want.view(np.uint8))
    g.close()


def test_registration_selectors_change_zero_padding_legality():
    """HostGraph.from_tflite(use_reference_bconv / use_indirect_bgemm) resolves LceBconv2d like
    RegisterLCECustomOps (lce_ops_register.h:25-53): the reference registration refuses zero
    padding with an odd channel count, the optimised ones refuse it with a fused activation
    (bconv2d.cc:188-200); the default accepts the union."""
    from compute_engine_b200.tflite_writer import TFLiteModel, bconv2d_options

    def model(cin, act):
        rng = np.random.default_rng(0)
        m = TFLiteModel()
        cw = (cin + 31) // 32
        xq = m.add_tensor("xq", (1, 6, 6, cw), np.int32)
        f = m.add_tensor("f", None, np.int32,
                         data=rng.integers(-2**31, 2**31 - 1, (8, 3, 3, cw), dtype=np.int64).astype(np.int32))
        mul = m.add_tensor("mul", None, np.float32, data=rng.uniform(0.1, 1, 8))
        bias = m.add_tensor("bias", None, np.float32, data=rng.uniform(0.1, 1, 8))
        y = m.add_tensor("y", (1, 6, 6, 8))
        m.add_op("LceBconv2d", [xq, f, mul, bias, -1], [y],
                 custom_options=bconv2d_options(cin, pad_values=0, activation=act))
        m.inputs, m.outputs = [xq], [y]
        return m.serialize()

    def prepares(blob, **kw):
        g = H.HostGraph.from_tflite(blob, device_arena=False, **kw)
        try:
            g.allocate_tensors()
            return True
        except H.HostError as e:
            assert "Zero-padding is only supported" in str(e)
            return False
        finally:
            g.close()

    odd, relu = model(33, 0), model(64, 1)
    assert prepares(odd) and prepares(relu)                                  # default: union
    assert not prepares(odd, use_reference_bconv=True) and prepares(relu, use_reference_bconv=True)
    assert prepares(odd, use_indirect_bgemm=True) and not prepares(relu, use_indirect_bgemm=True)
