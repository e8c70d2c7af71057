"""ctypes binding of the C++ graph host (liblce_b200_host.so: csrc/host/*).

``HostGraph`` is the Subgraph-role object: tensors + nodes driven through
``TfLiteRegistration {init, free, prepare, invoke}`` exactly like TFLite drives the
reference's ops (tensorflow/lite/core/subgraph.cc:1271,1302,1368). With
``device_arena=True`` activations stay in HBM between ops.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import build as _build

# TfLiteType (c_api_types.h:116-137)
kTfLiteFloat32, kTfLiteInt32, kTfLiteUInt8, kTfLiteInt64, kTfLiteBool, kTfLiteInt8 = 1, 2, 3, 4, 6, 9
_NP = {kTfLiteFloat32: np.float32, kTfLiteInt32: np.int32, kTfLiteUInt8: np.uint8,
       kTfLiteInt64: np.int64, kTfLiteBool: np.bool_, kTfLiteInt8: np.int8}
_TFL = {np.dtype(v): k for k, v in _NP.items()}


class HostError(RuntimeError):
    pass


_lib = None


def lib():
    global _lib
    if _lib is None:
        path = _build.host_lib_path()
        if not os.path.exists(path):
            raise HostError(f"{path} is missing: run __graft_entry__.build()")
        # the CUDA C-ABI library must be resolvable first (rpath $ORIGIN handles it)
        _lib = C.CDLL(path, mode=C.RTLD_GLOBAL)
        L = _lib
        L.lce_host_graph_create.restype = C.c_void_p
        L.lce_host_last_error.restype = C.c_char_p
        L.lce_host_tensor_name.restype = C.c_char_p
        L.lce_host_tensor_data.restype = C.c_void_p
        L.lce_host_tensor_bytes.restype = C.c_size_t
        L.lce_host_arena_bytes.restype = C.c_size_t
        L.lce_host_stream.restype = C.c_void_p
        L.lce_host_tensor_scale.restype = C.c_float
        L.lce_host_node_time_ms.restype = C.c_double
        L.lce_host_node_name.restype = C.c_char_p
        L.lce_host_flex_get_float.restype = C.c_float
        L.lce_host_flex_get_float.argtypes = [C.c_void_p, C.c_size_t, C.c_char_p, C.c_float]
        for name in ("lce_host_graph_destroy", "lce_host_last_error", "lce_host_allocate_tensors",
                     "lce_host_invoke", "lce_host_num_tensors", "lce_host_num_nodes",
                     "lce_host_arena_bytes", "lce_host_stream", "lce_host_num_inputs",
                     "lce_host_num_outputs"):
            getattr(L, name).argtypes = [C.c_void_p]
    return _lib


def flex_int_map(items: dict) -> bytes:
    """FlexBuffers map of integer attributes, as LCE/mlir/ir/lce_ops.cc:36-64 writes."""
    keys = b"".join(k.encode() + b"\0" for k in items)
    vals = (C.c_int64 * len(items))(*[int(v) for v in items.values()])
    out = (C.c_uint8 * 1024)()
    n = lib().lce_host_flex_write_int_map(keys, vals, len(items), out, C.c_size_t(1024))
    if n < 0:
        raise HostError("flexbuffer write failed")
    return bytes(out[:n])


def flex_get_int(blob: bytes, key: str):
    found = C.c_int()
    buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob) if blob else None
    v = lib().lce_host_flex_get_int(buf, C.c_size_t(len(blob)), key.encode(), C.byref(found))
    return v if found.value else None


def flex_get_float(blob: bytes, key: str, default=0.0):
    """FlexMap::AsFloat: a FLOAT, INT, UINT or BOOL value as float32; default for a missing key."""
    buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob) if blob else None
    return lib().lce_host_flex_get_float(buf, C.c_size_t(len(blob)), key.encode(), C.c_float(default))


def flex_get_bool(blob: bytes, key: str, default=False):
    buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob) if blob else None
    return bool(lib().lce_host_flex_get_bool(buf, C.c_size_t(len(blob)), key.encode(), int(bool(default))))


def flex_map_size(blob: bytes):
    buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob) if blob else None
    return lib().lce_host_flex_map_size(buf, C.c_size_t(len(blob)))


def bconv2d_options(channels_in, stride=(1, 1), dilation=(1, 1), padding=0, pad_values=1,
                    activation=0) -> bytes:
    return flex_int_map({"channels_in": channels_in, "dilation_height_factor": dilation[0],
                         "dilation_width_factor": dilation[1],
                         "fused_activation_function": activation, "pad_values": pad_values,
                         "padding": padding, "stride_height": stride[0],
                         "stride_width": stride[1]})


def bmaxpool_options(filter_hw, stride_hw, padding) -> bytes:
    return flex_int_map({"padding": padding, "stride_width": stride_hw[1],
                         "stride_height": stride_hw[0], "filter_width": filter_hw[1],
                         "filter_height": filter_hw[0]})


def device_count() -> int:
    return int(lib().lce_host_device_count())


def set_device(index: int):
    if lib().lce_host_set_device(int(index)) != 0:
        raise HostError(f"cannot select CUDA device {index}")


def get_device() -> int:
    return int(lib().lce_host_get_device())


def register_custom(name: str, registration_ptr: int):
    """Expose an external TfLiteRegistration* (e.g. the oracle test double) as `name`."""
    lib().lce_host_register_custom(name.encode(), C.c_void_p(registration_ptr))


class HostGraph:
    def __init__(self, device_arena=True):
        self._g = C.c_void_p(lib().lce_host_graph_create(1 if device_arena else 0))
        self.device_arena = device_arena
        self._keep = []

    def close(self):
        if self._g:
            lib().lce_host_graph_destroy(self._g)
            self._g = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _err(self):
        return (lib().lce_host_last_error(self._g) or b"").decode()

    def _check(self, rc, what):
        if rc != 0:
            raise HostError(f"{what}: {self._err()}")

    def add_tensor(self, dtype, dims, const=None, scale=0.0, zero_point=0, quant=False, name=""):
        t = dtype if isinstance(dtype, int) else _TFL[np.dtype(dtype)]
        d = (C.c_int * len(dims))(*dims)
        if const is not None:
            const = np.ascontiguousarray(const, _NP[t])
            self._keep.append(const)
            ptr, nbytes = const.ctypes.data_as(C.c_void_p), const.nbytes
            if const.size == 0:
                ptr = (C.c_uint8 * 1)()
        else:
            ptr, nbytes = None, 0
        return lib().lce_host_add_tensor(self._g, t, d, len(dims), ptr, C.c_size_t(nbytes),
                                         1 if quant else 0, C.c_float(scale), zero_point,
                                         name.encode())

    def add_custom_node(self, op_name, inputs, outputs, options=b""):
        i = (C.c_int * len(inputs))(*inputs)
        o = (C.c_int * len(outputs))(*outputs)
        buf = (C.c_uint8 * max(len(options), 1)).from_buffer_copy(options or b"\0")
        idx = lib().lce_host_add_custom_node(self._g, op_name.encode(), i, len(inputs), o,
                                             len(outputs), buf, C.c_size_t(len(options)))
        if idx < 0:
            raise HostError(self._err())
        return idx

    def set_io(self, inputs, outputs):
        i = (C.c_int * len(inputs))(*inputs)
        o = (C.c_int * len(outputs))(*outputs)
        lib().lce_host_set_io(self._g, i, len(inputs), o, len(outputs))

    def allocate_tensors(self):
        self._check(lib().lce_host_allocate_tensors(self._g), "AllocateTensors")

    def resize_input(self, tensor, dims):
        d = (C.c_int * len(dims))(*dims)
        self._check(lib().lce_host_resize_input(self._g, tensor, d, len(dims)), "ResizeInputTensor")

    def invoke(self):
        self._check(lib().lce_host_invoke(self._g), "Invoke")

    def enable_cuda_graph(self, on=True):
        self._check(lib().lce_host_enable_cuda_graph(self._g, 1 if on else 0), "EnableCudaGraph")

    def fuse_residual_blocks(self):
        """LceBconv2d -> ADD [-> LceQuantize] => one node. Call before allocate_tensors."""
        return lib().lce_host_fuse_residual_blocks(self._g)

    def fuse_float_glue(self):
        """MAX_POOL_2D(2x2 s1 VALID) -> DEPTHWISE_CONV_2D(3x3) => one node."""
        return lib().lce_host_fuse_float_glue(self._g)

    def fuse_dense_blocks(self):
        """BinaryDenseNet's MUL -> ADD -> LceQuantize -> LceBconv2d -> CONCATENATION layers and
        MeliusNet's improvement layers (the same up to LceBconv2d, whose output is added to the
        map's last channels through STRIDED_SLICE -> ADD -> CONCATENATION) => one node each, writing
        into the block's final map in place. Call before the other passes (fuse_residual_blocks
        would take an improvement layer's LceBconv2d -> ADD) and allocate_tensors."""
        return lib().lce_host_fuse_dense_blocks(self._g)

    def fuse_channel_gates(self):
        """LceBconv2d -> MUL(gate [B,1,1,C]) -> PRELU -> ADD(shortcut) [-> MUL -> ADD -> LceQuantize]
        (Real-to-Binary Net's gated block and the next block's BatchNorm and sign) => one node.
        Call before fuse_activation_chains and allocate_tensors."""
        return lib().lce_host_fuse_channel_gates(self._g)

    def fuse_spatial_scales(self):
        """LceBconv2d -> MUL(constant scale [1,OH,OW,C]) -> ADD(shortcut) [-> MUL -> ADD -> LceQuantize]
        (XNOR-Net++'s scaled block and the next block's BatchNorm and sign) => one node. Call
        before fuse_float_glue, fuse_activation_chains and allocate_tensors."""
        return lib().lce_host_fuse_spatial_scales(self._g)

    def fuse_binary_bases(self):
        """ABC-Net's layer: N x (ADD(x, u_n) -> LceQuantize), M * N LceBconv2d terms, their
        left-to-right ADD chain, MUL -> ADD (BatchNorm) [-> ADD(shortcut)] [-> the next layer's
        shifted signs] => one node; planes of a map without such a producer => one node. Call
        first in fuse_all: fuse_residual_blocks would take ADD(t_00, t_01) as a residual block."""
        return lib().lce_host_fuse_binary_bases(self._g)

    def fuse_pooled_signs(self):
        """MAX_POOL_2D -> MUL(scale) -> ADD(shift) -> LceQuantize (BinaryAlexNet's and XNOR-Net's
        pooled BatchNorm and sign) => one node that writes only the signs. Call before
        fuse_channel_gates, fuse_activation_chains and allocate_tensors."""
        return lib().lce_host_fuse_pooled_signs(self._g)

    def fuse_quantized_activations(self):
        """[MAX_POOL_2D ->] MAXIMUM(0) -> MINIMUM(1) -> MUL(3) -> ROUND -> DIV(3) -> CONV_2D or
        FULLY_CONNECTED with +-alpha weights (DoReFaNet's 2-bit activations) => a node that writes the
        level's bit planes and a plain LceBconv2d over three planes. Exact integer arithmetic, so not
        bit-identical to the float convolution it replaces (Graph::FuseQuantizedActivations states
        the bound). Call before allocate_tensors."""
        return lib().lce_host_fuse_quantized_activations(self._g)

    def fuse_grouped_conv_affine(self):
        """A grouped CONV_2D (filter [C, kh, kw, C_in / g], g > 1) -> MUL(scale [C]) -> ADD(shift [C])
        => one node whose kernel applies the BatchNorm in its epilogue. Bit-identical; an ungrouped
        CONV_2D is never matched. Call before allocate_tensors."""
        return lib().lce_host_fuse_grouped_conv_affine(self._g)

    def fuse_activation_chains(self):
        """ADD -> PRELU -> ADD [-> ADD -> LceQuantize] (ReActNet's RPReLU / RSign, each step
        optional) => the epilogue of the preceding fused LceBconv2d+ADD node, or one node.
        Call after fuse_residual_blocks and before allocate_tensors."""
        return lib().lce_host_fuse_activation_chains(self._g)

    def fuse_upsample_merges(self):
        """RESIZE_NEAREST_NEIGHBOR(u) -> ADD(skip) [-> LceQuantize] (a segmentation decoder's merge)
        => one node that reads u at each output pixel's nearest source pixel. Call before
        fuse_activation_chains and allocate_tensors."""
        return lib().lce_host_fuse_upsample_merges(self._g)

    def fuse_resize_argmax(self):
        """RESIZE_BILINEAR -> ARG_MAX over the channel axis (a segmentation head's labels) => one
        node that never writes the resized map. Call before allocate_tensors."""
        return lib().lce_host_fuse_resize_argmax(self._g)

    def fuse_subpixel_convs(self):
        """CONV_2D -> DEPTH_TO_SPACE [-> ADD(RESIZE_BILINEAR(img))] (a super-resolution tail) => one
        node that never writes the conv output, the shuffled map or the resized image. Call before
        allocate_tensors."""
        return lib().lce_host_fuse_subpixel_convs(self._g)

    def fuse_binary_transpose_convs(self):
        """LceDequantize -> TRANSPOSE_CONV (+-1 weights, kernel = stride) [-> ADD(skip)] [-> LceQuantize]
        (a binary learned upsampler) => one node that runs it as a 1x1 binary convolution on the b1
        tensor instruction and stores each column at its pixel-shuffled address. Call before
        fuse_residual_blocks and allocate_tensors."""
        return lib().lce_host_fuse_binary_transpose_convs(self._g)

    def fuse_binary_fully_connected(self):
        """LceDequantize -> FULLY_CONNECTED (+-alpha_o weights, N % 64 == 0) [-> MUL -> ADD] [-> LceQuantize]
        (a binary dense layer) => one node that runs it as a 1x1 binary convolution of its rows on the b1
        tensor instruction, with alpha, the bias, the BatchNorm and the next sign in the store.
        Bit-identical when every alpha_o is a power of two; otherwise within the bound
        Graph::FuseBinaryFullyConnected states. Call before allocate_tensors."""
        return lib().lce_host_fuse_binary_fully_connected(self._g)

    def fuse_binary_fc_max(self):
        """LceDequantize -> FULLY_CONNECTED (+-alpha_o weights, N % 64 == 0) [-> MUL -> ADD] -> REDUCE_MAX
        over the points of [B, P, N] [-> LceQuantize] (a binary PointNet's last shared layer and its max
        pool) => one node that runs the layer on the b1 tensor instruction and reduces each image's
        columns in its store, never writing the [B, P, N] map. The same bits as the unfused ops under
        fuse_binary_fully_connected. Call before fuse_binary_fully_connected and allocate_tensors."""
        return lib().lce_host_fuse_binary_fc_max(self._g)

    def fuse_residual_pairs(self):
        """Two consecutive LceBconv2d+ADD[+LceQuantize] blocks whose intermediate nothing else
        reads => one node that keeps it on chip. Call after the other fusions."""
        return lib().lce_host_fuse_residual_pairs(self._g)

    def fuse_all(self):
        return (self.fuse_binary_bases() + self.fuse_dense_blocks() + self.fuse_binary_transpose_convs()
                + self.fuse_binary_fc_max() + self.fuse_binary_fully_connected() + self.fuse_residual_blocks()
                + self.fuse_spatial_scales()
                + self.fuse_float_glue() + self.fuse_upsample_merges() + self.fuse_resize_argmax()
                + self.fuse_subpixel_convs()
                + self.fuse_grouped_conv_affine() + self.fuse_quantized_activations() + self.fuse_pooled_signs() + self.fuse_channel_gates() + self.fuse_activation_chains()
                + self.fuse_residual_pairs())

    # ---- profiling / async IO (bench.py) ----
    def enable_profiling(self, on=True):
        lib().lce_host_enable_profiling(self._g, 1 if on else 0)

    def reset_profile(self):
        lib().lce_host_reset_profile(self._g)

    def node_times_ms(self):
        return [lib().lce_host_node_time_ms(self._g, i) for i in range(self.num_nodes())]

    def node_name(self, i):
        return lib().lce_host_node_name(self._g, i).decode()

    def node_io(self, i):
        n = lib().lce_host_node_num_inputs(self._g, i)
        return ([lib().lce_host_node_input(self._g, i, k) for k in range(n)],
                [lib().lce_host_node_output(self._g, i, 0)])

    def node_outputs(self, i):
        """Every output of node i (node_io lists output 0 only)."""
        return [lib().lce_host_node_output(self._g, i, k)
                for k in range(lib().lce_host_node_num_outputs(self._g, i))]

    def synchronize(self):
        self._check(lib().lce_host_synchronize(self._g), "Synchronize")

    def write_ptr(self, t, ptr, nbytes):
        """Async copy from a raw (pinned host or device) pointer on the graph's stream."""
        self._check(lib().lce_host_tensor_write(self._g, t, C.c_void_p(ptr), C.c_size_t(nbytes)),
                    "WriteTensor")

    def read_ptr_async(self, t, ptr, nbytes):
        self._check(lib().lce_host_tensor_read_async(self._g, t, C.c_void_p(ptr),
                                                     C.c_size_t(nbytes)), "ReadTensorAsync")

    def preserve_all_tensors(self, on=True):
        lib().lce_host_preserve_all_tensors(self._g, 1 if on else 0)

    @classmethod
    def from_tflite(cls, model_bytes: bytes, device_arena=True, use_reference_bconv=False,
                    use_indirect_bgemm=False):
        """use_reference_bconv / use_indirect_bgemm: the selectors of RegisterLCECustomOps
        (LCE/tflite/kernels/lce_ops_register.h:25-53): which registration "LceBconv2d" resolves
        to -- its validation rules and, under zero padding, which of the reference's two results
        is reproduced (include/lce_b200_types.h)."""
        L = lib()
        L.lce_host_graph_from_tflite_ex.restype = C.c_void_p
        err = C.c_char_p()
        buf = (C.c_uint8 * len(model_bytes)).from_buffer_copy(model_bytes)
        h = L.lce_host_graph_from_tflite_ex(buf, C.c_size_t(len(model_bytes)),
                                            1 if device_arena else 0,
                                            1 if use_reference_bconv else 0,
                                            1 if use_indirect_bgemm else 0, C.byref(err))
        if not h:
            raise HostError((err.value or b'').decode())
        g = cls.__new__(cls)
        g._g = C.c_void_p(h)
        g.device_arena = device_arena
        g._keep = []
        return g

    def shape(self, t):
        n = lib().lce_host_tensor_ndims(self._g, t)
        return tuple(lib().lce_host_tensor_dim(self._g, t, i) for i in range(n))

    def dtype(self, t):
        return _NP[lib().lce_host_tensor_type(self._g, t)]

    def nbytes(self, t):
        return int(lib().lce_host_tensor_bytes(self._g, t))

    def data_ptr(self, t):
        return lib().lce_host_tensor_data(self._g, t)

    def in_arena(self, t):
        """Whether tensor t lives in the tensor arena (a constant does not)."""
        return bool(lib().lce_host_tensor_in_arena(self._g, t))

    def num_tensors(self):
        return lib().lce_host_num_tensors(self._g)

    def arena_bytes(self):
        return int(lib().lce_host_arena_bytes(self._g))

    def stream(self):
        return lib().lce_host_stream(self._g)

    def inputs(self):
        return [lib().lce_host_input(self._g, k) for k in range(lib().lce_host_num_inputs(self._g))]

    def outputs(self):
        return [lib().lce_host_output(self._g, k) for k in range(lib().lce_host_num_outputs(self._g))]

    def num_nodes(self):
        return lib().lce_host_num_nodes(self._g)

    def write(self, t, array):
        a = np.ascontiguousarray(array, self.dtype(t))
        if a.nbytes != self.nbytes(t):
            raise HostError(f"write: tensor {t} holds {self.nbytes(t)} bytes, got {a.nbytes}")
        self._keep_last = a
        self._check(lib().lce_host_tensor_write(self._g, t, a.ctypes.data_as(C.c_void_p),
                                                C.c_size_t(a.nbytes)), "WriteTensor")

    def read(self, t):
        out = np.empty(self.shape(t), self.dtype(t))
        if out.nbytes:
            self._check(lib().lce_host_tensor_read(self._g, t, out.ctypes.data_as(C.c_void_p),
                                                   C.c_size_t(out.nbytes)), "ReadTensor")
        return out
