"""A minimal FlatBuffers builder and a `.tflite` (schema v3, "TFL3") writer.

There is no TensorFlow, no flatbuffers package and no model zoo offline, so the
QuickNet / QuickNetLarge / Bi-RealNet-18 graphs the benchmark runs are SYNTHESISED:
correct topology, random weights (compute_engine_b200/zoo.py), serialised here into
real `.tflite` files that the C++ graph host reads back through its own reader.
Field ids follow tensorflow/lite/schema/schema.fbs: Model :1609,
OperatorCode :1467, SubGraph :1540, Tensor :210, Operator :1493, Buffer :1562,
QuantizationParameters :75, builtin option tables :806-1106.
"""
from __future__ import annotations

import struct

import numpy as np


class FlatBuilder:
    """Back-to-front builder: objects are pushed towards lower addresses; a
    position is the distance of an object's first byte from the END of the buffer."""

    def __init__(self):
        self.chunks = []
        self.size = 0
        self.minalign = 1

    def _push(self, b: bytes):
        self.chunks.append(bytes(b))
        self.size += len(b)

    def _prep(self, align, additional):
        self.minalign = max(self.minalign, align)
        pad = (-(self.size + additional)) % align
        if pad:
            self._push(b"\0" * pad)

    def string(self, s: str) -> int:
        b = s.encode()
        self._prep(4, len(b) + 1)
        self._push(b + b"\0")
        self._push(struct.pack("<I", len(b)))
        return self.size

    def bytes_vector(self, data: bytes, align=1) -> int:
        self._prep(max(4, align), len(data))
        if align > 4:
            self._prep(align, len(data))
        self._push(data)
        self._push(struct.pack("<I", len(data)))
        return self.size

    def scalar_vector(self, fmt: str, values) -> int:
        esz = struct.calcsize(fmt)
        data = np.asarray(values).astype({"i": "<i4", "f": "<f4", "q": "<i8", "B": "u1",
                                          "b": "i1"}[fmt]).tobytes()
        n = len(data) // esz
        self._prep(4, len(data))
        self._prep(esz, len(data))
        self._push(data)
        self._push(struct.pack("<I", n))
        return self.size

    def offset_vector(self, positions) -> int:
        self._prep(4, 4 * len(positions))
        for p in reversed(positions):
            self._push(struct.pack("<I", self.size + 4 - p))
        self._push(struct.pack("<I", len(positions)))
        return self.size

    def table(self, fields: dict) -> int:
        """fields: {field_id: (fmt, value)}; fmt in b B h i q f (scalars, inline) or
        'o' (offset to an already written object at position `value`). Fields equal
        to None are omitted (schema default)."""
        start = self.size
        slots = {}
        order = sorted((k for k, v in fields.items() if v is not None),
                       key=lambda k: -(4 if fields[k][0] == "o" else struct.calcsize(fields[k][0])))
        for fid in order:
            fmt, val = fields[fid]
            if fmt == "o":
                self._prep(4, 4)
                self._push(struct.pack("<I", self.size + 4 - val))
            else:
                sz = struct.calcsize(fmt)
                self._prep(sz, sz)
                self._push(struct.pack("<" + fmt, val))
            slots[fid] = self.size
        self._prep(4, 4)
        self._push(b"\0\0\0\0")            # soffset to the vtable, patched below
        patch_index = len(self.chunks) - 1
        table_pos = self.size
        n = (max(slots) + 1) if slots else 0
        vt = struct.pack("<HH", 4 + 2 * n, table_pos - start)
        for fid in range(n):
            vt += struct.pack("<H", table_pos - slots[fid] if fid in slots else 0)
        self._prep(2, len(vt))
        self._push(vt)
        self.chunks[patch_index] = struct.pack("<i", self.size - table_pos)
        return table_pos

    def finish(self, root_pos: int, identifier: bytes) -> bytes:
        self._prep(self.minalign, 8)
        self._push(identifier)
        self._push(struct.pack("<I", self.size + 4 - root_pos))
        return b"".join(reversed(self.chunks))


# TensorType (schema.fbs:39) and BuiltinOperator codes (schema.fbs:259-325)
TENSOR_TYPE = {np.dtype(np.float32): 0, np.dtype(np.int32): 2, np.dtype(np.uint8): 3,
               np.dtype(np.int64): 4, np.dtype(np.bool_): 6, np.dtype(np.int8): 9}
OP = {"ADD": 0, "AVERAGE_POOL_2D": 1, "CONV_2D": 3, "DEPTHWISE_CONV_2D": 4,
      "FULLY_CONNECTED": 9, "MAX_POOL_2D": 17, "MUL": 18, "RELU": 19, "RESHAPE": 22,
      "SOFTMAX": 25, "MEAN": 40, "CUSTOM": 32, "CONCATENATION": 2, "PAD": 34, "PADV2": 60,
      "DEQUANTIZE": 6, "PRELU": 54, "LOGISTIC": 14, "STRIDED_SLICE": 45, "SPLIT": 49,
      "DIV": 42, "MAXIMUM": 55, "MINIMUM": 57, "ROUND": 116, "RESIZE_BILINEAR": 23,
      "RESIZE_NEAREST_NEIGHBOR": 97, "ARG_MAX": 56, "DEPTH_TO_SPACE": 5,
      "TRANSPOSE_CONV": 67, "REDUCE_MAX": 82}
# BuiltinOptions union tags (schema_generated.h:1652-1694)
OPT_TAG = {"CONV_2D": 1, "DEPTHWISE_CONV_2D": 2, "AVERAGE_POOL_2D": 5, "MAX_POOL_2D": 5,
           "FULLY_CONNECTED": 8, "SOFTMAX": 9, "ADD": 11, "MUL": 21, "RESHAPE": 17, "MEAN": 27,
           "CONCATENATION": 10, "PAD": 22, "PADV2": 43, "STRIDED_SLICE": 32, "SPLIT": 35, "DIV": 29,
           "RESIZE_BILINEAR": 15, "RESIZE_NEAREST_NEIGHBOR": 74, "ARG_MAX": 40, "DEPTH_TO_SPACE": 94,
           "TRANSPOSE_CONV": 49, "REDUCE_MAX": 27}
PADDING = {"SAME": 0, "VALID": 1}
ACT = {"NONE": 0, "RELU": 1, "RELU_N1_TO_1": 2, "RELU6": 3}


class TFLiteModel:
    """Collects tensors / operators of one subgraph, then serialises."""

    def __init__(self, description="compute_engine_b200 synthetic model"):
        self.tensors = []     # dict(name, shape, dtype, data|None, scale, zero_point)
        self.ops = []         # dict(kind, inputs, outputs, options)
        self.inputs, self.outputs = [], []
        self.description = description

    def add_tensor(self, name, shape, dtype=np.float32, data=None, scale=None, zero_point=0):
        if data is not None:
            data = np.ascontiguousarray(data, dtype)
            shape = data.shape
        self.tensors.append({"name": name, "shape": tuple(int(s) for s in shape),
                             "dtype": np.dtype(dtype), "data": data, "scale": scale,
                             "zero_point": zero_point})
        return len(self.tensors) - 1

    def add_op(self, kind, inputs, outputs, **options):
        self.ops.append({"kind": kind, "inputs": list(inputs), "outputs": list(outputs),
                         "options": options})

    def _builtin_options(self, fb, kind, o):
        act = ACT[o.get("activation", "NONE")]
        if kind == "CONV_2D":
            return fb.table({0: ("b", PADDING[o["padding"]]), 1: ("i", o["stride"][1]),
                             2: ("i", o["stride"][0]), 3: ("b", act),
                             4: ("i", o.get("dilation", (1, 1))[1]),
                             5: ("i", o.get("dilation", (1, 1))[0])})
        if kind == "DEPTHWISE_CONV_2D":
            return fb.table({0: ("b", PADDING[o["padding"]]), 1: ("i", o["stride"][1]),
                             2: ("i", o["stride"][0]), 3: ("i", o.get("depth_multiplier", 1)),
                             4: ("b", act), 5: ("i", o.get("dilation", (1, 1))[1]),
                             6: ("i", o.get("dilation", (1, 1))[0])})
        if kind in ("MAX_POOL_2D", "AVERAGE_POOL_2D"):
            return fb.table({0: ("b", PADDING[o["padding"]]), 1: ("i", o["stride"][1]),
                             2: ("i", o["stride"][0]), 3: ("i", o["filter"][1]),
                             4: ("i", o["filter"][0]), 5: ("b", act)})
        if kind == "FULLY_CONNECTED":   # field 2, keep_num_dims, only when passed: other models keep their bytes
            keep = ("b", 1 if o["keep_num_dims"] else 0) if "keep_num_dims" in o else None
            return fb.table({0: ("b", act), 2: keep})
        if kind == "SOFTMAX":
            return fb.table({0: ("f", float(o.get("beta", 1.0)))})
        if kind in ("ADD", "MUL", "DIV"):
            return fb.table({0: ("b", act)})
        if kind == "RESHAPE":
            return fb.table({0: ("o", fb.scalar_vector("i", o["new_shape"]))})
        if kind in ("MEAN", "REDUCE_MAX"):   # ReducerOptions: keep_dims
            return fb.table({0: ("b", 1 if o.get("keep_dims", False) else 0)})
        if kind == "CONCATENATION":
            return fb.table({0: ("i", int(o.get("axis", 0))), 1: ("b", act)})
        if kind in ("PAD", "PADV2"):
            return fb.table({})
        if kind == "STRIDED_SLICE":   # StridedSliceOptions
            return fb.table({0: ("i", o.get("begin_mask", 0)), 1: ("i", o.get("end_mask", 0)),
                             2: ("i", o.get("ellipsis_mask", 0)), 3: ("i", o.get("new_axis_mask", 0)),
                             4: ("i", o.get("shrink_axis_mask", 0)),
                             5: ("b", 1) if o.get("offset") else None})
        if kind == "SPLIT":           # SplitOptions
            return fb.table({0: ("i", o["num_splits"])})
        if kind == "ARG_MAX":         # ArgMaxOptions: output_type, a TensorType
            return fb.table({0: ("b", TENSOR_TYPE[np.dtype(o["output_type"])])})
        if kind == "DEPTH_TO_SPACE":  # DepthToSpaceOptions: block_size
            return fb.table({0: ("i", int(o["block_size"]))})
        if kind == "TRANSPOSE_CONV":  # TransposeConvOptions: padding, stride_w, stride_h, fused activation
            return fb.table({0: ("b", PADDING[o["padding"]]), 1: ("i", o["stride"][1]),
                             2: ("i", o["stride"][0]), 3: ("b", act)})
        flags = [("b", 1) if o.get(f) else None for f in ("align_corners", "half_pixel_centers")]
        if kind == "RESIZE_BILINEAR":  # ResizeBilinearOptions (0, 1: the deprecated new_height / new_width)
            return fb.table({2: flags[0], 3: flags[1]})
        if kind == "RESIZE_NEAREST_NEIGHBOR":  # ResizeNearestNeighborOptions
            return fb.table({0: flags[0], 1: flags[1]})
        return None

    def serialize(self) -> bytes:
        fb = FlatBuilder()
        # buffers: index 0 is the empty sentinel (schema.fbs:1626)
        buffers = [fb.table({})]
        buf_index = []
        for t in self.tensors:
            if t["data"] is None:
                buf_index.append(0)
            else:
                vec = fb.bytes_vector(t["data"].tobytes(), align=16)
                buffers.append(fb.table({0: ("o", vec)}))
                buf_index.append(len(buffers) - 1)
        tensor_pos = []
        for t, b in zip(self.tensors, buf_index):
            q = None
            if t["scale"] is not None:
                q = fb.table({2: ("o", fb.scalar_vector("f", [t["scale"]])),
                              3: ("o", fb.scalar_vector("q", [t["zero_point"]]))})
            name = fb.string(t["name"])
            shape = fb.scalar_vector("i", t["shape"])
            tensor_pos.append(fb.table({0: ("o", shape), 1: ("b", TENSOR_TYPE[t["dtype"]]),
                                        2: ("I", b), 3: ("o", name),
                                        4: ("o", q) if q is not None else None}))
        # operator codes: one per distinct builtin / custom name
        codes, code_pos = {}, []
        for op in self.ops:
            key = op["kind"]
            if key not in codes:
                codes[key] = len(codes)
                if key in OP:
                    code = OP[key]
                    code_pos.append(fb.table({0: ("b", min(code, 127)), 2: ("i", 1),
                                              3: ("i", code)}))
                else:   # custom op: builtin_code CUSTOM (32) + custom_code string
                    name = fb.string(key)
                    code_pos.append(fb.table({0: ("b", 32), 1: ("o", name), 2: ("i", 1),
                                              3: ("i", 32)}))
        op_pos = []
        for op in self.ops:
            kind = op["kind"]
            ins = fb.scalar_vector("i", op["inputs"])
            outs = fb.scalar_vector("i", op["outputs"])
            fields = {0: ("I", codes[kind]), 1: ("o", ins), 2: ("o", outs)}
            if kind in OP:
                opt = self._builtin_options(fb, kind, op["options"])
                if opt is not None:
                    fields[3] = ("B", OPT_TAG[kind])
                    fields[4] = ("o", opt)
            else:
                fields[5] = ("o", fb.bytes_vector(op["options"].get("custom_options", b"")))
                fields[6] = ("b", 0)   # FLEXBUFFERS
            op_pos.append(fb.table(fields))
        sub = fb.table({0: ("o", fb.offset_vector(tensor_pos)),
                        1: ("o", fb.scalar_vector("i", self.inputs)),
                        2: ("o", fb.scalar_vector("i", self.outputs)),
                        3: ("o", fb.offset_vector(op_pos)),
                        4: ("o", fb.string("main"))})
        model = fb.table({0: ("I", 3), 1: ("o", fb.offset_vector(code_pos)),
                          2: ("o", fb.offset_vector([sub])),
                          3: ("o", fb.string(self.description)),
                          4: ("o", fb.offset_vector(buffers))})
        return fb.finish(model, b"TFL3")


# --------------------------------------------------------------------------- #
# FlexBuffers maps of scalars (the custom ops' custom_options), in pure Python so that a model can
# be serialised without loading any native library. An int map is the same bytes as
# csrc/host/flexbuffer_map.cc::WriteFlexIntMap (tests/test_host_ops.py compares them, and both
# reproduce the blobs the real flatbuffers library wrote into LCE/mlir/tests/legalize-lce.mlir:9,21).
# --------------------------------------------------------------------------- #
_FBT_INT, _FBT_FLOAT, _FBT_MAP, _FBT_BOOL = 1, 3, 9, 26


def flex_map(items: dict) -> bytes:
    """A map of int, bool and float scalars as flexbuffers::Builder writes it: keys sorted by their
    bytes, every value at the map's one byte width (the least that fits all of them). A Python float
    is Builder::Float (float32, at least 4 bytes), a numpy float64 Builder::Double (8 bytes); a float
    at byte width 8 is stored as a double, as the builder stores it."""
    keys = list(items)
    order = sorted(range(len(keys)), key=lambda i: keys[i].encode())
    vals = [items[k] for k in keys]
    min_log2w = 0
    for v in vals:
        if isinstance(v, np.float64):
            min_log2w = 3
        elif isinstance(v, (float, np.floating)):
            min_log2w = max(min_log2w, 2)
    for log2w in range(min_log2w, 4):
        w = 1 << log2w
        lim = 1 << (8 * w - 1)
        out = bytearray()
        key_pos = []
        for k in keys:
            key_pos.append(len(out))
            out += k.encode() + b"\0"

        def align():
            while len(out) % w:
                out.append(0)

        def put(v):
            out.extend(int(v & ((1 << (8 * w)) - 1)).to_bytes(w, "little"))

        fits = True
        align()
        put(len(keys))
        keys_vec = len(out)
        for i in order:
            off = len(out) - key_pos[i]
            if off >= (1 << (8 * w)):
                fits = False
            put(off)
        align()
        put(len(out) - keys_vec)
        put(w)
        put(len(keys))
        mp = len(out)
        types = []
        for i in order:
            v = vals[i]
            if isinstance(v, (bool, np.bool_)):
                put(int(v))
                types.append(_FBT_BOOL)
            elif isinstance(v, (float, np.floating)):
                out.extend(struct.pack("<f" if w == 4 else "<d", float(v)))
                types.append(_FBT_FLOAT)
            else:
                v = int(v)
                if v >= lim or v < -lim:
                    fits = False
                put(v)
                types.append(_FBT_INT)
        for t in types:
            out.append((t << 2) | log2w)
        align()
        if len(out) - mp >= (1 << (8 * w)):
            fits = False
        if not fits:
            continue
        put(len(out) - mp)
        out.append((_FBT_MAP << 2) | log2w)
        out.append(w)
        return bytes(out)
    raise ValueError("flexbuffer map does not fit 64-bit offsets")


def flex_int_map(items: dict) -> bytes:
    """A map of integers (the LCE ops' attributes): byte widths 1, 2 or 4."""
    out = flex_map({k: int(v) for k, v in items.items()})
    if out[-1] > 4:
        raise ValueError("flexbuffer map does not fit 32-bit offsets")
    return out


def detection_postprocess_options(max_detections=100, max_classes_per_detection=1, detections_per_class=100,
                                  num_classes=90, use_regular_nms=False, nms_score_threshold=1e-8,
                                  nms_iou_threshold=0.6, y_scale=10.0, x_scale=10.0, h_scale=5.0,
                                  w_scale=5.0, converter_keys=True) -> bytes:
    """custom_options of TFLite_Detection_PostProcess, with the keys the TF Object Detection API's
    export writes (export_tflite_ssd_graph_lib.py) and, with converter_keys, the two flags TF's
    converter adds."""
    items = {"max_detections": max_detections, "max_classes_per_detection": max_classes_per_detection,
             "detections_per_class": detections_per_class, "use_regular_nms": bool(use_regular_nms),
             "nms_score_threshold": float(nms_score_threshold), "nms_iou_threshold": float(nms_iou_threshold),
             "num_classes": num_classes, "y_scale": float(y_scale), "x_scale": float(x_scale),
             "h_scale": float(h_scale), "w_scale": float(w_scale)}
    if converter_keys:
        items.update({"_output_quantized": True, "_support_output_type_float_in_quantized_op": True})
    return flex_map(items)


def bconv2d_options(channels_in, stride=(1, 1), dilation=(1, 1), padding=0, pad_values=1,
                    activation=0) -> bytes:
    """custom_options of LceBconv2d (keys as LCE/mlir/ir/lce_ops.cc:36-52)."""
    return flex_int_map({"channels_in": channels_in, "dilation_height_factor": dilation[0],
                         "dilation_width_factor": dilation[1],
                         "fused_activation_function": activation, "pad_values": pad_values,
                         "padding": padding, "stride_height": stride[0],
                         "stride_width": stride[1]})


def bmaxpool_options(filter_hw, stride_hw, padding) -> bytes:
    return flex_int_map({"padding": padding, "stride_width": stride_hw[1],
                         "stride_height": stride_hw[0], "filter_width": filter_hw[1],
                         "filter_height": filter_hw[0]})
