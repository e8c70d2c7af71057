"""Synthetic model zoo: the model families the graph host runs, emitted as real
`.tflite` graphs with the op sequence the LCE converter produces (LceQuantize ->
LceBconv2d with folded BatchNorm multiplier/bias and fused ReLU -> ADD shortcut ...),
random weights (seeded), correct topology.

The topologies are NOT in /root/reference (they live in larq-zoo, absent offline);
they are restated from the public QuickNet / Bi-Real Net descriptions:
  QuickNet(-Large, -Small): stem [conv3x3 s2 -> BN/ReLU -> depthwise3x3 s2 -> conv1x1 -> BN],
    the first conv filters[0] // 4 wide, sections of residual blocks [sign -> binary conv3x3
    (one-padding, ReLU fused, BN folded) -> + shortcut] with filters (64,128,256,512) and blocks
    (4,4,4,4) / (6,8,12,6), or filters (32,64,256,512) and blocks (4,4,4,4) for QuickNetSmall
    (larq-zoo's QuickNetSmallFactory),
    transitions [ReLU? no: maxpool2x2 s1 -> blur depthwise3x3 s2 -> conv1x1 -> BN],
    head [ReLU -> global average pool -> dense 1000 -> softmax].
  Bi-RealNet-18: conv7x7 s2 + BN + maxpool3x3 s2; 16 binary conv3x3 (zero padding,
    per-channel scale folded into the multiplier) each with its own shortcut,
    downsampling shortcuts avgpool2x2 s2 -> conv1x1 -> BN; head as above.
"""
from __future__ import annotations

import numpy as np

# Pure Python on purpose (numpy + the flatbuffer / flexbuffer writers of tflite_writer.py): no
# native library is loaded, so bench.py's reference arm can synthesise the very same model bytes
# by loading these two files alone (importlib, not the package).
try:
    from .tflite_writer import TFLiteModel, bconv2d_options, detection_postprocess_options
except ImportError:      # loaded as a stand-alone file next to tflite_writer.py
    from tflite_writer import TFLiteModel, bconv2d_options, detection_postprocess_options


# Quantisation of an int8 image input (`input_type="int8"`): what the converter attaches to the
# input tensor with inference_input_type=tf.int8; N(0,1) images span about +-4.
INPUT_SCALE, INPUT_ZERO_POINT = 4.0 / 127.0, 0


def quantize_images(x, scale=INPUT_SCALE, zero_point=INPUT_ZERO_POINT):
    """float images -> the int8 tensor an int8-input model expects."""
    return np.clip(np.rint(np.asarray(x, np.float32) / np.float32(scale)) + zero_point, -128, 127).astype(np.int8)


class _Builder:
    def __init__(self, seed, batch, name):
        self.rng = np.random.default_rng(seed)
        self.m = TFLiteModel(name)
        self.batch = batch
        self.n = 0

    def _name(self, p):
        self.n += 1
        return f"{p}_{self.n}"

    def act(self, shape, dtype=np.float32):
        return self.m.add_tensor(self._name("t"), shape, dtype)

    def image_input(self, shape, input_type):
        """The graph's input: float32 images, or int8 images + the DEQUANTIZE the converter
        places behind an int8 input (then a step ships a quarter of the bytes to the device)."""
        if input_type in ("float32", np.float32, None):
            x = self.m.add_tensor("input", shape, np.float32)
            self.m.inputs = [x]
            return x
        if input_type not in ("int8", np.int8):
            raise ValueError(f"unsupported input_type {input_type!r}")
        q = self.m.add_tensor("input", shape, np.int8, scale=INPUT_SCALE, zero_point=INPUT_ZERO_POINT)
        self.m.inputs = [q]
        x = self.act(shape)
        self.m.add_op("DEQUANTIZE", [q], [x])
        return x

    def const(self, data, dtype=np.float32, name="w"):
        return self.m.add_tensor(self._name(name), None, dtype, data=data)

    def bn(self, c):
        """BatchNorm folded to y = x * scale + shift."""
        scale = self.rng.uniform(0.5, 1.5, c).astype(np.float32)
        shift = self.rng.uniform(-0.5, 0.5, c).astype(np.float32)
        return scale, shift

    def batchnorm(self, t, ts, activation="NONE"):
        """An unfolded BatchNorm as the converter leaves it: MUL(scale) -> ADD(shift)."""
        scale, shift = self.bn(ts[3])
        u = self.act(ts)
        self.m.add_op("MUL", [t, self.const(scale, name="bn_scale")], [u])
        return self.add(u, self.const(shift, name="bn_shift"), ts, activation)

    # ---- float builtins ----
    def conv(self, x, xs, cout, k, stride, padding="SAME", activation="NONE", bn=True,
             use_bias=True, binary=False):
        """binary: +-1 weights, what the converter leaves of a binary kernel on a float input."""
        b, h, w, cin = xs
        if binary:
            wt = (self.rng.integers(0, 2, (cout, k, k, cin), dtype=np.int8) * 2 - 1).astype(np.float32)
        else:
            wt = self.rng.standard_normal((cout, k, k, cin)).astype(np.float32) * np.float32(
                1.0 / np.sqrt(k * k * cin))
        bias = np.zeros(cout, np.float32)
        if bn:
            s, t = self.bn(cout)
            wt = wt * s[:, None, None, None]
            bias = t
        oh = -(-h // stride) if padding == "SAME" else (h - k) // stride + 1
        ow = -(-w // stride) if padding == "SAME" else (w - k) // stride + 1
        y = self.act((b, oh, ow, cout))
        self.m.add_op("CONV_2D", [x, self.const(wt), self.const(bias, name="b") if use_bias else -1],
                      [y], padding=padding, stride=(stride, stride), activation=activation)
        return y, (b, oh, ow, cout)

    def depthwise(self, x, xs, k, stride, padding="SAME", blur=False, bn=False, activation="NONE"):
        b, h, w, c = xs
        if blur:   # blurpool: fixed binomial kernel
            a = np.array([1.0, 2.0, 1.0], np.float32)
            kern = np.outer(a, a) / 16.0
            wt = np.broadcast_to(kern[None, :, :, None], (1, k, k, c)).astype(np.float32).copy()
        else:
            wt = self.rng.standard_normal((1, k, k, c)).astype(np.float32) / np.float32(k)
        bias = np.zeros(c, np.float32)
        if bn:
            s, t = self.bn(c)
            wt = wt * s[None, None, None, :]
            bias = t
        oh = -(-h // stride) if padding == "SAME" else (h - k) // stride + 1
        ow = -(-w // stride) if padding == "SAME" else (w - k) // stride + 1
        y = self.act((b, oh, ow, c))
        self.m.add_op("DEPTHWISE_CONV_2D", [x, self.const(wt), self.const(bias, name="b")], [y],
                      padding=padding, stride=(stride, stride), depth_multiplier=1, activation=activation)
        return y, (b, oh, ow, c)

    def pool(self, kind, x, xs, k, stride, padding):
        b, h, w, c = xs
        oh = -(-h // stride) if padding == "SAME" else (h - k) // stride + 1
        ow = -(-w // stride) if padding == "SAME" else (w - k) // stride + 1
        y = self.act((b, oh, ow, c))
        self.m.add_op(kind, [x], [y], padding=padding, stride=(stride, stride), filter=(k, k))
        return y, (b, oh, ow, c)

    def add(self, a, b_, shape, activation="NONE"):
        y = self.act(shape)
        self.m.add_op("ADD", [a, b_], [y], activation=activation)
        return y

    def relu(self, x, shape):
        y = self.act(shape)
        self.m.add_op("RELU", [x], [y])
        return y

    def transpose_conv(self, x, xs, out_shape, binary=False):
        """TRANSPOSE_CONV 2x2 / stride 2 (SAME) from xs to out_shape with bias. binary: larq's
        QuantConv2DTranspose(ste_sign, ste_sign) as the converter leaves it, LceQuantize -> LceDequantize
        -> TRANSPOSE_CONV with +-1 weights."""
        cin, cout = xs[3], out_shape[3]
        if binary:
            x = self.quantize(x, xs)
            deq = self.act(xs)
            self.m.add_op("LceDequantize", [x], [deq], custom_options=b"")
            x = deq
            wt = (self.rng.integers(0, 2, (cout, 2, 2, cin), dtype=np.int8) * 2 - 1).astype(np.float32)
        else:
            wt = self.rng.standard_normal((cout, 2, 2, cin)).astype(np.float32) * np.float32(1.0 / np.sqrt(cin))
        bias = self.rng.uniform(-0.5, 0.5, cout).astype(np.float32)
        y = self.act(out_shape)
        self.m.add_op("TRANSPOSE_CONV", [self.const(np.array(out_shape, np.int32), np.int32, "output_shape"),
                                         self.const(wt), x, self.const(bias, name="b")], [y],
                      padding="SAME", stride=(2, 2), activation="NONE")
        return y

    # ---- LCE custom ops ----
    def quantize(self, x, xs):
        b, h, w, c = xs
        y = self.act((b, h, w, (c + 31) // 32), np.int32)
        self.m.add_op("LceQuantize", [x], [y], custom_options=b"")
        return y

    def bconv(self, xq, xs, cout, k=3, stride=1, pad_values=1, activation="RELU", dilation=1,
              padding="SAME", bitpacked=False, fold_bn=True, groups=1):
        """LceBconv2d with float output; BN (and for Bi-RealNet the kernel scale)
        folded into post_activation_multiplier / bias like the converter does
        (LCE/mlir/transforms/optimize_patterns_common.td:39-113). bitpacked: int32 output, the
        signs the next binary layer reads, with synthetic int32 thresholds [cout] around half the
        accumulators' range K = k * k * cin (inputs 2 and 3 absent) in place of the BN.
        fold_bn=False: nothing is folded, post_activation_multiplier 1 and bias 0.
        groups > 1: a grouped layer, filter [cout, k, k, cin / groups / 32 words] (cin / groups a
        multiple of 32), channels_in still cin. Each group's signs and then its BN (or thresholds)
        are drawn in turn, as `groups` ungrouped layers of cin / groups -> cout / groups would
        draw them, and concatenated along the output channels."""
        b, h, w, cin = xs
        if cin % groups or cout % groups or (groups > 1 and (cin // groups) % 32):
            raise ValueError(f"groups={groups} needs cin / groups a multiple of 32 and cout divisible")
        cin_g, cout_g = cin // groups, cout // groups
        kk = k * k * cin_g
        filts, thrs, muls, shifts = [], [], [], []
        for _ in range(groups):
            signs = self.rng.integers(0, 2, (cout_g, k, k, cin_g), dtype=np.int8) * 2 - 1
            bits = np.zeros((cout_g, k, k, ((cin_g + 31) // 32) * 32), np.uint32)
            bits[..., :cin_g] = signs < 0
            filts.append((bits.reshape(cout_g, k, k, -1, 32) << np.arange(32, dtype=np.uint32)).sum(
                -1, dtype=np.uint64).astype(np.uint32).view(np.int32))
            if bitpacked:
                thrs.append(np.rint(kk / 2 + self.rng.standard_normal(cout_g) * np.sqrt(kk) * 0.75).astype(np.int32))
            elif fold_bn:
                s, t = self.bn(cout_g)
                muls.append((s / np.float32(kk) * np.float32(4.0)).astype(np.float32))
                shifts.append(t)
            else:
                muls.append(np.ones(cout_g, np.float32))
                shifts.append(np.zeros(cout_g, np.float32))
        filt = np.concatenate(filts)
        if padding == "SAME":
            oh, ow = -(-h // stride), -(-w // stride)
        else:
            oh, ow = (h - k) // stride + 1, (w - k) // stride + 1
        act_code = {"NONE": 0, "RELU": 1}[activation]
        opts = bconv2d_options(cin, (stride, stride), (dilation, dilation), {"SAME": 0, "VALID": 1}[padding],
                               pad_values, act_code)
        if bitpacked:
            thr = np.concatenate(thrs)
            y = self.act((b, oh, ow, (cout + 31) // 32), np.int32)
            self.m.add_op("LceBconv2d", [xq, self.const(filt, np.int32, "bfilter"), -1, -1,
                                         self.const(thr, np.int32, "thr")], [y], custom_options=opts)
            return y, (b, oh, ow, cout)
        mul, t = np.concatenate(muls), np.concatenate(shifts)
        y = self.act((b, oh, ow, cout))
        self.m.add_op("LceBconv2d",
                      [xq, self.const(filt, np.int32, "bfilter"), self.const(mul, name="pmul"),
                       self.const(t, name="pbias"), -1], [y], custom_options=opts)
        return y, (b, oh, ow, cout)

    def head(self, x, xs, classes=1000, relu=True):
        b, h, w, c = xs
        if relu:
            x = self.relu(x, xs)
        axes = self.const(np.array([1, 2], np.int32), np.int32, "axes")
        pooled = self.act((b, c))
        self.m.add_op("MEAN", [x, axes], [pooled], keep_dims=False)
        wt = self.rng.standard_normal((classes, c)).astype(np.float32) / np.float32(np.sqrt(c))
        logits = self.act((b, classes))
        self.m.add_op("FULLY_CONNECTED", [pooled, self.const(wt),
                                          self.const(np.zeros(classes, np.float32), name="b")],
                      [logits])
        probs = self.act((b, classes))
        self.m.add_op("SOFTMAX", [logits], [probs], beta=1.0)
        return probs


def quicknet(batch=1, blocks=(4, 4, 4, 4), filters=(64, 128, 256, 512), seed=0, image=224,
             name="QuickNet", input_type="float32"):
    """Returns the serialized .tflite bytes."""
    g = _Builder(seed, batch, name)
    x, xs = _quicknet_encoder(g, batch, image, input_type, blocks, filters)[-1]
    probs = g.head(x, xs)
    g.m.outputs = [probs]
    return g.m.serialize()


def _quicknet_encoder(g, batch, image, input_type, blocks, filters):
    """QuickNet's stem, sections and transitions; returns each section's final map (x, shape)."""
    xs = (batch, image, image, 3)
    x = g.image_input(xs, input_type)
    # stem
    x, xs = g.conv(x, xs, filters[0] // 4, 3, 2, activation="RELU")
    x, xs = g.depthwise(x, xs, 3, 2, bn=True)
    x, xs = g.conv(x, xs, filters[0], 1, 1)
    sections = []
    for si, (nb, f) in enumerate(zip(blocks, filters)):
        if si > 0:   # transition block
            x, xs = g.pool("MAX_POOL_2D", x, xs, 2, 1, "VALID")
            x, xs = g.depthwise(x, xs, 3, 2, blur=True)
            x, xs = g.conv(x, xs, f, 1, 1)
        for _ in range(nb):
            q = g.quantize(x, xs)
            y, _ = g.bconv(q, xs, f, pad_values=1, activation="RELU")
            x = g.add(y, x, xs)
        sections.append((x, xs))
    return sections


def quicknet_seg(batch=1, seed=0, image=224, input_type="float32", classes=21, decoder_blocks=2, labels=None,
                 upsample="nearest"):
    """A binary segmentation network: QuickNet's encoder, then a decoder of three stages that merge
    the coarse map with the encoder's skip maps as TF2's UpSampling2D and Keras' Add emit them, then a
    per-pixel classifier at full resolution. Each stage, for (coarse, skip) = (s4, s3), (d3, s2),
    (d2, s1): CONV_2D 1x1 to the skip's channels (BatchNorm folded, no activation) ->
    RESIZE_NEAREST_NEIGHBOR x2 (half_pixel_centers) -> ADD(skip) -> `decoder_blocks` residual blocks
    [LceQuantize -> LceBconv2d 3x3 (one-padding, ReLU, BatchNorm folded) -> ADD shortcut]. Head:
    CONV_2D 1x1 64 -> classes with bias -> RESIZE_BILINEAR to (image, image) (half_pixel_centers), the
    logits [B, image, image, classes]. With labels="int64" or "int32" the head ends in ARG_MAX over
    the channel axis (the axis a constant int32 -1), as tf.argmax(logits, axis=-1) converts, and the
    output is the label map [B, image, image] of that type. image must be a multiple of 32 (the
    encoder halves it five times and the decoder doubles it back).
    upsample picks how each stage brings the coarse map to the skip's size and channels:
    "nearest" the CONV_2D 1x1 -> RESIZE_NEAREST_NEIGHBOR above; "transpose" one float TRANSPOSE_CONV
    2x2 / stride 2 with bias (Keras' Conv2DTranspose); "binary_transpose" larq's
    QuantConv2DTranspose(ste_sign, ste_sign) as the converter leaves it without a binary transposed
    op: LceQuantize -> LceDequantize -> TRANSPOSE_CONV 2x2 / stride 2 with +-1 weights and a bias."""
    if upsample not in ("nearest", "transpose", "binary_transpose"):
        raise ValueError(f"quicknet_seg upsample must be 'nearest', 'transpose' or 'binary_transpose', "
                         f"not {upsample!r}")
    if image % 32:
        raise ValueError(f"quicknet_seg needs an image size that is a multiple of 32, not {image}")
    if labels not in (None, "int32", "int64"):
        raise ValueError(f"quicknet_seg labels must be None, 'int32' or 'int64', not {labels!r}")
    g = _Builder(seed, batch, "QuickNetSeg")
    sections = _quicknet_encoder(g, batch, image, input_type, (4, 4, 4, 4), (64, 128, 256, 512))
    x, xs = sections[-1]

    def size(h, w):
        return g.const(np.array([h, w], np.int32), np.int32, "size")

    for skip, ss in reversed(sections[:-1]):
        if upsample == "nearest":
            x, xs = g.conv(x, xs, ss[3], 1, 1)
            up = g.act(ss)
            g.m.add_op("RESIZE_NEAREST_NEIGHBOR", [x, size(ss[1], ss[2])], [up], half_pixel_centers=True)
        else:
            up = g.transpose_conv(x, xs, ss, binary=upsample == "binary_transpose")
        x, xs = g.add(up, skip, ss), ss
        for _ in range(decoder_blocks):
            q = g.quantize(x, xs)
            y, _ = g.bconv(q, xs, xs[3], pad_values=1, activation="RELU")
            x = g.add(y, x, xs)
    b, h, w, c = xs
    wt = g.rng.standard_normal((classes, 1, 1, c)).astype(np.float32) / np.float32(np.sqrt(c))
    bias = g.rng.uniform(-0.5, 0.5, classes).astype(np.float32)
    logits = g.act((b, h, w, classes))
    g.m.add_op("CONV_2D", [x, g.const(wt), g.const(bias, name="b")], [logits], padding="SAME",
               stride=(1, 1), activation="NONE")
    out = g.act((b, image, image, classes))
    g.m.add_op("RESIZE_BILINEAR", [logits, size(image, image)], [out], half_pixel_centers=True)
    if labels is not None:
        logits, out = out, g.act((b, image, image), np.dtype(labels))
        g.m.add_op("ARG_MAX", [logits, g.const(np.array(-1, np.int32), np.int32, "axis")], [out],
                   output_type=np.dtype(labels))
    g.m.outputs = [out]
    return g.m.serialize()


def binary_srnet(batch=1, seed=0, image=64, input_type="float32", scale=2, channels=64, blocks=16, residual=True):
    """A binary super-resolution network in EDSR-baseline's layout. Head: CONV_2D 3x3, 3 -> `channels`,
    with bias. Body: `blocks` residual blocks [LceQuantize -> LceBconv2d 3x3 (one-padding, BatchNorm
    folded, no activation) -> ADD shortcut], then the long skip ADD(body, head). Tail: CONV_2D 3x3,
    `channels` -> 3 * scale^2, with bias -> DEPTH_TO_SPACE(scale), and with `residual` an ADD of the
    image resized to the output's size by RESIZE_BILINEAR (half_pixel_centers), so the network learns
    the difference to a bilinear upscale. The tail is ESPCN's single sub-pixel convolution, not EDSR's
    wider upsampler (a 64 -> 256 convolution and a shuffle per factor 2). image is an int or an (h, w)
    pair; the output is [B, scale * h, scale * w, 3]. With input_type="int8" the DEQUANTIZE output
    feeds both the head and the resize."""
    if scale not in (2, 3, 4):
        raise ValueError(f"binary_srnet needs scale 2, 3 or 4, not {scale}")
    h, w = (image, image) if isinstance(image, int) else (int(image[0]), int(image[1]))
    g = _Builder(seed, batch, "BinarySRNet")
    xs = (batch, h, w, 3)
    img = g.image_input(xs, input_type)

    def conv3x3(t, cin, cout):
        wt = g.rng.standard_normal((cout, 3, 3, cin)).astype(np.float32) * np.float32(1.0 / np.sqrt(9 * cin))
        bias = g.rng.uniform(-0.1, 0.1, cout).astype(np.float32)
        y = g.act((batch, h, w, cout))
        g.m.add_op("CONV_2D", [t, g.const(wt), g.const(bias, name="b")], [y], padding="SAME", stride=(1, 1),
                   activation="NONE")
        return y

    ts = (batch, h, w, channels)
    head = x = conv3x3(img, 3, channels)
    for _ in range(blocks):
        q = g.quantize(x, ts)
        y, _ = g.bconv(q, ts, channels, pad_values=1, activation="NONE")
        x = g.add(y, x, ts)
    x = g.add(x, head, ts)
    sub = conv3x3(x, channels, 3 * scale * scale)
    out_shape = (batch, scale * h, scale * w, 3)
    out = g.act(out_shape)
    g.m.add_op("DEPTH_TO_SPACE", [sub], [out], block_size=scale)
    if residual:
        up = g.act(out_shape)
        size = g.const(np.array([scale * h, scale * w], np.int32), np.int32, "size")
        g.m.add_op("RESIZE_BILINEAR", [img, size], [up], half_pixel_centers=True)
        out = g.add(out, up, out_shape)
    g.m.outputs = [out]
    return g.m.serialize()


def ssd_anchors(grids, min_scale=0.2, max_scale=0.95):
    """The TF Object Detection API's SSD anchors (anchor_generators/multiple_grid_anchor_generator.py,
    create_ssd_anchors with its defaults) for feature maps of `grids` [(h, w), ...], in float32 as
    TFLite_Detection_PostProcess reads them: [N, 4] rows of (y_center, x_center, height, width),
    ordered by (row, column, anchor) as a head's [B, h, w, A * 4] map reshapes to [B, h * w * A, 4].
    The lowest map gets (0.1, 1), (s, 2), (s, 1/2); every other map (s, r) for the aspect ratios
    r in (1, 2, 3, 1/2, 1/3) and (sqrt(s * s_next), 1), with the scales s spread evenly over
    [min_scale, max_scale] and 1 after the last."""
    f32 = np.float32
    n = len(grids)
    scales = [min_scale + (max_scale - min_scale) * i / (n - 1) for i in range(n)] + [1.0]
    out = []
    for layer, (h, w) in enumerate(grids):
        s, s_next = scales[layer], scales[layer + 1]
        if layer == 0:
            specs = [(0.1, 1.0), (s, 2.0), (s, 0.5)]
        else:
            specs = [(s, r) for r in (1.0, 2.0, 3.0, 0.5, 1.0 / 3.0)] + [(np.sqrt(s * s_next), 1.0)]
        sc = np.array([p[0] for p in specs], f32)
        ar = np.sqrt(np.array([p[1] for p in specs], f32))
        heights, widths = sc / ar, sc * ar
        yc = (np.arange(h, dtype=f32) * f32(1.0 / h) + f32(0.5 / h)).astype(f32)
        xc = (np.arange(w, dtype=f32) * f32(1.0 / w) + f32(0.5 / w)).astype(f32)
        a = np.empty((h, w, len(specs), 4), f32)
        a[..., 0] = yc[:, None, None]
        a[..., 1] = xc[None, :, None]
        a[..., 2] = heights
        a[..., 3] = widths
        out.append(a.reshape(-1, 4))
    return np.concatenate(out).astype(f32)


def quicknet_ssd(batch=1, seed=0, image=224, input_type="float32", classes=20, postprocess=True,
                 use_regular_nms=False):
    """A binary SSDLite detector: QuickNet's encoder, then on its 28x28x128, 14x14x256 and 7x7x512
    maps (at 224) a head of A = 3, 6 and 6 anchors per cell: DEPTHWISE_CONV_2D 3x3 (BatchNorm folded,
    RELU) -> CONV_2D 1x1 to A * 4 box encodings and another to A * (classes + 1) class logits, each
    RESHAPEd to [B, h * w * A, 4 | classes + 1]. The maps are joined by CONCATENATION on axis 1, the
    logits go through LOGISTIC, and TFLite_Detection_PostProcess (the TF OD API's export defaults:
    100 detections, 1 class each, 100 per class, score threshold 1e-8, IoU threshold 0.6, scales
    10, 10, 5, 5) turns them into the outputs [boxes [B, 100, 4], classes, scores [B, 100],
    num_detections [B]], with the anchors of ssd_anchors(). postprocess=False leaves the op out: the
    outputs are then the box encodings [B, N, 4] and the class scores [B, N, classes + 1]."""
    if image % 32:
        raise ValueError(f"quicknet_ssd needs an image size that is a multiple of 32, not {image}")
    g = _Builder(seed, batch, "QuickNetSSD")
    sections = _quicknet_encoder(g, batch, image, input_type, (4, 4, 4, 4), (64, 128, 256, 512))
    boxes, logits, grids = [], [], []
    for (x, xs), a in zip(sections[1:], (3, 6, 6)):
        b, h, w, _ = xs
        t, ts = g.depthwise(x, xs, 3, 1, bn=True, activation="RELU")
        for width, maps in ((4, boxes), (classes + 1, logits)):
            y, _ = g.conv(t, ts, a * width, 1, 1)
            r = g.act((b, h * w * a, width))
            g.m.add_op("RESHAPE", [y], [r], new_shape=[-1, h * w * a, width])
            maps.append(r)
        grids.append((h, w))
    anchors = ssd_anchors(grids)
    n = anchors.shape[0]
    enc = g.act((batch, n, 4))
    g.m.add_op("CONCATENATION", boxes, [enc], axis=1)
    cat = g.act((batch, n, classes + 1))
    g.m.add_op("CONCATENATION", logits, [cat], axis=1)
    scores = g.act((batch, n, classes + 1))
    g.m.add_op("LOGISTIC", [cat], [scores])
    if not postprocess:
        g.m.outputs = [enc, scores]
        return g.m.serialize()
    outs = [g.act((batch, 100, 4)), g.act((batch, 100)), g.act((batch, 100)), g.act((batch,))]
    g.m.add_op("TFLite_Detection_PostProcess", [enc, scores, g.const(anchors, name="anchors")], outs,
               custom_options=detection_postprocess_options(num_classes=classes, use_regular_nms=use_regular_nms))
    g.m.outputs = outs
    return g.m.serialize()


def quicknet_large(batch=1, seed=0, image=224, input_type="float32"):
    return quicknet(batch, blocks=(6, 8, 12, 6), seed=seed, image=image, name="QuickNetLarge",
                    input_type=input_type)


def quicknet_small(batch=1, seed=0, image=224, input_type="float32"):
    """QuickNetSmall, restated from larq-zoo (sota/quicknet.py, QuickNetSmallFactory): QuickNet
    with section filters (32, 64, 256, 512) and four blocks per section, so the stem is CONV_2D
    3x3/s2 3 -> 8 (filters[0] // 4) -> DEPTHWISE 3x3/s2 -> CONV_2D 1x1 8 -> 32. 16 LceBconv2d."""
    return quicknet(batch, filters=(32, 64, 256, 512), seed=seed, image=image, name="QuickNetSmall",
                    input_type=input_type)


def birealnet18(batch=1, seed=0, image=224, input_type="float32"):
    g = _Builder(seed, batch, "BiRealNet18")
    xs = (batch, image, image, 3)
    x = g.image_input(xs, input_type)
    x, xs = g.conv(x, xs, 64, 7, 2)
    x, xs = g.pool("MAX_POOL_2D", x, xs, 3, 2, "SAME")
    cin = 64
    for stage, f in enumerate((64, 128, 256, 512)):
        for blk in range(4):
            stride = 2 if (stage > 0 and blk == 0) else 1
            q = g.quantize(x, xs)
            y, ys = g.bconv(q, xs, f, stride=stride, pad_values=0, activation="NONE")
            if stride == 2 or cin != f:
                s, ss = g.pool("AVERAGE_POOL_2D", x, xs, 2, 2, "VALID")
                s, ss = g.conv(s, ss, f, 1, 1)
            else:
                s = x
            x, xs = g.add(y, s, ys), ys
            cin = f
    probs = g.head(x, xs, relu=False)
    g.m.outputs = [probs]
    return g.m.serialize()


def reactnet_a(batch=1, seed=0, image=224, input_type="float32"):
    """ReActNet-A, restated from the public description (Liu et al., ECCV 2020): MobileNet-V1
    shaped. Stem CONV_2D 3x3/s2 3 -> 32 (BN folded, no activation), then 13 blocks with output
    widths [64, 128, 128, 256, 256, 512 x 6, 1024, 1024], stride 2 where the width changes (not
    32 -> 64). Each block, in the converter's op order:
      RSign [ADD(shift) -> LceQuantize] -> LceBconv2d 3x3 C -> C (pad_values 1, BN folded, no
      activation) -> ADD(shortcut; AVERAGE_POOL_2D 2x2/s2 VALID of x at stride 2) -> RPReLU
      [ADD(shift) -> PRELU(alpha [1,1,C]) -> ADD(shift)] = out1 -> RSign -> 1x1 LceBconv2d C -> C
      -> ADD(out1) (width doubling: two such 1x1 convolutions on the same signs, each + out1,
      then CONCATENATION on channels) -> RPReLU.
    Head MEAN -> FULLY_CONNECTED 1000 -> SOFTMAX. 31 LceBconv2d, 26 PRELU."""
    def conv3x3(g, q, xs, c, stride):
        return g.bconv(q, xs, c, stride=stride, pad_values=1, activation="NONE")
    return _reactnet_backbone(batch, seed, image, input_type, "ReActNetA", conv3x3)


def _reactnet_backbone(batch, seed, image, input_type, name, conv3x3):
    """ReActNet-A's graph (see reactnet_a) with each block's 3x3 binary convolution written by
    conv3x3(g, signs, xs, C, stride) -> (y, ys)."""
    g = _Builder(seed, batch, name)
    xs = (batch, image, image, 3)
    x = g.image_input(xs, input_type)
    x, xs = g.conv(x, xs, 32, 3, 2)

    def shift(t, ts):
        return g.add(t, g.const(g.rng.uniform(-0.2, 0.2, ts[3]).astype(np.float32), name="shift"), ts)

    def rsign(t, ts):
        return g.quantize(shift(t, ts), ts)

    def rprelu(t, ts):
        u = g.act(ts)
        alpha = g.const(g.rng.uniform(0.05, 0.5, (1, 1, ts[3])).astype(np.float32), name="alpha")
        g.m.add_op("PRELU", [shift(t, ts), alpha], [u])
        return shift(u, ts)

    widths = [32, 64, 128, 128, 256, 256] + [512] * 6 + [1024, 1024]
    for cin, cout in zip(widths[:-1], widths[1:]):
        stride = 2 if cout != cin and cin != 32 else 1
        # the shortcut first: the convolution's epilogue can then add it (Graph::FuseResidualBlocks)
        sc = x if stride == 1 else g.pool("AVERAGE_POOL_2D", x, xs, 2, 2, "VALID")[0]
        y, ys = conv3x3(g, rsign(x, xs), xs, cin, stride)
        out1 = rprelu(g.add(y, sc, ys), ys)
        q = rsign(out1, ys)
        halves = []
        for _ in range(cout // cin):
            z, _ = g.bconv(q, ys, cin, k=1, pad_values=1, activation="NONE")
            halves.append(g.add(z, out1, ys))
        xs = ys[:3] + (cout,)
        if len(halves) == 1:
            z = halves[0]
        else:
            z = g.act(xs)
            g.m.add_op("CONCATENATION", halves, [z], axis=3)
        x = rprelu(z, xs)
    probs = g.head(x, xs, relu=False)
    g.m.outputs = [probs]
    return g.m.serialize()


def binary_mobilenet(batch=1, seed=0, image=224, input_type="float32", group_channels=32,
                     group_conv="native"):
    """A binary MobileNet in the manner of Phan et al. ("Binarizing MobileNet via Evolution-based
    Searching", CVPR 2020): grouped binary convolutions in place of the depthwise ones. The paper's
    searched per-layer group counts are not available offline, so the topology is restated with a
    fixed group width on ReActNet-A's MobileNet-V1 backbone and converter op order (reactnet_a):
    each block's 3x3 LceBconv2d C -> C runs in C / group_channels groups (the first block's
    32-channel layer, with group_channels = 32, stays one group); the 1x1 halves, shortcuts, RSign
    and RPReLU are ReActNet-A's.
    group_conv="native": each grouped layer is one grouped LceBconv2d (filter [C, 3, 3,
    group_channels / 32 words], channels_in C). group_conv="split": SPLIT of the packed signs on
    axis 3 into the groups' words, one ungrouped LceBconv2d per group, CONCATENATION on channels:
    the same weights, drawn in the same order, and bit for bit the same result."""
    if group_conv not in ("split", "native"):
        raise ValueError(f"group_conv must be 'split' or 'native', not {group_conv!r}")
    if group_channels < 32 or group_channels % 32:
        raise ValueError(f"group_channels must be a positive multiple of 32, not {group_channels}")

    def conv3x3(g, q, xs, c, stride):
        groups = max(c // group_channels, 1)
        if group_conv == "native" or groups == 1:
            return g.bconv(q, xs, c, stride=stride, pad_values=1, activation="NONE", groups=groups)
        b, h, w, _ = xs
        cg = c // groups
        axis = g.const(np.array(3, np.int32), np.int32, "axis")
        parts = [g.act((b, h, w, cg // 32), np.int32) for _ in range(groups)]
        g.m.add_op("SPLIT", [axis, q], parts, num_splits=groups)
        ys = [g.bconv(p, (b, h, w, cg), cg, stride=stride, pad_values=1, activation="NONE") for p in parts]
        out_s = ys[0][1][:3] + (c,)
        z = g.act(out_s)
        g.m.add_op("CONCATENATION", [y for y, _ in ys], [z], axis=3)
        return z, out_s

    name = "BinaryMobileNet" if group_conv == "native" else "BinaryMobileNetSplit"
    return _reactnet_backbone(batch, seed, image, input_type, name, conv3x3)


def realtobinarynet(batch=1, seed=0, image=224, input_type="float32", pad_values=0):
    """Real-to-Binary Net, restated from the paper (Martinez et al., ICLR 2020): ResNet-18 with
    Bi-Real's one shortcut per binary convolution, 4 stages x 4 blocks at 64 / 128 / 256 / 512
    channels (16 LceBconv2d), each binary convolution's output scaled by a gate computed from the
    block's real-valued input. In the converter's op order:
      stem CONV_2D 7x7/s2 3 -> 64 (BN folded) -> PRELU -> MAX_POOL_2D 3x3/s2 SAME;
      block x [B,H,W,Cin] -> [B,H',W',Cout] (stride 2 and Cout = 2 Cin on the first block of
      stages 2-4): the shortcut first (x, or AVERAGE_POOL_2D 2x2/s2 VALID -> CONV_2D 1x1, BN
      folded); the gate MEAN(x, [1, 2]) -> FULLY_CONNECTED Cin -> Cin/8 (RELU, no bias) ->
      FULLY_CONNECTED Cin/8 -> Cout (no bias) -> LOGISTIC -> RESHAPE [-1, 1, 1, Cout]; the main
      path MUL(x, bn_scale) -> ADD(bn_shift) -> LceQuantize -> LceBconv2d 3x3 (stride s,
      `pad_values`, no fused activation) -> MUL(gate) -> PRELU(alpha [1, 1, Cout]) -> ADD(shortcut);
      head PRELU -> MEAN -> FULLY_CONNECTED 1000 -> SOFTMAX.
    The BatchNorm after each binary convolution is folded into its post_activation multiplier and
    bias, before the gate: a simplification of the paper's block, which changes nothing measured
    with synthetic weights. The RESHAPE's -1 batch dimension keeps the graph resizable."""
    g = _Builder(seed, batch, "RealToBinaryNet")
    xs = (batch, image, image, 3)
    x = g.image_input(xs, input_type)

    def prelu(t, ts):
        u = g.act(ts)
        alpha = g.const(g.rng.uniform(0.05, 0.5, (1, 1, ts[3])).astype(np.float32), name="alpha")
        g.m.add_op("PRELU", [t, alpha], [u])
        return u

    def dense(t, cin, cout, activation="NONE"):
        wt = g.rng.standard_normal((cout, cin)).astype(np.float32) / np.float32(np.sqrt(cin))
        y = g.act((batch, cout))
        g.m.add_op("FULLY_CONNECTED", [t, g.const(wt), -1], [y], activation=activation)
        return y

    def gate(t, ts, cout):
        axes = g.const(np.array([1, 2], np.int32), np.int32, "axes")
        pooled = g.act((batch, ts[3]))
        g.m.add_op("MEAN", [t, axes], [pooled], keep_dims=False)
        z = dense(dense(pooled, ts[3], ts[3] // 8, "RELU"), ts[3] // 8, cout)
        s = g.act((batch, cout))
        g.m.add_op("LOGISTIC", [z], [s])
        r = g.act((batch, 1, 1, cout))
        g.m.add_op("RESHAPE", [s], [r], new_shape=[-1, 1, 1, cout])
        return r

    x, xs = g.conv(x, xs, 64, 7, 2)
    x = prelu(x, xs)
    x, xs = g.pool("MAX_POOL_2D", x, xs, 3, 2, "SAME")
    for stage, cout in enumerate((64, 128, 256, 512)):
        for blk in range(4):
            stride = 2 if (stage > 0 and blk == 0) else 1
            if stride == 2:
                s, ss = g.pool("AVERAGE_POOL_2D", x, xs, 2, 2, "VALID")
                s, _ = g.conv(s, ss, cout, 1, 1)
            else:
                s = x
            gt = gate(x, xs, cout)
            scale, shift = g.bn(xs[3])
            t = g.act(xs)
            g.m.add_op("MUL", [x, g.const(scale, name="bn_scale")], [t])
            t = g.add(t, g.const(shift, name="bn_shift"), xs)
            y, ys = g.bconv(g.quantize(t, xs), xs, cout, stride=stride, pad_values=pad_values,
                            activation="NONE")
            u = g.act(ys)
            g.m.add_op("MUL", [y, gt], [u])
            x, xs = g.add(prelu(u, ys), s, ys), ys
    probs = g.head(prelu(x, xs), xs, relu=False)
    g.m.outputs = [probs]
    return g.m.serialize()


def xnornetpp(batch=1, seed=0, image=224, input_type="float32", pad_values=0):
    """XNOR-Net++, restated from the paper (Bulat & Tzimiropoulos, BMVC 2019) on the ResNet-18
    backbone of birealnet18, with synthetic weights, in the converter's op order:
      stem CONV_2D 7x7/s2 3 -> 64 (BN folded, RELU) -> MAX_POOL_2D 3x3/s2 SAME;
      4 stages x 4 blocks at 64 / 128 / 256 / 512 channels, stride 2 and Cout = 2 Cin on the first
      block of stages 2-4; each block on x [B,H,W,Cin], in XNOR order: the shortcut first (x, or
      AVERAGE_POOL_2D 2x2/s2 VALID -> CONV_2D 1x1, BN folded); MUL(x, bn_scale) -> ADD(bn_shift) ->
      LceQuantize -> LceBconv2d 3x3 SAME (stride s, `pad_values`, no fused activation, float output,
      post_activation multiplier 1 and bias 0: nothing is folded into it) -> MUL(Gamma) ->
      ADD(shortcut);
      head MEAN -> FULLY_CONNECTED 1000 -> SOFTMAX, as in birealnet18.
    Gamma is the paper's learned output scale in its factorised form alpha[C] x beta[OH] x gamma[OW],
    all positive, alpha scaled by 1 / K (K = 9 Cin, so Gamma also normalises the accumulator), folded
    into one constant [1, OH, OW, Cout] as the converter leaves it. 16 LceBconv2d, 16 Gamma MULs."""
    g = _Builder(seed, batch, "XNORNetPP")
    xs = (batch, image, image, 3)
    x = g.image_input(xs, input_type)
    x, xs = g.conv(x, xs, 64, 7, 2, activation="RELU")
    x, xs = g.pool("MAX_POOL_2D", x, xs, 3, 2, "SAME")
    for stage, cout in enumerate((64, 128, 256, 512)):
        for blk in range(4):
            stride = 2 if (stage > 0 and blk == 0) else 1
            if stride == 2:
                s, ss = g.pool("AVERAGE_POOL_2D", x, xs, 2, 2, "VALID")
                s, _ = g.conv(s, ss, cout, 1, 1)
            else:
                s = x
            t = g.batchnorm(x, xs)
            y, ys = g.bconv(g.quantize(t, xs), xs, cout, stride=stride, pad_values=pad_values,
                            activation="NONE", fold_bn=False)
            _, oh, ow, _ = ys
            alpha = g.rng.uniform(0.5, 1.5, cout).astype(np.float32) / np.float32(9 * xs[3])
            beta = g.rng.uniform(0.5, 1.5, oh).astype(np.float32)
            gamma = g.rng.uniform(0.5, 1.5, ow).astype(np.float32)
            scale = (beta[:, None, None] * gamma[None, :, None] * alpha[None, None, :]).astype(np.float32)
            u = g.act(ys)
            g.m.add_op("MUL", [y, g.const(scale.reshape(1, oh, ow, cout), name="gamma")], [u])
            x, xs = g.add(u, s, ys), ys
    probs = g.head(x, xs, relu=False)
    g.m.outputs = [probs]
    return g.m.serialize()


def abcnet(batch=1, seed=0, image=224, input_type="float32", bases=(3, 3), pad_values=1):
    """ABC-Net (Lin et al., NeurIPS 2017), restated from the paper on the ResNet-18 backbone with
    synthetic weights, in the converter's op order; bases = (M, N) weight bases and shifted
    activation signs.
      ABC(x, C_out, k, stride): for n = 0..N-1, s_n = ADD(x, u_n) with u_n a one-element float
      constant (the paper's v_n - 0.5, spread around 0) -> q_n = LceQuantize(s_n); then, n outer and
      m inner, t_nm = LceBconv2d(q_n, B_m) k x k SAME (stride, `pad_values`, float output, no fused
      activation, post_activation_multiplier gamma_nm [C_out] = the synthetic alpha_m * beta_n,
      post_activation_bias 0), the M filters B_m shared by every n; y = ADD(...ADD(ADD(t_00, t_01),
      t_02)..., t_{N-1,M-1}), left to right in that order.
      stem CONV_2D 7x7/s2 3 -> 64 (BN folded, RELU) -> MAX_POOL_2D 3x3/s2 SAME;
      4 stages x 2 basic blocks at 64 / 128 / 256 / 512 channels, stride 2 on the first block of
      stages 2-4; a block on x: the shortcut first (x, or CONV_2D 1x1 with the block's stride, BN
      folded); h = ADD(MUL(ABC(x, f, 3, s), bn_scale), bn_shift, RELU);
      z = ADD(MUL(ABC(h, f, 3, 1), bn_scale'), bn_shift'); out = ADD(z, shortcut, RELU);
      head MEAN -> FULLY_CONNECTED 1000 -> SOFTMAX.
    16 ABC layers, 16 * M * N LceBconv2d. Not in MODELS."""
    m_bases, n_planes = bases
    g = _Builder(seed, batch, "ABCNet")
    xs = (batch, image, image, 3)
    x = g.image_input(xs, input_type)
    x, xs = g.conv(x, xs, 64, 7, 2, activation="RELU")
    x, xs = g.pool("MAX_POOL_2D", x, xs, 3, 2, "SAME")
    shifts = [0.0] if n_planes == 1 else list(np.linspace(-0.6, 0.6, n_planes))

    def abc(t, ts, cout, k, stride):
        b, h, w, cin = ts
        qs = [g.quantize(g.add(t, g.const(np.array(u, np.float32), name="shift"), ts), ts) for u in shifts]
        filts = []
        for _ in range(m_bases):
            signs = g.rng.integers(0, 2, (cout, k, k, cin), dtype=np.int8) * 2 - 1
            bits = (signs < 0).astype(np.uint32).reshape(cout, k, k, cin // 32, 32)
            filt = (bits << np.arange(32, dtype=np.uint32)).sum(-1, dtype=np.uint64).astype(np.uint32).view(np.int32)
            filts.append(g.const(filt, np.int32, "bfilter"))
        alpha = [g.rng.uniform(0.5, 1.5, cout).astype(np.float32) * np.float32(4.0 / (k * k * cin))
                 for _ in range(m_bases)]
        beta = g.rng.uniform(0.5, 1.5, n_planes).astype(np.float32)
        oh, ow = -(-h // stride), -(-w // stride)
        ys = (b, oh, ow, cout)
        opts = bconv2d_options(cin, (stride, stride), (1, 1), 0, pad_values, 0)
        y = None
        for n in range(n_planes):
            for m in range(m_bases):
                t_nm = g.act(ys)
                g.m.add_op("LceBconv2d", [qs[n], filts[m], g.const((alpha[m] * beta[n]).astype(np.float32), name="pmul"),
                                          g.const(np.zeros(cout, np.float32), name="pbias"), -1], [t_nm],
                           custom_options=opts)
                y = t_nm if y is None else g.add(y, t_nm, ys)
        return y, ys

    for stage, f in enumerate((64, 128, 256, 512)):
        for blk in range(2):
            stride = 2 if (stage > 0 and blk == 0) else 1
            s = g.conv(x, xs, f, 1, stride)[0] if stride == 2 or xs[3] != f else x
            y, ys = abc(x, xs, f, 3, stride)
            h = g.batchnorm(y, ys, "RELU")
            z = g.batchnorm(abc(h, ys, f, 3, 1)[0], ys)
            x, xs = g.add(z, s, ys, "RELU"), ys
    probs = g.head(x, xs, relu=False)
    g.m.outputs = [probs]
    return g.m.serialize()


def binarydensenet(batch=1, seed=0, image=224, input_type="float32", pad_values=0,
                   layers=(6, 6, 6, 5), reduction=(2.7, 2.7, 2.2), dilation=(1, 1, 1, 1),
                   name="BinaryDenseNet28"):
    """BinaryDenseNet, restated from the paper (Bethge et al., 2019) with the block parameters of
    its 28 / 37 / 37-Dilated / 45 variants. In the converter's op order:
      stem CONV_2D 7x7/s2 3 -> 64 (BN folded, RELU) -> MAX_POOL_2D 3x3/s2 SAME;
      dense layer x_j [B,H,W,C_j] -> MUL(bn_scale) -> ADD(bn_shift) -> LceQuantize -> LceBconv2d
      3x3 (C_j -> 64, stride 1, SAME, `pad_values`, the block's dilation, no activation) = y_j,
      x_{j+1} = CONCATENATION([x_j, y_j], axis 3);
      transition MUL -> ADD (BN) -> MAX_POOL_2D 2x2/s2 VALID (not before a dilated block) -> RELU
      -> CONV_2D 1x1 to round(C // reduction / 32) * 32 channels, no bias;
      head MUL -> ADD (BN) -> RELU -> MEAN -> FULLY_CONNECTED 1000 -> SOFTMAX."""
    g = _Builder(seed, batch, name)
    xs = (batch, image, image, 3)
    x = g.image_input(xs, input_type)
    batchnorm = g.batchnorm
    x, xs = g.conv(x, xs, 64, 7, 2, activation="RELU")
    x, xs = g.pool("MAX_POOL_2D", x, xs, 3, 2, "SAME")
    for blk, n in enumerate(layers):
        if blk > 0:
            cout = int(round(xs[3] // reduction[blk - 1] / 32)) * 32
            x = batchnorm(x, xs)
            if dilation[blk] == 1:
                x, xs = g.pool("MAX_POOL_2D", x, xs, 2, 2, "VALID")
            x = g.relu(x, xs)
            x, xs = g.conv(x, xs, cout, 1, 1, bn=False, use_bias=False)
        for _ in range(n):
            t = batchnorm(x, xs)
            y, _ = g.bconv(g.quantize(t, xs), xs, 64, pad_values=pad_values, activation="NONE",
                           dilation=dilation[blk])
            xs = xs[:3] + (xs[3] + 64,)
            z = g.act(xs)
            g.m.add_op("CONCATENATION", [x, y], [z], axis=3)
            x = z
    probs = g.head(batchnorm(x, xs), xs)
    g.m.outputs = [probs]
    return g.m.serialize()


def binarydensenet28(batch=1, seed=0, image=224, input_type="float32", pad_values=0):
    return binarydensenet(batch, seed, image, input_type, pad_values)


def binarydensenet37(batch=1, seed=0, image=224, input_type="float32", pad_values=0):
    return binarydensenet(batch, seed, image, input_type, pad_values, layers=(6, 8, 12, 6),
                          reduction=(3.3, 3.3, 4), name="BinaryDenseNet37")


def binarydensenet37_dilated(batch=1, seed=0, image=224, input_type="float32", pad_values=0):
    return binarydensenet(batch, seed, image, input_type, pad_values, layers=(6, 8, 12, 6),
                          reduction=(3.3, 3.3, 4), dilation=(1, 1, 2, 4),
                          name="BinaryDenseNet37Dilated")


def binarydensenet45(batch=1, seed=0, image=224, input_type="float32", pad_values=0):
    return binarydensenet(batch, seed, image, input_type, pad_values, layers=(6, 12, 14, 8),
                          reduction=(2.7, 3.3, 4), name="BinaryDenseNet45")


def meliusnet(batch=1, seed=0, image=224, input_type="float32", pad_values=0, blocks=(4, 5, 4, 6),
              transitions=(160, 224, 256), name="MeliusNet22", group_conv="split"):
    """MeliusNet, restated from the paper (Bethge et al., 2020) and larq-zoo's MeliusNet22 with
    synthetic weights, in the converter's op order:
      stem CONV_2D 3x3/s2 3 -> 32 (BN folded, RELU); a grouped convolution 32 -> 32 in 4 groups,
      built as larq-zoo's group_conv builds it (tf.split -> one Conv2D per group -> concat):
      SPLIT(axis 3, 4) -> 4x CONV_2D 3x3 SAME 8 -> 8 (no bias) -> CONCATENATION -> MUL -> ADD(RELU),
      the BatchNorm and activation after the concatenation; the same 32 -> 64 in 8 groups (8x
      CONV_2D 4 -> 8); MAX_POOL_2D 3x3/s2 SAME;
      with group_conv="native" each of the two grouped convolutions is instead one grouped CONV_2D
      (filter [32, 3, 3, 8] and [64, 3, 3, 4], what Keras Conv2D(groups=g) converts to), then the same
      MUL -> ADD(RELU): its filter is the split form's per-group filters, drawn in the same order and
      concatenated along the output channels, and every other tensor is the split form's, so both
      forms compute the same function (the default "split" model's bytes are unchanged);
      sections of `blocks` MeliusBlocks (64 -> 320, 160 -> 480, 224 -> 480, 256 -> 640 channels
      at the default), each a dense layer and then an improvement layer on the map x [B,H,W,C]:
        dense layer MUL(bn_scale) -> ADD(bn_shift) -> LceQuantize -> LceBconv2d 3x3 C -> 64
        (`pad_values`, no activation) = y, CONCATENATION([x, y], axis 3), as BinaryDenseNet's;
        improvement layer MUL -> ADD -> LceQuantize, then a = STRIDED_SLICE(x)[..., :C-64] and
        b = STRIDED_SLICE(x)[..., C-64:] (constant int32 begin / end / strides, begin_mask and
        end_mask on the whole axes, the channel bound -64), then LceBconv2d 3x3 C -> 64 = y,
        ADD(b, y) and CONCATENATION([a, ADD], axis 3): y is added to the map's last 64 channels;
      transition after every section but the last: MUL -> ADD (BN) -> MAX_POOL_2D 2x2/s2 VALID ->
      RELU -> CONV_2D 1x1 to `transitions[i]` channels, no bias;
      head MUL -> ADD (BN) -> RELU -> MEAN -> FULLY_CONNECTED 1000 -> SOFTMAX.
    Simplifications: larq-zoo's transition convolutions are grouped; these are ungrouped. The
    slices come before the binary convolution, an order the converter may emit. 38 LceBconv2d,
    38 STRIDED_SLICE, 2 SPLIT, 16 CONV_2D and 40 CONCATENATION at the default; with
    group_conv="native" no SPLIT, 6 CONV_2D and 38 CONCATENATION."""
    if group_conv not in ("split", "native"):
        raise ValueError(f"group_conv must be 'split' or 'native', not {group_conv!r}")
    native = group_conv == "native"
    g = _Builder(seed, batch, name)
    xs = (batch, image, image, 3)
    x = g.image_input(xs, input_type)

    def group_conv(t, ts, cout, groups):
        if native:
            cin = ts[3] // groups
            # the split form's g.conv draws, group by group, concatenated along O
            wt = np.concatenate([g.rng.standard_normal((cout // groups, 3, 3, cin)).astype(np.float32) *
                                 np.float32(1.0 / np.sqrt(9 * cin)) for _ in range(groups)])
            y = g.act(ts[:3] + (cout,))
            g.m.add_op("CONV_2D", [t, g.const(wt), -1], [y], padding="SAME", stride=(1, 1), activation="NONE")
            ts = ts[:3] + (cout,)
            return g.batchnorm(y, ts, "RELU"), ts
        axis = g.const(np.array(3, np.int32), np.int32, "axis")
        parts = [g.act(ts[:3] + (ts[3] // groups,)) for _ in range(groups)]
        g.m.add_op("SPLIT", [axis, t], parts, num_splits=groups)
        ys = [g.conv(p, ts[:3] + (ts[3] // groups,), cout // groups, 3, 1, bn=False, use_bias=False)[0]
              for p in parts]
        ts = ts[:3] + (cout,)
        z = g.act(ts)
        g.m.add_op("CONCATENATION", ys, [z], axis=3)
        return g.batchnorm(z, ts, "RELU"), ts

    def last_channels(t, ts, first):
        """t[..., :C-64] (first) or t[..., C-64:]: the channel bound is -64, begin_mask /
        end_mask cover the whole axes."""
        out = g.act(ts[:3] + (ts[3] - 64 if first else 64,))
        vec = lambda v: g.const(np.array(v, np.int32), np.int32, "ss")
        lo, hi = (0, -64) if first else (-64, 0)
        g.m.add_op("STRIDED_SLICE", [t, vec([0, 0, 0, lo]), vec([0, 0, 0, hi]), vec([1, 1, 1, 1])], [out],
                   begin_mask=0b1111 if first else 0b0111, end_mask=0b0111 if first else 0b1111)
        return out

    x, xs = g.conv(x, xs, 32, 3, 2, activation="RELU")
    x, xs = group_conv(x, xs, 32, 4)
    x, xs = group_conv(x, xs, 64, 8)
    x, xs = g.pool("MAX_POOL_2D", x, xs, 3, 2, "SAME")
    for sec, n in enumerate(blocks):
        if sec > 0:
            x = g.batchnorm(x, xs)
            x, xs = g.pool("MAX_POOL_2D", x, xs, 2, 2, "VALID")
            x = g.relu(x, xs)
            x, xs = g.conv(x, xs, transitions[sec - 1], 1, 1, bn=False, use_bias=False)
        for _ in range(n):
            # dense layer
            y, _ = g.bconv(g.quantize(g.batchnorm(x, xs), xs), xs, 64, pad_values=pad_values,
                           activation="NONE")
            xs = xs[:3] + (xs[3] + 64,)
            z = g.act(xs)
            g.m.add_op("CONCATENATION", [x, y], [z], axis=3)
            x = z
            # improvement layer, the slices before the convolution
            q = g.quantize(g.batchnorm(x, xs), xs)
            a, b = last_channels(x, xs, True), last_channels(x, xs, False)
            y, _ = g.bconv(q, xs, 64, pad_values=pad_values, activation="NONE")
            s = g.add(b, y, xs[:3] + (64,))
            z = g.act(xs)
            g.m.add_op("CONCATENATION", [a, s], [z], axis=3)
            x = z
    probs = g.head(g.batchnorm(x, xs), xs)
    g.m.outputs = [probs]
    return g.m.serialize()


def meliusnet22(batch=1, seed=0, image=224, input_type="float32", pad_values=0):
    return meliusnet(batch, seed, image, input_type, pad_values)


def _alexnet(g, x, xs, widths, pad_values, flatten=False):
    """The binary trunk BinaryAlexNet and XNOR-Net share, after the stem's map x: pooled sign ->
    LceBconv2d 5x5 (float) -> pooled sign -> two LceBconv2d 3x3 with bitpacked output -> LceBconv2d
    3x3 (float) -> pooled sign -> LceBconv2d VALID over the whole pooled map (bitpacked). A pooled
    sign is MAX_POOL_2D 3x3/s2 VALID -> MUL(bn_scale) -> ADD(bn_shift) -> LceQuantize. Returns the
    packed signs of the last layer and their shape.
    flatten (widths without the last): the trunk ends at the last pooled BatchNorm, flattened as larq's
    Flatten converts, ADD -> RESHAPE [-1, OH * OW * C]; returns that float map and its width."""
    def pooled_sign(t, ts):
        t, ts = g.pool("MAX_POOL_2D", t, ts, 3, 2, "VALID")
        return g.quantize(g.batchnorm(t, ts), ts), ts

    c2, c3, c4, c5 = widths[:4]
    q, qs = pooled_sign(x, xs)
    y, ys = g.bconv(q, qs, c2, k=5, pad_values=pad_values, activation="NONE")
    q, qs = pooled_sign(y, ys)
    q, qs = g.bconv(q, qs, c3, pad_values=pad_values, activation="NONE", bitpacked=True)
    q, qs = g.bconv(q, qs, c4, pad_values=pad_values, activation="NONE", bitpacked=True)
    y, ys = g.bconv(q, qs, c5, pad_values=pad_values, activation="NONE")
    if flatten:
        y, ys = g.pool("MAX_POOL_2D", y, ys, 3, 2, "VALID")
        y = g.batchnorm(y, ys)
        k = ys[1] * ys[2] * ys[3]
        flat = g.act((ys[0], k))
        g.m.add_op("RESHAPE", [y], [flat], new_shape=[-1, k])
        return flat, k
    q, qs = pooled_sign(y, ys)
    return g.bconv(q, qs, widths[4], k=qs[1], pad_values=pad_values, activation="NONE", padding="VALID",
                   bitpacked=True)


def _binary_dense(g, x, k, n, alpha=None, bias=None, activation="NONE"):
    """larq's QuantDense(ste_sign, ste_sign) on a float [B, k] map as the converter leaves it (LCE has no
    binary dense op): LceQuantize -> LceDequantize -> FULLY_CONNECTED with weights +-alpha_o (alpha None:
    +-1.0, larq's ste_sign kernel) and the bias (None: absent). Returns the [B, n] output."""
    b = g.batch
    q = g.act((b, (k + 31) // 32), np.int32)
    g.m.add_op("LceQuantize", [x], [q], custom_options=b"")
    deq = g.act((b, k))
    g.m.add_op("LceDequantize", [q], [deq], custom_options=b"")
    wt = (g.rng.integers(0, 2, (n, k), dtype=np.int8) * 2 - 1).astype(np.float32)
    if alpha is not None:
        wt = wt * alpha[:, None]
    y = g.act((b, n))
    g.m.add_op("FULLY_CONNECTED", [deq, g.const(wt), -1 if bias is None else g.const(bias, name="b")], [y],
               activation=activation)
    return y


def binaryalexnet(batch=1, seed=0, image=224, input_type="float32", pad_values=0, dense="conv"):
    """BinaryAlexNet, restated from larq-zoo with synthetic weights, in the converter's op order
    (shapes at 224):
      stem CONV_2D 11x11/s4 SAME 3 -> 64 with +-1 float weights (a binary kernel on the float image,
      which the converter leaves a float convolution), no bias, no activation -> [B,56,56,64];
      MAX_POOL_2D 3x3/s2 VALID -> MUL -> ADD (the BatchNorm after the pool) -> LceQuantize;
      LceBconv2d 5x5 SAME 64 -> 192 (float output, `pad_values`, no activation) -> pooled sign
      as above -> 13x13;
      LceBconv2d 3x3 192 -> 384 and 384 -> 384 with bitpacked output (int32 signs, inputs 2 and 3
      absent, input 4 the int32 thresholds [C_out]);
      LceBconv2d 3x3 384 -> 256 (float) -> pooled sign -> 6x6;
      the dense blocks as convolutions: LceBconv2d VALID with a filter covering the pooled map
      (6x6 at 224) 256 -> 4096, bitpacked; 1x1 4096 -> 4096, bitpacked; 1x1 4096 -> 1000, float;
      RESHAPE [-1, 1000] -> SOFTMAX.
    Simplification: larq-zoo flattens the pooled map and applies dense layers; flattening an NHWC
    map and a dense layer over it is exactly a VALID convolution over the whole map, which keeps
    those layers binary. The BatchNorm that follows each binary layer with bitpacked output is
    folded into its thresholds. 7 LceBconv2d (4 bitpacked), 3 pooled signs.
    dense="fully_connected": larq-zoo's head as the converter leaves it instead: the last pooled
    BatchNorm flattened (ADD -> RESHAPE [-1, 9216]), then three times LceQuantize -> LceDequantize ->
    FULLY_CONNECTED (+-1.0 weights, no bias) -> MUL -> ADD (the BatchNorm, not folded), 4096, 4096 and
    1000 wide, then SOFTMAX. 4 LceBconv2d (2 bitpacked), 2 pooled signs and the flattened one."""
    if dense not in ("conv", "fully_connected"):
        raise ValueError(f"binaryalexnet dense must be 'conv' or 'fully_connected', not {dense!r}")
    g = _Builder(seed, batch, "BinaryAlexNet")
    xs = (batch, image, image, 3)
    x = g.image_input(xs, input_type)
    x, xs = g.conv(x, xs, 64, 11, 4, bn=False, use_bias=False, binary=True)
    if dense == "fully_connected":
        x, k = _alexnet(g, x, xs, (192, 384, 384, 256), pad_values, flatten=True)
        for n in (4096, 4096, 1000):
            y = _binary_dense(g, x, k, n)
            x = g.batchnorm(y, (batch, 1, 1, n))
            k = n
        probs = g.act((batch, 1000))
        g.m.add_op("SOFTMAX", [x], [probs], beta=1.0)
        g.m.outputs = [probs]
        return g.m.serialize()
    q, qs = _alexnet(g, x, xs, (192, 384, 384, 256, 4096), pad_values)
    q, qs = g.bconv(q, qs, 4096, k=1, pad_values=pad_values, activation="NONE", padding="VALID",
                    bitpacked=True)
    y, ys = g.bconv(q, qs, 1000, k=1, pad_values=pad_values, activation="NONE", padding="VALID")
    logits = g.act((batch, 1000))
    g.m.add_op("RESHAPE", [y], [logits], new_shape=[-1, 1000])
    probs = g.act((batch, 1000))
    g.m.add_op("SOFTMAX", [logits], [probs], beta=1.0)
    g.m.outputs = [probs]
    return g.m.serialize()


def xnornet(batch=1, seed=0, image=224, input_type="float32", pad_values=0, dense="conv"):
    """XNOR-Net, restated from larq-zoo with synthetic weights, in the converter's op order (shapes
    at 224):
      stem CONV_2D 11x11/s4 SAME 3 -> 96 (BN folded, RELU) -> [B,56,56,96];
      MAX_POOL_2D 3x3/s2 VALID -> MUL -> ADD (BN) -> LceQuantize;
      LceBconv2d 5x5 SAME 96 -> 256 (float output, `pad_values`, no activation) -> pooled sign;
      LceBconv2d 3x3 256 -> 384 and 384 -> 384, bitpacked (int32 thresholds [C_out]);
      LceBconv2d 3x3 384 -> 256 (float) -> pooled sign -> 6x6;
      LceBconv2d 6x6 VALID 256 -> 4096, bitpacked; LceBconv2d 1x1 4096 -> 4096, float with fused
      RELU (BN folded);
      RESHAPE [-1, 4096] -> FULLY_CONNECTED 1000 (BN folded into its weights and bias) -> SOFTMAX.
    The per-channel weight scale of XNOR-Net's binary layers folds into each post-activation
    multiplier, so with synthetic weights it changes nothing. The first dense layer is restated as
    a VALID convolution over the whole pooled map, as in binaryalexnet. 6 LceBconv2d (3
    bitpacked), 3 pooled signs.
    dense="fully_connected": the two 4096-wide layers as the converter leaves larq's QuantDense with
    XNOR-Net's kernel scale instead: the last pooled BatchNorm flattened (ADD -> RESHAPE [-1, 9216]),
    then LceQuantize -> LceDequantize -> FULLY_CONNECTED 9216 -> 4096 and LceQuantize -> LceDequantize
    -> FULLY_CONNECTED 4096 -> 4096 (RELU), each with weights +-alpha_o, alpha_o the row's mean |w|
    times its folded BatchNorm scale (not powers of two), and the folded shift as the bias; then the
    float classifier as above. 4 LceBconv2d (2 bitpacked), 2 pooled signs and the flattened one."""
    if dense not in ("conv", "fully_connected"):
        raise ValueError(f"xnornet dense must be 'conv' or 'fully_connected', not {dense!r}")
    g = _Builder(seed, batch, "XNORNet")
    xs = (batch, image, image, 3)
    x = g.image_input(xs, input_type)
    x, xs = g.conv(x, xs, 96, 11, 4, activation="RELU")
    if dense == "fully_connected":
        x, k = _alexnet(g, x, xs, (256, 384, 384, 256), pad_values, flatten=True)
        for act in ("NONE", "RELU"):
            s, t = g.bn(4096)
            alpha = (g.rng.uniform(0.5, 1.5, 4096).astype(np.float32) * s / np.float32(np.sqrt(k)))
            x = _binary_dense(g, x, k, 4096, alpha=alpha, bias=t, activation=act)
            k = 4096
        flat = x
    else:
        q, qs = _alexnet(g, x, xs, (256, 384, 384, 256, 4096), pad_values)
        y, ys = g.bconv(q, qs, 4096, k=1, pad_values=pad_values, activation="RELU", padding="VALID")
        flat = g.act((batch, 4096))
        g.m.add_op("RESHAPE", [y], [flat], new_shape=[-1, 4096])
    wt = g.rng.standard_normal((1000, 4096)).astype(np.float32) / np.float32(np.sqrt(4096))
    s, t = g.bn(1000)
    logits = g.act((batch, 1000))
    g.m.add_op("FULLY_CONNECTED", [flat, g.const(wt * s[:, None]), g.const(t, name="b")], [logits])
    probs = g.act((batch, 1000))
    g.m.add_op("SOFTMAX", [logits], [probs], beta=1.0)
    g.m.outputs = [probs]
    return g.m.serialize()


def dorefanet(batch=1, seed=0, image=224, input_type="float32"):
    """DoReFaNet (Zhou et al., 2016: 1-bit weights, 2-bit activations), restated from larq-zoo's
    DoReFaNet with synthetic weights; larq-zoo's source is not available offline, so the topology is
    restated from its public description. In the converter's op order (shapes at 224):
      stem CONV_2D 12x12/s4 VALID 3 -> 96 (BN folded into weights and bias, no activation) ->
      [B,54,54,96];
      quantised block Q(C_out, k, pool): the 2-bit activation quantiser round(clip(x, 0, 1) * 3) / 3 as
      MAXIMUM(x, 0) -> MINIMUM(., 1) -> MUL(., 3) -> ROUND -> DIV(., 3) with one-element constants, then
      CONV_2D k x k SAME stride 1 with no fused activation, whose weights are +-alpha_o: the
      magnitude-aware sign's per-channel scale times the folded BatchNorm scale, one float32 value
      per output channel, so |w| is bitwise constant within a channel and the converter cannot emit
      an LceBconv2d (the input is not binary); the bias is the folded BatchNorm shift; then, if
      `pool`, MAX_POOL_2D 3x3/s2;
      Q(256, 5, SAME pool) -> 27x27, Q(384, 3, SAME pool) -> 14x14, Q(384, 3), Q(256, 3, VALID pool)
      -> [B,6,6,256];
      RESHAPE [-1, 9216] -> quantiser -> FULLY_CONNECTED 9216 -> 4096 (+-alpha_o, bias) -> quantiser
      -> FULLY_CONNECTED 4096 -> 4096 (+-alpha_o, bias) -> MAXIMUM(0) -> MINIMUM(1) (a clip, not a
      quantiser) -> FULLY_CONNECTED 4096 -> 1000 with float weights -> SOFTMAX.
    6 quantisers, 5 CONV_2D, 3 FULLY_CONNECTED, 3 MAX_POOL_2D."""
    g = _Builder(seed, batch, "DoReFaNet")
    xs = (batch, image, image, 3)
    x = g.image_input(xs, input_type)

    def scalar_op(kind, t, ts, value):
        y = g.act(ts)
        g.m.add_op(kind, [t, g.const(np.array(value, np.float32), name="q")], [y])
        return y

    def clip(t, ts):
        return scalar_op("MINIMUM", scalar_op("MAXIMUM", t, ts, 0.0), ts, 1.0)

    def quantiser(t, ts):
        t = scalar_op("MUL", clip(t, ts), ts, 3.0)
        r = g.act(ts)
        g.m.add_op("ROUND", [t], [r])
        return scalar_op("DIV", r, ts, 3.0)

    def binary_weights(shape):
        """+-alpha_o of `shape` [C_out, ...], and the bias: pre-activations spread around [0, 1]."""
        fan_in = int(np.prod(shape[1:]))
        s, t = g.bn(shape[0])
        alpha = (g.rng.uniform(0.5, 1.5, shape[0]).astype(np.float32) * s / np.float32(np.sqrt(fan_in)))
        sign = (g.rng.integers(0, 2, shape, dtype=np.int8) * 2 - 1).astype(np.float32)
        return sign * alpha.reshape((-1,) + (1,) * (len(shape) - 1)), t + np.float32(0.5)

    def qconv(t, ts, cout, k, pool):
        b, h, w, cin = ts
        wt, bias = binary_weights((cout, k, k, cin))
        y = g.act((b, h, w, cout))
        g.m.add_op("CONV_2D", [quantiser(t, ts), g.const(wt), g.const(bias, name="b")], [y], padding="SAME",
                   stride=(1, 1), activation="NONE")
        ys = (b, h, w, cout)
        return g.pool("MAX_POOL_2D", y, ys, 3, 2, pool) if pool else (y, ys)

    def qdense(t, cin, cout):
        wt, bias = binary_weights((cout, cin))
        y = g.act((batch, cout))
        g.m.add_op("FULLY_CONNECTED", [quantiser(t, (batch, cin)), g.const(wt), g.const(bias, name="b")], [y])
        return y

    x, xs = g.conv(x, xs, 96, 12, 4, padding="VALID")
    x, xs = qconv(x, xs, 256, 5, "SAME")
    x, xs = qconv(x, xs, 384, 3, "SAME")
    x, xs = qconv(x, xs, 384, 3, None)
    x, xs = qconv(x, xs, 256, 3, "VALID")
    flat_c = xs[1] * xs[2] * xs[3]
    flat = g.act((batch, flat_c))
    g.m.add_op("RESHAPE", [x], [flat], new_shape=[-1, flat_c])
    x = qdense(qdense(flat, flat_c, 4096), 4096, 4096)
    x = clip(x, (batch, 4096))
    wt = g.rng.standard_normal((1000, 4096)).astype(np.float32) / np.float32(np.sqrt(4096))
    logits = g.act((batch, 1000))
    g.m.add_op("FULLY_CONNECTED", [x, g.const(wt), g.const(np.zeros(1000, np.float32), name="b")], [logits])
    probs = g.act((batch, 1000))
    g.m.add_op("SOFTMAX", [logits], [probs], beta=1.0)
    g.m.outputs = [probs]
    return g.m.serialize()


def binary_pointnet(batch=1, seed=0, points=1024, classes=40, widths=(64, 64, 64, 128, 1024), head=(512, 256),
                    alpha=None):
    """BiPointNet (Qin et al., ICLR 2021): vanilla PointNet classification without the T-Nets, its shared
    MLPs binary, with synthetic weights, in the op order the converter leaves larq's layers in:
      input float32 [B, P, 3] (P = `points`);
      stem FULLY_CONNECTED 3 -> widths[0] (float weights, bias, keep_num_dims) -> MUL -> ADD, the BatchNorm
      unfolded, without a RELU: the next layer takes its signs, which after a RELU would all be +1;
      each further width n: LceQuantize -> LceDequantize -> FULLY_CONNECTED(+-alpha weights, no bias,
      keep_num_dims) [B, P, n] -> MUL -> ADD (the BatchNorm), larq's QuantDense on [B, P, C];
      REDUCE_MAX over the points (axis 1) -> [B, widths[-1]], the global max pool (BiPointNet's EMA-max
      offset, here about the expected max of the last layer's dot products over P points, is a constant
      before the max, so it is folded into the last shift);
      the head: for each width in `head` LceQuantize -> LceDequantize -> FULLY_CONNECTED(+-alpha) -> MUL
      -> ADD, then a float FULLY_CONNECTED -> `classes` with bias and SOFTMAX.
    alpha=None: +-1.0 weights. alpha="lsr": each binary layer's weights +-alpha with one scale per layer
    that is not a power of two, BiPointNet's layer-wise scale recovery. Not in MODELS."""
    if alpha not in (None, "lsr"):
        raise ValueError(f"binary_pointnet alpha must be None or 'lsr', not {alpha!r}")
    g = _Builder(seed, batch, "BiPointNet")
    b = batch
    x = g.m.add_tensor("input", (b, points, 3), np.float32)
    g.m.inputs = [x]

    def bn_tail(y, shape, n, activation="NONE", offset=0.0):
        scale, shift = g.bn(n)
        shift = (shift - np.float32(offset) * scale).astype(np.float32)
        u = g.act(shape)
        g.m.add_op("MUL", [y, g.const(scale, name="bn_scale")], [u])
        return g.add(u, g.const(shift, name="bn_shift"), shape, activation)

    def binary_layer(x, lead, k, n, offset=0.0):
        q = g.act(lead + ((k + 31) // 32,), np.int32)
        g.m.add_op("LceQuantize", [x], [q], custom_options=b"")
        deq = g.act(lead + (k,))
        g.m.add_op("LceDequantize", [q], [deq], custom_options=b"")
        wt = (g.rng.integers(0, 2, (n, k), dtype=np.int8) * 2 - 1).astype(np.float32)
        if alpha == "lsr":
            a = np.float32(g.rng.uniform(0.3, 0.9))   # never a power of two
            wt = wt * a
        y = g.act(lead + (n,))
        keep = {"keep_num_dims": True} if len(lead) > 1 else {}
        g.m.add_op("FULLY_CONNECTED", [deq, g.const(wt), -1], [y], activation="NONE", **keep)
        return bn_tail(y, lead + (n,), n, offset=offset * float(np.abs(wt[0, 0])))

    wt = g.rng.standard_normal((widths[0], 3)).astype(np.float32) / np.float32(np.sqrt(3.0))
    y = g.act((b, points, widths[0]))
    g.m.add_op("FULLY_CONNECTED", [x, g.const(wt), g.const(g.rng.uniform(-0.5, 0.5, widths[0]).astype(np.float32),
                                                            name="b")],
               [y], activation="NONE", keep_num_dims=True)
    x = bn_tail(y, (b, points, widths[0]), widths[0])
    # the EMA-max offset: about the expected max over P points of a +-1 dot product of K terms (sd sqrt(K)),
    # so the pooled features' signs depend on the points
    lnp = np.log(max(points, 2))
    e_max = np.sqrt(2 * lnp) - (np.log(lnp) + np.log(4 * np.pi)) / (2 * np.sqrt(2 * lnp))
    for i, (k, n) in enumerate(zip(widths[:-1], widths[1:])):
        last = i == len(widths) - 2
        x = binary_layer(x, (b, points), k, n, offset=np.sqrt(k) * e_max if last and points > 1 else 0.0)
    feat = g.act((b, widths[-1]))
    g.m.add_op("REDUCE_MAX", [x, g.const(np.array([1], np.int32), np.int32, "axes")], [feat], keep_dims=False)
    x, k = feat, widths[-1]
    for n in head:
        x = binary_layer(x, (b,), k, n)
        k = n
    wt = g.rng.standard_normal((classes, k)).astype(np.float32) / np.float32(np.sqrt(k))
    logits = g.act((b, classes))
    g.m.add_op("FULLY_CONNECTED", [x, g.const(wt), g.const(np.zeros(classes, np.float32), name="b")], [logits],
               activation="NONE")
    probs = g.act((b, classes))
    g.m.add_op("SOFTMAX", [logits], [probs], beta=1.0)
    g.m.outputs = [probs]
    return g.m.serialize()


MODELS = {"quicknet": quicknet, "quicknet_large": quicknet_large, "quicknet_small": quicknet_small,
          "birealnet18": birealnet18,
          "reactnet_a": reactnet_a, "realtobinarynet": realtobinarynet,
          "binarydensenet28": binarydensenet28, "binarydensenet37": binarydensenet37,
          "binarydensenet37_dilated": binarydensenet37_dilated,
          "binarydensenet45": binarydensenet45, "meliusnet22": meliusnet22,
          "binaryalexnet": binaryalexnet, "xnornet": xnornet, "dorefanet": dorefanet}
