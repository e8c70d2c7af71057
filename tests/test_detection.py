"""Binary SSD detection graphs: TFLite_Detection_PostProcess (lce_b200_f32_detection_postprocess and the
graph host's custom op), FlexBuffers floats and bools, and the zoo's quicknet_ssd.

CPU: a numpy restatement of TFLite's kernel (detection_postprocess.cc) on hand-built cases with known
answers, the FlexBuffers reader and writer, Prepare's shapes and refusals, the model's node lists, the
other models' bytes, and the kernels' build.
GPU: the op bit for bit against the restatement in both NMS modes, each image of a batch against the
image alone, the whole graph op by op and fused against unfused, arena independence and CUDA-graph
replay, and Interpreter.predict over mini-batches."""
import collections
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import tflite_ref as R
from compute_engine_b200 import host as H
from compute_engine_b200 import tflite_writer as W
from compute_engine_b200 import zoo
from compute_engine_b200.tflite_writer import TFLiteModel

F32 = np.float32
OP = "TFLite_Detection_PostProcess"
DEFAULTS = dict(max_detections=100, max_classes_per_detection=1, detections_per_class=100, num_classes=20,
                use_regular_nms=0, nms_score_threshold=1e-8, nms_iou_threshold=0.6, y_scale=10.0, x_scale=10.0,
                h_scale=5.0, w_scale=5.0)


# ------------------------- numpy restatement of TFLite's kernel ------------------------- #
def decode(enc, anchors, o):
    """DecodeCenterSizeBoxes, every step rounded in float32, exp in float64 rounded once."""
    ys, xs, hs, ws = (F32(o[k]) for k in ("y_scale", "x_scale", "h_scale", "w_scale"))
    y, x, h, w = (np.ascontiguousarray(enc[:, k], F32) for k in range(4))
    ya, xa, ha, wa = (anchors[:, k].astype(F32) for k in range(4))
    with np.errstate(all="ignore"):
        yc = ((y / ys) * ha) + ya
        xc = ((x / xs) * wa) + xa
        hh = (F32(0.5) * np.exp((h / hs).astype(np.float64)).astype(F32)) * ha
        hw = (F32(0.5) * np.exp((w / ws).astype(np.float64)).astype(F32)) * wa
        return np.stack([yc - hh, xc - hw, yc + hh, xc + hw], 1).astype(F32)


def _mx(a, b):   # std::max<float>
    return np.where(a < b, b, a)


def _mn(a, b):   # std::min<float>
    return np.where(b < a, b, a)


def iou(bi, bj):
    """ComputeIntersectionOverUnion of box bi (the selected one) with each row of bj."""
    with np.errstate(all="ignore"):
        ai = (bi[2] - bi[0]) * (bi[3] - bi[1])
        aj = (bj[:, 2] - bj[:, 0]) * (bj[:, 3] - bj[:, 1])
        inter = _mx(_mn(bi[2], bj[:, 2]) - _mx(bi[0], bj[:, 0]), F32(0)) * \
            _mx(_mn(bi[3], bj[:, 3]) - _mx(bi[1], bj[:, 1]), F32(0))
        v = (inter / ((ai + aj) - inter)).astype(F32)
    return np.where((ai <= 0) | (aj <= 0), F32(0), v)


def nms(boxes, scores, o, max_out):
    """NonMaxSuppressionSingleClassHelper: SelectDetectionsAboveScoreThreshold, the stable descending
    sort (ties to the lower anchor, -0 as +0), then greedy suppression at IoU > threshold."""
    keep = np.flatnonzero(scores >= F32(o["nms_score_threshold"]))
    cand = keep[np.argsort(-scores[keep].astype(np.float64), kind="stable")]
    out_size = min(len(cand), max_out)
    active = np.ones(len(cand), bool)
    sel, pos = [], 0
    while len(sel) < out_size:
        nz = np.flatnonzero(active[pos:])
        if not len(nz):
            break
        i = pos + int(nz[0])
        sel.append(int(cand[i]))
        active[i] = False
        rest = np.flatnonzero(active[i + 1:]) + i + 1
        if len(rest):
            active[rest[iou(boxes[cand[i]], boxes[cand[rest]]) > F32(o["nms_iou_threshold"])]] = False
        pos = i + 1
    return sel


def top_classes(cs, k):
    """DecreasingPartialArgSort per anchor: ArgMaxVector for one class (first maximum, a NaN in class 0
    stays), else score descending, class ascending, NaN last."""
    n, c = cs.shape
    if k == 1:
        best, bv = np.zeros(n, np.int64), cs[:, 0].copy()
        for j in range(1, c):
            up = cs[:, j] > bv
            bv = np.where(up, cs[:, j], bv)
            best = np.where(up, j, best)
        return best[:, None]
    out = np.empty((n, k), np.int64)
    idx = np.arange(c)
    for a in range(n):
        v = cs[a].astype(np.float64)
        out[a] = np.lexsort((idx, -np.where(np.isnan(v), 0, v), np.isnan(v)))[:k]
    return out


def postprocess_image(enc, scores, anchors, o):
    """One image: enc [N, K], scores [N, S], anchors [N, 4] -> (boxes [D, 4], classes [D], scores [D], num)."""
    dec = decode(enc, anchors, o)
    c, md, mc = o["num_classes"], o["max_detections"], o["max_classes_per_detection"]
    cs = scores[:, scores.shape[1] - c:].astype(F32)
    d = md * mc
    ob, oc, osc = np.zeros((d, 4), F32), np.zeros(d, F32), np.zeros(d, F32)
    if not o["use_regular_nms"]:
        kc = min(mc, c)
        cls = top_classes(cs, kc)
        sel = nms(dec, cs[np.arange(len(cs)), cls[:, 0]], o, md)
        for r, a in enumerate(sel):
            for col in range(kc):
                ob[mc * r + col] = dec[a]
                oc[mc * r + col] = cls[a, col]
                osc[mc * r + col] = cs[a, cls[a, col]]
        return ob, oc, osc, len(sel)
    entries = []
    for k in range(c):
        entries += [(float(cs[a, k]), k, a) for a in nms(dec, cs[:, k], o, o["detections_per_class"])]
    top = sorted(entries, key=lambda e: -e[0])[:md]   # stable: class order, then each class's order
    for i, (s, k, a) in enumerate(top):
        ob[i], oc[i], osc[i] = dec[a], k, s
    return ob, oc, osc, len(top)


def postprocess_ref(enc, scores, anchors, **kw):
    o = dict(DEFAULTS, **kw)
    per = [postprocess_image(enc[b], scores[b], anchors, o) for b in range(enc.shape[0])]
    return (np.stack([p[0] for p in per]), np.stack([p[1] for p in per]), np.stack([p[2] for p in per]),
            np.array([p[3] for p in per], F32))


# ------------------------------- hand-built cases ------------------------------- #
def _anchors(*rows):
    """Anchors from corner boxes (ymin, xmin, ymax, xmax): zero encodings decode to those boxes."""
    a = np.array(rows, F32).reshape(-1, 4)
    return np.stack([(a[:, 0] + a[:, 2]) / 2, (a[:, 1] + a[:, 3]) / 2, a[:, 2] - a[:, 0], a[:, 3] - a[:, 1]], 1)


def _case(name):
    """(enc [1, N, K], scores [1, N, S], anchors, options) of a hand-built case."""
    unit = (0, 0, 1, 1)
    far = [(3 * i, 3 * i, 3 * i + 1, 3 * i + 1) for i in range(4)]
    kw = dict(num_classes=1, max_detections=4)
    if name == "score at threshold":
        a, s = _anchors(*far[:2]), [[0.5], [0.4999999]]
        kw["nms_score_threshold"] = 0.5
    elif name.startswith("iou at threshold"):
        a, s = _anchors(unit, (0, 0, 1, 0.5)), [[0.9], [0.8]]   # IoU exactly 0.5
        kw["nms_iou_threshold"] = 0.5 if name.endswith("kept") else 0.4999
    elif name == "identical boxes and scores":
        a, s = _anchors(unit, unit, unit), [[0.7], [0.7], [0.7]]
    elif name == "nan scores":
        a, s = _anchors(*far[:3]), [[np.nan, 0.1], [0.3, 0.9], [0.2, np.nan]]
        kw["num_classes"] = 2
    elif name == "zero-area box":
        a, s = _anchors(unit, (0.5, 0.5, 0.5, 0.5), unit, (0.5, 0.5, 0.5, 0.5)), [[0.9], [0.8], [0.7], [0.6]]
    elif name.startswith("label offset"):
        a, s = _anchors(*far[:3]), [[0.1, 0.2, 0.3], [0.9, 0.5, 0.1], [0.0, 0.1, 0.4]]
        kw["num_classes"] = 3 - int(name[-1])
    elif name == "k6":
        a, s = _anchors(*far[:3]), [[0.5], [0.7], [0.6]]
    elif name == "fewer classes than slots":
        a, s = _anchors(*far[:3]), [[0.1, 0.5, 0.2], [0.3, 0.2, 0.9], [0.4, 0.1, 0.3]]
        kw.update(num_classes=2, max_classes_per_detection=3)
    elif name == "nothing kept":
        a, s = _anchors(*far[:3]), [[0.1], [0.2], [0.3]]
        kw["nms_score_threshold"] = 0.5
    elif name.startswith("per class"):
        a = _anchors(*far)
        s = [[0, 0.9, 0.8], [0, 0.85, 0.7], [0, 0.6, 0.95], [0, 0.5, 0.4]]
        kw.update(num_classes=2, use_regular_nms=1, max_detections=3,
                  detections_per_class=1 if name.endswith("below") else 10)
    else:
        raise KeyError(name)
    s = np.array(s, F32)[None]
    k = 6 if name == "k6" else 4
    enc = np.zeros((1, len(a), k), F32)
    if k == 6:
        enc[..., 4:] = np.nan   # past the 4 coordinates nothing is read
    return enc, s, a, kw


CASES = {   # case: (the selected anchors in output order, their classes, num_detections)
    "score at threshold": ([0], [0], 1),
    "iou at threshold kept": ([0, 1], [0, 0], 2),
    "iou at threshold suppressed": ([0], [0], 1),
    "identical boxes and scores": ([0], [0], 1),
    "nan scores": ([1, 2], [1, 0], 2),   # anchor 0: NaN in class 0 is its maximum; anchor 2's NaN is passed over
    "zero-area box": ([0, 1, 3], [0, 0, 0], 3),
    "label offset 0": ([1, 2, 0], [0, 2, 2], 3),
    "label offset 1": ([1, 2, 0], [0, 1, 1], 3),
    "k6": ([1, 2, 0], [0, 0, 0], 3),
    "fewer classes than slots": ([1, 0, 2], None, 3),
    "nothing kept": ([], [], 0),
    "per class below": ([2, 0], [1, 0], 2),
    "per class above": ([2, 0, 1], [1, 0, 0], 3),
}


def _reference_case(name):
    enc, s, a, kw = _case(name)
    return (enc, s, a, kw), postprocess_ref(enc, s, a, **kw)


@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_on_known_answers(name):
    (enc, s, a, kw), (boxes, classes, scores, num) = _reference_case(name)
    want_sel, want_cls, want_num = CASES[name]
    assert num[0] == want_num
    o = dict(DEFAULTS, **kw)
    mc = o["max_classes_per_detection"] if not o["use_regular_nms"] else 1
    dec = decode(enc[0], a, o)
    for r, anchor in enumerate(want_sel):
        assert np.array_equal(boxes[0, mc * r], dec[anchor]), (r, anchor)
        if want_cls is not None:
            assert classes[0, mc * r] == want_cls[r]
    # every slot past the detections (and every class slot past num_classes) is zero
    used = np.zeros(boxes.shape[1], bool)
    kc = min(o["max_classes_per_detection"], o["num_classes"]) if not o["use_regular_nms"] else 1
    for r in range(want_num):
        used[mc * r: mc * r + kc] = True
    assert not boxes[0, ~used].any() and not classes[0, ~used].any() and not scores[0, ~used].any()


def test_reference_details():
    # fewer classes than slots: each detection has two classes, descending, then a zero slot
    _, (b, c, s, n) = _reference_case("fewer classes than slots")
    assert c[0, :3].tolist() == [1, 0, 0] and s[0, :3].tolist() == [F32(0.9), F32(0.2), 0]
    # the regular merge keeps class order on equal scores
    enc = np.zeros((1, 2, 4), F32)
    a = _anchors((0, 0, 1, 1), (3, 3, 4, 4))
    sc = np.array([[[0.5, 0.5], [0.5, 0.5]]], F32)
    _, c, _, n = postprocess_ref(enc, sc, a, num_classes=2, use_regular_nms=1, max_detections=3)
    assert n[0] == 3 and c[0].tolist() == [0, 0, 1]
    # -0.0 sorts as +0.0: the lower anchor first
    sc = np.array([[[0.0], [-0.0]]], F32)[:, ::-1].copy()
    b, _, s, n = postprocess_ref(enc, sc, a, num_classes=1, nms_score_threshold=-1.0)
    assert n[0] == 2 and np.array_equal(b[0, 0], decode(enc[0], a, DEFAULTS)[0])


# ------------------------------- FlexBuffers ------------------------------- #
def test_flex_map_reads_floats_ints_and_bools():
    blob = W.flex_map({"f": 0.6, "i": 7, "t": True, "n": -3})
    assert blob[-1] == 4   # float32 values: byte width 4
    assert H.flex_get_float(blob, "f") == F32(0.6) and H.flex_get_int(blob, "i") == 7
    assert H.flex_get_bool(blob, "t") and not H.flex_get_bool(blob, "missing")
    assert H.flex_get_float(blob, "i") == 7.0 and H.flex_get_float(blob, "missing", 2.5) == 2.5
    assert H.flex_get_bool(blob, "missing", True) and H.flex_get_int(blob, "n") == -3
    wide = W.flex_map({"d": np.float64(1e-8), "i": 1 << 40, "b": False})
    assert wide[-1] == 8
    assert H.flex_get_float(wide, "d") == F32(1e-8) and not H.flex_get_bool(wide, "b", True)
    assert H.flex_get_float(wide, "i") == float(1 << 40)
    assert H.flex_map_size(wide) == 3


def test_converter_style_options_parse():
    blob = W.detection_postprocess_options(num_classes=90, use_regular_nms=True, nms_iou_threshold=0.5)
    assert H.flex_map_size(blob) == 13 and H.flex_get_bool(blob, "_output_quantized")
    for k, v in (("max_detections", 100), ("max_classes_per_detection", 1), ("detections_per_class", 100),
                 ("num_classes", 90)):
        assert H.flex_get_int(blob, k) == v
    for k, v in (("nms_score_threshold", 1e-8), ("nms_iou_threshold", 0.5), ("y_scale", 10), ("w_scale", 5)):
        assert H.flex_get_float(blob, k) == F32(v)
    assert H.flex_get_bool(blob, "use_regular_nms")


@pytest.mark.parametrize("items", [{"channels_in": 3, "stride_height": 1}, {"a": 70000, "b": -5, "channels_in": 3072},
                                   {"padding": 1, "filter_height": 2, "filter_width": 2, "stride_width": 2}])
def test_flex_int_map_bytes_are_unchanged(items):
    assert W.flex_int_map(items) == H.flex_int_map(items) == W.flex_map(items)


# --------------------------------- host op --------------------------------- #
def _det_graph(b=2, n=6, k=4, s=4, options=None, anchors=None, anchors_const=True, dtype=np.float32,
               anchors_shape=None, scores_shape=None):
    m = TFLiteModel()
    enc = m.add_tensor("enc", (b, n, k), dtype)
    sc = m.add_tensor("scores", scores_shape or (b, n, s), dtype)
    if anchors is None:
        anchors = _anchors(*[(i, i, i + 1, i + 1) for i in range(n)])
    if anchors_const:
        an = m.add_tensor("anchors", None, np.float32, data=np.asarray(anchors, F32).reshape(anchors_shape or (-1, 4)))
    else:
        an = m.add_tensor("anchors", anchors_shape or (n, 4), np.float32)
    outs = [m.add_tensor(f"o{i}", sh) for i, sh in enumerate(((b, 10, 4), (b, 10), (b, 10), (b,)))]
    opts = options if options is not None else W.detection_postprocess_options(num_classes=s - 1, max_detections=10)
    m.add_op(OP, [enc, sc, an], outs, custom_options=opts)
    m.inputs = [enc, sc] + ([] if anchors_const else [an])
    m.outputs = outs
    return m.serialize()


@pytest.mark.parametrize("mc,b", [(1, 2), (3, 1), (2, 5)])
def test_host_prepares_the_output_shapes(mc, b):
    opts = W.detection_postprocess_options(num_classes=3, max_detections=7, max_classes_per_detection=mc)
    g = H.HostGraph.from_tflite(_det_graph(b=2, options=opts), device_arena=False)
    g.resize_input(g.inputs()[0], (b, 6, 4))
    g.resize_input(g.inputs()[1], (b, 6, 4))
    g.allocate_tensors()
    assert [g.shape(t) for t in g.outputs()] == [(b, 7 * mc, 4), (b, 7 * mc), (b, 7 * mc), (b,)]
    g.close()


def _opts(**kw):
    base = dict(num_classes=3, max_detections=10)
    base.update(kw)
    return W.detection_postprocess_options(**base)


REFUSALS = {
    "uint8 inputs": (dict(dtype=np.uint8), "must be float32"),
    "2-D box encodings": (dict(k=None), "must be 3-D"),
    "short box rows": (dict(k=3), "shapes must be"),
    "anchor count": (dict(anchors_shape=(3, 8), anchors=_anchors(*[(i, i, i + 1, i + 1) for i in range(6)])),
                     "shapes must be"),
    "score rows": (dict(scores_shape=(2, 5, 4)), "shapes must be"),
    "num_classes 0": (dict(options=_opts(num_classes=0)), "num_classes must be in"),
    "num_classes too many": (dict(options=_opts(num_classes=5)), "num_classes must be in"),
    "max_detections 0": (dict(options=_opts(max_detections=0)), "max_detections must be at least 1"),
    "max_classes_per_detection 0": (dict(options=_opts(max_classes_per_detection=0)),
                                    "max_classes_per_detection must be at least 1"),
    "detections_per_class 0": (dict(options=_opts(detections_per_class=0, use_regular_nms=True)),
                               "detections_per_class must be at least 1"),
    "iou 0": (dict(options=_opts(nms_iou_threshold=0.0)), r"nms_iou_threshold must be in \(0, 1\]"),
    "iou above 1": (dict(options=_opts(nms_iou_threshold=1.5)), r"nms_iou_threshold must be in \(0, 1\]"),
    "dynamic anchors": (dict(anchors_const=False), "anchors must be a constant"),
    "negative anchor height": (dict(anchors=np.array([[0.5, 0.5, -1, 1]] * 6, F32)), "must be finite and non-negative"),
    "nan anchor width": (dict(anchors=np.array([[0.5, 0.5, 1, np.nan]] * 6, F32)), "must be finite and non-negative"),
    "too many anchors": (dict(n=None), "anchors are more than the"),
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_host_refuses(case):
    kw, message = REFUSALS[case]
    kw = dict(kw)
    if case == "2-D box encodings":
        m = TFLiteModel()
        enc = m.add_tensor("enc", (2, 24))
        sc = m.add_tensor("scores", (2, 6, 4))
        an = m.add_tensor("anchors", None, np.float32, data=_anchors(*[(i, i, i + 1, i + 1) for i in range(6)]))
        outs = [m.add_tensor(f"o{i}", (1,)) for i in range(4)]
        m.add_op(OP, [enc, sc, an], outs, custom_options=_opts())
        m.inputs, m.outputs = [enc, sc], outs
        blob = m.serialize()
    elif case == "too many anchors":
        n = 40000
        blob = _det_graph(n=n, anchors=np.tile(np.array([[0.5, 0.5, 1, 1]], F32), (n, 1)))
    else:
        blob = _det_graph(**kw)
    g = H.HostGraph.from_tflite(blob, device_arena=False)
    with pytest.raises(H.HostError, match=message):
        g.allocate_tensors()
    g.close()


def test_max_anchors_covers_ssd():
    from compute_engine_b200 import capi
    assert capi.detection_max_anchors() >= 16384


def test_the_op_resolves_in_every_resolver():
    blob = zoo.quicknet_ssd(batch=1, image=64)
    for kw in ({}, {"use_reference_bconv": True}):
        g = H.HostGraph.from_tflite(blob, device_arena=False, **kw)
        g.allocate_tensors()
        g.close()


# ----------------------------------- model ----------------------------------- #
SSD_COUNTS = {(3, ""): 11, (4, ""): 7, (17, ""): 3, (32, "LceQuantize"): 16, (32, "LceBconv2d"): 16, (0, ""): 16,
              (22, ""): 6, (2, ""): 2, (14, ""): 1}


@pytest.mark.parametrize("postprocess", [True, False])
@pytest.mark.parametrize("input_type", ["float32", "int8"])
def test_quicknet_ssd_ops_and_shapes(postprocess, input_type):
    m = R.parse(zoo.quicknet_ssd(batch=2, input_type=input_type, postprocess=postprocess))
    kinds = collections.Counter((o["code"], o["custom"]) for o in m["ops"])
    want = dict(SSD_COUNTS)
    if input_type == "int8":
        want[(6, "")] = 1
    if postprocess:
        want[(32, OP)] = 1
    assert kinds == want
    shapes = [m["tensors"][i]["shape"] for i in m["outputs"]]
    if not postprocess:
        assert shapes == [(2, 3822, 4), (2, 3822, 21)]
        return
    assert shapes == [(2, 100, 4), (2, 100), (2, 100), (2,)]
    op = m["ops"][-1]
    blob = bytes(op["custom_options"])
    assert H.flex_get_int(blob, "num_classes") == 20 and not H.flex_get_bool(blob, "use_regular_nms")
    assert H.flex_get_float(blob, "nms_iou_threshold") == F32(0.6)
    anchors = m["tensors"][op["inputs"][2]]["data"]
    assert anchors.shape == (3822, 4) and np.array_equal(anchors, zoo.ssd_anchors([(28, 28), (14, 14), (7, 7)]))


def test_ssd_anchors_follow_the_grid_generator():
    a = zoo.ssd_anchors([(2, 2), (1, 1)])
    assert a.shape == (2 * 2 * 3 + 6, 4) and a.dtype == F32
    assert np.array_equal(a[0], F32([0.25, 0.25, 0.1, 0.1]))
    assert a[1, 2] == F32(0.2) / np.sqrt(F32(2)) and a[1, 3] == F32(0.2) * np.sqrt(F32(2))
    assert np.array_equal(a[3, :2], F32([0.25, 0.75]))   # (row 0, column 1), anchor 0
    assert np.array_equal(a[12], F32([0.5, 0.5, 0.95, 0.95]))
    assert a[17, 2] == F32(np.sqrt(0.95 * 1.0))


def test_quicknet_ssd_is_not_registered():
    assert "quicknet_ssd" not in zoo.MODELS and zoo.quicknet_ssd not in zoo.MODELS.values()
    with pytest.raises(ValueError, match="multiple of 32"):
        zoo.quicknet_ssd(image=100)


SSD_FUSED_TAIL = (["builtin:4", "builtin:3", "builtin:22", "builtin:3", "builtin:22"] * 3 +
                  ["builtin:2", "builtin:2", "builtin:14", OP])


def test_quicknet_ssd_fused_node_list():
    g = H.HostGraph.from_tflite(zoo.quicknet_ssd(batch=2, input_type="int8"), device_arena=True)
    g.fuse_all()
    names = [g.node_name(i) for i in range(g.num_nodes())]
    g.close()
    g = H.HostGraph.from_tflite(zoo.quicknet(batch=2, input_type="int8"), device_arena=True)
    g.fuse_all()
    backbone = [g.node_name(i) for i in range(g.num_nodes())]
    g.close()
    # QuickNet's fused backbone up to its head, then the detection heads and the op, unfused
    k = backbone.index("builtin:19") if "builtin:19" in backbone else len(backbone) - 3
    assert names == backbone[:k] + SSD_FUSED_TAIL


def test_other_models_keep_their_bytes():
    import hashlib
    from test_segmentation import MODEL_HASHES
    for name, make in zoo.MODELS.items():
        assert hashlib.sha256(make(batch=1, seed=0)).hexdigest()[:16] == MODEL_HASHES[name], name


def test_detection_kernels_compile_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(repo, "compute_engine_b200", "csrc", "lce_b200_detect.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas=-v",
                        "-cubin", "-I", os.path.join(repo, "include"), src, "-o", str(tmp_path / "detect.cubin")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    props = re.findall(r"Function properties for (\S*detection_\S*)\n\s*(.*)", r.stderr)
    assert len(props) == 4, r.stderr   # decode, NMS in both modes, merge
    for name, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)


# ----------------------------------- GPU ----------------------------------- #
def _same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _gpu(enc, scores, anchors, **kw):
    import torch
    from compute_engine_b200 import capi
    o = dict(DEFAULTS, **kw)
    t = [torch.from_numpy(np.ascontiguousarray(v, F32)).cuda() for v in (enc, scores, anchors)]
    out = capi.detection_postprocess(*t, **o)
    torch.cuda.synchronize()
    return tuple(v.cpu().numpy() for v in out)


def _compare(got, want, inputs):
    names = ("boxes", "classes", "scores", "num_detections")
    for name, g, w in zip(names, got, want):
        if not _same_bits(g, w):
            bad = np.argwhere(g.view(np.uint32) != w.view(np.uint32))[0]
            b = int(bad[0])
            msg = f"{name} differ first at {tuple(bad)}: kernel {g[tuple(bad)]!r}, reference {w[tuple(bad)]!r}"
            if name == "boxes":
                j = int(bad[1])
                row = w[b, j]
                enc, _, anchors = inputs
                hit = np.flatnonzero((decode(enc[b], anchors, DEFAULTS) == row).all(1))
                msg += f"; reference box {row}, anchor(s) {hit[:4]}, encodings {enc[b, hit[:1]]}, anchors {anchors[hit[:1]]}"
            pytest.fail(msg)


def _random(rng, b, n, c, k=4, offset=1, adversarial=False):
    if adversarial:   # few distinct boxes and scores: ties and dense overlaps everywhere
        anchors = _anchors(*[(y, x, y + 1, x + 1) for y in (0, 0.25, 0.5) for x in (0, 0.25, 0.5)])
        anchors = anchors[rng.integers(0, len(anchors), n)]
        enc = (rng.integers(-2, 3, (b, n, k)) * 0.5).astype(F32)
        scores = (rng.integers(0, 5, (b, n, c + offset)) / 4).astype(F32)
        scores[rng.random(scores.shape) < 0.02] = -0.0
    else:
        yx = rng.random((n, 2), dtype=F32)
        hw = rng.uniform(0.05, 0.5, (n, 2)).astype(F32)
        anchors = np.concatenate([yx, hw], 1)
        enc = rng.standard_normal((b, n, k), dtype=F32)
        scores = rng.random((b, n, c + offset), dtype=F32)
    return enc, scores, anchors


GPU_CASES = [(mode, b, kind) for mode in (0, 1) for b in (1, 3) for kind in ("random", "adversarial")]


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_gpu_known_answers(name):
    (enc, s, a, kw), want = _reference_case(name)
    _compare(_gpu(enc, s, a, **kw), want, (enc, s, a))


@pytest.mark.gpu
@pytest.mark.parametrize("regular,b,kind", GPU_CASES)
def test_gpu_matches_the_reference(regular, b, kind):
    rng = np.random.default_rng(regular * 10 + b + (kind == "adversarial") * 100)
    for n, c, k, offset, kw in ((500, 5, 4, 1, {}), (777, 3, 6, 0, dict(max_classes_per_detection=2)),
                                (3822, 20, 4, 1, dict(nms_iou_threshold=0.3, detections_per_class=40)),
                                (64, 4, 4, 1, dict(max_detections=7, max_classes_per_detection=5,
                                                   nms_score_threshold=0.5))):
        enc, scores, anchors = _random(rng, b, n, c, k, offset, kind == "adversarial")
        o = dict(kw, num_classes=c, use_regular_nms=regular)
        _compare(_gpu(enc, scores, anchors, **o), postprocess_ref(enc, scores, anchors, **o), (enc, scores, anchors))


@pytest.mark.gpu
@pytest.mark.parametrize("regular", [0, 1])
def test_gpu_at_the_anchor_limit(regular):
    from compute_engine_b200 import capi
    n = capi.detection_max_anchors()
    enc, scores, anchors = _random(np.random.default_rng(7 + regular), 1, n, 3)
    o = dict(num_classes=3, use_regular_nms=regular, max_detections=150)
    _compare(_gpu(enc, scores, anchors, **o), postprocess_ref(enc, scores, anchors, **o), (enc, scores, anchors))


@pytest.mark.gpu
@pytest.mark.parametrize("regular", [0, 1])
def test_gpu_batch_256_equals_each_image_alone(regular):
    enc, scores, anchors = _random(np.random.default_rng(3), 256, 3822, 20)
    scores[5:9] = (np.round(scores[5:9] * 4) / 4).astype(F32)   # a few images full of ties
    o = dict(num_classes=20, use_regular_nms=regular)
    got = _gpu(enc, scores, anchors, **o)
    for b in (0, 5, 8, 131, 255):
        alone = _gpu(enc[b:b + 1], scores[b:b + 1], anchors, **o)
        for g, a in zip(got, alone):
            assert _same_bits(g[b:b + 1], a), b
    for b in (0, 6, 255):
        want = postprocess_ref(enc[b:b + 1], scores[b:b + 1], anchors, **o)
        _compare(tuple(v[b:b + 1] for v in got), want, (enc[b:b + 1], scores[b:b + 1], anchors))


def _logistic_ref(x):
    import torch
    return torch.sigmoid(torch.from_numpy(x)).numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("regular", [False, True])
def test_gpu_quicknet_ssd_op_by_op(regular):
    """The unfused graph at batch 4, op by op on the device's own inputs: every LCE op, ADD and the
    post-processing bit exact, the other float builtins within the torch fp32 reference's tolerance."""
    blob = zoo.quicknet_ssd(batch=1, seed=9, use_regular_nms=regular)
    m = R.parse(blob)
    x = np.random.default_rng(3).standard_normal((4, 224, 224, 3)).astype(F32)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.preserve_all_tensors(True)
    g.resize_input(g.inputs()[0], x.shape)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    exact = collections.Counter()
    o = {k: v for k, v in DEFAULTS.items()}
    o.update(use_regular_nms=int(regular))
    for op in m["ops"]:
        act = [i for i in op["inputs"] if i >= 0 and m["tensors"][i]["data"] is None]
        vals = {i: g.read(i) for i in act}
        if op["custom"] == OP:
            want = postprocess_ref(vals[op["inputs"][0]], vals[op["inputs"][1]], m["tensors"][op["inputs"][2]]["data"],
                                   **o)
            got = [g.read(t) for t in op["outputs"]]
            _compare(got, want, (vals[op["inputs"][0]], vals[op["inputs"][1]], m["tensors"][op["inputs"][2]]["data"]))
            assert (got[3] > 0).all()
            exact[OP] += 1
            continue
        if op["code"] == 14:
            want = _logistic_ref(vals[op["inputs"][0]])
        else:
            sub = {"tensors": m["tensors"], "ops": [op], "inputs": act, "outputs": [op["outputs"][0]]}
            want = R.run(sub, [vals[i] for i in act])[0][0]
        got = g.read(op["outputs"][0])
        assert got.shape == want.shape, (op["code"], op["custom"])
        if op["code"] in (0, 2, 22, 32):
            assert _same_bits(got, want.astype(got.dtype)), (op["code"], op["custom"])
            exact[op["custom"] or op["code"]] += 1
        else:
            scale = max(1.0, float(np.abs(want).max()))
            assert np.allclose(got, want, rtol=1e-4, atol=1e-5 * scale), (op["code"], np.abs(got - want).max())
    assert exact == {"LceBconv2d": 16, "LceQuantize": 16, 0: 16, 22: 6, 2: 2, OP: 1}
    g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("regular", [False, True])
def test_gpu_quicknet_ssd_fused_equals_unfused(regular):
    blob = zoo.quicknet_ssd(batch=1, seed=4, input_type="int8", use_regular_nms=regular)
    x = zoo.quantize_images(np.random.default_rng(256).standard_normal((256, 224, 224, 3), dtype=F32))
    outs = {}
    for fuse in (False, True):
        g = H.HostGraph.from_tflite(blob, device_arena=True)
        if fuse:
            assert g.fuse_all() > 0
        g.resize_input(g.inputs()[0], x.shape)
        g.allocate_tensors()
        g.write(g.inputs()[0], x)
        g.invoke()
        outs[fuse] = [g.read(t) for t in g.outputs()]
        g.close()
    assert [o.shape for o in outs[True]] == [(256, 100, 4), (256, 100), (256, 100), (256,)]
    assert (outs[True][3] > 0).all()
    for a, b in zip(outs[False], outs[True]):
        assert _same_bits(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("regular", [False, True])
def test_gpu_quicknet_ssd_does_not_depend_on_the_arena(regular):
    import test_arena_independence as A
    blob = zoo.quicknet_ssd(batch=1, seed=0, use_regular_nms=regular)
    fails = A.check_arena_independence(blob, (A.BATCH, 224, 224, 3), "float32", fuse=True)
    assert not fails, "quicknet_ssd:\n" + "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("batch_size", [3, 5])
def test_gpu_interpreter_predict_over_mini_batches(batch_size):
    from compute_engine_b200.interpreter import Interpreter
    blob = zoo.quicknet_ssd(batch=1, image=64, seed=2, input_type="int8")
    x = zoo.quantize_images(np.random.default_rng(1).standard_normal((11, 64, 64, 3), dtype=F32))
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    g.fuse_all()
    g.resize_input(g.inputs()[0], x.shape)
    g.allocate_tensors()
    g.write(g.inputs()[0], x)
    g.invoke()
    want = [g.read(t) for t in g.outputs()]
    g.close()
    it = Interpreter(blob, batch_size=batch_size)
    got = it.predict(x)
    it.close()
    assert len(got) == 4
    for a, b in zip(got, want):
        assert _same_bits(np.asarray(a), b)
