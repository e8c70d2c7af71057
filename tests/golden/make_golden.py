#!/usr/bin/env python
"""Mint the golden vectors under tests/golden/ from the REFERENCE ITSELF.

Runs only in the build container (needs oracle/_ref/liblce_ref.so, i.e. the
reference's own headers compiled from /root/reference by oracle/Makefile). The
resulting ``lce_golden_*.npz`` parts are committed; the GPU box and the CPU test-suite
only read it. Inputs are regenerated from the recorded seeds by
``lce_testlib.make_bconv_case`` so only outputs (or, for the full-size config-1
case, SHA-256 digests of the outputs) are stored.

The case list re-runs the parameter grids of the reference's own op tests with
fixed seeds (they use std::random_device): bconv2d_test.cc:790-856 (SmallTest /
BigTest shapes), bmaxpool_test.cc:204-218, quantization_test.cc:121-130,
bitpack_test.cc:102-109.

Usage:  python tests/golden/make_golden.py
"""
import glob
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import lce_testlib as L  # noqa: E402


def bconv_specs():
    """(batch,h,w,cin, fh,fw,cout, groups, stride, dilation, padding, pad_value,
    activation, out_type) -- a pruned walk of the reference's BigTest grid plus
    SmallTest shapes, the 16-bit-overflow shape and QuickNet-like shapes."""
    specs = []
    S, V = L.PADDING_SAME, L.PADDING_VALID
    shapes = [(1, 7, 7, 4), (3, 8, 5, 64), (2, 7, 7, 96), (1, 8, 5, 128),
              (1, 7, 7, 192), (1, 8, 5, 256), (1, 7, 7, 512), (1, 4, 4, 64)]
    filters = [(1, 1, 1), (3, 3, 1), (2, 3, 2), (1, 1, 3), (3, 3, 4), (2, 3, 5),
               (1, 1, 6), (3, 3, 7), (2, 3, 32), (3, 3, 64)]
    i = 0
    for shape in shapes:
        for filt in filters:
            for groups in (1, 2, 4):
                b, h, w, c = shape
                fh, fw, co = filt
                if groups > 1 and (c % groups or co % groups or (c // groups) % 32):
                    continue
                # rotate through the remaining axes instead of the full product
                stride = ((1, 1), (2, 3))[i % 2]
                dil = ((1, 1), (3, 2))[(i // 2) % 2]
                pad, pv = ((V, 1), (S, 0), (S, 1))[i % 3]
                act = (L.ACT_NONE, L.ACT_RELU)[(i // 3) % 2]
                ot = (L.OUT_FLOAT, L.OUT_INT8, L.OUT_BITPACKED)[(i // 5) % 3]
                i += 1
                if pad == S and pv == 0 and c % 2:
                    pv = 1
                if pad == V and ((fh - 1) * dil[0] + 1 > h or (fw - 1) * dil[1] + 1 > w):
                    dil = (1, 1)
                specs.append((b, h, w, c, fh, fw, co, groups, stride, dil, pad,
                              pv, act, ot))
    # other activations
    for act in (L.ACT_RELU6, L.ACT_RELU_N1_TO_1):
        for ot in (L.OUT_FLOAT, L.OUT_INT8):
            specs.append((2, 6, 6, 64, 3, 3, 32, 1, (1, 1), (1, 1), S, 1, act, ot))
    # 16-bit accumulator overflow shape (bconv2d_test.cc:818-833)
    for ot in (L.OUT_FLOAT, L.OUT_BITPACKED):
        specs.append((1, 6, 6, 3072, 5, 5, 4, 1, (1, 1), (1, 1), S, 1,
                      L.ACT_RELU, ot))
    # QuickNet / Bi-RealNet-like layers at reduced spatial size
    for c, hw in ((64, 14), (128, 10), (256, 7), (512, 7)):
        specs.append((2, hw, hw, c, 3, 3, c, 1, (1, 1), (1, 1), S, 1, L.ACT_RELU,
                      L.OUT_FLOAT))
        specs.append((2, hw, hw, c, 3, 3, c, 1, (1, 1), (1, 1), S, 0, L.ACT_NONE,
                      L.OUT_FLOAT))
    specs.append((1, 14, 14, 64, 3, 3, 128, 1, (2, 2), (1, 1), S, 0, L.ACT_NONE,
                  L.OUT_FLOAT))
    return specs


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    if L.load_ref() is None:
        sys.exit("oracle/_ref/liblce_ref.so missing: run `make -C oracle` here")
    arrays, index = {}, {"bconv": [], "bconv_full": [], "bconv_zpc": [], "quantize": [],
                         "dequantize": [], "bmaxpool": []}

    for n, s in enumerate(bconv_specs()):
        (b, h, w, c, fh, fw, co, g, st, dl, pad, pv, act, ot) = s
        seed = 1000 + n
        case = L.make_bconv_case(seed, b, h, w, c, fh, fw, co, g, st, dl, pad, pv,
                                 act, ot)
        out = L.bconv2d(case.desc, case.inp, case.filt, case.mul, case.bias,
                        case.thr, impl="ref", kind=0)
        key = f"bconv_{n}"
        arrays[key] = out
        index["bconv"].append({"key": key, "seed": seed, "spec": list(s)})

    # Zero padding as the OPTIMISED kernels compute it -- what the reference's default
    # registration returns: Kernel4x2Portable with one-padding, OutputTransform, then
    # zero_padding_correction::ApplyCorrection (kind 1 of oracle/ref_shim.cc). Float output, no
    # activation (bconv2d.cc:188-200), odd channel counts included.
    for n, (b, h, w, c, fh, fw, co, st, dl) in enumerate([
            (2, 8, 8, 64, 3, 3, 32, (1, 1), (1, 1)), (1, 16, 16, 128, 3, 3, 64, (2, 2), (1, 1)),
            (2, 7, 7, 96, 3, 3, 16, (1, 1), (1, 1)), (1, 12, 12, 32, 5, 5, 8, (1, 1), (2, 2)),
            (1, 9, 11, 64, 3, 3, 8, (2, 1), (1, 1)), (1, 5, 5, 33, 3, 3, 8, (1, 1), (1, 1)),
            (1, 6, 6, 64, 5, 5, 8, (2, 2), (1, 1)), (3, 7, 7, 512, 3, 3, 64, (1, 1), (1, 1)),
            (1, 14, 14, 256, 3, 3, 128, (2, 2), (1, 1)), (1, 10, 7, 100, 2, 3, 12, (1, 2), (1, 1))]):
        seed = 5000 + n
        case = L.make_bconv_case(seed, b, h, w, c, fh, fw, co, 1, st, dl, L.PADDING_SAME, 0,
                                 L.ACT_NONE, L.OUT_FLOAT)
        key = f"bconv_zpc_{n}"
        arrays[key] = L.bconv2d(case.desc, case.inp, case.filt, case.mul, case.bias, None,
                                impl="ref", kind=1)
        index["bconv_zpc"].append({"key": key, "seed": seed,
                                   "spec": [b, h, w, c, fh, fw, co, list(st), list(dl)]})

    # config 1: 56x56x256 -> 256, k3 s1 SAME.
    # Outputs are 0.1-3.2 MB each, so only digests are stored.
    n = 0
    for pv in (1, 0):
        for act in (L.ACT_NONE, L.ACT_RELU):
            for ot in (L.OUT_FLOAT, L.OUT_INT8, L.OUT_BITPACKED):
                seed = n % 4
                case = L.make_bconv_case(seed, 1, 56, 56, 256, 3, 3, 256, 1,
                                         (1, 1), (1, 1), L.PADDING_SAME, pv, act,
                                         ot)
                ref0 = L.bconv2d(case.desc, case.inp, case.filt, case.mul,
                                 case.bias, case.thr, impl="ref", kind=0)
                entry = {"seed": seed, "pad_value": pv, "activation": act,
                         "out_type": ot, "sha256_reference_kernel": digest(ref0)}
                legal_opt = not (pv == 0 and (ot != L.OUT_FLOAT or act != L.ACT_NONE))
                if legal_opt:
                    ref1 = L.bconv2d(case.desc, case.inp, case.filt, case.mul,
                                     case.bias, case.thr, impl="ref", kind=1)
                    if pv == 1:
                        assert digest(ref1) == digest(ref0)
                    entry["sha256_indirect_kernel"] = digest(ref1)
                index["bconv_full"].append(entry)
                n += 1

    # LceQuantize / LceDequantize grids (bitpack_test.cc:102-109,
    # quantization_test.cc:121-130).
    rng = np.random.default_rng(7)
    n = 0
    for rows in (1, 2, 3, 8, 10, 15, 64):
        for cols in (1, 3, 16, 32, 33, 63, 64, 128):
            xf = rng.uniform(-1.5, 1.5, (rows, cols)).astype(np.float32)
            # sprinkle the special values the bit semantics hinge on
            flat = xf.reshape(-1)
            specials = np.array([-0.0, 0.0, np.nan, -np.nan, -1e-30, -1e-45,
                                 1e-45, -np.inf, np.inf], np.float32)
            flat[: min(flat.size, specials.size)] = specials[: flat.size]
            key = f"q_f32_{n}"
            arrays[key + "_in"] = xf
            arrays[key] = L.quantize(xf, impl="ref")
            index["quantize"].append({"key": key, "type": "f32", "zero_point": 0})
            for zp in (-1000, -1, 0, 23, 127, 128):
                xi = rng.integers(-128, 128, (rows, cols), dtype=np.int8)
                key = f"q_i8_{n}_{zp}"
                arrays[key + "_in"] = xi
                arrays[key] = L.quantize(xi, zero_point=zp, impl="ref")
                index["quantize"].append({"key": key, "type": "i8", "zero_point": zp})
            xb = rng.integers(0, 2, (rows, cols), dtype=np.uint8).astype(np.bool_)
            key = f"q_b_{n}"
            arrays[key + "_in"] = xb
            arrays[key] = L.quantize(xb, impl="ref")
            index["quantize"].append({"key": key, "type": "bool", "zero_point": 1})
            n += 1
    for n, (shape, ch) in enumerate([((1, 4, 4), 1), ((2, 3, 3), 31), ((1, 5, 2), 32),
                                     ((1, 2, 2), 33), ((3, 1, 1), 64), ((1, 3, 3), 68),
                                     ((1, 2, 3), 130), ((1, 1, 2), 200)]):
        packed = rng.integers(-2**31, 2**31, shape + (L.cdiv(ch, 32),),
                              dtype=np.int64).astype(np.int32)
        for t, scale, zp in ((L.T_FLOAT, 1.0, 0), (L.T_BOOL, 1.0, 0),
                             (L.T_INT8, 1.0, 0), (L.T_INT8, 0.05, 3),
                             (L.T_INT8, 0.007, -100), (L.T_INT8, 0.3, 127)):
            key = f"dq_{n}_{t}_{zp}"
            arrays[key + "_in"] = packed
            arrays[key] = L.dequantize(packed, ch, t, scale, zp, impl="ref").view(
                np.uint8 if t == L.T_BOOL else L._NP_T[t])
            index["dequantize"].append({"key": key, "channels": ch, "type": t,
                                        "scale": scale, "zero_point": zp})

    # LceBMaxPool2d grid (bmaxpool_test.cc:204-218 shapes, pruned).
    n = 0
    for (b, h, w, ch) in ((1, 7, 7, 1), (4, 8, 5, 2), (1, 12, 9, 3), (2, 56, 56, 2)):
        for (fh, fw) in ((1, 1), (2, 2), (3, 3), (2, 3)):
            for (sh, sw) in ((1, 1), (2, 2), (2, 3)):
                for pad in (L.PADDING_SAME, L.PADDING_VALID):
                    if pad == L.PADDING_VALID and (fh > h or fw > w):
                        continue
                    x = rng.integers(-2**31, 2**31, (b, h, w, ch),
                                     dtype=np.int64).astype(np.int32)
                    d = L.BMaxPoolDesc(b, h, w, ch, fh, fw, sh, sw, pad)
                    key = f"mp_{n}"
                    arrays[key + "_in"] = x
                    arrays[key] = L.bmaxpool(d, x, impl="ref")
                    index["bmaxpool"].append({"key": key, "desc": [b, h, w, ch, fh,
                                                                   fw, sh, sw, pad]})
                    n += 1

    # parts of under 1 MB each (tests/lce_testlib.py load_golden_arrays merges them)
    for old in glob.glob(os.path.join(HERE, "lce_golden_*.npz")):
        os.remove(old)
    keys, part, n_parts = list(arrays), {}, 0
    for i, k in enumerate(keys):
        part[k] = arrays[k]
        if sum(v.nbytes for v in part.values()) >= 800_000 or i == len(keys) - 1:
            np.savez_compressed(os.path.join(HERE, f"lce_golden_{n_parts}.npz"), **part)
            part, n_parts = {}, n_parts + 1
    with open(os.path.join(HERE, "lce_golden.json"), "w") as f:
        json.dump({"generator": "tests/golden/make_golden.py",
                   "reference": "larq/compute-engine e6860fcf core headers via "
                                "oracle/ref_shim.cc (kReference kernel unless "
                                "stated)", "index": index}, f, indent=1)
    sz = sum(os.path.getsize(p) for p in glob.glob(os.path.join(HERE, "lce_golden_*.npz")))
    print(f"wrote {len(arrays)} arrays, {sz/1e6:.2f} MB;",
          {k: len(v) for k, v in index.items()})


if __name__ == "__main__":
    main()
