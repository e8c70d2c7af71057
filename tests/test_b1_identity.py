"""The b1 inner product of the mma.sync kernel (compute_engine_b200/csrc/lce_b200_imma.cuh),
checked in numpy:

    popc(a ^ w) = popc(w) + popc(a) - 2 * popc(a & w)

with popc(a & w) and popc(a) as BMMA.AND.POPC sums. The fragment layout is mirrored from the
kernel: A rows [k-slice][pixel][8 words], the plan-time weight image of pack_weights_b1_kernel,
the registers thread (gid, tig) hands to mma.sync m16n8k256 / m16n8k128, and the k positions
PTX gives those registers. Padding words (out-of-bounds taps, the K tail) are 0."""
import numpy as np

M32 = 0xFFFFFFFF


def popc(x):
    return bin(int(x) & M32).count("1")


def a_rows(acts, Kw):
    """gather_tile<kSliceRows>: [slice][pixel][8 words], K padded with 0 words."""
    n_slices = -(-Kw // 8)
    out = np.zeros((n_slices, acts.shape[0], 8), dtype=np.uint64)
    for k in range(Kw):
        out[k // 8, :, k % 8] = acts[:, k]
    return out


def pack_weights_b1(filt, Kw):
    """pack_weights_b1_kernel for one 8-channel sub-tile: [slice][lane] = (b0, b1)."""
    n_slices = -(-Kw // 8)
    Kwp = (Kw + 3) & ~3
    img = np.zeros((n_slices, 32, 2), dtype=np.uint64)
    for s in range(n_slices):
        tail = s * 8 + 4 >= Kwp
        for lane in range(32):
            ch, tig = lane >> 2, lane & 3
            k0 = s * 8 + (tig if tail else 2 * tig)
            img[s, lane, 0] = filt[ch, k0] if k0 < Kw else 0
            img[s, lane, 1] = filt[ch, k0 + 1] if not tail and k0 + 1 < Kw else 0
    return img


def a_regs(A, s, gid, tig, tail):
    """compute_chunk_b1: the A registers of thread (gid, tig) for one m16 tile."""
    if tail:
        return [A[s, gid, tig], A[s, gid + 8, tig]]
    lo, hi = A[s, gid], A[s, gid + 8]
    return [lo[2 * tig], hi[2 * tig], lo[2 * tig + 1], hi[2 * tig + 1]]


def mma_and_popc(A, B, s, tail, ones=False):
    """D[16][8] of one mma.sync ... b1 and.popc, from the per-thread registers by PTX's fragment
    layout: A element (r, k) sits in thread (r % 8, (k % 128) // 32), register
    (k >= 128) * 2 + (r >= 8); B element (k, n) in thread (n, (k % 128) // 32), register k >= 128."""
    K = 128 if tail else 256
    d = np.zeros((16, 8), dtype=np.int64)
    for r in range(16):
        for n in range(8):
            for k32 in range(K // 32):
                tig, hi = k32 % 4, k32 // 4
                a = a_regs(A, s, r % 8, tig, tail)[hi * 2 + (r >= 8)]
                b = M32 if ones else B[s, n * 4 + tig, hi]
                d[r, n] += popc(int(a) & int(b))
    return d


def b1_accumulators(acts, filt):
    Kw = acts.shape[1]
    A, B = a_rows(acts, Kw), pack_weights_b1(filt, Kw)
    acc = np.zeros((16, 8), dtype=np.int64)
    pa = np.zeros((16, 8), dtype=np.int64)
    Kwp = (Kw + 3) & ~3
    for s in range(A.shape[0]):
        tail = s * 8 + 4 >= Kwp
        acc += mma_and_popc(A, B, s, tail)
        pa += mma_and_popc(A, B, s, tail, ones=True)
    wpop = np.array([sum(popc(v) for v in filt[n]) for n in range(8)])
    return wpop[None, :] + pa - 2 * acc


def xor_popc(acts, filt):
    return np.array([[sum(popc(int(a) ^ int(w)) for a, w in zip(acts[r], filt[n]))
                      for n in range(8)] for r in range(16)])


def test_and_popc_identity_per_word():
    rng = np.random.default_rng(0)
    words = rng.integers(0, 2**32, (400, 2), dtype=np.uint64)
    words[:4] = [[0, 0], [M32, 0], [0, M32], [M32, M32]]
    for a, w in words:
        assert popc(a ^ w) == popc(w) + popc(a) - 2 * popc(int(a) & int(w))


def test_fragments_give_xor_popcount_for_every_k_tail():
    """Full k256 slices, a k128 tail (Kw % 8 in 1..4) and zero words up to a full slice
    (Kw % 8 in 5..7): each (pixel, channel) gets sum_k popc(a ^ w) over the real K words."""
    rng = np.random.default_rng(1)
    for Kw in (1, 3, 4, 5, 8, 12, 18, 23, 36):
        acts = rng.integers(0, 2**32, (16, Kw), dtype=np.uint64)
        filt = rng.integers(0, 2**32, (8, Kw), dtype=np.uint64)
        assert np.array_equal(b1_accumulators(acts, filt), xor_popc(acts, filt)), Kw


def test_out_of_bounds_taps_gather_zero_words():
    """A tap outside the image gathers 0 words: it adds popc(w), the reference's one-padding;
    the zero-padding correction at scale 1 then adds channels_in / 2 - popc(w of the tap)."""
    rng = np.random.default_rng(2)
    taps, cw = 9, 2
    Kw = taps * cw
    acts = rng.integers(0, 2**32, (16, Kw), dtype=np.uint64)
    filt = rng.integers(0, 2**32, (8, Kw), dtype=np.uint64)
    oob = [0, 1, 2]                                   # top row of a 3x3 window
    for t in oob:
        acts[:, t * cw:(t + 1) * cw] = 0
    acc = b1_accumulators(acts, filt)
    inb = [k for k in range(Kw) if k // cw not in oob]
    tap_popc = [[sum(popc(v) for v in filt[n, t * cw:(t + 1) * cw]) for t in range(taps)]
                for n in range(8)]
    one_pad = np.array([[sum(popc(int(acts[r, k]) ^ int(filt[n, k])) for k in inb)
                         + sum(tap_popc[n][t] for t in oob) for n in range(8)] for r in range(16)])
    assert np.array_equal(acc, one_pad)
    zp_half = cw * 32 // 2
    corrected = acc + np.array([sum(zp_half - tap_popc[n][t] for t in oob) for n in range(8)])[None, :]
    want = one_pad - np.array([sum(tap_popc[n][t] for t in oob) for n in range(8)])[None, :] \
        + len(oob) * zp_half
    assert np.array_equal(corrected, want)


def test_scale_one_epilogue_matches_the_int8_scale():
    """The b1 accumulators are popc(a ^ w) itself: OutputTransform's acc << 1 and the raw store
    read them directly, where the int8 inner product's 8 * acc needs >> 2 and >> 3."""
    for acc in (0, 1, 7, 255, 12345, 25600):
        assert (acc << 1) == ((8 * acc) >> 2)
        assert acc == ((8 * acc) >> 3)
