"""Whole graphs whose results must not depend on what the tensor arena holds or where each tensor
sits in it, and CUDA-graph replays that must recompute everything from the new input.

Every other graph test starts from a fresh cudaMalloc arena, which is usually zeroed, and replays
the images it ran eagerly. A kernel that leaves output elements unwritten whose right value is 0, a
kernel that reads bytes its node does not own (the 64-byte slack PlanArena leaves behind each
tensor, a neighbouring tensor, a tensor missing from a fused node's IO lists, 0 * NaN), or a replay
that recomputes nothing, passes there. Here each graph runs under these variants, and each must give
the same bytes as the anchor: the same graph, eager, every tensor kept (preserve_all_tensors), the
arena zeroed by a memset before the input is written.
  P-A, P-B  every tensor kept, the arena filled with 0xFF (float NaN, int32 -1) or 0x7F (float
            3.4e38, int32 0x7F7F7F7F). Every tensor any node writes is compared with the anchor's,
            and a mismatch names the first node, in execution order, whose output differs. The
            arena bytes that belong to no tensor (past each tensor's 64 bytes of slack) must still
            hold the poison.
  R-A, R-B  the reused arena (the planner's own layout, the one bench.py times), poisoned: the
            graph's outputs. With P-x passing, a failure here is aliasing: a fused node reading a
            tensor missing from its IO lists, or writing past its tensor's slack.
  shrunk    the graph planned and run at twice the batch, then re-planned at the test batch in the
            same arena, which holds the larger run's tensors at other offsets (what Interpreter
            does across mini-batch sizes).
  replay    a CUDA graph captured on images x0, then replayed on x1 with the arena filled with 0xFF
            and on x2 with 0x7F: each must equal the anchor on that input, and the two must differ.
The zeroed anchor is also run twice, so that a kernel whose result varies from run to run is told
apart from one that depends on the arena. Nothing is compared with a poison value: a packed word
may legitimately be -1.

The arena is filled with cudaMemset from the CUDA runtime torch loads (the host library links
cudart statically; both use the device's primary context). The CPU tests check the two host
accessors this relies on and that every family of the zoo is covered.
"""
import ctypes as C
import sys

import numpy as np
import pytest

import tflite_ref as R
from compute_engine_b200 import host as H
from compute_engine_b200 import zoo

POISON = (("A", 0xFF), ("B", 0x7F))
BATCH = 8

# the graphs bench.py times, at its batch sizes
BENCHMARKED = [("quicknet", 256), ("quicknet_large", 128), ("quicknet_small", 256)]

# every other family, and the variants built outside zoo.MODELS
FAMILIES = {name: (zoo.MODELS[name], {}) for name in zoo.MODELS if name not in dict(BENCHMARKED)}
FAMILIES.update({
    "abcnet-3x3": (zoo.abcnet, dict(bases=(3, 3))),
    "xnornetpp-pad0": (zoo.xnornetpp, dict(pad_values=0)),
    "xnornetpp-pad1": (zoo.xnornetpp, dict(pad_values=1)),
    "binary_mobilenet": (zoo.binary_mobilenet, {}),
    "meliusnet-native-groups": (zoo.meliusnet, dict(group_conv="native")),
    "realtobinarynet-pad1": (zoo.realtobinarynet, dict(pad_values=1)),
})

# one unfused graph per family: float builtins and stand-alone LCE ops
UNFUSED = {"quicknet": (zoo.quicknet, {}), "abcnet": (zoo.abcnet, {}),
           "xnornetpp": (zoo.xnornetpp, {}), "binary_mobilenet": (zoo.binary_mobilenet, {})}
UNFUSED.update({name: (zoo.MODELS[name], {}) for name in (
    "birealnet18", "reactnet_a", "realtobinarynet", "binarydensenet28", "meliusnet22",
    "binaryalexnet", "xnornet", "dorefanet")})


@pytest.fixture(autouse=True)
def _release_snapshots():
    """The arena snapshots are torch tensors of up to a few GB: give their memory back to the
    device after each test rather than leave it in torch's cache for the rest of the suite."""
    yield
    torch = sys.modules.get("torch")
    if torch is not None and torch.cuda.is_initialized():
        torch.cuda.empty_cache()


# ------------------------------------------------------------------ arena access
_RT = None


def cudart():
    global _RT
    if _RT is None:
        import torch  # noqa: F401  (loads libcudart.so.12 into the process)
        rt = C.CDLL("libcudart.so.12")
        rt.cudaMemset.argtypes = [C.c_void_p, C.c_int, C.c_size_t]
        rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
        _RT = rt
    return _RT


def arena(g):
    """(base, bytes) of g's tensor arena. PlanArena puts its largest tensor at offset 0, so the base
    is the lowest address of a placed arena tensor; every placed tensor must lie inside."""
    placed = [t for t in range(g.num_tensors()) if g.in_arena(t) and g.data_ptr(t)]
    base, n = min(g.data_ptr(t) for t in placed), g.arena_bytes()
    for t in placed:
        assert base <= g.data_ptr(t) and g.data_ptr(t) + g.nbytes(t) <= base + n, (t, base, n)
    return base, n


def fill(g, byte):
    base, n = arena(g)
    rt = cudart()
    g.synchronize()
    assert rt.cudaMemset(C.c_void_p(base), byte, C.c_size_t(n)) == 0
    assert rt.cudaDeviceSynchronize() == 0
    g.synchronize()


def snapshot(g):
    """A device copy of the whole arena, and its base address."""
    import torch
    base, n = arena(g)
    g.synchronize()
    s = torch.empty(n, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    assert cudart().cudaMemcpy(C.c_void_p(s.data_ptr()), C.c_void_p(base), C.c_size_t(n), 3) == 0
    assert cudart().cudaDeviceSynchronize() == 0
    return base, s


def written(g):
    """(node, tensor) for every tensor a node writes, each under the first node that writes it."""
    seen, out = set(), []
    for i in range(g.num_nodes()):
        for t in g.node_outputs(i):
            if t >= 0 and t not in seen:
                seen.add(t)
                out.append((i, t))
    return out


def stray_write(g, snap, byte):
    """None, or where a node wrote arena bytes that belong to no tensor: past a tensor and the 64
    bytes of slack PlanArena leaves behind it. With every tensor kept no two tensors share bytes, so
    after a run on an arena filled with `byte` those bytes must still hold it."""
    import torch
    base, s = snap
    owned = torch.zeros(s.numel(), dtype=torch.bool, device=s.device)
    ends = []
    for t in range(g.num_tensors()):
        if g.in_arena(t) and g.data_ptr(t):
            o = g.data_ptr(t) - base
            owned[o:o + g.nbytes(t) + 64] = True
            ends.append((o + g.nbytes(t), t))
    bad = ((s != byte) & ~owned).nonzero().flatten()
    if len(bad) == 0:
        return None
    at = int(bad[0])
    end, t = max((e, t) for e, t in ends if e <= at)
    writers = [g.node_name(i) for i, u in written(g) if u == t]
    return (f"{len(bad)} bytes outside every tensor changed, the first {at - end} bytes past the end "
            f"of tensor {t} {g.shape(t)} {np.dtype(g.dtype(t))} (written by {writers or 'the host'})")


def first_difference(g, want, got):
    """None, or the first node (execution order) with an output whose bytes differ between two
    snapshots of the same graph's arena."""
    (base, a), (base2, b) = want, got
    assert base == base2
    for i, t in written(g):
        o, n = g.data_ptr(t) - base, g.nbytes(t)
        x, y = a[o:o + n], b[o:o + n]
        if bool((x == y).all()):
            continue
        bad = (x != y).nonzero().flatten()
        dt = np.dtype(g.dtype(t))
        k = int(bad[0]) // dt.itemsize
        av = x[k * dt.itemsize:(k + 1) * dt.itemsize].cpu().numpy().view(dt)[0]
        bv = y[k * dt.itemsize:(k + 1) * dt.itemsize].cpu().numpy().view(dt)[0]
        ins = [g.shape(s) for s in g.node_io(i)[0] if s >= 0]
        return (f"node {i} {g.node_name(i)} {ins} -> tensor {t} {g.shape(t)} {dt}: {len(bad)} of {n} "
                f"bytes differ, first at element {np.unravel_index(k, g.shape(t))} "
                f"(anchor {av!r}, here {bv!r})")
    return None


# ------------------------------------------------------------------ running the variants
UNPAIRED = ("fuse_binary_bases", "fuse_dense_blocks", "fuse_residual_blocks", "fuse_spatial_scales",
            "fuse_float_glue", "fuse_grouped_conv_affine", "fuse_quantized_activations",
            "fuse_pooled_signs", "fuse_channel_gates", "fuse_activation_chains")


def graph(blob, shape, fuse, preserve):
    """fuse: True (fuse_all), False, or "unpaired" (fuse_all's passes but fuse_residual_pairs)."""
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    if fuse == "unpaired":
        assert sum(getattr(g, p)() for p in UNPAIRED) > 0
    elif fuse:
        assert g.fuse_all() > 0
    g.preserve_all_tensors(preserve)
    g.resize_input(g.inputs()[0], shape)
    g.allocate_tensors()
    return g


def put(g, x):
    g.write(g.inputs()[0], x)
    g.invoke()
    return [g.read(t) for t in g.outputs()]


def run(g, x, byte):
    fill(g, byte)
    return put(g, x)


def same(a, b):
    return all(p.dtype == q.dtype and p.shape == q.shape and
               np.array_equal(p.view(np.uint8), q.view(np.uint8)) for p, q in zip(a, b))


def describe(want, got):
    for k, (p, q) in enumerate(zip(want, got)):
        bits = f"u{p.dtype.itemsize}"
        bad = np.argwhere(p.view(bits) != q.view(bits))
        if len(bad):
            first = tuple(bad[0])
            return (f"output {k}: {len(bad)} of {p.size} elements differ, first at {first} "
                    f"(anchor {p[first]!r}, here {q[first]!r})")
    return "outputs equal"


def images(shape, input_type, seed):
    x = np.random.default_rng(seed).standard_normal(shape, dtype=np.float32)
    return zoo.quantize_images(x) if input_type == "int8" else x


def check_arena_independence(blob, shape, input_type, fuse=True):
    """Runs every variant of the module docstring; returns the list of failures."""
    xs = [images(shape, input_type, 100 + k) for k in range(3)]
    fails = []

    # anchors, then P-A / P-B on the same layout
    g = graph(blob, shape, fuse, preserve=True)
    want = [run(g, x, 0) for x in xs]
    if same(want[1], want[2]):
        fails.append("the anchors of x1 and x2 are equal: the replay check needs them apart")
    anchor = (run(g, xs[0], 0), snapshot(g))
    if not same(anchor[0], want[0]):
        fails.append(f"anchor run twice: {describe(want[0], anchor[0])}")
    for tag, byte in POISON:
        out = run(g, xs[0], byte)
        snap = snapshot(g)
        d = first_difference(g, anchor[1], snap)
        if d is not None:
            fails.append(f"P-{tag}: {d}")
        elif not same(out, want[0]):
            fails.append(f"P-{tag}: {describe(want[0], out)}")
        d = stray_write(g, snap, byte)
        if d is not None:
            fails.append(f"P-{tag}: {d}")
        del snap
    del anchor
    g.close()

    # shrunk: planned and run at twice the batch first, then re-planned in the same arena
    big = (2 * shape[0],) + tuple(shape[1:])
    g = graph(blob, big, fuse, preserve=False)
    put(g, images(big, input_type, 99))
    bytes_big = g.arena_bytes()
    g.resize_input(g.inputs()[0], shape)
    g.allocate_tensors()
    assert g.arena_bytes() == bytes_big
    out = put(g, xs[0])
    if not same(out, want[0]):
        fails.append(f"shrunk: {describe(want[0], out)}")

    # R-A / R-B on the reused layout
    for tag, byte in POISON:
        out = run(g, xs[0], byte)
        if not same(out, want[0]):
            fails.append(f"R-{tag}: {describe(want[0], out)}")

    # replay of new inputs: the eager pass, the capture on x0, then x1 and x2 on poisoned arenas
    g.enable_cuda_graph(True)
    put(g, xs[0])
    out = put(g, xs[0])
    if not same(out, want[0]):
        fails.append(f"capture on x0: {describe(want[0], out)}")
    replayed = []
    for (tag, byte), k in zip(POISON, (1, 2)):
        out = run(g, xs[k], byte)
        replayed.append(out)
        if not same(out, want[k]):
            fails.append(f"replay of x{k} on arena {tag}: {describe(want[k], out)}")
    if same(replayed[0], replayed[1]):
        fails.append("the replays of x1 and x2 gave the same outputs")
    g.close()
    return fails


# ------------------------------------------------------------------ CPU
def test_every_zoo_family_is_covered():
    assert set(zoo.MODELS) <= set(FAMILIES) | set(dict(BENCHMARKED))
    makers = {make for make, _ in FAMILIES.values()} | {zoo.MODELS[n] for n, _ in BENCHMARKED}
    for name in ("abcnet", "xnornetpp", "binary_mobilenet", "meliusnet", "realtobinarynet"):
        assert getattr(zoo, name) in makers
    assert {make for make, _ in UNFUSED.values()} >= {zoo.quicknet, zoo.birealnet18, zoo.reactnet_a,
                                                      zoo.abcnet, zoo.xnornetpp, zoo.dorefanet}


def test_unpaired_passes_are_fuse_all_but_the_pairs():
    blob = zoo.quicknet(batch=1, image=224, seed=1, input_type="int8")
    names = []
    for passes in (("fuse_all",), UNPAIRED + ("fuse_residual_pairs",), UNPAIRED):
        g = H.HostGraph.from_tflite(blob, device_arena=True)
        for p in passes:
            getattr(g, p)()
        names.append([g.node_name(i) for i in range(g.num_nodes())])
        g.close()
    assert names[0] == names[1] and names[2] != names[1]
    assert not any(n.count("LceBconv2d") > 1 for n in names[2])


def test_node_outputs_lists_every_output():
    g = H.HostGraph.from_tflite(zoo.quicknet(batch=1, image=224, seed=1, input_type="int8"),
                                device_arena=True)
    g.fuse_all()
    counts = set()
    for i in range(g.num_nodes()):
        outs = g.node_outputs(i)
        assert outs[0] == g.node_io(i)[1][0]
        assert len(outs) == (2 if g.node_name(i).endswith("+LceQuantize") else 1), g.node_name(i)
        counts.add(len(outs))
    assert counts == {1, 2}
    g.close()


def test_in_arena_tells_the_constants_apart():
    blob = zoo.dorefanet(batch=1, image=64, seed=1)
    m = R.parse(blob)
    g = H.HostGraph.from_tflite(blob, device_arena=True)
    assert g.num_tensors() == len(m["tensors"])
    for t, e in enumerate(m["tensors"]):
        assert g.in_arena(t) == (e["data"] is None), (t, e["name"])
    # the DoReFaNet pass adds a bit-plane map (arena) and per-layer constants (not)
    g.fuse_all()
    added = range(len(m["tensors"]), g.num_tensors())
    kinds = {g.in_arena(t) for t in added}
    assert kinds == {True, False}
    g.close()


# ------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name,batch", BENCHMARKED)
def test_gpu_benchmarked_graph_does_not_depend_on_the_arena(name, batch):
    """The int8 graphs bench.py times, at its shapes."""
    blob = zoo.MODELS[name](batch=1, seed=0, input_type="int8")
    fails = check_arena_independence(blob, (batch, 224, 224, 3), "int8")
    assert not fails, f"{name} batch {batch}:\n" + "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(FAMILIES))
def test_gpu_family_does_not_depend_on_the_arena(case):
    make, kw = FAMILIES[case]
    blob = make(batch=1, seed=0, image=224, **kw)
    fails = check_arena_independence(blob, (BATCH, 224, 224, 3), "float32")
    assert not fails, f"{case}:\n" + "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("passes", ["unfused", "unpaired"])
def test_gpu_quicknet_at_the_benchmark_batch_without_fusion_or_pairs(passes):
    """QuickNet at bench.py's batch with its float builtins and stand-alone LCE ops, and fused
    except for the residual pairs."""
    blob = zoo.quicknet(batch=1, seed=0, input_type="int8")
    fails = check_arena_independence(blob, (256, 224, 224, 3), "int8",
                                     fuse=False if passes == "unfused" else "unpaired")
    assert not fails, f"quicknet {passes}:\n" + "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("name,image", [("quicknet", 100), ("reactnet_a", 160)])
def test_gpu_odd_image_does_not_depend_on_the_arena(name, image):
    """An odd batch, and for QuickNet an odd image: a partial pixel tile at every layer (ReActNet-A's
    shortcuts need the image to halve evenly five times)."""
    blob = zoo.MODELS[name](batch=1, seed=0, image=image, input_type="int8")
    fails = check_arena_independence(blob, (7, image, image, 3), "int8")
    assert not fails, f"{name} {image}x{image}:\n" + "\n".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(UNFUSED))
def test_gpu_unfused_graph_does_not_depend_on_the_arena(case):
    make, kw = UNFUSED[case]
    blob = make(batch=1, seed=0, image=224, **kw)
    fails = check_arena_independence(blob, (BATCH, 224, 224, 3), "float32", fuse=False)
    assert not fails, f"{case} unfused:\n" + "\n".join(fails)
