"""Python front-end with the reference's ``Interpreter`` interface
(LCE/tflite/python/interpreter.py:6-58, interpreter_base.py:36-95): same constructor
flags and properties, ``predict`` on numpy arrays -- but TRUE batching: the reference
feeds one sample at a time (interpreter_base.py:10-27 yields batch-1 inputs because
the converter pins the batch to 1, LCE/mlir/transforms/set_batch_size.cc:9-22); here
``predict`` resizes the input tensors to the whole (mini-)batch, re-runs every op's
``prepare`` -- what TFLite's ResizeInputTensor + AllocateTensors does -- and runs the
graph once per mini-batch on the device, replaying a captured CUDA graph.

``devices=[...]`` shards every mini-batch over several GPUs of the box from ONE process: the
model bytes are loaded onto each device once (constants are replicated; there is no transfer
between devices afterwards), image i of a mini-batch goes to device i * D // n, all devices run
concurrently on their own streams, and the outputs come back in input order. (bench.py's
multi-GPU runs use one process per GPU instead, as the measurement contract asks.)
"""
from __future__ import annotations

import ctypes as C
from typing import Iterator, List, Optional, Sequence, Union

import numpy as np

from . import host as _host

Data = Union[np.ndarray, List[np.ndarray]]

__all__ = ["Interpreter"]


class Interpreter:
    def __init__(self, flatbuffer_model: bytes, num_threads: int = 1,
                 use_reference_bconv: bool = False, use_indirect_bgemm: bool = False,
                 use_xnnpack: bool = False, batch_size: Optional[int] = None,
                 use_cuda_graph: bool = True, fuse: bool = True,
                 devices: Optional[Sequence[int]] = None):
        """flatbuffer_model: a serialized LCE model (`.tflite` bytes).
        num_threads / use_xnnpack: accepted for interface parity; the device path has no CPU
        threads to configure. use_reference_bconv / use_indirect_bgemm: as in the reference
        (interpreter.py:40-58 -> RegisterLCECustomOps), they choose the registration LceBconv2d
        resolves to: Register_BCONV_2D_REF (the reference kernel's validation rules and, under
        zero padding, its integer result) or Register_BCONV_2D_OPT_INDIRECT_BGEMM / the default
        (the optimised kernels' rules and their float zero-padding correction).
        batch_size: mini-batch used by predict (default: all). fuse: apply the graph-level fusions
        (residual-block tail into LceBconv2d's epilogue, max-pool + blur-pool); the outputs are
        bit-identical either way, with two exceptions: a 2-bit-activation layer (DoReFaNet's quantiser
        in front of a float CONV_2D or FULLY_CONNECTED with +-alpha weights) runs fused as an exact
        integer binary convolution over bit planes, whose result is the real value rounded twice,
        where the float layer rounds after each of its K terms; the two differ by up to about
        K * 2^-24 * sum |a| |w| per output, which can flip a level of the next quantiser at a near-tie
        (HostGraph.fuse_quantized_activations). And a binary dense layer (LceDequantize ->
        FULLY_CONNECTED with +-alpha_o weights) whose alpha_o are not all powers of two (XNOR-Net's
        scaled or BatchNorm-folded kernels) runs fused as fl(fl(alpha_o * D) + bias) with D the exact
        +-1 dot product, the real value rounded twice, where the float layer rounds after each of its K
        terms; the two differ by up to about K * 2^-24 * K * alpha_o per output (sum |a| |w| = K *
        alpha_o), which can flip the next sign at a near-tie (HostGraph.fuse_binary_fully_connected);
        with every alpha_o a power of two (+-1.0 kernels included) it is bit-identical. devices: CUDA
        device indices to shard mini-batches over (default: the current device only)."""
        if use_reference_bconv and use_indirect_bgemm:
            import warnings
            warnings.warn("'use_reference_bconv' and `use_indirect_bgemm` are both set to true. "
                          "use_indirect_bgemm==true will have no effect.")
        self.devices = list(devices) if devices is not None else [None]
        if not self.devices:
            raise ValueError("devices must name at least one CUDA device")
        self._graphs = []
        self.fused_nodes_removed = 0
        try:
            for d in self.devices:
                with _on_device(d):
                    g = _host.HostGraph.from_tflite(bytes(flatbuffer_model), device_arena=True,
                                                    use_reference_bconv=use_reference_bconv,
                                                    use_indirect_bgemm=use_indirect_bgemm)
                    self._graphs.append(g)
                    self.fused_nodes_removed = g.fuse_all() if fuse else 0
                    g.allocate_tensors()
                    if use_cuda_graph:
                        g.enable_cuda_graph(True)
        except _host.HostError as e:
            for g in self._graphs:
                g.close()
            raise ValueError(f"Could not build the interpreter: {e}") from None
        self._g = self._graphs[0]
        self.num_threads = num_threads
        self.batch_size = batch_size
        self._cur_batch = [None] * len(self._graphs)

    # ---- properties, as in interpreter_base.py:40-78 ----
    def _types(self, idx):
        return [np.dtype(self._g.dtype(t)).type for t in idx]

    @property
    def input_types(self) -> list:
        return self._types(self._g.inputs())

    @property
    def input_shapes(self) -> list:
        return [self._g.shape(t) for t in self._g.inputs()]

    @property
    def input_scales(self) -> list:
        return [self._scale(t) for t in self._g.inputs()]

    @property
    def input_zero_points(self) -> list:
        return [self._zp(t) for t in self._g.inputs()]

    @property
    def output_types(self) -> list:
        return self._types(self._g.outputs())

    @property
    def output_shapes(self) -> list:
        return [self._g.shape(t) for t in self._g.outputs()]

    @property
    def output_scales(self) -> list:
        return [self._scale(t) for t in self._g.outputs()]

    @property
    def output_zero_points(self) -> list:
        return [self._zp(t) for t in self._g.outputs()]

    def _scale(self, t):
        s = _host.lib().lce_host_tensor_scale(self._g._g, t)
        return float(s) if s != 0.0 else None

    def _zp(self, t):
        s = _host.lib().lce_host_tensor_scale(self._g._g, t)
        return int(_host.lib().lce_host_tensor_zero_point(self._g._g, t)) if s != 0.0 else None

    # ---- execution ----
    def _set_batch(self, gi, n):
        if n == self._cur_batch[gi]:
            return
        g = self._graphs[gi]
        for t in g.inputs():
            shape = list(g.shape(t))
            shape[0] = n
            g.resize_input(t, shape)
        g.allocate_tensors()
        self._cur_batch[gi] = n

    def _run(self, inputs: List[np.ndarray]) -> List[np.ndarray]:
        n = inputs[0].shape[0]
        D = len(self._graphs)
        # image i -> device i * D // n: contiguous, ordered shards (compute_engine_b200.parallel.shard_range)
        bounds = [(k * n) // D for k in range(D + 1)]
        active = [k for k in range(D) if bounds[k + 1] > bounds[k]]
        for k in active:                       # launch everywhere first: the devices overlap
            lo, hi = bounds[k], bounds[k + 1]
            with _on_device(self.devices[k]):
                g = self._graphs[k]
                self._set_batch(k, hi - lo)
                for t, a in zip(g.inputs(), inputs):
                    want = g.shape(t)
                    part = a[lo:hi]
                    if tuple(part.shape) != tuple(want):
                        raise ValueError(f"input shape {part.shape} does not match {want}")
                    g.write(t, part)
                g.invoke()
        parts = []
        for k in active:                       # then gather in input order
            with _on_device(self.devices[k]):
                g = self._graphs[k]
                parts.append([g.read(t) for t in g.outputs()])
        return [np.concatenate(col) for col in zip(*parts)]

    def predict(self, x: Union[Data, Iterator[Data]], verbose: int = 0) -> Data:
        """Generates output predictions for the input samples (leading dim = samples)."""
        if isinstance(x, np.ndarray):
            inputs = [x]
        elif isinstance(x, list):
            inputs = list(x)
        elif hasattr(x, "__next__") and hasattr(x, "__iter__"):
            items = list(x)
            if items and isinstance(items[0], np.ndarray):
                inputs = [np.stack(items)]
            else:
                inputs = [np.stack(col) for col in zip(*items)]
        else:
            raise ValueError(
                "Expected either a list of inputs or a Numpy array with implicit initial "
                f"batch dimension or an iterator yielding one of the above. Received: {x}")
        n = inputs[0].shape[0]
        bs = self.batch_size or n
        chunks = []
        for lo in range(0, n, bs):
            chunks.append(self._run([a[lo:lo + bs] for a in inputs]))
        outputs = [np.concatenate(parts) for parts in zip(*chunks)]
        if len(self._g.outputs()) == 1:
            return outputs[0]
        return outputs

    # device-resident API used by bench.py: no host copies
    @property
    def graph(self):
        return self._g

    def close(self):
        for d, g in zip(self.devices, self._graphs):
            with _on_device(d):
                g.close()


class _on_device:
    """Make CUDA device `index` current for the duration of the block (None: leave it alone)."""

    def __init__(self, index):
        self.index, self.prev = index, None

    def __enter__(self):
        if self.index is not None:
            self.prev = _host.get_device()
            _host.set_device(self.index)

    def __exit__(self, *exc):
        if self.index is not None and self.prev is not None and self.prev >= 0:
            _host.set_device(self.prev)
        return False
