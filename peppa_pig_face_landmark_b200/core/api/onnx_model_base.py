"""ONNXEngine — same surface as the reference's wrapper around onnxruntime
(the reference's Skps/core/api/onnx_model_base.py:6-27): construct from a path to an .onnx
file, call with one NCHW float32 array, get the list of graph outputs back as numpy arrays.
Here the graph is lowered to a fused plan and executed by hand-written sm_90a kernels through
the C-ABI in include/skps_b200.h; PyTorch/numpy objects are only containers for memory.
"""
import ctypes as C

import numpy as np

from ... import lowering
from ... import runtime as rt
from ...onnx_loader import load_onnx


class ONNXEngine:
    def __init__(self, onnx_f, device="cuda", max_batch=1, use_tc=True):
        if "cuda" not in str(device):
            raise RuntimeError("ONNXEngine: this build executes on a CUDA device only (got device=%r)" % (device,))
        torch = rt.require_cuda()
        self.lib = rt.load_library()
        self.device = torch.device(device if ":" in str(device) else "cuda:%d" % torch.cuda.current_device())
        g = load_onnx(onnx_f)
        shp = g.input_shapes[g.inputs[0]]
        if len(shp) != 4 or shp[1] != 3 or min(shp[2:]) <= 0:
            raise ValueError("ONNXEngine: unsupported input shape %s in %s" % (shp, onnx_f))
        self.in_hw = (int(shp[2]), int(shp[3]))
        self.plan = lowering.lower(onnx_f, self.in_hw, name=str(onnx_f), use_tc=use_tc)
        words, blob = self.plan.serialize()
        self._words, self._blob = words, blob
        self.max_batch = int(max_batch)
        h = C.c_void_p()
        rt.check(self.lib.skps_engine_create(words.ctypes.data, words.size, blob.ctypes.data, blob.size,
                                             self.max_batch, self.device.index or 0, C.byref(h)))
        self.handle = h
        self.n_out = self.lib.skps_engine_num_outputs(h)
        self.out_elems = [self.lib.skps_engine_output_elems(h, i) for i in range(self.n_out)]
        self.stream = torch.cuda.Stream(device=self.device)
        self.macs_per_sample = self.plan.macs
        self.launches = self.lib.skps_engine_launches_per_forward(h)

    def __del__(self):
        h = getattr(self, "handle", None)
        if h is not None and h.value:
            self.lib.skps_engine_destroy(h)
            self.handle = None

    # ------------------------------------------------------------------ reference contract
    def __call__(self, data):
        """data: float32 (N,3,H,W) host array, N <= max_batch -> [ndarray, ...] (graph-output order)."""
        data = np.ascontiguousarray(data, dtype=np.float32)
        if data.ndim != 4 or data.shape[1] != 3 or tuple(data.shape[2:]) != self.in_hw:
            raise ValueError("ONNXEngine: got input %s, expected (N,3,%d,%d)" % (data.shape, *self.in_hw))
        n = data.shape[0]
        outs = [np.empty((n, e), np.float32) for e in self.out_elems]
        arr = (C.c_void_p * self.n_out)(*[o.ctypes.data for o in outs])
        rt.check(self.lib.skps_engine_forward_host_f32(self.handle, data.ctypes.data, n, arr,
                                                       self.stream.cuda_stream))
        return self._shape(outs, n)

    # ------------------------------------------------------------------ additive entry points
    def run_u8(self, nhwc_u8):
        """uint8 (N,H,W,3) host pixels (before the /255) -> list of outputs; H2D and D2H included."""
        x = np.ascontiguousarray(nhwc_u8, dtype=np.uint8)
        if x.ndim != 4 or x.shape[3] != 3 or tuple(x.shape[1:3]) != self.in_hw:
            raise ValueError("ONNXEngine.run_u8: got %s, expected (N,%d,%d,3)" % (x.shape, *self.in_hw))
        n = x.shape[0]
        outs = [np.empty((n, e), np.float32) for e in self.out_elems]
        arr = (C.c_void_p * self.n_out)(*[o.ctypes.data for o in outs])
        rt.check(self.lib.skps_engine_forward_host_u8(self.handle, x.ctypes.data, n, arr, self.stream.cuda_stream))
        return self._shape(outs, n)

    def stream_u8(self, batches):
        """Streaming variant of run_u8 for throughput: iterate over uint8 (N,H,W,3) host batches (pinned memory for
        full overlap) and yield their outputs in order.  Two batches are in flight: while one computes, the next
        one's pixels are copied to the GPU on a second stream; results land in pinned host buffers."""
        torch = rt.require_cuda()
        pin = [[torch.empty((self.max_batch, e), dtype=torch.float32).pin_memory() for e in self.out_elems]
               for _ in range(2)]
        arrs = [(C.c_void_p * self.n_out)(*[t.data_ptr() for t in pin[s]]) for s in range(2)]
        pending = []            # (slot, batch size, keep-alive input)

        def finish():
            slot, n, _keep = pending.pop(0)
            rt.check(self.lib.skps_engine_wait(self.handle, slot))
            return self._shape([t[:n].numpy().copy() for t in pin[slot]], n)

        i = 0
        for x in batches:
            x = np.ascontiguousarray(x, dtype=np.uint8)
            if x.ndim != 4 or x.shape[3] != 3 or tuple(x.shape[1:3]) != self.in_hw:
                raise ValueError("ONNXEngine.stream_u8: got %s, expected (N,%d,%d,3)" % (x.shape, *self.in_hw))
            if len(pending) == 2:
                yield finish()
            slot = i & 1
            rt.check(self.lib.skps_engine_submit_host_u8(self.handle, slot, x.ctypes.data, x.shape[0], arrs[slot]))
            pending.append((slot, x.shape[0], x))
            i += 1
        while pending:
            yield finish()

    def forward_device(self, x_u8, outputs=None, stream=None):
        """x_u8: torch uint8 CUDA tensor (N,H,W,3); outputs: optional list of float32 CUDA tensors.
        Asynchronous on `stream` (default: this engine's stream); returns the output tensors."""
        torch = rt.require_cuda()
        n = x_u8.shape[0]
        if outputs is None:
            outputs = [torch.empty((n, e), dtype=torch.float32, device=self.device) for e in self.out_elems]
        arr = (C.c_void_p * self.n_out)(*[o.data_ptr() for o in outputs])
        s = stream if stream is not None else self.stream
        rt.check(self.lib.skps_engine_forward(self.handle, x_u8.data_ptr(), n, arr, s.cuda_stream))
        return outputs

    def input_ptr(self):
        return self.lib.skps_engine_input_ptr(self.handle)

    def output_ptr(self, i):
        return self.lib.skps_engine_output_ptr(self.handle, i)

    def read_buffer(self, idx, batch):
        """Debug/parity: internal activation buffer idx as (batch,H,W,C) numpy."""
        h, w, c, dt = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
        rt.check(self.lib.skps_engine_buffer_dims(self.handle, idx, C.byref(h), C.byref(w), C.byref(c), C.byref(dt)))
        out = np.empty((batch, h.value, w.value, c.value), np.uint8 if dt.value == 1 else np.float32)
        rt.check(self.lib.skps_engine_read_buffer(self.handle, idx, batch, out.ctypes.data))
        return out

    def _shape(self, outs, n):
        if self.n_out == 1:                       # detector: (N, rows, 16), 15120 rows at 384x640
            return [outs[0].reshape(n, -1, 16)]
        return outs                               # landmark net: (N,196), (N,98)
