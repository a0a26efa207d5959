"""What FaceDetector, FaceLandmark and FaceAnaImages share around a call: the check of its frames, the check and
allocation of result buffers given as {name: (shape, dtype name)}, and the growable pinned staging that uploads a call's
descriptors and host pixels with one copy."""
import collections

from .device_frames import (FrameLayout, check_cuda_frame, check_host_frame, check_layout, check_rotate, is_cuda_tensor,
                            is_tensor, upright_hw)

MAX_SIDE = 1 << 20         # largest frame side a call takes: keeps every row pitch and crop coordinate in int32

Frames = collections.namedtuple("Frames", "frames shapes cuda turns", defaults=(None,))
Frames.__doc__ = """A call's checked frames: the frames (host frames C-contiguous), the FrameLayout of each (H, W, row
pitch and plane pitch in bytes, layout code, all as stored; host frames are packed BGR), whether they are CUDA tensors,
and the quarter turns clockwise that make each upright (check_rotate; Frames.upright gives the upright sizes)."""
Frames.upright = property(lambda self: [upright_hw(f.H, f.W, t) for f, t in zip(self.shapes, self.turns)])
Frames.turned = property(lambda self: any(self.turns))


def check_frames(frames, device, layout="bgr", rotate=0):
    """Frames of a call, checked before anything is enqueued: all HxWx3 uint8 BGR numpy arrays, or all torch.uint8 CUDA
    tensors on `device` in layout `layout` that check_cuda_frame takes, with sides in 1..MAX_SIDE, stored turned by
    rotate= (check_rotate: one angle for the call or one per frame).  ValueError otherwise, for a mix of the two, for a
    layout other than "bgr" and for a turn with host frames."""
    frames = list(frames)
    on_dev = [is_cuda_tensor(f) for f in frames]
    cuda = bool(on_dev) and all(on_dev)
    if any(on_dev) and not cuda:
        raise ValueError("one call takes either host frames or CUDA frames, got both (frames %s are CUDA)"
                         % [i for i, d in enumerate(on_dev) if d])
    check_layout(layout, cuda or not frames)
    turns = check_rotate(rotate, len(frames), cuda or not frames)
    if cuda:
        shapes = [check_cuda_frame(f, device, (MAX_SIDE, MAX_SIDE), layout) for f in frames]
    else:
        frames = [check_host_frame(f) for f in frames]
        shapes = [FrameLayout(f.shape[0], f.shape[1], 3 * f.shape[1], 0, 0) for f in frames]
    for H, W, *_ in shapes:
        if not (0 < H <= MAX_SIDE and 0 < W <= MAX_SIDE):
            raise ValueError("frame %dx%d: sides must be in 1..%d" % (H, W, MAX_SIDE))
    return Frames(frames, shapes, cuda, turns)


def new_buffers(fields, device):
    """{name: empty tensor on device} for fields {name: (shape, dtype name)}."""
    import torch
    return {k: torch.empty(shape, dtype=getattr(torch, dt), device=device) for k, (shape, dt) in fields.items()}


def check_out(out, fields, device, busy):
    """ValueError unless `out` can take a call whose results are fields {name: (shape for this call, dtype name)}: a dict
    with the same keys, each value a contiguous tensor of the field's dtype on `device` with the field's trailing
    dimensions and at least its leading one, sharing no tensor with the dicts in `busy` (the out= of the calls still in
    flight, None for calls without)."""
    import torch
    if not isinstance(out, dict) or set(out) != set(fields):
        raise ValueError("out: expected a dict with keys %s (see new_results())" % sorted(fields))
    for k, (shape, dt) in fields.items():
        t, dt = out[k], getattr(torch, dt)
        if (not isinstance(t, torch.Tensor) or t.dtype != dt or t.device != device or not t.is_contiguous()
                or t.dim() != len(shape) or tuple(t.shape[1:]) != shape[1:] or t.shape[0] < shape[0]):
            got = ("%s %s on %s" % (t.dtype, tuple(t.shape), t.device)) if is_tensor(t) else type(t).__name__
            raise ValueError("out[%r]: expected a contiguous %s tensor (>= %d%s) on %s, got %s"
                             % (k, dt, shape[0], "".join(", %d" % v for v in shape[1:]), device, got))
    taken = {t.data_ptr() for b in busy if b is not None for t in b.values()}
    if any(t.data_ptr() in taken for t in out.values()):
        raise ValueError("out: these buffers belong to a call still in flight; collect() it first")


def grow(t, n, make):
    """t when it holds n elements, else make(max(n, 2 * len(t)))."""
    if t is not None and t.shape[0] >= n:
        return t
    return make(max(n, 0 if t is None else 2 * t.shape[0], 1))


def pad16(n):
    return (n + 15) // 16 * 16


class Staging:
    """A pinned host byte buffer and a device byte buffer that grow with the calls, and the upload of one into the other
    on a copy stream of their own; `copied` is recorded there after every upload."""

    def __init__(self, device):
        import torch
        self.device = device
        self.copy = torch.cuda.Stream(device=device)
        self.copied = torch.cuda.Event()
        self.host = self.dev = None

    def reserve(self, nbytes, done):
        """Room for nbytes, once the last upload has left the pinned buffer: (host buffer as a numpy array, device
        address).  A buffer too small is replaced after `done` has been synchronised: the event after which nothing
        reads the old ones."""
        import torch
        if self.host is None or self.host.shape[0] < nbytes:
            done.synchronize()
            self.host = grow(self.host, nbytes, lambda k: torch.empty((k,), dtype=torch.uint8).pin_memory())
            self.dev = grow(self.dev, nbytes, lambda k: torch.empty((k,), dtype=torch.uint8, device=self.device))
        self.copied.synchronize()
        return self.host.numpy(), self.dev.data_ptr()

    def send(self, nbytes, after):
        """Uploads the first nbytes on the copy stream once the event `after` (the last read of the device buffer) has
        completed, and records `copied`; the stream that reads the upload waits for `copied`."""
        import torch
        if nbytes:
            self.copy.wait_event(after)
            with torch.cuda.stream(self.copy):
                self.dev[:nbytes].copy_(self.host[:nbytes], non_blocking=True)
        self.copied.record(self.copy)
