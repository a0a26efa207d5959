"""Execution plan: the flat op list the CUDA engine (csrc/engine.cu) runs.

A plan is what `lowering.lower()` makes out of one of the reference's .onnx files:
  * buffers  — NHWC activations in HBM (float32, or uint8 for the network input),
               sized per sample; the engine allocates them for `max_batch`.
  * views    — (buffer, channel offset, channel stride, C, H, W).  Concat, Slice and
               the ShuffleNetV2 channel shuffle never move data: producers write
               through a view straight into the consumer's buffer.
  * ops      — fused kernels (conv+bias+act+residual, depthwise, decode, ...).
  * weights  — one float32 blob; ops carry offsets into it.

`Plan.serialize()` produces the int32 words + float blob handed through the C-ABI
(include/skps_b200.h: skps_engine_create).
"""
import numpy as np

# ---- op types (keep in sync with csrc/plan.h) ------------------------------------
OP_CONV = 1           # dense conv (any k/stride/dilation), +bias +act +residual, optional per-(n,cin) input scale
OP_DWCONV = 2         # depthwise conv +bias +act
OP_MAXPOOL2 = 3       # 2x2 stride 2, ceil_mode
OP_RESIZE_NEAREST = 4  # asymmetric/floor nearest to the output view's H,W
OP_UPSAMPLE_BILINEAR2X = 5  # half_pixel bilinear x2
OP_COPY = 6           # channel-view copy
OP_GAP = 7            # global average pool -> (N,1,1,C)
OP_AFFINE_ACT = 8     # per-channel x*s+t then act (explicit BatchNormalization)
OP_SCSE = 9           # x*cse[n,c] + x*sse[n,h,w]
OP_DET_DECODE = 10    # yolov5-face head decode -> (N,rows,16)
OP_HM_DECODE = 11     # heat-map argmax + offset decode -> (N,196),(N,98)
OP_SCALE_CH = 12      # x * gate[n,c]  (squeeze-excite applied ahead of a tensor-core conv)
OP_UPCAT_DW = 13      # depthwise3x3(concat(bilinear_x2(low), skip)) without materialising the up-sampled tensor
OP_ADDN = 14          # act(sum of up to 4 inputs), each optionally nearest-upsampled by 2^k (HRNet fuse layers)
OP_SE_FC = 15         # squeeze-excite gate: per-tile channel sums -> mean -> 1x1 -> act -> 1x1 -> act  (N,1,1,C)
OP_DWPW = 16          # act(conv1x1(dw_act(depthwise3x3(x | concat(bilinear_x2(low), x))))): the depthwise output lives in smem only (csrc/conv_xf.cu)

OP_GAP_SSE = 18       # scSE front end in one pass over x: per-tile channel sums (-> OP_SE_FC = cSE) and the sSE map act(x . w + b)

OP_STEM_BLOCK = 17    # uint8 input -> stem 3x3 s2 -> dw3x3 -> 1x1 16->16 (+shortcut) -> 1x1 16->E -> dw3x3 s2, one kernel (csrc/stem_block.cu)

OP_NAMES = {v: k for k, v in dict(globals()).items() if k.startswith("OP_")}

ACT_NONE, ACT_RELU, ACT_HSWISH, ACT_SILU, ACT_SIGMOID, ACT_HSIGMOID = range(6)

DT_F32, DT_U8, DT_SPLIT16 = 0, 1, 2     # SPLIT16: float16 hi plane + float16 lo plane, v = hi + lo

OP_WORDS = 64
VIEW_WORDS = 6
BUF_WORDS = 4


class Buf:
    def __init__(self, idx, C, H, W, dtype=DT_F32, name=""):
        self.idx, self.C, self.H, self.W, self.dtype, self.name = idx, C, H, W, dtype, name

    @property
    def elems(self):
        return self.C * self.H * self.W


class View:
    """Channel window onto a buffer.  Logical channel j lives at c_off + j*c_stride."""

    def __init__(self, buf, c_off, c_stride, C):
        self.buf, self.c_off, self.c_stride, self.C = buf, c_off, c_stride, C

    @property
    def H(self):
        return self.buf.H

    @property
    def W(self):
        return self.buf.W

    def sub(self, off, C, stride=1):
        return View(self.buf, self.c_off + off * self.c_stride, self.c_stride * stride, C)

    def words(self):
        return [self.buf.idx, self.c_off, self.c_stride, self.C, self.buf.H, self.buf.W]

    def __repr__(self):
        return "V(b%d[%d:+%d*%d] %dx%dx%d)" % (self.buf.idx, self.c_off, self.C, self.c_stride,
                                                self.buf.H, self.buf.W, self.buf.C)


_NOVIEW = [-1, 0, 1, 0, 0, 0]


class Op:
    def __init__(self, type, ins, outs, act=ACT_NONE, k=(1, 1), s=(1, 1), p=(0, 0), d=(1, 1),
                 w=None, b=None, flags=0, ints=(), floats=(), name=""):
        self.type, self.ins, self.outs, self.act = type, list(ins), list(outs), act
        self.k, self.s, self.p, self.d = k, s, p, d
        self.w, self.b = w, b                # numpy float32 arrays (already in kernel layout) or None
        self.flags, self.ints, self.floats, self.name = flags, list(ints), list(floats), name
        self.w_off = self.b_off = -1
        self.w2 = None                       # FLAG_TC: lo-plane weight matrix; its blob offset goes to ints[2]
        self.extra = None                    # op-specific float32 table; its blob offset goes to ints[extra_slot]
        self.extra_slot = 0
        self.extra2 = None                   # second float32 table; its blob offset goes to ints2[0]
        self.ints2 = [0, 0]

    def __repr__(self):
        return "%s %s -> %s act=%d k=%s s=%s d=%s %s" % (OP_NAMES[self.type], self.ins, self.outs,
                                                         self.act, self.k, self.s, self.d, self.name)


FLAG_IN_U8 = 1        # conv reads uint8 input and divides by 255 (first layer)
FLAG_TC = 2           # conv runs on the tensor-core path: w = hi matrix, w2 = lo matrix (float16 bytes in the blob)
FLAG_RES_FIRST = 4    # conv: act(conv + bias + residual) (ResNet/HRNet blocks) instead of act(conv + bias) + residual
FLAG_MMA = 16         # 3x3 conv with few channels on the halo-tile mma.sync kernel (csrc/conv_mma.cu): w = packed fp16 hi/lo
FLAG_XF = 32          # tensor-core 1x1 conv whose input is scaled by ins[2] = gate[n,c] inside the kernel (csrc/conv_xf.cu, XF_SCALE)
FLAG_HM_PART = 64     # heat-map head conv writes per-tile (max, first arg-max) rows to outs[1] instead of the map; OP_HM_DECODE reads them from ins[2]
FLAG_GAP_PARTIAL = 8  # depthwise conv also writes per-tile channel sums of its output to outs[1] ([tiles][C] per sample)
DW_TILE_W = 16


def dw_tile_rows(k, s):
    """Output rows per tile of csrc/dw_tma.cu (rows of the per-tile channel-sum buffer): 16 for 5x5 stride-1 layers, else 8."""
    return 16 if (k == 5 and s == 1) else 8


class Plan:
    def __init__(self, name):
        self.name = name
        self.bufs = []
        self.ops = []
        self.input = None        # View of the network input (uint8 NHWC)
        self.outputs = []        # Views of the outputs
        self.macs = 0            # conv MACs per sample (algorithmic work)

    def new_buf(self, C, H, W, dtype=DT_F32, name=""):
        b = Buf(len(self.bufs), C, H, W, dtype, name)
        self.bufs.append(b)
        return b

    # ------------------------------------------------------------------ serialization
    def pack_weights(self):
        """Concatenate all op weights/biases into one float32 blob (16-byte aligned pieces)."""
        parts = []
        off = 0

        def put(a):
            nonlocal off
            a = np.ascontiguousarray(a, dtype=np.float32).reshape(-1)
            pad = (-a.size) % 4
            start = off
            parts.append(a)
            if pad:
                parts.append(np.zeros(pad, np.float32))
            off += a.size + pad
            return start
        def put_raw(a):
            # float16 matrices travel as raw bytes inside the float32 blob
            raw = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
            pad = (-raw.size) % 16
            if pad:
                raw = np.concatenate([raw, np.zeros(pad, np.uint8)])
            return put(raw.view(np.float32))
        for op in self.ops:
            if op.flags & FLAG_MMA:
                op.w_off = put_raw(op.w)
            elif op.flags & FLAG_TC:
                op.w_off = put_raw(op.w)
                lo_off = put_raw(op.w2)
                op.ints = list(op.ints[:2]) + [lo_off] + list(op.ints[3:])
            else:
                op.w_off = put(op.w) if op.w is not None else -1
            op.b_off = put(op.b) if op.b is not None else -1
            if op.extra is not None:
                ints = list(op.ints) + [0] * (4 - len(op.ints))
                ints[op.extra_slot] = put(op.extra)
                op.ints = ints
            if op.extra2 is not None:
                op.ints2 = [put(op.extra2), 0]
        # tail slack: kernels that read weight rows in whole 16-byte / 64-channel pieces never run past the allocation
        parts.append(np.zeros(256, np.float32))
        return np.concatenate(parts)

    def serialize(self):
        blob = self.pack_weights()
        bw = []
        for b in self.bufs:
            bw += [b.C, b.H, b.W, b.dtype]
        ow = []
        for op in self.ops:
            w = [op.type, op.act]
            for i in range(3):
                w += op.ins[i].words() if i < len(op.ins) and op.ins[i] is not None else _NOVIEW
            for i in range(2):
                w += op.outs[i].words() if i < len(op.outs) else _NOVIEW
            w += [op.k[0], op.k[1], op.s[0], op.s[1], op.p[0], op.p[1], op.d[0], op.d[1]]
            w += [op.w_off, op.b_off, op.flags]
            ints = list(op.ints) + [0] * (4 - len(op.ints))
            w += ints[:4]
            fl = np.asarray(list(op.floats) + [0.0] * (8 - len(op.floats)), np.float32)[:8]
            w += fl.view(np.int32).tolist()
            w += op.ins[3].words() if len(op.ins) > 3 and op.ins[3] is not None else _NOVIEW     # 4th input (OP_ADDN)
            w += list(op.ints2)
            assert len(w) <= OP_WORDS, len(w)
            w += [0] * (OP_WORDS - len(w))
            ow += w
        header = np.array([0x534B5053, 1, len(self.bufs), len(self.ops),
                           self.input.buf.idx, len(self.outputs)] +
                          [v.buf.idx for v in self.outputs] + [0] * (2 - len(self.outputs)), np.int32)
        words = np.concatenate([header, np.array(bw, np.int32), np.array(ow, np.int32)])
        return words, blob

    def bytes_per_sample(self, op):
        """Activation bytes one sample moves through `op` (inputs + outputs), for traffic estimates."""
        tot = 0
        for v in list(op.ins) + list(op.outs):
            if v is not None:
                tot += v.C * v.buf.H * v.buf.W * (1 if v.buf.dtype == DT_U8 else 4)
        return tot


# ---- tensor-core (wgmma) convolution support ---------------------------------------------------
TC_BK = 64            # channels per k-block (csrc/conv_tc.cu)


def tc_tiling(cout):
    """Split Cout into n_tiles equal UMMA-N tiles (multiple of 16, <= 256)."""
    c16 = -(-cout // 16) * 16
    n_tiles = -(-c16 // 256)
    n_tile = -(-(-(-c16 // n_tiles)) // 16) * 16
    return n_tile, n_tiles


def split_fp16(a):
    """v -> (hi, lo) float16 with v ~= hi + lo (22 significant bits)."""
    a = np.asarray(a, dtype=np.float32)
    hi = a.astype(np.float16)
    lo = (a - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def pack_tc_weights(w_ockk, n_tile, n_tiles):
    """[Cout][kh][kw][Cin] float32 -> (hi, lo, out_scale): float16 matrices (n_tiles*n_tile,
    taps*cchunks*64) with K index = (tap*cchunks + chunk)*64 + ci_in_chunk, zero padded in both
    dimensions.  The weights are pre-multiplied by an exact power of two so that the lo parts stay
    in float16's normal range; the kernel multiplies the accumulator by out_scale = 2^-s."""
    cout, kh, kw, cin = w_ockk.shape
    wmax = float(np.abs(w_ockk).max())
    s_exp = int(np.floor(np.log2(8192.0 / wmax))) if wmax > 0 else 0
    w_ockk = (w_ockk * np.float32(2.0 ** s_exp)).astype(np.float32)
    cch = -(-cin // TC_BK)
    rows = n_tile * n_tiles
    m = np.zeros((rows, kh * kw, cch * TC_BK), np.float32)
    m[:cout, :, :cin] = w_ockk.reshape(cout, kh * kw, cin)
    m = m.reshape(rows, kh * kw * cch * TC_BK)
    hi, lo = split_fp16(m)
    return hi, lo, float(2.0 ** (-s_exp))


def upcat_effective_weights(w9c):
    """Depthwise 3x3 over a bilinear x2 (half_pixel) up-sampled map == a 3x3 stencil on the LOW-res map whose
    weights depend only on the output pixel's row/column class.  w9c: [9][C] (ky*3+kx major) ->
    [4][4][3][3][C] float32 indexed (class_y, class_x, a, b): out[y][x] = bias + sum_ab W[cy][cx][a][b] *
    low[clamp(y//2 + a - 1)][clamp(x//2 + b - 1)].  Classes: 0 = first row/col (the conv's zero padding removes
    tap 0), 1 = even, 2 = odd, 3 = last row/col (tap 2 removed).  Per dimension U[2m] = .25 L[m-1] + .75 L[m],
    U[2m+1] = .75 L[m] + .25 L[m+1] with edge-clamped indices (model.py:176 F.interpolate(scale_factor=2,
    mode='bilinear'))."""
    E = np.array([[.75, .25, 0], [.25, .75, 0], [0, .75, .25]])
    O = np.array([[.25, .75, 0], [0, .75, .25], [0, .25, .75]])
    E0, O1 = E.copy(), O.copy()
    E0[0] = 0
    O1[2] = 0
    R = [E0, E, O, O1]
    w = np.asarray(w9c, np.float64).reshape(3, 3, -1)
    out = np.zeros((4, 4, 3, 3, w.shape[-1]))
    for cy in range(4):
        for cx in range(4):
            out[cy, cx] = np.einsum("ykc,ya,kb->abc", w, R[cy], R[cx])
    return np.ascontiguousarray(out.astype(np.float32))


def pack_upcat_class_weights(w9c):
    """upcat_effective_weights() re-laid for csrc/conv_xf.cu: [C/32][cy 4][cx 4][tap 9][32] float32, so that one 5-D TMA box
    (32 ch, 9 taps, 3 column classes, 3 row classes) fetches what one output tile of a 32-channel sub-chunk needs."""
    e = upcat_effective_weights(w9c)                       # [4][4][3][3][C]
    C = e.shape[-1]
    assert C % 32 == 0
    e = e.reshape(4, 4, 9, C // 32, 32).transpose(3, 0, 1, 2, 4)
    return np.ascontiguousarray(e, dtype=np.float32)


def pack_mma_weights(w_ockk):
    """[Cout][3][3][Cin] float32 -> (packed, out_scale): float16 array [tap][plane hi/lo][Cout][Cin] for
    csrc/conv_mma.cu, pre-multiplied by an exact power of two like pack_tc_weights."""
    cout, kh, kw, cin = w_ockk.shape
    wmax = float(np.abs(w_ockk).max())
    s_exp = int(np.floor(np.log2(8192.0 / wmax))) if wmax > 0 else 0
    w = (w_ockk * np.float32(2.0 ** s_exp)).astype(np.float32)
    hi, lo = split_fp16(w.transpose(1, 2, 0, 3).reshape(kh * kw, cout, cin))        # [tap][Cout][Cin]
    return np.ascontiguousarray(np.stack([hi, lo], axis=1)), float(2.0 ** (-s_exp))
