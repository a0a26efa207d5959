"""Op-isolated check of the CUDA engine: every plan op is re-run on the GPU from the buffers the previous ops left and
compared element by element with the same op evaluated in float64 (oracle.plan_interp.PlanInterp.step) from the engine's
OWN inputs, so an error in one kernel cannot hide in the drift that builds up layer by layer.  Split-fp16 buffers read
back as hi + lo, which is exactly the operand the next kernel uses.

Every output element must lie within a bound derived from the op's arithmetic (comments at each constant); data movement
must be bit-exact, the heat-map partial maxima and arg-max decode are checked as maxima within the bound.

Usage:  python tools/op_report.py detector H W | student | teacher     [batch]
"""
import os
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch                                       # noqa: E402
import torch.nn.functional as F                    # noqa: E402

from peppa_pig_face_landmark_b200 import plan as P  # noqa: E402
from oracle.plan_interp import PlanInterp, rd, split16_round, _act  # noqa: E402

KERNELS = {0: "misc", 1: "tc", 2: "tct", 3: "hm", 4: "mma", 5: "xf", 6: "simt", 7: "dw_tma", 8: "dw", 9: "upcat_tma",
           10: "upcat", 11: "stem_block", 12: "pw", 13: "fpw"}
K_MISC, K_TC, K_TCT, K_HM, K_MMA, K_XF, K_SIMT, K_DW_TMA, K_DW, K_UPCAT_TMA, K_UPCAT, K_STEM, K_PW, K_FPW = range(14)
# conv_fpw runs conv_xf's layers on the same A producer (csrc/xf_producer.h) and epilogue: the same tensor-core bound applies
TENSOR_CORE = (K_TC, K_TCT, K_HM, K_MMA, K_XF, K_PW, K_FPW)
PW_BM = 128                    # pixels per conv_pw tile: the tiles run over the flat (n, y, x) index of the batch

U = 2.0 ** -24                 # unit roundoff of float32 (round to nearest)


def gamma(n):
    """Higham's gamma_n = n u / (1 - n u): |fl(sum of n products) - exact| <= gamma_n * sum |x_i w_i| in any summation
    order, with or without FMA; a bias add and the conversion of the input count as one more rounding each (gamma_{K+2})."""
    return n * U / (1 - n * U)


# Tensor-core convolutions (conv_tc/tct/hm/mma/xf): operands are fp16 hi + lo pairs (22 significant bits, the lo*lo
# product dropped), accumulated in fp32 by the tensor core.  Per output:
#     (2^-19 + n_acc 2^-23) sum|x||w|  +  2^-23 sum|w|
# 2^-19 sum|x||w| is the operand error (~2^-22 relative per operand, both operands, the dropped lo*lo product) with
# a factor 2 to spare -- the form of test_conv_tc_gpu's element-wise test, which uses random (cancelling) data.
# n_acc 2^-23 sum|x||w| is the fp32 accumulate: the MMA adds its 16-product groups into the accumulator with at most
# one ulp (2^-23, truncation) of the running sum, whose magnitude never exceeds sum|x||w|, and there are
# n_acc = 3 ceil(K/16) such updates (hi*hi, hi*lo and lo*hi each).  Real activations do not cancel: on the student's
# ASPP 3x3 convs (K = 1440) interior elements reach 2x the first term alone, in conv_tc and conv_tct alike.
# 2^-23 sum|w| is the format's absolute floor: below ~2^-3 the lo plane is a float16 subnormal, so an operand is only
# good to 2^-25 absolute (times |w| summed; a factor 4 for the weight side and the accumulate).
TC_REL, TC_ABS, TC_ACC = 2.0 ** -19, 2.0 ** -23, 2.0 ** -23


def tc_rel(K):
    """Relative coefficient of the tensor-core bound for K products per output (see above)."""
    return TC_REL + 3 * (-(-K // 16)) * TC_ACC
# Rounding a result into the split-fp16 format: |v - (hi + lo)| <= 2^-11 * 2^-11 |v| (lo keeps 11 bits of v - hi), and
# 2^-25 absolute where lo is subnormal.
SPLIT_REL, SPLIT_ABS = 2.0 ** -22, 2.0 ** -25
# Lipschitz constants of the activations: a pre-activation error e moves the output by at most L * e.
#   relu 1;  h-swish x*clamp(x/6+1/2) has slope x/3 + 1/2 <= 3/2 on [-3, 3];  SiLU's slope peaks at 1.0998 (x ~ 2.4);
#   sigmoid 1/4;  hard-sigmoid 1/6.
LIP = {P.ACT_NONE: 1.0, P.ACT_RELU: 1.0, P.ACT_HSWISH: 1.5, P.ACT_SILU: 1.1, P.ACT_SIGMOID: 0.25, P.ACT_HSIGMOID: 1 / 6}
TINY = 2.0 ** -100             # absolute floor: SiLU/sigmoid of very negative inputs flush to 0 where e^x underflows


def act_eval(z, y, a):
    """Bound on the rounding of evaluating activation `a` in float32 at pre-activation z (y = exact act(z)).
    h-swish / hard-sigmoid: t = fl(fl(z * c) + 1/2) is off by u(|z|/6 + |t|) <= u(|z|/6 + 1), times |z| for the product,
    plus the product's own rounding: 2^-23 (|z| (|z|/6 + 1) + |y|) keeps a factor 2.  sigmoid: expf is good to 2 ulp, the
    add and the divide to 1/2 ulp each: 4u relative, SiLU one more product: 5u; 2^-21 = 8u covers both."""
    if a in (P.ACT_NONE, P.ACT_RELU):
        return torch.zeros_like(z)
    if a == P.ACT_HSWISH:
        return 2.0 ** -23 * (z.abs() * (z.abs() / 6 + 1) + y.abs())
    if a == P.ACT_HSIGMOID:
        return 2.0 ** -23 * (z.abs() / 6 + 1)
    return 2.0 ** -21 * y.abs() + TINY


def _chw(t):
    return t.permute(0, 3, 1, 2)


def _hwc(t):
    return t.permute(0, 2, 3, 1)


def _t(a):
    return torch.from_numpy(np.asarray(a)).double()


class OpCheck:
    """Result of one op: worst err/bound ratio and where it happened."""

    def __init__(self, index, op, kernel, info, cls):
        self.index, self.op, self.kernel, self.info, self.cls = index, op, kernel, list(info), cls
        self.ratio, self.where, self.edge, self.note = 0.0, None, None, ""

    @property
    def ok(self):
        return self.ratio <= 1.0

    @property
    def name(self):
        return "%s#%d(%s)" % (P.OP_NAMES[self.op.type], self.index, self.op.name)

    def __str__(self):
        return "%4d %-16s %-10s %-14s ratio %.3e  worst (n,y,x,c)=%s edge_tile=%s %s" % (
            self.index, P.OP_NAMES[self.op.type][3:], KERNELS[self.kernel], self.info, self.ratio, self.where, self.edge,
            self.note)


def kernel_class(op, kernel):
    t = op.type
    if t in (P.OP_COPY, P.OP_MAXPOOL2, P.OP_RESIZE_NEAREST):
        return "exact"
    if t == P.OP_DET_DECODE:
        return "det_decode"
    if t == P.OP_HM_DECODE or (t == P.OP_CONV and op.flags & P.FLAG_HM_PART):
        return "hm"
    if kernel == K_FPW:
        return KERNELS[K_XF]            # conv_xf's layers, operands and epilogue: reported in conv_xf's class
    if kernel in TENSOR_CORE:
        return KERNELS[kernel]
    return KERNELS[kernel] if kernel != K_MISC else "fp32:" + P.OP_NAMES[t][3:].lower()


# --------------------------------------------------------------------------------------------------- float64 bounds
class Bounds:
    """Element-wise error bounds of one op's outputs, given the inputs (float64 buffers, a dict idx -> (N,H,W,C))
    and, for ops inside a fused stem block, a bound on the error of each input buffer (`ein`)."""

    def __init__(self, interp, bufs, fp32_pipes=False):
        self.interp, self.bufs, self.fp32 = interp, bufs, fp32_pipes
        self.ein = {}                                   # buffer idx -> (N,H,W,C) error bound of the buffer's contents

    def _e(self, v):
        e = self.ein.get(v.buf.idx)
        return rd({v.buf.idx: e}, v) if e is not None else torch.zeros_like(rd(self.bufs, v))

    def _finish(self, op, z, E, out_view, residual=True):
        """Residual (ins[1] of a conv / DWPW) and activation after a pre-activation z with error bound E;
        returns (y, bound of y)."""
        res = rd(self.bufs, op.ins[1]) if residual and len(op.ins) > 1 and op.ins[1] is not None else None
        L = LIP[op.act]
        if res is not None and op.flags & P.FLAG_RES_FIRST:
            z = z + res
            E = E + self._e(op.ins[1]) + U * z.abs()     # one rounding for the add
            y = _act(z, op.act)
            B = L * E + act_eval(z, y, op.act)
        else:
            y = _act(z, op.act)
            B = L * E + act_eval(z, y, op.act)
            if res is not None:
                y = y + res
                B = B + self._e(op.ins[1]) + U * y.abs()
        if out_view.buf.dtype == P.DT_SPLIT16:
            B = B + SPLIT_REL * y.abs() + SPLIT_ABS
        return y, B

    def conv_pre(self, op, kernel):
        """Pre-activation z = conv(x [* gate], w) + b of an OP_CONV and its error bound."""
        x = rd(self.bufs, op.ins[0])
        ex = self._e(op.ins[0])
        if op.ins[2] is not None:
            g = rd(self.bufs, op.ins[2])
            x, ex = x * g, ex * g.abs()
        w = _t(getattr(op, 'w_ref', op.w)).permute(0, 3, 1, 2)
        padc = op.outs[0].C - w.shape[0]
        if padc > 0:
            w = torch.cat([w, torch.zeros((padc,) + tuple(w.shape[1:]), dtype=w.dtype)])
        b = _t(op.b) if op.b is not None else torch.zeros(w.shape[0], dtype=torch.float64)
        kw = dict(stride=op.s, padding=tuple(op.p), dilation=op.d)
        z = _hwc(F.conv2d(_chw(x), w, b, **kw))
        mag = _hwc(F.conv2d(_chw(x.abs()), w.abs(), b.abs(), **kw))
        E = _hwc(F.conv2d(_chw(ex), w.abs(), **kw))      # error carried in by the input (stem block only)
        if kernel in TENSOR_CORE and not self.fp32:
            wsum = _hwc(F.conv2d(_chw(torch.ones_like(x)), w.abs(), **kw))
            E = E + tc_rel(w.shape[1] * w.shape[2] * w.shape[3]) * mag + TC_ABS * wsum
        else:
            K = w.shape[1] * w.shape[2] * w.shape[3]
            E = E + gamma(K + 2) * mag
        return z, E

    def dw_pre(self, x, ex, w9, b, k, s, p, d, n_up=0):
        """Depthwise conv (fp32 on the CUDA cores in every kernel); n_up > 0: the first n_up channels are a bilinear x2
        up-sample (4 more products per tap: gamma over 9 taps + 4 + bias + input)."""
        C = x.shape[-1]
        w = _t(w9).T.reshape(C, 1, k[0], k[1])
        bb = _t(b)
        kw = dict(stride=s, padding=tuple(p), dilation=d, groups=C)
        z = _hwc(F.conv2d(_chw(x), w, bb, **kw))
        mag = _hwc(F.conv2d(_chw(x.abs()), w.abs(), bb.abs(), **kw))
        K = k[0] * k[1] + (4 if n_up else 0)
        E = gamma(K + 2) * mag + _hwc(F.conv2d(_chw(ex), w.abs(), **kw))
        return z, E

    def _up(self, v):
        lo = _chw(rd(self.bufs, v))
        up = _hwc(F.interpolate(lo, scale_factor=2, mode="bilinear", align_corners=False))
        # bilinear weights are non-negative: the up-sample of |low| bounds |up(low)| and carries |error| the same way
        eu = _hwc(F.interpolate(_chw(self._e(v)), scale_factor=2, mode="bilinear", align_corners=False))
        return up, eu

    def op_bounds(self, op, kernel):
        """-> list of (output view, float64 reference, bound) for every output this op stores."""
        t = op.type
        if t == P.OP_CONV:
            z, E = self.conv_pre(op, kernel)
            y, B = self._finish(op, z, E, op.outs[0])
            return [(op.outs[0], y, B)]
        if t in (P.OP_DWCONV, P.OP_UPCAT_DW):
            if t == P.OP_DWCONV:
                x, ex = rd(self.bufs, op.ins[0]), self._e(op.ins[0])
                z, E = self.dw_pre(x, ex, op.w, op.b, op.k, op.s, op.p, op.d)
            else:
                up, eu = self._up(op.ins[0])
                x = torch.cat([up, rd(self.bufs, op.ins[1])], -1)
                ex = torch.cat([eu, self._e(op.ins[1])], -1)
                z, E = self.dw_pre(x, ex, op.w, op.b, (3, 3), (1, 1), (1, 1), (1, 1), n_up=up.shape[-1])
            y, B = self._finish(op, z, E, op.outs[0], residual=False)        # ins[1] of OP_UPCAT_DW is the skip input
            out = [(op.outs[0], y, B)]
            if t == P.OP_DWCONV and op.flags & P.FLAG_GAP_PARTIAL:
                th, tw = P.dw_tile_rows(op.k[0], op.s[0]), P.DW_TILE_W
                Ho, Wo = y.shape[1], y.shape[2]
                tiles = [(a, c) for a in range(0, Ho, th) for c in range(0, Wo, tw)]
                n = th * tw
                # per-tile sums of the (rounded) outputs: their bounds plus gamma_n of the sum of magnitudes
                s = torch.stack([y[:, a:a + th, c:c + tw].sum(dim=(1, 2)) for a, c in tiles], 1)
                sb = torch.stack([B[:, a:a + th, c:c + tw].sum(dim=(1, 2)) * (1 + gamma(n)) +
                                  gamma(n) * y[:, a:a + th, c:c + tw].abs().sum(dim=(1, 2)) for a, c in tiles], 1)
                N = y.shape[0]
                out.append((op.outs[1], s.reshape(N, len(tiles), 1, -1), sb.reshape(N, len(tiles), 1, -1)))
            return out
        if t == P.OP_DWPW:
            x, ex = rd(self.bufs, op.ins[0]), self._e(op.ins[0])
            n_up = 0
            if op.ins[2] is not None:
                up, eu = self._up(op.ins[2])
                n_up = up.shape[-1]
                x, ex = torch.cat([up, x], -1), torch.cat([eu, ex], -1)
            zd, Ed = self.dw_pre(x, ex, op.dw_w, op.dw_b, (3, 3), (1, 1), (1, 1), (1, 1), n_up=n_up)
            d = _act(zd, op.dw_act)
            # the depthwise result enters the pointwise MMA as fp16 hi + lo (kept in fp32 by the stem block: harmless)
            Ed = LIP[op.dw_act] * Ed + act_eval(zd, d, op.dw_act) + SPLIT_REL * d.abs() + SPLIT_ABS
            w = _t(op.w_ref).permute(0, 3, 1, 2)
            b = _t(op.b) if op.b is not None else torch.zeros(w.shape[0], dtype=torch.float64)
            z = _hwc(F.conv2d(_chw(d), w, b))
            mag = _hwc(F.conv2d(_chw(d.abs()), w.abs(), b.abs()))
            # the fp32 depthwise stage's error propagates through |w_pw|
            E = _hwc(F.conv2d(_chw(Ed), w.abs()))
            if kernel in TENSOR_CORE and not self.fp32:
                E = E + tc_rel(w.shape[1]) * mag + TC_ABS * _hwc(F.conv2d(_chw(torch.ones_like(d)), w.abs()))
            else:
                E = E + gamma(w.shape[1] + 2) * mag
            y, B = self._finish(op, z, E, op.outs[0])
            return [(op.outs[0], y, B)]
        if t == P.OP_GAP_SSE:
            x = rd(self.bufs, op.ins[0])
            N = x.shape[0]
            ws, bs = op.w_ref
            parts = x.reshape(N, -1, 32, x.shape[-1])
            s = parts.sum(dim=2)
            sb = gamma(32) * parts.abs().sum(dim=2)
            z = (x * _t(ws)).sum(-1, keepdim=True) + float(bs[0])
            mag = (x.abs() * _t(ws).abs()).sum(-1, keepdim=True) + abs(float(bs[0]))
            y = _act(z, op.act)
            B = LIP[op.act] * gamma(x.shape[-1] + 2) * mag + act_eval(z, y, op.act)
            return [(op.outs[0], s.reshape(N, s.shape[1], 1, -1), sb.reshape(N, s.shape[1], 1, -1)), (op.outs[1], y, B)]
        if t == P.OP_SE_FC:
            w1, w2 = (_t(a) for a in op.w_ref)
            Cr = op.ints[1]
            b1, b2 = _t(op.b[:Cr]), _t(op.b[Cr:])
            part = rd(self.bufs, op.ins[0])
            N, tiles = part.shape[0], part.shape[1] * part.shape[2]
            hw = float(op.ints[3])
            mean = part.sum(dim=(1, 2)) / hw
            # per-tile sums then a divide: gamma_{tiles + 1}
            Em = gamma(tiles + 1) * part.abs().sum(dim=(1, 2)) / hw
            z1 = mean @ w1.T + b1
            h = _act(z1, op.act)
            E1 = gamma(w1.shape[1] + 2) * (mean.abs() @ w1.abs().T + b1.abs()) + Em @ w1.abs().T
            Eh = LIP[op.act] * E1 + act_eval(z1, h, op.act)
            z2 = h @ w2.T + b2
            g = _act(z2, op.ints[2])
            E2 = gamma(w2.shape[1] + 2) * (h.abs() @ w2.abs().T + b2.abs()) + Eh @ w2.abs().T
            Bg = LIP[op.ints[2]] * E2 + act_eval(z2, g, op.ints[2])
            return [(op.outs[0], g.reshape(N, 1, 1, -1), Bg.reshape(N, 1, 1, -1))]
        if t == P.OP_GAP:
            x = rd(self.bufs, op.ins[0])
            y = x.mean(dim=(1, 2), keepdim=True)
            return [(op.outs[0], y, gamma(x.shape[1] * x.shape[2] + 1) * x.abs().mean(dim=(1, 2), keepdim=True))]
        if t == P.OP_AFFINE_ACT:
            x = rd(self.bufs, op.ins[0])
            z = x * _t(op.w) + _t(op.b)
            E = gamma(2) * (x.abs() * _t(op.w).abs() + _t(op.b).abs())
            y, B = self._finish(op, z, E, op.outs[0], residual=False)
            return [(op.outs[0], y, B)]
        if t == P.OP_SCSE:
            x = rd(self.bufs, op.ins[0])
            a, b = x * rd(self.bufs, op.ins[1]), x * rd(self.bufs, op.ins[2])
            y = a + b
            return [(op.outs[0], y, gamma(2) * (a.abs() + b.abs()) + (SPLIT_REL * y.abs() + SPLIT_ABS
                                                                       if op.outs[0].buf.dtype == P.DT_SPLIT16 else 0))]
        if t == P.OP_SCALE_CH:
            y = rd(self.bufs, op.ins[0]) * rd(self.bufs, op.ins[1])
            return [(op.outs[0], y, U * y.abs() + (SPLIT_REL * y.abs() + SPLIT_ABS
                                                   if op.outs[0].buf.dtype == P.DT_SPLIT16 else 0))]
        if t == P.OP_ADDN:
            o = op.outs[0]
            xs = []
            for v in op.ins:
                if v is None:
                    continue
                x = rd(self.bufs, v)
                f = o.H // x.shape[1]
                if f > 1:
                    x = x.repeat_interleave(f, 1).repeat_interleave(f, 2)
                xs.append(x)
            z = sum(xs)
            E = gamma(len(xs)) * sum(x.abs() for x in xs)
            y, B = self._finish(op, z, E, o, residual=False)
            return [(o, y, B)]
        if t == P.OP_UPSAMPLE_BILINEAR2X:
            up, _ = self._up(op.ins[0])
            return [(op.outs[0], up, gamma(6) * self._up_abs(op.ins[0]))]
        raise NotImplementedError(P.OP_NAMES[t])

    def _up_abs(self, v):
        return _hwc(F.interpolate(_chw(rd(self.bufs, v).abs()), scale_factor=2, mode="bilinear", align_corners=False))


def ratio_of(got, ref, bound):
    """Element-wise |got - ref| / bound (bound 0: bit-exact, any difference is infinitely far); NaN counts as infinite."""
    err = (got - ref).abs()
    r = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                    torch.where(err > 0, torch.full_like(err, float("inf")), torch.zeros_like(err)))
    return torch.where(torch.isnan(r) | torch.isnan(got), torch.full_like(r, float("inf")), r)


def det_decode_bound(op, heads):
    """Bound of the yolov5-face decode per element.  Every output is a short chain of float32 operations on one sigmoid
    (2^-21 relative, see act_eval) or one head value: 2^-20 (16 ulp) of the sum of the magnitudes of its terms covers the
    sigmoid error doubled / squared and the 3-4 roundings of the chain."""
    c = op.w
    rows = []
    N = heads[0].shape[0]
    for si, h in enumerate(heads):
        stride = float(c[si * 7])
        an = _t(c[si * 7 + 1: si * 7 + 7].reshape(3, 2))[None, :, None, None, :]
        H, W = h.shape[1], h.shape[2]
        t = h.reshape(N, H, W, 3, 16).permute(0, 3, 1, 2, 4)
        gy, gx = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
        grid = torch.stack([gx, gy], -1)[None, None]
        sg = torch.sigmoid(t)
        parts = [(sg[..., 0:2] * 2 + 0.5 + grid) * stride, (sg[..., 2:4] * 2) ** 2 * an.abs(), sg[..., 4:5]]
        for k in range(5):
            parts.append((t[..., 5 + 2 * k: 7 + 2 * k] * an).abs() + grid * stride)
        parts.append(sg[..., 15:16])
        rows.append(torch.cat(parts, -1).reshape(N, -1, 16))
    return 2.0 ** -20 * torch.cat(rows, 1).reshape(N, -1, 1, 16)


# --------------------------------------------------------------------------------------------------- the engine side
class EngineOps:
    """The CUDA engine as check_ops() drives it: one forward, then op by op re-run / read back."""

    def __init__(self, eng, batch):
        from peppa_pig_face_landmark_b200 import runtime as rt
        self.eng, self.batch, self.rt = eng, batch, rt
        self.lib = rt.load_library()
        self.plan = eng.plan

    def forward(self, x_u8):
        self.eng.run_u8(x_u8)

    def op_kernel(self, i):
        import ctypes as C
        info = (C.c_int32 * 4)()
        k = self.lib.skps_engine_op_kernel(self.eng.handle, i, info)
        assert k >= 0, "op_kernel: bad op index %d" % i
        return k, tuple(info)

    def read(self, idx):
        return torch.from_numpy(self.eng.read_buffer(idx, self.batch))

    def run_op(self, i):
        self.rt.check(self.lib.skps_engine_run_op(self.eng.handle, i, self.batch, self.eng.stream.cuda_stream))
        self.eng.stream.synchronize()

    def op_grid(self, i):
        """(CTAs, work units) of op i's launch if it runs a persistent kernel, else (0, 0)."""
        import ctypes as C
        g = (C.c_int32 * 2)()
        self.rt.check(self.lib.skps_engine_op_grid(self.eng.handle, i, self.batch, g))
        return g[0], g[1]

    def set_num_sms(self, n):
        """Size the persistent kernels' grids for n SMs (0: the device's)."""
        self.rt.check(self.lib.skps_engine_set_num_sms(self.eng.handle, n))


class InterpOps:
    """The float32 PlanInterp standing in for the engine (the checker's own test, without a GPU).  Kernel ids are the
    ones the plan's flags ask for; no tiling is reported."""

    def __init__(self, plan, batch):
        self.plan, self.batch, self.interp = plan, batch, PlanInterp(plan)

    def forward(self, x_u8):
        self.x_u8 = torch.from_numpy(np.ascontiguousarray(x_u8))
        self.bufs = [torch.zeros(self.batch, b.H, b.W, b.C, dtype=torch.float32) for b in self.plan.bufs]
        self.bufs[self.plan.input.buf.idx] = self.x_u8.to(torch.float32) / np.float32(255.0)
        for op in self.plan.ops:
            self._step(op)

    def op_kernel(self, i):
        op = self.plan.ops[i]
        if op.type == P.OP_CONV:
            k = K_MMA if op.flags & P.FLAG_MMA else K_XF if op.flags & P.FLAG_XF else K_TC if op.flags & P.FLAG_TC \
                else K_SIMT
        else:
            k = {P.OP_DWCONV: K_DW, P.OP_DWPW: K_XF, P.OP_UPCAT_DW: K_UPCAT, P.OP_STEM_BLOCK: K_STEM}.get(op.type, K_MISC)
        return k, (0, 0, 0, 0)

    def read(self, idx):
        return self.x_u8.clone() if idx == self.plan.input.buf.idx else self.bufs[idx].clone()

    def run_op(self, i):
        self._step(self.plan.ops[i])

    def _step(self, op):
        self.interp.step(op, self.bufs)
        for v in op.outs:                      # what the engine stores in a split-fp16 buffer is hi + lo
            if v.buf.dtype == P.DT_SPLIT16:
                sl = (Ellipsis, slice(v.c_off, v.c_off + v.C * v.c_stride, v.c_stride))
                self.bufs[v.buf.idx][sl] = split16_round(self.bufs[v.buf.idx][sl])


def _views_in(op):
    vs = [v for v in op.ins if v is not None]
    if op.type == P.OP_STEM_BLOCK:
        vs = [op.ins[0]]
    return vs


def _stored(op):
    if op.type == P.OP_CONV and op.flags & P.FLAG_HM_PART:
        return [op.outs[1]]                                   # the heat map itself is not stored
    return list(op.outs)


# Output tile of every tiled kernel: kernel -> (f(info, H, W) -> (rows, columns) of one tile of an H x W output map, whether
# a tile can hang over the map's border).  info is the tiling skps_engine_op_kernel reports.  A kernel whose applicability
# test only takes maps made of whole tiles has no border tiles; launch_signature() asserts that of every launch it sees.
# conv_pw tiles the flat (n, y, x) pixel index of the batch instead (PW_BM); conv_simt's pixel tile is picked per launch
# from the SM count and is not reported, so it has no entry.
TILES = {
    # 128-pixel blocks of bw x bh = 128 / bw pixels of one image, ragged at the right and bottom border (tc_pick_bw);
    # maps under 128 pixels: ipt whole images per tile (bw = W, bh = ipt H), the batch's last tile partial
    K_TC: (lambda info, H, W: (info[1], info[0]), True),
    # whole-row store boxes: bh = 256 / W rows of the full width; tct_applicable takes only W | 256 and H % bh == 0
    K_TCT: (lambda info, H, W: (info[0], W), False),
    # 256-pixel blocks of whole rows; hm_shape_ok takes only W | 256 and (H W) % 256 == 0
    K_HM: (lambda info, H, W: (256 // W, W), False),
    # 8 x 16 pixel tiles over the (stride-1) map, ceil-divided (conv_mma.cu MT_H, MT_W)
    K_MMA: (lambda info, H, W: (8, 16), True),
    # 16 x 8 pixel tiles (xf_producer.h XF_TW, XF_TH), ceil-divided
    K_XF: (lambda info, H, W: (8, 16), True),
    # conv_xf's tiles; fpw_supported takes only H % 8 == W % 16 == 0
    K_FPW: (lambda info, H, W: (8, 16), False),
    # dw_tile_rows(k, s) rows x 16 columns, ceil-divided
    K_DW_TMA: (lambda info, H, W: (info[0], P.DW_TILE_W), True),
    # 8 x 16 output tiles for the up-sampled channels and a 3x3 stride-1 dw_tma launch (8 x 16) for the skip channels
    K_UPCAT_TMA: (lambda info, H, W: (8, 16), True),
    # 8 x 16 tiles of the quarter-resolution output; stem_block_supported takes only input maps with H % 32 == W % 64 == 0
    K_STEM: (lambda info, H, W: (8, 16), False),
    # the fallback depthwise kernel: one thread per 4 consecutive pixels of a row where W % 4 == 0, else per pixel
    K_DW: (lambda info, H, W: (1, 4 if W % 4 == 0 else 1), False),
}


def edge_tile(kernel, info, H, W, y, x, n=None, batch=None):
    """Whether output pixel (y, x) of an H x W map lies in a tile that hangs over the map's border (TILES); for conv_pw, and
    for conv_tc's multi-image tiles, whether pixel (n, y, x) lies in the last, partial tile of a batch of `batch` maps.
    None where the kernel's tiling is not known."""
    if kernel == K_PW or (kernel == K_TC and info[2] > 1):
        if n is None or batch is None:
            return None
        if kernel == K_TC:
            return bool(batch % info[2] and n >= batch // info[2] * info[2])
        rows = batch * H * W
        return bool(rows % PW_BM and (n * H + y) * W + x >= rows // PW_BM * PW_BM)
    if kernel not in TILES:
        return None
    tile, border = TILES[kernel]
    if not border:
        return False
    bh, bw = tile(info, H, W)
    if bh <= 0 or bw <= 0:                     # no tiling reported (the float32 interpreter standing in for the engine)
        return None
    return bool((x // bw + 1) * bw > W or (y // bh + 1) * bh > H)


def plan_structure(plan):
    """The sequence of (op type, op flags) of a plan: which ops the lowering emits, fused how, routed to which family."""
    return tuple((op.type, op.flags) for op in plan.ops)


def launch_signature(op, kernel, info, H, W, batch):
    """What decides which code paths one op's launch runs: the op's layer (type, flags, kernel size, stride, channels,
    activation), the kernel and its tiling (info), and where the map's border falls in the kernel's tile.  H x W is the
    op's output map.

    For the kernels in TILES the border is (H mod tile rows > 0, W mod tile columns > 0, the map is smaller than one
    tile).  Whether a side is ragged, not by how much, is what selects code: conv_tc masks every row of an edge tile
    (row_ok) and its TMA stores clip, dw_tma masks every pixel, conv_xf stores row by row, so the remainder itself picks
    no other path.  conv_xf adds whether the map is one tile across: it then loads a wider up-sample weight box (wcx,
    conv_xf.cu).  conv_pw: whether the last 128-pixel tile of the batch's batch H W pixels is partial.  conv_tc adds
    the images in the last multi-image tile (ipt > 1) and, with two pixel tiles per weight load (mt = 2), the parity
    of the launch's tile count.  A kernel without border tiles is asserted to have no ragged side.  The op's place in
    the plan is left out: the same layer at another place runs the same code."""
    info = tuple(int(v) for v in info)
    if kernel == K_PW:
        border = ((batch * H * W) % PW_BM > 0,)
    elif kernel in TILES:
        tile, has_border = TILES[kernel]
        th, tw = tile(info, H, W)
        border = (H % th > 0, W % tw > 0, H < th or W < tw)
        assert has_border or not (border[0] or border[1]), "%s has no border tiles, but its %dx%d tile does not " \
            "divide %dx%d" % (KERNELS[kernel], th, tw, H, W)
        if kernel == K_XF:
            border += (W <= tw,)
        if kernel == K_TC:
            bw, bh, ipt, mt = info
            if ipt > 1:
                border += (batch % ipt,)
            if mt == 2:
                tiles = -(-batch // ipt) if ipt > 1 else batch * (-(-H // bh)) * (-(-W // bw))
                border += (tiles % 2,)
    else:
        border = None
    layer = (op.type, op.flags, tuple(op.k), tuple(op.s), op.ins[0].C if op.ins and op.ins[0] is not None else 0,
             op.outs[0].C, op.act)
    return layer, kernel, info, border


def _to64(t, buf):
    if buf.dtype == P.DT_U8:
        return t.to(torch.float64) / 255.0
    return t.to(torch.float64)


def _fresh(bufs, views, batch):
    """Float64 output buffers for `views`: zeros, or a copy where the buffer is also read (so the inputs stay intact)."""
    for v in views:
        b = v.buf
        bufs[b.idx] = bufs[b.idx].clone() if b.idx in bufs else torch.zeros(batch, b.H, b.W, b.C, dtype=torch.float64)


def evaluate(op, kernel, info, interp, ins_raw, got_raw, batch):
    """Compare one op's outputs (`got_raw`: buffer idx -> engine buffer after the op, as read back) with the float64
    evaluation from its inputs (`ins_raw`: buffer idx -> engine buffer before the op).
    Returns (worst ratio, (n, y, x, c) of the worst element, rows) -- rows: (view, reference, bound, ratio) per output."""
    bufs = {k: _to64(x, interp.plan.bufs[k]) for k, x in ins_raw.items()}
    got64 = {k: _to64(x, interp.plan.bufs[k]) for k, x in got_raw.items()}
    t = op.type
    if t == P.OP_CONV and op.flags & P.FLAG_HM_PART:
        return _hm_partials(op, kernel, info, interp, bufs, got_raw, batch)
    if t == P.OP_HM_DECODE:
        return _hm_decode(op, bufs, ins_raw, got64)
    if t == P.OP_STEM_BLOCK:
        # the fused layers run on the FP32 pipes; each layer's bound carries the error of its inputs from the layer
        # before (Bounds.ein); only the block's last output is stored
        bd = Bounds(interp, dict(bufs), fp32_pipes=True)
        for sub in op.sub_ops:
            _fresh(bd.bufs, sub.outs, batch)
            for v, ref, B in bd.op_bounds(sub, kernel):
                e = bd.ein.get(v.buf.idx)
                e = torch.zeros_like(bd.bufs[v.buf.idx]) if e is None else e.clone()
                e[..., v.c_off: v.c_off + v.C * v.c_stride: v.c_stride] = B
                bd.ein[v.buf.idx] = e
                bd.bufs[v.buf.idx][..., v.c_off: v.c_off + v.C * v.c_stride: v.c_stride] = ref
        res = [(op.outs[0], rd(bd.bufs, op.outs[0]), rd(bd.ein, op.outs[0]))]
    elif t in (P.OP_COPY, P.OP_MAXPOOL2, P.OP_RESIZE_NEAREST):
        res = [(v, None, 0.0) for v in op.outs]                 # data movement: bit-exact
    elif t == P.OP_DET_DECODE:
        res = [(op.outs[0], None, det_decode_bound(op, [rd(bufs, v) for v in op.ins]))]
    else:
        res = Bounds(interp, dict(bufs)).op_bounds(op, kernel)
    # the reference values are PlanInterp.step's; where the bound code recomputed them (for the pre-activation terms)
    # the two must agree
    stem_outs = [v for sub in op.sub_ops for v in sub.outs] if t == P.OP_STEM_BLOCK else []
    _fresh(bufs, list(op.outs) + stem_outs, batch)
    interp.step(op, bufs, torch.float64)
    checks = []
    for v, ref, B in res:
        r = rd(bufs, v)
        if ref is None and v.buf.dtype == P.DT_SPLIT16:
            # data movement from a float32 buffer into a split-fp16 one stores hi = fp16(v), lo = fp16(v - hi): exact
            # once that rounding is applied (a no-op on values that already came from a split-fp16 buffer)
            r = split16_round(r.float()).double()
        if ref is not None:
            assert torch.allclose(r, ref, rtol=1e-9, atol=1e-9 * (float(r.abs().max()) + 1)), P.OP_NAMES[t]
        checks.append((v, r, B if torch.is_tensor(B) else torch.full_like(r, B)))
    return _worst(checks, got64)


def _worst(checks, got64):
    worst, where, rows = 0.0, None, []
    for v, ref, B in checks:
        got = rd(got64, v)
        r = ratio_of(got, ref, B)
        rows.append((v, ref, B, r))
        m = float(r.max()) if r.numel() else 0.0
        if m > worst or where is None:
            flat = int(torch.argmax(torch.nan_to_num(r, posinf=1e308)))
            worst, where = max(worst, m), tuple(int(i) for i in np.unravel_index(flat, tuple(r.shape)))
    return worst, where, rows


def _hm_tiles(kernel, info, H, W):
    """Tile id of every pixel (H, W) of a heat-map head: conv_tc's 128-pixel bw x bh tiles or conv_hm's 256-pixel runs."""
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    if kernel == K_TC:
        bw, bh = info[0], info[1]
        return (yy // bh) * ((W + bw - 1) // bw) + xx // bw
    return (yy * W + xx) // 256


def _part_rows(raw, n_tiles, C):
    """Per-tile partial rows of a heat-map head as read back: [N][tiles][ld] float32, ld/2 maxima then ld/2 int32
    arg-max pixel indices (their bits) -> (maxima float64, indices int64), first C channels."""
    N, ld = raw.shape[0], raw.shape[-1]
    rows = raw.reshape(N, -1, ld)[:, :n_tiles].contiguous()
    return rows[..., :C].double(), rows.view(torch.int32)[..., ld // 2: ld // 2 + C].long()


def _hm_partials(op, kernel, info, interp, bufs, got_raw, batch):
    """Heat-map head with per-tile (max, first arg-max) partials instead of the map: the per-tile maximum must match the
    float64 one within the conv's bound, and the reported pixel must lie in the tile and BE a maximum within the bound
    (its float64 score within twice the bound of the tile's float64 maximum: both scores the kernel compared can be off
    by one bound) -- the rule of test_conv_hm_transposed_head_matches_fp64_argmax."""
    bd = Bounds(interp, bufs)
    z, E = bd.conv_pre(op, kernel)                           # score maps: no activation, no residual
    C = getattr(op, 'w_ref', op.w).shape[0]                  # not the zero channels that pad the map to a width of 8
    z, E = z[..., :C].contiguous(), E[..., :C].contiguous()
    N, H, W, _ = z.shape
    tid = _hm_tiles(kernel, info, H, W).reshape(-1)
    T = int(tid.max()) + 1
    val, idx = _part_rows(got_raw[op.outs[1].buf.idx], T, C)
    zf, Ef = z.reshape(N, H * W, C), E.reshape(N, H * W, C)
    rmax = torch.full((N, T, C), -float("inf"), dtype=torch.float64)
    bmax = torch.zeros((N, T, C), dtype=torch.float64)
    rmax = rmax.scatter_reduce(1, tid[None, :, None].expand(N, -1, C), zf, "amax")
    bmax = bmax.scatter_reduce(1, tid[None, :, None].expand(N, -1, C), Ef, "amax")
    r_val = (val - rmax).abs() / bmax
    inside = (idx >= 0) & (idx < H * W)
    safe = torch.where(inside, idx, torch.zeros_like(idx))
    in_tile = inside & (tid[safe] == torch.arange(T)[None, :, None])
    picked = torch.gather(zf, 1, safe)
    r_pick = torch.where(in_tile, (rmax - picked) / (2 * bmax), torch.full_like(r_val, float("inf")))
    r = torch.maximum(r_val, r_pick)
    flat = int(torch.argmax(r))
    n, t, c = np.unravel_index(flat, tuple(r.shape))
    return float(r.max()), (int(n), int(t), -1, int(c)), [(op.outs[1], val, bmax, r)]


def _hm_decode(op, bufs, ins_raw, got64):
    """Arg-max decode over the head's per-tile partials: the score must be exactly the first largest partial maximum
    (a selection, no arithmetic), the x/y offsets the K-long dot product at that pixel (gamma_{K+2}), plus the add of the
    pixel column / row and the divide by W (2 more roundings)."""
    npts = op.ints[0]
    assert op.flags & P.FLAG_HM_PART and len(op.ins) > 2 and op.ins[2] is not None, "hm_decode without partials"
    pv = op.ins[2]
    assert pv.c_off == 0 and pv.c_stride == 1
    val, idx = _part_rows(ins_raw[pv.buf.idx], pv.H * pv.W, npts)
    N = val.shape[0]
    m = val.max(dim=1, keepdim=True).values
    big = torch.full_like(idx, 1 << 40)
    am = torch.where(val == m, idx, big).min(dim=1).values                 # first maximum over tiles: smallest pixel index
    score = m[:, 0]
    W = op.ins[0].W
    feat = rd(bufs, op.ins[1])
    f = feat.reshape(N, -1, feat.shape[-1])
    fa = torch.gather(f, 1, am[:, :, None].expand(N, npts, f.shape[-1]))
    wo, bo = _t(op.w), _t(op.b)
    ox = (fa * wo[:npts][None]).sum(-1) + bo[:npts]
    oy = (fa * wo[npts:][None]).sum(-1) + bo[npts:]
    mx = (fa.abs() * wo[:npts].abs()[None]).sum(-1) + bo[:npts].abs()
    my = (fa.abs() * wo[npts:].abs()[None]).sum(-1) + bo[npts:].abs()
    K = f.shape[-1]
    cx, cy = (am % W).double(), (am // W).double()
    xy = torch.stack([(cx + ox) / W, (cy + oy) / W], -1)
    bxy = torch.stack([(gamma(K + 2) * mx * (1 + gamma(2)) + gamma(2) * (cx + ox.abs())) / W,
                       (gamma(K + 2) * my * (1 + gamma(2)) + gamma(2) * (cy + oy.abs())) / W], -1)
    checks = [(op.outs[0], xy.reshape(N, 1, 1, -1), bxy.reshape(N, 1, 1, -1)),
              (op.outs[1], score.reshape(N, 1, 1, -1), torch.zeros_like(score).reshape(N, 1, 1, -1))]
    return _worst(checks, got64)


def check_ops(ex, x_u8, log=None, keep=None):
    """Run `x_u8` (N,H,W,3 uint8) through executor `ex` (EngineOps or InterpOps) once, then re-run every op in
    plan order and check it in isolation (re-running in order restores every op's inputs as the forward left them).
    Returns (list of OpCheck, dict op index -> (outputs as read back, rows of (view, reference, bound, ratio))) -- the
    dict only for the OpChecks `keep` accepts (the tensors of a whole large plan do not fit in host memory)."""
    batch = x_u8.shape[0]
    ex.forward(x_u8)
    plan = ex.plan
    interp = PlanInterp(plan)
    results, detail = [], {}
    for i, op in enumerate(plan.ops):
        kernel, info = ex.op_kernel(i)
        ins = {}
        for v in _views_in(op):
            ins.setdefault(v.buf.idx, ex.read(v.buf.idx))
        ex.run_op(i)
        got = {}
        for v in _stored(op):
            got.setdefault(v.buf.idx, ex.read(v.buf.idx))
        res = OpCheck(i, op, kernel, info, kernel_class(op, kernel))
        res.batch = batch
        res.ratio, res.where, rows = evaluate(op, kernel, info, interp, ins, got, batch)
        if res.where is not None and res.where[2] >= 0:
            o = op.outs[0]
            res.edge = edge_tile(kernel, info, o.H, o.W, res.where[1], res.where[2], res.where[0], batch)
        if keep is not None and keep(res):
            detail[i] = (got, rows)
        results.append(res)
        if log is not None:
            print(res, file=log, flush=True)
    return results, detail


def check_engine(eng, x_u8, log=None, keep=None):
    return check_ops(EngineOps(eng, x_u8.shape[0]), x_u8, log, keep)


def planted_ratio(op, got, rows, k, where, factor=8.0):
    """Add `factor` x the element's bound to one element (n, y, x, c) of output row k on a HOST COPY of what the kernel
    wrote, and return the comparator's worst ratio over that output (a working checker reports >= factor - 1)."""
    v, ref, B, _ = rows[k]
    g = {i: _to64(x, v.buf) if i == v.buf.idx else x for i, x in got.items()}
    n, y, x, c = where
    g[v.buf.idx] = g[v.buf.idx].clone()
    g[v.buf.idx][n, y, x, v.c_off + c * v.c_stride] += factor * float(B[n, y, x, c])
    return _worst([(v, ref, B)], g)[0]


def worst_per_class(results):
    out = {}
    for r in results:
        out[r.cls] = max(out.get(r.cls, 0.0), r.ratio)
    return out


def tc_geometry(r):
    """(Ho, Wo, bw, bh, ipt, mt, pixel tiles of the launch) of a conv_tc OpCheck."""
    o = r.op.outs[0]
    bw, bh, ipt, mt = r.info
    tiles = -(-r.batch // ipt) if ipt > 1 else r.batch * (-(-o.H // bh)) * (-(-o.W // bw))
    return o.H, o.W, bw, bh, ipt, mt, tiles


BRANCHES = ["tc bw=%d ragged %s" % (bw, side) for bw in (64, 32, 16, 8) for side in ("right", "bottom")] + [
    "tc ipt>1", "tc mt=2 odd tile count", "tc stride 2 ragged", "tct", "simt conv W<8",
    "dw_tma s1 W<16", "dw_tma s1 W>=16", "dw_tma s2 W<16", "dw_tma s2 W>=16", "upcat_tma", "dwpw H%8!=0", "stem block",
    "pw partial last tile", "pw N chunks > 1"]


def coverage(tagged):
    """Branch name -> ["plan:op index", ...] over (plan tag, OpCheck) pairs, for every name in BRANCHES."""
    cov = {b: [] for b in BRANCHES}
    for tag, r in tagged:
        hit = []
        o = r.op.outs[0]
        if r.kernel == K_TC:
            Ho, Wo, bw, bh, ipt, mt, tiles = tc_geometry(r)
            if ipt == 1 and Wo % bw:
                hit.append("tc bw=%d ragged right" % bw)
            if ipt == 1 and Ho % bh:
                hit.append("tc bw=%d ragged bottom" % bw)
            if ipt > 1:
                hit.append("tc ipt>1")
            if mt == 2 and tiles % 2:
                hit.append("tc mt=2 odd tile count")
            if r.op.s[0] == 2 and ipt == 1 and (Wo % bw or Ho % bh):
                hit.append("tc stride 2 ragged")
        elif r.kernel == K_TCT:
            hit.append("tct")
        elif r.kernel == K_PW:
            if (r.batch * o.H * o.W) % PW_BM:
                hit.append("pw partial last tile")
            if r.info[1] > 1:
                hit.append("pw N chunks > 1")
        elif r.kernel == K_SIMT and o.W < 8:
            hit.append("simt conv W<8")
        elif r.kernel == K_DW_TMA:
            hit.append("dw_tma s%d W%s16" % (r.op.s[0], "<" if o.W < 16 else ">="))
        elif r.kernel == K_UPCAT_TMA:
            hit.append("upcat_tma")
        elif r.kernel == K_STEM:
            hit.append("stem block")
        if r.op.type == P.OP_DWPW and o.H % 8:
            hit.append("dwpw H%8!=0")
        for h in hit:
            if h in cov:
                cov[h].append("%s:%d" % (tag, r.index))
    return cov


# The persistent kernels launch min(units, SMs) CTAs (conv_mma: SMs x its CTAs per SM), and each CTA walks units
# blockIdx.x, + gridDim.x, ...: the ring phases, conv_pw's alternating warpgroups, the reuse of the epilogue staging buffers
# and the stem block's prefetch only act from a CTA's second unit on.  A sweep with the grid capped below the SM count
# (skps_engine_set_num_sms) must reach these.
PERSISTENT = {K_TC: "tc", K_TCT: "tct", K_HM: "hm", K_PW: "pw", K_XF: "xf", K_FPW: "fpw", K_STEM: "stem_block",
              K_MMA: "mma"}
WALK_BRANCHES = ["%s >= 3 units per CTA" % PERSISTENT[k] for k in sorted(PERSISTENT)] + [
    "pw every CTA >= 4 units, last unit on each warpgroup"]


def units_per_cta(ctas, units):
    """Units each CTA of a persistent launch walks: CTA b takes units b, b + ctas, ... (ascending in b's order)."""
    return [len(range(b, units, ctas)) for b in range(ctas)]


def walk_coverage(walks):
    """Branch name -> ["plan:op index@cap", ...] for every name in WALK_BRANCHES, over (label, kernel, ctas, units)
    tuples, one per persistent launch.  conv_pw gives unit `local` of a CTA to warpgroup local % 2: with at least 4 units
    on every CTA each warpgroup takes at least 2, and a grid that does not divide the units leaves CTAs with an odd and
    CTAs with an even count, so the last unit falls on warpgroup 0 on some and on warpgroup 1 on others."""
    cov = {b: [] for b in WALK_BRANCHES}
    for label, kernel, ctas, units in walks:
        if kernel not in PERSISTENT or not ctas:
            continue
        per = units_per_cta(ctas, units)
        if max(per) >= 3:
            cov["%s >= 3 units per CTA" % PERSISTENT[kernel]].append(label)
        if kernel == K_PW and min(per) >= 4 and units % ctas:
            cov["pw every CTA >= 4 units, last unit on each warpgroup"].append(label)
    return cov


# --------------------------------------------------------------------------------------------------- inputs and plans
def detector_inputs(hw, batch=3):
    """A letterboxed real frame (four copies of test1.jpg on a 4K frame), uint8 noise and a near-uniform grey frame."""
    import frames
    from oracle import host_ref as H
    x, _ = H.letterbox(frames.frame_4k(), *hw)
    real = np.round(x[0].transpose(1, 2, 0) * 255).astype(np.uint8)
    return _with_noise(real, batch)


def detector_domain_sample():
    """Detector input sizes that take every value of each axis of the accepted range (check_detector_input): every h with
    w at the range's minimum, Skps.yml's default 640 and the maximum, every w with h at the minimum, the default 384 and
    the maximum -- the four corners included.  The minima bring the small maps, where conv_tc's multi-image tiles start."""
    from peppa_pig_face_landmark_b200.graph_tools import DET_INPUT_MAX as hi, DET_INPUT_MIN as lo
    hs, ws = range(lo[0], hi[0] + 1, 32), range(lo[1], hi[1] + 1, 32)
    return sorted({(h, w) for h in hs for w in (lo[1], 640, hi[1])} | {(h, w) for w in ws for h in (lo[0], 384, hi[0])})


def retarget_and_lower(args):
    """(hw, directory, keep) -> (hw, path, plan_structure of the plan): the shipped detector retargeted to hw, written to
    `path` in directory and lowered.  The file (2 MB at 128x128, 84 MB at 2176x3840) is deleted unless keep, and path is
    then None.  A module-level function so that a process pool can run it."""
    from peppa_pig_face_landmark_b200 import lowering
    from peppa_pig_face_landmark_b200.graph_tools import retarget_detector_input
    hw, d, keep = args
    src = os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained", "yolov5n-0.5.onnx")
    path = retarget_detector_input(src, os.path.join(d, "det_%dx%d.onnx" % hw), hw)
    try:
        structure = plan_structure(lowering.lower(path, hw))
    finally:
        if not keep:
            os.remove(path)
    return hw, path if keep else None, structure


def lower_detector_domain(sizes, directory, keep=False):
    """retarget_and_lower over `sizes` on every CPU: yields (hw, path, plan structure) in the order of `sizes`.  With
    keep, the caller deletes each file once done with it; the pool runs at most two sizes per worker ahead of the
    caller, so only those files exist at one time."""
    import multiprocessing
    from collections import deque
    from concurrent.futures import ProcessPoolExecutor
    n = min(16, os.cpu_count() or 1)
    todo = iter(sizes)
    with ProcessPoolExecutor(n, mp_context=multiprocessing.get_context("spawn")) as ex:
        ahead = deque()
        for hw in todo:
            ahead.append(ex.submit(retarget_and_lower, (hw, directory, keep)))
            if len(ahead) >= 2 * n:
                yield ahead.popleft().result()
        while ahead:
            yield ahead.popleft().result()


def greedy_cover(sigs):
    """{size: set of signatures} -> sizes whose signatures together are all of them: greedy weighted set cover at cost
    h w, i.e. repeatedly the size with the least cost per signature it adds (the smaller size on a tie)."""
    left = set().union(*sigs.values())
    cover = []
    while left:
        hw = min((hw for hw in sigs if sigs[hw] & left),
                 key=lambda hw: (hw[0] * hw[1] / len(sigs[hw] & left), hw[0] * hw[1], hw))
        cover.append(hw)
        left -= sigs[hw]
    return cover


def _with_noise(real, batch):
    rng = np.random.default_rng(1)
    h, w = real.shape[:2]
    out = [real, rng.integers(0, 256, (h, w, 3), dtype=np.uint8),
           (114 + rng.integers(0, 2, (h, w, 3))).astype(np.uint8)]
    while len(out) < batch:
        out.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
    return np.ascontiguousarray(np.stack(out[:batch]))


def crop_inputs(batch=3):
    import frames
    return _with_noise(frames.crop_variants(1)[0], batch)


def make_engine(which, hw=None, batch=3, device=None):
    """(engine, input batch) for which = detector (at input size hw), student or teacher; device: None (the current
    device) or the device the engine runs on."""
    from peppa_pig_face_landmark_b200.core.api.onnx_model_base import ONNXEngine
    dev = "cuda" if device is None else device
    pre = os.path.join(ROOT, "peppa_pig_face_landmark_b200", "pretrained")
    if which == "detector":
        from peppa_pig_face_landmark_b200.graph_tools import detector_onnx_for
        path = detector_onnx_for(os.path.join(pre, "yolov5n-0.5.onnx"), hw)
        return ONNXEngine(path, device=dev, max_batch=batch), detector_inputs(hw, batch)
    if which == "student":
        return ONNXEngine(os.path.join(pre, "kps_student.onnx"), device=dev, max_batch=batch), crop_inputs(batch)
    if which == "teacher":
        from peppa_pig_face_landmark_b200 import teacher_graph as T
        return ONNXEngine(T.ensure_teacher_onnx(256), device=dev, max_batch=batch), crop_inputs(batch)
    raise ValueError(which)


def report(which, hw=None, batch=3, out=sys.stdout):
    eng, x = make_engine(which, hw, batch)
    results, _ = check_engine(eng, x, log=out)
    print("worst err/bound per kernel class:", file=out)
    for k, v in sorted(worst_per_class(results).items()):
        print("  %-18s %.3e" % (k, v), file=out)
    bad = [r for r in results if not r.ok]
    for r in bad:
        print("FAIL %s kernel %s %s worst (n,y,x,c)=%s edge tile=%s ratio %.3e" % (
            r.name, KERNELS[r.kernel], r.info, r.where, r.edge, r.ratio), file=out)
    return results


if __name__ == "__main__":
    args = sys.argv[1:] or ["student"]
    which = args[0]
    hw = (int(args[1]), int(args[2])) if which == "detector" and len(args) > 2 else ((384, 640) if which == "detector" else None)
    rest = args[3:] if which == "detector" and len(args) > 2 else args[1:]
    batch = int(rest[0]) if rest else (2 if which == "teacher" else 3)
    res = report(which, hw, batch)
    sys.exit(0 if all(r.ok for r in res) else 1)
