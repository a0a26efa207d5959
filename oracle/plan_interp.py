"""ORACLE-side tool (test infrastructure): executes a lowered plan
(peppa_pig_face_landmark_b200.plan.Plan) with PyTorch CPU ops so that the
lowering — fusion patterns, concat/shuffle views, decode tails — can be checked
against oracle.onnx_exec without a GPU.  Mirrors the semantics csrc/ implements.

`run()` executes a whole plan in float32; `step()` executes one plan op on a buffer list, in float32 or
float64 (tools/op_report.py evaluates every engine op in float64 from the engine's own inputs)."""
import numpy as np
import torch
import torch.nn.functional as F

from peppa_pig_face_landmark_b200 import plan as P


def _act(x, a):
    if a == P.ACT_NONE:
        return x
    if a == P.ACT_RELU:
        return torch.relu(x)
    if a == P.ACT_SILU:
        return x * torch.sigmoid(x)
    if a == P.ACT_SIGMOID:
        return torch.sigmoid(x)
    hs = torch.clamp(x * np.float32(1.0 / 6.0) + 0.5, 0.0, 1.0)
    return x * hs if a == P.ACT_HSWISH else hs


def split16_round(x, lo_scale=1.0):
    """v -> hi + lo as the SPLIT16 activation format stores it: hi = fp16(v), lo = fp16((v - hi) * lo_scale) / lo_scale
    (float16 subnormals included).  Used to measure what the format alone costs (tools/split_error.py)."""
    hi = x.to(torch.float16).to(torch.float32)
    lo = ((x - hi) * lo_scale).to(torch.float16).to(torch.float32) / lo_scale
    return hi + lo


def rd(bufs, v):
    """The channel window of view `v` (N, H, W, C) in a buffer list."""
    return bufs[v.buf.idx][..., v.c_off: v.c_off + v.C * v.c_stride: v.c_stride]


def wr(bufs, v, val):
    bufs[v.buf.idx][..., v.c_off: v.c_off + v.C * v.c_stride: v.c_stride] = val


class PlanInterp:
    def __init__(self, plan, emulate_split=False, lo_scale=1.0):
        self.plan = plan
        self.emulate_split = emulate_split      # tensor-core convs and OP_DWPW: operands rounded to fp16 hi/lo, fp64 accumulate
        self.lo_scale = lo_scale
        # csrc/stem_block.cu runs the depthwise + 1x1 of its fused layers on the FP32 pipes
        self._fp32_dwpw = {id(op.sub_ops[1]) for op in plan.ops if op.type == P.OP_STEM_BLOCK}

    def run(self, x_nhwc, dump=None):
        """x: (N,H,W,3) uint8 (or float32 already /255 when the plan was lowered with input_u8=False)."""
        pl = self.plan
        N = x_nhwc.shape[0]
        bufs = [torch.zeros(N, b.H, b.W, b.C, dtype=torch.float32) for b in pl.bufs]
        xin = torch.from_numpy(np.ascontiguousarray(x_nhwc))
        if xin.dtype == torch.uint8:
            xin = xin.to(torch.float32) / np.float32(255.0)
        bufs[pl.input.buf.idx] = xin
        for op in pl.ops:
            self.step(op, bufs, dump=dump)
        return [rd(bufs, v).reshape(N, -1).numpy() if v.buf.W == 1 and v.buf.H == 1
                else rd(bufs, v).reshape(N, v.buf.H, v.C).numpy() for v in pl.outputs]

    def step(self, op, bufs, dtype=torch.float32, dump=None):
        """Execute one plan op on `bufs` (one (N, H, W, C) tensor per plan buffer, the input already divided by 255):
        reads its input views, writes its output views.  Weights, biases and decode constants are cast to `dtype`
        (float32 leaves them exactly as run() has always used them).  A fused stem block executes as the layers it
        replaces.  `dump`: optional list that receives (op, [output views]) per executed layer."""
        if op.type == P.OP_STEM_BLOCK:
            for sub in op.sub_ops:
                self.step(sub, bufs, dtype, dump)
            return

        def T(a):
            t = torch.from_numpy(a)
            return t if dtype == torch.float32 else t.to(dtype)

        N = bufs[op.outs[0].buf.idx].shape[0]
        t = op.type
        if t == P.OP_CONV:
            x = rd(bufs, op.ins[0])
            if op.ins[2] is not None:
                x = x * rd(bufs, op.ins[2])
            w = T(getattr(op, 'w_ref', op.w)).permute(0, 3, 1, 2).contiguous()
            bias = T(op.b) if op.b is not None else None
            padc = op.outs[0].C - w.shape[0]          # zero-padded output channels (odd-width heat map)
            if padc > 0:
                w = torch.cat([w, torch.zeros((padc,) + tuple(w.shape[1:]), dtype=w.dtype)])
            if self.emulate_split and (op.flags & (P.FLAG_TC | P.FLAG_MMA)):
                sc = np.float32(1.0 / op.floats[0])                     # the weights' power-of-two pre-scale
                y = F.conv2d(split16_round(x, self.lo_scale).permute(0, 3, 1, 2).double(),
                             (split16_round(w * sc) / sc).double(), bias.double() if bias is not None else None,
                             stride=op.s, padding=tuple(op.p), dilation=op.d).float()
            else:
                y = F.conv2d(x.permute(0, 3, 1, 2), w, bias, stride=op.s, padding=tuple(op.p), dilation=op.d)
            y = y.permute(0, 2, 3, 1)
            if op.ins[1] is not None and (op.flags & P.FLAG_RES_FIRST):
                y = _act(y + rd(bufs, op.ins[1]), op.act)          # conv-bn, += shortcut, relu
            else:
                y = _act(y, op.act)
                if op.ins[1] is not None:
                    y = y + rd(bufs, op.ins[1])
            wr(bufs, op.outs[0], y)
        elif t == P.OP_DWCONV:
            x = rd(bufs, op.ins[0])
            C = x.shape[-1]
            w = T(op.w).T.reshape(C, 1, op.k[0], op.k[1]).contiguous()
            y = F.conv2d(x.permute(0, 3, 1, 2), w, T(op.b), stride=op.s, padding=tuple(op.p),
                         dilation=op.d, groups=C)
            y = _act(y, op.act).permute(0, 2, 3, 1)
            wr(bufs, op.outs[0], y)
            if op.flags & P.FLAG_GAP_PARTIAL:
                # per-tile channel sums (8x16 output tiles, row-major), as csrc/dw_tma.cu writes them
                th, tw = P.dw_tile_rows(op.k[0], op.s[0]), P.DW_TILE_W
                Ho, Wo = y.shape[1], y.shape[2]
                parts = [y[:, a:a + th, b:b + tw].sum(dim=(1, 2)) for a in range(0, Ho, th) for b in range(0, Wo, tw)]
                wr(bufs, op.outs[1], torch.stack(parts, 1).reshape(N, len(parts), 1, -1))
        elif t == P.OP_GAP_SSE:
            x = rd(bufs, op.ins[0])                                                  # (N, H, W, C)
            ws, bs = op.w_ref
            parts = x.reshape(N, -1, 32, x.shape[-1]).sum(dim=2)                    # (N, tiles, C): 32-pixel tiles
            wr(bufs, op.outs[0], parts.reshape(N, parts.shape[1], 1, -1))
            wr(bufs, op.outs[1], _act((x * T(ws)).sum(-1, keepdim=True) + float(bs[0]), op.act))
        elif t == P.OP_SE_FC:
            w1, w2 = op.w_ref
            Cr = op.ints[1]
            mean = rd(bufs, op.ins[0]).sum(dim=(1, 2)) / np.float32(op.ints[3])          # (N, C)
            h = _act(mean @ T(w1).T + T(op.b[:Cr]), op.act)
            g = _act(h @ T(w2).T + T(op.b[Cr:]), op.ints[2])
            wr(bufs, op.outs[0], g.reshape(N, 1, 1, -1))
        elif t == P.OP_UPCAT_DW:
            low = rd(bufs, op.ins[0]).permute(0, 3, 1, 2)
            up = F.interpolate(low, scale_factor=2, mode="bilinear", align_corners=False)
            x = torch.cat([up, rd(bufs, op.ins[1]).permute(0, 3, 1, 2)], 1)
            C = x.shape[1]
            w = T(op.w).T.reshape(C, 1, 3, 3).contiguous()
            y = F.conv2d(x, w, T(op.b), padding=1, groups=C)
            wr(bufs, op.outs[0], _act(y, op.act).permute(0, 2, 3, 1))
        elif t == P.OP_DWPW:
            x = rd(bufs, op.ins[0]).permute(0, 3, 1, 2)
            if op.ins[2] is not None:
                low = rd(bufs, op.ins[2]).permute(0, 3, 1, 2)
                x = torch.cat([F.interpolate(low, scale_factor=2, mode="bilinear", align_corners=False), x], 1)
            C = x.shape[1]
            wd = T(op.dw_w).T.reshape(C, 1, 3, 3).contiguous()
            y = _act(F.conv2d(x, wd, T(op.dw_b), padding=1, groups=C), op.dw_act)
            w = T(op.w_ref).permute(0, 3, 1, 2).contiguous()
            bias = T(op.b) if op.b is not None else None
            if self.emulate_split and id(op) not in self._fp32_dwpw:     # the depthwise output enters the MMA as fp16 hi/lo
                sc = np.float32(1.0 / op.floats[0])
                y = F.conv2d(split16_round(y, self.lo_scale).double(), (split16_round(w * sc) / sc).double(),
                             bias.double() if bias is not None else None).float()
            else:
                y = F.conv2d(y, w, bias)
            y = y.permute(0, 2, 3, 1)
            if op.ins[1] is not None and (op.flags & P.FLAG_RES_FIRST):
                y = _act(y + rd(bufs, op.ins[1]), op.act)
            else:
                y = _act(y, op.act)
                if op.ins[1] is not None:
                    y = y + rd(bufs, op.ins[1])
            wr(bufs, op.outs[0], y)
        elif t == P.OP_MAXPOOL2:
            x = rd(bufs, op.ins[0]).permute(0, 3, 1, 2)
            wr(bufs, op.outs[0], F.max_pool2d(x, 2, 2, 0, ceil_mode=True).permute(0, 2, 3, 1))
        elif t == P.OP_RESIZE_NEAREST:
            x = rd(bufs, op.ins[0])
            o = op.outs[0]
            ys = (torch.arange(o.H) * x.shape[1]) // o.H
            xs = (torch.arange(o.W) * x.shape[2]) // o.W
            wr(bufs, o, x[:, ys][:, :, xs])
        elif t == P.OP_UPSAMPLE_BILINEAR2X:
            x = rd(bufs, op.ins[0]).permute(0, 3, 1, 2)
            y = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)
            wr(bufs, op.outs[0], y.permute(0, 2, 3, 1))
        elif t == P.OP_COPY:
            wr(bufs, op.outs[0], rd(bufs, op.ins[0]).clone())
        elif t == P.OP_GAP:
            wr(bufs, op.outs[0], rd(bufs, op.ins[0]).mean(dim=(1, 2), keepdim=True))
        elif t == P.OP_AFFINE_ACT:
            y = rd(bufs, op.ins[0]) * T(op.w) + T(op.b)
            wr(bufs, op.outs[0], _act(y, op.act))
        elif t == P.OP_SCSE:
            x = rd(bufs, op.ins[0])
            wr(bufs, op.outs[0], x * rd(bufs, op.ins[1]) + x * rd(bufs, op.ins[2]))
        elif t == P.OP_ADDN:
            o = op.outs[0]
            y = None
            for v in op.ins:
                if v is None:
                    continue
                x = rd(bufs, v)
                f = o.H // x.shape[1]
                if f > 1:
                    x = x.repeat_interleave(f, 1).repeat_interleave(f, 2)
                y = x if y is None else y + x
            wr(bufs, o, _act(y, op.act))
        elif t == P.OP_SCALE_CH:
            wr(bufs, op.outs[0], rd(bufs, op.ins[0]) * rd(bufs, op.ins[1]))
        elif t == P.OP_DET_DECODE:
            wr(bufs, op.outs[0], self._det_decode(op, [rd(bufs, v) for v in op.ins], N, dtype))
        elif t == P.OP_HM_DECODE:
            if len(op.ins) > 1 and op.ins[1] is not None:
                xy, sc = self._hm_decode_split(rd(bufs, op.ins[0]), rd(bufs, op.ins[1]), op.w, op.b, op.ints[0])
            else:
                xy, sc = self._hm_decode(rd(bufs, op.ins[0]), op.ints[0])
            wr(bufs, op.outs[0], xy.reshape(N, 1, 1, -1))
            wr(bufs, op.outs[1], sc.reshape(N, 1, 1, -1))
        else:
            raise NotImplementedError(t)
        if dump is not None:
            dump.append((op, [rd(bufs, o).clone() for o in op.outs]))

    @staticmethod
    def _det_decode(op, heads, N, dtype=torch.float32):
        c = op.w
        rows = []
        for si, h in enumerate(heads):
            stride = c[si * 7]
            anchors = torch.from_numpy(c[si * 7 + 1: si * 7 + 7].reshape(3, 2).copy()).to(dtype)
            H, W = h.shape[1], h.shape[2]
            t = h.reshape(N, H, W, 3, 16).permute(0, 3, 1, 2, 4)          # N,3,H,W,16
            gy, gx = torch.meshgrid(torch.arange(H, dtype=dtype), torch.arange(W, dtype=dtype), indexing="ij")
            grid = torch.stack([gx, gy], -1)[None, None]
            an = anchors[None, :, None, None, :]
            sg = torch.sigmoid(t)
            xy = (sg[..., 0:2] * 2.0 - 0.5 + grid) * stride
            wh = (sg[..., 2:4] * 2.0) ** 2 * an
            parts = [xy, wh, sg[..., 4:5]]
            for k in range(5):
                parts.append(t[..., 5 + 2 * k: 7 + 2 * k] * an + grid * stride)
            parts.append(sg[..., 15:16])
            rows.append(torch.cat(parts, -1).reshape(N, -1, 16))
        return torch.cat(rows, 1).reshape(N, -1, 1, 16)

    @staticmethod
    def _hm_decode_split(score_map, feat, w_off, b_off, npts):
        """Score maps only; the x/y offsets are the 1x1 conv rows npts..3*npts evaluated at the arg-max pixel."""
        N, H, W, C = score_map.shape
        flat = score_map.reshape(N, H * W, C)[..., :npts]
        m = flat.max(dim=1, keepdim=True).values
        ar = torch.arange(H * W).reshape(1, -1, 1)
        idx = torch.where(flat == m, ar, torch.full_like(ar, H * W)).min(dim=1).values     # N,npts
        sc = torch.gather(flat, 1, idx[:, None, :])[:, 0]
        f = feat.reshape(N, H * W, -1)
        fa = torch.gather(f, 1, idx[:, :, None].expand(N, npts, f.shape[-1]))               # N,npts,K
        wo = torch.from_numpy(w_off).to(sc.dtype)
        bo = torch.from_numpy(b_off).to(sc.dtype)
        ox = (fa * wo[:npts][None]).sum(-1) + bo[:npts]
        oy = (fa * wo[npts:][None]).sum(-1) + bo[npts:]
        x = ((idx % W).to(sc.dtype) + ox) / np.float32(W)
        y = ((idx // W).to(sc.dtype) + oy) / np.float32(W)
        return torch.stack([x, y], -1), sc

    @staticmethod
    def _hm_decode(hm, npts):
        N, H, W, C = hm.shape
        flat = hm.reshape(N, H * W, C)
        heat = flat[..., :npts]
        m = heat.max(dim=1, keepdim=True).values
        ar = torch.arange(H * W).reshape(1, -1, 1)
        idx = torch.where(heat == m, ar, torch.full_like(ar, H * W)).min(dim=1).values     # N,npts
        g = idx[:, None, :]
        sc = torch.gather(heat, 1, g)[:, 0]
        ox = torch.gather(flat[..., npts:2 * npts], 1, g)[:, 0]
        oy = torch.gather(flat[..., 2 * npts:3 * npts], 1, g)[:, 0]
        x = ((idx % W).to(sc.dtype) + ox) / np.float32(W)
        y = ((idx // W).to(sc.dtype) + oy) / np.float32(W)
        return torch.stack([x, y], -1), sc
