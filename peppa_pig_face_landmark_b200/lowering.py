"""ONNX graph -> fused execution plan (plan.Plan).

Replaces what onnxruntime's graph optimiser + kernels do for the reference
(the reference's Skps/core/api/onnx_model_base.py:14): the shipped graphs
(yolov5n-0.5.onnx, kps_student.onnx) are pattern-matched into the op set in
plan.py.  Patterns handled:

  Conv [+Sigmoid,Mul | +HardSigmoid,Mul | +Relu | +Sigmoid | +HardSigmoid] [+Add]   -> OP_CONV / OP_DWCONV
  Conv + Add(residual) + Relu (ResNet / HRNet blocks of the Teacher, model.py:302-345) -> OP_CONV, FLAG_RES_FIRST
  Add trees [+Relu] over branch tensors, nearest Resize x2^k folded in (HRNet fuse)    -> OP_ADDN
  dense-conv tensors whose channel count is not a multiple of 8 (HRNet 18/36)          -> zero-padded channels
  ReduceMean(2,3) / GlobalAveragePool                                               -> OP_GAP
  Mul(x, gate[N,C,1,1]) feeding a Conv (squeeze-excite)                             -> conv input scale
  Mul(x,cSE) + Mul(x,sSE) -> Add (scSE attention)                                   -> OP_SCSE
  Concat(axis=1), Slice(axis=1), Reshape-Transpose-Reshape channel shuffle          -> views (no data movement)
  Resize nearest / linear x2, MaxPool 2x2 ceil, BatchNormalization [+Relu]          -> small ops
  yolov5-face Detect tail (face_detector graph nodes 502-820)                       -> OP_DET_DECODE
  heat-map arg-max tail (kps graph nodes 201-410; model.py:511-554)                 -> OP_HM_DECODE

Post passes over the plan (each one a function below):
  _fuse_upsample_concat_dw   Resize(linear x2) -> Concat -> depthwise 3x3            -> OP_UPCAT_DW (no up-sampled tensor)
  _fold_affine_into_producers BatchNorm(+ReLU) over a Concat of conv outputs (ASPP)  -> folded into the producing convs
  _fuse_se_chain             depthwise -> GAP -> FC -> FC (squeeze-excite)           -> per-tile sums in the depthwise + OP_SE_FC
  _fuse_dw_pw                depthwise 3x3 / OP_UPCAT_DW -> 1x1 conv                 -> OP_DWPW (csrc/conv_xf.cu)
  _fuse_stem_block           stem 3x3 s2 -> dw+pw block -> 1x1 expand -> dw 3x3 s2    -> OP_STEM_BLOCK (csrc/stem_block.cu)
  _fuse_hm_partial           heat-map head conv -> arg-max                           -> per-tile (max, arg-max) rows, map not stored
  _fuse_gap_sse              scSE: GAP + FC + FC and the 1-channel sSE conv          -> OP_GAP_SSE + OP_SE_FC
Kernel selection for a dense conv happens in the engine (csrc/engine.cu): transposed wgmma kernel (conv_tct.cu) when
Cout fills the 128 accumulator rows, transposed arg-max head (conv_hm.cu), pixels-as-rows kernel (conv_tc.cu) otherwise.
"""
import numpy as np

from . import plan as P
from .onnx_loader import load_onnx


class LoweringError(RuntimeError):
    pass


def _fold(node, vals):
    """Constant-fold the small shape-arithmetic ops the exporters leave behind."""
    op, a = node.op, node.attrs
    x = [vals[i] if i != "" else None for i in node.inputs]
    if op == "Add":
        return x[0] + x[1]
    if op == "Sub":
        return x[0] - x[1]
    if op == "Mul":
        return x[0] * x[1]
    if op == "Div":
        if np.issubdtype(np.asarray(x[0]).dtype, np.integer):
            return np.trunc(np.asarray(x[0]) / np.asarray(x[1])).astype(np.int64)
        return x[0] / x[1]
    if op == "Gather":
        return np.take(x[0], x[1], axis=a.get("axis", 0))
    if op == "Concat":
        return np.concatenate([np.atleast_1d(v) for v in x], axis=a["axis"])
    if op == "Unsqueeze":
        out = np.asarray(x[0])
        for ax in sorted(a["axes"]):
            out = np.expand_dims(out, ax)
        return out
    if op == "Squeeze":
        return np.squeeze(x[0], axis=tuple(a["axes"]))
    if op == "Cast":
        return np.asarray(x[0]).astype({1: np.float32, 7: np.int64, 6: np.int32, 9: np.bool_}[a["to"]])
    if op == "Slice":
        data = np.asarray(x[0])
        starts, ends = np.atleast_1d(x[1]), np.atleast_1d(x[2])
        axes = np.atleast_1d(x[3]) if len(x) > 3 and x[3] is not None else np.arange(len(starts))
        steps = np.atleast_1d(x[4]) if len(x) > 4 and x[4] is not None else np.ones(len(starts), np.int64)
        idx = [slice(None)] * data.ndim
        for s, e, ax, st in zip(starts, ends, axes, steps):
            idx[int(ax)] = slice(int(s), int(min(e, np.iinfo(np.int64).max)), int(st))
        return data[tuple(idx)]
    raise LoweringError("cannot fold %s" % op)


def pad_channels(g, mult=8):
    """Zero-pad the channel count of tensors that live between dense convolutions up to a multiple of `mult`
    (HRNet-w18's 18- and 36-channel branches -> 24 and 40) so that they meet the 16-byte alignment the TMA-fed
    kernels need.  A tensor group = everything connected through Relu / Add / scale-Resize; it is padded only if
    every producer is a dense Conv and every other consumer is a dense Conv: producers get zero output rows
    (relu(0) = 0, 0 + 0 = 0 keeps the padding zero), consumers get zero input columns, so results are unchanged.
    The original channel counts stay in attrs['_macs'] for the algorithmic MAC count."""
    nodes, weights = g.nodes, dict(g.weights)
    prod = {o: i for i, n in enumerate(nodes) for o in n.outputs}
    uses = {}
    for i, n in enumerate(nodes):
        for x in n.inputs:
            uses.setdefault(x, []).append(i)
    parent = {}

    def find(a):
        parent.setdefault(a, a)
        while parent[a] != a:
            parent[a] = parent[parent[a]]
            a = parent[a]
        return a

    def data_inputs(n):
        if n.op == "Relu":
            return n.inputs[:1]
        if n.op == "Add":
            return n.inputs[:2]
        if n.op == "Resize" and not (len(n.inputs) > 3 and n.inputs[3] != ""):
            return n.inputs[:1]
        return None

    def dense(n):
        return n.op == "Conv" and n.attrs.get("group", 1) == 1 and n.inputs[1] in weights

    for n in nodes:
        di = data_inputs(n)
        if di:
            for x in di:
                parent[find(x)] = find(n.outputs[0])
    roots = {}
    for n in nodes:
        if dense(n):
            c = weights[n.inputs[1]].shape[0]
            if c % mult and c > mult:
                roots.setdefault(find(n.outputs[0]), c)
    if not roots:
        return g
    members = {}
    for name in list(parent) + [o for n in nodes for o in n.outputs]:
        r = find(name)
        if r in roots:
            members.setdefault(r, set()).add(name)
    todo = []
    for r, names in members.items():
        C, ok = roots[r], True
        for t in names:
            if t not in prod or t in g.outputs:
                ok = False
                break
            pn = nodes[prod[t]]
            if dense(pn):
                ok &= weights[pn.inputs[1]].shape[0] == C
            elif data_inputs(pn) is None:
                ok = False
            for ci in uses.get(t, []):
                cn = nodes[ci]
                di = data_inputs(cn)
                if di is not None and t in di:
                    continue
                ok &= dense(cn) and cn.inputs[0] == t and t not in cn.inputs[1:]
            if not ok:
                break
        if ok:
            todo.append((names, C))
    for names, C in todo:
        Cp = -(-C // mult) * mult
        for t in names:
            pn = nodes[prod[t]]
            if dense(pn) and weights[pn.inputs[1]].shape[0] == C:
                w = weights[pn.inputs[1]]
                pn.attrs.setdefault("_macs", [w.shape[0], w.shape[1]])
                weights[pn.inputs[1]] = np.concatenate([w, np.zeros((Cp - C,) + w.shape[1:], w.dtype)])
                if len(pn.inputs) > 2:
                    b = weights[pn.inputs[2]]
                    weights[pn.inputs[2]] = np.concatenate([b, np.zeros(Cp - C, b.dtype)])
            for ci in uses.get(t, []):
                cn = nodes[ci]
                if dense(cn) and cn.inputs[0] == t:
                    w = weights[cn.inputs[1]]
                    if w.shape[1] == C:
                        cn.attrs.setdefault("_macs", [w.shape[0], w.shape[1]])
                        weights[cn.inputs[1]] = np.concatenate(
                            [w, np.zeros((w.shape[0], Cp - C) + w.shape[2:], w.dtype)], axis=1)
    return g._replace(weights=weights)


class _T:
    """A logical NCHW tensor during lowering."""
    __slots__ = ("C", "H", "W", "home", "view", "scaled", "dtype")

    def __init__(self, C, H, W):
        self.C, self.H, self.W = C, H, W
        self.home = None      # (parent tensor name, c_off, c_stride) if it lives inside another tensor
        self.view = None
        self.scaled = None    # ('c', x, gate) / ('s', x, gate): lazily applied SE / sSE multiply
        self.dtype = P.DT_F32


_ACT_AFTER = {"Relu": P.ACT_RELU}


class _Lowerer:
    def __init__(self, graph, name, in_hw, input_u8=True, use_tc=True):
        self.use_tc = use_tc
        self.g = graph
        self.plan = P.Plan(name)
        self.nodes = graph.nodes
        self.vals = dict(graph.weights)       # name -> numpy constant
        self.t = {}                           # name -> _T
        self.uses = {}
        for i, n in enumerate(self.nodes):
            for x in n.inputs:
                self.uses.setdefault(x, []).append(i)
        self.prod = {o: i for i, n in enumerate(self.nodes) for o in n.outputs}
        self.add_inner = set()                # Add nodes folded into a later OP_ADDN
        self.absorbed = set()                 # node indices consumed by a fusion
        self.fused = {}                       # conv node idx -> dict(act, out, res)
        self.pending_copies = {}              # node idx -> [(src tensor, dst tensor)]
        self.in_hw = in_hw
        self.input_u8 = input_u8
        self.decode_derived = set()
        self.det_heads = []

    # ------------------------------------------------------------------ helpers
    def users(self, name):
        return [self.nodes[i] for i in self.uses.get(name, [])]

    def user_idx(self, name):
        return self.uses.get(name, [])

    def is_const(self, name):
        return name in self.vals

    def shape_of(self, name):
        t = self.t[name]
        return [1, t.C, t.H, t.W]

    # ------------------------------------------------------------------ pass A: shapes, fusions, homes
    def analyse(self):
        g = self.g
        inp = g.inputs[0]
        self.t[inp] = _T(3, self.in_hw[0], self.in_hw[1])
        self.input_name = inp
        for idx, n in enumerate(self.nodes):
            if idx in self.absorbed:
                continue
            self._analyse_node(idx, n)

    def _set(self, name, C, H, W):
        self.t[name] = _T(C, H, W)
        return self.t[name]

    def _analyse_node(self, idx, n):
        op = n.op
        if op == "Constant":
            self.vals[n.outputs[0]] = np.asarray(n.attrs["value"])
            return
        ins = n.inputs
        if any(i in self.decode_derived for i in ins):
            self.decode_derived.update(n.outputs)
            return
        if op == "Shape" and ins[0] in self.t:
            self.vals[n.outputs[0]] = np.array(self.shape_of(ins[0]), np.int64)
            return
        if all((i == "" or i in self.vals) for i in ins) and op not in ("Conv",):
            if op == "ConstantOfShape" or op == "Equal" or op == "Where" or op == "Expand":
                self.decode_derived.update(n.outputs)   # only appears inside decode tails
                return
            self.vals[n.outputs[0]] = _fold(n, self.vals)
            return
        x = self.t.get(ins[0])
        if op == "Conv":
            w = self.vals[ins[1]]
            a = n.attrs
            k, s, d, p = a["kernel_shape"], a["strides"], a["dilations"], a["pads"]
            Ho = (x.H + 2 * p[0] - d[0] * (k[0] - 1) - 1) // s[0] + 1
            Wo = (x.W + 2 * p[1] - d[1] * (k[1] - 1) - 1) // s[1] + 1
            out = n.outputs[0]
            self._set(out, w.shape[0], Ho, Wo)
            self._fuse_after_conv(idx, n, out)
            return
        if op in ("Relu", "Sigmoid", "HardSigmoid"):
            # stand-alone activation not fused into a conv: only BatchNormalization->Relu here
            self._set(n.outputs[0], x.C, x.H, x.W)
            return
        if op == "BatchNormalization":
            self._set(n.outputs[0], x.C, x.H, x.W)
            us = self.user_idx(n.outputs[0])
            if len(us) == 1 and self.nodes[us[0]].op == "Relu":
                self.absorbed.add(us[0])
                self.fused[idx] = dict(act=P.ACT_RELU, out=self.nodes[us[0]].outputs[0])
                self._set(self.nodes[us[0]].outputs[0], x.C, x.H, x.W)
            else:
                self.fused[idx] = dict(act=P.ACT_NONE, out=n.outputs[0])
            return
        if op in ("ReduceMean", "GlobalAveragePool"):
            if op == "ReduceMean":
                assert sorted(n.attrs["axes"]) == [2, 3] and n.attrs.get("keepdims", 1) == 1
            self._set(n.outputs[0], x.C, 1, 1)
            return
        if op == "MaxPool":
            assert n.attrs["kernel_shape"] == [2, 2] and n.attrs["strides"] == [2, 2] and n.attrs.get("ceil_mode", 0) == 1
            self._set(n.outputs[0], x.C, -(-x.H // 2), -(-x.W // 2))
            return
        if op == "Resize":
            if len(ins) > 3 and ins[3] != "" and np.asarray(self.vals[ins[3]]).size > 0:
                size = [int(v) for v in np.asarray(self.vals[ins[3]]).reshape(-1)[2:]]
            else:
                sc = np.asarray(self.vals[ins[2]]).reshape(-1)
                size = [int(np.floor(x.H * sc[2])), int(np.floor(x.W * sc[3]))]
            self._set(n.outputs[0], x.C, size[0], size[1])
            return
        if op == "Mul":
            a_, b_ = self.t.get(ins[0]), self.t.get(ins[1])
            if a_ is None or b_ is None:
                raise LoweringError("Mul with constant operand outside decode: %s" % n.name)
            big, small = (ins[0], ins[1]) if (a_.H * a_.W * a_.C >= b_.H * b_.W * b_.C) else (ins[1], ins[0])
            tb, ts = self.t[big], self.t[small]
            o = self._set(n.outputs[0], tb.C, tb.H, tb.W)
            if ts.H == 1 and ts.W == 1 and ts.C == tb.C:
                o.scaled = ("c", big, small)
            elif ts.C == 1 and ts.H == tb.H and ts.W == tb.W:
                o.scaled = ("s", big, small)
            else:
                raise LoweringError("unsupported Mul %s" % n.name)
            return
        if op == "Add":
            a_, b_ = self.t[ins[0]], self.t[ins[1]]
            if a_.scaled and b_.scaled and a_.scaled[1] == b_.scaled[1] and {a_.scaled[0], b_.scaled[0]} == {"c", "s"}:
                self._set(n.outputs[0], a_.C, a_.H, a_.W)
                return
            if a_.scaled or b_.scaled or a_.C != b_.C:
                raise LoweringError("unfused Add %s" % n.name)
            self._analyse_add(idx, n, a_, b_)
            return
        if op == "Concat":
            assert n.attrs["axis"] == 1
            parts = [self.t[i] for i in ins]
            C = sum(p.C for p in parts)
            out = n.outputs[0]
            shuffle = self._match_shuffle(idx, out, C, parts[0].H, parts[0].W)
            if shuffle is not None:
                out = shuffle
                assert len(parts) == 2 and parts[0].C == parts[1].C
            self._set(out, C, parts[0].H, parts[0].W)
            off = 0
            copies = []
            for gi, (nm, p) in enumerate(zip(ins, parts)):
                spec = (out, gi, 2) if shuffle is not None else (out, off, 1)
                if p.home is None and nm != self.input_name and not self._is_alias(nm):
                    p.home = spec
                else:
                    copies.append((nm, spec, p.C))
                off += p.C
            if copies:
                self.pending_copies[idx] = copies
            return
        if op == "Slice":
            starts = np.atleast_1d(self.vals[ins[1]])
            ends = np.atleast_1d(self.vals[ins[2]])
            axes = np.atleast_1d(self.vals[ins[3]]) if len(ins) > 3 else np.array([0])
            assert len(starts) == 1 and int(axes[0]) == 1
            s, e = int(starts[0]), int(min(int(ends[0]), x.C))
            o = self._set(n.outputs[0], e - s, x.H, x.W)
            o.home = (ins[0], s, 1)
            self.alias = getattr(self, "alias", set())
            self.alias.add(n.outputs[0])
            return
        if op == "Reshape" and ins[0] in self.t:
            shape = [int(v) for v in np.asarray(self.vals[ins[1]]).reshape(-1)]
            if len(shape) == 5 and shape[1] == 3 and shape[2] == 16:
                # Detect head: everything downstream is the decode tail
                self.det_heads.append(ins[0])
                self.decode_derived.update(n.outputs)
                return
            raise LoweringError("unsupported Reshape %s -> %s" % (n.name, shape))
        raise LoweringError("unsupported op %s (%s)" % (op, n.name))

    def _analyse_add(self, idx, n, a_, b_):
        """Plain tensor Add: part of an OP_ADDN (sum tree, nearest Resize operands read in place, trailing Relu)."""
        out = n.outputs[0]
        H, W = max(a_.H, b_.H), max(a_.W, b_.W)
        self._set(out, a_.C, H, W)
        us = self.user_idx(out)
        if len(us) == 1 and self.nodes[us[0]].op == "Add":
            other = [i for i in self.nodes[us[0]].inputs if i != out]
            if len(other) == 1 and other[0] in self.t and not self.t[other[0]].scaled:
                self.add_inner.add(idx)          # folded into the Add that consumes it
                return
        leaves = []

        def gather(name):
            pi = self.prod.get(name)
            if pi is not None and pi in self.add_inner:
                for i in self.nodes[pi].inputs:
                    gather(i)
                return
            pn = self.nodes[pi] if pi is not None else None
            if (pn is not None and pn.op == "Resize" and pn.attrs.get("mode") == "nearest"
                    and len(self.user_idx(name)) == 1 and pi not in self.absorbed):
                src = self.t[pn.inputs[0]]
                f = self.t[name].H // src.H
                if src.H * f == self.t[name].H and src.W * f == self.t[name].W and f & (f - 1) == 0 \
                        and src.home is None and not src.scaled:
                    self.absorbed.add(pi)
                    leaves.append(pn.inputs[0])
                    return
            leaves.append(name)

        for i in n.inputs:
            gather(i)
        if len(leaves) > 4:
            raise LoweringError("Add tree with %d operands at %s" % (len(leaves), n.name))
        act, cur = P.ACT_NONE, out
        if len(us) == 1 and self.nodes[us[0]].op == "Relu":
            self.absorbed.add(us[0])
            act, cur = P.ACT_RELU, self.nodes[us[0]].outputs[0]
            self._set(cur, a_.C, H, W)
        self.fused[idx] = dict(kind="addn", leaves=leaves, act=act, out=cur)

    def _is_alias(self, nm):
        return nm in getattr(self, "alias", set())

    def _match_shuffle(self, idx, out, C, H, W):
        us = self.user_idx(out)
        if len(us) != 1 or self.nodes[us[0]].op != "Reshape":
            return None
        r1 = self.nodes[us[0]]
        # the reshape target is a Constant node that may come later in file order
        shp = self._const_of(r1.inputs[1])
        if shp is None or list(shp) != [1, 2, C // 2, H, W]:
            return None
        u2 = self.user_idx(r1.outputs[0])
        tr = self.nodes[u2[0]]
        if len(u2) != 1 or tr.op != "Transpose" or tr.attrs["perm"] != [0, 2, 1, 3, 4]:
            return None
        u3 = self.user_idx(tr.outputs[0])
        r2 = self.nodes[u3[0]]
        shp2 = self._const_of(r2.inputs[1])
        if len(u3) != 1 or r2.op != "Reshape" or list(shp2) not in ([1, C, H, W], [1, -1, H, W]):
            return None
        self.absorbed.update([us[0], u2[0], u3[0]])
        return r2.outputs[0]

    def _const_of(self, name):
        if name in self.vals:
            return np.asarray(self.vals[name]).reshape(-1)
        for n in self.nodes:
            if n.op == "Constant" and n.outputs[0] == name:
                return np.asarray(n.attrs["value"]).reshape(-1)
        return None

    def _fuse_after_conv(self, idx, n, out):
        t = self.t[out]
        us = self.user_idx(out)
        ops = sorted(self.nodes[u].op for u in us)
        act, cur = P.ACT_NONE, out
        if ops == ["Slice"] * 3 and any(m.op == "ArgMax" for m in self.nodes):
            # heat-map head: the three Slices start the arg-max decode tail
            for u in us:
                self.absorbed.add(u)
                self.decode_derived.update(self.nodes[u].outputs)
            self.fused[idx] = dict(act=P.ACT_NONE, out=out, res=None)
            return
        if ops == ["Relu"]:
            act, cur = P.ACT_RELU, self.nodes[us[0]].outputs[0]
            self.absorbed.add(us[0])
        elif ops in (["Mul", "Sigmoid"], ["HardSigmoid", "Mul"]):
            gate = [u for u in us if self.nodes[u].op != "Mul"][0]
            mul = [u for u in us if self.nodes[u].op == "Mul"][0]
            gout = self.nodes[gate].outputs[0]
            if sorted(self.nodes[mul].inputs) == sorted([out, gout]) and self.user_idx(gout) == [mul]:
                act = P.ACT_SILU if self.nodes[gate].op == "Sigmoid" else P.ACT_HSWISH
                if act == P.ACT_HSWISH:
                    self._check_hsig(self.nodes[gate])
                cur = self.nodes[mul].outputs[0]
                self.absorbed.update([gate, mul])
        elif ops == ["Sigmoid"]:
            act, cur = P.ACT_SIGMOID, self.nodes[us[0]].outputs[0]
            self.absorbed.add(us[0])
        elif ops == ["HardSigmoid"]:
            self._check_hsig(self.nodes[us[0]])
            act, cur = P.ACT_HSIGMOID, self.nodes[us[0]].outputs[0]
            self.absorbed.add(us[0])
        res, res_first = None, False
        u2 = self.user_idx(cur)
        if len(u2) == 1 and self.nodes[u2[0]].op == "Add":
            add = self.nodes[u2[0]]
            other = [i for i in add.inputs if i != cur]
            if len(other) == 1 and other[0] in self.t and not self.t[other[0]].scaled \
                    and self.prod.get(other[0], -1) < idx:
                o = self.t[other[0]]
                if (o.C, o.H, o.W) == (t.C, t.H, t.W):
                    res = other[0]
                    self.absorbed.add(u2[0])
                    cur = add.outputs[0]
                    u3 = self.user_idx(cur)
                    if act == P.ACT_NONE and len(u3) == 1 and self.nodes[u3[0]].op == "Relu":
                        # conv-bn, += shortcut, relu (timm BasicBlock / Bottleneck): the activation follows the add
                        self.absorbed.add(u3[0])
                        act, cur, res_first = P.ACT_RELU, self.nodes[u3[0]].outputs[0], True
        if cur != out:
            self._set(cur, t.C, t.H, t.W)
        self.fused[idx] = dict(act=act, out=cur, res=res, res_first=res_first)

    @staticmethod
    def _check_hsig(node):
        al = node.attrs.get("alpha", 0.2)
        be = node.attrs.get("beta", 0.5)
        if abs(al - 1.0 / 6.0) > 1e-6 or be != 0.5:
            raise LoweringError("HardSigmoid alpha/beta %r/%r" % (al, be))

    # ------------------------------------------------------------------ views
    def view(self, name):
        t = self.t[name]
        if t.view is not None:
            return t.view
        if t.home is not None:
            parent, off, stride = t.home
            t.view = self.view(parent).sub(off, t.C, stride)
        else:
            # pixel rows of odd width (the 294-channel heat map) are padded to a multiple of 8 channels so
            # every kernel can use 16-byte vector stores; the view keeps the logical channel count
            ld = t.C if (t.C % 8 == 0 or t.C <= 8 or t.H * t.W == 1) else -(-t.C // 8) * 8
            b = self.plan.new_buf(ld, t.H, t.W, t.dtype, name)
            t.view = P.View(b, 0, 1, t.C)
        return t.view

    # ------------------------------------------------------------------ pass B: emission
    def emit(self):
        pl = self.plan
        tin = self.t[self.input_name]
        tin.dtype = P.DT_U8 if self.input_u8 else P.DT_F32
        pl.input = self.view(self.input_name)
        for idx, n in enumerate(self.nodes):
            if idx in self.absorbed or n.op == "Constant":
                continue
            if any(i in self.decode_derived for i in n.inputs) or n.outputs[0] in self.decode_derived:
                continue
            if n.outputs[0] in self.vals:
                continue
            self._emit_node(idx, n)
            if getattr(self, "done", False):
                break
        if self.det_heads:
            self._emit_det_decode()

    def _mma_eligible(self, xin, out_v, k, s, p, d, flags, gate):
        """csrc/conv_mma.cu: 3x3 stride-1 'same' convs with Cin == Cout in {24, 40} reading a SPLIT16-able view."""
        if not self.use_tc or (flags & P.FLAG_IN_U8) or gate is not None:
            return False
        if list(k) != [3, 3] or list(s) != [1, 1] or list(d) != [1, 1] or list(p[:2]) != [1, 1]:
            return False
        # the whole weight set stays resident (one 4-warp CTA per SM: 115 KB of shared memory), which pays off for the
        # thinnest layers only: just the 24-channel layers are routed here (not re-measured on H100)
        if xin.C != out_v.C or xin.C != 24 or xin.buf.dtype == P.DT_U8:
            return False
        if xin.c_stride != 1 or out_v.c_stride != 1 or (xin.buf.C | xin.c_off) % 8 or (out_v.buf.C | out_v.c_off) % 8:
            return False
        return xin.H >= 8 and xin.W >= 16

    def _tc_eligible(self, xin, k, s, p, d, flags, cout=0, gate=None):
        """Shapes csrc/conv_tc.cu handles: stride-1/2 'same' square convs whose 128-pixel output tiles are whole
        image-row blocks (or whole images for maps under 128 pixels), channel windows aligned for TMA
        (16-byte rows of float16)."""
        if not self.use_tc or (flags & P.FLAG_IN_U8) or xin.buf.dtype == P.DT_U8:
            return False
        if list(k) == [1, 1] and list(s) == [1, 1] and cout == 16 and xin.C <= 32 \
                and xin.H * xin.W >= 1024 and gate is None:
            return False          # HBM-bound thin pointwise layer: csrc/ops_misc.cu pw_small_kernel (CUDA cores)
        # stride-2 convs ride on TMA element strides
        if s[0] != s[1] or s[0] not in (1, 2) or k[0] != k[1] or d[0] != d[1] or p[0] != p[1] \
                or p[0] != d[0] * (k[0] - 1) // 2:
            return False
        if xin.c_stride != 1 or xin.C % 8 or xin.c_off % 8 or xin.buf.C % 8:
            return False
        if xin.H % s[0] or xin.W % s[0]:
            return False
        H, W = xin.H // s[0], xin.W // s[0]              # output map: 128-pixel tiles = row blocks, or whole images
        if W < 8:
            return False
        if H * W < 128:                                  # several whole images per tile
            return 128 % W == 0 and 128 % (H * W) == 0
        if (W % 128 == 0) if W >= 128 else (128 % W == 0 and H % (128 // W) == 0):
            return True
        # any other map: ragged bw x 128/bw tiles (mirrors csrc/conv_tc.cu tc_pick_bw)
        return any(bw <= W + 7 and 128 // bw <= H + 7 for bw in (64, 32, 16, 8))

    def _xf_scale_ok(self, xin, gate, out_v, k, s, cout):
        """Mirror of csrc/conv_xf.cu xf_supported() for XF_SCALE: 1x1 stride-1 conv, one N tile, 16x8 pixel tiles."""
        if list(k) != [1, 1] or list(s) != [1, 1] or P.tc_tiling(cout)[1] != 1:
            return False
        if gate.c_stride != 1 or (gate.buf.C | gate.c_off) % 4 or gate.buf.dtype != P.DT_F32:
            return False
        return xin.H >= 8 and xin.W >= 16 and -(-xin.C // 64) <= 16 and out_v.c_stride == 1

    def _conv_input(self, name):
        """Resolve a conv's input: plain view, or (view, gate view) for an SE-scaled tensor."""
        t = self.t[name]
        if t.scaled:
            kind, x, gate = t.scaled
            if kind != "c":
                raise LoweringError("sSE-scaled tensor feeding a conv")
            return self.view(x), self.view(gate)
        return self.view(name), None

    def _emit_node(self, idx, n):
        pl, op = self.plan, n.op
        ins = n.inputs
        if op == "Conv":
            f = self.fused[idx]
            a = n.attrs
            w = self.vals[ins[1]].astype(np.float32)
            b = self.vals[ins[2]].astype(np.float32) if len(ins) > 2 else None
            k, s, d, p = a["kernel_shape"], a["strides"], a["dilations"], a["pads"]
            assert p[0] == p[2] and p[1] == p[3]
            groups = a.get("group", 1)
            xin, gate = self._conv_input(ins[0])
            out_t = self.t[f["out"]]
            hm_split = None
            if groups == 1 and list(k) == [1, 1] and self._is_hm_head(f["out"]) and gate is None \
                    and w.shape[0] % 3 == 0 and b is not None:
                # heat-map head (model.py:511-554 postp): only the score maps are needed densely; the x/y offset maps are
                # read at ONE pixel per landmark (the arg-max), so the conv computes the first third of its channels and the
                # decode kernel evaluates the two offset dot products at that pixel from the conv's input
                npts = w.shape[0] // 3
                hm_split = dict(npts=npts, xin=xin, w=np.ascontiguousarray(w[npts:].reshape(2 * npts, -1)), b=b[npts:].copy())
                self.macs_unsplit = out_t.H * out_t.W * w.shape[1] * 2 * npts       # algorithmic MACs stay those of the graph
                w, b = w[:npts], b[:npts]
                out_t.C = npts
            out_v = self.view(f["out"])
            flags = P.FLAG_RES_FIRST if f.get("res_first") else 0
            if ins[0] == self.input_name and self.input_u8:
                flags |= P.FLAG_IN_U8
            mc = a.get("_macs", [w.shape[0], w.shape[1]])          # channel counts before pad_channels()
            assert xin.c_stride == 1, "strided input view"
            if groups == 1:
                wk = np.ascontiguousarray(w.transpose(0, 2, 3, 1))      # [Cout][kh][kw][Cin]
                res = self.view(f["res"]) if f.get("res") else None
                if self._mma_eligible(xin, out_v, k, s, p, d, flags, gate):
                    # few-channel 3x3 (HRNet 18/36-channel branches, padded to 24/40): halo tile fetched once, taps from smem
                    xin.buf.dtype = P.DT_SPLIT16
                    packed, out_scale = P.pack_mma_weights(wk)
                    o = P.Op(P.OP_CONV, [xin, res, None], [out_v], f["act"], k, s, p[:2], d, packed,
                             b if b is not None else np.zeros(out_v.C, np.float32), flags | P.FLAG_MMA, floats=[out_scale],
                             name=n.name)
                elif self._tc_eligible(xin, k, s, p, d, flags, out_v.C, gate):
                    # tensor-core path (csrc/conv_tc.cu): float16 hi/lo operands, input buffer in SPLIT16 format
                    xf_flag = 0
                    if gate is not None and self._xf_scale_ok(xin, gate, out_v, k, s, w.shape[0]):
                        # squeeze-excite scale applied to the A tiles in shared memory by the conv kernel itself
                        # (csrc/conv_xf.cu, XF_SCALE): the expanded tensor is read once, no separate scale pass
                        xf_flag = P.FLAG_XF
                    elif gate is not None:
                        # squeeze-excite scale cannot ride on a TMA-fed operand: apply it in its own pass
                        sb = pl.new_buf(xin.C, xin.H, xin.W, P.DT_SPLIT16, n.name + ":se_scaled")
                        sv = P.View(sb, 0, 1, xin.C)
                        pl.ops.append(P.Op(P.OP_SCALE_CH, [xin, gate], [sv], name=n.name + ":se_scale"))
                        xin, gate = sv, None
                    xin.buf.dtype = P.DT_SPLIT16
                    wk_tc, b_tc = wk, b
                    if (out_v.C % 8 and out_v.c_off == 0 and out_v.c_stride == 1 and out_v.buf.C % 8 == 0
                            and out_v.buf.C - out_v.C < 8):
                        # odd channel count (the 294-wide heat map): also write the buffer's zero padding channels so
                        # the epilogue can use whole 16-byte groups / TMA stores; consumers keep the logical view
                        padc = out_v.buf.C - out_v.C
                        wk_tc = np.concatenate([wk, np.zeros((padc,) + wk.shape[1:], np.float32)])
                        b_tc = np.concatenate([b if b is not None else np.zeros(out_v.C, np.float32),
                                               np.zeros(padc, np.float32)])
                        out_v = P.View(out_v.buf, 0, 1, out_v.buf.C)
                    n_tile, n_tiles = P.tc_tiling(wk_tc.shape[0])
                    hi, lo, out_scale = P.pack_tc_weights(wk_tc, n_tile, n_tiles)
                    b = b_tc
                    o = P.Op(P.OP_CONV, [xin, res, gate if xf_flag else None], [out_v], f["act"], k, s, p[:2], d, hi, b,
                             flags | P.FLAG_TC | xf_flag, ints=[n_tile, n_tiles, 0, 0], floats=[out_scale], name=n.name)
                    o.w2 = lo
                else:
                    o = P.Op(P.OP_CONV, [xin, res, gate], [out_v], f["act"], k, s, p[:2], d, wk, b, flags,
                             name=n.name)
                o.w_ref = wk
                pl.macs += mc[0] * out_t.H * out_t.W * mc[1] * k[0] * k[1]
                if hm_split is not None:
                    pl.macs += self.macs_unsplit
                    self.hm_split = hm_split
            else:
                assert groups == w.shape[0] and w.shape[1] == 1 and gate is None and not f.get("res")
                wk = np.ascontiguousarray(w.reshape(w.shape[0], -1).T)    # [kh*kw][C]
                o = P.Op(P.OP_DWCONV, [xin], [out_v], f["act"], k, s, p[:2], d, wk,
                         b if b is not None else np.zeros(w.shape[0], np.float32), flags, name=n.name)
                pl.macs += out_t.C * out_t.H * out_t.W * k[0] * k[1]
            pl.ops.append(o)
            self._maybe_hm_decode(f["out"])
            return
        if op in ("ReduceMean", "GlobalAveragePool"):
            pl.ops.append(P.Op(P.OP_GAP, [self.view(ins[0])], [self.view(n.outputs[0])], name=n.name))
            return
        if op == "MaxPool":
            pl.ops.append(P.Op(P.OP_MAXPOOL2, [self.view(ins[0])], [self.view(n.outputs[0])], name=n.name))
            return
        if op == "Resize":
            a = n.attrs
            src, dst = self.view(ins[0]), self.view(n.outputs[0])
            if a["mode"] == "nearest":
                assert a["coordinate_transformation_mode"] == "asymmetric" and a["nearest_mode"] == "floor"
                pl.ops.append(P.Op(P.OP_RESIZE_NEAREST, [src], [dst], name=n.name))
            else:
                assert a["mode"] == "linear" and a["coordinate_transformation_mode"] == "half_pixel"
                assert dst.H == 2 * src.H and dst.W == 2 * src.W
                pl.ops.append(P.Op(P.OP_UPSAMPLE_BILINEAR2X, [src], [dst], name=n.name))
            return
        if op == "BatchNormalization":
            f = self.fused[idx]
            sc, bi, mean, var = [self.vals[i].astype(np.float32) for i in ins[1:5]]
            eps = np.float32(n.attrs.get("epsilon", 1e-5))
            inv = (sc / np.sqrt(var + eps)).astype(np.float32)
            shift = (bi - mean * inv).astype(np.float32)
            pl.ops.append(P.Op(P.OP_AFFINE_ACT, [self.view(ins[0])], [self.view(f["out"])], f["act"],
                               w=inv, b=shift, name=n.name))
            return
        if op == "Concat":
            for src, spec, C in self.pending_copies.get(idx, []):
                parent, off, stride = spec
                dst = self.view(parent).sub(off, C, stride)
                pl.ops.append(P.Op(P.OP_COPY, [self.view(src)], [dst], name=n.name + ":copy"))
            return
        if op == "Mul":
            return      # lazily-applied SE / scSE scale
        if op == "Add" and idx in self.add_inner:
            return
        if op == "Add" and self.fused.get(idx, {}).get("kind") == "addn":
            f = self.fused[idx]
            pl.ops.append(P.Op(P.OP_ADDN, [self.view(x) for x in f["leaves"]], [self.view(f["out"])], f["act"],
                               name=n.name))
            return
        if op == "Add":
            a_, b_ = self.t[ins[0]], self.t[ins[1]]
            c_t, s_t = (a_, b_) if a_.scaled[0] == "c" else (b_, a_)
            x = c_t.scaled[1]
            pl.ops.append(P.Op(P.OP_SCSE, [self.view(x), self.view(c_t.scaled[2]), self.view(s_t.scaled[2])],
                               [self.view(n.outputs[0])], name=n.name))
            return
        if op == "Slice":
            return
        raise LoweringError("emit: unsupported %s %s" % (op, n.name))

    # ------------------------------------------------------------------ decode tails
    def _is_hm_head(self, name):
        us = self.users(name)
        return bool(us) and len(us) == 3 and all(u.op == "Slice" for u in us) and any(n.op == "ArgMax" for n in self.nodes)

    def _maybe_hm_decode(self, name):
        us = self.users(name)
        if not self._is_hm_head(name):
            return
        t = self.t[name]
        bounds = sorted(int(np.atleast_1d(self._const_of(u.inputs[1]))[0]) for u in us)
        npts = bounds[1]
        split = getattr(self, "hm_split", None)
        if bounds != [0, npts, 2 * npts] or t.C != (npts if split else 3 * npts):
            raise LoweringError("unexpected heat-map slicing %s" % bounds)
        mods = [n for n in self.nodes if n.op == "Mod"]
        side = int(np.asarray(self._const_of(mods[0].inputs[1])).reshape(-1)[0])
        if side != t.W or t.H != t.W:
            raise LoweringError("heat-map side %d vs %dx%d" % (side, t.H, t.W))
        pl = self.plan
        xy = pl.new_buf(2 * npts, 1, 1, P.DT_F32, "output")
        sc = pl.new_buf(npts, 1, 1, P.DT_F32, "score")
        vxy, vsc = P.View(xy, 0, 1, 2 * npts), P.View(sc, 0, 1, npts)
        if split:
            xin = split["xin"]
            pl.ops.append(P.Op(P.OP_HM_DECODE, [self.view(name), xin], [vxy, vsc], w=split["w"], b=split["b"],
                               ints=[npts, xin.C], name="hm_decode"))
        else:
            pl.ops.append(P.Op(P.OP_HM_DECODE, [self.view(name)], [vxy, vsc], ints=[npts], name="hm_decode"))
        # graph outputs are ['output' (1,196), 'score' (1,98)] in that order
        assert len(self.g.outputs) == 2
        pl.outputs = [vxy, vsc]
        self.done = True

    def _emit_det_decode(self):
        pl = self.plan
        assert len(self.det_heads) == 3
        views = [self.view(h) for h in self.det_heads]
        consts = []
        rows = 0
        for h in self.det_heads:
            t = self.t[h]
            stride, anchors = self._det_constants(h, t)
            consts += [stride] + anchors
            rows += 3 * t.H * t.W
        out = pl.new_buf(16, rows, 1, P.DT_F32, "output")     # (N, rows, 16) stored as H=rows, W=1, C=16
        ov = P.View(out, 0, 1, 16)
        pl.ops.append(P.Op(P.OP_DET_DECODE, views, [ov], w=np.array(consts, np.float32), ints=[rows],
                           name="det_decode"))
        pl.outputs = [ov]

    def _det_constants(self, head, t):
        """Dig stride and the three (w,h) anchors of one scale out of the Detect tail's constants."""
        # nodes downstream of this head until the next head
        start = [i for i, n in enumerate(self.nodes) if head in n.inputs][0]
        stride, anchors, grid_ok = None, None, False
        i = start
        seen_pow = False
        while i < len(self.nodes):
            n = self.nodes[i]
            if n.op == "Conv":
                break
            if n.op == "Pow":
                seen_pow = True
                mul = self.nodes[self.user_idx(n.outputs[0])[0]]
                c = [self._const_full(x) for x in mul.inputs if self._const_full(x) is not None][0]
                assert c.shape == (1, 3, t.H, t.W, 2) and np.ptp(c, axis=(2, 3)).max() == 0
                anchors = [float(v) for v in c[0, :, 0, 0, :].reshape(-1)]
            if n.op == "Sub" and stride is None:
                add = self.nodes[self.user_idx(n.outputs[0])[0]]
                grid = [self._const_full(x) for x in add.inputs if self._const_full(x) is not None][0]
                gx, gy = np.meshgrid(np.arange(t.W), np.arange(t.H))
                assert np.array_equal(grid[0, 0, :, :, 0], gx) and np.array_equal(grid[0, 2, :, :, 1], gy)
                grid_ok = True
                mul = self.nodes[self.user_idx(add.outputs[0])[0]]
                sc = [self._const_full(x) for x in mul.inputs if self._const_full(x) is not None][0]
                stride = float(np.asarray(sc).reshape(-1)[0])
            i += 1
        if not (seen_pow and grid_ok and stride and anchors):
            raise LoweringError("could not recover Detect constants for %s" % head)
        return stride, anchors

    def _const_full(self, name):
        if name in self.vals:
            return np.asarray(self.vals[name])
        for n in self.nodes:
            if n.op == "Constant" and n.outputs[0] == name:
                return np.asarray(n.attrs["value"])
        return None


def _fuse_upsample_concat_dw(pl):
    """Resize(linear x2) -> Concat(skip) -> depthwise 3x3 (the head of each DecoderBlock, model.py:133-196)
    becomes one OP_UPCAT_DW that interpolates on the fly; the up-sampled tensor is never written."""
    for d in list(pl.ops):
        if d.type != P.OP_DWCONV or list(d.k) != [3, 3] or list(d.s) != [1, 1] or list(d.d) != [1, 1] or list(d.p) != [1, 1]:
            continue
        x = d.ins[0]
        if x.c_off != 0 or x.c_stride != 1 or x.C != x.buf.C:
            continue
        ups = [u for u in pl.ops if u.type == P.OP_UPSAMPLE_BILINEAR2X and u.outs[0].buf is x.buf and u.outs[0].c_off == 0
               and u.outs[0].c_stride == 1]
        if len(ups) != 1:
            continue
        u = ups[0]
        cu = u.outs[0].C
        readers = [o for o in pl.ops if o is not d and any(v is not None and v.buf is x.buf and v.c_off < cu for v in o.ins)]
        low = u.ins[0]
        ok8 = all(v % 8 == 0 for v in (cu, x.C - cu, x.buf.C, low.C, low.buf.C, low.c_off,
                                      d.outs[0].buf.C, d.outs[0].c_off))
        if readers or low.c_stride != 1 or d.outs[0].c_stride != 1 or not ok8 or cu >= x.C:
            continue
        d.type = P.OP_UPCAT_DW
        x.buf.name += ":skip-only"         # the first `cu` channels of this buffer are never written any more
        d.ins = [low, P.View(x.buf, cu, 1, x.C - cu)]
        pl.ops.remove(u)


def _dw_tma_ok(op):
    """Mirror of csrc/dw_tma.cu dw_tma_supported(): layers the TMA-staged depthwise kernel takes."""
    k, s, d, p = op.k, op.s, op.d, op.p
    if k[0] != k[1] or s[0] != s[1] or d[0] != d[1] or p[0] != p[1]:
        return False
    if (k[0], s[0], d[0]) not in ((3, 1, 1), (3, 2, 1), (5, 1, 1), (5, 2, 1), (5, 1, 2)) or p[0] != d[0] * (k[0] - 1) // 2:
        return False
    x, o = op.ins[0], op.outs[0]
    if x.c_stride != 1 or o.c_stride != 1 or x.C != o.C or x.buf.dtype == P.DT_U8:
        return False
    return not ((x.C | x.buf.C | x.c_off | o.buf.C | o.c_off) & 7)


def _fuse_se_chain(pl):
    """depthwise -> GlobalAveragePool -> 1x1 (+Relu) -> 1x1 (+HardSigmoid): the pooling pass over the depthwise output
    disappears (the depthwise kernel writes per-tile channel sums, FLAG_GAP_PARTIAL) and the two tiny FCs become one
    OP_SE_FC launch.  mobilenetv3 squeeze-excite blocks of the student encoder (kps_student.onnx .../se/*)."""
    def same(a, b):
        return a is not None and b is not None and a.buf is b.buf and (a.c_off, a.c_stride, a.C) == (b.c_off, b.c_stride, b.C)

    def readers(v, skip):
        return [o for o in pl.ops if o not in skip and any(same(i, v) for i in o.ins)]

    for gap in list(pl.ops):
        if gap.type != P.OP_GAP:
            continue
        i = pl.ops.index(gap)
        dws = [o for o in pl.ops[:i] if o.type == P.OP_DWCONV and same(o.outs[0], gap.ins[0])]
        if len(dws) != 1 or not _dw_tma_ok(dws[0]) or len(dws[0].outs) != 1:
            continue
        dw = dws[0]
        fc1 = readers(gap.outs[0], [gap])
        if len(fc1) != 1 or fc1[0].type != P.OP_CONV or list(fc1[0].k) != [1, 1] or (fc1[0].flags & P.FLAG_TC) \
                or fc1[0].ins[1] is not None or fc1[0].ins[2] is not None:
            continue
        fc1 = fc1[0]
        fc2 = readers(fc1.outs[0], [fc1])
        if len(fc2) != 1 or fc2[0].type != P.OP_CONV or list(fc2[0].k) != [1, 1] or (fc2[0].flags & P.FLAG_TC) \
                or fc2[0].ins[1] is not None or fc2[0].ins[2] is not None:
            continue
        fc2 = fc2[0]
        C, Cr = dw.outs[0].C, fc1.outs[0].C
        if fc2.outs[0].C != C or fc1.ins[0].C != C or (C + Cr) * 8 * 4 > 96 * 1024 or C % 4:
            continue
        o = dw.outs[0]
        tiles = -(-o.H // P.dw_tile_rows(dw.k[0], dw.s[0])) * -(-o.W // P.DW_TILE_W)
        pb = pl.new_buf(C, tiles, 1, P.DT_F32, dw.name + ":tile_sums")
        pv = P.View(pb, 0, 1, C)
        dw.outs = [dw.outs[0], pv]
        dw.flags |= P.FLAG_GAP_PARTIAL
        w1 = fc1.w_ref.reshape(Cr, C)                    # [Cout][1][1][Cin]
        w2 = fc2.w_ref.reshape(C, Cr)
        b1 = fc1.b if fc1.b is not None else np.zeros(Cr, np.float32)
        b2 = fc2.b if fc2.b is not None else np.zeros(C, np.float32)
        se = P.Op(P.OP_SE_FC, [pv], [fc2.outs[0]], fc1.act, w=np.ascontiguousarray(w1.T),
                  b=np.concatenate([b1, b2]).astype(np.float32), ints=[0, Cr, fc2.act, o.H * o.W], name=fc1.name + ":se_fc")
        se.extra = np.ascontiguousarray(w2.T)
        se.w_ref = (w1, w2)
        pl.ops[pl.ops.index(fc2)] = se
        pl.ops.remove(fc1)
        pl.ops.remove(gap)


def _fuse_dw_pw(pl):
    """depthwise 3x3 (stride 1) [or the fused upsample+concat+depthwise] -> 1x1 conv becomes one OP_DWPW when the depthwise
    output has no other reader: transform warps of csrc/conv_xf.cu build the conv's A tiles in shared memory, the
    depthwise output never reaches HBM.  MobileNetV3 blocks without squeeze-excite (kps_student.onnx blocks.0.0, 1.1,
    3.1-3.3: conv_dw -> conv_pw[l]) and both DecoderBlock heads (model.py:133-196)."""
    def same(a, b):
        return a is not None and b is not None and a.buf is b.buf and (a.c_off, a.c_stride, a.C) == (b.c_off, b.c_stride, b.C)

    def ok8(v):
        return v.c_stride == 1 and not ((v.C | v.buf.C | v.c_off) & 7)

    for d in list(pl.ops):
        up = d.type == P.OP_UPCAT_DW
        if not up and not (d.type == P.OP_DWCONV and list(d.k) == [3, 3] and list(d.s) == [1, 1] and list(d.d) == [1, 1]
                           and list(d.p) == [1, 1] and not (d.flags & P.FLAG_GAP_PARTIAL)):
            continue
        mid = d.outs[0]
        readers = [o for o in pl.ops if o is not d and any(v is not None and v.buf is mid.buf for v in o.ins)]
        writers = [o for o in pl.ops if o is not d and any(v.buf is mid.buf for v in o.outs)]
        if len(readers) != 1 or writers or mid.buf in [v.buf for v in pl.outputs]:
            continue
        c = readers[0]
        if c.type != P.OP_CONV or list(c.k) != [1, 1] or list(c.s) != [1, 1] or not same(c.ins[0], mid) \
                or c.ins[2] is not None or (c.flags & (P.FLAG_MMA | P.FLAG_XF | P.FLAG_IN_U8)):
            continue
        out = c.outs[0]
        x = d.ins[1] if up else d.ins[0]
        low = d.ins[0] if up else None
        if not ok8(x) or x.buf.dtype not in (P.DT_F32, P.DT_SPLIT16) or out.H < 8 or out.W < 16:
            continue
        if up and (not ok8(low) or low.buf.dtype != P.DT_F32 or x.buf.dtype != P.DT_SPLIT16 or low.C % 64
                   or out.H % 8 or out.W % 16 or out.H < 16):
            continue
        K = x.C + (low.C if up else 0)
        n_tile, n_tiles = P.tc_tiling(out.C)
        if n_tiles != 1 or -(-K // 64) > 16:
            continue
        if c.flags & P.FLAG_TC:
            hi, lo, out_scale = c.w, c.w2, c.floats[0]
            n_tile = c.ints[0]
            bias = c.b
        else:
            hi, lo, out_scale = P.pack_tc_weights(c.w_ref, n_tile, n_tiles)
            bias = c.b if c.b is not None else np.zeros(out.C, np.float32)
        kpad = -(-K // 64) * 64
        dww = np.zeros((10, kpad), np.float32)
        dww[:9, :K] = d.w
        dww[9, :K] = d.b
        o = P.Op(P.OP_DWPW, [x, c.ins[1], low], [out], c.act, (1, 1), (1, 1), (0, 0), (1, 1), hi, bias,
                 (c.flags & P.FLAG_RES_FIRST) | P.FLAG_TC, ints=[n_tile, 1, 0, 0], floats=[out_scale, float(d.act)],
                 name=d.name + "+" + c.name.split("/")[-2] if "/" in c.name else d.name + "+pw")
        o.w2 = lo
        o.extra, o.extra_slot = dww, 3
        if up:
            o.extra2 = P.pack_upcat_class_weights(d.w[:, :low.C])
        o.w_ref, o.dw_w, o.dw_b, o.dw_act = c.w_ref, d.w, d.b, d.act
        out.buf.dtype = out.buf.dtype            # the output keeps the format its readers asked for
        pl.ops[pl.ops.index(c)] = o
        pl.ops.remove(d)


def _fuse_stem_block(pl):
    """uint8 input -> conv_stem 3x3 s2 (h-swish) -> [depthwise 3x3 + ReLU -> 1x1 16->16 + shortcut] -> 1x1 16->64 + ReLU ->
    depthwise 3x3 s2 + ReLU: the whole full-resolution head of the mobilenetv3 encoder (kps_student.onnx conv_stem,
    blocks.0.0, blocks.1.0/conv_pw + conv_dw) becomes ONE CUDA-core kernel (csrc/stem_block.cu); the 16- and 64-channel
    full-resolution tensors never reach HBM."""
    if len(pl.ops) < 4:
        return
    c0, b0, c1, d1 = pl.ops[0], pl.ops[1], pl.ops[2], pl.ops[3]

    def same(a, b):
        return a is not None and b is not None and a.buf is b.buf and (a.c_off, a.c_stride, a.C) == (b.c_off, b.c_stride, b.C)

    def whole(v):
        return v.c_off == 0 and v.c_stride == 1 and v.C == v.buf.C

    def single_use(v, users):
        return all(not any(i is not None and i.buf is v.buf for i in o.ins) for o in pl.ops if o not in users) \
            and v.buf not in [o.buf for o in pl.outputs]

    H, W = pl.input.buf.H, pl.input.buf.W
    ok = (c0.type == P.OP_CONV and (c0.flags & P.FLAG_IN_U8) and list(c0.k) == [3, 3] and list(c0.s) == [2, 2]
          and list(c0.p) == [1, 1] and c0.act == P.ACT_HSWISH and c0.outs[0].C == 16 and whole(c0.outs[0])
          and c0.ins[1] is None and c0.b is not None
          and b0.type == P.OP_DWPW and b0.ins[2] is None and same(b0.ins[0], c0.outs[0]) and same(b0.ins[1], c0.outs[0])
          and int(b0.dw_act) == P.ACT_RELU and b0.act == P.ACT_NONE and b0.outs[0].C == 16 and whole(b0.outs[0])
          and not (b0.flags & P.FLAG_RES_FIRST)
          and c1.type == P.OP_CONV and list(c1.k) == [1, 1] and list(c1.s) == [1, 1] and same(c1.ins[0], b0.outs[0])
          and c1.ins[1] is None and c1.ins[2] is None and c1.act == P.ACT_RELU and c1.outs[0].C == 64 and whole(c1.outs[0])
          and d1.type == P.OP_DWCONV and list(d1.k) == [3, 3] and list(d1.s) == [2, 2] and list(d1.p) == [1, 1]
          and list(d1.d) == [1, 1] and d1.act == P.ACT_RELU and same(d1.ins[0], c1.outs[0]) and len(d1.outs) == 1
          and d1.outs[0].c_stride == 1 and not ((d1.outs[0].buf.C | d1.outs[0].c_off) & 3)
          and H % 32 == 0 and W % 64 == 0
          and single_use(c0.outs[0], [b0]) and single_use(b0.outs[0], [c1]) and single_use(c1.outs[0], [d1]))
    if not ok:
        return
    E = 64
    sw = np.ascontiguousarray(c0.w_ref.transpose(1, 2, 3, 0).reshape(27, 16), np.float32)         # [(ky*3+kx)*3+ci][co]
    pw0 = np.ascontiguousarray(b0.w_ref.reshape(16, 16).T, np.float32)                              # [ci][co]
    pw1 = np.ascontiguousarray(c1.w_ref.reshape(E, 16).T, np.float32)                               # [ci][co]
    zeros = lambda n: np.zeros(n, np.float32)
    packed = np.concatenate([sw.reshape(-1), c0.b, b0.dw_w.reshape(-1), b0.dw_b, pw0.reshape(-1),
                             b0.b if b0.b is not None else zeros(16), pw1.reshape(-1),
                             c1.b if c1.b is not None else zeros(E)]).astype(np.float32)
    assert packed.size == 27 * 16 + 16 + 144 + 16 + 256 + 16 + 16 * E + E
    o = P.Op(P.OP_STEM_BLOCK, [pl.input], [d1.outs[0]], P.ACT_RELU, w=packed, name="stem_block:" + d1.name)
    o.extra = np.concatenate([d1.w.reshape(9, E), d1.b.reshape(1, E)]).astype(np.float32)           # [9][E] + [E]
    o.sub_ops = [c0, b0, c1, d1]                  # the layers it replaces (oracle/plan_interp.py executes these)
    pl.ops[0:4] = [o]


def _fuse_hm_partial(pl):
    """Heat-map head: the decode (model.py:511-554 postp) needs only the maximum and first arg-max of every score map, so the
    head conv's epilogue reduces each 128-pixel tile to (max, pixel index) per channel and the map itself is never stored
    (436 MB per 256-face batch written and read back otherwise).  Split-head plans only (scores separate from offsets)."""
    for dec in pl.ops:
        if dec.type != P.OP_HM_DECODE or len(dec.ins) < 2 or dec.ins[1] is None:
            continue
        hv = dec.ins[0]
        prods = [o for o in pl.ops if o.type == P.OP_CONV and o.outs[0].buf is hv.buf]
        readers = [o for o in pl.ops if o is not dec and any(i is not None and i.buf is hv.buf for i in o.ins)]
        if len(prods) != 1 or readers or not (prods[0].flags & P.FLAG_TC) or (prods[0].flags & (P.FLAG_XF | P.FLAG_MMA)):
            continue
        hm = prods[0]
        H, W = hv.H, hv.W
        exact = (W % 128 == 0) if W >= 128 else (128 % W == 0 and H % (128 // W) == 0)
        if hm.act != P.ACT_NONE or hm.ins[1] is not None or list(hm.s) != [1, 1] or not exact or hv.buf.C > 128:
            continue
        ldp = 128
        # 256-pixel row-block tiles run on the transposed head kernel (csrc/conv_hm.cu: channels as accumulator rows, the
        # arg-max is a per-thread scan); other shapes keep conv_tc's 128-pixel tiles and its reduce-scatter epilogue
        cin = hm.ins[0].C
        wide = (8 <= W <= 256 and 256 % W == 0 and (H * W) % 256 == 0
                and cin % 8 == 0 and cin <= 128 and hm.ints[1] == 1)
        pb = pl.new_buf(2 * ldp, (H * W) // (256 if wide else 128), 1, P.DT_F32, hm.name + ":tile_max")
        pv = P.View(pb, 0, 1, 2 * ldp)
        hm.outs = [hm.outs[0], pv]
        hm.flags |= P.FLAG_HM_PART
        dec.ins = [dec.ins[0], dec.ins[1], pv]
        dec.flags |= P.FLAG_HM_PART


def _fuse_gap_sse(pl):
    """scSE attention (model.py:117-130; DecoderBlock attention2): cSE = sigmoid(FC(relu(FC(mean(x))))) and sSE = sigmoid(conv1x1(x))
    both start with a full pass over x.  One kernel (OP_GAP_SSE) reads x once and writes per-tile channel sums and the sSE map;
    the cSE MLP becomes the squeeze-excite FC kernel on those sums (OP_SE_FC).  Replaces GlobalAveragePool + 3 convs."""
    def same(a, b):
        return a is not None and b is not None and a.buf is b.buf and (a.c_off, a.c_stride, a.C) == (b.c_off, b.c_stride, b.C)

    def readers(v, skip=()):
        return [o for o in pl.ops if o not in skip and any(same(i, v) for i in o.ins)]

    for sc in list(pl.ops):
        if sc.type != P.OP_SCSE:
            continue
        x, cse, sse = sc.ins[0], sc.ins[1], sc.ins[2]
        fc2 = [o for o in pl.ops if o.type == P.OP_CONV and same(o.outs[0], cse)]
        sconv = [o for o in pl.ops if o.type == P.OP_CONV and same(o.outs[0], sse)]
        if len(fc2) != 1 or len(sconv) != 1:
            continue
        fc2, sconv = fc2[0], sconv[0]
        fc1 = [o for o in pl.ops if o.type == P.OP_CONV and same(o.outs[0], fc2.ins[0])]
        if len(fc1) != 1:
            continue
        fc1 = fc1[0]
        gap = [o for o in pl.ops if o.type == P.OP_GAP and same(o.outs[0], fc1.ins[0])]
        if len(gap) != 1 or not same(gap[0].ins[0], x) or not same(sconv.ins[0], x):
            continue
        gap = gap[0]
        C, Cr, HW = x.C, fc1.outs[0].C, x.H * x.W
        ok = (all(list(o.k) == [1, 1] and list(o.s) == [1, 1] and o.ins[1] is None and (len(o.ins) < 3 or o.ins[2] is None)
                  for o in (fc1, fc2, sconv))
              and not (fc1.flags & P.FLAG_TC) and not (fc2.flags & P.FLAG_TC) and sconv.outs[0].C == 1
              and x.c_off == 0 and x.c_stride == 1 and x.C == x.buf.C and C == 256 and HW % 32 == 0
              and fc2.outs[0].C == C and (C + Cr) * 8 * 4 <= 96 * 1024
              and len(readers(gap.outs[0])) == 1 and len(readers(fc1.outs[0])) == 1
              and len(readers(cse)) == 1 and len(readers(sse)) == 1)
        if not ok:
            continue
        tiles = HW // 32
        pb = pl.new_buf(C, tiles, 1, P.DT_F32, gap.name + ":tile_sums")
        pv = P.View(pb, 0, 1, C)
        ws = sconv.w_ref.reshape(-1)[:C].astype(np.float32)
        bs = (sconv.b[:1] if sconv.b is not None else np.zeros(1, np.float32)).astype(np.float32)
        sse.buf.dtype = P.DT_F32
        g = P.Op(P.OP_GAP_SSE, [x], [pv, sse], sconv.act, w=ws, b=bs, name=gap.name + ":gap_sse")
        g.w_ref = (ws, bs)
        w1 = fc1.w_ref.reshape(Cr, C)
        w2 = fc2.w_ref.reshape(C, Cr)
        b1 = fc1.b if fc1.b is not None else np.zeros(Cr, np.float32)
        b2 = fc2.b if fc2.b is not None else np.zeros(C, np.float32)
        se = P.Op(P.OP_SE_FC, [pv], [fc2.outs[0]], fc1.act, w=np.ascontiguousarray(w1.T),
                  b=np.concatenate([b1, b2]).astype(np.float32), ints=[0, Cr, fc2.act, HW], name=fc1.name + ":se_fc")
        se.extra = np.ascontiguousarray(w2.T)
        se.w_ref = (w1, w2)
        i = min(pl.ops.index(o) for o in (gap, fc1, fc2, sconv))
        for o in (gap, fc1, fc2, sconv):
            pl.ops.remove(o)
        pl.ops[i:i] = [g, se]


def _fold_affine_into_producers(pl):
    """BatchNormalization (+ReLU) applied to a Concat of conv outputs (the ASPP tail, model.py Decoder/ASPP: conv1|conv2|conv3|
    pooled branch -> bn_act): a per-channel affine commutes with the channel concat, so it folds into every producing conv
    (rows of W and the bias scaled, the ReLU becomes the conv's activation) and the pass over the 256-channel tensor
    disappears.  A nearest-resize producer (the broadcast pooled branch, itself conv+ReLU) gets the affine on its 1x1 source
    tensor instead."""
    for a in list(pl.ops):
        if a.type != P.OP_AFFINE_ACT or a.act not in (P.ACT_NONE, P.ACT_RELU):
            continue
        vin, vout = a.ins[0], a.outs[0]
        if vin.c_off != 0 or vin.c_stride != 1 or vin.C != vin.buf.C or vout.c_off != 0 or vout.c_stride != 1 or vout.C != vout.buf.C:
            continue
        prods = [o for o in pl.ops if o is not a and any(v.buf is vin.buf for v in o.outs)]
        if any(i is not None and i.buf is vin.buf for o in pl.ops if o is not a for i in o.ins) or vin.buf in [v.buf for v in pl.outputs]:
            continue
        covered = np.zeros(vin.C, np.int32)
        ok = True
        for o in prods:
            v = o.outs[0]
            if v.c_stride != 1 or len(o.outs) != 1:
                ok = False
                break
            covered[v.c_off:v.c_off + v.C] += 1
            if o.type == P.OP_CONV:
                ok &= (o.act == P.ACT_NONE and (len(o.ins) < 2 or o.ins[1] is None) and (len(o.ins) < 3 or o.ins[2] is None)
                       and not (o.flags & (P.FLAG_XF | P.FLAG_MMA | P.FLAG_HM_PART)) and getattr(o, "w_ref", None) is not None
                       and o.w_ref.shape[0] == v.C)
            elif o.type == P.OP_RESIZE_NEAREST:
                src = o.ins[0]
                ok &= src.H * src.W == 1 and src.c_off == 0 and src.c_stride == 1 and src.C == src.buf.C == v.C and \
                    sum(1 for q in pl.ops for i in q.ins if i is not None and i.buf is src.buf) == 1
            else:
                ok = False
        if not ok or not (covered == 1).all():
            continue
        inv, shift = a.w.astype(np.float32), a.b.astype(np.float32)
        for o in prods:
            v = o.outs[0]
            sc, sh = inv[v.c_off:v.c_off + v.C], shift[v.c_off:v.c_off + v.C]
            if o.type == P.OP_CONV:
                w = (o.w_ref * sc[:, None, None, None]).astype(np.float32)
                b = ((o.b[:v.C] if o.b is not None else np.zeros(v.C, np.float32)) * sc + sh).astype(np.float32)
                o.w_ref = w
                if o.flags & P.FLAG_TC:
                    hi, lo, out_scale = P.pack_tc_weights(w, o.ints[0], o.ints[1])
                    o.w, o.w2, o.floats = hi, lo, [out_scale] + list(o.floats[1:])
                else:
                    o.w = w
                o.b = b
                o.act = a.act
            else:
                src = o.ins[0]
                pl.ops.insert(pl.ops.index(o), P.Op(P.OP_AFFINE_ACT, [src], [src], a.act, w=sc.copy(), b=sh.copy(),
                                                     name=a.name + ":pooled"))
                src.buf.name += ":folded_bn"       # no longer the ONNX tensor of that name
        # the consumers of the normalised tensor read the concat buffer itself
        vin.buf.dtype = vout.buf.dtype
        vin.buf.name = vout.buf.name              # it now holds the normalised tensor (tools/layer_report.py compares by name)
        for o in pl.ops:
            o.ins = [P.View(vin.buf, i.c_off, i.c_stride, i.C) if (i is not None and i.buf is vout.buf) else i for i in o.ins]
        pl.ops.remove(a)


def lower(onnx_path, in_hw, name=None, input_u8=True, use_tc=True):
    """Build the plan for one of the reference's graphs at a fixed input size.  use_tc routes every
    eligible dense conv to the wgmma kernel (float16 hi/lo split, see csrc/conv_tc.cu)."""
    g = pad_channels(load_onnx(onnx_path))
    lw = _Lowerer(g, name or onnx_path, in_hw, input_u8, use_tc)
    lw.analyse()
    lw.emit()
    _fuse_upsample_concat_dw(lw.plan)
    _fold_affine_into_producers(lw.plan)
    _fuse_se_chain(lw.plan)
    if use_tc:
        _fuse_dw_pw(lw.plan)
        if input_u8:
            _fuse_stem_block(lw.plan)
        _fuse_hm_partial(lw.plan)
        _fuse_gap_sse(lw.plan)
    if not lw.plan.outputs:
        raise LoweringError("no outputs produced for %s" % onnx_path)
    return lw.plan
