"""`.onnx` model files -> the reference's 3-key checkpoint dict, for `compiler.compile_checkpoint`.

The reference runs an `.onnx` file through OpenCV DNN (`TextDetBaseDNN`, basemodel.py:246-256), picked from the
suffix (inference.py:124-130).  This module reads such a file and rebuilds the checkpoint the torch backend loads,

    {'blk_det': {'cfg': dict, 'weights': state_dict}, 'text_seg': state_dict, 'text_det': state_dict}

so that the one compiler emits the engine program for it.  Two parts:

* `read_model(path or bytes)`: the subset of the protobuf wire format a model needs (ModelProto.graph: nodes with
  their inputs, outputs and attributes, initializers, graph inputs / outputs with static shapes), pure Python and
  numpy, without the `onnx` package.  Tensors come as `raw_data`, `float_data`, `int32_data` or `int64_data`.
  External data, an unknown data type and a truncated or corrupt file raise ValueError.
* `checkpoint_from_graph(graph)`: recognises the modules of the reference's network by data flow, walking from each
  output back to the graph input -- never by initializer names or node order, which the exporter and onnxsim do not keep -- and recovers the
  yolov5 cfg (width and depth multiples from channel counts and C3 repeats, nc from the Detect conv, anchors from the
  anchor-grid constants / stride), the weights and `head_act`.  Anything outside the supported yolov5s-v6 + UnetHead
  + DBHead structure raises ValueError naming the node.

What the `.onnx` path computes differs from the `.pt` path in four ways, all reproduced here (DESIGN.md section 4):
the network sees RGB (inference.py:72-83 with to_tensor=False, then `blobFromImage` without swapRB), so the stem's
input channels are reversed in the recovered weights and the engine keeps feeding its BGR page; the input size is
fixed by the file; the exporter folds Conv + BatchNorm in float32 itself (those convs arrive with a bias and no BN
entries, `compile_checkpoint` takes them as folded), while the BatchNorm after each ConvTranspose stays a node and is
folded by the compiler in float64 as for a `.pt` file; and the output order cv2 returns is irrelevant, since the
engine's outputs are named by what they are.
"""
import struct

import numpy as np

# ---------------------------------------------------------------------------------------------------------------
# protobuf wire format

_DTYPES = {1: np.float32, 2: np.uint8, 3: np.int8, 5: np.int16, 6: np.int32, 7: np.int64, 9: np.bool_,
           10: np.float16, 11: np.float64}


class _Msg:
    """One message: field number -> list of (wire type, value); value is an int (varint / fixed) or a memoryview."""

    def __init__(self, buf, what):
        self.fields = {}
        self.what = what
        pos, end = 0, len(buf)
        while pos < end:
            key, pos = _varint(buf, pos, what)
            num, wt = key >> 3, key & 7
            if num == 0:
                raise ValueError("corrupt ONNX file: field number 0 in %s" % what)
            if wt == 0:
                val, pos = _varint(buf, pos, what)
            elif wt == 1:
                if pos + 8 > end:
                    raise ValueError("truncated ONNX file: 64-bit field %d of %s" % (num, what))
                val, pos = struct.unpack_from("<Q", buf, pos)[0], pos + 8
            elif wt == 2:
                n, pos = _varint(buf, pos, what)
                if pos + n > end:
                    raise ValueError("truncated ONNX file: field %d of %s needs %d bytes, %d left"
                                     % (num, what, n, end - pos))
                val, pos = buf[pos:pos + n], pos + n
            elif wt == 5:
                if pos + 4 > end:
                    raise ValueError("truncated ONNX file: 32-bit field %d of %s" % (num, what))
                val, pos = struct.unpack_from("<I", buf, pos)[0], pos + 4
            else:
                raise ValueError("corrupt ONNX file: wire type %d of field %d in %s" % (wt, num, what))
            self.fields.setdefault(num, []).append((wt, val))

    def all(self, num):
        return [v for _wt, v in self.fields.get(num, [])]

    def one(self, num, default=None):
        v = self.fields.get(num)
        return v[-1][1] if v else default

    def str(self, num, default=""):
        v = self.one(num)
        return default if v is None else bytes(v).decode("utf-8", "replace")

    def strs(self, num):
        return [bytes(v).decode("utf-8", "replace") for v in self.all(num)]

    def sub(self, num, what):
        return [_Msg(v, what) for v in self.all(num)]

    def ints(self, num):
        """a repeated varint field, packed or not, as signed int64"""
        out = []
        for wt, v in self.fields.get(num, []):
            if wt == 0:
                out.append(v)
            elif wt == 2:
                pos = 0
                while pos < len(v):
                    x, pos = _varint(v, pos, self.what)
                    out.append(x)
            else:
                raise ValueError("corrupt ONNX file: field %d of %s is not an integer" % (num, self.what))
        return [x - (1 << 64) if x >= 1 << 63 else x for x in out]

    def packed(self, num, dtype):
        """a repeated fixed-width field (float32 / float64), packed or not"""
        dt = np.dtype(dtype)
        parts = []
        for wt, v in self.fields.get(num, []):
            if wt == 2:
                if len(v) % dt.itemsize:
                    raise ValueError("corrupt ONNX file: packed field %d of %s has %d bytes"
                                     % (num, self.what, len(v)))
                parts.append(np.frombuffer(v, dt))
            else:
                parts.append(np.array([v], np.uint32 if dt.itemsize == 4 else np.uint64).view(dt))
        return np.concatenate(parts) if parts else np.zeros((0,), dt)


def _varint(buf, pos, what):
    x, shift = 0, 0
    while True:
        if pos >= len(buf):
            raise ValueError("truncated ONNX file: varint in %s" % what)
        b = buf[pos]
        pos += 1
        x |= (b & 0x7F) << shift
        if not b & 0x80:
            return x, pos
        shift += 7
        if shift > 63:
            raise ValueError("corrupt ONNX file: varint longer than 10 bytes in %s" % what)


def _tensor(m, what):
    """TensorProto -> numpy array"""
    name = m.str(8)
    what = "tensor %r of %s" % (name, what)
    if m.one(14, 0) == 1 or m.all(13):
        raise ValueError("%s keeps its data in an external file, which is not supported" % what)
    dims = m.ints(1)
    dt = m.one(2, 0)
    if dt not in _DTYPES:
        raise ValueError("%s has ONNX data type %d, which is not supported" % (what, dt))
    dtype = np.dtype(_DTYPES[dt])
    count = int(np.prod(dims, dtype=np.int64)) if dims else 1
    raw = m.one(9)
    if raw is not None:
        if len(raw) != count * dtype.itemsize:
            raise ValueError("%s: raw_data has %d bytes, its shape %s needs %d"
                             % (what, len(raw), dims, count * dtype.itemsize))
        a = np.frombuffer(raw, dtype.newbyteorder("<")).astype(dtype)
    elif dt == 1:
        a = m.packed(4, np.float32)
    elif dt == 11:
        a = m.packed(10, np.float64)
    elif dt == 7:
        a = np.array(m.ints(7), np.int64)
    elif dt in (2, 3, 5, 6, 9):
        a = np.array(m.ints(5), np.int64).astype(dtype)
    elif dt == 10:
        a = np.array(m.ints(5), np.uint16).view(np.float16)
    else:
        a = np.zeros((0,), dtype)
    if a.size != count:
        raise ValueError("%s holds %d values, its shape %s needs %d" % (what, a.size, dims, count))
    return a.reshape(dims)


class Node:
    """A graph node: op_type, name, input / output value names, attributes (name -> int, float, bytes, ndarray or
    list)."""

    def __init__(self, op_type, name, inputs, outputs, attrs):
        self.op_type, self.name, self.inputs, self.outputs, self.attrs = op_type, name, inputs, outputs, attrs

    def __repr__(self):
        return "%s node %r (%s -> %s)" % (self.op_type, self.name, ", ".join(self.inputs), ", ".join(self.outputs))


def _attr(m, what):
    name = m.str(1)
    typ = m.one(20, 0)
    what = "attribute %r of %s" % (name, what)
    if typ == 1:
        return name, struct.unpack("<f", struct.pack("<I", m.one(2, 0)))[0]
    if typ == 2:
        v = m.one(3, 0)
        return name, v - (1 << 64) if v >= 1 << 63 else v
    if typ == 3:
        return name, bytes(m.one(4, b""))
    if typ == 4:
        return name, _tensor(_Msg(m.one(5, b""), what), what)
    if typ == 6:
        return name, [float(x) for x in m.packed(7, np.float32)]
    if typ == 7:
        return name, m.ints(8)
    if typ == 8:
        return name, [bytes(v) for v in m.all(9)]
    return name, None   # graphs, sparse tensors, type protos: no supported node has them


def _value_shape(m):
    """ValueInfoProto -> (name, shape list of int or str (symbolic) or None, elem_type)"""
    name = m.str(1)
    t = m.one(2)
    if t is None:
        return name, None, 0
    tt = _Msg(t, "type of %r" % name).one(1)
    if tt is None:
        return name, None, 0
    tt = _Msg(tt, "tensor type of %r" % name)
    shp = tt.one(2)
    if shp is None:
        return name, None, tt.one(1, 0)
    dims = []
    for d in _Msg(shp, "shape of %r" % name).sub(1, "dim of %r" % name):
        if d.one(1) is not None:
            dims.append(d.ints(1)[0])
        else:
            dims.append(d.str(2) or "?")
    return name, dims, tt.one(1, 0)


class Graph:
    """nodes (list of Node), initializers (name -> ndarray; `Constant` node values are added here too), inputs /
    outputs (list of (name, shape)), opset (default domain)."""

    def __init__(self, nodes, initializers, inputs, outputs, opset):
        self.nodes, self.initializers, self.inputs, self.outputs, self.opset = nodes, initializers, inputs, outputs, opset


def read_model(src):
    """Parses an ONNX file (path or bytes) into a Graph.  ValueError on anything it cannot read."""
    if isinstance(src, (bytes, bytearray, memoryview)):
        data = bytes(src)
    else:
        with open(src, "rb") as f:
            data = f.read()
    if not data:
        raise ValueError("empty ONNX file")
    model = _Msg(memoryview(data), "ModelProto")
    g = model.one(7)
    if g is None:
        raise ValueError("not an ONNX model: no graph (ModelProto field 7)")
    opset = 0
    for o in model.sub(8, "opset_import"):
        if o.str(1) in ("", "ai.onnx"):
            opset = o.ints(2)[0] if o.all(2) else 0
    g = _Msg(g, "GraphProto")
    inits = {}
    for t in g.sub(5, "GraphProto.initializer"):
        inits[t.str(8)] = _tensor(t, "the initializers")
    nodes = []
    for k, n in enumerate(g.sub(1, "GraphProto.node")):
        op, name = n.str(4), n.str(3)
        what = "%s node %r" % (op, name or "#%d" % k)
        attrs = dict(_attr(a, what) for a in n.sub(5, what))
        if n.str(7) not in ("", "ai.onnx"):
            raise ValueError("%s is in the custom domain %r, which is not supported" % (what, n.str(7)))
        node = Node(op, name or "#%d" % k, n.strs(1), n.strs(2), attrs)
        if op == "Constant":
            if not isinstance(attrs.get("value"), np.ndarray) or len(node.outputs) != 1:
                raise ValueError("%r: only tensor-valued Constant nodes are supported" % (node,))
            inits[node.outputs[0]] = attrs["value"]
            continue
        nodes.append(node)
    inputs = [_value_shape(v)[:2] for v in g.sub(11, "GraphProto.input")]
    inputs = [(n, s) for n, s in inputs if n not in inits]
    outputs = [_value_shape(v)[:2] for v in g.sub(12, "GraphProto.output")]
    return Graph(nodes, inits, inputs, outputs, opset)


# ---------------------------------------------------------------------------------------------------------------
# graph -> checkpoint

# yolov5 v6.0 (yolov5s.yaml) layer template: [from, base repeats, module, base args]; width / depth multiples, nc and
# anchors come from the graph.  Layer 0 is the 6x6 s2 Conv stem (a v5.0 Focus stem is not supported).
YOLOV5_V6_BACKBONE = [[-1, 1, "Conv", [64, 6, 2, 2]], [-1, 1, "Conv", [128, 3, 2]], [-1, 3, "C3", [128]],
                      [-1, 1, "Conv", [256, 3, 2]], [-1, 6, "C3", [256]], [-1, 1, "Conv", [512, 3, 2]],
                      [-1, 9, "C3", [512]], [-1, 1, "Conv", [1024, 3, 2]], [-1, 3, "C3", [1024]],
                      [-1, 1, "SPPF", [1024, 5]]]
YOLOV5_V6_HEAD = [[-1, 1, "Conv", [512, 1, 1]], [-1, 1, "nn.Upsample", [None, 2, "nearest"]],
                  [[-1, 6], 1, "Concat", [1]], [-1, 3, "C3", [512, False]],
                  [-1, 1, "Conv", [256, 1, 1]], [-1, 1, "nn.Upsample", [None, 2, "nearest"]],
                  [[-1, 4], 1, "Concat", [1]], [-1, 3, "C3", [256, False]],
                  [-1, 1, "Conv", [256, 3, 2]], [[-1, 14], 1, "Concat", [1]], [-1, 3, "C3", [512, False]],
                  [-1, 1, "Conv", [512, 3, 2]], [[-1, 10], 1, "Concat", [1]], [-1, 3, "C3", [1024, False]],
                  [[17, 20, 23], 1, "Detect", ["nc", "anchors"]]]
_WIDTHS = (0.25, 0.50, 0.75, 1.0, 1.25)
_DEPTHS = (0.33, 0.67, 1.0, 1.33)
_HEAD_ACT = {"leaky": "leaky", "relu": "relu", "silu": True}   # -> compile_checkpoint(head_act=)


def _unsupported(node, what):
    return ValueError("unsupported ONNX graph: %r, where %s was expected" % (node, what))


class _Walker:
    """Walks the graph backwards from a value to the node that computes it, checking each node against the module
    it must belong to.  Every recognised conv / deconv / BatchNorm writes its tensors into a state dict under the
    reference's parameter names."""

    def __init__(self, g):
        self.g = g
        self.prod = {o: n for n in g.nodes for o in n.outputs}

    def src(self, v, ops, what):
        n = self.prod.get(v)
        if n is None or n.op_type not in ops:
            raise _unsupported(n if n is not None else "graph value %r" % v, what)
        return n

    def const(self, n, i, what):
        if len(n.inputs) <= i or not n.inputs[i]:
            return None
        v = n.inputs[i]
        if v not in self.g.initializers:
            raise _unsupported(n, what + " with constant input %d" % i)
        return self.g.initializers[v]

    def act(self, v, what):
        """-> (kind, pre-activation value) of x * sigmoid(x), LeakyReLU(0.1) or ReLU"""
        n = self.src(v, ("Mul", "LeakyRelu", "Relu"), what + " (SiLU, LeakyReLU or ReLU)")
        if n.op_type == "LeakyRelu":
            if abs(n.attrs.get("alpha", 0.01) - 0.1) > 1e-6:
                raise _unsupported(n, "LeakyReLU(0.1)")
            return "leaky", n.inputs[0]
        if n.op_type == "Relu":
            return "relu", n.inputs[0]
        for x, s in (n.inputs, n.inputs[::-1]):
            p = self.prod.get(s)
            if p is not None and p.op_type == "Sigmoid" and p.inputs[0] == x:
                return "silu", x
        raise _unsupported(n, what + " (x * sigmoid(x))")

    def conv(self, v, what, k=None, s=1, p=None, act=True, sd=None, prefix=None):
        """a Conv (+ activation) whose BatchNorm the exporter folded; k None: any of 1 / 3.  -> dict(x, k, act, node)"""
        kind, pre = self.act(v, what) if act else (None, v)
        n = self.src(pre, ("Conv",), what + " (Conv with its BatchNorm folded)")
        w = self.const(n, 1, what)
        b = self.const(n, 2, what)
        a = n.attrs
        kk = int(w.shape[2]) if w is not None and w.ndim == 4 else -1
        pad = kk // 2 if p is None else p
        if (w is None or w.ndim != 4 or w.shape[2] != w.shape[3] or (k is not None and kk != k)
                or (k is None and kk not in (1, 3)) or a.get("group", 1) != 1 or any(d != 1 for d in a.get("dilations", [1, 1]))
                or list(a.get("strides", [1, 1])) != [s, s] or list(a.get("pads", [0, 0, 0, 0])) != [pad] * 4
                or a.get("auto_pad", b"NOTSET") not in (b"NOTSET", b"")):
            raise _unsupported(n, "%s: a %sx%s stride-%d Conv" % (what, k or "k", k or "k", s))
        if b is None:
            b = np.zeros((w.shape[0],), np.float32)
        if sd is not None:
            sd[prefix + ".weight"], sd[prefix + ".bias"] = w, b
        return dict(x=n.inputs[0], k=kk, act=kind, node=n, w=w)

    def concat(self, v, n_in, what, axis=1):
        n = self.src(v, ("Concat",), what)
        if n.attrs.get("axis") not in ((axis,) if axis == 1 else (-1, 4)) or len(n.inputs) != n_in:
            raise _unsupported(n, "%s: a Concat of %d tensors on axis %d" % (what, n_in, axis))
        return n.inputs

    def c3(self, v, sd, prefix):
        """C3 (common.py:126-138) computing v: cv3(cat(m(cv1(x)), cv2(x))) -> dict(x, n, shortcut, act)"""
        what = "C3 " + prefix
        cv3 = self.conv(v, what + ".cv3", 1, sd=sd, prefix=prefix + ".cv3.conv")
        m_out, cv2_out = self.concat(cv3["x"], 2, what + " concat")
        cv2 = self.conv(cv2_out, what + ".cv2", 1, sd=sd, prefix=prefix + ".cv2.conv")
        x = cv2["x"]
        acts, blocks, cur = {cv3["act"], cv2["act"]}, [], m_out
        while True:
            n = self.prod.get(cur)
            if n is not None and n.op_type == "Add":   # Bottleneck with shortcut: y + cv2(cv1(y))
                for y, r in (n.inputs, n.inputs[::-1]):
                    c2 = self.conv(r, what + " bottleneck cv2", 3) if self._is_conv(r, 3) else None
                    c1 = self.conv(c2["x"], what + " bottleneck cv1", 1) if c2 and self._is_conv(c2["x"], 1) else None
                    if c1 is not None and c1["x"] == y:
                        break
                else:
                    raise _unsupported(n, what + ": a Bottleneck residual x + cv2(cv1(x))")
                blocks.append((True, r))
                cur = y
                continue
            c = self.conv(cur, what + " cv1 or bottleneck", None)
            if c["k"] == 1:   # C3.cv1: must read the same x as cv2
                if c["x"] != x:
                    raise _unsupported(c["node"], what + ".cv1 reading the C3 input")
                self.conv(cur, what + ".cv1", 1, sd=sd, prefix=prefix + ".cv1.conv")
                acts.add(c["act"])
                break
            blocks.append((False, cur))
            cur = self.conv(c["x"], what + " bottleneck cv1", 1)["x"]
        blocks.reverse()
        for j, (_sc, r) in enumerate(blocks):
            c2 = self.conv(r, what + " bottleneck cv2", 3, sd=sd, prefix="%s.m.%d.cv2.conv" % (prefix, j))
            c1 = self.conv(c2["x"], what + " bottleneck cv1", 1, sd=sd, prefix="%s.m.%d.cv1.conv" % (prefix, j))
            acts |= {c1["act"], c2["act"]}
        if len(acts) != 1 or len({sc for sc, _r in blocks}) != 1:
            raise _unsupported(cv3["node"], what + " with one activation and one shortcut setting for all its convs")
        return dict(x=x, n=len(blocks), shortcut=blocks[0][0], act=acts.pop())

    def _is_conv(self, v, k):
        try:
            self.conv(v, "", k)
            return True
        except ValueError:
            return False

    def sppf(self, v, sd, prefix):
        """SPPF (common.py): cv2(cat(y, m(y), m(m(y)), m(m(m(y))))) with y = cv1(x), m = MaxPool 5 / 1 / 2"""
        what = "SPPF " + prefix
        cv2 = self.conv(v, what + ".cv2", 1, sd=sd, prefix=prefix + ".cv2.conv")
        ins = self.concat(cv2["x"], 4, what + " concat")
        for k in (3, 2, 1):
            mp = self.src(ins[k], ("MaxPool",), what + " MaxPool")
            a = mp.attrs
            if (mp.inputs[0] != ins[k - 1] or list(a.get("kernel_shape", [])) != [5, 5] or list(a.get("strides", [1, 1])) != [1, 1]
                    or list(a.get("pads", [0] * 4)) != [2] * 4 or a.get("ceil_mode", 0) or any(d != 1 for d in a.get("dilations", [1, 1]))):
                raise _unsupported(mp, what + ": MaxPool(5, 1, 2) of the previous pooling")
        cv1 = self.conv(ins[0], what + ".cv1", 1, sd=sd, prefix=prefix + ".cv1.conv")
        return dict(x=cv1["x"], act={cv1["act"], cv2["act"]})

    def upsample(self, v, what):
        n = self.src(v, ("Resize", "Upsample"), what + " (nearest x2 Resize)")
        scales = self.const(n, 2 if n.op_type == "Resize" and len(n.inputs) > 2 else 1, what)
        if n.attrs.get("mode", b"nearest") != b"nearest" or scales is None or scales.size == 0:
            scales = None
        if scales is None or [float(s) for s in scales.reshape(-1)] != [1.0, 1.0, 2.0, 2.0]:
            raise _unsupported(n, what + ": a nearest Resize with scales (1, 1, 2, 2)")
        return n.inputs[0]

    def deconv_bn_relu(self, v, sd, prefix, k, pad, what, bias):
        """Relu(BatchNorm(ConvTranspose(x))); the BatchNorm keeps its own node and goes into the dict as BN entries"""
        r = self.src(v, ("Relu",), what + " ReLU")
        bn = self.src(r.inputs[0], ("BatchNormalization",), what + " BatchNorm")
        if abs(bn.attrs.get("epsilon", 1e-5) - 1e-5) > 1e-9 or bn.attrs.get("training_mode", 0):
            raise _unsupported(bn, what + ": an eval-mode BatchNorm with eps 1e-5")
        ct = self.deconv(bn.inputs[0], sd, prefix[0], k, pad, what, bias)
        prm = [self.const(bn, i, what + " BatchNorm") for i in range(1, 5)]
        if any(p is None for p in prm):
            raise _unsupported(bn, what + " BatchNorm with constant parameters")
        for key, p in zip(("weight", "bias", "running_mean", "running_var"), prm):
            sd["%s.%s" % (prefix[1], key)] = p
        return ct

    def deconv(self, v, sd, prefix, k, pad, what, bias):
        n = self.src(v, ("ConvTranspose",), what + " ConvTranspose")
        w, b, a = self.const(n, 1, what), self.const(n, 2, what), n.attrs
        if (w is None or w.ndim != 4 or list(w.shape[2:]) != [k, k] or list(a.get("strides", [1, 1])) != [2, 2]
                or list(a.get("pads", [0] * 4)) != [pad] * 4 or a.get("group", 1) != 1
                or any(d != 1 for d in a.get("dilations", [1, 1])) or any(a.get("output_padding", [0, 0]))
                or "output_shape" in a or (b is not None and not bias)):
            raise _unsupported(n, "%s: a ConvTranspose %dx%d stride 2 pad %d%s" % (what, k, k, pad, "" if bias else " without bias"))
        sd[prefix + ".weight"] = w
        if bias:
            sd[prefix + ".bias"] = b if b is not None else np.zeros((w.shape[1],), np.float32)
        return n.inputs[0]

    def up_c3(self, v, sd, prefix, n_in):
        """double_conv_up_c3 (basemodel.py:21-32): ReLU(BN(ConvT4x4s2(C3(x)))) -> (C3 input values, act)"""
        x = self.deconv_bn_relu(v, sd, (prefix + ".conv.1", prefix + ".conv.2"), 4, 1, "double_conv_up_c3 " + prefix, False)
        c = self.head_c3(x, sd, prefix + ".conv.0")
        return (self.concat(c["x"], 2, prefix + " input") if n_in == 2 else [c["x"]]), c["act"]

    def head_c3(self, v, sd, prefix):
        c = self.c3(v, sd, prefix)
        if c["n"] != 1 or not c["shortcut"]:
            raise _unsupported(self.prod[v], "head C3 %s with one shortcut Bottleneck" % prefix)
        return c


def _const_through(W, v):
    """the constant behind Cast / Expand nodes (the exporter's anchor grid)"""
    while v not in W.g.initializers:
        n = W.prod.get(v)
        if n is None or n.op_type not in ("Cast", "Expand"):
            return None
        v = n.inputs[0]
    return W.g.initializers[v]


def _detect_level(W, v, S, down, sd, li):
    """one level of Detect (yolo.py:23-44, inplace=False): Reshape(cat(xy, wh, conf)) with
    y = sigmoid(Transpose(Reshape(conv(x)))) -> (conv input, anchors in px (na, 2), out channels)"""
    what = "Detect level %d" % li
    rs = W.src(v, ("Reshape",), what + " output Reshape")
    xy, wh, conf = W.concat(rs.inputs[0], 3, what + " (xy, wh, conf)", axis=-1)
    sig = W.src(conf, ("Slice",), what + " conf Slice").inputs[0]
    sn = W.src(sig, ("Sigmoid",), what + " Sigmoid")
    tr = W.src(sn.inputs[0], ("Transpose",), what + " Transpose")
    if list(tr.attrs.get("perm", [])) != [0, 1, 3, 4, 2]:
        raise _unsupported(tr, what + ": Transpose (0, 1, 3, 4, 2)")
    r5 = W.src(tr.inputs[0], ("Reshape",), what + " Reshape to (bs, na, no, ny, nx)")
    conv = W.conv(r5.inputs[0], what + " conv", 1, act=False)
    shp = W.const(r5, 1, what)
    g = S // down
    if shp is None or shp.size != 5 or list(shp.reshape(-1)[3:]) != [g, g]:
        raise _unsupported(r5, "%s: a Reshape to a constant (bs, na, no, %d, %d) (the %d px feature map of a %d px input)"
                           % (what, g, g, g, S))
    stride = S / g
    anchors = None
    mul = W.src(wh, ("Mul",), what + " wh = (2 sigmoid)^2 * anchor_grid")
    for a in mul.inputs:
        c = _const_through(W, a)
        if c is not None and c.ndim == 5 and c.shape[-1] == 2:
            anchors = np.asarray(c, np.float64)[0, :, 0, 0, :]
    mxy = W.src(xy, ("Mul",), what + " xy = (2 sigmoid - 0.5 + grid) * stride")
    strides = [W.g.initializers.get(a) for a in mxy.inputs]
    if anchors is None or not any(s is not None and s.size == 1 and float(s) == stride for s in strides):
        raise _unsupported(mul if anchors is None else mxy, "%s: the anchor grid and the stride %g" % (what, stride))
    na = anchors.shape[0]
    co = conv["w"].shape[0]
    if co % na or co // na < 6 or int(shp.reshape(-1)[1]) != na:
        raise _unsupported(conv["node"], what + ": a conv with na * (nc + 5) outputs")
    sd["model.24.m.%d.weight" % li] = conv["w"]
    sd["model.24.m.%d.bias" % li] = W.const(conv["node"], 2, what)
    return conv["x"], anchors, co // na


def checkpoint_from_graph(g):
    """Graph -> (checkpoint dict, head_act, input size S).  ValueError names the node where the graph leaves the
    supported yolov5s-v6 + UnetHead + DBHead structure."""
    if len(g.inputs) != 1:
        raise ValueError("unsupported ONNX graph: %d inputs, the detector has one (images)" % len(g.inputs))
    iname, shape = g.inputs[0]
    if shape is None or len(shape) != 4 or not all(isinstance(d, int) and d > 0 for d in shape):
        raise ValueError("unsupported ONNX graph: input %r has shape %s; the input size must be fixed at export "
                         "(dynamic=False)" % (iname, shape))
    if shape[1] != 3 or shape[2] != shape[3]:
        raise ValueError("unsupported ONNX graph: input %r has shape %s; a square 3-channel input is needed"
                         % (iname, shape))
    S = shape[2]
    W = _Walker(g)
    outs = {}
    for name, _shp in g.outputs:
        n = W.prod.get(name)
        if n is not None and n.op_type == "Concat" and all(W.prod.get(i) is not None and W.prod[i].op_type == "Reshape"
                                                           for i in n.inputs):
            outs.setdefault("blk", name)
        elif n is not None and n.op_type == "Sigmoid":
            outs.setdefault("seg", name)
        elif n is not None and n.op_type == "Concat" and len(n.inputs) == 2:
            outs.setdefault("det", name)
    if len(g.outputs) != 3 or len(outs) != 3:
        raise ValueError("unsupported ONNX graph: outputs %s; the detector has three (blk, seg, det)"
                         % [o for o, _s in g.outputs])
    ysd, ssd, dsd = {}, {}, {}

    # ---- text_det: DBHead (basemodel.py:83-125) --------------------------------------------------------------
    heads = set()
    xs = []
    for name, v in zip(("binarize", "thresh"), W.concat(outs["det"], 2, "DBHead output cat(shrink, threshold)")):
        s = W.src(v, ("Sigmoid",), "DBHead %s Sigmoid" % name)
        x = W.deconv(s.inputs[0], dsd, name + ".6", 2, 0, "DBHead " + name, True)
        x = W.deconv_bn_relu(x, dsd, (name + ".3", name + ".4"), 2, 0, "DBHead " + name, True)
        c = W.conv(x, "DBHead %s.0" % name, 3, sd=dsd, prefix=name + ".0")
        if c["act"] != "relu":
            raise _unsupported(c["node"], "DBHead %s.0 followed by ReLU" % name)
        xs.append(c["x"])
    if xs[0] != xs[1]:
        raise _unsupported(W.prod.get(xs[1]), "DBHead thresh reading the same features as binarize")
    c = W.conv(xs[0], "DBHead conv", 1, sd=dsd, prefix="conv.0")
    if c["act"] != "relu":
        raise _unsupported(c["node"], "DBHead conv followed by ReLU")
    (f128_d, du128), a1 = W.up_c3(c["x"], dsd, "upconv4", 2)
    (f64_d, u64_d), a2 = W.up_c3(du128, dsd, "upconv3", 2)
    heads |= {a1, a2}

    # ---- text_seg: UnetHead (basemodel.py:47-78) -------------------------------------------------------------
    s = W.src(outs["seg"], ("Sigmoid",), "UnetHead output Sigmoid")
    u512 = W.deconv(s.inputs[0], ssd, "upconv6.0", 4, 1, "UnetHead upconv6", False)
    (f256, u256), a = W.up_c3(u512, ssd, "upconv5", 2)
    heads.add(a)
    (f128, u128), a = W.up_c3(u256, ssd, "upconv4", 2)
    heads.add(a)
    (f64, u64), a = W.up_c3(u128, ssd, "upconv3", 2)
    heads.add(a)
    (f32, u32), a = W.up_c3(u64, ssd, "upconv2", 2)
    heads.add(a)
    (d16,), a = W.up_c3(u32, ssd, "upconv0", 1)
    heads.add(a)
    c = W.head_c3(d16, ssd, "down_conv1.conv")
    heads.add(c["act"])
    pool = W.src(c["x"], ("AveragePool",), "UnetHead down_conv1 AvgPool2d(2)")
    pa = pool.attrs
    if (list(pa.get("kernel_shape", [])) != [2, 2] or list(pa.get("strides", [1, 1])) != [2, 2]
            or any(pa.get("pads", [0] * 4)) or pa.get("ceil_mode", 0)):
        raise _unsupported(pool, "AvgPool2d(2, stride=2)")
    f3 = pool.inputs[0]
    if (f64_d, u64_d, f128_d) != (f64, u64, f128):
        raise _unsupported(W.prod.get(c["x"]), "DBHead reading the UnetHead's features (f80, f40, u40)")
    if len(heads) != 1:
        raise ValueError("unsupported ONNX graph: the head C3s use different activations %s" % sorted(heads))
    head_act = _HEAD_ACT[heads.pop()]

    # ---- blk_det: yolov5 v6 (yolo.py) ------------------------------------------------------------------------
    parts = W.concat(outs["blk"], 3, "Detect output cat of three levels")
    P, anchors, nos = [], [], []
    for li, (part, down) in enumerate(zip(parts, (8, 16, 32))):
        x, anc, no = _detect_level(W, part, S, down, ysd, li)
        P.append(x)
        anchors.append(anc)
        nos.append(no)
    if len(set(nos)) != 1 or len({a.shape for a in anchors}) != 1:
        raise _unsupported(W.prod[outs["blk"]], "Detect levels with one number of anchors and classes")
    val, n_of, yacts = {}, {}, set()

    def c3(i, v):
        c = W.c3(v, ysd, "model.%d" % i)
        n_of[i] = (c["n"], c["shortcut"])
        yacts.add(c["act"])
        return c["x"]

    def conv(i, v, k, s_, p=None):
        c = W.conv(v, "Conv model.%d" % i, k, s_, p, sd=ysd, prefix="model.%d.conv" % i)
        yacts.add(c["act"])
        return c["x"]

    val[17], val[20], val[23] = P
    a, val[10] = W.concat(c3(23, val[23]), 2, "model.22 Concat")
    if conv(21, a, 3, 2) != val[20]:
        raise _unsupported(W.prod[a], "model.21 Conv reading model.20")
    a, val[14] = W.concat(c3(20, val[20]), 2, "model.19 Concat")
    if conv(18, a, 3, 2) != val[17]:
        raise _unsupported(W.prod[a], "model.18 Conv reading model.17")
    a, val[4] = W.concat(c3(17, val[17]), 2, "model.16 Concat")
    if W.upsample(a, "model.15 Upsample") != val[14]:
        raise _unsupported(W.prod[a], "model.15 Upsample of model.14")
    val[13] = conv(14, val[14], 1, 1)
    a, val[6] = W.concat(c3(13, val[13]), 2, "model.12 Concat")
    if W.upsample(a, "model.11 Upsample") != val[10]:
        raise _unsupported(W.prod[a], "model.11 Upsample of model.10")
    val[9] = conv(10, val[10], 1, 1)
    sp = W.sppf(val[9], ysd, "model.9")
    yacts |= sp["act"]
    val[8] = sp["x"]
    val[7] = c3(8, val[8])
    for i in (7, 5):   # the C3 outputs 6 and 4 feed both the next Conv and the neck
        if conv(i, val[i], 3, 2) != val[i - 1]:
            raise _unsupported(W.prod.get(val[i]), "model.%d reading model.%d" % (i, i - 1))
        val[i - 2] = c3(i - 1, val[i - 1])
    val[2] = conv(3, val[3], 3, 2)
    val[1] = c3(2, val[2])
    val[0] = conv(1, val[1], 3, 2)
    try:
        img = conv(0, val[0], 6, 2, 2)
    except ValueError as ex:
        raise ValueError("%s (the yolov5 v6 stem Conv(3, c, 6, 2, 2) on the input; a v5.0 Focus stem is not "
                         "supported)" % ex) from None
    if img != iname:
        raise _unsupported(W.prod[val[0]], "the stem Conv reading the graph input %r" % iname)
    if (val[1], val[3], val[5], val[7], val[9]) != (f256, f128, f64, f32, f3):
        raise _unsupported(W.prod.get(f256), "the heads reading model.1, 3, 5, 7 and 9 of the backbone")
    if yacts != {"silu"}:
        raise ValueError("unsupported ONNX graph: the yolov5 convs use activations %s, SiLU expected" % sorted(yacts))
    # the network is fed RGB (inference.py:72-83, to_tensor=False, and blobFromImage without swapRB): reversing the
    # stem's input channels makes the engine's BGR page compute the same function
    ysd["model.0.conv.weight"] = np.ascontiguousarray(ysd["model.0.conv.weight"][:, ::-1])

    # ---- cfg: multiples from channel counts and repeats, nc and anchors from Detect -------------------------------
    na = anchors[0].shape[0]
    nc = nos[0] - 5
    anchors_px = [[float(v) for v in (a).reshape(-1)] for a in anchors]
    anchors_px = [[int(v) if v == int(v) else v for v in lv] for lv in anchors_px]
    layers = YOLOV5_V6_BACKBONE + YOLOV5_V6_HEAD
    c_out = {i: ysd["model.%d.cv3.conv.weight" % i].shape[0] if layers[i][2] == "C3" else
             ysd["model.%d.cv2.conv.weight" % i].shape[0] if layers[i][2] == "SPPF" else
             ysd["model.%d.conv.weight" % i].shape[0] for i in range(24) if layers[i][2] in ("Conv", "C3", "SPPF")}

    def fits(gw, gd):
        for i, (_f, n, m, args) in enumerate(layers[:24]):
            if m in ("Conv", "C3", "SPPF") and c_out[i] != int(np.ceil(args[0] * gw / 8) * 8):
                return False
            if m == "C3" and n_of[i] != ((max(round(n * gd), 1) if n > 1 else n), len(args) < 2 or args[1]):
                return False
        return True

    mult = [(gw, gd) for gw in _WIDTHS for gd in _DEPTHS if fits(gw, gd)]
    if not mult:
        raise ValueError("unsupported ONNX graph: channel counts %s and C3 repeats %s follow no yolov5 v6 width / "
                         "depth multiple" % ([c_out[i] for i in sorted(c_out)], [n_of[i] for i in sorted(n_of)]))
    gw, gd = mult[0]
    cfg = {"nc": nc, "depth_multiple": gd, "width_multiple": gw, "anchors": anchors_px,
           "backbone": [list(L) for L in YOLOV5_V6_BACKBONE], "head": [list(L) for L in YOLOV5_V6_HEAD]}
    strides = np.array([8.0, 16.0, 32.0])[:, None, None]
    ysd["model.24.anchors"] = np.stack(anchors) / strides
    ckpt = {"blk_det": {"cfg": cfg, "weights": ysd}, "text_seg": ssd, "text_det": dsd}
    return ckpt, head_act, S


def load_checkpoint(src):
    """An `.onnx` file (path or bytes) -> (checkpoint dict, head_act, input size); see checkpoint_from_graph."""
    return checkpoint_from_graph(read_model(src))
