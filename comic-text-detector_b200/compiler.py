"""Checkpoint -> engine program.

Host-side counterpart of the reference's model construction + weight preparation:
`get_base_det_models` (basemodel.py:211-220), `load_yolov5_ckpt` / `parse_model` / `Model.fuse`
(models/yolov5/yolo.py:285-311, 208-259, 185-192) and `fuse_conv_and_bn`
(utils/yolov5_utils.py:23-43).  It consumes the reference's 3-key checkpoint dict

    {'blk_det': {'cfg': dict, 'weights': state_dict}, 'text_seg': state_dict, 'text_det': state_dict}

folds EVERY BatchNorm (yolo eps 1e-3 per utils/yolov5_utils.py:59; the heads' live BNs,
eps 1e-5, basemodel.py:223, are folded too), eliminates torch.cat by K-concatenated conv
sources / channel-offset destinations, and emits the flat op list + weight blob that
`ctd_create` (include/ctd_b200.h) takes.  Pure numpy; no torch.nn, no CUDA.
"""
import numpy as np

# enum mirrors of include/ctd_b200.h
OP_STEM, OP_CONV, OP_DECONV4, OP_AVGPOOL2, OP_SPPF_POOL, OP_UPSAMPLE2, OP_DETECT, OP_SEG_TAIL, OP_DB_TAIL = range(9)
OP_S2D = 9  # reserved value of a retired op kind: never emitted, no engine kernel; the name stays for existing callers
ACT_NONE, ACT_SILU, ACT_LEAKY, ACT_RELU, ACT_SIGMOID = range(5)
MAX_SRC = 3


def _np(t):
    return t.detach().cpu().numpy().astype(np.float64) if hasattr(t, "detach") else np.asarray(t, np.float64)


def make_divisible(x, d):
    import math
    return math.ceil(x / d) * d


def parse_cfg(cfg):
    """Topology walk of the yolov5 cfg dict for the module kinds the shipped yolov5s cfg uses
    (Conv, C3, SPPF, nn.Upsample, Concat, Detect) -- models/yolov5/yolo.py:208-259."""
    gd, gw = cfg["depth_multiple"], cfg["width_multiple"]
    nc, anchors = cfg["nc"], cfg["anchors"]
    na = len(anchors[0]) // 2
    no = na * (nc + 5)
    ch = [cfg.get("ch", 3)]
    layers = []
    for i, (f, n, m, args) in enumerate(cfg["backbone"] + cfg["head"]):
        m = m if isinstance(m, str) else getattr(m, "__name__", str(m))
        args = [nc if a == "nc" else anchors if a == "anchors" else a for a in args]
        n = max(round(n * gd), 1) if n > 1 else n
        if m in ("Conv", "C3", "SPPF"):
            c1, c2 = ch[f], args[0]
            if c2 != no:
                c2 = make_divisible(c2 * gw, 8)
            L = dict(i=i, f=f, type=m, c1=c1, c2=c2)
            if m == "Conv":
                L.update(k=args[1] if len(args) > 1 else 1, s=args[2] if len(args) > 2 else 1,
                         p=args[3] if len(args) > 3 else None)
            elif m == "C3":
                L.update(n=n, shortcut=args[1] if len(args) > 1 else True)
            else:
                L.update(k=args[1] if len(args) > 1 else 5)
        elif m == "Concat":
            c2 = sum(ch[x] for x in f)
            L = dict(i=i, f=f, type=m, c2=c2)
        elif m == "Detect":
            c2 = None
            L = dict(i=i, f=f, type=m, nc=nc, anchors=anchors, ch=[ch[x] for x in f], c2=None)
        elif m in ("nn.Upsample", "Upsample"):
            c2 = ch[f]
            L = dict(i=i, f=f, type="Upsample", c2=c2)
        else:
            raise ValueError("cfg module %r is not part of the supported yolov5s graph" % (m,))
        layers.append(L)
        if i == 0:
            ch = []
        ch.append(c2)
    return layers


class Program:
    """Flat op list + buffer table + weight blob."""

    def __init__(self):
        self.ops = []
        self.bufs = []  # (channels, down)
        self.blob = bytearray()
        self.names = {}  # debug: name -> tensor

    def newbuf(self, channels, down):
        self.bufs.append((int(channels), int(down)))
        return len(self.bufs) - 1

    def tensor(self, buf, coff, c):
        return dict(buf=buf, coff=coff, c=c, down=self.bufs[buf][1])

    def add_blob(self, arr):
        pad = (-len(self.blob)) % 256
        self.blob += b"\0" * pad
        off = len(self.blob)
        self.blob += np.ascontiguousarray(arr).tobytes()
        return off

    def _op(self, kind, srcs, dst, **kw):
        op = dict(kind=kind, n_src=len(srcs), src_buf=[0] * MAX_SRC, src_coff=[0] * MAX_SRC, src_c=[0] * MAX_SRC,
                  dst_buf=-1, dst_coff=0, cout=0, cout_pad=0, ksize=1, stride=1, act=ACT_NONE, residual=0, aux=0,
                  w16_off=0, w32_off=0, b_off=0, p_off=0)
        assert 1 <= len(srcs) <= MAX_SRC
        for i, s in enumerate(srcs):
            op["src_buf"][i], op["src_coff"][i], op["src_c"][i] = s["buf"], s["coff"], s["c"]
        if dst is not None:
            op["dst_buf"], op["dst_coff"] = dst["buf"], dst["coff"]
        op.update(kw)
        self.ops.append(op)
        return op

    # ---- GEMM-shaped ops -------------------------------------------------------------------
    def _pack(self, wk, bias, cout):
        """wk: [phase][cout][K] float64 -> pads rows to a multiple of 16, stores fp16 + fp32 + bias."""
        cout_pad = (cout + 15) // 16 * 16
        nph, _, K = wk.shape
        wp = np.zeros((nph, cout_pad, K), np.float32)
        wp[:, :cout] = wk.astype(np.float32)
        bp = np.zeros((cout_pad,), np.float32)
        bp[:cout] = bias.astype(np.float32)
        return dict(cout=cout, cout_pad=cout_pad, w16_off=self.add_blob(wp.astype(np.float16)),
                    w32_off=self.add_blob(wp), b_off=self.add_blob(bp))

    def conv(self, srcs, w, b, stride, act, dst=None, residual=False):
        """w: [Co][Ci][k][k] (BN already folded), K order = (ky, kx, ci) with ci running over the
        concatenated sources."""
        co, ci, k, _ = w.shape
        assert ci == sum(s["c"] for s in srcs), (ci, [s["c"] for s in srcs])
        down = srcs[0]["down"] * stride
        if dst is None:
            dst = self.tensor(self.newbuf(co, down), 0, co)
        wk = w.transpose(0, 2, 3, 1).reshape(1, co, k * k * ci)
        self._op(OP_CONV, srcs, dst, ksize=k, stride=stride, act=act, residual=int(residual), **self._pack(wk, b, co))
        return self.tensor(dst["buf"], dst["coff"], co)

    def deconv4(self, srcs, w, b, act):
        """w: [Ci][Co][4][4] (torch ConvTranspose2d layout, BN folded). out = 2*in - 1 + k."""
        ci, co = w.shape[:2]
        assert ci == sum(s["c"] for s in srcs)
        KY = ((1, 3), (0, 2))  # phase parity -> kernel index of tap 0 (d=0 / +1) and tap 1 (d=-1 / 0)
        wk = np.zeros((4, co, 4 * ci), np.float64)
        for py in range(2):
            for px in range(2):
                for ty in range(2):
                    for tx in range(2):
                        t = ty * 2 + tx
                        wk[py * 2 + px, :, t * ci:(t + 1) * ci] = w[:, :, KY[py][ty], KY[px][tx]].T
        down = srcs[0]["down"] // 2
        dst = self.tensor(self.newbuf(co, down), 0, co)
        self._op(OP_DECONV4, srcs, dst, ksize=4, stride=2, act=act, **self._pack(wk, b, co))
        return dst

    def detect(self, src, w, b, level, stride, anchors_px):
        co = w.shape[0]
        wk = w.reshape(1, co, -1)
        prm = np.array([stride] + list(anchors_px), np.float32)
        self._op(OP_DETECT, [src], None, ksize=1, stride=1, aux=level, p_off=self.add_blob(prm), **self._pack(wk, b, co))


def fold_bn(w, conv_bias, sd, bn_prefix, eps, transposed=False):
    """(w, b) of conv followed by eval-mode BatchNorm -> single affine conv
    (same algebra as utils/yolov5_utils.py:23-43, carried out in float64).  A conv with a bias and no BatchNorm
    entries is one whose BatchNorm was already folded (the ONNX exporter does that, onnx_model.py): returned as is."""
    if conv_bias is not None and bn_prefix + ".weight" not in sd:
        return w, conv_bias
    g, beta = _np(sd[bn_prefix + ".weight"]), _np(sd[bn_prefix + ".bias"])
    mu, var = _np(sd[bn_prefix + ".running_mean"]), _np(sd[bn_prefix + ".running_var"])
    scale = g / np.sqrt(var + eps)
    if transposed:
        wf = w * scale[None, :, None, None]
    else:
        wf = w * scale[:, None, None, None]
    b0 = np.zeros_like(mu) if conv_bias is None else conv_bias
    return wf, (b0 - mu) * scale + beta


def compile_checkpoint(ckpt, head_act="leaky"):
    """Returns a Program for the full TextDetBase.forward graph (basemodel.py:240-244)."""
    P = Program()
    cfg = ckpt["blk_det"]["cfg"]
    ysd, ssd, dsd = ckpt["blk_det"]["weights"], ckpt["text_seg"], ckpt["text_det"]
    layers = parse_cfg(cfg)
    hact = {"leaky": ACT_LEAKY, "relu": ACT_RELU}.get(head_act, ACT_SILU if head_act is True else ACT_NONE)

    def bias(sd, key):   # only convs whose BatchNorm is already folded have one
        return _np(sd[key]) if key in sd else None

    def yconv(prefix):
        return fold_bn(_np(ysd[prefix + ".conv.weight"]), bias(ysd, prefix + ".conv.bias"), ysd, prefix + ".bn", 1e-3)

    def hconv(sd, prefix):
        return fold_bn(_np(sd[prefix + ".conv.weight"]), bias(sd, prefix + ".conv.bias"), sd, prefix + ".bn", 1e-5)

    def c3(srcs, get, prefix, n, shortcut, act):
        """C3.forward (common.py:137-138): cv3(cat(m(cv1(x)), cv2(x))); cv1||cv2 share x -> one GEMM."""
        w1, b1 = get(prefix + ".cv1")
        w2, b2 = get(prefix + ".cv2")
        c_ = w1.shape[0]
        down = srcs[0]["down"]
        Y = P.newbuf(2 * c_, down)
        P.conv(srcs, np.concatenate([w1, w2], 0), np.concatenate([b1, b2], 0), 1, act, dst=P.tensor(Y, 0, 2 * c_))
        cur = P.tensor(Y, 0, c_)
        for j in range(n):
            wa, ba = get("%s.m.%d.cv1" % (prefix, j))
            wb, bb = get("%s.m.%d.cv2" % (prefix, j))
            t = P.conv([cur], wa, ba, 1, act)
            # Bottleneck (common.py:103-104): x + cv2(cv1(x)), written in place over x
            P.conv([t], wb, bb, 1, act, dst=cur, residual=bool(shortcut))
        w3, b3 = get(prefix + ".cv3")
        if cur["buf"] == Y:
            return P.conv([P.tensor(Y, 0, 2 * c_)], w3, b3, 1, act)
        return P.conv([cur, P.tensor(Y, c_, c_)], w3, b3, 1, act)   # cv3(cat(m(cv1 x), cv2 x)): K-concatenated

    # ---- blk_det (yolo.py:115-134) -----------------------------------------------------------
    outs = []
    x = None
    for L in layers:
        i, f, t = L["i"], L["f"], L["type"]
        pfx = "model.%d" % i
        if i == 0:
            inp = None
        elif f == -1:
            inp = x
        elif isinstance(f, int):
            inp = outs[f]
        else:
            inp = [x if j == -1 else outs[j] for j in f]
        if t == "Conv":
            w, b = yconv(pfx)
            if i == 0:
                assert L["k"] == 6 and L["s"] == 2 and w.shape[1] == 3 and w.shape[0] <= 32, "stem must be Conv(3,<=32,6,2,2)"
                co = w.shape[0]
                dst = P.tensor(P.newbuf(co, 2), 0, co)
                w32 = w.transpose(0, 2, 3, 1).reshape(co, 108).astype(np.float32)
                bp = np.zeros((32,), np.float32)
                bp[:co] = b
                # tensor-core form: 6x6 s2 p2 over 3 channels == 3x3 s1 p1 over the 2x2 space-to-depth page
                # (ky = 2a+dy, kx = 2b+dx, s2d channel = (dy*2+dx)*3 + c, 12 -> 16 channels).  One K block per
                # filter ROW a: the 4-pixel window (x-1 .. x+2) x 16 channels = 64 contiguous fp16 of the padded
                # s2d buffer (the 4th pixel has zero weights), so K = 3 x 64.
                w3 = np.zeros((co, 16, 3, 3), np.float64)
                for dy in range(2):
                    for dx in range(2):
                        for c in range(3):
                            w3[:, (dy * 2 + dx) * 3 + c] = w[:, c, dy::2, dx::2]
                wwin = np.zeros((32, 3, 4, 16), np.float32)
                wwin[:co, :, :3, :] = w3.transpose(0, 2, 3, 1)  # [co][a][b][ch]
                s2d = P.tensor(P.newbuf(16, 2), 0, 16)
                P._op(OP_STEM, [s2d], dst, ksize=6, stride=2, act=ACT_SILU, cout=co, cout_pad=32,
                      w32_off=P.add_blob(w32), w16_off=P.add_blob(wwin.reshape(32, 192).astype(np.float16)),
                      b_off=P.add_blob(bp))
                x = [dst]
            else:
                x = [P.conv(inp, w, b, L["s"], ACT_SILU)]
        elif t == "C3":
            x = [c3(inp, yconv, pfx, L["n"], L["shortcut"], ACT_SILU)]
        elif t == "SPPF":
            w1, b1 = yconv(pfx + ".cv1")
            c_ = w1.shape[0]
            buf = P.newbuf(4 * c_, inp[0]["down"])
            P.conv(inp, w1, b1, 1, ACT_SILU, dst=P.tensor(buf, 0, c_))
            P._op(OP_SPPF_POOL, [P.tensor(buf, 0, c_)], None)
            w2, b2 = yconv(pfx + ".cv2")
            x = [P.conv([P.tensor(buf, 0, 4 * c_)], w2, b2, 1, ACT_SILU)]
        elif t == "Upsample":
            s = inp[0]
            assert len(inp) == 1
            dst = P.tensor(P.newbuf(s["c"], s["down"] // 2), 0, s["c"])
            P._op(OP_UPSAMPLE2, [s], dst)
            x = [dst]
        elif t == "Concat":
            x = [s for part in inp for s in part]
        elif t == "Detect":
            na = len(L["anchors"][0]) // 2
            anchors = _np(ysd[pfx + ".anchors"])  # (nl, na, 2), already / stride (yolo.py:85)
            for li, part in enumerate(inp):
                assert len(part) == 1
                stride = float(part[0]["down"])
                w = _np(ysd["%s.m.%d.weight" % (pfx, li)])
                b = _np(ysd["%s.m.%d.bias" % (pfx, li)])
                P.detect(part[0], w, b, li, stride, (anchors[li] * stride).reshape(-1))
            x = None
        outs.append(x)
    f256, f128, f64, f32, f3 = (outs[k][0] for k in (1, 3, 5, 7, 9))  # out_indices (yolo.py:286,310)

    # ---- text_seg: UnetHead.forward (basemodel.py:62-78) ---------------------------------------
    def up_c3(sd, srcs, pfx):
        """double_conv_up_c3 (basemodel.py:21-32)."""
        y = c3(srcs, lambda p_: hconv(sd, p_), pfx + ".conv.0", 1, True, hact)
        w, b = fold_bn(_np(sd[pfx + ".conv.1.weight"]), None, sd, pfx + ".conv.2", 1e-5, transposed=True)
        return P.deconv4([y], w, b, ACT_RELU)

    pooled = P.tensor(P.newbuf(f3["c"], f3["down"] * 2), 0, f3["c"])
    P._op(OP_AVGPOOL2, [f3], pooled)
    d16 = c3([pooled], lambda p_: hconv(ssd, p_), "down_conv1.conv", 1, True, hact)
    u32 = up_c3(ssd, [d16], "upconv0")
    u64 = up_c3(ssd, [f32, u32], "upconv2")
    u128 = up_c3(ssd, [f64, u64], "upconv3")
    u256 = up_c3(ssd, [f128, u128], "upconv4")
    u512 = up_c3(ssd, [f256, u256], "upconv5")
    w6 = _np(ssd["upconv6.0.weight"])  # (C,1,4,4)
    # tensor-core form: the four sub-pixel phases of ConvT 4x4 s2 p1 (C -> 1) as ONE 3x3 convolution with
    # 4 output channels (n = py*2+px; phase taps (d, k): parity 0 -> (0,1),(-1,3); parity 1 -> (0,2),(+1,0))
    ci6 = w6.shape[0]
    wc = np.zeros((16, 3, 3, ci6), np.float32)
    TAPS = (((0, 1), (-1, 3)), ((0, 2), (1, 0)))
    for py in range(2):
        for px in range(2):
            for dy, ky in TAPS[py]:
                for dx, kx in TAPS[px]:
                    wc[py * 2 + px, dy + 1, dx + 1, :] = w6[:, 0, ky, kx]
    P._op(OP_SEG_TAIL, [u512], None, p_off=P.add_blob(w6.reshape(w6.shape[0], 16).astype(np.float32)),
          w16_off=P.add_blob(wc.reshape(16, 9 * ci6).astype(np.float16)), cout=4, cout_pad=16)

    # ---- text_det: DBHead.forward (basemodel.py:106-125) ----------------------------------------
    du128 = up_c3(dsd, [f64, u64], "upconv3")
    dx = up_c3(dsd, [f128, du128], "upconv4")
    w, b = fold_bn(_np(dsd["conv.0.weight"]), _np(dsd["conv.0.bias"]), dsd, "conv.1", 1e-5)
    dx = P.conv([dx], w, b, 1, ACT_RELU)
    wb, bb = fold_bn(_np(dsd["binarize.0.weight"]), _np(dsd["binarize.0.bias"]), dsd, "binarize.1", 1e-5)
    wt, bt = fold_bn(_np(dsd["thresh.0.weight"]),
                     _np(dsd["thresh.0.bias"]) if "thresh.0.bias" in dsd else None, dsd, "thresh.1", 1e-5)
    assert wb.shape[0] == 16 and wt.shape[0] == 16, "DB tail kernel is specialised for inner_channels//4 == 16"
    t32 = P.conv([dx], np.concatenate([wb, wt], 0), np.concatenate([bb, bt], 0), 1, ACT_RELU)
    prm = []
    for name in ("binarize", "thresh"):
        w3, b3 = fold_bn(_np(dsd[name + ".3.weight"]), _np(dsd[name + ".3.bias"]), dsd, name + ".4", 1e-5, transposed=True)
        w6_, b6_ = _np(dsd[name + ".6.weight"]), _np(dsd[name + ".6.bias"])
        prm += [w3.reshape(-1), b3.reshape(-1), w6_.reshape(-1), b6_.reshape(-1)]  # 1024 + 16 + 64 + 1
    P._op(OP_DB_TAIL, [t32], None, p_off=P.add_blob(np.concatenate(prm).astype(np.float32)))
    P.names.update(f256=f256, f128=f128, f64=f64, f32=f32, f3=f3, u64=u64, u512=u512, t32=t32)
    P.nc = cfg["nc"]
    return P
