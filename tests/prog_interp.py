"""TEST INFRASTRUCTURE: a slow CPU interpreter of the engine program (op list + weight blob) in
torch fp32.  It executes exactly what comic-text-detector_b200/compiler.py emitted -- packed
weights, K-concatenated sources, channel-offset destinations, in-place residuals, deconv phases --
so the compiler / weight packing can be pinned against the oracle WITHOUT a GPU.  It shares no
code with the CUDA kernels."""
import numpy as np
import torch
import torch.nn.functional as F

from ctd_b200 import compiler as cc


def _act(x, a):
    if a == cc.ACT_SILU:
        return F.silu(x)
    if a == cc.ACT_LEAKY:
        return F.leaky_relu(x, 0.1)
    if a == cc.ACT_RELU:
        return F.relu(x)
    if a == cc.ACT_SIGMOID:
        return torch.sigmoid(x)
    return x


def _blob(prog, off, count, dtype):
    return torch.from_numpy(np.frombuffer(prog.blob, dtype=dtype, count=count, offset=off).copy())


class Interp:
    """Step-by-step interpreter.  storage='f32': exact fp32 reference of the program.  storage='f16': emulation of
    the tensor-core engine's numerics -- fp16 weights, every activation rounded to fp16 when it is stored, fp32
    accumulation, the stem in its space-to-depth window form, the seg tail in its 3x3 / 4-phase fp16 form."""

    def __init__(self, prog, pages, storage="f32"):
        self.prog, self.pages, self.f16 = prog, pages, storage == "f16"
        n, h, w, _ = pages.shape
        self.n, self.h, self.w = n, h, w
        self.bufs = [torch.zeros(n, c, h // d, w // d) for c, d in prog.bufs]  # NCHW here
        self.no = 5 + prog.nc
        rows = 3 * ((h // 8) * (w // 8) + (h // 16) * (w // 16) + (h // 32) * (w // 32))
        self.blks = torch.zeros(n, rows, self.no)
        self.mask = self.lines = None

    def q(self, x):
        return x.half().float() if self.f16 else x

    def buf_nhwc(self, b):
        return np.ascontiguousarray(self.bufs[b].permute(0, 2, 3, 1).numpy())

    def written(self, op):
        """(buf, coff, c) of the slice op writes, or None for ops writing engine outputs."""
        k = op["kind"]
        if k == cc.OP_SPPF_POOL:
            return op["src_buf"][0], op["src_coff"][0] + op["src_c"][0], 3 * op["src_c"][0]
        if op["dst_buf"] < 0:
            return None
        c = op["cout"] if k in (cc.OP_STEM, cc.OP_CONV, cc.OP_DECONV4) else op["src_c"][0]
        return op["dst_buf"], op["dst_coff"], c

    def step(self, i):
        prog, pages, bufs, n, h, w, no = self.prog, self.pages, self.bufs, self.n, self.h, self.w, self.no
        use_fp16_weights = self.f16
        op = prog.ops[i]
        k = op["kind"]
        srcs = [bufs[op["src_buf"][j]][:, op["src_coff"][j]:op["src_coff"][j] + op["src_c"][j]] for j in range(op["n_src"])]
        if k == cc.OP_STEM and use_fp16_weights:
            # tensor-core form of the stem: window-layout fp16 weights over the space-to-depth page
            x = torch.from_numpy(np.ascontiguousarray(pages.transpose(0, 3, 1, 2)).astype(np.float32) / 255).half().float()
            s2d = torch.zeros(n, 16, h // 2, w // 2)
            for dy in range(2):
                for dx in range(2):
                    s2d[:, (dy * 2 + dx) * 3:(dy * 2 + dx) * 3 + 3] = x[:, :, dy::2, dx::2]
            ww = _blob(prog, op["w16_off"], 32 * 192, np.float16).float().view(32, 3, 4, 16)[:op["cout"], :, :3]
            wt = ww.permute(0, 3, 1, 2)  # [co][ch][a][b]
            b = _blob(prog, op["b_off"], op["cout"], np.float32)
            y = _act(F.conv2d(s2d, wt, b, 1, 1), op["act"])
            bufs[op["dst_buf"]][:, op["dst_coff"]:op["dst_coff"] + op["cout"]] = self.q(y)
            return
        cin = sum(op["src_c"][:op["n_src"]])
        if k == cc.OP_STEM:
            x = torch.from_numpy(np.ascontiguousarray(pages.transpose(0, 3, 1, 2)).astype(np.float32) / 255)
            wt = _blob(prog, op["w32_off"], op["cout"] * 108, np.float32).view(op["cout"], 6, 6, 3).permute(0, 3, 1, 2)
            b = _blob(prog, op["b_off"], op["cout"], np.float32)
            y = _act(F.conv2d(x, wt, b, 2, 2), op["act"])
            bufs[op["dst_buf"]][:, op["dst_coff"]:op["dst_coff"] + op["cout"]] = y
        elif k in (cc.OP_CONV, cc.OP_DETECT):
            ks, st = op["ksize"], op["stride"]
            K = ks * ks * cin
            if use_fp16_weights:
                wk = _blob(prog, op["w16_off"], op["cout_pad"] * K, np.float16).float()
            else:
                wk = _blob(prog, op["w32_off"], op["cout_pad"] * K, np.float32)
            wt = wk.view(op["cout_pad"], ks, ks, cin)[:op["cout"]].permute(0, 3, 1, 2)
            b = _blob(prog, op["b_off"], op["cout_pad"], np.float32)[:op["cout"]]
            y = F.conv2d(torch.cat(srcs, 1), wt, b, st, ks // 2)
            if k == cc.OP_CONV:
                y = _act(y, op["act"])
                dst = bufs[op["dst_buf"]][:, op["dst_coff"]:op["dst_coff"] + op["cout"]]
                if op["residual"]:
                    y = y + dst
                bufs[op["dst_buf"]][:, op["dst_coff"]:op["dst_coff"] + op["cout"]] = self.q(y)
            else:
                prm = _blob(prog, op["p_off"], 7, np.float32)
                stride, anch = float(prm[0]), prm[1:].view(3, 2)
                bs, _, ny, nx = y.shape
                y = y.view(bs, 3, no, ny, nx).permute(0, 1, 3, 4, 2).sigmoid()
                yv, xv = torch.meshgrid([torch.arange(ny), torch.arange(nx)], indexing="ij")
                grid = torch.stack((xv, yv), 2).float()
                out = y.clone()
                out[..., 0:2] = (y[..., 0:2] * 2 - 0.5 + grid) * stride
                out[..., 2:4] = (y[..., 2:4] * 2) ** 2 * anch.view(1, 3, 1, 1, 2)
                r0 = sum(3 * (h // (8 << l)) * (w // (8 << l)) for l in range(op["aux"]))
                self.blks[:, r0:r0 + 3 * ny * nx] = out.reshape(bs, -1, no)
        elif k == cc.OP_DECONV4:
            K = 4 * cin
            wk = (_blob(prog, op["w16_off"], 4 * op["cout_pad"] * K, np.float16).float() if use_fp16_weights
                  else _blob(prog, op["w32_off"], 4 * op["cout_pad"] * K, np.float32)).view(4, op["cout_pad"], 4, cin)
            b = _blob(prog, op["b_off"], op["cout_pad"], np.float32)[:op["cout"]]
            x = torch.cat(srcs, 1)
            nb, _, ih, iw = x.shape
            out = torch.zeros(nb, op["cout"], 2 * ih, 2 * iw)
            d = ((0, -1), (1, 0))
            xp = F.pad(x, (1, 1, 1, 1))
            for ph in range(4):
                py, px = ph >> 1, ph & 1
                acc = torch.zeros(nb, op["cout"], ih, iw)
                for t in range(4):
                    dy, dx = d[py][t >> 1], d[px][t & 1]
                    xs = xp[:, :, 1 + dy:1 + dy + ih, 1 + dx:1 + dx + iw]
                    acc += torch.einsum("nchw,oc->nohw", xs, wk[ph, :op["cout"], t])
                out[:, :, py::2, px::2] = acc
            y = _act(out + b.view(1, -1, 1, 1), op["act"])
            bufs[op["dst_buf"]][:, op["dst_coff"]:op["dst_coff"] + op["cout"]] = self.q(y)
        elif k == cc.OP_AVGPOOL2:
            bufs[op["dst_buf"]][:, op["dst_coff"]:op["dst_coff"] + op["src_c"][0]] = self.q(F.avg_pool2d(srcs[0], 2, 2))
        elif k == cc.OP_SPPF_POOL:
            c = op["src_c"][0]
            c0 = op["src_coff"][0]
            y1 = F.max_pool2d(srcs[0], 5, 1, 2)
            y2 = F.max_pool2d(y1, 5, 1, 2)
            y3 = F.max_pool2d(y2, 5, 1, 2)
            B = bufs[op["src_buf"][0]]
            B[:, c0 + c:c0 + 2 * c], B[:, c0 + 2 * c:c0 + 3 * c], B[:, c0 + 3 * c:c0 + 4 * c] = y1, y2, y3
        elif k == cc.OP_UPSAMPLE2:
            bufs[op["dst_buf"]][:, op["dst_coff"]:op["dst_coff"] + op["src_c"][0]] = F.interpolate(srcs[0], scale_factor=2, mode="nearest")
        elif k == cc.OP_SEG_TAIL:
            c = op["src_c"][0]
            if use_fp16_weights and op["w16_off"] > 0:
                # tensor-core form: 3x3 conv with the 4 sub-pixel phases as output channels, fp16 weights
                wc = _blob(prog, op["w16_off"], 16 * 9 * c, np.float16).float().view(16, 3, 3, c)[:4].permute(0, 3, 1, 2)
                y = F.conv2d(srcs[0], wc, None, 1, 1)                       # [n][4][h][w], phase = py*2+px
                nb, _, ih, iw = y.shape
                out = torch.zeros(nb, 1, 2 * ih, 2 * iw)
                for py in range(2):
                    for px in range(2):
                        out[:, 0, py::2, px::2] = y[:, py * 2 + px]
                self.mask = torch.sigmoid(out)
            else:
                wt = _blob(prog, op["p_off"], c * 16, np.float32).view(c, 1, 4, 4)
                self.mask = torch.sigmoid(F.conv_transpose2d(srcs[0], wt, None, 2, 1))
        elif k == cc.OP_DB_TAIL:
            prm = _blob(prog, op["p_off"], 2 * 1105, np.float32)
            outs = []
            for b_ in range(2):
                q = prm[b_ * 1105:(b_ + 1) * 1105]
                w3, b3 = q[:1024].view(16, 16, 2, 2), q[1024:1040]
                w6, b6 = q[1040:1104].view(16, 1, 2, 2), q[1104:1105]
                x = srcs[0][:, b_ * 16:(b_ + 1) * 16]
                t = F.relu(F.conv_transpose2d(x, w3, b3, 2))
                outs.append(torch.sigmoid(F.conv_transpose2d(t, w6, b6, 2)))
            self.lines = torch.cat(outs, 1)


def run_program(prog, pages, use_fp16_weights=False, storage=None):
    """pages u8 [n][h][w][3] -> (blks, mask, lines) like the engine's net outputs.  storage='f16' emulates the
    tensor-core engine (fp16 weights AND fp16 activation storage); use_fp16_weights alone keeps fp32 activations."""
    it = Interp(prog, pages, storage or "f32")
    if use_fp16_weights and storage is None:
        it.f16 = True
        it.q = lambda x: x          # historical mode: fp16 weights, fp32 activations
    for i in range(len(prog.ops)):
        it.step(i)
    return it.blks, it.mask, it.lines
