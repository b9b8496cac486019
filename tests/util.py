"""Shared helpers for the parity tests."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import ctd_b200  # noqa: E402
from ctd_b200 import compiler as cc  # noqa: E402
from ctd_b200.binding import PREC_FP16_TC, PREC_FP32_SIMT, PREC_FP16_SIMT, PREC_SPLIT_TC  # noqa: E402

_CKPT_CACHE = {}


def get_checkpoint(seed=0, smooth=True):
    from oracle import synth
    key = (seed, smooth)
    if key not in _CKPT_CACHE:
        _CKPT_CACHE[key] = synth.make_checkpoint(seed, smooth=smooth)
    return _CKPT_CACHE[key]


def h16(a):
    """round to fp16 and back (what the fp16 engine stores)."""
    return np.asarray(a, np.float32).astype(np.float16).astype(np.float32)


def page_to_net_input(pages):
    """u8 [n][h][w][3] BGR -> f32 (n,3,h,w) BGR /255: what preprocess_img feeds the torch backend
    for net-sized pages (inference.py:72-83)."""
    return torch.from_numpy(np.ascontiguousarray(pages.transpose(0, 3, 1, 2)).astype(np.float32) / 255)


class SingleOp:
    """Builds a one-op program around Program.conv/deconv4 with writable source buffers."""

    def __init__(self, src_channels, down=1, extra_channels=0):
        self.P = cc.Program()
        self.P.nc = 2
        self.srcs = []
        for c in src_channels:
            # source tensors sit at a channel offset inside wider buffers to exercise slicing
            b = self.P.newbuf(c + extra_channels, down)
            self.srcs.append(self.P.tensor(b, extra_channels, c))

    def run(self, out_tensor, inputs, n, h, w, precision, dst_init=None, full_dst=False):
        """full_dst: return every channel of the destination buffer, not only the op's slice."""
        eng = ctd_b200.Engine(self.P, precision=precision, max_batch=n, max_h=h, max_w=w, skip_postproc=True)
        try:
            for t, arr in zip(self.srcs, inputs):
                ch = self.P.bufs[t["buf"]][0]
                full = np.zeros(arr.shape[:3] + (ch,), np.float32)
                full[..., t["coff"]:t["coff"] + t["c"]] = arr
                eng.debug_write(t, full, n, h, w)
            if dst_init is not None:
                eng.debug_write(out_tensor, dst_init, n, h, w)
            eng.forward(np.zeros((n, h, w, 3), np.uint8))
            if full_dst:
                return eng.debug_read(dict(out_tensor, coff=0, c=self.P.bufs[out_tensor["buf"]][0]))
            return eng.debug_read(out_tensor)
        finally:
            eng.close()


# ---------------------------------------------------------------------------------------------------------------
# Launch plan of conv_tc_kernel, replicated from conv_tc_plan (csrc/conv_tc.cu): the N-block width BN and the tile
# count decide which instantiation runs and how many tiles each persistent CTA loops over.
TILE_W, TILE_H = 16, 8
H100_SMS = 132


def pick_block_n(cout_pad):
    if cout_pad >= 128 and cout_pad % 128 == 0:
        return 128
    if cout_pad % 64 == 0:
        return 64
    if cout_pad % 32 == 0:
        return 32
    return 16


def tc_plan(cout, gh, gw, n_img, n_phase=1, split=False, num_sms=H100_SMS):
    """-> dict(bn, tiles, grid, tiles_per_cta, partial) of the conv_tc_kernel launch for a grid of gh x gw pixels."""
    cout_pad = (cout + 15) // 16 * 16
    spatial = n_img * -(-gw // TILE_W) * -(-gh // TILE_H) * n_phase
    bn = pick_block_n(cout_pad)
    while bn > 64 and spatial * (cout_pad // bn) <= num_sms // 2:
        bn //= 2
    if split and bn > 64:
        bn = 64
    tiles = spatial * (cout_pad // bn)
    grid = min(tiles, num_sms)
    return dict(bn=bn, tiles=tiles, grid=grid, tiles_per_cta=-(-tiles // grid),
                partial=gw % TILE_W != 0 or gh % TILE_H != 0)


# ---------------------------------------------------------------------------------------------------------------
# Elementwise error bound of one tensor-core convolution against a float64 reference:
#
#     |got - ref| <= a * |ref| + b(K) * M,      M = |bias| + conv(|X|, |W|)
#
# M bounds every partial sum the accumulator can hold, so b(K) * M covers the accumulation and operand rounding and
# a * |ref| the rounding of the stored result.  ref and M are float64 of the operands the kernel really used.
def fp16_tc_ab(K):
    """fp16 engine: fp16 operands (exact products), fp32 wgmma accumulation, fp16 output."""
    # a: 2^-11 is the fp16 rounding of the output (half an ulp of 11 significant bits); 2^-20 the fast exp /
    #    __fdividef of SiLU and sigmoid (a few fp32 ulps relative to the activation).
    a = 2.0 ** -11 + 2.0 ** -20
    # b: every K = 16 wgmma truncates its fp32 sum once on the way in and once into the accumulator (2 ulps, 2^-23
    #    relative to a partial sum <= M, per K step), +4 ulps for the bias add, activation and residual add in fp32;
    #    1.1 is the largest slope of the activations (SiLU: 1.0998), which carries the pre-activation error through.
    b = 1.1 * (2 * -(-K // 16) + 4) * 2.0 ** -23
    return a, b


def split_tc_ab(K):
    """split-fp16 engine: fp32 operands as fp16 hi + lo, promoted fp32 accumulation, fp32 output."""
    # a: the fp32 result rounding and the precise expf / division of the epilogue (2 ulps of 2^-24 = 2^-23) with 2x
    #    margin.
    a = 2.0 ** -22
    # b: hi + lo carries 22 significant bits of each operand (2^-23 relative each, so 2^-22 per product: 2^-21 is
    #    2x margin); each hi x hi wgmma (K = 16) lands in a fresh accumulator that is added to the running sum with
    #    round-to-nearest, one 2^-24 rounding per K step relative to a partial sum <= M.  The cross terms are
    #    2^-11 of the sum, so their tensor-core truncation (2^-23 of that) is below every term above.
    b = 2.0 ** -21 + -(-K // 16) * 2.0 ** -24
    return a, b


def simt_ab(K, fp16_out=False):
    """CUDA-core engines (conv_simt_kernel, stem_kernel): exact operands (fp32, or fp16 widened to fp32), one fp32
    FMA chain of K terms per output, fp32 epilogue, fp32 or fp16 output."""
    # a: expf is within 2 ulps (2^-22 relative), the 1 + e and the division of SiLU / sigmoid and the residual add
    #    round once each (3 x 2^-24): 1.75 x 2^-22 in all, under 2^-21.  An fp16 output adds its own rounding, 2^-11.
    a = 2.0 ** -21 + (2.0 ** -11 if fp16_out else 0.0)
    # b: every FMA rounds once, 2^-24 relative to a partial sum <= M; K FMAs, the bias add and 3 ulps of headroom for
    #    the activation's internal roundings (the +4 of fp16_tc_ab); 1.1 is SiLU's largest slope, which carries the
    #    pre-activation error through.
    b = 1.1 * (K + 4) * 2.0 ** -24
    return a, b


def bound_ratio(got, ref, M, a, b, ref_mag=None):
    """Elementwise |got - ref| / (a * |ref| + b * M) as float64 (torch or numpy in, same kind out).  ref_mag replaces
    |ref| in the bound where the output is computed through a cancellation (Detect box centres)."""
    if isinstance(ref, torch.Tensor):
        got = torch.as_tensor(got, device=ref.device).double()
        rm = ref.abs() if ref_mag is None else ref_mag
        return (got - ref).abs() / (a * rm + b * M + 1e-300)
    got = np.asarray(got, np.float64)
    rm = np.abs(ref) if ref_mag is None else ref_mag
    return np.abs(got - ref) / (a * rm + b * M + 1e-300)


def blob_tensor(prog, off, count, dtype, device="cuda"):
    """`count` values of `dtype` at byte offset `off` of the program's weight blob, as a torch tensor."""
    return torch.from_numpy(np.frombuffer(prog.blob, dtype=dtype, count=count, offset=off).copy()).to(device)


def nchw_f64(arr, img, device="cuda"):
    """image `img` of an engine buffer read as [n][h][w][c] -> float64 [1][c][h][w]."""
    return torch.from_numpy(np.ascontiguousarray(arr[img])).to(device).permute(2, 0, 1)[None].double()


def conv_ref_mag(x, w, bias, stride, pad):
    """float64 conv2d and its magnitude M = |bias| + conv(|x|, |w|); x [n][ci][h][w], w [co][ci][k][k]."""
    x, w, bias = x.double(), w.double(), bias.double()
    ref = torch.nn.functional.conv2d(x, w, bias, stride, pad)
    mag = torch.nn.functional.conv2d(x.abs(), w.abs(), bias.abs(), stride, pad)
    return ref, mag


def deconv4_ref_mag(x, wk, bias):
    """ConvTranspose 4x4 s2 p1 from the engine's packed phase weights wk [4][co][4 * ci] (K order = (tap, ci)) in
    float64: returns ref and M, both [n][co][2h][2w]."""
    x, wk, bias = x.double(), wk.double(), bias.double()
    n, ci, h, w = x.shape
    co = wk.shape[1]
    xp = torch.nn.functional.pad(x, (1, 1, 1, 1))
    d = ((0, -1), (1, 0))
    ref = x.new_zeros(n, co, 2 * h, 2 * w)
    mag = x.new_zeros(n, co, 2 * h, 2 * w)
    for ph in range(4):
        py, px = ph >> 1, ph & 1
        xs = torch.cat([xp[:, :, 1 + d[py][t >> 1]:1 + d[py][t >> 1] + h, 1 + d[px][t & 1]:1 + d[px][t & 1] + w]
                        for t in range(4)], 1)
        wp = wk[ph].view(co, 4 * ci, 1, 1)
        ref[:, :, py::2, px::2] = torch.nn.functional.conv2d(xs, wp, bias)
        mag[:, :, py::2, px::2] = torch.nn.functional.conv2d(xs.abs(), wp.abs(), bias.abs())
    return ref, mag


def act_f64(y, act):
    F = torch.nn.functional
    if act == cc.ACT_SILU:
        return F.silu(y)
    if act == cc.ACT_LEAKY:
        return F.leaky_relu(y, 0.1)
    if act == cc.ACT_RELU:
        return F.relu(y)
    if act == cc.ACT_SIGMOID:
        return torch.sigmoid(y)
    return y


def detect_decode_f64(y, mag, stride, anchors):
    """Detect decode (yolo.py:36-44) of the float64 head output y [n][3 * no][gh][gw] and its error bound terms.
    Returns (ref, M_out, ref_mag) laid out like the engine's rows [n][3 * gh * gw][no]: M_out is the magnitude M
    scaled by the decode's largest slope per column (sigmoid' <= 1/4; centres 2 s' stride <= stride / 2; sizes
    8 s s' anchor <= 32/27 anchor), ref_mag the magnitude of the decode's terms (centres subtract 0.5)."""
    n, c, gh, gw = y.shape
    no = c // 3
    s = torch.sigmoid(y).view(n, 3, no, gh, gw).permute(0, 1, 3, 4, 2)
    m = mag.view(n, 3, no, gh, gw).permute(0, 1, 3, 4, 2)
    gy, gx = torch.meshgrid(torch.arange(gh, device=y.device), torch.arange(gw, device=y.device), indexing="ij")
    grid = torch.stack((gx, gy), 2).double()
    anch = torch.as_tensor(np.asarray(anchors, np.float64), device=y.device).view(1, 3, 1, 1, 2)
    ref = s.clone()
    ref[..., 0:2] = (s[..., 0:2] * 2 - 0.5 + grid) * stride
    ref[..., 2:4] = (s[..., 2:4] * 2) ** 2 * anch
    slope = torch.full((no,), 0.25, dtype=torch.float64, device=y.device)
    slope[0:2] = 0.5 * stride
    mout = m * slope
    mout[..., 2:4] = m[..., 2:4] * (32.0 / 27.0) * anch
    rmag = ref.abs()
    rmag[..., 0:2] = (s[..., 0:2] * 2 + 0.5 + grid) * stride
    return ref.reshape(n, -1, no), mout.reshape(n, -1, no), rmag.reshape(n, -1, no)


def program_tc_plans(prog, n, h, w, split=False, num_sms=H100_SMS):
    """{op index: tc_plan} of every CONV / DECONV4 / DETECT op of a compiled program at batch shape n x h x w."""
    plans = {}
    for i, op in enumerate(prog.ops):
        if op["kind"] not in (cc.OP_CONV, cc.OP_DECONV4, cc.OP_DETECT):
            continue
        down = prog.bufs[op["src_buf"][0]][1]
        gh, gw = h // down, w // down
        if op["kind"] == cc.OP_DECONV4:
            plans[i] = tc_plan(op["cout"], gh, gw, n, 4, split, num_sms)
        else:
            plans[i] = tc_plan(op["cout"], gh // op["stride"], gw // op["stride"], n, 1, split, num_sms)
    return plans


# ---------------------------------------------------------------------------------------------------------------
# Kernel choice of sppf_pool_launch (csrc/simt.cu), replicated: the whole h x w plane of one 8-channel group, twice
# (ping-pong), must fit in 200 KB of shared memory for sppf_pool_tile_kernel; otherwise sppf_pool_kernel reads a
# 13 x 13 window per pixel from global memory.  h x w is the SPPF grid, the page at 1/32.
SPPF_SMEM_LIMIT = 200 * 1024


def sppf_uses_tile(h, w, elem_bytes):
    return 2 * h * w * 8 * elem_bytes <= SPPF_SMEM_LIMIT


# (precision, n, page h, page w, tile kernel?) of tests/test_gpu_thin_ops.py::test_sppf_both_kernels: each storage
# width at its exact tile limit and past it (tests/test_cpu_thin_ops_plan.py checks the sides without a GPU)
SPPF_SHAPES = [
    (PREC_SPLIT_TC, 1, 1024, 3200, True),       # 32 x 100 fp32: 204 800 B, the limit itself
    (PREC_FP32_SIMT, 2, 1856, 1856, False),     # 58 x 58 fp32, two images
    (PREC_SPLIT_TC, 1, 1024, 4096, False),      # 32 x 128 fp32
    (PREC_FP16_TC, 1, 2048, 3200, True),        # 64 x 100 fp16: 204 800 B
    (PREC_FP16_TC, 1, 2624, 2624, False),       # 82 x 82 fp16
]


def storage_bytes(prec):
    """bytes per stored activation: fp16 engines 2, fp32 and split-fp16 (fp32 master copy) 4."""
    return 2 if prec in (PREC_FP16_TC, PREC_FP16_SIMT) else 4
