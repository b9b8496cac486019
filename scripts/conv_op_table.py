#!/usr/bin/env python
"""Per-op table of the wgmma convolutions (conv_tc_kernel; the stem and seg tail: csrc/conv_ends.cu) of the flagship
program at one batch shape.

    python scripts/conv_op_table.py [--batch 16 --size 1024] [--gpu] [--runs 5] [--json FILE]

One row per tensor-core op (stem, CONV, DECONV4, DETECT, seg tail) of the synthetic checkpoint's program: the launch
plan conv_tc_plan picks (N-block width BN, tile shape, tiles, tiles per persistent CTA), the algorithmic FLOPs, the
least HBM traffic (every input read once, the weights read once, the output written once) and the operand bytes TMA
moves from L2 into shared memory (A = activation boxes, B = weight boxes; in conv_tc_kernel every K block of every tap
of every tile loads one A box and one B box, in the stem and seg-tail kernels every tile loads one halo box and every
CTA the weights once).  The plan is computed here from the same rules as csrc/conv_tc.cu (132 SMs).

With --gpu, the program also runs on cuda:0: each op's device time is the minimum over --runs un-graphed forwards
(Engine.profile_forward, CUDA events around every op), and the row adds the achieved TFLOP/s, operand TB/s and HBM
TB/s (least HBM bytes over time).  The totals end with one line per op kind (1x1 CONV, 3x3 CONV, DECONV4, DETECT,
stem, seg tail), with ms, TFLOP/s and HBM TB/s under --gpu.  The card's name and power limit are printed with the
table.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from ctd_b200 import compiler as cc  # noqa: E402

SMS = 132
TILE_W = 16
KIND = {cc.OP_STEM: "stem", cc.OP_CONV: "conv", cc.OP_DECONV4: "deconv4", cc.OP_DETECT: "detect",
        cc.OP_SEG_TAIL: "seg_tail"}


def pick_block_n(cout_pad):
    if cout_pad >= 128 and cout_pad % 128 == 0:
        return 128
    if cout_pad % 64 == 0:
        return 64
    if cout_pad % 32 == 0:
        return 32
    return 16


def k_block(src_c):
    kb = 64
    for c in src_c:
        if c % 64 != 0 and kb > 32:
            kb = 32
        if c % 32 != 0:
            kb = 16
    return kb


def tc_plan(cout_pad, gh, gw, n, n_phase, nhwc_store, tile_h=None, sms=SMS):
    """conv_tc_plan: BN from the 16x8 tile count, then 16x16 tiles for NHWC-store (CONV / DECONV4) ops that keep at
    least one tile per SM.  tile_h forces a tile height (model of one tile shape for every op)."""
    tiles_x = -(-gw // TILE_W)
    sp8 = n * tiles_x * -(-gh // 8) * n_phase
    bn = pick_block_n(cout_pad)
    while bn > 64 and sp8 * (cout_pad // bn) <= sms // 2:
        bn //= 2
    th = 8
    if tile_h is not None:
        th = tile_h
    elif nhwc_store and n * tiles_x * -(-gh // 16) * n_phase * (cout_pad // bn) >= sms:
        th = 16
    tiles = n * tiles_x * -(-gh // th) * n_phase * (cout_pad // bn)
    grid = min(tiles, sms)
    return bn, th, tiles, -(-tiles // grid)


def op_rows(prog, n, h, w, tile_h=None):
    rows = []
    for i, o in enumerate(prog.ops):
        kind = o["kind"]
        if kind not in KIND:
            continue
        src_c = list(o["src_c"][:o["n_src"]])
        cin = sum(src_c)
        cout, cout_pad = o["cout"], o["cout_pad"]
        if kind == cc.OP_STEM:
            # stem_tc_kernel (csrc/conv_ends.cu): 16x16 output tiles, each loading one box of 36 page rows x 144
            # bytes of u8 (its space-to-depth rows and their halo); the 12 KB of window weights once per CTA
            gh, gw, res = h // 2, w // 2, h // 2
            k, stride = 6, 2
            bn, th = 32, 16
            tiles = n * -(-gw // TILE_W) * -(-gh // th)
            grid = min(tiles, SMS)
            tpc = -(-tiles // grid)
            flops = 2.0 * n * gh * gw * 108 * cout
            hbm = n * h * w * 3 + cout_pad * 192 * 2 + n * gh * gw * cout * 2
            a_bytes = float(tiles) * (2 * th + 4) * 144
            b_bytes = float(grid) * cout_pad * 192 * 2
        elif kind == cc.OP_SEG_TAIL:
            # seg_tc_kernel (csrc/conv_ends.cu): 16x16 tiles of the 64-channel input, each loading one (16+2)^2-pixel
            # halo box; 9 taps x the first 8 of the 16 (4 phases, zero-padded) weight rows once per CTA (m64n8 MMAs);
            # f32 + u8 mask at twice the resolution
            down = prog.bufs[o["src_buf"][0]][1]
            sh, sw = h // down, w // down
            k, stride, gh, gw, res = 4, 2, sh, sw, sh
            bn, th = 8, 16
            tiles = n * -(-gw // TILE_W) * -(-gh // th)
            grid = min(tiles, SMS)
            tpc = -(-tiles // grid)
            flops = 2.0 * n * sh * sw * 16 * cin
            hbm = n * sh * sw * cin * 2 + cout_pad * 9 * cin * 2 + n * 4 * sh * sw * (4 + 1)
            a_bytes = float(tiles) * (th + 2) * (TILE_W + 2) * cin * 2
            b_bytes = float(grid) * bn * 9 * cin * 2
        else:
            down = prog.bufs[o["src_buf"][0]][1]
            sh, sw = h // down, w // down
            kb = k_block(src_c)
            if kind == cc.OP_DECONV4:
                k, stride, taps, n_phase, gh, gw = 4, 2, 4, 4, sh, sw
            else:
                k, stride, n_phase = o["ksize"], o["stride"], 1
                taps, gh, gw = k * k, sh // stride, sw // stride
            res = sh
            bn, th, tiles, tpc = tc_plan(cout_pad, gh, gw, n, n_phase, kind != cc.OP_DETECT, tile_h)
            if kind == cc.OP_DECONV4:
                flops = 2.0 * n * sh * sw * 16 * cin * cout
                out_b = n * 4 * sh * sw * cout * 2
            else:
                flops = 2.0 * n * gh * gw * taps * cin * cout
                out_b = n * gh * gw * cout * (4 if kind == cc.OP_DETECT else 2) * (2 if o["residual"] else 1)
            hbm = n * sh * sw * cin * 2 + n_phase * cout_pad * taps * cin * 2 + out_b
            its = taps * (cin // kb)                              # K iterations of a tile
            a_bytes = float(tiles) * its * th * TILE_W * kb * 2
            b_bytes = float(tiles) * its * bn * kb * 2
        rows.append(dict(op=i, kind=KIND[kind], k=k, stride=stride, res=res, cin=cin, cout=cout, bn=bn,
                         tile="16x%d" % th, tiles=tiles, tiles_per_cta=tpc, gflop=flops / 1e9, hbm_gb=hbm / 1e9,
                         a_gb=a_bytes / 1e9, b_gb=b_bytes / 1e9))
    return rows


def gpu_times(prog, n, h, w, runs):
    import numpy as np
    import torch
    import ctd_b200
    from oracle import synth
    pages = np.stack([synth.structured_page(1000 + i, h, w) for i in range(n)])
    dev = torch.from_numpy(pages).cuda()
    eng = ctd_b200.Engine(prog, max_batch=n, max_h=h, max_w=w)
    try:
        eng.forward_device(dev.data_ptr(), n, h, w)
        best = None
        for _ in range(runs):
            ms = eng.profile_forward(dev_ptr=dev.data_ptr(), shape=(n, h, w))[0]
            best = ms if best is None else np.minimum(best, ms)
    finally:
        eng.close()
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return [float(v) for v in best], q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=1024, help="square page size")
    ap.add_argument("--tile-h", type=int, choices=(8, 16), default=None,
                    help="model every CONV / DECONV4 / DETECT op at this tile height (CPU model only)")
    ap.add_argument("--gpu", action="store_true", help="add per-op device times measured on cuda:0")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the rows to this file")
    args = ap.parse_args()
    if args.gpu and args.tile_h is not None:
        ap.error("--tile-h models another plan; the GPU runs the plan of the build")
    from oracle import synth
    prog = cc.compile_checkpoint(synth.make_checkpoint(0, smooth=True))
    n, h, w = args.batch, args.size, args.size
    rows = op_rows(prog, n, h, w, args.tile_h)
    card = None
    if args.gpu:
        ms, card = gpu_times(prog, n, h, w, args.runs)
        for r in rows:
            r["ms"] = ms[r["op"]]
            r["tflops"] = r["gflop"] / r["ms"] if r["ms"] > 0 else 0.0
            r["operand_tbs"] = (r["a_gb"] + r["b_gb"]) / r["ms"] if r["ms"] > 0 else 0.0
            r["hbm_tbs"] = r["hbm_gb"] / r["ms"] if r["ms"] > 0 else 0.0
    print("conv_tc ops at %d x %d x %d fp16%s" % (n, h, w, ("; " + card) if card else " (CPU model, not measured)"))
    hdr = "%4s %-8s %2s %2s %5s %9s %4s %6s %6s %7s %10s %8s %6s %6s" % (
        "op", "kind", "k", "s", "res", "cin/cout", "BN", "tile", "tiles", "t/CTA", "GFLOP", "HBM GB", "A GB", "B GB")
    if args.gpu:
        hdr += " %7s %7s %7s %7s" % ("ms", "TFLOP/s", "opTB/s", "HBMTB/s")
    print(hdr)
    for r in rows:
        line = "%4d %-8s %2d %2d %5d %9s %4d %6s %6d %7d %10.2f %8.3f %6.2f %6.2f" % (
            r["op"], r["kind"], r["k"], r["stride"], r["res"], "%d/%d" % (r["cin"], r["cout"]), r["bn"], r["tile"],
            r["tiles"], r["tiles_per_cta"], r["gflop"], r["hbm_gb"], r["a_gb"], r["b_gb"])
        if args.gpu:
            line += " %7.3f %7.1f %7.2f %7.2f" % (r["ms"], r["tflops"], r["operand_tbs"], r["hbm_tbs"])
        print(line)
    gemm = [r for r in rows if r["kind"] in ("conv", "deconv4", "detect")]
    for name, sel in (("CONV/DECONV4/DETECT (%d ops)" % len(gemm), gemm), ("all %d tensor-core ops" % len(rows), rows)):
        t = {k: sum(r[k] for r in sel) for k in ("gflop", "hbm_gb", "a_gb", "b_gb")}
        line = "total %s: %.3f TFLOP, HBM %.2f GB, operands A %.2f + B %.2f = %.2f GB" % (
            name, t["gflop"] / 1e3, t["hbm_gb"], t["a_gb"], t["b_gb"], t["a_gb"] + t["b_gb"])
        if args.gpu:
            ms = sum(r["ms"] for r in sel)
            line += "; %.3f ms, %.1f TFLOP/s, operands %.2f TB/s" % (ms, t["gflop"] / ms, (t["a_gb"] + t["b_gb"]) / ms)
        print(line)
    groups = (("1x1 CONV", lambda r: r["kind"] == "conv" and r["k"] == 1),
              ("3x3 CONV", lambda r: r["kind"] == "conv" and r["k"] == 3),
              ("DECONV4", lambda r: r["kind"] == "deconv4"), ("DETECT", lambda r: r["kind"] == "detect"),
              ("stem", lambda r: r["kind"] == "stem"), ("seg tail", lambda r: r["kind"] == "seg_tail"))
    for name, pick in groups:
        sel = [r for r in rows if pick(r)]
        if not sel:
            continue
        t = {k: sum(r[k] for r in sel) for k in ("gflop", "hbm_gb", "a_gb", "b_gb")}
        line = "  %-8s %3d ops: %.3f TFLOP, HBM %.2f GB, operands %.2f GB" % (
            name, len(sel), t["gflop"] / 1e3, t["hbm_gb"], t["a_gb"] + t["b_gb"])
        if args.gpu:
            # HBM TB/s: least HBM bytes over device time
            ms = sum(r["ms"] for r in sel)
            line += "; %.3f ms, %.1f TFLOP/s, HBM %.2f TB/s" % (ms, t["gflop"] / ms, t["hbm_gb"] / ms)
        print(line)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"shape": [n, h, w], "card": card, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
