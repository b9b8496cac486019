"""-m gpu: every op the engine runs on CUDA cores (csrc/simt.cu), alone, at the benchmarked shapes, on every image of
the batch, against a reference computed here from the op's own inputs and the compiled program's blob.

Procedure, as in tests/test_gpu_conv_tc.py::test_bench_plans_per_op: `eng.forward(pages)`, then for each op read its
inputs, run only that op (`ctd_debug_run_ops`) and read what it wrote.  Criteria per op:

* UPSAMPLE2: the nearest copy, bit for bit.
* SPPF pools: slots [c,2c), [2c,3c), [3c,4c) equal float64 max_pool2d of slot 0 with k = 5 / 9 / 13, stride 1 and
  -inf padding, bit for bit; slot 0 is unchanged.
* AVGPOOL2: bit for bit the kernel's order in float32, (((tl + tr) + bl) + br) * 0.25 rounded to the storage type; and
  within one output rounding plus the three fp32 adds of float64: a |ref| + t + 3 * 2^-24 * mean(|x|), with a = 2^-24
  for fp32 and 2^-11 for fp16, and t = 2^-25 for fp16 (half its subnormal spacing), 0 for fp32.
* DB_TAIL: float64 ConvT 2x2 s2 -> +b3 -> ReLU -> ConvT 2x2 s2 -> +b6 -> sigmoid for both branches, from the op's fp32
  parameters (layout at db_tail_kernel).  Per output the kernel runs an fp32 FMA chain of 17 terms (b3 and 16 FMAs)
  for each of the 16 hidden channels, then one of 17 terms (b6 and 16 FMAs) over them.  Every FMA rounds once
  (2^-24): the first chains err by 16 * 2^-24 * M1, M1 = |b3| + sum |x| |w3|, carried through |w6|; the second by
  16 * 2^-24 * M2 with M2 <= M = |b6| + sum |w6| M1.  So the pre-sigmoid error is at most 32 * 2^-24 * M; the
  sigmoid's slope is at most 1/4, and its own error (expf within 2 ulps, the add and the division) is under 2^-21
  relative.  The bound is

      |lines - ref| <= 2^-21 |ref| + 0.25 * 34 * 2^-24 * M          (34 for 32: a 1.06x margin)

  The DB bitmap must be the engine's own lines[:, 0] > float32(0.3) at every pixel, exactly, and may differ from the
  float64 shrink map's only where |ref - 0.3| is within that bound.
* STEM on CUDA cores: float64 conv 6x6 s2 p2 of float32(u8) / 255 with the fp32 weights under simt_ab(108)
  (tests/util.py: one fp32 FMA chain of K terms).
* SEG_TAIL on CUDA cores: float64 ConvT 4x4 s2 p1 + sigmoid.  The kernel forms 16 tap partials per input pixel in FMA
  chains of C terms and adds 4 of them per output in 3 fp32 adds: (C + 3) * 2^-24 * M before the sigmoid (slope
  <= 1/4, so 0.25 M), 2^-21 relative after it.  mask_u8 equals trunc(mask * 255.0f) exactly.
* CONV / DECONV4 / DETECT on CUDA cores (conv_simt_kernel, in CTD_PREC_FP32_SIMT and CTD_PREC_FP16_SIMT): float64 of
  the op's packed weights under simt_ab(K); Detect rows through the decode as in test_bench_plans_per_op.

The weights are the rough synthetic checkpoint's.  The smooth one (the benchmark's) makes every ConvT 2x2 constant
over its taps and every ConvT 4x4 a symmetric bilinear kernel, so a transposed or swapped sub-pixel phase in the DB
tail, the seg tail or a deconvolution computes the same values there.

test_sppf_both_kernels runs the SPPF op of the real program alone on both sides of sppf_pool_launch's shared-memory
limit (sppf_pool_tile_kernel and sppf_pool_kernel), on the forward's own activations and on a crafted slot 0, with slots
1-3 filled with a sentinel first so that an element left unwritten fails.
"""
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import ctd_b200
from ctd_b200 import compiler as cc
from oracle import synth
from util import (PREC_FP16_TC, PREC_SPLIT_TC, PREC_FP32_SIMT, PREC_FP16_SIMT, get_checkpoint, simt_ab, bound_ratio,
                  conv_ref_mag, deconv4_ref_mag, act_f64, detect_decode_f64, blob_tensor, nchw_f64, storage_bytes,
                  sppf_uses_tile, SPPF_SHAPES)

pytestmark = pytest.mark.gpu

DEV = "cuda"
GEMM = (cc.OP_CONV, cc.OP_DECONV4, cc.OP_DETECT)
DB_THRESH = np.float32(0.3)     # the engine's db_thresh, a float32
SIGMOID_A = 2.0 ** -21          # expf (2 ulps), the add and the division of 1 / (1 + e), relative to the result
KIND_NAME = {cc.OP_STEM: "stem", cc.OP_CONV: "conv", cc.OP_DECONV4: "deconv4", cc.OP_AVGPOOL2: "avgpool2",
             cc.OP_SPPF_POOL: "sppf", cc.OP_UPSAMPLE2: "upsample2", cc.OP_DETECT: "detect",
             cc.OP_SEG_TAIL: "seg_tail", cc.OP_DB_TAIL: "db_tail"}


def _on_tensor_cores(prec, kind):
    """runs_on_tensor_cores (csrc/engine.cu): every other op runs a csrc/simt.cu kernel."""
    if prec == PREC_SPLIT_TC:
        return kind in GEMM
    if prec == PREC_FP16_TC:
        return kind in GEMM or kind in (cc.OP_STEM, cc.OP_SEG_TAIL)
    return False


def _t(prog, buf, coff, c):
    return dict(buf=buf, coff=coff, c=c, down=prog.bufs[buf][1])


PER_OP_SHAPES = [(PREC_FP16_TC, 16, 1024, 1024), (PREC_FP16_TC, 8, 640, 640), (PREC_FP16_TC, 8, 1536, 1536),
                 (PREC_SPLIT_TC, 1, 1024, 1024), (PREC_FP32_SIMT, 1, 1024, 1024), (PREC_FP16_SIMT, 2, 256, 320)]


@pytest.mark.parametrize("prec,n,h,w", PER_OP_SHAPES,
                         ids=["fp16_tc_16x1024", "fp16_tc_8x640", "fp16_tc_8x1536", "split_tc_1x1024",
                              "fp32_simt_1x1024", "fp16_simt_2x256x320"])
def test_cuda_core_ops_per_op(prec, n, h, w):
    t0 = time.time()
    prog = cc.compile_checkpoint(get_checkpoint(0, smooth=False))
    pages = np.stack([synth.structured_page(900 + i, h, w) for i in range(n)])
    fp16 = storage_bytes(prec) == 2
    eng = ctd_b200.Engine(prog, precision=prec, max_batch=n, max_h=h, max_w=w, skip_postproc=True)
    report = []     # (worst err/bound or None for an exact-only op, op, kind, K or note, elements that differ)
    try:
        eng.forward(pages)
        for i, op in enumerate(prog.ops):
            kind = op["kind"]
            if _on_tensor_cores(prec, kind):
                continue
            fn = {cc.OP_SPPF_POOL: _check_sppf, cc.OP_UPSAMPLE2: _check_upsample2, cc.OP_AVGPOOL2: _check_avgpool2,
                  cc.OP_DB_TAIL: _check_db_tail, cc.OP_SEG_TAIL: _check_seg_tail, cc.OP_STEM: _check_gemm}.get(
                      kind, _check_gemm)
            ratio, note, differ = fn(eng, prog, i, op, pages, fp16)
            report.append((ratio, i, KIND_NAME[kind], note, differ))
    finally:
        eng.close()
    print("%s %dx%dx%d: %d CUDA-core ops, %.0f s; worst err/bound per op (ratio, op, kind, K, elements that differ "
          "where exact):" % (_prec_name(prec), n, h, w, len(report), time.time() - t0))
    for r, i, k, note, d in sorted(report, key=lambda x: -1.0 if x[0] is None else x[0], reverse=True):
        print("  %s op %d %s %s%s" % ("exact" if r is None else "%.3g" % r, i, k, note, " differ %d" % d if d else ""))
    bad = [x for x in report if x[4] or (x[0] is not None and not x[0] <= 1.0)]
    assert not bad, "ops above the bound or not exact: %s" % bad[:10]


def _prec_name(prec):
    return {PREC_FP16_TC: "fp16_tc", PREC_SPLIT_TC: "split_tc", PREC_FP32_SIMT: "fp32_simt",
            PREC_FP16_SIMT: "fp16_simt"}[prec]


# ---------------------------------------------------------------------------------------------------------------
def _sppf_ref_differ(slot0, after, c):
    """elements of `after` (slots 0-3, [n][h][w][4c]) that differ from slot 0 unchanged and its float64 5 / 9 / 13
    max pools with -inf padding."""
    differ = int((after[..., :c] != slot0).sum())
    for img in range(slot0.shape[0]):
        x = nchw_f64(slot0, img)
        for slot, k in ((1, 5), (2, 9), (3, 13)):
            ref = F.max_pool2d(x, k, 1, k // 2)
            differ += int((nchw_f64(after[..., slot * c:(slot + 1) * c], img) != ref).sum())
    return differ


def _check_sppf(eng, prog, i, op, pages, fp16):
    n, h, w, _ = pages.shape
    b, o, c = op["src_buf"][0], op["src_coff"][0], op["src_c"][0]
    slot0 = eng.debug_read(_t(prog, b, o, c)).copy()
    eng.debug_run_ops(i, i, n, h, w)
    return None, "k5/9/13", _sppf_ref_differ(slot0, eng.debug_read(_t(prog, b, o, 4 * c)), c)


def _check_upsample2(eng, prog, i, op, pages, fp16):
    n, h, w, _ = pages.shape
    x = eng.debug_read(_t(prog, op["src_buf"][0], op["src_coff"][0], op["src_c"][0])).copy()
    eng.debug_run_ops(i, i, n, h, w)
    got = eng.debug_read(_t(prog, op["dst_buf"], op["dst_coff"], op["src_c"][0]))
    want = np.repeat(np.repeat(x, 2, axis=1), 2, axis=2)
    return None, "nearest", int((got != want).sum())


def _check_avgpool2(eng, prog, i, op, pages, fp16):
    n, h, w, _ = pages.shape
    x = eng.debug_read(_t(prog, op["src_buf"][0], op["src_coff"][0], op["src_c"][0])).copy()
    eng.debug_run_ops(i, i, n, h, w)
    got = eng.debug_read(_t(prog, op["dst_buf"], op["dst_coff"], op["src_c"][0]))
    tl, tr, bl, br = x[:, 0::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 0::2], x[:, 1::2, 1::2]
    want = (((tl + tr) + bl) + br) * np.float32(0.25)
    assert want.dtype == np.float32
    if fp16:
        want = want.astype(np.float16).astype(np.float32)
    x64 = x.astype(np.float64)
    ref = (x64[:, 0::2, 0::2] + x64[:, 0::2, 1::2] + x64[:, 1::2, 0::2] + x64[:, 1::2, 1::2]) / 4
    mag = (np.abs(x64[:, 0::2, 0::2]) + np.abs(x64[:, 0::2, 1::2]) + np.abs(x64[:, 1::2, 0::2])
           + np.abs(x64[:, 1::2, 1::2])) / 4
    # one output rounding: half an ulp, relative for normal values, 2^-25 absolute in fp16's subnormal range
    a, tiny = (2.0 ** -11, 2.0 ** -25) if fp16 else (2.0 ** -24, 0.0)
    ratio = float((np.abs(got - ref) / (a * np.abs(ref) + tiny + 3 * 2.0 ** -24 * mag + 1e-300)).max())
    return ratio, "2x2", int((got != want).sum())


def _check_db_tail(eng, prog, i, op, pages, fp16):
    n, h, w, _ = pages.shape
    x_all = eng.debug_read(_t(prog, op["src_buf"][0], op["src_coff"][0], op["src_c"][0])).copy()
    eng.debug_run_ops(i, i, n, h, w)
    lines = eng.net_outputs(want_blks=False, want_mask=False)[2]
    bitmap = eng.db_components(want_bitmap=True, want_labels=False)[0]
    # the bitmap is the engine's own shrink map against the float32 threshold, at every pixel
    differ = int((bitmap != (lines[:, 0] > DB_THRESH)).sum())
    prm = blob_tensor(prog, op["p_off"], 2 * 1105, np.float32).double()
    thr = float(DB_THRESH)
    worst = 0.0
    for img in range(n):
        x = nchw_f64(x_all, img)
        for br in range(2):
            p = prm[br * 1105:(br + 1) * 1105]
            w3, b3 = p[:1024].view(16, 16, 2, 2), p[1024:1040]
            w6, b6 = p[1040:1104].view(16, 1, 2, 2), p[1104:1105]
            xb = x[:, 16 * br:16 * br + 16]
            ref = torch.sigmoid(F.conv_transpose2d(F.relu(F.conv_transpose2d(xb, w3, b3, 2)), w6, b6, 2))
            m1 = F.conv_transpose2d(xb.abs(), w3.abs(), b3.abs(), 2)
            mag = F.conv_transpose2d(m1, w6.abs(), b6.abs(), 2)
            got = torch.from_numpy(lines[img, br][None, None]).to(DEV)
            bound = SIGMOID_A * ref.abs() + 0.25 * 34 * 2.0 ** -24 * mag
            worst = max(worst, float(((got.double() - ref).abs() / bound).max()))
            if br == 0:
                # against the float64 shrink map, only pixels within the bound of the threshold may flip
                bm = torch.from_numpy(bitmap[img][None, None]).to(DEV) != 0
                flip = bm != (ref > thr)
                differ += int((flip & ((ref - thr).abs() > bound)).sum())
    return worst, "K=17+17", differ


def _check_seg_tail(eng, prog, i, op, pages, fp16):
    n, h, w, _ = pages.shape
    c = op["src_c"][0]
    x_all = eng.debug_read(_t(prog, op["src_buf"][0], op["src_coff"][0], c)).copy()
    eng.debug_run_ops(i, i, n, h, w)
    mask = eng.net_outputs(want_blks=False, want_lines=False)[1]
    m8 = eng.mask_u8()
    differ = int((m8 != (mask[:, 0] * np.float32(255)).astype(np.uint8)).sum())
    wt = blob_tensor(prog, op["p_off"], c * 16, np.float32).double().view(c, 1, 4, 4)
    worst = 0.0
    for img in range(n):
        x = nchw_f64(x_all, img)
        ref = torch.sigmoid(F.conv_transpose2d(x, wt, None, 2, 1))
        mag = F.conv_transpose2d(x.abs(), wt.abs(), None, 2, 1)
        got = torch.from_numpy(mask[img][None]).to(DEV)
        worst = max(worst, float(bound_ratio(got, ref, 0.25 * mag, SIGMOID_A, (c + 3) * 2.0 ** -24).max()))
    return worst, "K=%d+3" % c, differ


def _check_gemm(eng, prog, i, op, pages, fp16):
    """conv_simt_kernel (CONV / DECONV4 / DETECT) and stem_kernel against float64 under simt_ab(K)."""
    n, h, w, _ = pages.shape
    kind = op["kind"]
    srcs = [(op["src_buf"][j], op["src_coff"][j], op["src_c"][j]) for j in range(op["n_src"])]
    ins = [] if kind == cc.OP_STEM else [eng.debug_read(_t(prog, *s)).copy() for s in srcs]
    dst_t = _t(prog, op["dst_buf"], op["dst_coff"], op["cout"]) if op["dst_buf"] >= 0 else None
    res_before = eng.debug_read(dst_t).copy() if op["residual"] else None
    eng.debug_run_ops(i, i, n, h, w, pages=pages if kind == cc.OP_STEM else None)
    got_all = eng.net_outputs(want_mask=False, want_lines=False)[0] if kind == cc.OP_DETECT else eng.debug_read(dst_t)
    cout, cout_pad = op["cout"], op["cout_pad"]
    # the weights the kernel reads: fp16 engines the fp16 copy, fp32 engines the fp32 one; the stem always fp32
    wdt, woff = (np.float16, op["w16_off"]) if fp16 and kind != cc.OP_STEM else (np.float32, op["w32_off"])
    bias = blob_tensor(prog, op["b_off"], cout, np.float32)
    worst = 0.0
    for img in range(n):
        if kind == cc.OP_STEM:
            x32 = pages[img].astype(np.float32) / np.float32(255)      # the kernel's float(u8) / 255.0f
            x = torch.from_numpy(np.ascontiguousarray(x32.transpose(2, 0, 1))[None]).to(DEV).double()
            wt = blob_tensor(prog, woff, cout * 108, wdt).view(cout, 6, 6, 3).permute(0, 3, 1, 2)
            K = 108
            ref, mag = conv_ref_mag(x, wt, bias, 2, 2)
        else:
            x = torch.cat([nchw_f64(a, img) for a in ins], 1)
            cin = x.shape[1]
            if kind == cc.OP_DECONV4:
                K = 4 * cin
                wk = blob_tensor(prog, woff, 4 * cout_pad * K, wdt).view(4, cout_pad, K)[:, :cout]
                ref, mag = deconv4_ref_mag(x, wk, bias)
            else:
                ks, st = op["ksize"], op["stride"]
                K = ks * ks * cin
                wt = blob_tensor(prog, woff, cout_pad * K, wdt).view(cout_pad, ks, ks, cin)[:cout].permute(0, 3, 1, 2)
                ref, mag = conv_ref_mag(x, wt, bias, st, ks // 2)
        a, b = simt_ab(K, fp16_out=fp16)
        if kind == cc.OP_DETECT:
            prm = blob_tensor(prog, op["p_off"], 7, np.float32).double().cpu().numpy()
            rf, mo, rmag = detect_decode_f64(ref, mag, float(prm[0]), prm[1:].reshape(3, 2))
            gh, gw = ref.shape[2], ref.shape[3]
            r0 = sum(3 * (h // (8 << l)) * (w // (8 << l)) for l in range(op["aux"]))
            got = torch.from_numpy(got_all[img, r0:r0 + 3 * gh * gw][None]).to(DEV)
            # fp32 rows: the decode's own roundings and the sigmoid (SIGMOID_A), the head output's error scaled by the
            # decode slope (in mo)
            r = float(bound_ratio(got, rf, mo, SIGMOID_A, b, ref_mag=rmag).max())
        else:
            ref = act_f64(ref, op["act"])
            if res_before is not None:
                ref = ref + nchw_f64(res_before, img)
            r = float(bound_ratio(nchw_f64(got_all, img), ref, mag, a, b).max())
        worst = max(worst, r)
    return worst, "K=%d" % K, 0


# ---------------------------------------------------------------------------------------------------------------
SENTINEL = 4096.0       # exact in fp16 and above every value slot 0 holds


def _crafted_slot0(n, gh, gw, c):
    """All values negative (so a 0 in place of the -inf padding shows at every border), drawn from 8 levels (exact
    ties everywhere), and a unique maximum at each corner and edge midpoint, different per image and channel.  All
    values are exact in fp16."""
    rng = np.random.default_rng(gh * 1000 + gw)
    x = -(1.0 + rng.integers(0, 8, (n, gh, gw, c)) / 4.0)
    spots = [(0, 0), (0, gw - 1), (gh - 1, 0), (gh - 1, gw - 1), (0, gw // 2), (gh - 1, gw // 2), (gh // 2, 0),
             (gh // 2, gw - 1)]
    ch = np.arange(c)
    for img in range(n):
        for k, (y, xx) in enumerate(spots):
            x[img, y, xx] = -(1 + k + 8 * img + 16 * (ch % 4)) / 256.0
    return x.astype(np.float32)


@pytest.mark.parametrize("prec,n,h,w,tile", SPPF_SHAPES,
                         ids=["%s_%dx%dx%d_%s" % ("f16" if storage_bytes(p) == 2 else "f32", n, h, w,
                                                  "tile" if t else "fallback") for p, n, h, w, t in SPPF_SHAPES])
def test_sppf_both_kernels(prec, n, h, w, tile):
    t0 = time.time()
    prog = cc.compile_checkpoint(get_checkpoint(0, smooth=False))
    (i, op), = [(i, op) for i, op in enumerate(prog.ops) if op["kind"] == cc.OP_SPPF_POOL]
    b, o, c = op["src_buf"][0], op["src_coff"][0], op["src_c"][0]
    ch, down = prog.bufs[b]
    gh, gw = h // down, w // down
    assert sppf_uses_tile(gh, gw, storage_bytes(prec)) == tile
    whole = _t(prog, b, 0, ch)
    pages = np.stack([synth.structured_page(700 + k, h, w) for k in range(n)])
    eng = ctd_b200.Engine(prog, precision=prec, max_batch=n, max_h=h, max_w=w, skip_postproc=True)
    results = {}
    try:
        eng.forward(pages)
        inputs = {"forward": eng.debug_read(whole).copy(), "crafted": None}
        inputs["crafted"] = inputs["forward"].copy()
        inputs["crafted"][..., o:o + c] = _crafted_slot0(n, gh, gw, c)
        for name, buf in inputs.items():
            buf[..., o + c:o + 4 * c] = SENTINEL
            eng.debug_write(whole, buf, n, h, w)
            eng.debug_run_ops(i, i, n, h, w)
            after = eng.debug_read(_t(prog, b, o, 4 * c))
            results[name] = _sppf_ref_differ(buf[..., o:o + c], after, c)
    finally:
        eng.close()
    print("sppf %s %dx%dx%d (grid %dx%d, %s kernel): elements that differ %s, %.0f s"
          % (_prec_name(prec), n, h, w, gh, gw, "tile" if tile else "fallback", results, time.time() - t0))
    assert not any(results.values()), results
