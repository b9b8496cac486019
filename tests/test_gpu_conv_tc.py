"""-m gpu: conv_tc_kernel (csrc/conv_tc.cu) pinned exactly, at every launch plan it has, and at the plans the
benchmark runs.

* Routing: one-hot weights make every output exactly one input value (or 0 in the padding), so the result must be
  EQUAL to a numpy emulation of the epilogue (fp32 bias add, ReLU, fp32 residual add, fp16 / fp32 store).  A wrong
  tap, border, parity map, deconvolution phase, K-concatenation, channel offset, image offset, tile origin or
  epilogue column then fails with zero tolerance.  ROUTING_CASES covers every N-block width BN of both precisions,
  with full and partial 16x8 tiles (tests/test_cpu_conv_tc_plan.py checks the coverage without a GPU).
* Split magnitude probe: a 1x1 identity convolution in split-fp16 mode must keep 22 significant bits for operands
  from 2^-20 to 2^8.
* Benchmarked plans: every tensor-core op of the real program, re-run alone on the engine's own buffers at the
  benchmark's batch shapes, against a float64 reference under the elementwise bound of tests/util.py.
"""
import time

import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200 import compiler as cc
from oracle import synth
from util import (SingleOp, PREC_FP16_TC, PREC_SPLIT_TC, get_checkpoint, tc_plan, fp16_tc_ab, split_tc_ab,
                  bound_ratio, conv_ref_mag, deconv4_ref_mag, act_f64, detect_decode_f64, program_tc_plans, blob_tensor,
                  nchw_f64)

pytestmark = pytest.mark.gpu

DEV = "cuda"


# ---------------------------------------------------------------------------------------------------------------
# routing cases: (name, precision, source channels, kind, k, stride, cout, act, residual, down, n, h, w, dst)
#   kind "conv" | "deconv"; down = resolution divisor of the sources; dst = (buffer channels, channel offset) of a
#   destination slice inside a wider buffer, or None for a fresh buffer
ROUTING_CASES = [
    ("f16_1x1_many", PREC_FP16_TC, [128], "conv", 1, 1, 128, cc.ACT_RELU, False, 1, 2, 256, 512, None),
    ("f16_3x3_partial_x", PREC_FP16_TC, [64, 64], "conv", 3, 1, 128, cc.ACT_NONE, True, 8, 4, 512, 960, (136, 8)),
    ("f16_3x3_partial", PREC_FP16_TC, [64], "conv", 3, 1, 64, cc.ACT_RELU, False, 16, 2, 192, 320, None),
    ("f16_3x3_3src", PREC_FP16_TC, [64, 32, 16], "conv", 3, 1, 64, cc.ACT_NONE, False, 1, 1, 64, 128, None),
    ("f16_3x3s2", PREC_FP16_TC, [32], "conv", 3, 2, 32, cc.ACT_NONE, False, 1, 1, 128, 256, None),
    ("f16_deconv4_partial", PREC_FP16_TC, [64], "deconv", 4, 2, 32, cc.ACT_RELU, False, 16, 2, 192, 320, None),
    ("f16_1x1_cout21", PREC_FP16_TC, [64, 32], "conv", 1, 1, 21, cc.ACT_RELU, False, 16, 2, 192, 320, (40, 8)),
    ("f16_3x3_bn16", PREC_FP16_TC, [32], "conv", 3, 1, 16, cc.ACT_RELU, False, 1, 1, 64, 64, None),
    ("f16_deconv4_bn16_batch3", PREC_FP16_TC, [128], "deconv", 4, 2, 16, cc.ACT_NONE, False, 16, 3, 192, 320, None),
    ("f16_3x3s2_many", PREC_FP16_TC, [64], "conv", 3, 2, 128, cc.ACT_NONE, False, 1, 2, 512, 512, None),
    ("f16_3x3_res_2src", PREC_FP16_TC, [32, 64], "conv", 3, 1, 64, cc.ACT_RELU, True, 1, 1, 64, 64, (72, 8)),
    ("split_1x1_many", PREC_SPLIT_TC, [128], "conv", 1, 1, 128, cc.ACT_RELU, False, 1, 2, 256, 512, None),
    ("split_3x3_res_partial", PREC_SPLIT_TC, [64, 32], "conv", 3, 1, 64, cc.ACT_NONE, True, 16, 2, 192, 320, (72, 8)),
    ("split_3x3s2_partial", PREC_SPLIT_TC, [32], "conv", 3, 2, 32, cc.ACT_RELU, False, 8, 2, 256, 320, None),
    ("split_deconv4", PREC_SPLIT_TC, [64], "deconv", 4, 2, 32, cc.ACT_NONE, False, 2, 1, 64, 128, None),
    ("split_3x3_3src_bn16", PREC_SPLIT_TC, [16, 32, 64], "conv", 3, 1, 16, cc.ACT_RELU, False, 1, 1, 64, 64, None),
    ("split_deconv4_bn16_partial", PREC_SPLIT_TC, [32], "deconv", 4, 2, 16, cc.ACT_RELU, False, 16, 2, 192, 320,
     None),
    ("split_1x1_cout20", PREC_SPLIT_TC, [64], "conv", 1, 1, 20, cc.ACT_NONE, False, 16, 2, 192, 320, (32, 8)),
    ("split_3x3s2_many", PREC_SPLIT_TC, [64], "conv", 3, 2, 64, cc.ACT_NONE, False, 1, 2, 512, 512, None),
]


def case_plan(case):
    """conv_tc_kernel launch plan of a routing case (tests/util.py replica of conv_tc_plan)."""
    _, prec, _, kind, _, stride, cout, _, _, down, n, h, w, _ = case
    gh, gw = h // down, w // down
    if kind == "conv":
        gh, gw = gh // stride, gw // stride
    return tc_plan(cout, gh, gw, n, 4 if kind == "deconv" else 1, split=prec == PREC_SPLIT_TC)


def _case_id(case):
    p = case_plan(case)
    return "%s-bn%d%s" % (case[0], p["bn"], "-partial" if p["partial"] else "")


def _one_hot_weights(rng, kind, cin, cout, k):
    """Every output channel reads exactly one (input channel, tap); channels and taps vary with the output channel
    so that all sources, K blocks and taps are exercised.  conv: [co][ci][k][k]; deconv: [ci][co][4][4]."""
    perm = rng.permutation(max(cin, cout))
    if kind == "conv":
        w = np.zeros((cout, cin, k, k), np.float64)
        for co in range(cout):
            t = (co * 5 + 3) % (k * k)
            w[co, perm[co] % cin, t // k, t % k] = 1.0
    else:
        w = np.zeros((cin, cout, 4, 4), np.float64)
        for co in range(cout):
            t = (co * 7 + 1) % 16
            w[perm[co] % cin, co, t // 4, t % 4] = 1.0
    return w


@pytest.mark.parametrize("case", ROUTING_CASES, ids=_case_id)
def test_routing_exact(case):
    name, prec, srcc, kind, k, stride, cout, act, residual, down, n, h, w, dstspec = case
    rng = np.random.default_rng(sum(map(ord, name)))
    cin = sum(srcc)
    so = SingleOp(srcc, down=down, extra_channels=8)
    wgt = _one_hot_weights(rng, kind, cin, cout, k)
    bias = rng.integers(-12, 13, cout) / 8.0            # k/8: exact in fp16 and fp32
    dst = dst_init = None
    odown = down * stride if kind == "conv" else down // 2
    oh, ow = h // odown, w // odown
    if dstspec is not None:
        dch, dcoff = dstspec
        dst = so.P.tensor(so.P.newbuf(dch, odown), dcoff, cout)
        dst_init = rng.standard_normal((n, oh, ow, dch)).astype(np.float16).astype(np.float32)
    if kind == "conv":
        out_t = so.P.conv(so.srcs, wgt, bias, stride, act, dst=dst, residual=residual)
    else:
        out_t = so.P.deconv4(so.srcs, wgt, bias, act)
    # fp16 values (lo plane = 0 in split mode), with exact zeros and signed values
    ins = [rng.standard_normal((n, h // down, w // down, c)).astype(np.float16).astype(np.float32) for c in srcc]
    got = so.run(out_t, ins, n, h, w, prec, dst_init=dst_init, full_dst=True)

    x = torch.from_numpy(np.concatenate(ins, -1)).permute(0, 3, 1, 2).to(DEV, torch.float64)
    wt = torch.from_numpy(wgt).to(DEV)
    if kind == "conv":
        y = torch.nn.functional.conv2d(x, wt, None, stride, k // 2)
    else:
        y = torch.nn.functional.conv_transpose2d(x, wt, None, 2, 1)
    y = y.permute(0, 2, 3, 1).cpu().numpy()
    assert np.array_equal(y, y.astype(np.float16).astype(np.float64)), "one-hot reference is not a copy"
    # epilogue emulation: fp32(acc + bias) -> activation -> (+ fp32 residual) -> store
    v = y.astype(np.float32) + bias.astype(np.float32)
    if act == cc.ACT_RELU:
        v = np.maximum(v, np.float32(0))
    coff = dstspec[1] if dstspec else 0
    if residual:
        v = v + dst_init[..., coff:coff + cout]
    if prec == PREC_FP16_TC:
        v = v.astype(np.float16).astype(np.float32)
    if dst_init is not None:
        want = dst_init.copy()
        want[..., coff:coff + cout] = v
    else:
        want = v
    assert got.shape == want.shape, (got.shape, want.shape)
    diff = got != want
    print("%s: %d of %d elements differ, plan %s" % (name, int(diff.sum()), diff.size, case_plan(case)))
    if diff.any():
        idx = np.argwhere(diff)[:8]
        raise AssertionError("%d elements differ; first (n, y, x, c): %s got %s want %s"
                             % (int(diff.sum()), idx.tolist(), got[diff][:8].tolist(), want[diff][:8].tolist()))


# ---------------------------------------------------------------------------------------------------------------
def _octave_table(vals, rel):
    octs = np.floor(np.log2(np.abs(vals))).astype(int)
    return {int(o): float(rel[octs == o].max()) for o in np.unique(octs)}


def _log_uniform(rng, size, lo=-20, hi=8):
    return (np.exp2(rng.uniform(lo, hi, size)) * rng.choice([-1.0, 1.0], size)).astype(np.float32)


def test_split_magnitude_probe():
    """1x1 convolutions in split-fp16 mode: |got - x w| <= 2^-21 |x w| + 2^-35 per element, for activations from
    2^-20 to 2^8 (w = 1) and for weights from 2^-20 to 2^8 (x = 1)."""
    rng = np.random.default_rng(7)
    n, h, w, c = 1, 64, 128, 64
    results = {}
    # activation sweep: identity weights
    so = SingleOp([c], down=1)
    out_t = so.P.conv(so.srcs, np.eye(c).reshape(c, c, 1, 1), np.zeros(c), 1, cc.ACT_NONE)
    x = _log_uniform(rng, (n, h, w, c))
    got = so.run(out_t, [x], n, h, w, PREC_SPLIT_TC).astype(np.float64)
    ref = x.astype(np.float64)
    results["activation"] = (ref, got)
    # weight sweep: dense log-uniform weights, pixel p carries x = 1 on channel p % c only, so out[p, co] = W[co, p % c]
    so = SingleOp([c], down=1)
    wgt = _log_uniform(rng, (c, c)).astype(np.float64)
    out_t = so.P.conv(so.srcs, wgt.reshape(c, c, 1, 1), np.zeros(c), 1, cc.ACT_NONE)
    sel = np.arange(h * w) % c
    xo = np.zeros((n, h * w, c), np.float32)
    xo[0, np.arange(h * w), sel] = 1.0
    got = so.run(out_t, [xo.reshape(n, h, w, c)], n, h, w, PREC_SPLIT_TC).astype(np.float64).reshape(h * w, c)
    ref = wgt.T[sel]                                     # [pixel][co] = W[co][p % c]
    results["weight"] = (ref, got)
    bad = []
    for kind, (ref, got) in results.items():
        err = np.abs(got - ref)
        rel = err / np.abs(ref)
        tab = _octave_table(ref.ravel(), rel.ravel())
        print("split probe, %s sweep: max relative error per octave (log2):" % kind)
        print("  " + " ".join("2^%d:%.1f" % (o, np.log2(max(e, 2.0 ** -60))) for o, e in sorted(tab.items())))
        viol = err > 2.0 ** -21 * np.abs(ref) + 2.0 ** -35
        if viol.any():
            bad.append("%s sweep: %d elements above the bound, largest |x| %g"
                       % (kind, int(viol.sum()), float(np.abs(ref[viol]).max())))
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------------------
# benchmarked plans
BENCH_SHAPES = [(PREC_FP16_TC, 16, 1024, 1024), (PREC_FP16_TC, 8, 640, 640), (PREC_FP16_TC, 8, 1536, 1536),
                (PREC_SPLIT_TC, 1, 1024, 1024)]


def _slices_overlap(a, b):
    return a[0] == b[0] and a[1] < b[1] + b[2] and b[1] < a[1] + a[2]


def _check_images(n):
    """Images whose results are compared: the first and the last of the batch.  Their tiles open and close every
    persistent CTA's tile loop (the n-block index varies fastest, then the image), so a carried pipeline state or
    an image offset that goes wrong shows in them; the float64 reference of all 16 pages would take minutes."""
    return sorted({0, n - 1})


@pytest.mark.parametrize("prec,n,h,w", BENCH_SHAPES,
                         ids=["fp16_16x1024", "fp16_8x640", "fp16_8x1536", "split_1x1024"])
def test_bench_plans_per_op(prec, n, h, w):
    t0 = time.time()
    split = prec == PREC_SPLIT_TC
    ck = get_checkpoint(0, True)
    prog = cc.compile_checkpoint(ck)
    pages = np.stack([synth.structured_page(900 + i, h, w) for i in range(n)])
    plans = program_tc_plans(prog, n, h, w, split)
    eng = ctd_b200.Engine(prog, precision=prec, max_batch=n, max_h=h, max_w=w, skip_postproc=True)
    report = []
    try:
        eng.forward(pages)
        for i, op in enumerate(prog.ops):
            kind = op["kind"]
            gemm = kind in (cc.OP_CONV, cc.OP_DECONV4, cc.OP_DETECT)
            tc_tail = not split and kind in (cc.OP_STEM, cc.OP_SEG_TAIL)
            if not (gemm or tc_tail):      # CUDA-core ops: tests/test_gpu_thin_ops.py
                continue
            srcs = [(op["src_buf"][j], op["src_coff"][j], op["src_c"][j]) for j in range(op["n_src"])]
            dsl = (op["dst_buf"], op["dst_coff"], op["cout"]) if op["dst_buf"] >= 0 else None
            if dsl is not None and kind != cc.OP_STEM:
                assert not any(_slices_overlap(s, dsl) for s in srcs), "op %d reads the slice it writes" % i
            ins = [] if kind == cc.OP_STEM else [eng.debug_read(dict(buf=b, coff=o, c=c, down=prog.bufs[b][1]))
                                                 for b, o, c in srcs]
            dst_t = dict(buf=dsl[0], coff=dsl[1], c=dsl[2], down=prog.bufs[dsl[0]][1]) if dsl else None
            res_before = eng.debug_read(dst_t).copy() if op["residual"] else None
            eng.debug_run_ops(i, i, n, h, w, pages=pages if kind == cc.OP_STEM else None)
            if kind == cc.OP_DETECT:
                got_all = eng.net_outputs(want_mask=False, want_lines=False)[0]
            elif kind == cc.OP_SEG_TAIL:
                got_all = eng.net_outputs(want_blks=False, want_lines=False)[1]
            else:
                got_all = eng.debug_read(dst_t)
            worst, K = 0.0, None
            for img in _check_images(n):
                r, K = _op_ratio(prog, op, ins, res_before, got_all, pages, img, split)
                worst = max(worst, r)
            # the stem's plan is fixed at BN = 32 (conv_tc_plan_stem), the seg tail's at 16
            bn = plans[i]["bn"] if i in plans else (32 if kind == cc.OP_STEM else 16)
            report.append((worst, i, kind, K, bn))
            del ins, got_all, res_before
    finally:
        eng.close()
    report.sort(reverse=True)
    print("%s %dx%dx%d: %d tensor-core ops, %.0f s; worst err/bound (ratio, op, kind, K, predicted BN): %s"
          % ("split_tc" if split else "fp16_tc", n, h, w, len(report), time.time() - t0,
             [("%.3g" % r, i, k, K, bn) for r, i, k, K, bn in report[:6]]))
    print("  predicted BN histogram:", {bn: sum(1 for x in report if x[4] == bn) for bn in sorted({x[4] for x in report})})
    bad = [x for x in report if not x[0] <= 1.0]
    assert not bad, "ops above the bound: %s" % bad[:10]


def _op_ratio(prog, op, ins, res_before, got_all, pages, img, split):
    """(max err/bound over image `img` of op's output, K)."""
    n, h, w, _ = pages.shape
    kind = op["kind"]
    cin = sum(op["src_c"][:op["n_src"]])
    cout, cout_pad = op["cout"], op["cout_pad"]
    wdt = np.float32 if split else np.float16
    wsz = 4 if split else 2
    woff = op["w32_off"] if split else op["w16_off"]
    bias = blob_tensor(prog, op["b_off"], cout, np.float32)
    if kind == cc.OP_STEM:
        # tensor-core stem: fp16 space-to-depth page (channel (dy * 2 + dx) * 3 + c) and the fp16 window weights
        pg = (torch.from_numpy(pages[img]).to(DEV).permute(2, 0, 1).float() / 255).half().double()
        x = torch.zeros(1, 16, h // 2, w // 2, dtype=torch.float64, device=DEV)
        for dy in range(2):
            for dx in range(2):
                x[0, (dy * 2 + dx) * 3:(dy * 2 + dx) * 3 + 3] = pg[:, dy::2, dx::2]
        ww = blob_tensor(prog, op["w16_off"], 32 * 192, np.float16).double().view(32, 3, 4, 16)[:cout, :, :3]
        ref, mag = conv_ref_mag(x, ww.permute(0, 3, 1, 2), bias, 1, 1)
        K = 192
    elif kind == cc.OP_SEG_TAIL:
        c = op["src_c"][0]
        x = nchw_f64(ins[0], img)
        wc = blob_tensor(prog, op["w16_off"], 16 * 9 * c, np.float16).double().view(16, 3, 3, c)[:4].permute(0, 3, 1, 2)
        y, mag = conv_ref_mag(x, wc, torch.zeros(4, device=DEV), 1, 1)
        K = 9 * c
        nb, _, ih, iw = y.shape
        ref = torch.zeros(1, 2 * ih, 2 * iw, dtype=torch.float64, device=DEV)
        m2 = torch.zeros_like(ref)
        for p in range(4):
            ref[:, p >> 1::2, p & 1::2] = torch.sigmoid(y[:, p])
            m2[:, p >> 1::2, p & 1::2] = 0.25 * mag[:, p]
        # fp32 sigmoid with expf (2^-21: a few ulps) over the accumulation error times the sigmoid's slope (in m2)
        b = fp16_tc_ab(K)[1]
        got = torch.from_numpy(got_all[img].reshape(1, 2 * ih, 2 * iw)).to(DEV)
        return float(bound_ratio(got, ref, m2, 2.0 ** -21, b).max()), K
    else:
        x = torch.cat([nchw_f64(a, img) for a in ins], 1)
        if kind == cc.OP_DECONV4:
            K = 4 * cin
            wk = blob_tensor(prog, woff, 4 * cout_pad * K, wdt).view(4, cout_pad, K)[:, :cout]
            ref, mag = deconv4_ref_mag(x, wk, bias)
        else:
            ks, st = op["ksize"], op["stride"]
            K = ks * ks * cin
            wt = blob_tensor(prog, woff, cout_pad * K, wdt).view(cout_pad, ks, ks, cin)[:cout].permute(0, 3, 1, 2)
            ref, mag = conv_ref_mag(x, wt, bias, st, ks // 2)
    a, b = split_tc_ab(K) if split else fp16_tc_ab(K)
    if kind == cc.OP_DETECT:
        prm = blob_tensor(prog, op["p_off"], 7, np.float32).double().cpu().numpy()
        rf, mo, rmag = detect_decode_f64(ref, mag, float(prm[0]), prm[1:].reshape(3, 2))
        gh, gw = ref.shape[2], ref.shape[3]
        r0 = sum(3 * (h // (8 << l)) * (w // (8 << l)) for l in range(op["aux"]))
        got = torch.from_numpy(got_all[img, r0:r0 + 3 * gh * gw][None]).to(DEV)
        # fp32 decode: a few ulps of the decode's terms (2^-21); the head output's error scaled by the decode slope
        return float(bound_ratio(got, rf, mo, 2.0 ** -21, b, ref_mag=rmag).max()), K
    ref = act_f64(ref, op["act"])
    if res_before is not None:
        ref = ref + nchw_f64(res_before, img)
    got = nchw_f64(got_all, img)
    return float(bound_ratio(got, ref, mag, a, b).max()), K

