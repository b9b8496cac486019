"""-m gpu: the convolution kernels (conv_tc_kernel and conv_simt_kernel, in all four precisions) on one-op convolution
and 4x4-deconvolution programs against a plain torch reference of the same op (fp16-rounded operands for the fp16
engines, so only accumulation order and the output rounding differ).  The tensor-core engines (fp16 and split-fp16)
are also held to the elementwise bound of tests/util.py, so a wrong value at a small output fails as well as one at
the largest.  The other CUDA-core kernels (stem, pools, upsample, seg and DB tails) are pinned per op in
tests/test_gpu_thin_ops.py."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from util import (SingleOp, h16, cc, PREC_FP16_TC, PREC_FP32_SIMT, PREC_FP16_SIMT, PREC_SPLIT_TC, fp16_tc_ab,
                  split_tc_ab, bound_ratio)

pytestmark = pytest.mark.gpu

ACTS = {cc.ACT_NONE: lambda x: x, cc.ACT_SILU: F.silu, cc.ACT_LEAKY: lambda x: F.leaky_relu(x, 0.1), cc.ACT_RELU: F.relu}


def _rand(rng, *shape, scale=1.0):
    return (rng.standard_normal(shape) * scale).astype(np.float32)


def _tol(prec, ref):
    m = float(np.abs(ref).max()) + 1e-6
    return (2e-5 if prec == PREC_FP32_SIMT else 2.5e-3) * m


CONV_CASES = [
    # (src channels, cout, k, stride, act, residual, h, w, n)
    ([64], 64, 1, 1, cc.ACT_SILU, False, 64, 64, 1),
    ([128], 128, 1, 1, cc.ACT_LEAKY, False, 64, 64, 2),
    ([256], 256, 1, 1, cc.ACT_NONE, False, 64, 64, 1),
    ([512], 512, 1, 1, cc.ACT_SILU, False, 64, 64, 1),
    ([64], 64, 3, 1, cc.ACT_SILU, True, 64, 64, 1),
    ([128], 128, 3, 1, cc.ACT_LEAKY, False, 64, 128, 1),
    ([64], 128, 3, 2, cc.ACT_SILU, False, 128, 128, 1),
    ([256], 512, 3, 2, cc.ACT_SILU, False, 64, 64, 2),
    ([32], 32, 1, 1, cc.ACT_SILU, False, 64, 64, 1),
    ([32], 32, 3, 1, cc.ACT_SILU, True, 64, 64, 1),
    ([32], 64, 3, 2, cc.ACT_SILU, False, 128, 128, 1),
    ([256, 512], 256, 1, 1, cc.ACT_LEAKY, False, 64, 64, 1),
    ([64, 128], 128, 1, 1, cc.ACT_LEAKY, False, 64, 64, 1),
    ([64], 32, 3, 1, cc.ACT_RELU, False, 64, 64, 1),
    ([64], 16, 3, 1, cc.ACT_RELU, False, 64, 64, 1),
    ([128], 64, 1, 1, cc.ACT_RELU, False, 192, 64, 1),
    ([16], 32, 3, 1, cc.ACT_SILU, False, 64, 128, 2),   # 16-channel K blocks (32-byte swizzle): the s2d stem
    ([16], 16, 1, 1, cc.ACT_NONE, False, 64, 64, 1),
    ([64, 64], 64, 3, 1, cc.ACT_LEAKY, False, 64, 128, 2),   # two sources, 64-channel K blocks
    ([32, 64], 64, 3, 1, cc.ACT_RELU, True, 128, 64, 1),     # 32-channel K blocks (64-byte swizzle)
    ([128], 32, 3, 1, cc.ACT_SILU, False, 64, 192, 1),
    ([256], 256, 3, 1, cc.ACT_LEAKY, True, 64, 64, 1),       # two 128-wide N blocks, residual
    ([128], 128, 3, 1, cc.ACT_SILU, True, 64, 64, 2),        # BN = 128 with residual
    ([64, 64], 128, 3, 1, cc.ACT_RELU, False, 128, 64, 1),   # two sources
    ([128, 64], 128, 1, 1, cc.ACT_SILU, False, 64, 192, 1),  # 1x1 over two sources
    ([128, 128], 512, 3, 1, cc.ACT_SILU, False, 64, 128, 1),  # two sources x four N blocks
    # (..., down): sources at 1/down resolution of the page
    ([64], 64, 3, 1, cc.ACT_SILU, True, 192, 320, 2, 16),      # 12x20 grid: partial tiles in x and y, batch 2
    ([128, 64], 128, 3, 2, cc.ACT_LEAKY, False, 512, 960, 2, 8),  # 32x60 grid: partial in x
    ([32], 96, 3, 1, cc.ACT_RELU, False, 192, 320, 3, 16),     # BN 32 x 3 N blocks, partial tiles, batch 3
    ([64], 128, 1, 1, cc.ACT_SILU, False, 512, 512, 2, 1),     # 4096 tiles: ~31 per persistent CTA
]


def _check_bound(prec, got, x, wgt, bias, ref, K, transposed=False, stride=1, pad=1):
    """Elementwise bound of the tensor-core engines; M = |bias| + conv(|x|, |w|) in float64."""
    if prec not in (PREC_FP16_TC, PREC_SPLIT_TC):
        return
    cf = F.conv_transpose2d if transposed else F.conv2d
    mag = cf(x.abs(), torch.from_numpy(wgt).double().abs(), torch.from_numpy(bias).double().abs(), stride, pad)
    a, b = fp16_tc_ab(K) if prec == PREC_FP16_TC else split_tc_ab(K)
    r = bound_ratio(got, ref, mag.permute(0, 2, 3, 1).numpy(), a, b)
    assert r.max() <= 1.0, "err/bound %.3g at %s" % (r.max(), np.unravel_index(np.argmax(r), r.shape))


def _conv_id(c):
    i = "c%s_o%d_k%d_s%d_r%d" % ("+".join(map(str, c[0])), c[1], c[2], c[3], int(c[5]))
    return i if len(c) < 10 else i + "_d%d_n%d_%dx%d" % (c[9], c[8], c[6], c[7])


@pytest.mark.parametrize("prec", [PREC_FP16_TC, PREC_FP32_SIMT, PREC_FP16_SIMT, PREC_SPLIT_TC])
@pytest.mark.parametrize("case", CONV_CASES, ids=_conv_id)
def test_conv(case, prec):
    srcc, cout, k, stride, act, residual, h, w, n = case[:9]
    down = case[9] if len(case) > 9 else 1
    rng = np.random.default_rng(hash((tuple(srcc), cout, k, stride)) % 2**32)
    cin = sum(srcc)
    so = SingleOp(srcc, down=down, extra_channels=8)
    wgt = _rand(rng, cout, cin, k, k, scale=1.0 / np.sqrt(cin * k * k))
    bias = _rand(rng, cout, scale=0.5)
    sh, sw = h // down, w // down
    ins = [_rand(rng, n, sh, sw, c) for c in srcc]
    dst = None
    dst_init = None
    if residual:
        db = so.P.newbuf(cout + 8, down * stride)
        dst = so.P.tensor(db, 8, cout)
        dst_init = _rand(rng, n, sh // stride, sw // stride, cout + 8)
    out_t = so.P.conv(so.srcs, wgt.astype(np.float64), bias.astype(np.float64), stride, act, dst=dst, residual=residual)
    if prec in (PREC_FP16_TC, PREC_FP16_SIMT):
        ins = [h16(a) for a in ins]
        wgt = h16(wgt)
        if dst_init is not None:
            dst_init = h16(dst_init)
    got = so.run(out_t, ins, n, h, w, prec, dst_init=dst_init)
    x = torch.from_numpy(np.concatenate(ins, -1)).permute(0, 3, 1, 2).double()
    ref = F.conv2d(x, torch.from_numpy(wgt).double(), torch.from_numpy(bias).double(), stride, k // 2)
    ref = ACTS[act](ref)
    if residual:
        ref = ref + torch.from_numpy(dst_init[..., 8:]).permute(0, 3, 1, 2).double()
    ref = ref.permute(0, 2, 3, 1).numpy()
    err = np.abs(got - ref).max()
    assert err <= _tol(prec, ref), "max abs err %g (ref max %g)" % (err, np.abs(ref).max())
    _check_bound(prec, got, x, wgt, bias, ref, cin * k * k, stride=stride, pad=k // 2)


DECONV_CASES = [([64], 32, 32, 32, 1), ([128], 64, 64, 64, 1), ([512], 256, 32, 32, 2), ([256], 128, 32, 64, 1),
                ([96], 64, 96, 32, 2),
                # (..., down): sources at 1/down of the page; 12x20 grid = partial tiles in x and y
                ([64], 32, 12, 20, 2, 16), ([128], 128, 12, 20, 3, 16), ([64], 64, 128, 128, 2, 2)]


def _deconv_id(c):
    i = "c%d_o%d_%dx%d" % (c[0][0], c[1], c[2], c[3])
    return i if len(c) < 6 else i + "_d%d_n%d" % (c[5], c[4])


@pytest.mark.parametrize("prec", [PREC_FP16_TC, PREC_FP32_SIMT, PREC_FP16_SIMT, PREC_SPLIT_TC])
@pytest.mark.parametrize("case", DECONV_CASES, ids=_deconv_id)
def test_deconv4(case, prec):
    srcc, cout, h, w, n = case[:5]
    down = case[5] if len(case) > 5 else 2
    rng = np.random.default_rng(cout * 7 + h)
    cin = sum(srcc)
    so = SingleOp(srcc, down=down, extra_channels=0)
    wgt = _rand(rng, cin, cout, 4, 4, scale=1.0 / np.sqrt(cin * 4))
    bias = _rand(rng, cout, scale=0.5)
    ins = [_rand(rng, n, h, w, c) for c in srcc]
    out_t = so.P.deconv4(so.srcs, wgt.astype(np.float64), bias.astype(np.float64), cc.ACT_RELU)
    if prec in (PREC_FP16_TC, PREC_FP16_SIMT):
        ins = [h16(a) for a in ins]
        wgt = h16(wgt)
    got = so.run(out_t, ins, n, down * h, down * w, prec)
    x = torch.from_numpy(np.concatenate(ins, -1)).permute(0, 3, 1, 2).double()
    ref = F.relu(F.conv_transpose2d(x, torch.from_numpy(wgt).double(), torch.from_numpy(bias).double(), 2, 1))
    ref = ref.permute(0, 2, 3, 1).numpy()
    assert got.shape == ref.shape
    err = np.abs(got - ref).max()
    assert err <= _tol(prec, ref), "max abs err %g (ref max %g)" % (err, np.abs(ref).max())
    _check_bound(prec, got, x, wgt, bias, ref, 4 * cin, transposed=True, stride=2, pad=1)
