"""-m gpu: every CUDA kernel against a plain torch fp32 reference of the same op (fp16-rounded
operands for the fp16 engines, so only accumulation order and the output rounding differ)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from util import SingleOp, h16, cc, PREC_FP16_TC, PREC_FP32_SIMT, PREC_FP16_SIMT

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
]


@pytest.mark.parametrize("prec", [PREC_FP16_TC, PREC_FP32_SIMT, PREC_FP16_SIMT])
@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "c%s_o%d_k%d_s%d_r%d" % ("+".join(map(str, c[0])), c[1], c[2], c[3], int(c[5])))
def test_conv(case, prec):
    srcc, cout, k, stride, act, residual, h, w, n = case
    rng = np.random.default_rng(hash((tuple(srcc), cout, k, stride)) % 2**32)
    cin = sum(srcc)
    so = SingleOp(srcc, down=1, extra_channels=8)
    wgt = _rand(rng, cout, cin, k, k, scale=1.0 / np.sqrt(cin * k * k))
    bias = _rand(rng, cout, scale=0.5)
    ins = [_rand(rng, n, h, w, c) for c in srcc]
    dst = None
    dst_init = None
    if residual:
        db = so.P.newbuf(cout + 8, stride)
        dst = so.P.tensor(db, 8, cout)
        dst_init = _rand(rng, n, h // stride, w // stride, cout + 8)
    out_t = so.P.conv(so.srcs, wgt.astype(np.float64), bias.astype(np.float64), stride, act, dst=dst, residual=residual)
    if prec != PREC_FP32_SIMT:
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


DECONV_CASES = [([64], 32, 32, 32, 1), ([128], 64, 64, 64, 1), ([512], 256, 32, 32, 2), ([256], 128, 32, 64, 1),
                ([96], 64, 96, 32, 2)]


@pytest.mark.parametrize("prec", [PREC_FP16_TC, PREC_FP32_SIMT, PREC_FP16_SIMT])
@pytest.mark.parametrize("case", DECONV_CASES, ids=lambda c: "c%d_o%d_%dx%d" % (c[0][0], c[1], c[2], c[3]))
def test_deconv4(case, prec):
    srcc, cout, h, w, n = case
    rng = np.random.default_rng(cout * 7 + h)
    cin = sum(srcc)
    so = SingleOp(srcc, down=2, extra_channels=0)
    wgt = _rand(rng, cin, cout, 4, 4, scale=1.0 / np.sqrt(cin * 4))
    bias = _rand(rng, cout, scale=0.5)
    ins = [_rand(rng, n, h, w, c) for c in srcc]
    out_t = so.P.deconv4(so.srcs, wgt.astype(np.float64), bias.astype(np.float64), cc.ACT_RELU)
    if prec != PREC_FP32_SIMT:
        ins = [h16(a) for a in ins]
        wgt = h16(wgt)
    got = so.run(out_t, ins, n, 2 * h, 2 * w, prec)
    x = torch.from_numpy(np.concatenate(ins, -1)).permute(0, 3, 1, 2).double()
    ref = F.relu(F.conv_transpose2d(x, torch.from_numpy(wgt).double(), torch.from_numpy(bias).double(), 2, 1))
    ref = ref.permute(0, 2, 3, 1).numpy()
    assert got.shape == ref.shape
    err = np.abs(got - ref).max()
    assert err <= _tol(prec, ref), "max abs err %g (ref max %g)" % (err, np.abs(ref).max())
