"""-m gpu: EVERY launch plan of the real network, one op at a time, against the CPU interpreter of the program
(tests/prog_interp.py) fed the SAME inputs ("teacher forcing"): the interpreter's buffers are written into the
engine, only op i runs (ctd_debug_run_ops), and the slice it wrote must match the interpreter's result for op i.
Nothing is amplified by the (ill-conditioned, random-weight) net, so the tolerances are those of one rounding:

  * CTD_PREC_FP16_TC (the benchmarked wgmma engine) vs the fp16-storage emulation: <= 2e-3 relative -- one fp16
    ulp (2^-10) where a value sits on a rounding boundary and the fp32 accumulation order differs;
  * CTD_PREC_SPLIT_TC (split-fp16 tensor-core engine) and CTD_PREC_FP32_SIMT (CUDA-core fp32 engine) vs the fp32
    interpreter: <= 1e-4 of (|ref| + 1 % of the tensor's scale) -- both sides round differently in fp32 (torch's
    oneDNN blocking vs the engine's K order / the tensor core's accumulator), measured 1e-6 .. 4e-5.

A wrong tap, border, K-concatenation, phase or residual shows up as an O(1) error in exactly the op that has it,
instead of hiding inside the net-level statistical tolerance of test_gpu_net.py."""
import numpy as np
import pytest

import ctd_b200
from ctd_b200 import compiler as cc
from oracle import synth
from prog_interp import Interp
from util import get_checkpoint, PREC_FP16_TC, PREC_SPLIT_TC, PREC_FP32_SIMT

pytestmark = pytest.mark.gpu


def _pages(n, h, w, seed=1000):
    return np.stack([synth.structured_page(seed + i, h, w) if i % 2 == 0 else synth.noise_page(seed + i, h, w)
                     for i in range(n)])


def _tensor(prog, buf):
    return dict(buf=buf, coff=0, c=prog.bufs[buf][0], down=prog.bufs[buf][1])


@pytest.mark.parametrize("prec,storage,rel", [(PREC_FP16_TC, "f16", 2e-3), (PREC_SPLIT_TC, "f32", 1e-4),
                                              (PREC_FP32_SIMT, "f32", 1e-4)], ids=["fp16_tc", "split_tc", "fp32_simt"])
@pytest.mark.parametrize("shape", [(2, 256, 320), (1, 192, 448)], ids=["2x256x320", "1x192x448"])
def test_every_op_matches_interpreter(prec, storage, rel, shape):
    n, h, w = shape
    ck = get_checkpoint(0, True)
    prog = ctd_b200.compiler.compile_checkpoint(ck)
    pages = _pages(n, h, w, seed=31)
    it = Interp(prog, pages, storage)
    eng = ctd_b200.Engine(prog, precision=prec, max_batch=n, max_h=h, max_w=w, skip_postproc=True)
    worst = []
    try:
        for i, op in enumerate(prog.ops):
            k = op["kind"]
            touched = set(op["src_buf"][:op["n_src"]])
            if op["dst_buf"] >= 0:
                touched.add(op["dst_buf"])
            if k == cc.OP_STEM:
                touched.discard(op["src_buf"][0])       # the s2d staging buffer is produced by the op itself
            for b in sorted(touched):
                eng.debug_write(_tensor(prog, b), it.buf_nhwc(b), n, h, w)
            eng.debug_run_ops(i, i, n, h, w, pages=pages if k == cc.OP_STEM else None)
            it.step(i)
            wr = it.written(op)
            if wr is not None:
                buf, coff, c = wr
                got = eng.debug_read(dict(buf=buf, coff=coff, c=c, down=prog.bufs[buf][1]))
                ref = it.buf_nhwc(buf)[..., coff:coff + c]
                pairs = [("buf", got, ref, rel)]
            elif k == cc.OP_DETECT:
                blks, _, _ = eng.net_outputs(want_mask=False, want_lines=False)
                r0 = sum(3 * (h // (8 << l)) * (w // (8 << l)) for l in range(op["aux"]))
                r1 = r0 + 3 * (h // (8 << op["aux"])) * (w // (8 << op["aux"]))
                pairs = [("blks", blks[:, r0:r1], it.blks[:, r0:r1].numpy(), rel)]
            elif k == cc.OP_SEG_TAIL:
                _, mask, _ = eng.net_outputs(want_blks=False, want_lines=False)
                pairs = [("mask", mask, it.mask.numpy(), rel)]
            else:
                _, _, lines = eng.net_outputs(want_blks=False, want_mask=False)
                pairs = [("lines", lines, it.lines.numpy(), rel)]
            for name, got, ref, r in pairs:
                scale = float(np.abs(ref).max()) + 1e-12
                err = np.abs(got - ref) / (np.abs(ref) + 0.01 * scale)
                e = float(err.max())
                worst.append((e, i, k, name))
    finally:
        eng.close()
    worst.sort(reverse=True)
    print("worst ops (rel err, op, kind):", [(float("%.3g" % e), i, k) for e, i, k, _ in worst[:8]],
          "median %.3g" % float(np.median([w[0] for w in worst])))
    bad = [(e, i, k, nm) for e, i, k, nm in worst if e > rel]
    assert not bad, "ops above %.3g: %s" % (rel, bad[:10])
