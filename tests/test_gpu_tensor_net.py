"""-m gpu: `ctd_b200.TextDetBase`, the network on float32 CUDA tensors (`ctd_forward_tensor`).

  * for x = u8 / 255 (what preprocess_img makes) the module's blks / mask / lines equal `Engine.forward` on the u8
    pages bit for bit, in all four precisions;
  * any other float input against the fp32 oracle (oracle/net_ref.py);
  * the oracle's post-processing chain on the module's tensors equals `ctd_b200.TextDetector`;
  * stream order on both sides of the call, shape changes, non-contiguous inputs and the refusals."""
import numpy as np
import pytest
import torch

import ctd_b200
from oracle import synth, pipeline_ref, textblock_ref
from oracle.net_ref import RefNet
from util import get_checkpoint, page_to_net_input, PREC_FP16_TC, PREC_FP32_SIMT, PREC_FP16_SIMT, PREC_SPLIT_TC

pytestmark = pytest.mark.gpu

PRECS = [(PREC_FP16_TC, "fp16_tc"), (PREC_SPLIT_TC, "split_tc"), (PREC_FP32_SIMT, "fp32_simt"),
         (PREC_FP16_SIMT, "fp16_simt")]

# The tolerances tests/test_gpu_net.py states for the whole forward against the fp32 oracle: max abs error of the maps,
# its mean, its 99.9th percentile and the relative error of the Detect rows.  The fp16 ones are statistical (fp16
# storage of every activation; see that file).
TOL = {PREC_FP32_SIMT: dict(maps=1e-3, maps_mean=1e-4, p999=1e-3, blks_rel=2e-3),
       PREC_SPLIT_TC: dict(maps=1e-3, maps_mean=1e-4, p999=1e-3, blks_rel=2e-3),
       PREC_FP16_TC: dict(maps=0.8, maps_mean=1.5e-2, p999=0.25, blks_rel=1.0)}


def _pages(n, h, w, seed=1000):
    return np.stack([synth.structured_page(seed + i, h, w) if i % 2 == 0 else synth.noise_page(seed + i, h, w)
                     for i in range(n)])


def _u8_outputs(ck, prec, pages, use_graph=False):
    n, h, w, _ = pages.shape
    eng = ctd_b200.Engine(ctd_b200.compiler.compile_checkpoint(ck), precision=prec, max_batch=n, max_h=h, max_w=w,
                          use_graph=use_graph)
    try:
        eng.forward(pages)
        return eng.net_outputs()
    finally:
        eng.close()


def _assert_same(got, want, what=""):
    for name, g, e in zip(("blks", "mask", "lines"), got, want):
        g = g.cpu().numpy() if isinstance(g, torch.Tensor) else g
        e = e.cpu().numpy() if isinstance(e, torch.Tensor) else e
        assert g.shape == e.shape, (what, name, g.shape, e.shape)
        assert np.array_equal(g, e), "%s %s: max diff %g" % (what, name, float(np.abs(g - e).max()))


@pytest.mark.parametrize("prec", [p for p, _ in PRECS], ids=[i for _, i in PRECS])
def test_identity_with_u8_path(prec):
    ck = get_checkpoint(0, True)
    pages = _pages(2, 256, 320)
    want = _u8_outputs(ck, prec, pages)
    mod = ctd_b200.TextDetBase(ck, precision=prec, max_batch=2, max_size=(256, 320))
    try:
        got = mod(page_to_net_input(pages).cuda())
        _assert_same(got, want, "prec %d" % prec)
    finally:
        mod.close()


def test_identity_with_u8_path_benchmark_batch():
    """16 pages of 1024 x 1024, fp16 tensor cores, the u8 engine under a CUDA graph (as bench.py runs it)"""
    ck = get_checkpoint(0, True)
    pages = _pages(16, 1024, 1024)
    want = _u8_outputs(ck, PREC_FP16_TC, pages, use_graph=True)
    mod = ctd_b200.TextDetBase(ck, max_batch=16, max_size=1024)
    try:
        x = page_to_net_input(pages).cuda()
        _assert_same(mod(x), want, "16x1024")
        _assert_same(mod(x), want, "16x1024, second call")
    finally:
        mod.close()


def _float_inputs(n, h, w, kind, seed):
    g = np.random.default_rng(seed)
    if kind == "u8_noise":
        x = page_to_net_input(_pages(n, h, w, seed)).numpy() + g.normal(0, 0.01, (n, 3, h, w)).astype(np.float32)
    else:
        x = g.uniform(-0.1, 1.1, (n, 3, h, w)).astype(np.float32)
    return torch.from_numpy(np.ascontiguousarray(x, np.float32))


@pytest.mark.parametrize("kind", ["u8_noise", "uniform"])
@pytest.mark.parametrize("prec", [PREC_SPLIT_TC, PREC_FP32_SIMT, PREC_FP16_TC], ids=["split_tc", "fp32_simt", "fp16_tc"])
def test_float_input_against_oracle(prec, kind):
    ck = get_checkpoint(0, True)
    n, h, w = 2, 256, 320
    x = _float_inputs(n, h, w, kind, 31)
    with torch.no_grad():
        rb, rm, rl = (t.numpy() for t in RefNet(ck)(x))
    mod = ctd_b200.TextDetBase(ck, precision=prec, max_batch=n, max_size=(h, w))
    try:
        blks, mask, lines = (t.cpu().numpy() for t in mod(x.cuda()))
    finally:
        mod.close()
    tol = TOL[prec]
    e_mask, e_lines = float(np.abs(mask - rm).max()), float(np.abs(lines - rl).max())
    m_mask, m_lines = float(np.abs(mask - rm).mean()), float(np.abs(lines - rl).mean())
    e_blks = float((np.abs(blks - rb) / (np.abs(rb) + 1.0)).max())
    msg = "prec %d %s: max err mask %.3g lines %.3g blks(rel) %.3g; mean err mask %.3g lines %.3g" % (
        prec, kind, e_mask, e_lines, e_blks, m_mask, m_lines)
    print(msg)
    assert e_mask <= tol["maps"] and e_lines <= tol["maps"], msg
    assert m_mask <= tol["maps_mean"] and m_lines <= tol["maps_mean"], msg
    assert e_blks <= tol["blks_rel"], msg
    for got, ref in ((mask, rm), (lines, rl)):
        d = np.abs(got - ref).ravel()
        assert float(np.partition(d, int(d.size * 0.999))[int(d.size * 0.999)]) <= tol["p999"], msg


def test_reference_chain_on_module_tensors():
    """INTEGRATION.md: `self.net = ctd_b200.TextDetBase(model_path, device='cuda', act=act)` under the reference's own
    post-processing (here the oracle's restatement of it) gives what ctd_b200.TextDetector gives"""
    ck = get_checkpoint(0, True)
    size = 512
    det = ctd_b200.TextDetector(ck, input_size=size, act="leaky")
    net = ctd_b200.TextDetBase(ck, device='cuda', act='leaky')
    key = lambda b: (tuple(int(v) for v in b.xyxy), np.array(b.lines).astype(int).tolist(), b.language,
                     bool(b.vertical), int(b.angle))
    try:
        for seed in (1000, 1003):
            page = synth.structured_page(seed, size, size)
            mask8, mask_refined, blk_list = det(page.copy())
            blks, mask, lines = net(page_to_net_input(page[None]).cuda())
            rmask, rref, rblk = pipeline_ref.postprocess_page(page.copy(), blks[0].cpu(), mask[0, 0].cpu(),
                                                              lines[0].cpu(), textblock_ref.group_output)
            assert len(blk_list) > 3 and [key(a) for a in blk_list] == [key(b) for b in rblk], seed
            assert np.array_equal(mask8, rmask) and np.array_equal(mask_refined, rref), seed
    finally:
        det.close()
        net.close()


def _sleep_ms(ms):
    """a kernel that keeps the current stream busy for about `ms` milliseconds"""
    torch.cuda._sleep(int(ms * 1e6))   # cycles at ~1-2 GHz: 0.5-1 ms per million


def test_stream_order_side_stream():
    ck = get_checkpoint(0, True)
    n, h, w = 2, 256, 320
    src = _float_inputs(n, h, w, "uniform", 5).cuda()
    mod = ctd_b200.TextDetBase(ck, max_batch=n, max_size=(h, w))
    try:
        want = [t.cpu() for t in mod(src)]
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        x = torch.zeros_like(src)
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            _sleep_ms(50)
            x.copy_(src)            # x is written only after the sleep: the engine must wait for it
            outs = mod(x)
            got = [t.clone() for t in outs]   # consumers enqueued right after the call, no synchronize
            s_done = torch.cuda.Event()
            s_done.record(s)
        s_done.synchronize()
        _assert_same(got, want, "side stream")
        _assert_same(outs, want, "side stream, the outputs themselves")
    finally:
        mod.close()


def test_stream_order_default_stream():
    ck = get_checkpoint(0, True)
    n, h, w = 1, 256, 256
    src = _float_inputs(n, h, w, "u8_noise", 6).cuda()
    mod = ctd_b200.TextDetBase(ck, max_batch=n, max_size=(h, w))
    try:
        want = [t.cpu() for t in mod(src)]
        x = torch.zeros_like(src)
        torch.cuda.synchronize()
        _sleep_ms(50)
        x.copy_(src)
        outs = mod(x)
        sums = [t.sum(dtype=torch.float64) for t in outs]   # consumers on the default stream, right after the call
        got = [t.clone() for t in outs]
        _assert_same(got, want, "default stream")
        for s, t in zip(sums, want):
            assert float(s) == float(t.sum(dtype=torch.float64))
    finally:
        mod.close()


def test_shape_sequence_and_views():
    ck = get_checkpoint(0, True)
    mod = ctd_b200.TextDetBase(ck, max_batch=3, max_size=(384, 512))
    try:
        shapes = [(2, 256, 384), (1, 128, 192), (2, 384, 512), (1, 64, 448), (2, 256, 384)]
        for i, (n, h, w) in enumerate(shapes):
            x = _float_inputs(n, h, w, "uniform" if i % 2 else "u8_noise", 40 + i).cuda()
            got = mod(x)
            alone = ctd_b200.TextDetBase(ck, max_batch=n, max_size=(h, w))
            try:
                _assert_same(got, alone(x), "shape %s" % ((n, h, w),))
            finally:
                alone.close()
        big = _float_inputs(2, 320, 448, "u8_noise", 60).cuda()
        flat = torch.empty((1 + big[:1].numel(),), device=big.device)
        unaligned = flat[1:].view(big[:1].shape)   # contiguous, 4 bytes past a 16-byte boundary
        unaligned.copy_(big[:1])
        views = {"channels_last": big[:, :, :256, :384].contiguous().to(memory_format=torch.channels_last),
                 "slice": big[:, :, 40:296, 64:448],
                 "batch slice": big[1:],
                 "unaligned": unaligned}
        for name, v in views.items():
            assert name in ("batch slice", "unaligned") or not v.is_contiguous()
            _assert_same(mod(v), mod(v.contiguous()), name)
    finally:
        mod.close()


def test_refusals_leave_module_usable():
    ck = get_checkpoint(0, True)
    n, h, w = 2, 128, 192
    mod = ctd_b200.TextDetBase(ck, max_batch=n, max_size=(h, w))
    try:
        x = _float_inputs(n, h, w, "uniform", 7).cuda()
        want = [t.cpu() for t in mod(x)]
        bad = {"cpu tensor": x.cpu(),
               "numpy array": x.cpu().numpy(),
               "float16": x.half(),
               "float64": x.double(),
               "3-d": x[0],
               "4 channels": torch.cat([x, x[:, :1]], 1),
               "H not a multiple of 64": x[:, :, :96],
               "W not a multiple of 64": x[:, :, :, :160],
               "H above max_size": torch.zeros((1, 3, h + 64, w), device=x.device),
               "W above max_size": torch.zeros((1, 3, h, w + 64), device=x.device),
               "N = 0": x[:0],
               "N above max_batch": torch.cat([x, x[:1]], 0)}
        if torch.cuda.device_count() > 1:
            bad["other device"] = x.to("cuda:1")
        for name, b in bad.items():
            with pytest.raises(ValueError):
                mod(b)
            _assert_same(mod(x), want, "after refusing %s" % name)
        with pytest.raises(ValueError):
            ctd_b200.TextDetBase("model.onnx")
        with pytest.raises(ValueError):
            ctd_b200.TextDetBase(ck, device="cpu")
    finally:
        mod.close()
