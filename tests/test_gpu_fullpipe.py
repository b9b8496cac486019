"""-m gpu: the full-page pipeline behind the C ABI -- ctd_detect_page (one page, any size) and ctd_submit_full /
ctd_collect (batches, two in flight, host group stage on the engine's worker thread, refine_mask on the resident
pages) -- against the oracle chain on the engine's own maps and against each other."""
import numpy as np
import pytest
import torch

import ctd_b200
from ctd_b200 import multigpu
from oracle import pipeline_ref, synth, textblock_ref
from util import get_checkpoint

pytestmark = pytest.mark.gpu


def _blk_key(b):
    return (tuple(int(v) for v in b.xyxy), np.array(b.lines).astype(int).tolist(), b.language, bool(b.vertical),
            float(b.font_size), int(b.angle))


@pytest.mark.parametrize("mode", [0, 1])
def test_submit_full_equals_detect_page_and_oracle(mode):
    ck = get_checkpoint(0, True)
    prog = ctd_b200.compiler.compile_checkpoint(ck)
    B, H, W = 3, 512, 512
    eng = ctd_b200.Engine(prog, max_batch=B, max_h=H, max_w=W, use_graph=True)
    one = ctd_b200.Engine(prog, max_batch=1, max_h=H, max_w=W)
    try:
        lay = eng.results_layout()
        batches = [np.stack([synth.structured_page(7000 + 10 * k + i, H, W) for i in range(B)]) for k in range(4)]
        host_in = [torch.from_numpy(pg).pin_memory() for pg in batches]
        host_out = [torch.zeros((lay["total_bytes"],), dtype=torch.uint8).pin_memory() for _ in batches]
        pending = []
        for k in range(len(batches)):
            if len(pending) == 2:
                eng.collect(pending.pop(0))
            eng.submit_full(k & 1, host_in[k].data_ptr(), B, H, W, host_out[k].data_ptr(), refine_mode=mode)
            pending.append(k & 1)
        while pending:
            eng.collect(pending.pop(0))
        n_blocks = 0
        for k, pg in enumerate(batches):
            got = multigpu.unpack_arena(host_out[k].numpy(), lay, B, H, W, full=True)
            for i in range(B):
                assert got["block_flags"][i] == 0
                # (a) the blocking single-page call
                m1, r1, rec, lines, dist = one.detect_page(pg[i], H, W, refine_mode=mode)
                b1 = ctd_b200.textblock.blocks_from_records(rec, lines, dist)
                assert np.array_equal(got["mask"][i], m1)
                assert [_blk_key(a) for a in got["blocks"][i]] == [_blk_key(b) for b in b1]
                assert np.array_equal(got["mask_refined"][i], r1), int((got["mask_refined"][i] != r1).sum())
                n_blocks += len(b1)
            # (b) the oracle chain on the engine's own maps (first page of every batch: the oracle's refine is slow)
            one.forward(pg[:1])
            blks, mf, lf = one.net_outputs()
            rmask, rref, rblk = pipeline_ref.postprocess_page(pg[0].copy(), blks[0], mf[0, 0], lf[0], textblock_ref.group_output,
                                                              refine_mode=mode)
            assert [_blk_key(a) for a in got["blocks"][0]] == [_blk_key(b) for b in rblk]
            assert np.array_equal(got["mask_refined"][0], rref)
        assert n_blocks > 10
    finally:
        eng.close()
        one.close()


def test_submit_full_device_pages_and_device_arena():
    """pages already resident in HBM (bench `value` leg) + the device copy of the results a multi-GPU gather moves"""
    ck = get_checkpoint(0, True)
    prog = ctd_b200.compiler.compile_checkpoint(ck)
    B, H, W = 2, 256, 256
    eng = ctd_b200.Engine(prog, max_batch=B, max_h=H, max_w=W, use_graph=True)
    try:
        lay = eng.results_layout()
        pages = np.stack([synth.structured_page(8000 + i, H, W) for i in range(B)])
        dev = torch.from_numpy(pages).cuda()
        out_a = torch.zeros((lay["total_bytes"],), dtype=torch.uint8).pin_memory()
        out_b = torch.zeros((lay["total_bytes"],), dtype=torch.uint8).pin_memory()
        eng.submit_full(0, dev.data_ptr(), B, H, W, out_a.data_ptr(), pages_on_device=True)
        eng.collect(0)
        host = torch.from_numpy(pages).pin_memory()
        eng.submit_full(1, host.data_ptr(), B, H, W, out_b.data_ptr())
        eng.collect(1)
        a = multigpu.unpack_arena(out_a.numpy(), lay, B, H, W, full=True)
        b = multigpu.unpack_arena(out_b.numpy(), lay, B, H, W, full=True)
        assert np.array_equal(a["mask"], b["mask"]) and np.array_equal(a["mask_refined"], b["mask_refined"])
        for i in range(B):
            assert [_blk_key(x) for x in a["blocks"][i]] == [_blk_key(y) for y in b["blocks"][i]]
        # the device copy holds the same bytes for the sections the pipeline fills
        base, _st = eng.device_arena(1)

        class _DevArr:
            def __init__(self, ptr, nbytes):
                self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3}
        d = torch.as_tensor(_DevArr(base, lay["total_bytes"]), device="cuda").cpu().numpy()
        dd = multigpu.unpack_arena(d, lay, B, H, W, full=True)
        assert np.array_equal(dd["mask"], b["mask"]) and np.array_equal(dd["mask_refined"], b["mask_refined"])
        for i in range(B):
            assert [_blk_key(x) for x in dd["blocks"][i]] == [_blk_key(y) for y in b["blocks"][i]]
    finally:
        eng.close()


def _bytes(x):
    """a collected result as host bytes and shapes, CUDA tensors copied back, nesting kept"""
    if x is None:
        return None
    if isinstance(x, (list, tuple)):
        return [_bytes(v) for v in x]
    if isinstance(x, torch.Tensor):
        x = x.cpu().numpy()
    return x.shape, np.ascontiguousarray(x).tobytes()


def _collected(items):
    """collect_pages items as mask, mask_refined, blocks and crops (the line and distance arrays past a page's own
    entries are not results)"""
    return [[_bytes(it[0]), _bytes(it[1]),
             [_blk_key(b) for b in ctd_b200.textblock.blocks_from_records(it[2], it[3], it[4])], _bytes(list(it[5:]))]
            for it in items]


def test_slots_reused_across_host_device_and_pages_batches():
    """one handle's two slots run, in turn, ctd_submit_full on host pages (slot 0), ctd_submit_pages with crops and
    results on the device (slot 1), ctd_submit_full on device pages (slot 0) and ctd_submit_pages with neither
    (slot 1): every batch computes what it computes on a fresh handle, and a slot hands out crops or device results
    only when its last batch made them"""
    prog = ctd_b200.compiler.compile_checkpoint(get_checkpoint(0, True))
    B, N = 2, 256

    def engine():
        return ctd_b200.Engine(prog, max_batch=B, max_h=N, max_w=N, use_graph=True)

    net_pages = torch.from_numpy(np.stack([synth.structured_page(9100 + i, N, N) for i in range(B)])).pin_memory()
    dev_pages = net_pages.cuda()
    pages_a = [synth.structured_page(9200, 361, 251), synth.structured_page(9201, 414, 292)]
    pages_b = [synth.structured_page(9300, 200, 150), synth.structured_page(9301, 2 * N, 2 * N)]

    def run(eng, kind):
        out = torch.zeros((eng.results_layout()["total_bytes"],), dtype=torch.uint8).pin_memory()
        pages = dev_pages if kind == "device" else net_pages
        eng.submit_full(0, pages.data_ptr(), B, N, N, out.data_ptr(), pages_on_device=kind == "device")
        return out

    def arena(eng, out):
        lay = eng.results_layout()
        got = multigpu.unpack_arena(out.numpy(), lay, B, N, N, full=True)
        return (out[:lay["phase_a_bytes"]].numpy().tobytes(), _bytes(got["mask_refined"]),
                [[_blk_key(b) for b in blks] for blks in got["blocks"]])

    eng = engine()
    try:
        out_host = run(eng, "host")
        eng.submit_pages(1, pages_a, N, N, textheight=32, device_results=True)
        eng.collect(0)
        got_a = eng.collect_pages(1)
        got_host = arena(eng, out_host)
        out_dev = run(eng, "device")
        eng.submit_pages(1, pages_b, N, N)
        eng.collect(0)
        got_dev = arena(eng, out_dev)
        got_b = eng.collect_pages(1)
        # neither slot's last batch asked for crops, and neither left its results on the device.  The destinations
        # are valid device memory with room for pages_a's [mask | mask_refined | crops] (slot 1 still holds that
        # batch's page entries), so only the slot's state can refuse the copy.
        dst = [torch.empty((2 * p.shape[0] * p.shape[1] + (32 << 20),), dtype=torch.uint8, device="cuda")
               for p in pages_a]
        ptrs = (ctd_b200.binding.C.c_void_p * B)(*[d.data_ptr() for d in dst])
        for slot in (0, 1):
            with pytest.raises(ctd_b200.CtdError, match="ctd_submit_pages batch with a textheight"):
                eng.collect_regions(slot, [[], []])
            assert eng.lib.ctd_collect_device(eng.h, slot, ptrs) == -1
            assert b"results on the device" in eng.lib.ctd_last_error(eng.h)
    finally:
        eng.close()
    assert sum(len(p[2]) for p in got_a) > 0 and any(c is not None for p in got_a for blk in p[5] for c in blk)
    assert all(isinstance(p[0], torch.Tensor) and p[0].is_cuda for p in got_a)
    ref = {}
    for kind in ("host", "device"):
        one = engine()
        try:
            out = run(one, kind)
            one.collect(0)
            ref[kind] = arena(one, out)
        finally:
            one.close()
    for key, pages, kw in (("a", pages_a, dict(textheight=32, device_results=True)), ("b", pages_b, {})):
        one = engine()
        try:
            one.submit_pages(0, pages, N, N, **kw)
            ref[key] = one.collect_pages(0)
        finally:
            one.close()
    assert got_host == ref["host"]
    assert got_dev == ref["device"]
    assert _collected(got_a) == _collected(ref["a"])
    assert _collected(got_b) == _collected(ref["b"])


def test_keep_undetected_on_page_larger_than_net_input():
    """ADVICE r1 (high): keep_undetected_mask=True on a page with more pixels than the net input used to fail with
    'image larger than the workspace'."""
    det = ctd_b200.TextDetector(get_checkpoint(0, True), input_size=256, act="leaky")
    try:
        for shape in [(360, 250), (700, 1000)]:
            page = synth.structured_page(5, shape[0], shape[1])
            mask, mask_refined, blk_list = det(page.copy(), keep_undetected_mask=True)
            assert mask.shape == shape and mask_refined.shape == shape
            m0, r0, b0 = det(page.copy(), keep_undetected_mask=False)
            assert np.all((mask_refined | r0) == mask_refined)          # the undetected pass only adds pixels
            assert [_blk_key(a) for a in blk_list] == [_blk_key(b) for b in b0]
    finally:
        det.close()
