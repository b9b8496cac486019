"""-m gpu: the drop-in `TextDetector` end to end.  The network runs in fp16 on tensor cores, so its maps differ
from the fp32 reference within the stated tolerance (tests/test_gpu_net.py); everything AFTER the network is
checked exactly: the oracle post-processing chain is run on the engine's own maps and must reproduce the
detector's outputs (mask, mask_refined, blocks) -- SURVEY section 4 tier 3/4."""
import numpy as np
import pytest

import ctd_b200
from oracle import pipeline_ref, synth, textblock_ref
from util import get_checkpoint

pytestmark = pytest.mark.gpu


def _blk_key(b):
    return (tuple(int(v) for v in b.xyxy), np.array(b.lines).astype(int).tolist(), b.language, bool(b.vertical),
            float(b.font_size), int(b.angle))


@pytest.mark.parametrize("keep_undetected", [False, True])
@pytest.mark.parametrize("mode", [0, 1])
def test_text_detector_matches_oracle_chain(mode, keep_undetected):
    ck = get_checkpoint(0, True)
    det = ctd_b200.TextDetector(ck, input_size=512, act="leaky")
    try:
        for seed in (1000, 1003):
            img = synth.structured_page(seed, 512, 512)
            mask, mask_refined, blk_list = det(img.copy(), refine_mode=mode, keep_undetected_mask=keep_undetected)
            det.net.forward(img[None])
            blks, mf, lf = det.net.net_outputs()
            # the oracle chain (cv2 / numpy restatement of the reference, with the python restatement of group_output)
            # on the engine's own maps must reproduce the native pipeline exactly: blocks, mask, mask_refined
            rmask, rref, rblk = pipeline_ref.postprocess_page(img.copy(), blks[0], mf[0, 0], lf[0], textblock_ref.group_output,
                                                              refine_mode=mode, keep_undetected_mask=keep_undetected)
            assert mask.shape == (512, 512) and mask.dtype == np.uint8
            assert [_blk_key(a) for a in blk_list] == [_blk_key(b) for b in rblk]
            assert np.array_equal(mask_refined, rref), int((mask_refined != rref).sum())
            assert np.array_equal(mask, rmask)
            assert len(blk_list) > 3
    finally:
        det.close()


def test_submit_full_phase_a_matches_blocking_forward():
    """ctd_submit_full/ctd_collect (two batches in flight, copies on side streams) must deliver result arenas whose
    phase-A section is byte-identical to the blocking ctd_forward + ctd_get_* path, in submission order, for different
    pages per batch."""
    import torch
    from ctd_b200 import multigpu
    ck = get_checkpoint(0, True)
    prog = ctd_b200.compiler.compile_checkpoint(ck)
    B, H, W = 2, 256, 256
    eng = ctd_b200.Engine(prog, max_batch=B, max_h=H, max_w=W, use_graph=True)
    try:
        batches = [np.stack([synth.structured_page(3000 + 10 * k + i, H, W) for i in range(B)]) for k in range(5)]
        want = []
        for pg in batches:
            eng.forward(pg)
            boxes, scores = eng.text_lines()
            want.append((eng.mask_u8().copy(), eng.detections(), boxes, scores))
        lay = eng.results_layout()
        assert multigpu.arena_layout(B, H, W)["phase_a_bytes"] == lay["phase_a_bytes"]
        host_in = [torch.from_numpy(pg).pin_memory() for pg in batches]
        host_out = [torch.zeros((lay["total_bytes"],), dtype=torch.uint8).pin_memory() for _ in batches]
        pending = []
        for k in range(len(batches)):
            if len(pending) == 2:
                eng.collect(pending.pop(0))
            eng.submit_full(k & 1, host_in[k].data_ptr(), B, H, W, host_out[k].data_ptr())
            pending.append(k & 1)
        with pytest.raises(ctd_b200.binding.CtdError):
            eng.submit_full(pending[0], host_in[0].data_ptr(), B, H, W, host_out[0].data_ptr())  # slot still in flight
        while pending:
            eng.collect(pending.pop(0))
        for k, (mask, dets, boxes, scores) in enumerate(want):
            got = multigpu.unpack_arena(host_out[k].numpy(), lay, B, H, W)
            assert np.array_equal(got["mask"], mask)
            for i in range(B):
                assert np.array_equal(got["det"][i], dets[i])
                assert np.array_equal(got["line_boxes"][i], boxes[i]) and np.array_equal(got["line_scores"][i], scores[i])
                assert len(boxes[i]) > 0
    finally:
        eng.close()


def test_two_workspaces_interleaved_equal_single():
    """Two engines (workspaces) on one GPU with batches alternating between them and `ctd_join` ordering the streams
    (what bench.py times) must give exactly the results of one engine used serially."""
    ck = get_checkpoint(0, True)
    prog = ctd_b200.compiler.compile_checkpoint(ck)
    B, H, W = 2, 256, 256
    batches = [np.stack([synth.structured_page(4000 + 10 * k + i, H, W) for i in range(B)]) for k in range(4)]
    single = ctd_b200.Engine(prog, max_batch=B, max_h=H, max_w=W)
    try:
        want = []
        for pg in batches:
            single.forward(pg)
            want.append((single.mask_u8().copy(), single.detections(), single.text_lines()))
    finally:
        single.close()
    engs = [ctd_b200.Engine(prog, max_batch=B, max_h=H, max_w=W) for _ in range(2)]
    try:
        got = []
        for rnd in range(2):                      # 2 rounds x 2 engines, both forwards in flight before any read
            for k, e in enumerate(engs):
                e.forward(batches[2 * rnd + k])
            engs[0].join(engs[1])
            for e in engs:
                got.append((e.mask_u8().copy(), e.detections(), e.text_lines()))
        for (m0, d0, (b0, s0)), (m1, d1, (b1, s1)) in zip(want, got):
            assert np.array_equal(m0, m1)
            for i in range(B):
                assert np.array_equal(d0[i], d1[i]) and np.array_equal(b0[i], b1[i]) and np.array_equal(s0[i], s1[i])
        with pytest.raises(ctd_b200.binding.CtdError):
            engs[0].lib.ctd_join.restype  # noqa: B018  (attribute exists)
            engs[0]._ck(engs[0].lib.ctd_join(engs[0].h, None))
    finally:
        for e in engs:
            e.close()
