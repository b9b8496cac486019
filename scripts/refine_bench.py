"""Throughput of refine_mask on caller block lists (ctd_submit_refine) against the detector that made the blocks.

Workload: the 64 seeded pages of scripts/pages_bench.py at input_size 1024, detected once with
`detect_batch(keep_undetected_mask=False)` to get each page's (page, mask, blk_list), without the blocks whose window
is empty (the reference's refine_mask raises on them; the detector drops their windows, so its mask_refined is the
same without them; "dropped" counts them).  Arms, each run once to warm up
and then --reps times (the oracle once); each figure is the median pass (a pass ends when the last result is on the
host, or on the device for device_results):

  detect_stream_b16       the detector itself at max_batch 16 (network + post-processing + refine), for scale
  refine_stream_b16       MaskRefiner(max_batch=16).refine_stream, host results
  refine_stream_b16_dev   the same with device_results=True
  refine_mask_per_page    ctd_b200.refine_mask, one blocking call per page
  oracle_cpu              oracle/postproc_ref.refine_mask on --cpu-pages pages (one host thread)

Every GPU arm's mask_refined must equal the detector's own, byte for byte.  Prints one JSON line with pages/s and
blocks/s per arm and the card's name and power limit, read in the same run.

    python scripts/refine_bench.py [--pages 64] [--cpu-pages 4]"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from pages_bench import NET, card, workload  # noqa: E402


def timed(fn, reps):
    out = fn()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return out, statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=64)
    ap.add_argument("--cpu-pages", type=int, default=4)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    import numpy as np
    import torch
    import ctd_b200
    from ctd_b200 import binding
    from oracle import postproc_ref, synth
    ck = synth.make_checkpoint(0, smooth=True)
    pages = workload(args.pages)
    det = ctd_b200.TextDetector(ck, input_size=NET, act="leaky", max_batch=16)
    ref = ctd_b200.MaskRefiner(max_batch=16)
    try:
        detected = det.detect_batch(pages, keep_undetected_mask=False)
        items = []
        for p, (m, _mr, b) in zip(pages, detected):
            st = binding.refine_plan([p.shape[:2]], np.array([x.xyxy for x in b], np.int32).reshape(-1, 4), [len(b)])[2]
            items.append((p, m, [x for x, s in zip(b, st) if s == 0]))
        want = [mr for _m, mr, _b in detected]
        n_blocks = sum(len(b) for _p, _m, b in items)
        line = {"card": card(), "pages": len(pages), "blocks": n_blocks,
                "dropped": sum(len(d[2]) for d in detected) - n_blocks, "input_size": NET, "arms": {}}

        def arm(name, fn, n_pages, blocks, outs=None, reps=args.reps):
            got, dt = timed(fn, reps)
            if outs is not None:
                for g, w in zip(outs(got), want):
                    assert np.array_equal(g, w), name
            line["arms"][name] = {"pages_per_s": round(n_pages / dt, 2), "blocks_per_s": round(blocks / dt, 1)}

        arm("detect_stream_b16", lambda: list(det.detect_stream(pages)), len(pages), n_blocks,
            lambda got: [g[1] for g in got])
        arm("refine_stream_b16", lambda: list(ref.refine_stream(items)), len(pages), n_blocks,
            lambda got: [g[1] for g in got])

        def dev():
            out = list(ref.refine_stream(items, device_results=True))
            torch.cuda.synchronize()
            return out
        arm("refine_stream_b16_dev", dev, len(pages), n_blocks, lambda got: [g[1].cpu().numpy() for g in got])
        arm("refine_mask_per_page", lambda: [ctd_b200.refine_mask(p, m, b) for p, m, b in items], len(pages),
            n_blocks, lambda got: got)
        k = min(args.cpu_pages, len(items))
        arm("oracle_cpu", lambda: [postproc_ref.refine_mask(p, m, [x.xyxy for x in b]) for p, m, b in items[:k]], k,
            sum(len(b) for _p, _m, b in items[:k]), lambda got: got, reps=1)
        line["equal_to_detector"] = True
    finally:
        ref.close()
        det.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
