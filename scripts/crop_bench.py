"""Throughput of the OCR crops of a caller's block list: the blocking per-page `TextDetector.get_transformed_regions`
against `RegionCropper.crop_stream` (ctd_submit_regions: lines planned on the engine's worker threads, one
k_warp_regions launch per batch, CUDA pages read where they are).

Workload: the 64 seeded pages of scripts/stream_regions_bench.py at input_size 1024, textheight 48, max_batch 16.  The
blocks come from `detect_stream` and are round-tripped through `to_dict` and json (`TextBlock(**d)`), as a caller that
edits or stores them has them; that happens before any timed region.  Every arm runs the workload once to warm up, then
twice timed; the time ends when the last crop is in the caller's hands.

    python scripts/crop_bench.py [--out DIR] [--profile]

Arms: (b) `get_transformed_regions` block by block (a page where some line raises cannot be cut in one call; the blocks
that raise are skipped), as stream_regions_bench.py's arm (b) does after the stream; `crop_stream` with host results;
`crop_stream(device_results=True)`; and the latter with the pages as CUDA tensors.  Reported per arm: pages/s, lines/s
and crop Mpx/s, with the card's name and power limit read in the same run.

--profile: a separate run.  Device time of k_warp_regions per batch (torch.profiler, CUDA activity) for host and CUDA
pages, and per batch the host time of the line records (`regions.line_records`, on the caller's thread) and of the
plans (`ctd_region_plan`, which the worker runs on its host threads; timed here on one thread).  Prints one JSON line."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from stream_regions_bench import MAX_BATCH, NET, SIZES, TEXTHEIGHT, _count, card, workload  # noqa: E402


def blocks_of(det, pages):
    """the detector's blocks of every page, through to_dict, json and TextBlock(**d)"""
    from ctd_b200.annotations import NumpyEncoder
    from ctd_b200.textblock import TextBlock
    out = []
    for _m, _r, blks in det.detect_stream(pages, refine_mode=0):
        out.append([TextBlock(**d) for d in json.loads(json.dumps([b.to_dict() for b in blks], cls=NumpyEncoder))])
    return out


def run_arm(det, cropper, items, arm):
    """one pass -> (lines cropped, crop pixels)"""
    from ctd_b200 import CtdError
    lines = px = 0
    if arm == "b":
        for img, blks in items:
            crops = []
            for b in blks:
                try:
                    crops += det.get_transformed_regions(img, [b], TEXTHEIGHT)
                except CtdError:
                    pass
            nl, npx = _count(crops)
            lines, px = lines + nl, px + npx
        return lines, px
    for crops in cropper.crop_stream(items, TEXTHEIGHT, device_results=arm != "host"):
        nl, npx = _count(crops)
        lines, px = lines + nl, px + npx
    if arm != "host":
        import torch
        torch.cuda.synchronize()
    return lines, px


def profile(cropper, items, cuda_items):
    import numpy as np
    import torch
    from ctd_b200 import binding, regions
    n_batches = (len(items) + MAX_BATCH - 1) // MAX_BATCH
    out = {"batches": n_batches}
    rec_ms, plan_ms = [], []
    for k in range(n_batches):
        batch = items[k * MAX_BATCH:(k + 1) * MAX_BATCH]
        t0 = time.perf_counter()
        recs = [regions.line_records(blks)[0] for _img, blks in batch]
        t1 = time.perf_counter()
        for (img, _b), rec in zip(batch, recs):
            binding.region_plan(rec, img.shape[1], img.shape[0], TEXTHEIGHT)
        t2 = time.perf_counter()
        rec_ms.append((t1 - t0) * 1e3)
        plan_ms.append((t2 - t1) * 1e3)
    out["line_records_ms_per_batch"] = round(float(np.mean(rec_ms)), 3)
    out["plan_ms_per_batch_one_thread"] = round(float(np.mean(plan_ms)), 3)
    for name, its in (("host_pages", items), ("cuda_pages", cuda_items)):
        run_arm(None, cropper, its, "device")
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            lines, px = run_arm(None, cropper, its, "device")
            torch.cuda.synchronize()
        us, cnt = 0.0, 0
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA and "k_warp_regions" in ev.name:
                us += ev.time_range.elapsed_us()
                cnt += 1
        out[name] = {"launches": cnt, "device_us": round(us, 1), "device_us_per_batch": round(us / max(cnt, 1), 1),
                     "lines": lines, "crop_bytes": px * 3,
                     "crop_gb_per_s": round(px * 3 / (us * 1e-6) / 1e9, 1) if us > 0 else None}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--pages", type=int, default=64)
    args = ap.parse_args()
    import torch
    import ctd_b200
    from oracle import synth
    pages = workload(args.pages)
    line = {"card": card(), "pages": len(pages), "input_size": NET, "sizes": SIZES, "textheight": TEXTHEIGHT,
            "max_batch": MAX_BATCH, "arms": {}}
    det = ctd_b200.TextDetector(synth.make_checkpoint(0, smooth=True), input_size=NET, act="leaky",
                                max_batch=MAX_BATCH)
    cropper = ctd_b200.RegionCropper(max_batch=MAX_BATCH)
    try:
        blocks = blocks_of(det, pages)
        items = list(zip(pages, blocks))
        cuda_items = [(torch.from_numpy(p).cuda(), b) for p, b in items]
        torch.cuda.synchronize()
        if args.profile:
            line["profile"] = profile(cropper, items, cuda_items)
        else:
            arms = [("b", "get_transformed_regions_per_block", items), ("host", "crop_stream", items),
                    ("device", "crop_stream_device_results", items),
                    ("device", "crop_stream_device_results_cuda_pages", cuda_items)]
            for arm, name, its in arms:
                run_arm(det, cropper, its, arm)
                t0 = time.perf_counter()
                r1 = run_arm(det, cropper, its, arm)
                r2 = run_arm(det, cropper, its, arm)
                dt = time.perf_counter() - t0
                line["arms"][name] = {
                    "pages_per_s": round(2 * len(its) / dt, 2), "lines_per_s": round((r1[0] + r2[0]) / dt, 1),
                    "crop_mpx_per_s": round((r1[1] + r2[1]) / dt / 1e6, 2), "lines_per_pass": r1[0],
                    "crop_mpx_per_pass": round(r1[1] / 1e6, 2)}
                print(name, line["arms"][name], flush=True)
    finally:
        cropper.close()
        det.close()
    line["card_after"] = card()
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "crop_bench%s.json" % ("_profile" if args.profile else "")), "w") as f:
            f.write(json.dumps(line, indent=1))


if __name__ == "__main__":
    main()
