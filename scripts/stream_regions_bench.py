"""Throughput of "detect + OCR crops" over pages of any size: the batched stream alone, the stream followed by the
blocking per-page `get_transformed_regions`, and the stream cutting the crops itself (`detect_stream(textheight=)`,
ctd_submit_pages with a textheight: planned on the engine's worker threads, one k_warp_regions launch per batch on the
pages already in device memory).

Workload: the 64 seeded synthetic pages of scripts/pages_bench.py (oracle/synth.structured_page) at input_size 1024,
refine_mode INPAINT, textheight 48, max_batch 16.  Every arm runs the workload once to warm up, then twice timed; the
time ends when the last result is on the host.

    python scripts/stream_regions_bench.py [--out DIR] [--profile]

Arms: (a) `detect_stream`; (b) `detect_stream` + `get_transformed_regions` on every yielded page (a page on which the
reference raises for some line is cropped block by block, skipping the blocks that raise: counted as
`pages_with_raising_lines`); (c) `detect_stream(textheight=48)`.  Reported per arm: pages/s, lines/s and crop Mpx/s
(lines and crop pixels of the pass, the same for (b) and (c) up to the lines (b) has to skip).

--profile: a separate run.  Host split of one pass of (a) and (c): wall time, caller-thread time waiting in
Engine.collect and assembling the crops in Engine.collect_regions; the planner's time for every line of the pass on one
host thread.  Then one pass each of (a) and (c) under torch.profiler (CUDA activity): device time of k_warp_regions per
batch and its achieved GB/s from the crop bytes it writes (its page reads are gathers of 4 taps per pixel, mostly from
L2), and the device time of all device-to-host copies.  Prints one JSON line either way."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [(1654, 1170), (1170, 1654), (2048, 1446), (1200, 800), (1024, 1024)]
NET = 1024
TEXTHEIGHT = 48
MAX_BATCH = 16


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True)
    except OSError:
        return "unknown"
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def workload(n=64):
    from oracle import synth
    return [synth.structured_page(10_000 + i, *SIZES[i % len(SIZES)]) for i in range(n)]


def _count(crops):
    lines = px = 0
    for blk in crops:
        for c in blk:
            if c is not None:
                lines += 1
                px += c.shape[0] * c.shape[1]
    return lines, px


def run_arm(det, pages, arm):
    """one pass -> (lines cropped, crop pixels, pages with a raising line)"""
    from ctd_b200 import CtdError
    lines = px = raising = 0
    if arm == "a":
        for _m, _r, blks in det.detect_stream(pages, refine_mode=0):
            lines += sum(len(b.lines) for b in blks)
    elif arm == "b":
        for img, (_m, _r, blks) in zip(pages, det.detect_stream(pages, refine_mode=0)):
            try:
                crops = det.get_transformed_regions(img, blks, TEXTHEIGHT)
            except CtdError:
                raising += 1
                crops = []
                for b in blks:
                    try:
                        crops += det.get_transformed_regions(img, [b], TEXTHEIGHT)
                    except CtdError:
                        pass
            nl, npx = _count(crops)
            lines, px = lines + nl, px + npx
    else:
        for _m, _r, blks, crops in det.detect_stream(pages, refine_mode=0, textheight=TEXTHEIGHT):
            nl, npx = _count(crops)
            lines, px = lines + nl, px + npx
            raising += any(c is None for blk in crops for c in blk)
    return lines, px, raising


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--pages", type=int, default=64)
    args = ap.parse_args()
    import ctd_b200
    from oracle import synth
    ck = synth.make_checkpoint(0, smooth=True)
    pages = workload(args.pages)
    line = {"card": card(), "pages": len(pages), "input_size": NET, "sizes": SIZES, "textheight": TEXTHEIGHT,
            "max_batch": MAX_BATCH, "arms": {}}
    det = ctd_b200.TextDetector(ck, input_size=NET, act="leaky", max_batch=MAX_BATCH)
    try:
        if args.profile:
            line["profile"] = profile(det, pages)
        else:
            names = {"a": "detect_stream", "b": "detect_stream+get_transformed_regions",
                     "c": "detect_stream_textheight"}
            for arm in ("a", "b", "c"):
                run_arm(det, pages, arm)
                t0 = time.perf_counter()
                r1 = run_arm(det, pages, arm)
                r2 = run_arm(det, pages, arm)
                dt = time.perf_counter() - t0
                line["arms"][names[arm]] = {
                    "pages_per_s": round(2 * len(pages) / dt, 2), "lines_per_s": round((r1[0] + r2[0]) / dt, 1),
                    "crop_mpx_per_s": round((r1[1] + r2[1]) / dt / 1e6, 2), "lines_per_pass": r1[0],
                    "crop_mpx_per_pass": round(r1[1] / 1e6, 2), "pages_with_raising_lines": r1[2]}
                print(names[arm], line["arms"][names[arm]], flush=True)
    finally:
        det.close()
    line["card_after"] = card()
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "stream_regions_bench%s.json" % ("_profile" if args.profile else "")), "w") as f:
            f.write(json.dumps(line, indent=1))


def split(det, pages, arm):
    """host clock of one pass of arm (a) or (c), and the caller-thread time inside Engine.collect (waiting for the
    batch) and Engine.collect_regions (copying each page's crops out and building the per-line views), in ms"""
    eng = det.net
    t = {"collect_wait": 0.0, "collect_regions": 0.0}

    def timed(key, fn):
        def w(*a, **k):
            t0 = time.perf_counter()
            try:
                return fn(*a, **k)
            finally:
                t[key] += time.perf_counter() - t0
        return w

    eng.collect = timed("collect_wait", eng.collect)
    eng.collect_regions = timed("collect_regions", eng.collect_regions)
    try:
        t0 = time.perf_counter()
        run_arm(det, pages, arm)
        t["pass"] = time.perf_counter() - t0
    finally:
        del eng.collect, eng.collect_regions
    return {k: round(v * 1e3, 1) for k, v in t.items()}


def plan_ms(det, pages):
    """ctd_region_plan of every line of the pass on one host thread, ms (the worker runs it on its host threads)"""
    from ctd_b200 import binding, textblock
    total = 0.0
    for img, (_m, _r, blks) in zip(pages, det.detect_stream(pages, refine_mode=0)):
        rec, _keys = textblock.region_lines(blks)
        t0 = time.perf_counter()
        binding.region_plan(rec, img.shape[1], img.shape[0], TEXTHEIGHT)
        total += time.perf_counter() - t0
    return round(total * 1e3, 1)


def profile(det, pages):
    import torch
    out = {"batches": (len(pages) + MAX_BATCH - 1) // MAX_BATCH}
    for arm in ("a", "c"):
        run_arm(det, pages, arm)
        out["host_split_ms_" + arm] = split(det, pages, arm)
    out["plan_ms_one_thread"] = plan_ms(det, pages)
    for arm in ("a", "c"):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            lines, px, _r = run_arm(det, pages, arm)
            torch.cuda.synchronize()
        us, cnt, d2h_us = 0.0, 0, 0.0
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            if "k_warp_regions" in ev.name:
                us += ev.time_range.elapsed_us()
                cnt += 1
            elif "DtoH" in ev.name:
                d2h_us += ev.time_range.elapsed_us()
        out["d2h_device_ms_" + arm] = round(d2h_us / 1e3, 2)
        if arm == "c":
            b = px * 3
            out.update({"launches": cnt, "device_us": round(us, 1), "device_us_per_batch": round(us / max(cnt, 1), 1),
                        "crop_bytes": b, "lines": lines,
                        "gb_per_s": round(b / (us * 1e-6) / 1e9, 1) if us > 0 else None})
    return out


if __name__ == "__main__":
    main()
