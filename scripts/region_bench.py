"""Throughput of the text-line crops: `TextDetector.get_transformed_regions` on the blocks the detector finds on
synthetic 1024 x 1024 pages, against the same crops through the cv2 restatement of the reference method
(tests/region_ref.py) on the host's CPU cores.

Reports, per page: the host-clock time of the blocking call (plan + page upload + launch + copy back), the kernel's
device time (torch.profiler CUDA activity, in a separate pass), lines/s and output Mpx/s, the CPU baseline's time with
the thread count cv2 used, and the card's name and power limit read in the same run.  Prints one JSON line; with
--out also writes it to a file.

    python scripts/region_bench.py --pages 16 --textheight 48 --reps 20
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # the measurement still stands; say why the limit is missing
        q = "unavailable (%s)" % e
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=16)
    ap.add_argument("--textheight", type=int, default=48)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import cv2
    import torch
    import ctd_b200
    from oracle import synth
    import region_ref

    det = ctd_b200.TextDetector(synth.make_checkpoint(0, smooth=True), input_size=1024, act="leaky")
    th = a.textheight
    pages, blocks = [], []
    for s in range(a.pages):
        page = synth.structured_page(5000 + s, 1024, 1024)
        _, _, blk_list = det(page.copy())
        keep = []   # blocks on which the reference raises for some line are left out of the workload
        for blk in blk_list:
            try:
                for i in range(len(blk.lines)):
                    region_ref.transformed_region(blk, page, i, th)
                keep.append(blk)
            except Exception:
                pass
        pages.append(page)
        blocks.append(keep)
    n_lines = sum(len(b.lines) for bl in blocks for b in bl)
    crops = [det.get_transformed_regions(p, bl, th) for p, bl in zip(pages, blocks)]   # warm-up + output check
    n_px = sum(c.shape[0] * c.shape[1] for page in crops for bc in page for c in bc)
    for p, bl, got in zip(pages, blocks, crops):
        for blk, g in zip(bl, got):
            for i, c in enumerate(g):
                assert np.array_equal(c, region_ref.transformed_region(blk, p, i, th))

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.reps):
        for p, bl in zip(pages, blocks):
            det.get_transformed_regions(p, bl, th)
    gpu_s = (time.perf_counter() - t0) / (a.reps * a.pages)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.reps):
            for p, bl in zip(pages, blocks):
                det.get_transformed_regions(p, bl, th)
        torch.cuda.synchronize()
    k_us = [e.device_time for e in prof.events() if "k_warp_regions" in e.name]
    kernel_s = (sum(k_us) / len(k_us) * 1e-6) if k_us else float("nan")

    cpu_reps = max(1, a.reps // 4)
    t0 = time.perf_counter()
    for _ in range(cpu_reps):
        for p, bl in zip(pages, blocks):
            for blk in bl:
                for i in range(len(blk.lines)):
                    region_ref.transformed_region(blk, p, i, th)
    cpu_s = (time.perf_counter() - t0) / (cpu_reps * a.pages)

    name, limit = card()
    res = {
        "workload": "%d synthetic 1024x1024 pages, textheight %d" % (a.pages, th),
        "lines_per_page": n_lines / a.pages, "output_mpx_per_page": n_px / a.pages / 1e6,
        "gpu_ms_per_page": gpu_s * 1e3, "kernel_us_per_page": kernel_s * 1e6, "kernel_launches_seen": len(k_us),
        "gpu_lines_per_s": n_lines / a.pages / gpu_s, "gpu_mpx_per_s": n_px / a.pages / gpu_s / 1e6,
        "kernel_mpx_per_s": n_px / a.pages / kernel_s / 1e6,
        "cpu_ms_per_page": cpu_s * 1e3, "cpu_lines_per_s": n_lines / a.pages / cpu_s,
        "cpu_cores": os.cpu_count(), "cv2_threads": cv2.getNumThreads(),
        "speedup_vs_cpu": cpu_s / gpu_s, "card": name, "power_limit_and_max_sm_clock": limit,
    }
    det.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
