"""Throughput of JPEG files encoded on the GPU (`ctd_b200.JpegEncoder`, csrc/jpeg_enc.cu) against cv2.imencode('.jpg').

Workload: the 64 seeded synthetic pages of scripts/pages_bench.py (1654x1170, 1170x1654, 2048x1446, 1200x800 and
1024x1024) plus the golden scan tests/golden/AisazuNihaIrarenai-003.jpg decoded by cv2: 65 BGR pages, each encoded at
cv2's defaults (quality 95, 4:2:0) and at 4:4:4 with optimised Huffman tables.

Arms (each run once to warm up, then timed `--reps` times; the median is reported, and the slowest and fastest
pass as `mpx_s_range`), per setting:
  - JpegEncoder.encode in batches of 16, from numpy pages (uploaded through the encoder's pinned staging) and from
    CUDA pages already on the device; files on the host either way;
  - cv2.imencode on one host thread, and on --threads host threads through a thread pool.
Every GPU file is checked against cv2's before anything is timed.

--profile: a separate run under torch.profiler (CUDA activity) of one encode of the CUDA pages per setting, in batches
of 16: device time per kernel and per page.

    python scripts/jpeg_encode_bench.py [--out DIR] [--reps 3] [--threads N] [--profile]

Prints one JSON line, with the card's name and power limit."""
import argparse
import json
import os
import statistics
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(ROOT)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

BATCH = 16
SETTINGS = {"default": [], "444_optimize": [7, 0x111111, 3, 1]}
KERNELS = ["jpeg_block_kernel", "jpeg_symbol_kernel", "jpeg_table_kernel", "jpeg_header_kernel", "scan_",
           "jpeg_stuff_kernel", "jpeg_copy_kernel"]


def timed(fn, reps):
    """(median, fastest, slowest) seconds of `reps` timed calls after one warm-up call"""
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t)
    return statistics.median(ts), min(ts), max(ts)


def encode_all(enc, imgs, params):
    out = []
    for i in range(0, len(imgs), BATCH):
        out += enc.encode(imgs[i:i + BATCH], params)
    return out


def pages():
    import cv2
    from pages_bench import workload
    golden = cv2.imdecode(np.fromfile(os.path.join(ROOT, "tests", "golden", "AisazuNihaIrarenai-003.jpg"), np.uint8),
                          cv2.IMREAD_COLOR)
    return workload(64) + [golden]


def profile(enc, dev, params):
    import torch
    encode_all(enc, dev, params)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        encode_all(enc, dev, params)
        torch.cuda.synchronize()
    t = {k: [0.0, 0] for k in KERNELS + ["memcpy", "memset"]}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        for k in t:
            if k in ev.name or (k in ("memcpy", "memset") and k in ev.name.lower()):
                t[k][0] += ev.time_range.elapsed_us()
                t[k][1] += 1
                break
    return {k: {"launches": c, "device_us_per_page": round(us / len(dev), 1)} for k, (us, c) in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import cv2
    import torch
    import ctd_b200
    from pages_bench import card
    if not torch.cuda.is_available():
        raise SystemExit("jpeg_encode_bench.py measures the GPU encoder: no GPU visible")
    imgs = pages()
    dev = [torch.from_numpy(p).cuda() for p in imgs]
    torch.cuda.synchronize()
    mpx = sum(p.shape[0] * p.shape[1] for p in imgs) / 1e6
    line = {"card": card(), "pages": len(imgs), "mpx": round(mpx, 1), "threads": args.threads, "settings": {}}
    enc = ctd_b200.JpegEncoder(0)
    try:
        for name, params in SETTINGS.items():
            ref = [cv2.imencode(".jpg", p, params)[1] for p in imgs]
            for src in (imgs, dev):
                got = encode_all(enc, src, params)
                assert all(np.array_equal(g, r) for g, r in zip(got, ref)), "GPU encode differs from cv2"
            if args.profile:
                line["settings"][name] = {"profile": profile(enc, dev, params)}
                continue
            t_host = timed(lambda: encode_all(enc, imgs, params), args.reps)
            t_dev = timed(lambda: encode_all(enc, dev, params), args.reps)
            t_cpu1 = timed(lambda: [cv2.imencode(".jpg", p, params) for p in imgs], args.reps)
            with ThreadPoolExecutor(args.threads) as ex:
                t_cpun = timed(lambda: list(ex.map(lambda p: cv2.imencode(".jpg", p, params), imgs)), args.reps)
            arm = lambda t: {"mpx_s": round(mpx / t[0], 1), "ms_per_page": round(t[0] / len(imgs) * 1e3, 3),
                             "mpx_s_range": [round(mpx / t[2], 1), round(mpx / t[1], 1)]}
            line["settings"][name] = {"mb_jpeg": round(sum(r.size for r in ref) / 1e6, 2),
                                      "gpu_batch16_host_pages": arm(t_host), "gpu_batch16_cuda_pages": arm(t_dev),
                                      "cv2_1thread": arm(t_cpu1), "cv2_%dthreads" % args.threads: arm(t_cpun)}
    finally:
        enc.close()
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "jpeg_encode_bench%s.json" % ("_profile" if args.profile else "")), "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
