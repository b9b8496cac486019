"""Throughput of PNG files encoded on the GPU (`ctd_b200.PngEncoder`, csrc/png.cu) and of `model2annotations`,
which writes every page and its refined mask as PNGs.

Workload: the 64 seeded synthetic pages of scripts/pages_bench.py (1654x1170, 1170x1654, 2048x1446, 1200x800 and
1024x1024) and their refined masks (REFINEMASK_ANNOTATION, keep_undetected_mask, the 1024 net).

Arms (each run once to warm up, then timed `--reps` times; the median is reported):
  1. encode alone: Mpx/s of PngEncoder.encode in batches of 16 (numpy pages in, files on the host out), for the pages
     and for the masks, against cv2.imencode('.png') on one host thread and on --threads host threads;
  2. model2annotations on the pages written as baseline JPEG files (quality 90, 4:2:0, as scripts/jpeg_bench.py
     makes them): "before" is the page-by-page writer (cv2.imread, detect_stream, write_annotations with cv2's PNG
     encode), "after" is `annotations.model2annotations` (GPU JPEG decode, device-results stream, GPU PNG encode).
     Pages/s and the caller thread's CPU ms per page; the two output directories must be identical.

    python scripts/png_bench.py [--out DIR] [--reps 3] [--threads 16]

Prints one JSON line, with the card's name and power limit."""
import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

NET = 1024
BATCH = 16


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t)
    return statistics.median(ts)


def imencode(img):
    import cv2
    return cv2.imencode(".png", img)[1]


def encode_all(enc, imgs):
    out = []
    for i in range(0, len(imgs), BATCH):
        out += enc.encode(imgs[i:i + BATCH])
    return out


def before(det, paths, out_dir):
    """the page-by-page writer: cv2 reads, the stream detects, write_annotations writes with cv2"""
    from ctd_b200 import annotations
    from ctd_b200.inference import REFINEMASK_ANNOTATION
    from collections import deque
    os.makedirs(out_dir, exist_ok=True)
    read = deque()

    def imgs():
        for p in paths:
            read.append(annotations.imread(p))
            yield read[-1]
    for p, (_m, refined, blks) in zip(paths, det.detect_stream(imgs(), refine_mode=REFINEMASK_ANNOTATION,
                                                               keep_undetected_mask=True)):
        annotations.write_annotations(out_dir, os.path.basename(p), read.popleft(), refined, blks)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=min(16, os.cpu_count() or 1))
    args = ap.parse_args()
    import cv2
    import torch
    import ctd_b200
    from ctd_b200 import annotations
    from ctd_b200.inference import REFINEMASK_ANNOTATION
    from oracle import synth
    from pages_bench import card, workload
    if not torch.cuda.is_available():
        raise SystemExit("png_bench.py measures the GPU encoder: no GPU visible")
    pages = workload(64)
    ck = synth.make_checkpoint(0, smooth=True)
    det = ctd_b200.TextDetector(ck, input_size=NET, act="leaky", max_batch=8)
    tmp = tempfile.mkdtemp(prefix="png_bench_")
    line = {"card": card(), "pages": len(pages), "arms": {}}
    try:
        masks = [r[1] for r in det.detect_stream(pages, refine_mode=REFINEMASK_ANNOTATION, keep_undetected_mask=True)]
        enc = ctd_b200.PngEncoder(0)
        try:
            for name, imgs in (("pages", pages), ("masks", masks)):
                mpx = sum(i.shape[0] * i.shape[1] for i in imgs) / 1e6
                got = encode_all(enc, imgs)
                assert all(np.array_equal(g, imencode(i)) for g, i in zip(got, imgs)), "GPU encode differs from cv2"
                t_gpu = timed(lambda: encode_all(enc, imgs), args.reps)
                t_cpu1 = timed(lambda: [imencode(i) for i in imgs], args.reps)
                with ThreadPoolExecutor(args.threads) as ex:
                    t_cpun = timed(lambda: list(ex.map(imencode, imgs)), args.reps)
                line["arms"]["encode_" + name] = {
                    "mpx": round(mpx, 1), "mb_png": round(sum(g.size for g in got) / 1e6, 2),
                    "gpu_batch16_mpx_s": round(mpx / t_gpu, 1), "cv2_1thread_mpx_s": round(mpx / t_cpu1, 1),
                    "cv2_%dthreads_mpx_s" % args.threads: round(mpx / t_cpun, 1),
                    "gpu_ms_per_image": round(t_gpu / len(imgs) * 1e3, 3),
                    "cv2_1thread_ms_per_image": round(t_cpu1 / len(imgs) * 1e3, 3)}
        finally:
            enc.close()
        src = os.path.join(tmp, "src")
        os.makedirs(src)
        for i, p in enumerate(pages):
            cv2.imwrite(os.path.join(src, "page%02d.jpg" % i), p, [cv2.IMWRITE_JPEG_QUALITY, 90,
                                                                   cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                                                   cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420])
        paths = annotations.find_all_imgs(src, abs_path=True)

        def run(kind, k):
            out_dir = os.path.join(tmp, "%s%d" % (kind, k))
            t0, c0 = time.perf_counter(), time.thread_time()
            if kind == "before":
                before(det, paths, out_dir)
            else:
                annotations.model2annotations(None, src, out_dir, detector=det)
            return time.perf_counter() - t0, time.thread_time() - c0, out_dir

        runs = {"before": [], "after": []}
        for k in range(args.reps + 1):          # alternate the two; the first pass of each is the warm-up
            for kind in ("before", "after"):
                r = run(kind, k)
                if k:
                    runs[kind].append(r)
        for kind, rs in runs.items():
            wall = statistics.median(r[0] for r in rs)
            cpu = statistics.median(r[1] for r in rs)
            line["arms"]["model2annotations_" + kind] = {"pages_s": round(len(paths) / wall, 1),
                                                         "caller_cpu_ms_per_page": round(cpu / len(paths) * 1e3, 2)}
        a, b = runs["before"][-1][2], runs["after"][-1][2]
        same = sorted(os.listdir(a)) == sorted(os.listdir(b)) and all(
            open(os.path.join(a, f), "rb").read() == open(os.path.join(b, f), "rb").read() for f in os.listdir(a))
        line["arms"]["identical"] = bool(same)
        assert same, "model2annotations' files differ from the page-by-page writer's"
    finally:
        det.close()
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "png_bench.json"), "w") as f:
            f.write(json.dumps(line, indent=1))


if __name__ == "__main__":
    main()
