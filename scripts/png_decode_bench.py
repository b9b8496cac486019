"""Throughput of PNG pages decoded on the GPU (`ctd_b200.PngDecoder`, csrc/png_dec.cu), of a detection stream fed
with PNG files, and of `model2annotations` on a directory of PNG pages.

Workload: the 64 seeded synthetic pages of scripts/pages_bench.py (1654x1170, 1170x1654, 2048x1446, 1200x800 and
1024x1024) as three sets of files: cv2's own PNGs (`cv2.imencode('.png')`: SUB filter, level 1, Z_RLE), PIL level 6
with adaptive filters (Paeth common), and greyscale `L` PNGs written by PIL.

Arms (each run once to warm up, then timed `--reps` times; the median is reported):
  1. decode alone, per set: Mpx/s of PngDecoder.decode in batches of 16 (the time ends when decode returns: its pages
     are complete), against cv2.imdecode on one host thread and on --threads host threads;
  2. detect_stream(cv2.imdecode(f) for f in files) against detect_stream(files) on the cv2 set: pages/s and the caller
     thread's CPU time per page; the results must be identical;
  3. model2annotations on a directory of the first 16 cv2-set pages, with PNG pages decoded by cv2 (before) and on the
     GPU (after): pages/s; the written files must be identical.

    python scripts/png_decode_bench.py [--out DIR] [--profile]

--profile: a separate run under torch.profiler (CUDA activity) of one decode of every set in batches of 16: device
microseconds per page of each decode kernel, deflate blocks and self-synchronisation rounds.  Prints one JSON line either way."""
import argparse
import io
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


def sets():
    import cv2
    from PIL import Image
    from pages_bench import workload
    pages = workload(64)

    def pil(img, mode):
        im = Image.fromarray(np.ascontiguousarray(img[..., ::-1]), "RGB").convert(mode)
        b = io.BytesIO()
        im.save(b, "PNG", compress_level=6)
        return b.getvalue()
    return {"cv2": [cv2.imencode(".png", p)[1].tobytes() for p in pages],
            "pil_level6": [pil(p, "RGB") for p in pages],
            "grey_L": [pil(p, "L") for p in pages]}


def imdecode(f):
    import cv2
    return cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR)


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t)
    return statistics.median(ts)


def decode_all(dec, fs):
    out = []
    for i in range(0, len(fs), BATCH):
        out += dec.decode(fs[i:i + BATCH])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=8)
    args = ap.parse_args()
    import torch
    import ctd_b200
    from ctd_b200 import annotations
    from oracle import synth
    from pages_bench import card
    if not torch.cuda.is_available():
        raise SystemExit("png_decode_bench.py measures the GPU decoder: no GPU visible")
    fsets = sets()
    line = {"card": card(), "arms": {}}
    if args.profile:
        line["profile"] = {name: profile(fs) for name, fs in fsets.items()}
        return emit(line, args)
    dec = ctd_b200.PngDecoder(0)
    try:
        for name, fs in fsets.items():
            mpx = sum(i["height"] * i["width"] for i in map(ctd_b200.png_probe, fs)) / 1e6
            got = decode_all(dec, fs)
            assert all(isinstance(g, torch.Tensor) for g in got), dec.last_status
            assert all(np.array_equal(g.cpu().numpy(), imdecode(f)) for g, f in zip(got, fs)), "GPU decode differs"
            del got
            t_gpu = timed(lambda: decode_all(dec, fs), args.reps)
            t_cpu1 = timed(lambda: [imdecode(f) for f in fs], args.reps)
            with ThreadPoolExecutor(args.threads) as ex:
                t_cpun = timed(lambda: list(ex.map(imdecode, fs)), args.reps)
            line["arms"]["decode_" + name] = {
                "files": len(fs), "mpx": round(mpx, 2), "mb_encoded": round(sum(map(len, fs)) / 1e6, 2),
                "gpu_batch16_mpx_s": round(mpx / t_gpu, 1), "cv2_1thread_mpx_s": round(mpx / t_cpu1, 1),
                "cv2_%dthreads_mpx_s" % args.threads: round(mpx / t_cpun, 1),
                "gpu_ms_per_page": round(t_gpu / len(fs) * 1e3, 3)}
    finally:
        dec.close()
    fs = fsets["cv2"]
    ck = synth.make_checkpoint(0, smooth=True)
    det = ctd_b200.TextDetector(ck, input_size=NET, act="leaky", max_batch=BATCH)
    try:
        res = {}

        def stream(encoded):
            t0, c0 = time.perf_counter(), time.thread_time()
            out = list(det.detect_stream(fs if encoded else (imdecode(f) for f in fs)))
            return out, time.perf_counter() - t0, time.thread_time() - c0

        for name, enc in (("stream_host_decode", False), ("stream_files", True)):
            stream(enc)
            runs = [stream(enc) for _ in range(args.reps)]
            res[name] = runs[-1][0]
            line["arms"][name] = {"pages_s": round(len(fs) / statistics.median(r[1] for r in runs), 1),
                                  "caller_cpu_ms_per_page": round(statistics.median(r[2] for r in runs) / len(fs) * 1e3, 2)}
        same = all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and
                   repr([vars(x) for x in a[2]]) == repr([vars(x) for x in b[2]])
                   for a, b in zip(res["stream_host_decode"], res["stream_files"]))
        line["arms"]["stream_identical"] = bool(same)
        assert same, "the two streams differ"
    finally:
        det.close()
    # model2annotations on a PNG directory: PNGs through cv2 (the JPEG decoder's fallback) against the GPU
    tmp = tempfile.mkdtemp(prefix="png_decode_bench_")
    try:
        src = os.path.join(tmp, "src")
        os.makedirs(src)
        for i, f in enumerate(fs[:16]):
            with open(os.path.join(src, "p%02d.png" % i), "wb") as fh:
                fh.write(f)
        det = ctd_b200.TextDetector(ck, input_size=NET, act="leaky", max_batch=8)
        try:
            outs = {}
            for name in ("annotations_cv2_decode", "annotations_gpu_decode"):
                if name == "annotations_cv2_decode":
                    det.png_decoder = det.jpeg_decoder   # PNG files to the JPEG decoder, which hands them to cv2
                else:
                    del det.png_decoder
                dst = os.path.join(tmp, name)

                def run():
                    shutil.rmtree(dst, ignore_errors=True)
                    annotations.model2annotations(None, src, dst, detector=det)
                line["arms"][name] = {"pages_s": round(16 / timed(run, args.reps), 1)}
                outs[name] = {n: open(os.path.join(dst, n), "rb").read() for n in sorted(os.listdir(dst))}
            same = outs["annotations_cv2_decode"] == outs["annotations_gpu_decode"]
            line["arms"]["annotations_identical"] = bool(same)
            assert same, "model2annotations wrote different files"
        finally:
            det.close()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    emit(line, args)


def emit(line, args):
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "png_decode_bench%s.json" % ("_profile" if args.profile else "")), "w") as f:
            f.write(json.dumps(line, indent=1))


KERNELS = ["png_inflate_kernel", "png_adler_kernel", "png_unfilter_kernel", "png_convert_kernel"]


def profile(fs):
    import torch
    import ctd_b200
    dec = ctd_b200.PngDecoder(0)
    try:
        blocks = rounds = 0
        for i in range(0, len(fs), BATCH):
            dec.decode(fs[i:i + BATCH])
            b, r = dec.last_stats()
            blocks, rounds = blocks + b, rounds + r
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            decode_all(dec, fs)
            torch.cuda.synchronize()
    finally:
        dec.close()
    t = {k: [0.0, 0] for k in KERNELS + ["memcpy HtoD"]}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        for k in t:
            if k in ev.name or (k == "memcpy HtoD" and "HtoD" in ev.name):
                t[k][0] += ev.time_range.elapsed_us()
                t[k][1] += 1
                break
    out = {k: {"launches": c, "device_us_per_page": round(us / len(fs), 1)} for k, (us, c) in t.items()}
    out["blocks"], out["sync_rounds"] = blocks, rounds
    out["rounds_per_chunk_upper"] = round(rounds / max(1, blocks), 2)
    return out


if __name__ == "__main__":
    main()
