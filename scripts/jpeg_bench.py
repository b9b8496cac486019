"""Throughput of JPEG pages decoded on the GPU (`ctd_b200.JpegDecoder`, csrc/jpeg.cu) and of a detection stream fed
with encoded files.

Workload: the 64 seeded synthetic pages of scripts/pages_bench.py (1654x1170, 1170x1654, 2048x1446, 1200x800 and
1024x1024), encoded once with cv2 at quality 90, 4:2:0, plus the golden scan tests/golden/AisazuNihaIrarenai-003.jpg.

Arms (each run once to warm up, then timed `--reps` times; the median is reported):
  1. decode alone: Mpx/s of JpegDecoder.decode in batches of 16 (the time ends when decode returns: its pages are
     complete), against cv2.imdecode on one host thread and on --threads host threads;
  2. detect_stream(cv2.imdecode(f) for f in files): decoding on the caller thread;
  3. detect_stream(files): the encoded files, decoded on the GPU batch by batch.
For arms 2 and 3: pages/s and the caller thread's CPU time per page (time.thread_time); their results must be
identical (masks, mask_refined, blocks).  --sub-bits: also time arm 1 at these subsequence lengths.

    python scripts/jpeg_bench.py [--out DIR] [--profile] [--sub-bits 256,1024,4096]

--profile: a separate run under torch.profiler (CUDA activity) of one decode of every file in batches of 16: device
microseconds per page of each decode kernel and the bytes each one must move.  Prints one JSON line either way."""
import argparse
import json
import os
import statistics
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

GOLDEN = os.path.join(ROOT, "tests", "golden", "AisazuNihaIrarenai-003.jpg")
NET = 1024
BATCH = 16


def files():
    import cv2
    from pages_bench import workload
    out = []
    for p in workload(64):
        ok, e = cv2.imencode(".jpg", p, [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                         cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420])
        out.append(e.tobytes())
    out.append(open(GOLDEN, "rb").read())
    return out


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
    ap.add_argument("--threads", type=int, default=min(16, os.cpu_count() or 1))
    ap.add_argument("--sub-bits", default="")
    args = ap.parse_args()
    import torch
    import ctd_b200
    from oracle import synth
    from pages_bench import card
    if not torch.cuda.is_available():
        raise SystemExit("jpeg_bench.py measures the GPU decoder: no GPU visible")
    fs = files()
    mpx = sum(i["height"] * i["width"] for i in map(ctd_b200.jpeg_probe, fs)) / 1e6
    line = {"card": card(), "files": len(fs), "mpx": round(mpx, 2), "mb_encoded": round(sum(map(len, fs)) / 1e6, 2),
            "arms": {}}
    if args.profile:
        line["profile"] = profile(fs)
        return emit(line, args)
    dec = ctd_b200.JpegDecoder(0)
    try:
        got = decode_all(dec, fs)
        assert all(isinstance(g, torch.Tensor) for g in got), dec.last_status
        assert all(np.array_equal(g.cpu().numpy(), imdecode(f)) for g, f in zip(got, fs)), "GPU decode differs from cv2"
        del got
        t_gpu = timed(lambda: decode_all(dec, fs), args.reps)
    finally:
        dec.close()
    t_cpu1 = timed(lambda: [imdecode(f) for f in fs], args.reps)
    with ThreadPoolExecutor(args.threads) as ex:
        t_cpun = timed(lambda: list(ex.map(imdecode, fs)), args.reps)
    line["arms"]["decode"] = {"gpu_batch16_mpx_s": round(mpx / t_gpu, 1), "cv2_1thread_mpx_s": round(mpx / t_cpu1, 1),
                              "cv2_%dthreads_mpx_s" % args.threads: round(mpx / t_cpun, 1),
                              "gpu_ms_per_page": round(t_gpu / len(fs) * 1e3, 3),
                              "cv2_1thread_ms_per_page": round(t_cpu1 / len(fs) * 1e3, 3)}
    for sb in [int(x) for x in args.sub_bits.split(",") if x]:
        d = ctd_b200.JpegDecoder(0, subsequence_bits=sb)
        try:
            line["arms"]["decode"]["gpu_sub%d_mpx_s" % sb] = round(mpx / timed(lambda: decode_all(d, fs), args.reps), 1)
        finally:
            d.close()
    # arms 2 and 3: the stream
    ck = synth.make_checkpoint(0, smooth=True)
    det = ctd_b200.TextDetector(ck, input_size=NET, act="leaky", max_batch=BATCH)
    try:
        res = {}

        def stream(encoded):
            t0, c0 = time.perf_counter(), time.thread_time()
            src = fs if encoded else (imdecode(f) for f in fs)
            out = list(det.detect_stream(src))
            return out, time.perf_counter() - t0, time.thread_time() - c0

        for name, enc in (("stream_host_decode", False), ("stream_encoded", True)):
            stream(enc)
            runs = [stream(enc) for _ in range(args.reps)]
            wall = statistics.median(r[1] for r in runs)
            cpu = statistics.median(r[2] for r in runs)
            res[name] = runs[-1][0]
            line["arms"][name] = {"pages_s": round(len(fs) / wall, 1), "caller_cpu_ms_per_page": round(cpu / len(fs) * 1e3, 2)}
        same = all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and
                   [vars(x) for x in a[2]].__repr__() == [vars(x) for x in b[2]].__repr__()
                   for a, b in zip(res["stream_host_decode"], res["stream_encoded"]))
        line["arms"]["identical"] = bool(same)
        assert same, "the two streams differ"
    finally:
        det.close()
    emit(line, args)


def emit(line, args):
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "jpeg_bench%s.json" % ("_profile" if args.profile else "")), "w") as f:
            f.write(json.dumps(line, indent=1))


KERNELS = ["jpeg_sync_kernel", "jpeg_scan_kernel", "jpeg_write_kernel", "jpeg_idct_kernel", "jpeg_color_kernel"]


def profile(fs):
    import torch
    import ctd_b200
    dec = ctd_b200.JpegDecoder(0)
    try:
        decode_all(dec, fs)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            decode_all(dec, fs)
            torch.cuda.synchronize()
    finally:
        dec.close()
    t = {k: [0.0, 0] for k in KERNELS + ["memcpy HtoD", "memset"]}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        for k in t:
            if k in ev.name or (k == "memcpy HtoD" and "HtoD" in ev.name) or (k == "memset" and "Memset" in ev.name):
                t[k][0] += ev.time_range.elapsed_us()
                t[k][1] += 1
                break
    infos = [ctd_b200.jpeg_probe(f) for f in fs]
    px = sum(i["height"] * i["width"] for i in infos)
    ecs = sum(i["ecs_bytes"] for i in infos)
    blocks = sum(-(-i["frame_height"] // 16) * -(-i["frame_width"] // 16) * 6 for i in infos)
    # bytes each kernel must move at least: the sync rounds read the scan bits (per round), the write pass reads the
    # bits and writes the coefficients, the IDCT reads coefficients and writes planes, the colour pass reads the
    # planes (Y + 2 quarter-size chroma) and writes BGR
    need = {"jpeg_sync_kernel": ecs, "jpeg_scan_kernel": 0, "jpeg_write_kernel": ecs + blocks * 128,
            "jpeg_idct_kernel": blocks * (128 + 64), "jpeg_color_kernel": blocks * 64 + px * 3}
    out = {}
    for k, (us, cnt) in t.items():
        b = need.get(k)
        out[k] = {"launches": cnt, "device_us_per_page": round(us / len(fs), 2)}
        if b:
            out[k]["bytes_per_page"] = int(b / len(fs))
            out[k]["gb_per_s"] = round(b / (us * 1e-6) / 1e9, 1) if us > 0 else None
    return out


if __name__ == "__main__":
    main()
