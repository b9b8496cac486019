"""Cost of the detector's pre-processing on the GPU (`ctd_preprocess_pages`, preprocess.py) and of
`NetworkDetector(TextDetBase)` against `TextDetector`.

Workload: 16 pages of the any-size mix of scripts/stream_regions_bench.py, input_size 1024, max_batch 16.

  * the kernel (`letterbox_tensor_kernel`): its mean device time per 16-page batch from torch.profiler (CUDA activity,
    a separate pass), in f32 and f16, and the bytes it moves per batch, computed here from the shapes: the output
    (16 x 3 x 1024 x 1024 elements) written and every source page read once.  Its achieved bytes/s is given against
    the H100 SXM data-sheet HBM3 bandwidth, 3.35 TB/s;
  * `Preprocessor.preprocess_batch` pages/s from numpy pages and from CUDA pages (the time ends when the tensor is
    complete on the device), against the oracle's CPU restatement of the reference's `preprocess_img`
    (oracle/preprocess_ref.py, cv2 + numpy, device='cuda': the upload included), page by page;
  * `NetworkDetector(TextDetBase).detect_stream` against `TextDetector.detect_stream` on the same numpy pages
    (`--repeat` passes over the 16 pages per stream), alternated run by run, `--runs` runs each.

    python scripts/preprocess_bench.py [--repeat 4] [--runs 3] [--oracle-pages 16]

Prints one JSON line, with the card's name and power limit read in the same run."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from stream_regions_bench import SIZES, card  # noqa: E402

NET = 1024
MAX_BATCH = 16
HBM_BYTES_PER_S = 3.35e12


def kernel_ms(pre, pages, half, reps=20):
    import torch
    from torch.profiler import ProfilerActivity, profile
    pre.run(pages, half=half)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            pre.run(pages, half=half)
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events() if "letterbox_tensor_kernel" in e.name]
    return (sum(times) / len(times) / 1000.0, len(times)) if times else (None, 0)


def pages_per_s(fn, n_pages, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return n_pages * reps / (time.perf_counter() - t0)


def stream_pages_s(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    k = sum(1 for _ in fn())
    torch.cuda.synchronize()
    return k / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=4, help="passes over the 16 pages per timed stream")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--oracle-pages", type=int, default=16)
    args = ap.parse_args()
    import torch
    import ctd_b200
    from oracle import preprocess_ref, synth
    from util import get_checkpoint
    if not torch.cuda.is_available():
        raise SystemExit("preprocess_bench.py measures on the GPU; no CUDA device is visible")
    pages = [synth.structured_page(21_000 + i, *SIZES[i % len(SIZES)]) for i in range(MAX_BATCH)]
    out = {"card": card(), "input_size": NET, "max_batch": MAX_BATCH, "pages": [list(p.shape[:2]) for p in pages]}
    pre = ctd_b200.Preprocessor(NET, max_batch=MAX_BATCH)
    try:
        cuda_pages = [torch.from_numpy(p).cuda() for p in pages]
        src_bytes = sum(p.size for p in pages)
        for name, half in (("f32", False), ("f16", True)):
            ms, launches = kernel_ms(pre, cuda_pages, half)
            nbytes = MAX_BATCH * 3 * NET * NET * (2 if half else 4) + src_bytes
            r = {"kernel_ms_per_batch": ms, "launches_profiled": launches, "bytes_per_batch": nbytes}
            if ms:
                r["bytes_per_s"] = nbytes / (ms / 1000.0)
                r["share_of_3_35_TBps"] = nbytes / (ms / 1000.0) / HBM_BYTES_PER_S
            out["kernel_" + name] = r
        out["preprocess_batch_numpy_pages_s"] = pages_per_s(lambda: pre.preprocess_batch(pages), MAX_BATCH, 10)
        out["preprocess_batch_cuda_pages_s"] = pages_per_s(lambda: pre.preprocess_batch(cuda_pages), MAX_BATCH, 20)
        k = args.oracle_pages
        t0 = time.perf_counter()
        for i in range(k):
            preprocess_ref.preprocess_img(pages[i % len(pages)], (NET, NET), 'cuda')
        torch.cuda.synchronize()
        out["oracle_cpu_preprocess_img_pages_s"] = k / (time.perf_counter() - t0)
    finally:
        pre.close()
    ck = get_checkpoint(0, True)
    det = ctd_b200.TextDetector(ck, input_size=NET, act="leaky", max_batch=MAX_BATCH)
    base = ctd_b200.TextDetBase(ck, max_batch=MAX_BATCH, max_size=NET)
    nd = ctd_b200.NetworkDetector(base, NET, max_batch=MAX_BATCH)
    try:
        imgs = pages * args.repeat
        for fn in (lambda: nd.detect_stream(imgs), lambda: det.detect_stream(imgs)):   # warm-up
            for _ in fn():
                pass
        r = {}
        for _ in range(args.runs):   # alternated run by run
            r.setdefault("network_detector_pages_s", []).append(stream_pages_s(lambda: nd.detect_stream(imgs)))
            r.setdefault("text_detector_pages_s", []).append(stream_pages_s(lambda: det.detect_stream(imgs)))
        out["detect_stream"] = r
    finally:
        det.close()
        nd.close()
        base.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
