"""Throughput of the detector's post-processing on a caller's network outputs: `PostProcessor.postprocess_stream`
(ctd_submit_outputs) against `TextDetector.detect_stream` (ctd_submit_pages: the same work plus the letterbox and the
forward) on the same pages.

Workloads, input_size 1024, max_batch 16: (a) 16 seeded net-sized 1024x1024 pages, (b) 16 pages of the any-size mix of
scripts/stream_regions_bench.py.  The network outputs are those of `TextDetBase` on the host-letterboxed pages (float32
CUDA tensors, one batched forward per workload, made before any timed region); each stream item is a per-page slice
`blks[i], mask[i], lines_map[i]` of them, read where it is.  Every arm streams the workload `--repeat` times in one
stream (so two batches are in flight), once to warm up and then `--runs` times timed; the time ends when the last
result is in the caller's hands.

Also reported:
  * the ingest kernel (`gather_outputs_kernel`): its mean device time per batch from torch.profiler (CUDA activity, in a
    separate pass after the timed ones) and the bytes it moves per batch, computed here from the shapes: per page the
    mask, channel 0 of lines_map and the A rows of blks read, and the u8 mask, the u8 bitmap, the f32 lines plane and the
    workspace's blks rows written.  Its achieved bytes/s is given against the H100 SXM data-sheet HBM3 bandwidth,
    3.35 TB/s;
  * the oracle's CPU restatement of the same stages (tests/pages_ref.py on oracle/postproc_ref.py: torch CPU NMS,
    numpy / cv2 mask, DB boxes, group_output, refine_mask), timed on `--oracle-pages` pages of each workload.  It is a
    restatement written for this project's tests, not the reference's own code, and its time is labelled as such.

    python scripts/postprocess_bench.py [--repeat 4] [--runs 3] [--oracle-pages 2]

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


def pages_of(kind):
    from oracle import synth
    if kind == "net":
        return [synth.structured_page(20_000 + i, NET, NET) for i in range(MAX_BATCH)]
    return [synth.structured_page(21_000 + i, *SIZES[i % len(SIZES)]) for i in range(MAX_BATCH)]


def outputs_of(base, pages):
    import numpy as np
    from ctd_b200.inference import letterbox
    from util import page_to_net_input
    boxed = np.stack([letterbox(p, (NET, NET))[0] for p in pages])
    return base(page_to_net_input(boxed).cuda())


def ingest_bytes(blks, n):
    """bytes gather_outputs_kernel reads and writes for n pages of these outputs (see the module docstring)"""
    from ctd_b200.postprocess import workspace_rows
    _n, a, no = blks.shape
    px = NET * NET
    read = px * 4 + px * 4 + a * no * 4
    write = px + px + px * 4 + workspace_rows(NET, NET) * no * 4
    return n * (read + write)


def time_stream(fn, runs):
    import torch
    for _ in fn():   # warm-up
        pass
    torch.cuda.synchronize()
    best = []
    for _ in range(runs):
        t0 = time.perf_counter()
        k = sum(1 for _ in fn())
        torch.cuda.synchronize()
        best.append(k / (time.perf_counter() - t0))
    return best


def ingest_kernel_ms(post, items):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in post.postprocess_stream(items):
            pass
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events() if "gather_outputs_kernel" in e.name]
    return (sum(times) / len(times) / 1000.0, len(times)) if times else (None, 0)


def oracle_s_per_page(pages, blks, mask, lines, k):
    from ctd_b200.inference import letterbox_geometry
    from oracle import textblock_ref
    from pages_ref import postprocess_page_any_size
    t0 = time.perf_counter()
    for i in range(k):
        p, b, m, ln = pages[i], blks[i].cpu().numpy(), mask[i, 0].cpu().numpy(), lines[i].cpu().numpy()
        unpad = letterbox_geometry(p.shape[:2], (NET, NET))[1][::-1]
        postprocess_page_any_size(p.copy(), (NET, NET), unpad, b, m, ln, textblock_ref.group_output)
    return (time.perf_counter() - t0) / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=4, help="passes over the 16 pages per timed stream")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--oracle-pages", type=int, default=2)
    args = ap.parse_args()
    import torch
    import ctd_b200
    from util import get_checkpoint
    if not torch.cuda.is_available():
        raise SystemExit("postprocess_bench.py measures on the GPU; no CUDA device is visible")
    ck = get_checkpoint(0, True)
    det = ctd_b200.TextDetector(ck, input_size=NET, act="leaky", max_batch=MAX_BATCH)
    base = ctd_b200.TextDetBase(ck, max_batch=MAX_BATCH, max_size=NET)
    post = ctd_b200.PostProcessor(input_size=NET, max_batch=MAX_BATCH)
    out = {"card": card(), "input_size": NET, "max_batch": MAX_BATCH, "repeat": args.repeat}
    try:
        for kind in ("net", "mix"):
            pages = pages_of(kind)
            blks, mask, lines = outputs_of(base, pages)
            torch.cuda.synchronize()
            items = [(p, blks[i], mask[i], lines[i]) for i, p in enumerate(pages)] * args.repeat
            imgs = pages * args.repeat
            r = {}
            # alternate the arms run by run, so both see the same state of a shared machine
            for _ in range(args.runs):
                r.setdefault("postprocess_stream_pages_s", []).extend(
                    time_stream(lambda: post.postprocess_stream(items), 1))
                r.setdefault("detect_stream_pages_s", []).extend(time_stream(lambda: det.detect_stream(imgs), 1))
            ms, launches = ingest_kernel_ms(post, items)
            nbytes = ingest_bytes(blks, MAX_BATCH)
            r["ingest_kernel_ms_per_batch"] = ms
            r["ingest_kernel_launches_profiled"] = launches
            r["ingest_bytes_per_batch"] = nbytes
            if ms:
                r["ingest_bytes_per_s"] = nbytes / (ms / 1000.0)
                r["ingest_share_of_3_35_TBps"] = nbytes / (ms / 1000.0) / HBM_BYTES_PER_S
            r["oracle_cpu_restatement_s_per_page"] = oracle_s_per_page(pages, blks, mask, lines, args.oracle_pages)
            out[kind] = r
    finally:
        det.close()
        post.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
