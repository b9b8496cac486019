"""Post-processing of float16 network outputs: `PostProcessor(half=True).postprocess_stream` on the same outputs as
float16, as float32, and as `.float()` then float32 (what users of an fp16 network had to do before), and the ingest
kernel's time and bytes for f16 and f32 batches.

Workload: 16 seeded net-sized 1024x1024 pages, input_size 1024, max_batch 16.  The outputs are `TextDetBase(half=True)`
on the host-letterboxed pages, as float16 CUDA tensors, and their float32 copies, all made before any timed region;
each stream item is a per-page slice.  The arms alternate run by run (`--runs` each, after one warm-up each), each
streaming the 16 pages `--repeat` times; the `.float()` arm converts every page's three maps inside the timed stream.

The ingest kernel (`gather_outputs_kernel`): mean device time per batch from torch.profiler in a separate pass per
dtype, and the bytes it moves per batch from the shapes (per page: mask, channel 0 of lines_map and the A rows of blks
read at the element size, the u8 mask, u8 bitmap, f32 lines plane and f32 workspace blks rows written), against the H100
SXM data-sheet HBM3 bandwidth, 3.35 TB/s.

    python scripts/postprocess_f16_bench.py [--repeat 4] [--runs 3]

Prints one JSON line, with the card's name and power limit read in the same run."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from postprocess_bench import HBM_BYTES_PER_S, MAX_BATCH, NET, ingest_kernel_ms, pages_of, time_stream  # noqa: E402
from stream_regions_bench import card  # noqa: E402


def ingest_bytes(blks, n, esz):
    """bytes gather_outputs_kernel reads and writes for n pages whose maps have esz-byte elements"""
    from ctd_b200.postprocess import workspace_rows
    _n, a, no = blks.shape
    px = NET * NET
    return n * (px * esz * 2 + a * no * esz + px + px + px * 4 + workspace_rows(NET, NET) * no * 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=4, help="passes over the 16 pages per timed stream")
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    import ctd_b200
    from ctd_b200.inference import letterbox
    from util import get_checkpoint, page_to_net_input
    if not torch.cuda.is_available():
        raise SystemExit("postprocess_f16_bench.py measures on the GPU; no CUDA device is visible")
    base = ctd_b200.TextDetBase(get_checkpoint(0, True), max_batch=MAX_BATCH, max_size=NET, half=True)
    post = ctd_b200.PostProcessor(input_size=NET, max_batch=MAX_BATCH, half=True)
    out = {"card": card(), "input_size": NET, "max_batch": MAX_BATCH, "repeat": args.repeat}
    try:
        pages = pages_of("net")
        boxed = np.stack([letterbox(p, (NET, NET))[0] for p in pages])
        o16 = base(page_to_net_input(boxed).cuda().half())
        o32 = tuple(t.float() for t in o16)
        torch.cuda.synchronize()
        items16 = [(p, o16[0][i], o16[1][i], o16[2][i]) for i, p in enumerate(pages)] * args.repeat
        items32 = [(p, o32[0][i], o32[1][i], o32[2][i]) for i, p in enumerate(pages)] * args.repeat

        def converted():
            for p, b, m, ln in items16:
                yield p, b.float(), m.float(), ln.float()

        arms = {"f16_pages_s": lambda: post.postprocess_stream(items16),
                "f32_pages_s": lambda: post.postprocess_stream(items32),
                "float_then_f32_pages_s": lambda: post.postprocess_stream(converted())}
        for name, fn in arms.items():
            time_stream(fn, 0)   # warm-up
        for _ in range(args.runs):
            for name, fn in arms.items():
                out.setdefault(name, []).extend(time_stream(fn, 1))
        for dt, items, esz in (("f16", items16, 2), ("f32", items32, 4)):
            ms, launches = ingest_kernel_ms(post, items)
            nbytes = ingest_bytes(o16[0], MAX_BATCH, esz)
            r = {"ms_per_batch": ms, "launches_profiled": launches, "bytes_per_batch": nbytes}
            if ms:
                r["bytes_per_s"] = nbytes / (ms / 1000.0)
                r["share_of_3_35_TBps"] = nbytes / (ms / 1000.0) / HBM_BYTES_PER_S
            out["ingest_" + dt] = r
    finally:
        base.close()
        post.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
