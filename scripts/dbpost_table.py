#!/usr/bin/env python
"""Per-kernel table of the DB post-processing (launch_db_post: ccl_launch in csrc/postproc.cu, segrep_launch in
csrc/segrep.cu) on the benchmark's batch.

    python scripts/dbpost_table.py [--batch 16 --size 1024] [--gpu] [--lib FILE] [--json FILE]

The batch is the one bench.py measures: the synthetic checkpoint of seed 0 and structured_page(1000 + i) for i < B,
on the fp16 tensor-core engine.  One row per DB post kernel: its launches per forward, the bytes it moves per page
pixel by a model read off the kernels (below), and with --gpu its device time summed over its launches in one warmed
ctd_forward (torch.profiler CUDA activity, in a run of its own) and the modelled bytes over that time.  The memsets
enqueued on the DB post-processing's stream are a row of their own.  The header gives the card's name and power limit,
read in the same command.  --lib runs another build of libctd_b200.so (a parent's, to alternate it with this tree's).

Without --gpu the script prints the byte model only.  A library that still launches flag_scan_seg_kernel is a parent
build, and the table uses the parent's byte model for it.

Byte model, per page pixel and launch (HBM: a 16 x 1024^2 batch has 16.8 M pixels, so one int32 plane is 67 MB, over
the 50 MB L2).  Kernels whose traffic does not scale with the page area (the seams, the per-page scans, the
per-contour geometry) count 0.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# kernel name: bytes per page pixel and launch, for the kernels of this tree.  The kernels that only a parent build has
# (before the label plane was built on demand and the flag plane was dropped) stay listed, so that --lib can time one;
# where a kernel of the same name moved more bytes there, the parent's figure is in its comment.
MODEL = {
    # ccl_launch
    "ccl_local_kernel": 5.0,         # bitmap 1 in; L 4 out (parent: + keymin 4 out)
    "ccl_border_kernel": 0.0,
    "ccl_flatten_kernel": 8.0,       # L 4 in, L 4 out, a count per warp
    # ccl_number_launch: on demand only, not in a forward
    "ccl_key_kernel": 8.0,           # L 4 in, keymin atomics of one block row per component (+ its memset 4)
    # parent only
    "ccl_flatten_key_kernel": 8.0,   # L 4 in, L 4 out (+ keymin atomics of one block row per component)
    "ccl_markfirst_kernel": 4.0,     # L 4 in
    "ccl_scan_seg_kernel": 2.0,      # one flag per 2x2 block: 1 in + 1 out
    "ccl_scan_top_kernel": 0.0,
    "ccl_relabel_kernel": 8.0,       # L 4 in, labels 4 out
    # segrep_launch
    "bg_local_kernel": 5.0,          # bitmap 1 in, Lb 4 out
    "bg_border_kernel": 0.0,
    "bg_flatten_kernel": 8.0,        # Lb 4 in, 4 out
    "mark_outside_kernel": 0.0,
    "roots_kernel": 8.0,             # Lf 4 + Lb 4 in (parent: + flag 4 out)
    "flag_scan_seg_kernel": 8.0,     # parent only: flag 4 in, 4 out
    "flag_scan_top_kernel": 0.0,
    "rows_init_kernel": 7.8,         # parent only: rowmin + rowmax, n x 1000 contours x h rows x 8 B
    "assign_cid_kernel": 8.0,        # Lf 4 + Lb 4 in, cid at roots (parent: flag 4 in, cid 4 out)
    "accumulate_kernel": 14.0,       # pred 4 + Lf 4 + Lb 4 in, parent / cid at roots (+ double atomics per run)
    "tree_kernel": 0.0,              # the root list (parent: Lf 4 + Lb 4 in)
    "contour_order_kernel": 0.0,
    "contour_kernel": 0.0,
    "rows_clear_kernel": 0.0,        # the rows of each contour's y range
}
PARENT_BPP = {"ccl_local_kernel": 9.0, "roots_kernel": 12.0, "tree_kernel": 8.0}


def card():
    return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def kernel_key(name):
    m = re.search(r"\b([a-z_0-9]+_kernel)\b", name)
    return m.group(1) if m and m.group(1) in MODEL else None


def gpu_run(n, h, w, lib=None):
    import numpy as np
    import torch
    from torch.profiler import profile, ProfilerActivity
    import ctd_b200
    if lib:
        ctd_b200.binding.LIB_PATH = os.path.abspath(lib)   # read when the library is first loaded, below
    from oracle import synth
    ck = synth.make_checkpoint(0, smooth=True)
    prog = ctd_b200.compiler.compile_checkpoint(ck)
    pages = np.stack([synth.structured_page(1000 + i, h, w) for i in range(n)])
    dev = torch.from_numpy(pages).cuda()
    eng = ctd_b200.Engine(prog, max_batch=n, max_h=h, max_w=w, use_graph=False)
    try:
        for _ in range(3):
            eng.forward_device(dev.data_ptr(), n, h, w)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.forward_device(dev.data_ptr(), n, h, w)
            torch.cuda.synchronize()
    finally:
        eng.close()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    events = [ev for ev in trace.get("traceEvents", []) if ev.get("cat") in ("kernel", "gpu_memset")]
    # the DB post-processing's stream: the one its first kernel ran on
    streams = {ev.get("args", {}).get("stream") for ev in events if ev.get("cat") == "kernel" and kernel_key(ev["name"])}
    times, counts = {}, {}
    span0, span1, other_ms = None, None, 0.0
    for ev in events:
        dur = ev.get("dur", 0.0) * 1e-3
        if ev.get("cat") == "kernel":
            k = kernel_key(ev.get("name", ""))
            if k is None:
                other_ms += dur
                continue
        elif ev.get("args", {}).get("stream") in streams:
            k = "memset"
        else:
            continue
        times[k] = times.get(k, 0.0) + dur
        counts[k] = counts.get(k, 0) + 1
        t0, t1 = ev["ts"], ev["ts"] + ev.get("dur", 0.0)
        span0 = t0 if span0 is None else min(span0, t0)
        span1 = t1 if span1 is None else max(span1, t1)
    span = (span1 - span0) * 1e-3 if span0 is not None else 0.0
    return times, counts, other_ms, span, card()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=1024, help="square page size")
    ap.add_argument("--gpu", action="store_true", help="run the batch on cuda:0 and add the measured device times")
    ap.add_argument("--lib", default=None, help="with --gpu: another build of libctd_b200.so to run")
    ap.add_argument("--json", default=None, help="also write the rows to this file")
    args = ap.parse_args()
    n, h, w = args.batch, args.size, args.size
    px = n * h * w
    if not args.gpu:
        print("DB post-processing byte model per page pixel and launch (CPU model; --gpu measures the batch)")
        for k, b in MODEL.items():
            print("%-24s %6.2f" % (k, b))
        return
    times, counts, other_ms, span, cardq = gpu_run(n, h, w, lib=args.lib)
    parent = "flag_scan_seg_kernel" in counts   # a build from before the flag plane was dropped
    print("DB post-processing at %d x %d x %d (%s); %s" % (n, h, w, args.lib or "this tree", cardq))
    print("%-24s %8s %6s %8s %8s %7s" % ("kernel", "launches", "B/px", "GB", "ms", "TB/s"))
    rows = []
    tot_ms = tot_gb = 0.0
    for k in list(MODEL) + ["memset"]:
        if k not in counts:
            continue
        b = PARENT_BPP.get(k, MODEL.get(k, 0.0)) if parent else MODEL.get(k, 0.0)
        gb = b * counts[k] * px / 1e9
        ms = times[k]
        tot_ms += ms
        tot_gb += gb
        rows.append(dict(kernel=k, launches=counts[k], bytes_per_px=b, gb=gb, ms=ms))
        print("%-24s %8d %6.2f %8.3f %8.3f %7s" % (k, counts[k], b, gb, ms, "%.2f" % (gb / ms) if ms > 0 and gb > 0 else "-"))
    print("DB post total: %.3f ms device time in %d launches, %.2f GB modelled (%.2f TB/s); first start to last end "
          "%.3f ms; other kernels of the forward: %.3f ms"
          % (tot_ms, sum(counts.values()), tot_gb, tot_gb / tot_ms if tot_ms > 0 else 0.0, span, other_ms))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"shape": [n, h, w], "lib": args.lib, "card": cardq, "rows": rows, "dbpost_ms": tot_ms,
                       "span_ms": span, "other_ms": other_ms}, f, indent=1)


if __name__ == "__main__":
    main()
