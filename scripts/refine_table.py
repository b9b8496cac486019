#!/usr/bin/env python
"""Per-kernel table of refine_mask (csrc/refine_mk.cu) on the benchmark's batch.

    python scripts/refine_table.py [--batch 16 --size 1024] [--gpu | --passes] [--mode 0] [--json FILE] [--lib FILE]

The batch is the one bench.py measures: the synthetic checkpoint of seed 0 and structured_page(1000 + i) for i < B,
on the fp16 tensor-core engine.  One row per refine kernel: its launches per batch, the bytes it moves per window
pixel by a model read off the kernels (below), and with --gpu its device time summed over its launches in one warmed
ctd_submit_full + ctd_collect (torch.profiler CUDA activity, in a run of its own) and the modelled bytes over that
time.  The header gives the batch's windows (expand_textwindow(.., 16) of every block the engine returned), their
chunks and window pixels, and the card's name and power limit, read in the same command.

Without --gpu (or without a GPU) the script prints the byte model per window pixel only: the windows come from the
network's output, so their pixel count needs the engine.

--passes measures how the time of k_label_local divides among its passes, per round.  It runs the same batch on a
second build of the library, compiled with -DCTD_REFINE_PASS_CLOCKS into --passes-dir (built there by csrc/build.sh if
it holds no library yet; the shipped library is not touched), in which thread 0 of every k_label_local CTA adds the
clock64() ticks between pass boundaries to a global table.  The table printed is each pass's share of the summed CTA
ticks of the round's launch: a share of CTA residency, not of the launch's wall time.  It also counts, per round, the
word seams that runs cross (pass 1 links each to its run's first pixel; they were shared unions before) and the shared
unions of vertical and diagonal contacts in pass 2.  --lib runs --gpu on another
build of the library (a parent's, to alternate it with this tree's).

Byte model, per window pixel and launch (HBM; the window planes of a batch are ~1 GB, far over the 50 MB L2):
  k_phase0        mask (+ halo rows) 1 + image 3 in; grey 1 + pred, merged bits 0.25 out             5.25
  k_xor           mask 1 + grey 1 + image 3 in; six candidate bit planes 0.75 out                    5.75
  k_label_local   source, merged, pred bits 0.375 in; 16-bit label out 2                             2.375
  k_merge         source, merged bits 0.25 (labels are read at run starts only)                      0.25
  k_dilate        merged bits (+ halo) in, tmp bits out (inpaint mode only)                          0.25
  k_or            merged bits (the set pixels' atomics on mask_refined are not counted)              0.125
The bit planes hold 32 pixels per 4-byte word: 0.125 B per pixel and plane.  The per-window kernels (k_decide1,
k_decide2), k_union_border (the first row of each chunk) and the kernels that walk the per-chunk root lists (k_flat1,
k_top_a, k_top_b, k_decide_roots) move a negligible number of bytes.  Rounds a window skips
(nproc < 4) still launch but return at once: the model counts every round of every window, so it is an upper bound on
the bytes of rounds 0..3.
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

CHUNK_PX = 8192   # kRefineChunkPx (csrc/kernels.h)

# name: (bytes per window pixel and launch, launches per batch in inpaint mode, pixels it sweeps: "all" / "multi")
MODEL = {
    "k_phase0": (5.25, 1, "all"),
    "k_decide1": (0, 1, "all"),
    "k_xor": (5.75, 1, "all"),
    "k_decide2": (0, 1, "all"),
    "k_label_local": (2.375, 5, "all"),
    "k_union_border": (0, 5, "multi"),
    "k_flat1": (0, 5, "multi"),
    "k_top_a": (0, 1, "all"),
    "k_top_b": (0, 1, "all"),
    "k_decide_roots": (0, 5, "all"),
    "k_merge": (0.25, 1, "all"),
    "k_dilate": (0.25, 1, "all"),
    "k_or": (0.125, 1, "all"),
}


def plan_chunks(wins):
    """RefineJob::add (csrc/pipeline.cu): chunks of whole rows, or row segments of <= CHUNK_PX pixels"""
    n_chunks = n_multi = 0
    px = multi_px = 0
    for x1, y1, x2, y2 in wins:
        rw, rh = x2 - x1, y2 - y1
        if rw <= 0 or rh <= 0:
            continue
        rows_per = max(1, CHUNK_PX // rw)
        if rows_per >= 8:
            rows_per &= ~3
        nc = -(-rh // rows_per) * -(-rw // CHUNK_PX)
        n_chunks += nc
        px += rw * rh
        if nc > 1:
            n_multi += nc
            multi_px += rw * rh
    return n_chunks, n_multi, px, multi_px


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q


# g_pass_clocks[round][i] (csrc/refine_mk.cu): the merge of the round before, then the labelling's passes
PASSES = ["merge r-1", "pass 1", "-", "pass 2", "pass 3a", "pass 3b", "pass 3c"]
# g_pass_counts[round][i]: word seams that a run crosses, and the shared unions of vertical and diagonal contacts
COUNTS = ["seams", "contacts"]


def build_passes_lib(build_dir):
    lib = os.path.join(build_dir, "libctd_b200.so")
    if not os.path.isfile(lib):
        subprocess.run(["bash", os.path.join(ROOT, "comic-text-detector_b200", "csrc", "build.sh"),
                        "-DCTD_REFINE_PASS_CLOCKS"], env=dict(os.environ, CTD_BUILD_DIR=os.path.abspath(build_dir)),
                       check=True)
    return lib


def print_passes(clk, counts, cardq):
    print("k_label_local, share of the summed CTA clock ticks per pass and round, and union counts; %s" % cardq)
    print("%-6s %10s " % ("round", "Mticks") + " ".join("%10s" % p for p in PASSES + COUNTS))
    for r in range(5):
        tot = float(sum(clk[r]))
        if tot > 0:
            print("%-6d %10.1f " % (r, tot / 1e6) + " ".join("%9.1f%%" % (100.0 * c / tot) for c in clk[r][0:7])
                  + " " + " ".join("%10d" % c for c in counts[r]))


def gpu_run(n, h, w, mode, lib=None, passes=False):
    import numpy as np
    import torch
    from torch.profiler import profile, ProfilerActivity
    import ctd_b200
    if lib:
        ctd_b200.binding.LIB_PATH = os.path.abspath(lib)   # read when the library is first loaded, below
    from ctd_b200 import multigpu
    from oracle import postproc_ref, synth
    ck = synth.make_checkpoint(0, smooth=True)
    prog = ctd_b200.compiler.compile_checkpoint(ck)
    pages = np.stack([synth.structured_page(1000 + i, h, w) for i in range(n)])
    dev = torch.from_numpy(pages).cuda()
    eng = ctd_b200.Engine(prog, max_batch=n, max_h=h, max_w=w, use_graph=True)
    lay = eng.results_layout()
    out = torch.empty((lay["total_bytes"],), dtype=torch.uint8).pin_memory()
    try:
        for _ in range(3):
            eng.submit_full(0, dev.data_ptr(), n, h, w, out.data_ptr(), refine_mode=mode, pages_on_device=True)
            eng.collect(0)
        torch.cuda.synchronize()
        if passes:
            import ctypes
            clk = (ctypes.c_ulonglong * (5 * 8 + 5 * 2))()   # ticks [5][8], then counts [5][2]
            fn = ctd_b200.binding.load_library().ctd_refine_pass_clocks
            fn(clk)   # drop the warm-up's ticks
            eng.submit_full(0, dev.data_ptr(), n, h, w, out.data_ptr(), refine_mode=mode, pages_on_device=True)
            eng.collect(0)
            torch.cuda.synchronize()
            if fn(clk) != 0:
                raise RuntimeError("ctd_refine_pass_clocks failed")
            return ([[int(clk[8 * r + i]) for i in range(8)] for r in range(5)],
                    [[int(clk[40 + 2 * r + i]) for i in range(2)] for r in range(5)], card())
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.submit_full(0, dev.data_ptr(), n, h, w, out.data_ptr(), refine_mode=mode, pages_on_device=True)
            eng.collect(0)
            torch.cuda.synchronize()
        a = multigpu.unpack_arena(out.numpy(), lay, n, h, w, full=True)
    finally:
        eng.close()
    wins = [postproc_ref.expand_textwindow((h, w), [int(v) for v in b.xyxy[:4]], expand_r=16)
            for blocks in a["blocks"] for b in blocks]
    times, counts, other_ms = {}, {}, 0.0
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    for ev in trace.get("traceEvents", []):
        if ev.get("cat") != "kernel":
            continue
        m = re.search(r"\b(k_[a-z0-9_]+)\(", ev.get("name", ""))
        if m and m.group(1) in MODEL:
            times[m.group(1)] = times.get(m.group(1), 0.0) + ev.get("dur", 0.0) * 1e-3
            counts[m.group(1)] = counts.get(m.group(1), 0) + 1
        else:
            other_ms += ev.get("dur", 0.0) * 1e-3
    return wins, times, counts, other_ms, card()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=1024, help="square page size")
    ap.add_argument("--mode", type=int, choices=(0, 1), default=0, help="refine mode (0 = inpaint, as the benchmark)")
    ap.add_argument("--gpu", action="store_true", help="run the batch on cuda:0 and add the measured device times")
    ap.add_argument("--passes", action="store_true", help="pass shares of k_label_local on a -DCTD_REFINE_PASS_CLOCKS build")
    ap.add_argument("--passes-dir", default=None, help="build directory of that library (default: a temporary one)")
    ap.add_argument("--lib", default=None, help="with --gpu: another build of libctd_b200.so to run")
    ap.add_argument("--json", default=None, help="also write the rows to this file")
    args = ap.parse_args()
    n, h, w = args.batch, args.size, args.size
    names = [k for k in MODEL if not (k == "k_dilate" and args.mode == 1)]
    if args.passes:
        with tempfile.TemporaryDirectory() as td:
            clk, counts, cardq = gpu_run(n, h, w, args.mode, lib=build_passes_lib(args.passes_dir or td), passes=True)
        print_passes(clk, counts, cardq)
        if args.json:
            with open(args.json, "w") as f:
                json.dump({"shape": [n, h, w], "mode": args.mode, "card": cardq, "passes": PASSES, "ticks": clk,
                           "counts": COUNTS, "unions": counts}, f)
        return
    if not args.gpu:
        print("refine_mask byte model per window pixel (CPU model; --gpu measures the batch)")
        print("%-15s %8s %6s %6s" % ("kernel", "launches", "B/px", "sweeps"))
        tot = 0
        for k in names:
            b, l, sel = MODEL[k]
            tot += b * l if sel == "all" else 0
            print("%-15s %8d %6.3f %6s" % (k, l, b, sel))
        print("total over every window pixel: %.2f B (+ %d B per pixel of multi-chunk windows)"
              % (tot, sum(MODEL[k][0] * MODEL[k][1] for k in names if MODEL[k][2] == "multi")))
        return
    wins, times, counts, other_ms, cardq = gpu_run(n, h, w, args.mode, lib=args.lib)
    n_chunks, n_multi, px, multi_px = plan_chunks(wins)
    print("refine_mask at %d x %d x %d, mode %d; %s" % (n, h, w, args.mode, cardq))
    print("windows %d, chunks %d (%d in multi-chunk windows), window pixels %.2f M (%.2f M in multi-chunk windows)"
          % (len(wins), n_chunks, n_multi, px / 1e6, multi_px / 1e6))
    print("%-15s %8s %6s %8s %8s %7s" % ("kernel", "launches", "B/px", "GB", "ms", "TB/s"))
    rows = []
    tot_ms = tot_gb = 0.0
    for k in names:
        b, _l, sel = MODEL[k]
        launches = counts.get(k, 0)
        gb = b * launches * (px if sel == "all" else multi_px) / 1e9
        ms = times.get(k, 0.0)
        tot_ms += ms
        tot_gb += gb
        rows.append(dict(kernel=k, launches=launches, bytes_per_px=b, gb=gb, ms=ms))
        print("%-15s %8d %6.3f %8.3f %8.3f %7s" % (k, launches, b, gb, ms, "%.2f" % (gb / ms) if ms > 0 and gb > 0 else "-"))
    print("refine total: %.3f ms, %.2f GB modelled (%.2f TB/s); other kernels of the step: %.3f ms"
          % (tot_ms, tot_gb, tot_gb / tot_ms if tot_ms > 0 else 0.0, other_ms))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"shape": [n, h, w], "mode": args.mode, "card": cardq, "windows": len(wins), "chunks": n_chunks,
                       "multi_chunks": n_multi, "window_px": px, "rows": rows, "refine_ms": tot_ms,
                       "other_ms": other_ms}, f, indent=1)


if __name__ == "__main__":
    main()
