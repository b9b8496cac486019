"""Throughput of the batched stream with pages and results in GPU memory: `detect_stream(textheight=48)` fed numpy pages
or torch.uint8 CUDA pages, yielding numpy results or CUDA tensors (`device_results=True`; ctd_submit_pages with device
pages, one batched strided gather launch per batch, ctd_collect_device).

Workload: the 64 seeded synthetic pages of scripts/stream_regions_bench.py (DESIGN §7.4) at input_size 1024,
refine_mode INPAINT, textheight 48, max_batch 16.  Every arm runs the workload once to warm up, then twice timed; the
host clock stops when the last result of the second pass is usable (numpy results are host arrays; CUDA results are
complete when yielded).

    python scripts/device_stream_bench.py [--out DIR] [--profile]

Arms: (1) numpy pages -> numpy results (§7.4 arm c); (2) CUDA pages, uploaded once before timing -> numpy results;
(3) CUDA pages -> CUDA results; (4) numpy pages -> CUDA results.  Before timing, every arm's results are compared with
arm 1's, byte for byte (masks, mask_refined, crops, block boxes and lines).

--profile: a separate run.  Caller-thread time of one pass of each arm (host clock, and the part spent waiting in
Engine.collect); then one pass of arm 3 under torch.profiler (CUDA activity): device time of gather_pages_kernel per
batch and its achieved GB/s from the bytes it reads plus the bytes it writes (2 x the page bytes, from the shapes).
Prints one JSON line either way."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [(1654, 1170), (1170, 1654), (2048, 1446), (1200, 800), (1024, 1024)]
NET = 1024
TEXTHEIGHT = 48
MAX_BATCH = 16
ARMS = {"1": "numpy->numpy", "2": "cuda->numpy", "3": "cuda->cuda", "4": "numpy->cuda"}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True)
    except OSError:
        return "unknown"
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def workload(n=64):
    from oracle import synth
    return [synth.structured_page(10_000 + i, *SIZES[i % len(SIZES)]) for i in range(n)]


def run_arm(det, pages, cuda_pages, arm, keep=False):
    """one pass -> (lines cropped, the items if keep)"""
    src = cuda_pages if arm in ("2", "3") else pages
    items = []
    lines = 0
    for item in det.detect_stream(src, refine_mode=0, textheight=TEXTHEIGHT, device_results=arm in ("3", "4")):
        lines += sum(c is not None for blk in item[3] for c in blk)
        if keep:
            items.append(item)
    return lines, items


def _host(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else x


def same_results(got, ref):
    """byte equality of two passes' items: masks, mask_refined, crops, block boxes and lines"""
    if len(got) != len(ref):
        return False
    for g, r in zip(got, ref):
        if not (np.array_equal(_host(g[0]), r[0]) and np.array_equal(_host(g[1]), r[1])):
            return False
        if [(list(b.xyxy), np.asarray(b.lines).tolist()) for b in g[2]] != \
                [(list(b.xyxy), np.asarray(b.lines).tolist()) for b in r[2]]:
            return False
        for gb, rb in zip(g[3], r[3]):
            if len(gb) != len(rb):
                return False
            for gc, rc in zip(gb, rb):
                if (gc is None) != (rc is None) or (rc is not None and not np.array_equal(_host(gc), rc)):
                    return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--pages", type=int, default=64)
    args = ap.parse_args()
    import torch
    import ctd_b200
    from oracle import synth
    ck = synth.make_checkpoint(0, smooth=True)
    pages = workload(args.pages)
    line = {"card": card(), "pages": len(pages), "input_size": NET, "sizes": SIZES, "textheight": TEXTHEIGHT,
            "max_batch": MAX_BATCH, "arms": {}}
    det = ctd_b200.TextDetector(ck, input_size=NET, act="leaky", max_batch=MAX_BATCH)
    try:
        cuda_pages = [torch.from_numpy(p).cuda() for p in pages]   # uploaded once, before any timing
        torch.cuda.synchronize()
        if args.profile:
            line["profile"] = profile(det, pages, cuda_pages)
        else:
            _n, ref = run_arm(det, pages, cuda_pages, "1", keep=True)
            for arm in ARMS:
                _n, items = run_arm(det, pages, cuda_pages, arm, keep=True)   # the check pass is the warm-up
                same = same_results(items, ref)
                del items
                t0 = time.perf_counter()
                l1, _ = run_arm(det, pages, cuda_pages, arm)
                l2, _ = run_arm(det, pages, cuda_pages, arm)
                dt = time.perf_counter() - t0
                line["arms"][ARMS[arm]] = {"pages_per_s": round(2 * len(pages) / dt, 2),
                                           "lines_per_s": round((l1 + l2) / dt, 1), "lines_per_pass": l1,
                                           "same_as_arm_1": same}
                print(ARMS[arm], line["arms"][ARMS[arm]], flush=True)
    finally:
        det.close()
    line["card_after"] = card()
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "device_stream_bench%s.json" % ("_profile" if args.profile else "")), "w") as f:
            f.write(json.dumps(line, indent=1))
    if not args.profile and not all(a["same_as_arm_1"] for a in line["arms"].values()):
        sys.exit("an arm's results differ from arm 1's")


def host_split(det, pages, cuda_pages, arm):
    """host clock of one pass and the caller-thread time inside Engine.collect (waiting for the batch), in ms"""
    eng = det.net
    t = {"collect_wait": 0.0}
    collect = eng.collect

    def timed(*a, **k):
        t0 = time.perf_counter()
        try:
            return collect(*a, **k)
        finally:
            t["collect_wait"] += time.perf_counter() - t0

    eng.collect = timed
    try:
        t0 = time.perf_counter()
        run_arm(det, pages, cuda_pages, arm)
        t["pass"] = time.perf_counter() - t0
    finally:
        del eng.collect
    return {k: round(v * 1e3, 1) for k, v in t.items()}


def profile(det, pages, cuda_pages):
    import torch
    out = {"batches": (len(pages) + MAX_BATCH - 1) // MAX_BATCH, "caller_ms": {}}
    for arm in ARMS:
        run_arm(det, pages, cuda_pages, arm)
        out["caller_ms"][ARMS[arm]] = host_split(det, pages, cuda_pages, arm)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run_arm(det, pages, cuda_pages, "3")
        torch.cuda.synchronize()
    us, cnt = 0.0, 0
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and "gather_pages_kernel" in ev.name:
            us += ev.time_range.elapsed_us()
            cnt += 1
    moved = 2 * sum(p.size for p in pages)   # every page byte read once and written once
    out.update({"gather_launches": cnt, "gather_device_us": round(us, 1),
                "gather_device_us_per_batch": round(us / max(cnt, 1), 1), "gather_bytes_moved": moved,
                "gather_gb_per_s": round(moved / (us * 1e-6) / 1e9, 1) if us > 0 else None})
    return out


if __name__ == "__main__":
    main()
