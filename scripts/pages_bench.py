"""Throughput of pages of any size through the whole `TextDetector.__call__` chain: page by page (`__call__`, one
blocking ctd_detect_page per page) against `TextDetector.detect_stream` (ctd_submit_pages, batches of max_batch pages,
two in flight), with refine_undetected_mask off and on (on = model2annotations' mode).

Workload: 64 seeded synthetic pages (oracle/synth.structured_page) at input_size 1024 in a scan-like mix of sizes:
1654x1170 (the reference's example page), 1170x1654, 2048x1446, 1200x800 and 1024x1024 -- the letterbox and the mask
back-projection run for every page but the last size.  Every arm runs the workload once to warm up (launch plans,
grown buffers), then twice timed; the time ends when the last result is on the host.

    python scripts/pages_bench.py [--out DIR] [--profile]

--profile: a separate run under torch.profiler (CUDA activity) of detect_stream at max_batch 16: device time of the
letterbox and back-projection kernels and their achieved GB/s from the bytes they must move (letterbox: the page in,
net_h * net_w * 3 out; back-projection: the unpadded mask crop in, ih * iw out).  Prints one JSON line either way."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [(1654, 1170), (1170, 1654), (2048, 1446), (1200, 800), (1024, 1024)]
NET = 1024


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


def run_arm(det, pages, batched, keep):
    if batched:
        out = list(det.detect_stream(pages, refine_mode=0, keep_undetected_mask=keep))
    else:
        out = [det(p, refine_mode=0, keep_undetected_mask=keep) for p in pages]
    return sum(len(o[2]) for o in out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--pages", type=int, default=64)
    args = ap.parse_args()
    import ctd_b200
    from ctd_b200 import binding
    from oracle import synth
    ck = synth.make_checkpoint(0, smooth=True)
    pages = workload(args.pages)
    mpx = sum(p.shape[0] * p.shape[1] for p in pages) / 1e6
    _plan, in_bytes, _rb = binding.pages_plan([p.shape[:2] for p in pages], NET, NET)
    line = {"card": card(), "pages": len(pages), "input_size": NET, "sizes": SIZES, "arms": {}}
    if args.profile:
        line["profile"] = profile(ck, pages)
    else:
        for max_batch in (1, 8, 16):
            det = ctd_b200.TextDetector(ck, input_size=NET, act="leaky", max_batch=max_batch)
            try:
                for keep in (False, True):
                    batched = max_batch > 1
                    run_arm(det, pages, batched, keep)
                    t0 = time.perf_counter()
                    blocks = run_arm(det, pages, batched, keep) + run_arm(det, pages, batched, keep)
                    dt = time.perf_counter() - t0
                    name = ("detect_stream_b%d" % max_batch if batched else "call_per_page") + ("_keep" if keep else "")
                    line["arms"][name] = {
                        "pages_per_s": round(2 * len(pages) / dt, 2), "mpx_per_s": round(2 * mpx / dt, 2),
                        "h2d_bytes_per_page": int(in_bytes / len(pages)) if batched else
                        int(sum(p.nbytes for p in pages) / len(pages)),
                        "blocks_per_pass": blocks // 2}
                    print(name, line["arms"][name], flush=True)
            finally:
                det.close()
        line["card_after"] = card()
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "pages_bench%s.json" % ("_profile" if args.profile else "")), "w") as f:
            f.write(json.dumps(line, indent=1))


def profile(ck, pages):
    import torch
    import ctd_b200
    from ctd_b200 import binding
    det = ctd_b200.TextDetector(ck, input_size=NET, act="leaky", max_batch=16)
    try:
        run_arm(det, pages, True, False)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            run_arm(det, pages, True, False)
            torch.cuda.synchronize()
        t = {"letterbox_batch_kernel": [0.0, 0], "backproject_batch_kernel": [0.0, 0]}
        for ev in prof.events():
            for k in t:
                if k in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA:
                    t[k][0] += ev.time_range.elapsed_us()
                    t[k][1] += 1
        ent, _ib, _rb = binding.pages_plan([p.shape[:2] for p in pages], NET, NET)
        lb_bytes = sum(int(p.nbytes) + NET * NET * 3 for p in pages)
        bp_bytes = sum(int(e["unpad_h"]) * int(e["unpad_w"]) + int(e["ih"]) * int(e["iw"]) for e in ent)
        out = {}
        for k, b in (("letterbox_batch_kernel", lb_bytes), ("backproject_batch_kernel", bp_bytes)):
            us, cnt = t[k]
            out[k] = {"launches": cnt, "device_us": round(us, 1), "bytes": b,
                      "gb_per_s": round(b / (us * 1e-6) / 1e9, 1) if us > 0 else None}
        return out
    finally:
        det.close()


if __name__ == "__main__":
    main()
