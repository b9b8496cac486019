"""Cost of the float-tensor network path (`ctd_b200.TextDetBase`, ctd_forward_tensor) against the u8 device path.

Workload: batches of 16 seeded synthetic 1024 x 1024 pages, fp16 tensor cores, the network only (skip_postproc).
  arm "tensor": TextDetBase on the pages as float32 CUDA tensors [16][3][1024][1024] (u8 / 255): the input pre-pass,
                the forward (CUDA graph) and the three device-to-device output copies into fresh torch tensors;
  arm "u8":     Engine.forward_device on the same pages as u8 [16][1024][1024][3] in device memory (CUDA graph), its
                outputs left in the engine.
Both arms compute the same network outputs bit for bit (checked before timing).  The arms alternate in one run, each
round timing --iters batches with a host clock that stops after a device synchronise.

    python scripts/tensor_net_bench.py [--rounds 5] [--iters 20] [--profile] [--out DIR]

--profile: a separate run.  A few batches of each arm under torch.profiler (CUDA activity): the device time per page of
the pre-pass (nchw_to_hwc_kernel), the stem on each page type (stem_tc_kernel<__half> / <unsigned char>) and the
device-to-device copies, with their achieved GB/s from the bytes the shapes say they move.  Prints one JSON line
either way, with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N, S = 16, 1024


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True)
    except OSError:
        return "unknown"
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def byte_model(n=N, h=S, w=S, nc=2):
    """bytes per page each piece moves, from the shapes"""
    px = h * w
    rows = 3 * ((h // 8) * (w // 8) + (h // 16) * (w // 16) + (h // 32) * (w // 32))
    return {"prepass": px * 3 * 4 + px * 3 * 2,          # f32 NCHW in, fp16 HWC out
            "stem_f16_read": px * 3 * 2, "stem_u8_read": px * 3,
            "copies": 2 * (rows * (5 + nc) * 4 + px * 4 + px * 2 * 4)}   # read + write of blks, mask, lines


def setup():
    import torch
    import ctd_b200
    from ctd_b200.binding import PREC_FP16_TC
    from oracle import synth
    if not torch.cuda.is_available():
        raise SystemExit("tensor_net_bench.py measures on the GPU; no CUDA device is visible")
    ck = synth.make_checkpoint(0, smooth=True)
    pages = np.stack([synth.structured_page(1000 + i, S, S) for i in range(N)])
    u8 = torch.from_numpy(pages).cuda()
    x = torch.from_numpy(np.ascontiguousarray(pages.transpose(0, 3, 1, 2)).astype(np.float32) / 255).cuda()
    mod = ctd_b200.TextDetBase(ck, precision=PREC_FP16_TC, max_batch=N, max_size=S)
    eng = ctd_b200.Engine(ctd_b200.compiler.compile_checkpoint(ck), precision=PREC_FP16_TC, max_batch=N, max_h=S,
                          max_w=S, use_graph=True, skip_postproc=True)
    return torch, mod, eng, u8, x


def check_same(torch, mod, eng, u8, x):
    got = [t.cpu().numpy() for t in mod(x)]
    eng.forward_device(u8.data_ptr(), N, S, S)
    want = eng.net_outputs()
    return all(np.array_equal(g, e) for g, e in zip(got, want))


def arm_tensor(torch, mod, eng, u8, x, iters):
    for _ in range(iters):
        mod(x)


def arm_u8(torch, mod, eng, u8, x, iters):
    for _ in range(iters):
        eng.forward_device(u8.data_ptr(), N, S, S)


ARMS = {"tensor": arm_tensor, "u8": arm_u8}


def timed(torch, fn, ctx, iters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn(*ctx, iters)
    torch.cuda.synchronize()   # the engine's stream and torch's: a device-wide synchronise
    return time.perf_counter() - t0


def run_timing(args):
    torch, *ctx = setup()
    ctx = (torch, *ctx)
    same = check_same(*ctx)
    for fn in ARMS.values():
        timed(torch, fn, ctx, max(2, args.iters // 4))   # warm-up: graphs captured, allocator primed
    rates = {k: [] for k in ARMS}
    for _ in range(args.rounds):
        for k, fn in ARMS.items():
            rates[k].append(N * args.iters / timed(torch, fn, ctx, args.iters))
    med = {k: float(np.median(v)) for k, v in rates.items()}
    return {"card": card(), "pages_per_batch": N, "size": S, "identical_outputs": bool(same),
            "pages_per_s": {k: [round(r, 1) for r in v] for k, v in rates.items()},
            "median_pages_per_s": {k: round(v, 1) for k, v in med.items()},
            "tensor_ms_per_page_extra": round(1e3 / med["tensor"] - 1e3 / med["u8"], 4)}


def run_profile(args):
    from torch.profiler import profile, ProfilerActivity
    torch, *ctx = setup()
    ctx = (torch, *ctx)
    for fn in ARMS.values():
        timed(torch, fn, ctx, 3)
    iters = 5
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for fn in ARMS.values():
            fn(*ctx, iters)
        torch.cuda.synchronize()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        prof.export_chrome_trace(os.path.join(args.out, "tensor_net.pt.trace.json"))
    dev = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        dev[e.key] = dev.get(e.key, 0.0) + t
    pick = lambda pred: sum(v for k, v in dev.items() if pred(k))
    pages = iters * N
    us = {"prepass": pick(lambda k: "nchw_to_hwc_kernel" in k),
          "stem_f16": pick(lambda k: "stem_tc_kernel" in k and "__half" in k),
          "stem_u8": pick(lambda k: "stem_tc_kernel" in k and "unsigned char" in k),
          "copies_dtod": pick(lambda k: "Memcpy DtoD" in k)}
    per_page = {k: v / pages for k, v in us.items()}   # microseconds per page
    bm = byte_model()
    gbs = {"prepass": bm["prepass"], "stem_f16": bm["stem_f16_read"], "stem_u8": bm["stem_u8_read"],
           "copies_dtod": bm["copies"]}
    return {"card": card(), "profile": True, "pages": pages,
            "us_per_page": {k: round(v, 2) for k, v in per_page.items()},
            "GB_per_s": {k: (round(gbs[k] / (per_page[k] * 1e3), 1) if per_page[k] else None) for k in per_page},
            "bytes_per_page": bm,
            "kernels": sorted(((k, round(v / pages, 2)) for k, v in dev.items() if v), key=lambda kv: -kv[1])[:12]}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="directory for the profiler trace")
    args = ap.parse_args()
    res = run_profile(args) if args.profile else run_timing(args)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
