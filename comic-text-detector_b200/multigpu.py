"""Page sharding + result gather for one-process-per-GPU runs (SURVEY section 8e).

Pages are independent (reference inference.py:141-178 is pure per image), so the only
"communication" is a gather of fixed-size per-rank result arenas to rank 0.  The functions are
backend-agnostic (`nccl` on GPUs, `gloo` in the CPU tests)."""
import numpy as np


def shard_range(n_pages, rank, world):
    """Contiguous shard [lo, hi) of `n_pages` for `rank`; shards differ by at most one page."""
    base, rem = divmod(int(n_pages), int(world))
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def arena_layout(max_batch, max_h, max_w):
    """Byte offsets of the phase-A section of an engine's result arena for an engine created with
    (max_batch, max_h, max_w) -- the first phase_a_bytes of what ctd_submit_full delivers.  Mirrors engine.cu (256-byte
    aligned fields) without a GPU; prefer `Engine.results_layout()`, which asks the library and also covers
    mask_refined and the block sections."""
    al = lambda v: (v + 255) // 256 * 256
    o_det = al(max_batch * max_h * max_w)
    o_cnt = o_det + al(max_batch * 300 * 6 * 4)
    o_nl = o_cnt + al(max_batch * 4)
    o_lb = o_nl + al(max_batch * 4)
    o_ls = o_lb + al(max_batch * 1000 * 8 * 2)
    o_lc = o_ls + al(max_batch * 1000 * 4)
    return dict(mask=0, mask_u8=0, det=o_det, det_count=o_cnt, n_labels=o_nl, line_boxes=o_lb, line_scores=o_ls,
                line_count=o_lc, total=o_lc + al(max_batch * 4), phase_a_bytes=o_lc + al(max_batch * 4))


def gather_arenas(local_arena, dist, rank, world, dst=0):
    """One collective: every rank contributes its uint8 arena tensor; rank `dst` gets the list."""
    import torch
    out = [torch.empty_like(local_arena) for _ in range(world)] if rank == dst else None
    dist.gather(local_arena, gather_list=out, dst=dst)
    return out


def unpack_arena(arena_u8, layout, n, h, w, full=False):
    """arena bytes (numpy uint8) of a batch of n pages of h x w -> dict.  `layout` is `Engine.results_layout()` (or
    `arena_layout(max_batch, max_h, max_w)` for the phase-A section): the offsets depend on the shape the ENGINE was
    created for, not on the shape of this batch.  full=True also unpacks mask_refined and the per-page blocks
    (ctd_submit_full)."""
    lay = layout
    a = np.asarray(arena_u8)
    m0 = lay.get("mask_u8", lay.get("mask", 0))
    mask = a[m0:m0 + n * h * w].reshape(n, h, w)
    det = a[lay["det"]:lay["det"] + n * 300 * 6 * 4].view(np.float32).reshape(n, 300, 6)
    cnt = a[lay["det_count"]:lay["det_count"] + n * 4].view(np.int32)
    nl = a[lay["n_labels"]:lay["n_labels"] + n * 4].view(np.int32)
    lb = a[lay["line_boxes"]:lay["line_boxes"] + n * 1000 * 16].view(np.int16).reshape(n, 1000, 4, 2)
    ls = a[lay["line_scores"]:lay["line_scores"] + n * 1000 * 4].view(np.float32).reshape(n, 1000)
    lc = a[lay["line_count"]:lay["line_count"] + n * 4].view(np.int32)
    out = dict(mask=mask, det=[det[i, :cnt[i]] for i in range(n)], n_labels=nl,
               line_boxes=[lb[i, :lc[i]] for i in range(n)], line_scores=[ls[i, :lc[i]] for i in range(n)])
    if full:
        from .binding import decode_block_section
        from .textblock import blocks_from_records
        out["mask_refined"] = a[lay["mask_refined"]:lay["mask_refined"] + n * h * w].reshape(n, h, w)
        blocks, flags = [], []
        for i in range(n):
            sec = a[lay["blocks"] + i * lay["blocks_stride"]:lay["blocks"] + (i + 1) * lay["blocks_stride"]]
            hdr, rec, lines, dist = decode_block_section(sec, lay)
            blocks.append(blocks_from_records(rec, lines, dist))
            flags.append(int(hdr[3]))
        out["blocks"], out["block_flags"] = blocks, flags
    return out
