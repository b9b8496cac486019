"""The batches tests/test_gpu_gather.py runs through gather_pages_kernel (csrc/gather.cu), and a model of the copy path
each of their rows takes, which tests/test_cpu_gather_cases.py checks with no GPU.

A device image is a view of a flat u8 storage tensor, given by its sizes, strides and storage offset (`View`).  The
gather copies row y of an image from src + y * stride_h to dst + y * iw * ch, where dst is the slot's plane base
(cudaMalloc: 256-aligned) plus the image's page_off (3 P_i, a multiple of 768) or mask_off (P_i, a multiple of 256)
from the plan, and src is the storage's data pointer (the CUDA caching allocator hands out 512-aligned blocks) plus
the offset.  Both addresses are therefore known modulo 256, which fixes the copy path of every row, its byte head
and its byte tail (`row_path`)."""
from collections import namedtuple

import numpy as np
import torch

from ctd_b200 import binding

NET = 256
MAX_BATCH = 6
SENTINEL = 0xA5

# sizes, strides (elements = bytes), storage offset, and the storage bytes the view spans
View = namedtuple("View", "size stride offset nbytes")
# one image of a batch: a page ([h][w][3]) or a mask ([h][w]); view None: a host (numpy) image
Img = namedtuple("Img", "h w view")
# job "pages": ctd_submit_pages (pages only); "refine": ctd_submit_refine with no blocks (masks[i] goes with pages[i])
Case = namedtuple("Case", "name job pages masks")


def _view(t):
    size, stride, off = tuple(t.shape), tuple(t.stride()), t.storage_offset()
    return View(size, stride, off, off + sum((n - 1) * s for n, s in zip(size, stride)) + 1)


def meta(*size):
    return torch.empty(size, dtype=torch.uint8, device="meta")


def host(h, w):
    return Img(h, w, None)


def window(h, w, ch, off, pitch):
    """rows of w * ch contiguous bytes, `pitch` bytes apart, the first at byte `off` of a larger buffer"""
    size, stride = ((h, w, 3), (pitch, 3, 1)) if ch == 3 else ((h, w), (pitch, 1))
    return Img(h, w, _view(meta(off + h * pitch).as_strided(size, stride, off)))


def dev(h, w, ch, t):
    """an image given as a torch expression on meta tensors"""
    assert tuple(t.shape) == ((h, w, 3) if ch == 3 else (h, w)), t.shape
    return Img(h, w, _view(t))


def _phase_sweep(ch, widths, job):
    """every source offset 0..15 of contiguous-row windows at each width, MAX_BATCH images per batch.  The row pitch is
    odd, so the source phase of successive rows moves on; at least 17 rows, so a row of an odd number of bytes meets
    every destination phase"""
    imgs = []
    for w in widths:
        for off in range(16):
            imgs.append(window(17 + (5 * off + w) % 23, w, ch, off, (w * ch | 1) + 2 * (off % 7)))
    cases = []
    for b in range(0, len(imgs), MAX_BATCH):
        part = imgs[b:b + MAX_BATCH]
        name = "%s_phases_%d" % ("page" if ch == 3 else "mask", b // MAX_BATCH)
        if ch == 3:
            cases.append(Case(name, job, part, None))
        else:
            cases.append(Case(name, job, [host(i.h, i.w) for i in part], part))
    return cases


def _generic_pages():
    h, w = 37, 23
    return [
        dev(h, w, 3, meta(3, h, w).permute(1, 2, 0)),                               # channels-first
        dev(h, w, 3, meta(w, h, 3).transpose(0, 1)),                                # a transposed page
        dev(h, w, 3, meta(h, w, 6)[..., ::2]),                                      # pixel stride 6, channel stride 2
        dev(h, w, 3, meta(1, w, 3).expand(h, w, 3)),                                # one row repeated
        dev(h, w, 3, meta(h, 1, 3).expand(h, w, 3)),                                # one column repeated
        dev(h, w, 3, meta(h, w, 1).expand(h, w, 3)),                                # grey: one byte per pixel
    ]


def _generic_masks():
    h, w = 37, 23
    return [dev(h, w, 1, meta(h, w, 3)[..., c]) for c in range(3)] + [
        dev(h, w, 1, meta(w, h).t()),                                               # a transposed mask
        dev(h, w, 1, meta(1, w).expand(h, w)),                                      # one row repeated
        dev(h, w, 1, meta(h, 1).expand(h, w)),                                      # one column repeated
    ]


def _big(ch):
    # 7016 x 4960 cut from a 7020 x 4963 image at row 2, column 1: an odd byte offset and an odd row pitch
    t = meta(7020, 4963, 3)[2:7018, 1:4961] if ch == 3 else meta(7020, 4963)[2:7018, 1:4961]
    return dev(7016, 4960, ch, t)


# one-row and one-column images between tall ones: the row search of the kernel meets a page boundary at every step
_THIN = [(300, 7), (1, 50), (200, 5), (40, 1), (1, 1), (257, 3)]


def _mixed(pattern, shapes, ch, seed):
    """pattern: 'H' a host image, 'D' a device window (its offset and pitch varied with its index)"""
    out = []
    for i, (p, (h, w)) in enumerate(zip(pattern, shapes)):
        k = seed + i
        out.append(host(h, w) if p == "H" else window(h, w, ch, (7 * k) % 16, w * ch + 1 + 2 * (k % 5)))
    return out


CASES = (
    _phase_sweep(3, [1, 2, 5, 7, 16, 43], "pages")
    + _phase_sweep(1, [1, 2, 5, 7, 16, 48, 129], "refine")
    + [
        Case("page_generic", "pages", _generic_pages(), None),
        Case("page_generic_refine", "refine", _generic_pages(), [host(37, 23)] * 6),
        Case("mask_generic", "refine", [host(37, 23)] * 6, _generic_masks()),
        Case("thin_pages", "pages", _mixed("DDDDDD", _THIN, 3, 0), None),
        Case("thin_refine", "refine", _mixed("DDDDDD", _THIN, 3, 3), _mixed("DDDDDD", _THIN, 1, 5)),
        # host and device images in every run pattern; full and partial batches
        Case("host_first", "pages", _mixed("HHDDDD", _THIN, 3, 1), None),
        Case("host_middle", "pages", _mixed("DHHD", _THIN[:4], 3, 2), None),
        Case("host_last", "pages", _mixed("DDDDH", _THIN[:5], 3, 4), None),
        Case("host_all", "pages", _mixed("HHH", _THIN[:3], 3, 0), None),
        Case("host_runs_refine", "refine", _mixed("HDHHDH", _THIN, 3, 6), _mixed("DHDDHD", _THIN, 1, 7)),
        Case("host_all_refine", "refine", _mixed("HHHH", _THIN[:4], 3, 0), _mixed("HHHH", _THIN[:4], 1, 0)),
        Case("big", "refine", [_big(3), host(33, 17)], [_big(1), host(33, 17)]),
    ]
)


def row_path(s, d, nb):
    """copy path of one fast-path row of nb bytes from source address s to destination address d (both modulo 256):
    (path, head, words, tail), path 'w16', 'w4' or 'shift1' .. 'shift3' (the byte shift of the funnel-shifted words)"""
    phase = (s ^ d) & 15
    wide = 16 if phase == 0 else 4
    head = min(nb, (wide - d % wide) % wide)
    words = (nb - head) // wide
    tail = nb - head - words * wide
    if phase & 3 == 0:
        return ("w16" if wide == 16 else "w4"), head, words, tail
    return "shift%d" % ((s + head) % 4), head, words, tail


def is_fast(img, ch):
    st = img.view.stride
    return st[1] == 1 if ch == 1 else (st[2] == 1 and st[1] == 3)


def image_paths(img, ch, dst_off):
    """the paths of an image's rows: {'generic3'} / {'generic1'} for the byte-per-thread paths, else per row
    (path, head > 0, tail > 0) for rows with at least one word, and 'short' for a row shorter than one word"""
    if not is_fast(img, ch):
        return {"generic%d" % ch}
    nb = img.w * ch
    out = set()
    for y in range(img.h):
        path, head, words, tail = row_path((img.view.offset + y * img.view.stride[0]) % 256, (dst_off + y * nb) % 256,
                                           nb)
        if nb < 4:
            out.add("short")
        elif words:
            out.add((path, head > 0, tail > 0))
    return out


def shapes(imgs):
    return [(i.h, i.w) for i in imgs]


def plan(case):
    """(page entries, bytes of the packed pages, bytes of the mask plane) of the case's batch, from the planner its
    job's submit checks the entries against"""
    if case.job == "pages":
        entries, in_bytes, _res = binding.pages_plan(shapes(case.pages), NET, NET)
        return entries, in_bytes, 0
    n = len(case.pages)
    entries, _win, _st, in_bytes, _res = binding.refine_plan(shapes(case.pages), np.zeros((0, 4), np.int32), [0] * n)
    return entries, in_bytes // 5 * 3, in_bytes // 5


def case_paths(case):
    """{(kind, path)}: kind 'page' or 'mask', path as image_paths gives it, over the case's device images"""
    entries, _pb, _mb = plan(case)
    out = set()
    for kind, imgs, ch, key in (("page", case.pages, 3, "page_off"), ("mask", case.masks or [], 1, "mask_off")):
        for img, e in zip(imgs, entries):
            if img.view is not None:
                out |= {(kind, p) for p in image_paths(img, ch, int(e[key]))}
    return out
