"""TEST INFRASTRUCTURE ONLY: `TextBlock.get_transformed_region` (reference utils/textblock.py:162-194) restated with
numpy + cv2, statement for statement, plus the per-line plan fields the native `ctd_region_plan` returns.  It needs no
reference tree and no GPU; tests/test_cpu_regions.py checks it against the unmodified reference byte for byte."""
import cv2
import numpy as np

LANG_LIST = ["eng", "ja", "unknown"]
MAX_SIDE = 32767   # crops with a side this long or longer are refused by the native planner (status 2)


def _geometry(lines, idx, language, vertical, font_size, im_w, im_h, textheight):
    src_pts = np.array(lines[idx], dtype=np.float64)
    if language == "eng" or (language == "unknown" and not vertical):
        e_size = font_size / 3
        src_pts[..., 0] += np.array([-e_size, e_size, e_size, -e_size])
        src_pts[..., 1] += np.array([-e_size, -e_size, e_size, e_size])
        src_pts[..., 0] = np.clip(src_pts[..., 0], 0, im_w)
        src_pts[..., 1] = np.clip(src_pts[..., 1], 0, im_h)
    middle_pnt = (src_pts[[1, 2, 3, 0]] + src_pts) / 2
    vec_v = middle_pnt[2] - middle_pnt[0]
    vec_h = middle_pnt[1] - middle_pnt[3]
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.linalg.norm(vec_v) / np.linalg.norm(vec_h)
    if not vertical:
        h = int(textheight)
        w = int(round(textheight / ratio))
    else:
        w = int(textheight)
        h = int(round(textheight * ratio))
    dst_pts = np.array([[0, 0], [w - 1, 0], [w - 1, h - 1], [0, h - 1]]).astype(np.float32)
    return src_pts, dst_pts, w, h


def transformed_region(blk, img, idx, textheight):
    """the reference method on a block-like object (lines, language, vertical, font_size); raises where it raises"""
    im_h, im_w = img.shape[:2]
    src_pts, dst_pts, w, h = _geometry(blk.lines, idx, blk.language, blk.vertical, blk.font_size, im_w, im_h, textheight)
    M, _ = cv2.findHomography(src_pts, dst_pts, cv2.RANSAC, 5.0)
    region = cv2.warpPerspective(img, M, (w, h))
    if blk.vertical:
        region = cv2.rotate(region, cv2.ROTATE_90_COUNTERCLOCKWISE)
    return region


def plan_line(lines, idx, language, vertical, font_size, im_w, im_h, textheight):
    """dict(status, out_h, out_w, rotate, homography, inverse) as ctd_region_plan should fill it (status 1: the
    reference raises; 2: a side of MAX_SIDE px or more)"""
    try:
        src_pts, dst_pts, w, h = _geometry(lines, idx, language, vertical, font_size, im_w, im_h, textheight)
    except (ZeroDivisionError, ValueError, OverflowError):
        return dict(status=1)
    if w >= MAX_SIDE or h >= MAX_SIDE:
        return dict(status=2)
    M, _ = cv2.findHomography(src_pts, dst_pts, cv2.RANSAC, 5.0)
    if M is None:
        return dict(status=1)
    _, inv = cv2.invert(M, flags=cv2.DECOMP_LU)
    ww, wh = (im_w, im_h) if (w <= 0 or h <= 0) else (w, h)
    out_h, out_w = (ww, wh) if vertical else (wh, ww)
    return dict(status=0, out_h=out_h, out_w=out_w, rotate=int(bool(vertical)), homography=M, inverse=inv)


def warp_with_inverse(img, inverse, out_h, out_w, rotate):
    """cv2.warpPerspective sampling with a given inverse matrix (WARP_INVERSE_MAP) + the rotation: what the kernel
    computes for one plan entry"""
    ww, wh = (out_h, out_w) if rotate else (out_w, out_h)
    region = cv2.warpPerspective(img, np.asarray(inverse, np.float64), (ww, wh), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP)
    if rotate:
        region = cv2.rotate(region, cv2.ROTATE_90_COUNTERCLOCKWISE)
    return region
