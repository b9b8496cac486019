"""TEST INFRASTRUCTURE ONLY (oracle): the part of `TextDetector.__call__` after the network
(reference inference.py:148-178) restated on top of oracle/postproc_ref.py, for net-sized pages.
`group_output_fn` is injected: the build-container tests pass the UNMODIFIED reference function, the GPU-box
tests pass the host implementation that tests/test_cpu_textblock.py pins against the reference."""
import numpy as np
import torch

from oracle import postproc_ref


def undetected_blocks(mask_pred, mask_refined, blk_xyxy):
    """utils/textmask.py:136-153: the blocks of refine_undetected_mask's second refine_mask (mutates mask_pred in place
    like the reference)."""
    import cv2
    mask_pred[np.where(mask_refined > 30)] = 0
    _, pred_t = cv2.threshold(mask_pred, 30, 255, cv2.THRESH_BINARY)
    n, labels, stats, _c = cv2.connectedComponentsWithStats(pred_t, 4, cv2.CV_16U)
    valid = np.where(stats[:, -1] > 50)[0]
    extra = []
    if len(valid) > 0:
        for li in valid[1:]:
            x, y, w, h, area = stats[li]
            bbox = [x, y, x + w, y + h]
            score = -1
            for b in blk_xyxy:
                x1, y1, x2, y2 = max(b[0], bbox[0]), max(b[1], bbox[1]), min(b[2], bbox[2]), min(b[3], bbox[3])
                s = -1 if (y2 < y1 or x2 < x1) else (y2 - y1) * (x2 - x1)   # union_area, imgproc_utils.py:13-20
                if s > score:
                    score = s
            if score / w / h < 0.5:
                extra.append([int(v) for v in bbox])
    return extra


def refine_undetected_mask(img, mask_pred, mask_refined, blk_xyxy, make_window_list, refine_mode, tie_order="stable"):
    """utils/textmask.py:135-156 (mutates mask_pred in place like the reference)."""
    import cv2
    extra = undetected_blocks(mask_pred, mask_refined, blk_xyxy)
    if len(extra) > 0:
        mask_refined = cv2.bitwise_or(mask_refined, postproc_ref.refine_mask(img, mask_pred, extra, refine_mode, tie_order))
    return mask_refined


def postprocess_page(img, blks, mask_f32, lines_f32, group_output_fn, conf_thresh=0.4, nms_thresh=0.35,
                     refine_mode=0, keep_undetected_mask=False, tie_order="stable"):
    """img u8 [H,W,3]; blks f32 [A,7]; mask_f32 [H,W]; lines_f32 [2,H,W] -> (mask u8, mask_refined u8, blk_list)."""
    im_h, im_w = img.shape[:2]
    det = postproc_ref.non_max_suppression(torch.as_tensor(blks)[None], conf_thresh, nms_thresh)[0].numpy()
    # resize_ratio == (1.0, 1.0) for net-sized pages (inference.py:148)
    det[..., [0, 2]] = det[..., [0, 2]] * 1.0
    det[..., [1, 3]] = det[..., [1, 3]] * 1.0
    b = (det[..., 0:4].astype(np.int32), det[..., 5].astype(np.int32), np.round(det[..., 4], 3))
    mask = (np.asarray(mask_f32) * 255).astype(np.uint8)          # postprocess_mask
    boxes, scores = postproc_ref.seg_represent(np.asarray(lines_f32)[0], 0.3)
    idx = np.where(scores > 0.6)
    lines = boxes[idx]
    if lines.size == 0:
        lines = []
    else:
        lines = lines.astype(np.float64)
        lines[..., 0] *= 1.0
        lines[..., 1] *= 1.0
        lines = lines.astype(np.int32)
    blk_list = group_output_fn(b, lines, im_w, im_h, mask)
    wins = [blk.xyxy for blk in blk_list]
    mask_refined = postproc_ref.refine_mask(img, mask, wins, refine_mode, tie_order)
    if keep_undetected_mask:
        mask_refined = refine_undetected_mask(img, mask, mask_refined, wins, None, refine_mode, tie_order)
    return mask, mask_refined, blk_list
