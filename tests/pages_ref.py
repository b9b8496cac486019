"""TEST INFRASTRUCTURE ONLY (oracle): the part of `TextDetector.__call__` after the network (reference
inference.py:148-178) for a page of ANY size, the sibling of oracle/pipeline_ref.postprocess_page (which covers
net-sized pages, whose resize ratios are 1.0).  It restates inference.py:148 (resize_ratio), 158-172 (the mask crop +
cv2.resize back to the page, the ratio casts of the text lines) and postprocess_yolo's ratio cast of the boxes
(inference.py:101-114), on top of the same oracle stages."""
import numpy as np
import torch

from oracle import pipeline_ref, postproc_ref


def postprocess_page_any_size(img, net_hw, unpad_hw, blks, mask_f32, lines_f32, group_output_fn, conf_thresh=0.4,
                              nms_thresh=0.35, refine_mode=0, keep_undetected_mask=False):
    """img u8 [H,W,3] (the page); net_hw = input_size; unpad_hw = the letterboxed size; blks f32 [A,7], mask_f32 [h,w],
    lines_f32 [2,h,w] = the network's outputs on the letterboxed page -> (mask u8, mask_refined u8, blk_list)."""
    import cv2
    im_h, im_w = img.shape[:2]
    dh, dw = net_hw[0] - unpad_hw[0], net_hw[1] - unpad_hw[1]
    resize_ratio = (im_w / (net_hw[1] - dw), im_h / (net_hw[0] - dh))
    det = postproc_ref.non_max_suppression(torch.as_tensor(blks)[None], conf_thresh, nms_thresh)[0].numpy()
    det[..., [0, 2]] = det[..., [0, 2]] * resize_ratio[0]
    det[..., [1, 3]] = det[..., [1, 3]] * resize_ratio[1]
    b = (det[..., 0:4].astype(np.int32), det[..., 5].astype(np.int32), np.round(det[..., 4], 3))
    mask = (np.asarray(mask_f32) * 255).astype(np.uint8)
    boxes, scores = postproc_ref.seg_represent(np.asarray(lines_f32)[0], 0.3)
    idx = np.where(scores > 0.6)
    lines = boxes[idx]
    mask = mask[:mask.shape[0] - dh, :mask.shape[1] - dw]
    mask = cv2.resize(mask, (im_w, im_h), interpolation=cv2.INTER_LINEAR)
    if lines.size == 0:
        lines = []
    else:
        lines = lines.astype(np.float64)
        lines[..., 0] *= resize_ratio[0]
        lines[..., 1] *= resize_ratio[1]
        lines = lines.astype(np.int32)
    blk_list = group_output_fn(b, lines, im_w, im_h, mask)
    # a block whose expanded window is an empty slice refines nothing (cv2 refuses the empty crop; the engine skips
    # the window, RefineJob::add)
    wins = []
    for blk in blk_list:
        x1, y1, x2, y2 = postproc_ref.expand_textwindow(img.shape, blk.xyxy, expand_r=16)
        if x2 > x1 and y2 > y1:
            wins.append(blk.xyxy)
    mask_refined = postproc_ref.refine_mask(img, mask, wins, refine_mode)
    if keep_undetected_mask:
        mask_refined = pipeline_ref.refine_undetected_mask(img, mask, mask_refined, [b.xyxy for b in blk_list], None,
                                                           refine_mode)
    return mask, mask_refined, blk_list
