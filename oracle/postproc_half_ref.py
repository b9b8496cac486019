"""TEST INFRASTRUCTURE ONLY (oracle): the reference's post-processing on float16 network outputs, the stages of
`TextDetector.__call__` (inference.py:148-178) that a `.half()` network's outputs take, restated on top of
oracle/postproc_ref.py and oracle/pipeline_ref.py.  On half tensors the reference does its arithmetic in half:

* non_max_suppression (yolov5_utils.py:136-182): `obj > conf_thres` and `conf > conf_thres` compare against
  half(conf_thres); `x[:, 5:] *= x[:, 4:5]` and xywh2xyxy round to half; torch.cat((box, conf, j.float()), 1) widens
  the rows to float32 before the class offset and torchvision's NMS.  postproc_ref.non_max_suppression is the
  reference's code line for line, so on a half tensor it does exactly this;
* postprocess_mask (inference.py:85-99): `img * 255` is a float16 numpy product (NEP 50), then numpy's float16 ->
  uint8 cast;
* SegDetectorRepresenter (db_utils.py:54-72): `pred > 0.3` compares against half(0.3); box_score_fast widens a float16
  map to float32 (db_utils.py:209-210).  A float16 value p satisfies `p > half(t)` exactly when float32(p) >
  float32(half(t)), so postproc_ref.seg_represent on the widened map with the threshold half(t) is the half binarize.
"""
import numpy as np
import torch

from oracle import pipeline_ref, postproc_ref


def non_max_suppression_half(prediction, conf_thres=0.4, iou_thres=0.35):
    """yolov5_utils.non_max_suppression on a float16 (N, A, 5 + nc) prediction -> list of float32 (n, 6) tensors"""
    return postproc_ref.non_max_suppression(torch.as_tensor(prediction).half(), conf_thres, iou_thres)


def mask_u8_half(mask):
    """postprocess_mask on a float16 map: (p * 255) in float16, then astype(np.uint8)"""
    return (np.asarray(mask, np.float16) * 255).astype(np.uint8)


def binarize_half(pred, thresh=0.3):
    """SegDetectorRepresenter.binarize on a float16 map: pred > half(thresh)"""
    return np.asarray(pred, np.float16) > np.float16(thresh)


def seg_represent_half(pred, thresh=0.3):
    """SegDetectorRepresenter(thresh)(batch, pred[None, None]) for one float16 map: the bitmap `pred > half(thresh)`,
    contour scores on the map widened to float32"""
    return postproc_ref.seg_represent(np.asarray(pred, np.float16).astype(np.float32), float(np.float16(thresh)))


def postprocess_page_half(img, blks, mask, lines, group_output_fn, conf_thresh=0.4, nms_thresh=0.35, refine_mode=0,
                          keep_undetected_mask=False):
    """pipeline_ref.postprocess_page for float16 outputs of a net-sized page: img u8 [H,W,3]; blks f16 [A,7]; mask
    f16 [H,W]; lines f16 [2,H,W] -> (mask u8, mask_refined u8, blk_list)"""
    im_h, im_w = img.shape[:2]
    det = non_max_suppression_half(np.asarray(blks, np.float16)[None], conf_thresh, nms_thresh)[0].numpy()
    b = (det[..., 0:4].astype(np.int32), det[..., 5].astype(np.int32), np.round(det[..., 4], 3))
    mask_u8 = mask_u8_half(mask)
    boxes, scores = seg_represent_half(np.asarray(lines)[0], 0.3)
    lines_kept = boxes[np.where(scores > 0.6)]
    lines_kept = [] if lines_kept.size == 0 else lines_kept.astype(np.float64).astype(np.int32)
    blk_list = group_output_fn(b, lines_kept, im_w, im_h, mask_u8)
    # a block whose expanded window is an empty slice refines nothing (cv2 refuses the empty crop; the engine skips
    # the window), as in tests/pages_ref.py
    wins = []
    for blk in blk_list:
        x1, y1, x2, y2 = postproc_ref.expand_textwindow(img.shape, blk.xyxy, expand_r=16)
        if x2 > x1 and y2 > y1:
            wins.append(blk.xyxy)
    mask_refined = postproc_ref.refine_mask(img, mask_u8, wins, refine_mode)
    if keep_undetected_mask:
        mask_refined = pipeline_ref.refine_undetected_mask(img, mask_u8, mask_refined, [k.xyxy for k in blk_list], None,
                                                           refine_mode)
    return mask_u8, mask_refined, blk_list


def golden_inputs(seed=0, net=256, nc=2):
    """the crafted float16 outputs of tests/golden/half_ref_256.npz, (blks [A][5 + nc], mask [1][H][W], lines
    [2][H][W]) of one net x net page, made to hit every half rule:
    * mask: every float16 value in [0, 1] (the 131 whose half product truncates differently among them), then
      random values;
    * lines: text-line bars at 0.9 ringed by pixels of exactly half(0.3) (background in half, foreground after
      .float()), on noise below 0.3;
    * blks: candidates with random half boxes (corners that round), class scores that tie after rounding, rows tied
      on score, and obj / class scores just around half(0.4)."""
    rng = np.random.default_rng(seed)
    a = 3 * ((net // 8) ** 2 + (net // 16) ** 2 + (net // 32) ** 2)
    unit = np.arange(0x3c01, dtype=np.uint16).view(np.float16)   # +0 .. 1.0
    mask = rng.uniform(0, 1, net * net).astype(np.float16)
    mask[:unit.size] = unit
    mask = mask.reshape(1, net, net)
    l0 = rng.uniform(0, 0.29, (net, net)).astype(np.float16)
    h03 = np.float16(0.3)
    for k in range(12):
        y, x = 12 + 20 * k, 16 + 13 * (k % 5)
        length = 60 + 9 * k
        l0[y - 1:y + 6, x - 1:x + length + 1] = h03
        l0[y:y + 5, x:x + length] = np.float16(0.9)
    lines = np.stack([l0, np.zeros_like(l0)])   # channel 1 (the threshold map) is never read
    b = np.zeros((a, 5 + nc), np.float16)
    b[:, 0:2] = rng.uniform(0, net, (a, 2))
    b[:, 2:4] = rng.uniform(0.01, 40, (a, 2))
    b[:, 4] = rng.uniform(0, 0.39, a)
    b[:, 5:] = rng.uniform(0, 1, (a, nc))
    cand = rng.choice(a, 400, replace=False)
    b[cand, 4] = rng.uniform(0.4, 1, cand.size)
    b[cand, 5] = rng.uniform(0.8, 1, cand.size)
    b[cand, 6] = rng.uniform(0, 1, cand.size)
    # class scores equal in half once multiplied, different in float: best class = the first in half
    b[cand[:40], 5] = np.float16(0.9)
    b[cand[:40], 6] = np.float16(0.9) + np.float16(0.0004)
    # obj / scores straddling half(0.4): the float product passes 0.4 where the half one does not
    b[cand[40:80], 4] = np.float16(0.40039062)
    b[cand[40:80], 5] = np.float16(0.9995)
    # rows that tie on score only in half (NMS order by row)
    b[cand[80:120], 4] = np.float16(0.75)
    b[cand[80:120], 5] = (np.float16(0.9) + rng.uniform(0, 0.0004, 40)).astype(np.float16)
    # corners that round in half: a large cx and a w whose half is far below its last place
    b[cand[120:200], 0] = rng.integers(130, 250, 80).astype(np.float16) + np.float16(0.125)
    b[cand[120:200], 2] = np.float16(0.0078125) * rng.integers(1, 60, 80).astype(np.float16)
    return b, mask, lines
