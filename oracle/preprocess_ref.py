"""Restatement of the reference's `preprocess_img` (inference.py:72-83) and the `letterbox` it calls
(utils/imgproc_utils.py:86-117, auto=False, scaleup=True) with cv2 + numpy + torch, for the tests of
`ctd_b200.preprocess_img` / `Preprocessor`.  Pinned against the reference itself in tests/test_cpu_preprocess.py."""
import cv2
import numpy as np
import torch


def letterbox_size(shape_hw, new_shape):
    """(r, (unpad_w, unpad_h), dw, dh): r = min(H / h, W / w), the resized size round(size * r) with Python's round
    (half to even), and the bottom / right padding"""
    r = min(new_shape[0] / shape_hw[0], new_shape[1] / shape_hw[1])
    new_unpad = int(round(shape_hw[1] * r)), int(round(shape_hw[0] * r))
    return r, new_unpad, new_shape[1] - new_unpad[0], new_shape[0] - new_unpad[1]


def preprocess_img(img, input_size=(1024, 1024), device='cpu', bgr2rgb=True, half=False, to_tensor=True):
    """-> (img_in, (r, r), dw, dh): img_in float32 (float16 with half) [1][3][H][W] on `device`, or with
    to_tensor=False the letterboxed u8 [H][W][3] page as numpy"""
    if not isinstance(input_size, tuple):
        input_size = (input_size, input_size)
    if bgr2rgb:
        img = cv2.cvtColor(img, cv2.COLOR_BGR2RGB)
    r, (uw, uh), dw, dh = letterbox_size(img.shape[:2], input_size)
    if (img.shape[1], img.shape[0]) != (uw, uh):
        img = cv2.resize(img, (uw, uh), interpolation=cv2.INTER_LINEAR)
    out = np.zeros((input_size[0], input_size[1], 3), np.uint8)
    out[:uh, :uw] = img
    if not to_tensor:
        return out, (r, r), int(dw), int(dh)
    chw = np.ascontiguousarray(out.transpose(2, 0, 1)[::-1])
    x = torch.from_numpy(chw[None].astype(np.float32) / np.float32(255)).to(device)
    if half:
        x = x.half()
    return x, (r, r), int(dw), int(dh)
