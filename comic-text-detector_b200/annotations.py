"""Annotation writer on top of the H100 detector: the on-disk formats of the reference's batch tool
`model2annotations` (inference.py:19-70) --

  <name>.txt        YOLO labels of the text blocks: "1 cx cy w h" per block, normalised, '\\n'-joined without a
                    trailing newline (imgproc_utils.py:22-29 `get_yololabel_strings`, :40-51 `xyxy2yolo`)
  line-<name>.txt   one text line per row, 8 integers x1 y1 .. x4 y4 (`np.savetxt(.., fmt='%d')`)
  <name>.json       `[blk.to_dict() ...]` through a numpy-aware JSON encoder (io_utils.py:16-28), optional
  <name>.png        the page re-encoded as PNG;  mask-<name>.png  the refined mask (io_utils.py:48-53 `imwrite`)

-- produced with refine_mode=REFINEMASK_ANNOTATION, keep_undetected_mask=True like the reference.  SURVEY 8f row f2.
`traverse_by_dict` reads such a directory back and refines each page's mask with the blocks of its json, as the
reference's second tool does.
"""
import glob
import json
import os
import os.path as osp
from collections import deque
from pathlib import Path

import numpy as np

from .inference import REFINEMASK_ANNOTATION, REFINEMASK_INPAINT, TextDetector
from .kernel_jobs import check_page, decode_files
from .png import is_png, png_probe
from .textblock import TextBlock

IMG_EXT = (".bmp", ".jpg", ".png", ".jpeg")


class NumpyEncoder(json.JSONEncoder):
    """arrays -> lists, numpy scalars -> Python scalars (io_utils.py:16-28)."""

    def default(self, obj):
        if isinstance(obj, np.ndarray):
            return obj.tolist()
        if isinstance(obj, np.bool_):
            return bool(obj)
        if isinstance(obj, np.floating):
            return float(obj)
        if isinstance(obj, np.integer):
            return int(obj)
        return json.JSONEncoder.default(self, obj)


def find_all_imgs(img_dir, abs_path=False):
    """io_utils.py:30-41: every file of `img_dir` whose suffix is an image extension, in glob order."""
    out = []
    for fp in glob.glob(osp.join(img_dir, "*")):
        name = osp.basename(fp)
        if Path(name).suffix.lower() in IMG_EXT:
            out.append(fp if abs_path else name)
    return out


def imread(path, read_type=None):
    import cv2
    return cv2.imdecode(np.fromfile(path, dtype=np.uint8), cv2.IMREAD_COLOR if read_type is None else read_type)


def png_path(img_path, ext=".png"):
    """io_utils.py:48-53's file name: the suffix is REPLACED by `ext` (first occurrence of the suffix string)."""
    suffix = Path(img_path).suffix
    return img_path.replace(suffix, ext) if suffix != "" else img_path + ext


def imwrite(img_path, img, ext=".png"):
    """io_utils.py:48-53"""
    import cv2
    cv2.imencode(ext, img)[1].tofile(png_path(img_path, ext))


def xyxy2yolo(xyxy, w, h):
    """imgproc_utils.py:40-51: [x1,y1,x2,y2] -> normalised [cx,cy,w,h] (float64); None for no boxes."""
    if len(xyxy) == 0:
        return None
    a = np.array(xyxy)
    if a.ndim == 1:
        a = a[None]
    yolo = np.copy(a).astype(np.float64)
    yolo[:, [0, 2]] = yolo[:, [0, 2]] / w
    yolo[:, [1, 3]] = yolo[:, [1, 3]] / h
    yolo[:, [2, 3]] -= yolo[:, [0, 1]]
    yolo[:, [0, 1]] += yolo[:, [2, 3]] / 2
    return yolo


def get_yololabel_strings(clslist, labellist):
    """imgproc_utils.py:22-29"""
    rows = [str(int(c)) + " " + " ".join(str(e) for e in xywh) for c, xywh in zip(clslist, labellist)]
    return "\n".join(rows)


def write_labels(save_dir, imgname, im_h, im_w, blk_list, save_json=False):
    """the text files of `write_annotations`: <name>.txt, line-<name>.txt (when there are lines), <name>.json"""
    imname = imgname.replace(Path(imgname).suffix, "")
    polys, blk_xyxy, blk_dicts = [], [], []
    for blk in blk_list:
        polys += blk.lines
        blk_xyxy.append(blk.xyxy)
        blk_dicts.append(blk.to_dict())
    yolo = xyxy2yolo(blk_xyxy, im_w, im_h)
    label = get_yololabel_strings([1] * len(yolo), yolo) if yolo is not None else ""
    with open(osp.join(save_dir, imname + ".txt"), "w", encoding="utf8") as f:
        f.write(label)
    if len(polys) != 0:
        np.savetxt(osp.join(save_dir, "line-" + imname + ".txt"), np.array(polys).reshape(-1, 8), fmt="%d")
    if save_json:
        with open(osp.join(save_dir, imname + ".json"), "w", encoding="utf8") as f:
            f.write(json.dumps(blk_dicts, ensure_ascii=False, cls=NumpyEncoder))
    return imname


def write_annotations(save_dir, imgname, img, mask_refined, blk_list, save_json=False):
    """The per-page part of `model2annotations` (inference.py:33-70) for an already detected page, PNGs by cv2."""
    im_h, im_w = img.shape[:2]
    imname = write_labels(save_dir, imgname, im_h, im_w, blk_list, save_json)
    imwrite(osp.join(save_dir, imgname), img)
    imwrite(osp.join(save_dir, "mask-" + imname + ".png"), mask_refined)


def _read_pages(imglist, det, failed):
    """(path, page) for each file in order, decoded in batches of det.max_batch as the detector decodes encoded pages
    (baseline JPEGs and PNGs on the GPU into CUDA pages, every other file by cv2).  A file that cannot be read ends the pages
    there: its error goes to `failed`."""
    for b0 in range(0, len(imglist), det.max_batch):
        paths = imglist[b0:b0 + det.max_batch]
        pages = decode_files([np.fromfile(p, dtype=np.uint8) for p in paths], det.png_decoder, det.jpeg_decoder)
        for img_path, img in zip(paths, pages):
            try:
                img = check_page(img, det.device_index)
            except ValueError as ex:
                failed.append(ValueError("%s: %s" % (img_path, ex)))
                return
            yield img_path, img


def model2annotations(model_path, img_dir_list, save_dir, save_json=False, detector=None):
    """`model2annotations(model_path, img_dir_list, save_dir, save_json)` of the reference (inference.py:19-70).

    The files are those `write_annotations` writes page by page, byte for byte.  Pages are read in batches of the
    detector's max_batch and decoded with its JpegDecoder and PngDecoder; a page decoded on the GPU stays there for the
    detection and for its PNG, so a directory of PNG pages (such as this tool's own output) is read on the GPU too.  The refined masks stay on the GPU (detect_stream's device_results), and both PNGs of every page of
    a batch of results are encoded in one PngEncoder call."""
    from .png import PngEncoder
    if isinstance(img_dir_list, str):
        img_dir_list = [img_dir_list]
    # batches of up to 8 pages (scripts/pages_bench.py: the fastest of the measured batch sizes)
    det = detector if detector is not None else TextDetector(model_path=model_path, input_size=1024, act="leaky",
                                                             max_batch=8)
    os.makedirs(save_dir, exist_ok=True)
    enc = None
    try:
        imglist = []
        for d in img_dir_list:
            imglist += find_all_imgs(d, abs_path=True)
        enc = PngEncoder(det.device_index)
        # pages are decoded while the previous batches run on the GPU (TextDetector.detect_stream); results come back
        # in input order, so each one is written with the page it belongs to.  A page that cannot be read ends the
        # stream there: every page before it is still written, then the error is raised, as page by page.
        read, failed, done = deque(), [], []

        def pages():
            for img_path, img in _read_pages(imglist, det, failed):
                read.append((img_path, img))
                yield img

        def flush():
            files = enc.encode([x for _p, img, mask, _b in done for x in (img, mask)])
            for k, (img_path, img, _mask, blk_list) in enumerate(done):
                imgname = osp.basename(img_path)
                imname = write_labels(save_dir, imgname, img.shape[0], img.shape[1], blk_list, save_json)
                files[2 * k].tofile(png_path(osp.join(save_dir, imgname)))
                files[2 * k + 1].tofile(png_path(osp.join(save_dir, "mask-" + imname + ".png")))
            done.clear()

        for _mask, mask_refined, blk_list in det.detect_stream(pages(), refine_mode=REFINEMASK_ANNOTATION,
                                                                keep_undetected_mask=True, device_results=True):
            img_path, img = read.popleft()
            done.append((img_path, img, mask_refined, blk_list))
            if len(done) == det.max_batch:
                flush()
        if done:
            flush()
        if failed:
            raise failed[0]
    finally:
        if enc is not None:
            enc.close()
        if detector is None:
            det.close()


def read_grey(bufs, png_decoder):
    """encoded masks (1-D np.uint8 arrays) -> what `cv2.imdecode(buf, cv2.IMREAD_GRAYSCALE)` returns for each: for a
    greyscale PNG (colour type 0) the GPU decodes, channel 0 of png_decoder()'s page (a strided CUDA view; cv2 reads
    such a file to equal grey and colour pages), for every other file cv2's grey decode on the host"""
    import cv2
    grey = [i for i, b in enumerate(bufs) if is_png(b) and png_probe(b)["color_type"] == 0]
    out = [None] * len(bufs)
    if grey:
        for i, page in zip(grey, png_decoder().decode([bufs[i] for i in grey])):
            out[i] = None if page is None else page[..., 0]
    for i, b in enumerate(bufs):
        if out[i] is None:
            out[i] = cv2.imdecode(b, cv2.IMREAD_GRAYSCALE)
    return out


def traverse_by_dict(img_dir_list, dict_dir, refiner=None):
    """The reference's `traverse_by_dict(img_dir_list, dict_dir)` (inference.py:180-200) without its display: for
    every image of `img_dir_list` in `find_all_imgs` order, the blocks of `dict_dir/<name>.json` (`TextBlock(**d)` for
    each dict; FileNotFoundError when it is missing) and the mask `dict_dir/mask-<name>.png` (read as
    `cv2.imread(path, IMREAD_GRAYSCALE)` reads it) refine the page's mask with REFINEMASK_INPAINT.  A generator of
    `(img_path, img, mask_refined, blk_list)`: img is the page as decoded (a CUDA tensor where the GPU decodes it, else
    cv2's numpy page), mask_refined a numpy array equal to the reference's `refine_mask(img, mask, blk_list)`.

    Pages and masks are read in batches of the refiner's max_batch (a MaskRefiner; one is made and closed here when
    none is given) and decoded on the GPU where it takes them (JPEG and PNG pages, greyscale PNG masks)."""
    from .textmask import MaskRefiner
    if isinstance(img_dir_list, str):
        img_dir_list = [img_dir_list]
    ref = refiner if refiner is not None else MaskRefiner()
    try:
        imglist = []
        for d in img_dir_list:
            imglist += find_all_imgs(d, abs_path=True)
        read = deque()

        def items():
            for b0 in range(0, len(imglist), ref.max_batch):
                paths = imglist[b0:b0 + ref.max_batch]
                blks, mask_paths = [], []
                for img_path in paths:
                    imgname = osp.basename(img_path)
                    imname = imgname.replace(Path(imgname).suffix, "")
                    mask_paths.append(osp.join(dict_dir, "mask-" + imname + ".png"))
                    with open(osp.join(dict_dir, imname + ".json"), "r", encoding="utf8") as f:
                        blks.append([TextBlock(**d) for d in json.loads(f.read())])
                pages = decode_files([np.fromfile(p, dtype=np.uint8) for p in paths], ref.png_decoder, ref.jpeg_decoder)
                masks = read_grey([np.fromfile(p, dtype=np.uint8) for p in mask_paths], ref.png_decoder)
                for img_path, img, mask_path, mask, blk_list in zip(paths, pages, mask_paths, masks, blks):
                    if img is None:
                        raise ValueError("%s could not be decoded (cv2.imdecode returns None)" % img_path)
                    if mask is None:
                        raise ValueError("%s could not be decoded (cv2.imdecode returns None)" % mask_path)
                    read.append((img_path, img, blk_list))
                    yield img, mask, blk_list

        for _mask, mask_refined in ref.refine_stream(items(), refine_mode=REFINEMASK_INPAINT):
            img_path, img, blk_list = read.popleft()
            yield img_path, img, mask_refined, blk_list
    finally:
        if refiner is None:
            ref.close()
