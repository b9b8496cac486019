"""not-gpu: the annotation writer (comic-text-detector_b200/annotations.py, SURVEY 8f row f2) against the UNMODIFIED
reference's own writer code path (`model2annotations`' per-page body, inference.py:33-70, run with the reference's
TextBlock / xyxy2yolo / get_yololabel_strings / NumpyEncoder / imwrite) on identical grouping results: every file
byte-identical.  Live against the reference tree where it is present, always against the goldens it produced;
the format itself is also checked stand-alone."""
import hashlib
import json
import os
import os.path as osp
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ctd_b200 import annotations as ann  # noqa: E402
from ctd_b200 import textblock as tb  # noqa: E402
from oracle import ref_shim  # noqa: E402
from test_cpu_textblock import make_case  # noqa: E402

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="/root/reference not present on this box")


def _reference_page_writer(ns, save_dir, imgname, img, mask_refined, blk_list, save_json):
    """inference.py:33-70 with the reference's own helpers (nothing of ours on this path)."""
    from pathlib import Path
    io_utils = sys.modules["utils.io_utils"]
    ip = ns.imgproc_utils
    im_h, im_w = img.shape[:2]
    imname = imgname.replace(Path(imgname).suffix, '')
    polys, blk_xyxy, blk_dict_list = [], [], []
    for blk in blk_list:
        polys += blk.lines
        blk_xyxy.append(blk.xyxy)
        blk_dict_list.append(blk.to_dict())
    blk_xyxy = ip.xyxy2yolo(blk_xyxy, im_w, im_h)
    yolo_label = ip.get_yololabel_strings([1] * len(blk_xyxy), blk_xyxy) if blk_xyxy is not None else ''
    with open(osp.join(save_dir, imname + '.txt'), 'w', encoding='utf8') as f:
        f.write(yolo_label)
    if len(polys) != 0:
        np.savetxt(osp.join(save_dir, 'line-' + imname + '.txt'), np.array(polys).reshape(-1, 8), fmt='%d')
    if save_json:
        with open(osp.join(save_dir, imname + '.json'), 'w', encoding='utf8') as f:
            f.write(json.dumps(blk_dict_list, ensure_ascii=False, cls=io_utils.NumpyEncoder))
    io_utils.imwrite(osp.join(save_dir, imgname), img)
    io_utils.imwrite(osp.join(save_dir, 'mask-' + imname + '.png'), mask_refined)


SEEDS = [0, 3, 5, 11, 17]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "annotations_ref.json")


def annotation_case(seed):
    """(file name, page, mask_refined, grouping input) of one seed: the same inputs on both writers."""
    blks, lines, w, h, mask = make_case(seed)
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    return ("page %d.jpg" % seed, img, mask, (blks[0].copy(), blks[1].copy(), blks[2].copy()),
            lines.copy() if len(lines) else [], w, h)


def _write_ours(d, seed):
    name, img, mask, blks, lines, w, h = annotation_case(seed)
    ours = tb.group_output(blks, lines, w, h, mask.copy())
    ann.write_annotations(str(d), name, img, mask, ours, save_json=True)


def _assert_json_equal(f, ja, jb):
    """same blocks, same keys, same values (key ORDER follows each class's attribute order)"""
    assert len(ja) == len(jb)
    for x, y in zip(ja, jb):
        for k in y:
            assert k in x, (f, k)
            if k in ("distance", "vec", "norm", "weight", "font_size"):
                # float fields of the native group_output: glibc acos/sin vs numpy's SIMD kernels may differ in
                # the last ulp; the TYPE written (int vs float) must still agree
                assert type(x[k]) is type(y[k]), (f, k, x[k], y[k])
                assert np.allclose(np.array(x[k], np.float64), np.array(y[k], np.float64), rtol=1e-12, atol=0,
                                   equal_nan=True), (f, k)
            else:
                assert x[k] == y[k], (f, k)


@needs_ref
@pytest.mark.parametrize("seed", SEEDS)
def test_files_equal_reference_writer(tmp_path, seed):
    ns = ref_shim.load()
    name, img, mask, blks, lines, w, h = annotation_case(seed)
    theirs = ns.textblock.group_output(blks, lines, w, h, mask.copy())
    da, db = tmp_path / "ours", tmp_path / "ref"
    da.mkdir(); db.mkdir()
    _write_ours(da, seed)
    _reference_page_writer(ns, str(db), name, img, mask, theirs, True)
    fa, fb = sorted(os.listdir(da)), sorted(os.listdir(db))
    assert fa == fb and len(fa) >= 4
    for f in fa:
        a, b = (da / f).read_bytes(), (db / f).read_bytes()
        if f.endswith(".json"):
            _assert_json_equal(f, json.loads(a), json.loads(b))
        else:
            assert a == b, f


@pytest.mark.parametrize("seed", SEEDS)
def test_files_equal_reference_goldens(tmp_path, seed):
    """the same comparison against what the reference's writer produced for these inputs
    (tests/golden/annotations_ref.json, written by oracle/make_golden_ref.py): file names, the bytes of every
    non-JSON file (sha256) and the JSON content"""
    gold = json.load(open(GOLDEN))[str(seed)]
    _write_ours(tmp_path, seed)
    assert sorted(os.listdir(tmp_path)) == sorted(gold)
    for f, g in gold.items():
        data = (tmp_path / f).read_bytes()
        if f.endswith(".json"):
            _assert_json_equal(f, json.loads(data), g["json"])
        else:
            assert hashlib.sha256(data).hexdigest() == g["sha256"], f


def test_label_and_line_formats(tmp_path):
    blk = tb.TextBlock([10, 20, 110, 220], lines=[[[10, 20], [110, 20], [110, 60], [10, 60]]])
    img = np.zeros((400, 200, 3), np.uint8)
    ann.write_annotations(str(tmp_path), "p.png", img, np.zeros((400, 200), np.uint8), [blk], save_json=True)
    assert (tmp_path / "p.txt").read_text() == "1 0.3 0.3 0.5 0.5"
    assert (tmp_path / "line-p.txt").read_text() == "10 20 110 20 110 60 10 60\n"
    assert json.loads((tmp_path / "p.json").read_text())[0]["xyxy"] == [10, 20, 110, 220]
    assert (tmp_path / "p.png").exists() and (tmp_path / "mask-p.png").exists()
    ann.write_annotations(str(tmp_path), "q.jpg", img, np.zeros((400, 200), np.uint8), [], save_json=False)
    assert (tmp_path / "q.txt").read_text() == "" and not (tmp_path / "line-q.txt").exists()
    assert ann.find_all_imgs(str(tmp_path)) and all(f.endswith(".png") for f in ann.find_all_imgs(str(tmp_path)))
