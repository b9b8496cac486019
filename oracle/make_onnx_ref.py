"""TEST INFRASTRUCTURE ONLY (oracle): the reference's ONNX model and what its OpenCV-DNN backend computes on it.

The reference ships its detector as an ONNX file too, run through `cv2.dnn` (`TextDetBaseDNN`, basemodel.py:246-256,
picked from the suffix in inference.py:124-130).  This recipe makes such a file from the synthetic checkpoint and
records the unmodified reference's results on it, for tests/test_cpu_onnx.py and tests/test_gpu_onnx.py:

* `export(size)` restates `export_onnx`'s module edits (utils/export.py:30-47: export-friendly SiLU, Detect with
  inplace=False and onnx_dynamic=False) and writes `TextDetBase(synth.make_checkpoint(0))` at opset 11 with constant
  folding and the names images / blk, seg, det, as examples.ipynb does, through torch's TorchScript exporter.  The
  exporter's one import of the `onnx` package (the hook that inserts custom onnxscript functions, of which this model
  has none) is bypassed; nothing else is changed.
* for input sizes 512 and 1024, `oracle/_ref/ctd_<size>.onnx` plus `oracle/_ref/onnx_ref_<size>.npz` /
  `onnx_ref_<size>.json`: the `cv2.dnn` net outputs (blk, seg, det as `TextDetBaseDNN.__call__` returns them) and the
  full `(mask, mask_refined, blk_list)` of the reference's `TextDetector(model_path=<onnx>)` on seeded
  `synth.structured_page`s, net-sized and not, with keep_undetected_mask off and on.

`build()` runs it when the reference tree exists; elsewhere it does nothing.  Usage, from the repository root:
    python -m oracle.make_onnx_ref [size ...]
"""
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "oracle", "_ref")
SIZES = (512, 1024)
CKPT_SEED = 0

# (seed, h, w, keep_undetected_mask) per input size: net-sized pages and pages of other shapes.  The reference's
# refine_mask raises on a block with an empty window, which many synthetic pages of other shapes have; these are pages
# it completes (a page where it raises is recorded with the error and no results)
PAGES = {
    512: [(31, 512, 512, False), (32, 512, 512, True), (32, 640, 640, True), (33, 380, 610, False),
          (34, 820, 560, True), (36, 300, 300, False)],
    1024: [(41, 1024, 1024, False), (42, 1024, 1024, True), (43, 1280, 1280, True), (44, 600, 600, False)],
}


def onnx_path(size):
    return os.path.join(OUT, "ctd_%d.onnx" % size)


def results_paths(size):
    return os.path.join(OUT, "onnx_ref_%d.npz" % size), os.path.join(OUT, "onnx_ref_%d.json" % size)


def export(ns, size, path):
    """export_onnx (utils/export.py:30-47) without onnx.checker / onnxsim, which need the onnx package."""
    import torch
    import torch.nn as nn
    from torch.onnx._internal.torchscript_exporter import onnx_proto_utils
    from oracle import synth

    class SiLU(nn.Module):  # export-friendly version of nn.SiLU() (utils/export.py:18-21)
        @staticmethod
        def forward(x):
            return x * torch.sigmoid(x)

    ck = synth.make_checkpoint(CKPT_SEED)
    with tempfile.TemporaryDirectory() as d:
        f = os.path.join(d, "ck.pt")
        torch.save(ck, f)
        model = ns.basemodel.TextDetBase(f, device="cpu", act="leaky").eval()
    for _k, m in model.named_modules():
        if isinstance(m, ns.common.Conv):
            if isinstance(m.act, nn.SiLU):
                m.act = SiLU()
        elif isinstance(m, ns.yolo.Detect):
            m.inplace = False
            m.onnx_dynamic = False
    im = torch.zeros(1, 3, size, size)
    hook = onnx_proto_utils._add_onnxscript_fn
    onnx_proto_utils._add_onnxscript_fn = lambda model_bytes, custom_opsets: model_bytes
    try:
        torch.onnx.export(model, im, path, verbose=False, opset_version=11, training=torch.onnx.TrainingMode.EVAL,
                          do_constant_folding=True, input_names=["images"], output_names=["blk", "seg", "det"],
                          dynamo=False)
    finally:
        onnx_proto_utils._add_onnxscript_fn = hook


def reference_results(ns, size, path):
    """the unmodified reference opencv backend on PAGES[size]"""
    from oracle import synth
    det = ns.inference.TextDetector(model_path=path, input_size=size, device="cpu", act="leaky")
    assert det.backend == "opencv"
    arrays, meta = {}, []
    for k, (seed, h, w, keep) in enumerate(PAGES[size]):
        page = synth.structured_page(seed, h, w)
        img_in, _ratio, _dw, _dh = ns.inference.preprocess_img(page, input_size=det.input_size, to_tensor=False)
        # cv2 returns the outputs in its own order (the reference swaps them back, inference.py:151-155): they are
        # named here by shape, blk [1][A][no], seg [1][1][S][S], det [1][2][S][S]
        for o in det.net(img_in):
            arrays["%s_%d" % ("blk" if o.ndim == 3 else "seg" if o.shape[1] == 1 else "det", k)] = o
        try:
            mask, mask_refined, blk_list = det(page.copy(), keep_undetected_mask=keep)
        except Exception as ex:   # the reference's refine_mask fails on a block whose window is empty
            meta.append(dict(seed=seed, h=h, w=w, keep_undetected_mask=keep, error=repr(ex)))
            continue
        arrays.update({"mask_%d" % k: mask, "mask_refined_%d" % k: mask_refined})
        meta.append(dict(seed=seed, h=h, w=w, keep_undetected_mask=keep,
                         blocks=[dict(xyxy=[int(v) for v in b.xyxy], lines=np.array(b.lines).astype(int).tolist(),
                                      language=b.language, vertical=bool(b.vertical), font_size=float(b.font_size),
                                      angle=int(b.angle)) for b in blk_list]))
    return arrays, meta


def make(ns, size):
    os.makedirs(OUT, exist_ok=True)
    path = onnx_path(size)
    if all(os.path.isfile(p) for p in (path,) + results_paths(size)):
        print("make_onnx_ref: %s and its results exist" % os.path.relpath(path, ROOT))
        return
    export(ns, size, path)
    arrays, meta = reference_results(ns, size, path)
    npz, js = results_paths(size)
    np.savez_compressed(npz, **arrays)
    with open(js, "w") as f:
        json.dump(dict(size=size, ckpt_seed=CKPT_SEED, pages=meta), f, indent=1)
    for p in (path, npz, js):
        print("wrote", os.path.relpath(p, ROOT), os.path.getsize(p), "bytes")


def main(sizes=SIZES):
    from oracle import ref_shim
    if not ref_shim.available():
        print("make_onnx_ref: no reference tree, nothing to do")
        return
    ns = ref_shim.load()
    for size in sizes:
        make(ns, int(size))


if __name__ == "__main__":
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    main(sys.argv[1:] or SIZES)
