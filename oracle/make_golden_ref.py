"""TEST INFRASTRUCTURE ONLY (oracle): goldens the UNMODIFIED reference produces for the tests that compare with it,
so that those comparisons also run where the reference tree is absent:

* tests/golden/seg_represent_ref.npz: `SegDetectorRepresenter(thresh=0.3)` boxes / scores for every map of
  tests/stress_maps.CASES;
* tests/golden/annotations_ref.json: per seed of tests/test_cpu_annotations.py, the files the reference's
  `model2annotations` per-page body writes (sha256 of each file; the parsed content of the .json file);
* tests/golden/net_ref_128x192.npz: the reference `TextDetBase` forward (blks, mask, lines) on the page and
  checkpoint of tests/test_cpu_oracle.py::test_net_ref_is_bit_identical_to_reference.

Needs the reference tree (oracle/ref_shim.py).  Usage, from the repository root:
    python -m oracle.make_golden_ref
"""
import hashlib
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
GOLD = os.path.join(ROOT, "tests", "golden")


def seg_represent(ns):
    import stress_maps
    rep = ns.db_utils.SegDetectorRepresenter(thresh=0.3)
    out = {}
    for name, f in stress_maps.CASES.items():
        b, s = rep(None, torch.from_numpy(f())[None, None])
        out["boxes_" + name] = np.asarray(b[0])
        out["scores_" + name] = np.asarray(s[0])
    np.savez_compressed(os.path.join(GOLD, "seg_represent_ref.npz"), **out)


def annotations(ns):
    from test_cpu_annotations import SEEDS, _reference_page_writer, annotation_case
    out = {}
    for seed in SEEDS:
        name, img, mask, blks, lines, w, h = annotation_case(seed)
        theirs = ns.textblock.group_output(blks, lines, w, h, mask.copy())
        with tempfile.TemporaryDirectory() as d:
            _reference_page_writer(ns, d, name, img, mask, theirs, True)
            files = {}
            for f in sorted(os.listdir(d)):
                data = open(os.path.join(d, f), "rb").read()
                files[f] = {"sha256": hashlib.sha256(data).hexdigest()}
                if f.endswith(".json"):
                    files[f]["json"] = json.loads(data)
        out[str(seed)] = files
    json.dump(out, open(os.path.join(GOLD, "annotations_ref.json"), "w"), indent=0, sort_keys=True)


def net(ns):
    from oracle import synth
    from util import page_to_net_input
    ck = synth.make_checkpoint(0, smooth=False, bn_calibrate=128)
    with tempfile.TemporaryDirectory() as d:
        f = os.path.join(d, "ck.pt")
        torch.save(ck, f)
        model = ns.basemodel.TextDetBase(f, device="cpu", act="leaky")
    x = page_to_net_input(np.stack([synth.structured_page(3, 128, 192)]))
    with torch.no_grad():
        b, m, l = model(x)
    np.savez_compressed(os.path.join(GOLD, "net_ref_128x192.npz"), blks=b.numpy(), mask=m.numpy(), lines=l.numpy())


def main():
    from oracle import ref_shim
    assert ref_shim.available(), "needs the reference tree (see oracle/ref_shim.py)"
    ns = ref_shim.load()
    seg_represent(ns)
    annotations(ns)
    net(ns)
    for f in ("seg_represent_ref.npz", "annotations_ref.json", "net_ref_128x192.npz"):
        print("wrote", f, os.path.getsize(os.path.join(GOLD, f)), "bytes")


if __name__ == "__main__":
    main()
