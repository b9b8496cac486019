"""not-gpu: `.onnx` models (comic-text-detector_b200/onnx_model.py) -- the protobuf reader against OpenCV's own parse,
the checkpoint recovered from the graph against the source checkpoint, the compiled program interpreted on the CPU
against OpenCV DNN's forward, the refusals, and the `.pt` compiler's output pinned to its hash.

The models and OpenCV's outputs come from oracle/make_onnx_ref.py (run by build() where the reference tree exists);
the tests that need them skip, naming the missing file, when they are absent."""
import hashlib
import json
import os

import numpy as np
import pytest

import ctd_b200
from ctd_b200 import compiler as cc
from ctd_b200 import onnx_model as om
from oracle import synth
from prog_interp import run_program

REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")
SIZE = 512


def _ref_file(name):
    p = os.path.join(REF, name)
    if not os.path.isfile(p):
        pytest.skip("%s is missing (made by oracle/make_onnx_ref.py where the reference tree exists)" % p)
    return p


@pytest.fixture(scope="module")
def onnx_file():
    return _ref_file("ctd_%d.onnx" % SIZE)


@pytest.fixture(scope="module")
def recovered(onnx_file):
    return om.load_checkpoint(onnx_file)


@pytest.fixture(scope="module")
def programs(recovered):
    ck, act, _s = recovered
    return cc.compile_checkpoint(ck, act), cc.compile_checkpoint(synth.make_checkpoint(0), "leaky")


# ---- reader ---------------------------------------------------------------------------------------------------
def test_reader_matches_opencv_parse(onnx_file):
    """every Convolution, Deconvolution and BatchNorm parameter the reader returns equals cv2's bit for bit"""
    import cv2
    g = om.read_model(onnx_file)
    net = cv2.dnn.readNetFromONNX(onnx_file)
    order = {"Conv": (1, 2), "ConvTranspose": (1, 2), "BatchNormalization": (3, 4, 1, 2)}  # cv2 BN: mean, var, w, b
    n = 0
    for node in g.nodes:
        if node.op_type not in order:
            continue
        lid = net.getLayerId("onnx_node!" + node.name)
        assert lid >= 0, node
        ours = [g.initializers[node.inputs[i]] for i in order[node.op_type] if i < len(node.inputs)]
        assert len(net.getLayer(lid).blobs) == len(ours), node
        for k, a in enumerate(ours):
            b = net.getParam(lid, k)
            assert a.dtype == np.float32 and a.size == b.size, node
            assert np.array_equal(a.reshape(-1).view(np.uint32), b.reshape(-1).view(np.uint32)), (node, k)
        n += 1
    assert n == 103 + 12 + 9   # every conv, every ConvTranspose and the nine BatchNorms that stay nodes


def _varint(x):
    out = bytearray()
    while True:
        b = x & 0x7F
        x >>= 7
        out.append(b | (0x80 if x else 0))
        if not x:
            return bytes(out)


def _field(num, val):
    """protobuf field: int -> varint, bytes -> length-delimited"""
    if isinstance(val, int):
        return _varint(num << 3) + _varint(val)
    return _varint(num << 3 | 2) + _varint(len(val)) + val


def _model(graph_fields):
    return _field(1, 7) + _field(8, _field(2, 11)) + _field(7, b"".join(graph_fields))


def _input(name, dims):
    shape = b"".join(_field(1, _field(1, d) if isinstance(d, int) else _field(2, d.encode())) for d in dims)
    return _field(11, _field(1, name.encode()) + _field(2, _field(1, _field(1, 1) + _field(2, shape))))


def test_reader_tensor_encodings():
    raw = np.arange(6, dtype=np.float32).reshape(2, 3)
    t_raw = _field(1, 2) + _field(1, 3) + _field(2, 1) + _field(8, b"raw") + _field(9, raw.tobytes())
    t_flt = _field(1, 2) + _field(2, 1) + _field(8, b"flt") + _field(4, np.float32([1.5, -2]).tobytes())
    t_i64 = _field(1, 3) + _field(2, 7) + _field(8, b"i64") + _field(7, b"".join(_varint(v % (1 << 64)) for v in (4, -1, 7)))
    g = om.read_model(_model([_field(5, t) for t in (t_raw, t_flt, t_i64)]))
    assert np.array_equal(g.initializers["raw"], raw)
    assert np.array_equal(g.initializers["flt"], np.float32([1.5, -2]))
    assert g.initializers["i64"].tolist() == [4, -1, 7]


@pytest.mark.parametrize("tensor, msg", [
    (_field(1, 2) + _field(2, 1) + _field(8, b"ext") + _field(14, 1), "external file"),
    (_field(1, 2) + _field(2, 8) + _field(8, b"str"), "data type 8"),
    (_field(1, 4) + _field(2, 1) + _field(8, b"short") + _field(9, b"\0" * 8), "raw_data has 8 bytes"),
])
def test_reader_refuses_tensors(tensor, msg):
    with pytest.raises(ValueError, match=msg):
        om.read_model(_model([_field(5, tensor)]))


def test_reader_refuses_truncated_and_corrupt_files(onnx_file):
    data = open(onnx_file, "rb").read()
    for cut in (len(data) // 2, len(data) - 1, 5):
        with pytest.raises(ValueError, match="truncated"):
            om.read_model(data[:cut])
    with pytest.raises(ValueError, match="empty"):
        om.read_model(b"")
    with pytest.raises(ValueError, match="corrupt|truncated|no graph"):
        om.read_model(b"\x0f" + data[1:64])


@pytest.mark.parametrize("dims, msg", [([1, 3, "height", "width"], "fixed at export"),
                                       ([1, 3, 512, 640], "square")])
def test_refuses_dynamic_and_non_square_inputs(dims, msg):
    with pytest.raises(ValueError, match=msg):
        om.checkpoint_from_graph(om.read_model(_model([_input("images", dims)])))


# ---- graph -> checkpoint -> program ---------------------------------------------------------------------------
def test_recovered_cfg(recovered):
    ck, act, size = recovered
    cfg = ck["blk_det"]["cfg"]
    src = synth.YOLOV5S_CFG
    assert size == SIZE and act == "leaky"
    assert (cfg["nc"], cfg["width_multiple"], cfg["depth_multiple"]) == (src["nc"], src["width_multiple"], src["depth_multiple"])
    assert cfg["anchors"] == src["anchors"]
    assert cc.parse_cfg(cfg) == cc.parse_cfg(src)
    assert np.array_equal(ck["blk_det"]["weights"]["model.24.anchors"],
                          synth.make_checkpoint(0)["blk_det"]["weights"]["model.24.anchors"].numpy())


def _weights(P, op):
    """float32 views of every weight / bias / parameter region an op reads"""
    f = lambda off, n: np.frombuffer(P.blob, np.float32, n, off)
    k, cin = op["kind"], sum(op["src_c"][:op["n_src"]])
    if k == cc.OP_STEM:
        return [f(op["w32_off"], op["cout"] * 108).reshape(op["cout"], 6, 6, 3), f(op["b_off"], op["cout"])]
    if k in (cc.OP_CONV, cc.OP_DETECT, cc.OP_DECONV4):
        K = 16 * cin if k == cc.OP_DECONV4 else op["ksize"] ** 2 * cin
        out = [f(op["w32_off"], op["cout_pad"] * K), f(op["b_off"], op["cout_pad"])]
        return out + ([f(op["p_off"], 7)] if k == cc.OP_DETECT else [])
    if k == cc.OP_SEG_TAIL:
        return [f(op["p_off"], 16 * cin)]
    if k == cc.OP_DB_TAIL:
        return [f(op["p_off"], 2 * 1105)]
    return []


def test_program_equals_pt_program_but_for_weight_rounding(programs):
    """Same buffers and op list, field for field; the stem is the source stem with its input channels reversed; every
    weight agrees within the float32 rounding of the exporter's Conv + BatchNorm folding.  Bound: 2^-21 of the
    tensor's largest magnitude (the exporter folds w * gamma / sqrt(var + eps) and beta - mu * scale with a few
    float32 roundings of 2^-24 each; the compiler folds in float64 and rounds once; measured: 1.6e-7 = 2.7 * 2^-24)."""
    po, pp = programs
    assert po.bufs == pp.bufs and po.nc == pp.nc
    assert po.ops == pp.ops            # kinds, sources, destinations, shapes, activations and blob offsets
    assert len(po.blob) == len(pp.blob)
    worst = 0.0
    for a, b in zip(po.ops, pp.ops):
        wa, wb = _weights(po, a), _weights(pp, b)
        if a["kind"] == cc.OP_STEM:
            wb[0] = wb[0][..., ::-1]
            assert np.abs(wa[0] - _weights(pp, b)[0]).max() > 1e-2   # reversing the channels is not a no-op
        for x, y in zip(wa, wb):
            err = float(np.abs(x - y).max() / max(np.abs(y).max(), 1e-30))
            worst = max(worst, err)
    assert worst < 2.0 ** -21, worst


def test_emulated_forward_matches_opencv_dnn(programs):
    """The ONNX program interpreted in fp32 (tests/prog_interp.py) on the BGR page against what cv2.dnn computed on
    the reference's RGB blob.  Tolerance 1e-3, the bound the `.pt` program is held to against the torch forward
    (cv2.dnn and torch differ by up to 5.6e-4 on the net maps; this distance measured 1.4e-4 at 256 px)."""
    arrs = np.load(_ref_file("onnx_ref_%d.npz" % SIZE))
    meta = json.load(open(_ref_file("onnx_ref_%d.json" % SIZE)))
    k = next(i for i, p in enumerate(meta["pages"]) if (p["h"], p["w"]) == (SIZE, SIZE))
    p = meta["pages"][k]
    page = synth.structured_page(p["seed"], p["h"], p["w"])
    blks, mask, lines = run_program(programs[0], page[None])
    assert float(np.abs(mask.numpy() - arrs["seg_%d" % k]).max()) < 1e-3
    assert float(np.abs(lines.numpy() - arrs["det_%d" % k]).max()) < 1e-3
    rb = arrs["blk_%d" % k]
    assert float((np.abs(blks.numpy() - rb) / (np.abs(rb) + 1)).max()) < 1e-3


# ---- refusals -------------------------------------------------------------------------------------------------
def test_refuses_unsupported_node(onnx_file):
    data = open(onnx_file, "rb").read()
    assert data.count(b"MaxPool") >= 3
    with pytest.raises(ValueError, match=r"MinPool node '/blk_det/model\.9/m_2/MinPool'"):
        om.load_checkpoint(data.replace(b"MaxPool", b"MinPool"))


def test_refuses_mismatched_input_size(onnx_file):
    """raised while reading the model, before an engine exists"""
    with pytest.raises(ValueError, match="exported for 512 x 512 input"):
        ctd_b200.TextDetector(onnx_file, input_size=1024)


# ---- the `.pt` compiler stays byte-identical ------------------------------------------------------------------
# sha256 of the blob, then of json([ops, bufs]), as the parent commit's compiler emitted them.  The checkpoints skip
# the BN re-estimation (bn_calibrate=0): that forward's float rounding depends on the CPU, the seeded init does not.
PT_PROGRAM_SHA256 = {
    (True, "leaky"): "ab9bfae654beb1ff73bc4caee72240de122ef5573d59a9dab2817a9915e463c2",
    (True, "relu"): "a337b1ec668b2d063473bed3363bdeefe07c34897e5a9f5000f08221d92e360c",
    (True, True): "644b394c3c6a20fda88229ee31a8e13b804ad1eae6753e2728cba54bd32bf1d5",
    (False, "leaky"): "bdab826b649a9787143f2e7699daa6e541b28ec5266847b2c4c1738db8eafa7d",
}


@pytest.mark.parametrize("smooth, act", list(PT_PROGRAM_SHA256))
def test_pt_program_bytes_unchanged(smooth, act):
    P = cc.compile_checkpoint(synth.make_checkpoint(0, smooth=smooth, bn_calibrate=0), act)
    h = hashlib.sha256(bytes(P.blob))
    h.update(json.dumps([P.ops, P.bufs], sort_keys=True).encode())
    assert h.hexdigest() == PT_PROGRAM_SHA256[(smooth, act)]
