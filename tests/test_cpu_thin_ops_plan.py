"""CPU: the shapes of tests/test_gpu_thin_ops.py::test_sppf_both_kernels fall on the sides of sppf_pool_launch's
shared-memory limit they claim, so that the GPU test cannot drift to one SPPF kernel unnoticed."""
from util import cc, get_checkpoint, sppf_uses_tile, storage_bytes, SPPF_SHAPES, SPPF_SMEM_LIMIT


def _sppf_grid_down():
    prog = cc.compile_checkpoint(get_checkpoint(0, True))
    (op,) = [op for op in prog.ops if op["kind"] == cc.OP_SPPF_POOL]
    return prog.bufs[op["src_buf"][0]][1]


def test_sppf_rule_matches_launch():
    # sppf_pool_launch: 2 planes x h x w x 8 channels of the storage type, at most 200 KB
    assert sppf_uses_tile(32, 100, 4) and not sppf_uses_tile(32, 101, 4)
    assert sppf_uses_tile(64, 100, 2) and not sppf_uses_tile(64, 101, 2)
    assert sppf_uses_tile(40, 80, 4) and not sppf_uses_tile(58, 58, 4)     # 1280 x 2560 pages; 1856^2
    assert sppf_uses_tile(80, 80, 2) and not sppf_uses_tile(82, 82, 2)     # 2560^2; 2624^2


def test_sppf_shapes_on_both_sides():
    down = _sppf_grid_down()
    assert down == 32
    sides = set()
    for prec, n, h, w, tile in SPPF_SHAPES:
        gh, gw = h // down, w // down
        e = storage_bytes(prec)
        assert h % down == 0 and w % down == 0 and h % 64 == 0 and w % 64 == 0
        assert sppf_uses_tile(gh, gw, e) == tile, (prec, h, w)
        if tile:   # the tile shapes sit exactly at the limit
            assert 2 * gh * gw * 8 * e == SPPF_SMEM_LIMIT, (prec, h, w)
        sides.add((e, tile))
        if not tile and e == 4:
            sides.add(("fallback batch", n > 1))
    assert sides >= {(4, True), (4, False), (2, True), (2, False), ("fallback batch", True)}, sides
