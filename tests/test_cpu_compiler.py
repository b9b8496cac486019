"""not-gpu: the host compiler (BN folding, weight packing, graph wiring) pinned against the oracle
by interpreting the emitted program on the CPU."""
import numpy as np
import pytest
import torch

import ctd_b200
from oracle import synth
from oracle.net_ref import RefNet
from prog_interp import run_program
from util import page_to_net_input


@pytest.fixture(scope="module")
def ck():
    return synth.make_checkpoint(0, smooth=False, bn_calibrate=256)


def test_program_structure(ck):
    prog = ctd_b200.compiler.compile_checkpoint(ck)
    kinds = [o["kind"] for o in prog.ops]
    cc = ctd_b200.compiler
    assert kinds.count(cc.OP_STEM) == 1 and kinds.count(cc.OP_DETECT) == 3 and kinds.count(cc.OP_DECONV4) == 7
    assert kinds.count(cc.OP_SEG_TAIL) == 1 and kinds.count(cc.OP_DB_TAIL) == 1
    # 115 reference conv/deconv layers: cv1||cv2 fused per C3 (18 of them), binarize.0||thresh.0 fused, the two
    # ConvT2x2 pairs and the seg ConvT live in the tails
    n_gemm = kinds.count(cc.OP_CONV) + kinds.count(cc.OP_DECONV4) + kinds.count(cc.OP_DETECT)
    assert n_gemm == 92
    for o in prog.ops:
        if o["kind"] in (cc.OP_CONV, cc.OP_DECONV4):
            assert o["cout_pad"] % 16 == 0 and o["w16_off"] % 256 == 0 and o["b_off"] % 256 == 0
            for i in range(o["n_src"]):
                assert o["src_c"][i] % 16 == 0 and o["src_coff"][i] % 8 == 0


def test_stem_window_weights_match_direct_form(ck):
    """the tensor-core (space-to-depth window) weights of the stem compute the same conv as the direct 6x6 form"""
    prog = ctd_b200.compiler.compile_checkpoint(ck)
    pages = np.stack([synth.noise_page(3, 64, 128)])
    b16, m16, l16 = run_program(prog, pages, use_fp16_weights=True)
    b32, m32, l32 = run_program(prog, pages)
    # fp16 weight rounding through the whole net: statistical bound (a wrong tap mapping gives mean errors ~0.1)
    assert float((m16 - m32).abs().max()) < 0.3 and float((m16 - m32).abs().mean()) < 5e-3


def test_program_matches_oracle(ck):
    """fp32 weights: the interpreted program equals the oracle forward to fp32 rounding."""
    prog = ctd_b200.compiler.compile_checkpoint(ck)
    pages = np.stack([synth.structured_page(7, 128, 192)])
    blks, mask, lines = run_program(prog, pages)
    rb, rm, rl = RefNet(ck)(page_to_net_input(pages))
    assert float((mask - rm).abs().max()) < 1e-3
    assert float((lines - rl).abs().max()) < 1e-3
    assert float(((blks - rb).abs() / (rb.abs() + 1)).max()) < 1e-3
