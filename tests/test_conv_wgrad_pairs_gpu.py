"""Paired work units in the wgmma weight-gradient kernel (skd_set_wgrad_pairing 0 / 1 / 2) leave every dW bit as it was: each case
is torch.equal across the three modes, with the same (BLOCK_N, linear, splits) plan, in both K-block modes.  Both pair kinds:
adjacent Cout tiles (Cout >= 256, BLOCK_N 128) and one unit per consumer warpgroup (Cout <= 64, BLOCK_N <= 64).  Cases: the step's
weight-gradient shapes of both kinds at reduced batch with more than one split, ragged Cout (320, 384: one pair and a single tile),
Cout 64 and 48 with stride 2 and dilation 2, channel-pitched x and dy, and a launch that pairs some groups but not all."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from structure_knowledge_distillation_b200 import ops as o
    return o


def _pitched(t, pitch, off, g):
    n, c, h, w = t.shape
    buf = torch.randn(n, h, w, pitch, device="cuda", generator=g)
    buf[..., off:off + c] = t.permute(0, 2, 3, 1)
    return buf.permute(0, 3, 1, 2)[:, off:off + c]


def _run(ops, L, xc, dyc, k, s, p, d, mode):
    L.skd_set_wgrad_pairing(mode)
    dw = ops.conv2d_wgrad(xc, dyc, (k, k), s, p, d)
    plan, pairs = (ctypes.c_int * 3)(), (ctypes.c_int * 1)()
    L.skd_conv_wgrad_last_plan(plan)
    L.skd_conv_wgrad_last_pairs(pairs)
    return dw, list(plan), pairs[0]


# (N, Cin, H, W, Cout, k, stride, pad, dil, x pitch, dy pitch); the first eight are the step's shapes that pair
CASES = [
    (2, 512, 65, 129, 512, 3, 1, 4, 4, 0, 0),    # layer4 3x3 d4 512->512
    (2, 256, 65, 129, 512, 3, 1, 4, 4, 0, 0),    # layer4 3x3 d4 256->512
    (2, 256, 65, 129, 256, 3, 1, 2, 2, 0, 0),    # layer3 3x3 d2 256->256
    (2, 128, 65, 129, 256, 3, 1, 2, 2, 0, 0),    # layer3 3x3 d2 128->256
    (2, 256, 65, 129, 512, 1, 1, 0, 1, 0, 0),    # layer4 downsample 1x1 256->512
    (2, 128, 65, 129, 256, 1, 1, 0, 1, 0, 0),    # layer3 downsample 1x1 128->256
    (2, 64, 129, 257, 64, 3, 1, 1, 1, 0, 0),     # layer1 3x3 64->64
    (1, 64, 256, 512, 64, 3, 1, 1, 1, 0, 0),     # stem conv2 3x3 64->64
    (2, 256, 33, 41, 320, 3, 1, 1, 1, 0, 0),     # Cout 320: one pair, the ragged 64-row tile single
    (2, 128, 33, 41, 384, 3, 1, 1, 1, 0, 0),     # Cout 384: one pair, the odd full tile single
    (2, 64, 33, 31, 64, 3, 2, 1, 1, 0, 0),       # Cout 64, stride 2
    (1, 64, 40, 37, 48, 3, 1, 2, 2, 0, 0),       # Cout 48, dilation 2
    (2, 32, 45, 51, 64, 1, 1, 0, 1, 0, 0),       # Cout 64, 1x1, BLOCK_N 32
    (1, 128, 40, 37, 48, 3, 1, 2, 2, 0, 0),      # Cout 48 with BLOCK_N 128: no pairs
    (2, 128, 37, 45, 256, 3, 1, 1, 1, 160, 288), # channel-pitched x and dy
    (2, 256, 21, 23, 512, 3, 2, 1, 1, 320, 544), # channel-pitched, stride 2
    (2, 64, 19, 21, 48, 3, 2, 1, 1, 80, 96),     # channel-pitched, Cout 48, stride 2
]
STEP = CASES[:8]


@pytest.mark.parametrize("case", CASES)
def test_wgrad_pairs_bit_identical(ops, case):
    from structure_knowledge_distillation_b200._cabi import lib
    L = lib()
    N, Cin, H, W, Cout, k, s, p, d, ldx, ldy = case
    g = torch.Generator(device="cuda").manual_seed(sum(case) + 11)
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g)
    OH, OW = (H + 2 * p - d * (k - 1) - 1) // s + 1, (W + 2 * p - d * (k - 1) - 1) // s + 1
    dy = torch.randn(N, Cout, OH, OW, device="cuda", generator=g)
    xc = _pitched(x, ldx, 16, g) if ldx else ops.to_nhwc(x)
    dyc = _pitched(dy, ldy, 32, g) if ldy else ops.to_nhwc(dy)
    pairs_legal = (Cin > 64 and Cout >= 256) or (Cin <= 64 and Cout <= 64)
    try:
        for linear in (1, 0):
            L.skd_set_wgrad_linear(linear)
            ref, plan0, pairs0 = _run(ops, L, xc, dyc, k, s, p, d, 0)
            assert pairs0 == 0
            if case in STEP:
                assert plan0[2] > 1, plan0
            for mode in (1, 2):
                dw, plan, pairs = _run(ops, L, xc, dyc, k, s, p, d, mode)
                assert plan == plan0, (mode, linear, plan, plan0)
                assert pairs == 0 if not pairs_legal else (mode == 1 or pairs > 0), (mode, pairs)
                assert torch.equal(dw, ref), (mode, linear, pairs, float((dw - ref).abs().max()))
    finally:
        L.skd_set_wgrad_linear(1)
        L.skd_set_wgrad_pairing(1)


def test_wgrad_pairs_partial():
    """Mode 1 pairs some groups of the layer4 3x3 d4 512->512 shape at batch 8 (4 splits, 288 groups) but not all, and the result is
    bit for bit that of single units."""
    from structure_knowledge_distillation_b200 import ops
    from structure_knowledge_distillation_b200._cabi import lib
    L = lib()
    N, C, H, W, k, d = 8, 512, 65, 129, 3, 4
    g = torch.Generator(device="cuda").manual_seed(5)
    xc = ops.to_nhwc(torch.randn(N, C, H, W, device="cuda", generator=g))
    dyc = ops.to_nhwc(torch.randn(N, C, H, W, device="cuda", generator=g))
    try:
        out = {}
        for mode in (0, 1, 2):
            out[mode] = _run(ops, L, xc, dyc, k, 1, d, d, mode)
    finally:
        L.skd_set_wgrad_pairing(1)
    groups = 4 * 2 * 9 * 4
    assert out[0][1] == out[1][1] == out[2][1] == [128, 1, 4], [out[m][1] for m in out]
    assert out[0][2] == 0 and 0 < out[1][2] < groups and out[2][2] == groups, [out[m][2] for m in out]
    assert torch.equal(out[1][0], out[0][0]) and torch.equal(out[2][0], out[0][0])


def test_wgrad_wg_pairs_layer1():
    """Layer1's 3x3 64->64 at batch 8 (129x257, 29 splits, 261 units): mode 1 runs 130 units in pairs, one per consumer warpgroup,
    and the last alone, all in one wave, bit for bit what single units give."""
    from structure_knowledge_distillation_b200 import ops
    from structure_knowledge_distillation_b200._cabi import lib
    L = lib()
    N, C, H, W = 8, 64, 129, 257
    g = torch.Generator(device="cuda").manual_seed(6)
    xc = ops.to_nhwc(torch.randn(N, C, H, W, device="cuda", generator=g))
    dyc = ops.to_nhwc(torch.randn(N, C, H, W, device="cuda", generator=g))
    try:
        out = {mode: _run(ops, L, xc, dyc, 3, 1, 1, 1, mode) for mode in (0, 1, 2)}
    finally:
        L.skd_set_wgrad_pairing(1)
    assert out[0][1] == out[1][1] == out[2][1] == [64, 1, 29], [out[m][1] for m in out]
    assert [out[m][2] for m in (0, 1, 2)] == [0, 130, 130], [out[m][2] for m in out]
    assert torch.equal(out[1][0], out[0][0]) and torch.equal(out[2][0], out[0][0])
