"""The wgmma weight-gradient kernel against float64: dY fragments fed to the tensor core from registers at every Cin tile width
(BLOCK_N 32 / 64 / 128), Cout <= 64 (the second consumer warpgroup's rows out of range) with 1x1, stride 2 and dilation 2, ragged Cout,
channel-pitched x / dy and a split-K launch at the student's layer4 shape.  Each case is within the TF32 bound, bit for bit the same on
a second run, and the two K-block modes (32 consecutive pixels through TMA im2col, pixel rectangles) agree."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from structure_knowledge_distillation_b200 import ops as o
    return o


def rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _pitched(t, pitch, off, g):
    """NHWC copy of t (N,C,H,W) as channels off .. off+C of a wider buffer of `pitch` channels (the rest random)."""
    n, c, h, w = t.shape
    buf = torch.randn(n, h, w, pitch, device="cuda", generator=g)
    buf[..., off:off + c] = t.permute(0, 2, 3, 1)
    return buf.permute(0, 3, 1, 2)[:, off:off + c]


def _wgrad_both_modes(ops, xc, dyc, k, s, p, d):
    from structure_knowledge_distillation_b200._cabi import lib
    out = {}
    try:
        for linear in (1, 0):
            lib().skd_set_wgrad_linear(linear)
            a = ops.conv2d_wgrad(xc, dyc, (k, k), s, p, d)
            b = ops.conv2d_wgrad(xc, dyc, (k, k), s, p, d)
            assert torch.equal(a, b), ("run to run", linear)
            out[linear] = a
    finally:
        lib().skd_set_wgrad_linear(1)
    return out[1], out[0]


# (N, Cin, H, W, Cout, k, stride, pad, dil, x pitch, dy pitch)
CASES = [
    (2, 64, 33, 31, 64, 3, 1, 1, 1, 0, 0),       # Cout 64: warpgroup 1's rows out of range
    (2, 64, 20, 17, 64, 1, 1, 0, 1, 0, 0),       # Cout 64, 1x1
    (2, 64, 33, 31, 64, 3, 2, 1, 1, 0, 0),       # Cout 64, stride 2
    (1, 128, 40, 37, 32, 3, 1, 2, 2, 0, 0),      # dilation 2, BLOCK_N 128, Cout one 32-channel chunk
    (2, 32, 21, 19, 128, 3, 1, 1, 1, 0, 0),      # BLOCK_N 32
    (2, 64, 21, 19, 128, 3, 1, 1, 1, 0, 0),      # BLOCK_N 64
    (1, 128, 21, 19, 256, 3, 1, 1, 1, 0, 0),     # BLOCK_N 128, two Cout tiles
    (2, 96, 17, 23, 100, 3, 1, 1, 1, 0, 0),      # Cout 100: ragged inside the fourth 32-row chunk; Cin 96 ragged in a 128 tile
    (2, 64, 19, 21, 128, 3, 1, 1, 1, 96, 160),   # channel-pitched x and dy
    (2, 64, 19, 21, 48, 3, 2, 1, 1, 80, 96),     # channel-pitched, Cout 48, stride 2
]


@pytest.mark.parametrize("case", CASES)
def test_conv_wgrad_cases(ops, case):
    N, Cin, H, W, Cout, k, s, p, d, ldx, ldy = case
    g = torch.Generator(device="cuda").manual_seed(sum(case) + 3)
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g)
    OH, OW = (H + 2 * p - d * (k - 1) - 1) // s + 1, (W + 2 * p - d * (k - 1) - 1) // s + 1
    dy = torch.randn(N, Cout, OH, OW, device="cuda", generator=g)
    dw_ref = torch.nn.grad.conv2d_weight(x.double(), (Cout, Cin, k, k), dy.double(), s, p, d).permute(0, 2, 3, 1)
    xc = _pitched(x, ldx, 16, g) if ldx else ops.to_nhwc(x)
    dyc = _pitched(dy, ldy, 32, g) if ldy else ops.to_nhwc(dy)
    a, b = _wgrad_both_modes(ops, xc, dyc, k, s, p, d)
    assert rel(a, dw_ref) < 2e-3 and rel(b, dw_ref) < 2e-3, (rel(a, dw_ref), rel(b, dw_ref))
    assert rel(a, b) < 1e-3, rel(a, b)


def test_conv_wgrad_layer4_splitk(ops):
    """The student's layer4 3x3 d4 512->512 at batch 8 (65x129 maps): a split-K launch (several partial planes added in fixed order);
    checked against float64 on the first 64 output channels."""
    from structure_knowledge_distillation_b200._cabi import lib
    N, C, H, W, k, d = 8, 512, 65, 129, 3, 4
    assert lib().skd_conv2d_wgrad_sm100_workspace_floats(N, H, W, C, C, k, k, 1, d, d) > C * k * k * C, "expected split-K"
    g = torch.Generator(device="cuda").manual_seed(41)
    x = torch.randn(N, C, H, W, device="cuda", generator=g)
    dy = torch.randn(N, C, H, W, device="cuda", generator=g)
    a, b = _wgrad_both_modes(ops, ops.to_nhwc(x), ops.to_nhwc(dy), k, 1, d, d)
    dw_ref = torch.nn.grad.conv2d_weight(x.double(), (64, C, k, k), dy[:, :64].double(), 1, d, d).permute(0, 2, 3, 1)
    assert rel(a[:64], dw_ref) < 2e-3 and rel(b[:64], dw_ref) < 2e-3, (rel(a[:64], dw_ref), rel(b[:64], dw_ref))
    assert rel(a, b) < 1e-3, rel(a, b)
