"""oracle/student_kernels_ref.py -- the float64 restatements the ESPNet and MobileNetV2 student kernels are tested against -- held
against torch float64 autograd and a few values worked by hand.  No GPU needed."""
import pytest
import torch
import torch.nn.functional as F

from oracle import student_kernels_ref as R

EPS, MOM = 1e-3, 0.1


def _rows(P, C, seed, scale=1.0, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(P, C, generator=g, dtype=torch.float64) * scale + shift, g


def test_stats_and_running_update_match_batchnorm2d():
    x, g = _rows(37, 5, 0, 2.0, 0.5)
    mean, var = R.bn_stats(x)
    bn = torch.nn.BatchNorm2d(5, eps=EPS, momentum=R.f32(MOM)).double().train()
    rm0, rv0 = torch.randn(5, generator=g, dtype=torch.float64), torch.rand(5, generator=g, dtype=torch.float64) + 0.5
    bn.running_mean.copy_(rm0)
    bn.running_var.copy_(rv0)
    bn(x.T.reshape(1, 5, 37, 1))
    rm, rv = R.running_update(rm0, rv0, mean, var, 37, MOM)
    assert torch.allclose(rm, bn.running_mean, rtol=1e-14, atol=1e-14)
    assert torch.allclose(rv, bn.running_var, rtol=1e-14, atol=1e-14)
    assert torch.allclose(var, x.var(0, unbiased=False), rtol=1e-14)
    # by hand: rows 1, 3 -> mean 2, var 1; unbiased 2; running from (0, 1) at momentum 0.5: (1, 1.5)
    m, v = R.bn_stats(torch.tensor([[1.0], [3.0]]))
    assert float(m) == 2.0 and float(v) == 1.0
    rm, rv = R.running_update(torch.zeros(1), torch.ones(1), m, v, 2, 0.5)
    assert float(rm) == 1.0 and float(rv) == 1.5
    # one row: the biased variance 0 goes in unchanged
    _, rv1 = R.running_update(torch.zeros(1), torch.ones(1), torch.zeros(1), torch.zeros(1), 1, 0.5)
    assert float(rv1) == 0.5


def _autograd(x, g, mean, var, w, b, alpha, kind, training):
    """torch float64 autograd of act(bn(x)): with batch statistics (training) through F.batch_norm, else from the fixed (mean, var);
    eps is the float32 value the kernels take."""
    xl = x.clone().requires_grad_(True)
    wl, bl = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    al = alpha.clone().requires_grad_(True) if alpha is not None else None
    X = xl.T.unsqueeze(0).unsqueeze(-1)                              # (1, C, P, 1)
    if training:
        z = F.batch_norm(X, None, None, wl, bl, True, 0.0, R.f32(EPS))
    else:
        z = F.batch_norm(X, mean, var, wl, bl, False, 0.0, R.f32(EPS))
    if kind == "prelu":
        y = F.prelu(z, al) if al is not None else z
    elif kind == "relu6":
        y = F.hardtanh(z, 0.0, 6.0)
    else:
        y = z
    y.backward(g.T.unsqueeze(0).unsqueeze(-1))
    return y[0, :, :, 0].T.detach(), xl.grad, wl.grad, bl.grad, al.grad if al is not None else None


@pytest.mark.parametrize("kind,with_alpha", [("prelu", True), ("prelu", False), ("relu6", False), ("linear", False)])
@pytest.mark.parametrize("training", [True, False])
def test_bn_act_forward_backward_match_autograd(kind, with_alpha, training):
    P, C = 53, 6
    x, gen = _rows(P, C, 1, 1.5, 0.3)
    w = torch.randn(C, generator=gen, dtype=torch.float64)
    b = torch.randn(C, generator=gen, dtype=torch.float64) * (3.0 if kind == "relu6" else 0.5) + (3.0 if kind == "relu6" else 0.0)
    alpha = torch.rand(C, generator=gen, dtype=torch.float64) * 0.5 if with_alpha else None
    g = torch.randn(P, C, generator=gen, dtype=torch.float64)
    if training:
        mean, var = R.bn_stats(x)
    else:
        mean, var = torch.randn(C, generator=gen, dtype=torch.float64) * 0.3, torch.rand(C, generator=gen, dtype=torch.float64) + 0.5
    y_t, dx_t, dw_t, db_t, da_t = _autograd(x, g, mean, var, w, b, alpha, kind, training)
    _, z, _ = R.bn_z(x, mean, var, w, b, EPS)
    y = R.prelu(z, alpha) if kind == "prelu" else R.relu6(z) if kind == "relu6" else z
    assert torch.allclose(y, y_t, rtol=1e-12, atol=1e-12)
    ref = R.bn_act_backward(x, g, mean, var, w, b, EPS, kind, training, alpha)
    assert torch.allclose(ref["dx"], dx_t, rtol=1e-10, atol=1e-12)
    assert torch.allclose(ref["dweight"], dw_t, rtol=1e-10, atol=1e-12)
    assert torch.allclose(ref["dbias"], db_t, rtol=1e-10, atol=1e-12)
    if da_t is not None:
        assert torch.allclose(ref["dalpha"], da_t, rtol=1e-10, atol=1e-12)
    assert torch.allclose(ref["coef"][0], ref["dbias"] / P) and torch.allclose(ref["coef"][1], ref["dweight"] / P)
    assert bool((ref["dx_mag"] >= ref["dx"].abs() * (1 - 1e-12)).all())


def test_kinks_follow_torch():
    """z exactly 0 (PReLU, ReLU6) and exactly 6 (ReLU6), with running statistics so that x == mean gives z == b: the reference's
    branches are torch's -- PReLU takes the slope at 0, ReLU6 passes nothing at 0 or 6."""
    x = torch.tensor([[2.0, 2.0, 2.0], [2.0, 2.0, 2.0]], dtype=torch.float64)
    mean, var = torch.full((3,), 2.0, dtype=torch.float64), torch.ones(3, dtype=torch.float64)
    w = torch.tensor([1.5, -0.5, 2.0], dtype=torch.float64)
    g = torch.tensor([[1.0, -2.0, 3.0], [0.5, 4.0, -1.0]], dtype=torch.float64)
    alpha = torch.tensor([0.25, 0.5, 0.125], dtype=torch.float64)
    b0 = torch.zeros(3, dtype=torch.float64)
    for kind, b, al in (("prelu", b0, alpha), ("relu6", b0, None), ("relu6", b0 + 6, None)):
        _, dx_t, dw_t, db_t, da_t = _autograd(x, g, mean, var, w, b, al, kind, False)
        ref = R.bn_act_backward(x, g, mean, var, w, b, EPS, kind, False, al)
        assert torch.equal(ref["dz"], g * alpha if kind == "prelu" else torch.zeros_like(g))
        assert torch.allclose(ref["dx"], dx_t, rtol=1e-14, atol=0) and torch.allclose(ref["dbias"], db_t, rtol=1e-14, atol=0)
        assert torch.equal(ref["dweight"], torch.zeros(3, dtype=torch.float64)) and torch.equal(dw_t, ref["dweight"])
        if kind == "relu6":
            assert torch.equal(dx_t, torch.zeros_like(dx_t)) and torch.equal(db_t, torch.zeros(3, dtype=torch.float64))
        else:
            assert torch.equal(ref["dalpha"], torch.zeros(3, dtype=torch.float64)) and torch.equal(da_t, ref["dalpha"])
            assert torch.allclose(ref["dbias"], (alpha * g).sum(0), rtol=1e-15)


def test_esp_combine_and_its_adjoint():
    P, n1, n = 9, 3, 2
    gen = torch.Generator().manual_seed(4)
    d = [torch.randn(P, k, generator=gen, dtype=torch.float64, requires_grad=True) for k in (n1, n, n, n, n)]
    res = torch.randn(P, n1 + 4 * n, generator=gen, dtype=torch.float64, requires_grad=True)
    v, mag = R.esp_combine(*d, res)
    a1 = d[1]
    a2 = a1 + d[2]
    a3 = a2 + d[3]
    a4 = a3 + d[4]
    want = torch.cat([d[0], a1, a2, a3, a4], 1) + res
    assert torch.allclose(v, want, rtol=1e-15) and bool((mag >= v.abs() * (1 - 1e-15)).all())
    gc = torch.randn(P, n1 + 4 * n, generator=gen, dtype=torch.float64)
    want.backward(gc)
    got = R.esp_combine_backward(gc, n1, n)
    for a, t in zip(got, d):
        assert torch.allclose(a, t.grad, rtol=1e-14, atol=1e-15)
    assert torch.equal(res.grad, gc)
    # by hand, one row, n1 = 1, n = 1: g = (1, 2, 3, 4, 5) -> d1 = 1, d2 = 14, d4 = 12, d8 = 9, d16 = 5
    one = R.esp_combine_backward(torch.tensor([[1.0, 2.0, 3.0, 4.0, 5.0]]), 1, 1)
    assert [float(t) for t in one] == [1.0, 14.0, 12.0, 9.0, 5.0]


@pytest.mark.parametrize("stride,dil,h,w", [(1, 1, 7, 9), (2, 1, 7, 8), (1, 2, 6, 5), (2, 4, 9, 11), (1, 1, 1, 6), (2, 2, 5, 1)])
def test_depthwise_matches_autograd(stride, dil, h, w):
    gen = torch.Generator().manual_seed(h * w + dil)
    x = torch.randn(2, 8, h, w, generator=gen, dtype=torch.float64, requires_grad=True)
    wt = torch.randn(8, 1, 3, 3, generator=gen, dtype=torch.float64, requires_grad=True)
    y = F.conv2d(x, wt, None, stride, dil, dil, 8)
    ref, mag = R.dwconv3x3(x.detach(), wt.detach(), stride, dil)
    assert y.shape[2:] == ((h - 1) // stride + 1, (w - 1) // stride + 1)
    assert torch.allclose(ref, y, rtol=1e-14, atol=1e-14) and bool((mag >= ref.abs() * (1 - 1e-14)).all())
    dy = torch.randn(y.shape, generator=gen, dtype=torch.float64)
    y.backward(dy)
    dx, _ = R.dwconv3x3_dgrad(dy, wt.detach(), tuple(x.shape), stride, dil)
    dw, _ = R.dwconv3x3_wgrad(x.detach(), dy, stride, dil)
    assert torch.allclose(dx, x.grad, rtol=1e-13, atol=1e-13) and torch.allclose(dw, wt.grad, rtol=1e-13, atol=1e-13)
    # the fused statistics are those of the output
    m, v = R.bn_stats(ref.permute(0, 2, 3, 1).reshape(-1, 8))
    assert torch.allclose(m, ref.mean((0, 2, 3))) and torch.allclose(v, ref.var((0, 2, 3), unbiased=False))


def test_avgpool_divides_every_window_by_nine():
    x = torch.arange(1.0, 10.0, dtype=torch.float64).reshape(1, 1, 3, 3)
    y, _ = R.avgpool3x3s2(x)
    # output (0, 0) sees x[0:2, 0:2] = 1 + 2 + 4 + 5 = 12 (the padded taps count): 12 / 9
    assert y.shape == (1, 1, 2, 2) and float(y[0, 0, 0, 0]) == 12.0 / 9.0 and float(y[0, 0, 1, 1]) == (5 + 6 + 8 + 9) / 9.0
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(2, 3, 7, 10, generator=gen, dtype=torch.float64)
    assert torch.allclose(R.avgpool3x3s2(x)[0], torch.nn.AvgPool2d(3, 2, 1)(x), rtol=1e-15)


@pytest.mark.parametrize("h,w,H,W", [(46, 61, 360, 480), (360, 480, 46, 61), (5, 7, 5, 7), (1, 6, 4, 9), (6, 1, 1, 3), (3, 4, 1, 1),
                                     (65, 129, 64, 128)])
def test_resample_pinned_and_adjoint(h, w, H, W):
    gen = torch.Generator().manual_seed(h + W)
    x = torch.randn(2, 3, h, w, generator=gen, dtype=torch.float64, requires_grad=True)
    y = R.resample(x, H, W)
    pinned, mag = R.resample_pinned(x.detach(), H, W)
    # the float32 taps move the source coordinate by a few float32 ulps of max(h, w), each unit of which moves a value by at most
    # twice the largest input
    shift = 4 * 2.0 ** -24 * max(h, w) * 2
    assert torch.allclose(pinned, y, rtol=0, atol=shift * float(x.detach().abs().max())) and bool((mag >= pinned.abs() * (1 - 1e-14)).all())
    dy = torch.randn(y.shape, generator=gen, dtype=torch.float64)
    y.backward(dy)
    adj, amag, chain = R.resample_adjoint_pinned(dy, h, w)
    assert torch.allclose(adj, x.grad, rtol=0, atol=shift * float(amag.max()))
    # pinned adjoint is the exact transpose of the pinned forward: <M x, dy> = <x, M^T dy>
    lhs = float((pinned * dy).sum())
    rhs = float((x.detach() * adj).sum())
    assert abs(lhs - rhs) <= 1e-12 * float((mag * dy.abs()).sum())
    assert chain >= 2
    # each row of an axis matrix sums to 1 up to float32 rounding of (1 - l) + l
    for n_in, n_out in ((h, H), (w, W)):
        M = R.axis_matrix(n_in, n_out)
        assert torch.allclose(M.sum(1), torch.ones(n_out, dtype=torch.float64), rtol=0, atol=2 ** -23)
