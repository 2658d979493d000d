"""TEST INFRASTRUCTURE -- float64 restatements of the ESPNet (csrc/espnet.cu) and MobileNetV2 (csrc/mobilenet.cu) student kernels, on
[P][C] rows (NHWC pixels by channels) or (N, C, H, W) maps.  Each returns the value and, where a test bounds a float32 evaluation
elementwise, the sum of the magnitudes of the terms that value adds (`mag`).

The activation masks are taken from a float32 z supplied by the caller (`z32`: the kernel's own rounding of the BatchNorm output) so
that a reference branch never differs from the kernel's at a point float32 rounding moved across a kink; without it they are taken
from the float64 z.  The kinks follow torch: PReLU takes the slope branch where z <= 0, ReLU6 passes the gradient where 0 < z < 6.

tests/test_student_kernels_ref_cpu.py holds these against torch float64 autograd; tests/test_student_kernels_float64_gpu.py holds
the kernels against these."""
import torch
import torch.nn.functional as F


def f32(v):
    """The float32 value of a Python float (the kernels take momentum, eps as float)."""
    return float(torch.tensor(v, dtype=torch.float32))


# ---------------------------------------------------------------------------------------------- BatchNorm statistics
def bn_stats(x):
    """-> mean, biased variance of the channels of x [P][C] (float64)."""
    x = x.double()
    return x.mean(0), x.var(0, unbiased=False)


def running_update(rm, rv, mean, var, P, momentum):
    """torch's BatchNorm2d running statistics: (1 - m) r + m batch, with the unbiased variance n / (n - 1) (the biased one at n = 1)."""
    m = f32(momentum)
    ub = var * (P / (P - 1)) if P > 1 else var
    return (1 - m) * rm.double() + m * mean, (1 - m) * rv.double() + m * ub


# ---------------------------------------------------------------------------------------------- BatchNorm + activation
def bn_z(x, mean, var, w, b, eps):
    """-> xhat, z = xhat * w + b (float64) from the given (float32) statistics."""
    invstd = 1.0 / (var.double() + f32(eps)).sqrt()
    xhat = (x.double() - mean.double()) * invstd
    return xhat, xhat * w.double() + b.double(), invstd


def z_float32(x, mean, var, w, b, eps):
    """z rounded step by step as the kernels form it: ((x - mean) * invstd) * w + b, invstd = 1 / sqrt(var + eps), all float32."""
    invstd = 1.0 / torch.sqrt(var.float() + f32(eps))
    return ((x.float() - mean.float()) * invstd) * w.float() + b.float()


def prelu(z, alpha):
    """PReLU with per-channel slope (alpha None: identity, plain BatchNorm)."""
    return z if alpha is None else torch.where(z > 0, z, alpha.double() * z)


def relu6(z):
    return z.clamp(0.0, 6.0)


def act_dz(z, g, kind, alpha=None, z32=None):
    """dL/dz of the activation: kind "prelu" (slope where z <= 0; alpha None: 1) or "relu6" (g where 0 < z < 6) or "linear"."""
    zm = z if z32 is None else z32.double()
    g = g.double()
    if kind == "prelu":
        return g if alpha is None else torch.where(zm > 0, g, alpha.double() * g)
    if kind == "relu6":
        return torch.where((zm > 0) & (zm < 6), g, torch.zeros_like(g))
    return g


def bn_act_backward(x, g, mean, var, w, b, eps, kind, training, alpha=None, z32=None):
    """BatchNorm (+ activation) backward from the given statistics, as the kernels split it: the reduce pass (dweight = sum dz xhat,
    dbias = sum dz, dalpha = sum_{z <= 0} z g, coef = (mean dz, mean dz xhat)) and the input gradient, w invstd (dz - coef0 - xhat
    coef1) with batch statistics, w invstd dz with running statistics.  -> dict of float64 tensors; `*_mag` are the sums of the
    magnitudes of the terms each value adds."""
    P = x.shape[0]
    xhat, z, invstd = bn_z(x, mean, var, w, b, eps)
    dz = act_dz(z, g, kind, alpha, z32)
    zm = z if z32 is None else z32.double()
    k = w.double() * invstd
    out = dict(xhat=xhat, z=z, dz=dz, k=k, dweight=(dz * xhat).sum(0), dbias=dz.sum(0), dweight_mag=(dz * xhat).abs().sum(0),
               dbias_mag=dz.abs().sum(0))
    if kind == "prelu" and alpha is not None:
        neg = ~(zm > 0)
        out["dalpha"] = torch.where(neg, z * g.double(), torch.zeros_like(z)).sum(0)
        out["dalpha_mag"] = torch.where(neg, (z * g.double()).abs(), torch.zeros_like(z)).sum(0)
    out["coef"] = torch.stack([out["dbias"] / P, out["dweight"] / P])
    if training:
        c0, c1 = out["coef"]
        out["dx"] = (dz - c0 - xhat * c1) * k
        out["dx_mag"] = (dz.abs() + c0.abs() + (xhat * c1).abs()) * k.abs()
    else:
        out["dx"] = dz * k
        out["dx_mag"] = (dz * k).abs()
    return out


# ---------------------------------------------------------------------------------------------- ESP module combine
def esp_combine(d1, d2, d4, d8, d16, res=None):
    """[d1 | d2 | d2 + d4 | d2 + d4 + d8 | d2 + d4 + d8 + d16] (+ res) on [P][.] rows -> (value, sum of magnitudes)."""
    d1, d2, d4, d8, d16 = (t.double() for t in (d1, d2, d4, d8, d16))
    a1 = d2
    a2 = a1 + d4
    a3 = a2 + d8
    a4 = a3 + d16
    v = torch.cat([d1, a1, a2, a3, a4], 1)
    m1 = d2.abs()
    m2 = m1 + d4.abs()
    m3 = m2 + d8.abs()
    m4 = m3 + d16.abs()
    mag = torch.cat([d1.abs(), m1, m2, m3, m4], 1)
    if res is not None:
        v = v + res.double()
        mag = mag + res.double().abs()
    return v, mag


def esp_combine_backward(gc, n1, n):
    """Adjoint of esp_combine for the gradient gc [P][n1 + 4n] of the combine: d1 = g[:n1]; the fused branches get the suffix sums of
    the four n-wide slices, d16 = g4, d8 = g3 + g4, d4 = g2 + g3 + g4, d2 = g1 + g2 + g3 + g4; the residual gets gc itself."""
    gc = gc.double()
    g = [gc[:, n1 + q * n:n1 + (q + 1) * n] for q in range(4)]
    d16 = g[3]
    d8 = g[2] + d16
    d4 = g[1] + d8
    d2 = g[0] + d4
    return gc[:, :n1], d2, d4, d8, d16


# ---------------------------------------------------------------------------------------------- depthwise 3x3
def dwconv3x3(x, w, stride, dilation):
    """Depthwise 3x3 (groups = C, padding = dilation) of (N, C, H, W) -> (value, sum of |w| |x| over the taps)."""
    c = x.shape[1]
    y = F.conv2d(x.double(), w.double(), None, stride, dilation, dilation, c)
    mag = F.conv2d(x.double().abs(), w.double().abs(), None, stride, dilation, dilation, c)
    return y, mag


def dwconv3x3_dgrad(dy, w, x_shape, stride, dilation):
    """-> (dx, sum of magnitudes) of the depthwise convolution of an input of x_shape."""
    c = x_shape[1]
    gi = torch.nn.grad.conv2d_input
    dx = gi(x_shape, w.double(), dy.double(), stride, dilation, dilation, c)
    mag = gi(x_shape, w.double().abs(), dy.double().abs(), stride, dilation, dilation, c)
    return dx, mag


def dwconv3x3_wgrad(x, dy, stride, dilation):
    """-> (dweight (C, 1, 3, 3), sum of magnitudes)."""
    c = x.shape[1]
    gw = torch.nn.grad.conv2d_weight
    dw = gw(x.double(), (c, 1, 3, 3), dy.double(), stride, dilation, dilation, c)
    mag = gw(x.double().abs(), (c, 1, 3, 3), dy.double().abs(), stride, dilation, dilation, c)
    return dw, mag


# ---------------------------------------------------------------------------------------------- pooling and resampling
def avgpool3x3s2(x):
    """nn.AvgPool2d(3, 2, 1) with count_include_pad (every window divides by 9) of (N, C, H, W) -> (value, sum of |taps| / 9)."""
    return (F.avg_pool2d(x.double(), 3, 2, 1, count_include_pad=True),
            F.avg_pool2d(x.double().abs(), 3, 2, 1, count_include_pad=True))


def resample(x, H, W):
    """F.interpolate(bilinear, align_corners=True) in float64, the unpinned reference."""
    return F.interpolate(x.double(), size=(H, W), mode="bilinear", align_corners=True)


def axis_matrix(n_in, n_out):
    """The interpolation matrix M [n_out][n_in] of one axis, in float64 from the kernels' float32 taps: r = (n_in - 1) / (n_out - 1)
    and f = o * r in float32, i0 = min(int(f), n_in - 1), i1 = min(i0 + 1, n_in - 1), l = f - i0; M[o][i0] += 1 - l, M[o][i1] += l,
    each weight a float32 and a clamped tap (i0 == i1) the float32 sum of both (up_at / adj_weight)."""
    one = lambda v: torch.tensor(float(v), dtype=torch.float32)
    r = one(n_in - 1) / one(n_out - 1) if n_out > 1 else one(0)
    f = torch.arange(n_out, dtype=torch.float32) * r
    i0 = f.to(torch.int64).clamp(max=n_in - 1)
    i1 = (i0 + 1).clamp(max=n_in - 1)
    lo = f - i0.float()
    hi = 1.0 - lo
    M = torch.zeros(n_out, n_in, dtype=torch.float32)
    o = torch.arange(n_out)
    M[o, i0] = hi
    M[o, i1] = M[o, i1] + lo                  # float32: the clamped tap gets fl((1 - l) + l)
    return M.double()


def resample_pinned(x, H, W):
    """The resample with the kernels' own float32 weights: out = My x Mx^T per plane -> (value, sum of magnitudes)."""
    My, Mx = axis_matrix(x.shape[2], H).to(x.device), axis_matrix(x.shape[3], W).to(x.device)
    xd = x.double()
    return My @ xd @ Mx.T, My.abs() @ xd.abs() @ Mx.abs().T


def resample_adjoint_pinned(dout, h, w):
    """Adjoint of resample_pinned: dsrc = My^T dout Mx per plane -> (value, sum of magnitudes, longest float32 addition chain of an
    element: the output rows plus output columns that reach it)."""
    H, W = dout.shape[2:]
    My, Mx = axis_matrix(h, H).to(dout.device), axis_matrix(w, W).to(dout.device)
    g = dout.double()
    chain = int((My != 0).sum(0).max()) + int((Mx != 0).sum(0).max())
    return My.T @ g @ Mx, My.abs().T @ g.abs() @ Mx.abs(), chain
