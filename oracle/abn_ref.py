"""TEST INFRASTRUCTURE -- stored outputs of the reference's own ABN kernels (libs/src/bn.cu, built into oracle/_ref/libbn_ref.so by
`make -C oracle REF=<reference checkout>`), so that tests/test_kernels_gpu.py compares the C ABI against them on any machine.

    python -m oracle.abn_ref [OUT]        (needs a GPU and oracle/_ref/libbn_ref.so; writes tests/golden/bn_ref.pt by default)

Inputs are drawn on the CPU from fixed seeds (identical on every machine); z and dx of the large shapes are kept as a fixed sample
of positions (cases.sample_large)."""
import ctypes
import os
import sys

import torch
import torch.nn.functional as F

from . import cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libbn_ref.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "bn_ref.pt")

ABN_SHAPES = [(2, 5, 7 * 3), (8, 64, 33 * 65), (3, 19, 1001), (1, 128, 4), (4, 256, 65 * 129), (2, 7, 1)]
ACT_SIZES = (1, 7, 1024, 4099)
EPS = 1e-5


def abn_inputs(N, C, S):
    """x, weight, bias, dz of one ABN case (CPU, float32)."""
    g = torch.Generator().manual_seed(N * 1000 + C)
    x = torch.randn(N, C, S, generator=g) * 2 + 0.5
    w = torch.randn(C, generator=g); b = torch.randn(C, generator=g)
    w[0] = -abs(w[0])                                      # exercise the sign-corrected dweight (bn.cu:217-223)
    dz = torch.randn(N, C, S, generator=g)
    return x, w, b, dz


def run_abi(lib, pre, N, C, S, x, w, b, dz, stream):
    """mean/var -> forward (in place) -> edz/eydz -> backward through the raw-pointer ABI of bn.h (ours: pre = "skd_")."""
    vp, fl = ctypes.c_void_p, ctypes.c_float
    dev = x.device
    mean = torch.empty(C, device=dev); var = torch.empty(C, device=dev)
    z = x.clone()
    f = lambda name: getattr(lib, pre + name)
    assert f("bn_mean_var_cuda")(N, C, S, vp(x.data_ptr()), vp(mean.data_ptr()), vp(var.data_ptr()), vp(stream))
    assert f("bn_forward_cuda")(N, C, S, vp(z.data_ptr()), vp(mean.data_ptr()), vp(var.data_ptr()), vp(w.data_ptr()),
                                vp(b.data_ptr()), vp(z.data_ptr()), vp(z.data_ptr()), fl(EPS), vp(stream))     # in place
    edz = torch.empty(C, device=dev); eydz = torch.empty(C, device=dev)
    assert f("bn_edz_eydz_cuda")(N, C, S, vp(z.data_ptr()), vp(dz.data_ptr()), vp(w.data_ptr()), vp(b.data_ptr()),
                                 vp(edz.data_ptr()), vp(eydz.data_ptr()), fl(EPS), vp(stream))
    dx = torch.empty_like(x); dw = torch.zeros(C, device=dev); db = torch.zeros(C, device=dev)
    assert f("bn_backward_cuda")(N, C, S, vp(dz.data_ptr()), vp(z.data_ptr()), vp(var.data_ptr()), vp(w.data_ptr()),
                                 vp(b.data_ptr()), vp(edz.data_ptr()), vp(eydz.data_ptr()), vp(dx.data_ptr()),
                                 vp(dw.data_ptr()), vp(db.data_ptr()), fl(EPS), vp(stream))
    torch.cuda.synchronize()
    return dict(mean=mean, var=var, z=z, edz=edz, eydz=eydz, dx=dx, dw=dw, db=db)


def act_inputs(n):
    """elu output e, leaky-relu output y (slope 0.01) and an incoming gradient d of one activation case (CPU, float32)."""
    g = torch.Generator().manual_seed(n)
    x = torch.randn(n, generator=g)
    return F.elu(x), torch.where(x < 0, x * 0.01, x), torch.randn(n, generator=g)


def run_act_backward(lib, pre, e, y, d):
    """elu backward (bn.cu:348-362) on e and leaky-relu backward on y, each on a copy of d."""
    vp = ctypes.c_void_p
    st = torch.cuda.current_stream().cuda_stream
    fe, fl = getattr(lib, pre + "elu_backward_cuda"), getattr(lib, pre + "leaky_relu_backward_cuda")
    fe.restype = fl.restype = ctypes.c_int
    fe.argtypes = [ctypes.c_int, vp, vp, vp]
    fl.argtypes = [ctypes.c_int, vp, vp, ctypes.c_float, vp]
    d1, d2 = d.clone(), d.clone()
    assert fe(e.numel(), e.data_ptr(), d1.data_ptr(), st) == 1
    assert fl(y.numel(), y.data_ptr(), d2.data_ptr(), 0.01, st) == 1
    torch.cuda.synchronize()
    return d1, d2


def main(out=GOLDEN):
    ref = ctypes.CDLL(REF_LIB)
    st = torch.cuda.current_stream().cuda_stream
    gold = {"abn": {}, "act": {}}
    for N, C, S in ABN_SHAPES:
        x, w, b, dz = (t.cuda() for t in abn_inputs(N, C, S))
        r = run_abi(ref, "_", N, C, S, x, w, b, dz, st)
        gold["abn"][(N, C, S)] = {k: cases.sample_large(v.cpu()) for k, v in r.items()}
    for n in ACT_SIZES:
        e, y, d = (t.cuda() for t in act_inputs(n))
        d_elu, d_leaky = run_act_backward(ref, "_", e, y, d)
        gold["act"][n] = dict(elu=d_elu.cpu(), leaky=d_leaky.cpu())
    gold["device"] = torch.cuda.get_device_name()
    torch.save(gold, out)
    print("wrote", out)


if __name__ == "__main__":
    main(*sys.argv[1:])
