"""The ESPNet-C / ESPNet (csrc/espnet.cu) and MobileNetV2 (csrc/mobilenet.cu) student kernels against float64, at every shape the
students' training steps and evaluation forwards launch them with.

At those shapes the kernels take paths small shapes never reach: hundreds of row splits (capped at (P + 31) / 32), a second channel
chunk past 256 channels (or channel quads), idle threads where 256 % C != 0, grid-stride loops that go round many times.  A guard
records every call of the kernels' `ops` wrappers during one eager step and the eval forwards of each student and fails on a
signature STEP_LAUNCHES lacks; each row of the table, and synthetic rows for the edges no step reaches, is then run twice on
NaN-filled buffers (NaN in every pitch tail) and held elementwise against oracle/student_kernels_ref.py, with bounds stated relative to
the sum of the magnitudes of each element's terms.  The BatchNorm + activation kinks (PReLU at z = 0, ReLU6 at z = 0 and 6) are
pinned exactly with rows whose z is exactly b.
"""
import inspect

import pytest
import torch

pytestmark = pytest.mark.gpu

# ---------------------------------------------------------------------------------------------- launch signatures
RECORDED = ("bnprelu_stats", "bnprelu_apply", "bnprelu_bwd_reduce", "bnprelu_bwd_dx", "esp_combine", "esp_bwd_dx", "avgpool3x3s2",
            "resample_nhwc", "resample_adjoint_nhwc", "dwconv3x3_fwd", "dwconv3x3_dgrad", "dwconv3x3_wgrad", "bnact_apply",
            "bnact_bwd_reduce", "bnact_bwd_dx")


def _signature(ops, name, a):
    """The launch signature of one wrapper call: everything the kernel's geometry and branches depend on (rows or N/H/W, channels,
    pitches, padded widths, stride / dilation, mode flags), none of the values."""
    if name == "bnprelu_stats":
        P, c, ld = ops._rows(a["x"])
        return (name, P, c, ld, a["running_mean"] is not None)
    if name == "esp_combine":
        d1, d2 = a["branches"][:2]
        P, n1, ld1 = ops._rows(d1)
        _, n, ldn = ops._rows(d2)
        ldr = ops._rows(a["residual"])[2] if a["residual"] is not None else 0
        return (name, P, n1, ld1, n, ldn, ldr, ops._rows(a["out"])[2], bool(a["stats"]), a["running_mean"] is not None)
    if name == "bnprelu_apply":
        P, c, ld = ops._rows(a["x"])
        cw = a["out_channels"] or c
        ldo = ops._rows(a["out"])[2] if a["out"] is not None else cw
        return (name, P, c, ld, cw, ldo, a["alpha"] is not None)
    if name == "bnprelu_bwd_reduce":
        P, c, ld = ops._rows(a["x"])
        return (name, P, c, ld, ops._rows(a["dout"])[2], a["alpha"] is not None)
    if name == "bnprelu_bwd_dx":
        P, c, ld = ops._rows(a["x"])
        return (name, P, c, ld, ops._rows(a["dout"])[2], a["dx_channels"] or c, bool(a["training"]), a["alpha"] is not None)
    if name == "esp_bwd_dx":
        P, c, ld = ops._rows(a["x"])
        return (name, P, a["n1"], a["n"], ld, ops._rows(a["dout"])[2], bool(a["training"]), a["alpha"] is not None,
                bool(a["want_dres"]))
    if name == "avgpool3x3s2":
        n, c, h, w, lds = ops.nhwc_meta(a["src"])
        return (name, n, h, w, c, lds, ops.nhwc_meta(a["out"])[4])
    if name == "resample_nhwc":
        t = a["t"]
        n, c, h, w = t.shape
        _, sc, sp = ops.pixel_strides(t)
        return (name, n, c, h, w, a["h"], a["w"], "nhwc" if sc == 1 else "nchw", sp if sc == 1 else 1)
    if name == "resample_adjoint_nhwc":
        n, c, H, W = a["dout"].shape
        return (name, n, c, H, W, a["h"], a["w"], a["channels"] or c)
    if name == "dwconv3x3_fwd":
        n, c, h, w = a["x"].shape
        return (name, n, c, h, w, a["stride"], int(a["dilation"]), bool(a["stats"]), a["running_mean"] is not None)
    if name == "dwconv3x3_dgrad":
        n, c, h, w = a["x_shape"]
        return (name, n, c, h, w, a["stride"], int(a["dilation"]))
    if name == "dwconv3x3_wgrad":
        n, c, h, w = a["x"].shape
        return (name, n, c, h, w, a["stride"], int(a["dilation"]))
    if name == "bnact_apply":
        P, c, ld = ops._rows(a["x"])
        ldr = ops._rows(a["residual"])[2] if a["residual"] is not None else 0
        return (name, P, c, ld, bool(a["relu6"]), ldr)
    if name == "bnact_bwd_reduce":
        P, c, ld = ops._rows(a["x"])
        return (name, P, c, ld, ops._rows(a["dout"])[2], bool(a["relu6"]))
    if name == "bnact_bwd_dx":
        P, c, ld = ops._rows(a["x"])
        return (name, P, c, ld, ops._rows(a["dout"])[2], bool(a["relu6"]), bool(a["training"]))
    raise KeyError(name)


def record_launches(monkeypatch, ops, fn):
    """Run fn() with every wrapper in RECORDED logging its call's signature, then calling through; -> the set of signatures."""
    seen = set()
    for name in RECORDED:
        orig = getattr(ops, name)
        sig = inspect.signature(orig)

        def logged(*args, _orig=orig, _sig=sig, _name=name, **kwargs):
            b = _sig.bind(*args, **kwargs)
            b.apply_defaults()
            seen.add(_signature(ops, _name, b.arguments))
            return _orig(*args, **kwargs)
        monkeypatch.setattr(ops, name, logged)
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        monkeypatch.undo()
    return seen


STUDENT_STEPS = (("espnet_c", 16, 360, 480), ("espnet", 16, 360, 480), ("mobilenetv2", 8, 512, 1024))
EVAL_HW = (1024, 2048)


def run_student(student, batch, h, w):
    """One eager distillation step at the student's benchmark configuration (Pi + Pa + Ho wgan-gp), then the eval-mode forward of
    one whole 1024x2048 image at batch 1 and of the image with its mirror at batch 2."""
    from oracle import port
    from structure_knowledge_distillation_b200.networks.evaluate import _scores, zoom_image
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    torch.manual_seed(0)
    m = NetModel(make_args(batch_size=batch, pi=True, pa=True, ho=True, adv_loss_type="wgan-gp", student=student))
    images, labels = port.synthetic_batch(batch, h, w, seed=1)
    m.set_input((images, labels, None, None))
    m.optimize_parameters()
    s = m.student.eval()
    image = torch.randn(1, 3, *EVAL_HW, generator=torch.Generator().manual_seed(3)).cuda() * 40.0
    for flip in (False, True):
        _scores(s, zoom_image(image, 1.0, flip))
    torch.cuda.synchronize()
    del m, s
    torch.cuda.empty_cache()


# The distinct signatures of one eager step of each student at its benchmark configuration (ESPNet-C and ESPNet: batch 16 at 360x480;
# MobileNetV2: batch 8 at 512x1024; Pi + Pa + Ho wgan-gp) and of its eval-mode forwards of a 1024x2048 image at batch 1 and 2.
STEP_LAUNCHES = frozenset([
    ('avgpool3x3s2', 1, 1024, 2048, 3, 4, 20),                                   # espnet_c, espnet
    ('avgpool3x3s2', 1, 512, 1024, 3, 20, 132),                                  # espnet_c, espnet
    ('avgpool3x3s2', 16, 180, 240, 3, 20, 132),                                  # espnet_c, espnet
    ('avgpool3x3s2', 16, 360, 480, 3, 4, 20),                                    # espnet_c, espnet
    ('avgpool3x3s2', 2, 1024, 2048, 3, 4, 20),                                   # espnet_c, espnet
    ('avgpool3x3s2', 2, 512, 1024, 3, 20, 132),                                  # espnet_c, espnet
    ('bnact_apply', 1048576, 16, 16, False, 0),                                  # mobilenetv2
    ('bnact_apply', 1048576, 32, 32, True, 0),                                   # mobilenetv2
    ('bnact_apply', 1048576, 96, 96, True, 0),                                   # mobilenetv2
    ('bnact_apply', 131072, 144, 144, True, 0),                                  # mobilenetv2
    ('bnact_apply', 131072, 24, 24, False, 0),                                   # mobilenetv2
    ('bnact_apply', 131072, 24, 24, False, 24),                                  # mobilenetv2
    ('bnact_apply', 131072, 96, 96, True, 0),                                    # mobilenetv2
    ('bnact_apply', 262144, 144, 144, True, 0),                                  # mobilenetv2
    ('bnact_apply', 262144, 24, 24, False, 0),                                   # mobilenetv2
    ('bnact_apply', 262144, 24, 24, False, 24),                                  # mobilenetv2
    ('bnact_apply', 262144, 96, 96, True, 0),                                    # mobilenetv2
    ('bnact_apply', 32768, 144, 144, True, 0),                                   # mobilenetv2
    ('bnact_apply', 32768, 160, 160, False, 0),                                  # mobilenetv2
    ('bnact_apply', 32768, 160, 160, False, 160),                                # mobilenetv2
    ('bnact_apply', 32768, 192, 192, True, 0),                                   # mobilenetv2
    ('bnact_apply', 32768, 32, 32, False, 0),                                    # mobilenetv2
    ('bnact_apply', 32768, 32, 32, False, 32),                                   # mobilenetv2
    ('bnact_apply', 32768, 320, 320, False, 0),                                  # mobilenetv2
    ('bnact_apply', 32768, 384, 384, True, 0),                                   # mobilenetv2
    ('bnact_apply', 32768, 576, 576, True, 0),                                   # mobilenetv2
    ('bnact_apply', 32768, 64, 64, False, 0),                                    # mobilenetv2
    ('bnact_apply', 32768, 64, 64, False, 64),                                   # mobilenetv2
    ('bnact_apply', 32768, 96, 96, False, 0),                                    # mobilenetv2
    ('bnact_apply', 32768, 96, 96, False, 96),                                   # mobilenetv2
    ('bnact_apply', 32768, 960, 960, True, 0),                                   # mobilenetv2
    ('bnact_apply', 524288, 16, 16, False, 0),                                   # mobilenetv2
    ('bnact_apply', 524288, 32, 32, True, 0),                                    # mobilenetv2
    ('bnact_apply', 524288, 96, 96, True, 0),                                    # mobilenetv2
    ('bnact_apply', 65536, 144, 144, True, 0),                                   # mobilenetv2
    ('bnact_apply', 65536, 160, 160, False, 0),                                  # mobilenetv2
    ('bnact_apply', 65536, 160, 160, False, 160),                                # mobilenetv2
    ('bnact_apply', 65536, 192, 192, True, 0),                                   # mobilenetv2
    ('bnact_apply', 65536, 32, 32, False, 0),                                    # mobilenetv2
    ('bnact_apply', 65536, 32, 32, False, 32),                                   # mobilenetv2
    ('bnact_apply', 65536, 320, 320, False, 0),                                  # mobilenetv2
    ('bnact_apply', 65536, 384, 384, True, 0),                                   # mobilenetv2
    ('bnact_apply', 65536, 576, 576, True, 0),                                   # mobilenetv2
    ('bnact_apply', 65536, 64, 64, False, 0),                                    # mobilenetv2
    ('bnact_apply', 65536, 64, 64, False, 64),                                   # mobilenetv2
    ('bnact_apply', 65536, 96, 96, False, 0),                                    # mobilenetv2
    ('bnact_apply', 65536, 96, 96, False, 96),                                   # mobilenetv2
    ('bnact_apply', 65536, 960, 960, True, 0),                                   # mobilenetv2
    ('bnact_bwd_dx', 1048576, 16, 16, 16, False, True),                          # mobilenetv2
    ('bnact_bwd_dx', 1048576, 32, 32, 32, True, True),                           # mobilenetv2
    ('bnact_bwd_dx', 1048576, 96, 96, 96, True, True),                           # mobilenetv2
    ('bnact_bwd_dx', 262144, 144, 144, 144, True, True),                         # mobilenetv2
    ('bnact_bwd_dx', 262144, 24, 24, 24, False, True),                           # mobilenetv2
    ('bnact_bwd_dx', 262144, 96, 96, 96, True, True),                            # mobilenetv2
    ('bnact_bwd_dx', 65536, 144, 144, 144, True, True),                          # mobilenetv2
    ('bnact_bwd_dx', 65536, 160, 160, 160, False, True),                         # mobilenetv2
    ('bnact_bwd_dx', 65536, 192, 192, 192, True, True),                          # mobilenetv2
    ('bnact_bwd_dx', 65536, 32, 32, 32, False, True),                            # mobilenetv2
    ('bnact_bwd_dx', 65536, 320, 320, 320, False, True),                         # mobilenetv2
    ('bnact_bwd_dx', 65536, 384, 384, 384, True, True),                          # mobilenetv2
    ('bnact_bwd_dx', 65536, 576, 576, 576, True, True),                          # mobilenetv2
    ('bnact_bwd_dx', 65536, 64, 64, 64, False, True),                            # mobilenetv2
    ('bnact_bwd_dx', 65536, 96, 96, 96, False, True),                            # mobilenetv2
    ('bnact_bwd_dx', 65536, 960, 960, 960, True, True),                          # mobilenetv2
    ('bnact_bwd_reduce', 1048576, 16, 16, 16, False),                            # mobilenetv2
    ('bnact_bwd_reduce', 1048576, 32, 32, 32, True),                             # mobilenetv2
    ('bnact_bwd_reduce', 1048576, 96, 96, 96, True),                             # mobilenetv2
    ('bnact_bwd_reduce', 262144, 144, 144, 144, True),                           # mobilenetv2
    ('bnact_bwd_reduce', 262144, 24, 24, 24, False),                             # mobilenetv2
    ('bnact_bwd_reduce', 262144, 96, 96, 96, True),                              # mobilenetv2
    ('bnact_bwd_reduce', 65536, 144, 144, 144, True),                            # mobilenetv2
    ('bnact_bwd_reduce', 65536, 160, 160, 160, False),                           # mobilenetv2
    ('bnact_bwd_reduce', 65536, 192, 192, 192, True),                            # mobilenetv2
    ('bnact_bwd_reduce', 65536, 32, 32, 32, False),                              # mobilenetv2
    ('bnact_bwd_reduce', 65536, 320, 320, 320, False),                           # mobilenetv2
    ('bnact_bwd_reduce', 65536, 384, 384, 384, True),                            # mobilenetv2
    ('bnact_bwd_reduce', 65536, 576, 576, 576, True),                            # mobilenetv2
    ('bnact_bwd_reduce', 65536, 64, 64, 64, False),                              # mobilenetv2
    ('bnact_bwd_reduce', 65536, 96, 96, 96, False),                              # mobilenetv2
    ('bnact_bwd_reduce', 65536, 960, 960, 960, True),                            # mobilenetv2
    ('bnprelu_apply', 1048576, 16, 16, 16, 16, True),                            # espnet_c, espnet
    ('bnprelu_apply', 1048576, 19, 20, 20, 20, True),                            # espnet_c, espnet
    ('bnprelu_apply', 131072, 131, 132, 132, 132, True),                         # espnet_c, espnet
    ('bnprelu_apply', 131072, 19, 19, 20, 20, True),                             # espnet
    ('bnprelu_apply', 131072, 38, 40, 40, 40, True),                             # espnet
    ('bnprelu_apply', 131072, 64, 64, 64, 64, True),                             # espnet_c, espnet
    ('bnprelu_apply', 172800, 131, 132, 132, 132, True),                         # espnet_c, espnet
    ('bnprelu_apply', 172800, 19, 19, 20, 20, True),                             # espnet
    ('bnprelu_apply', 172800, 38, 40, 40, 40, True),                             # espnet
    ('bnprelu_apply', 172800, 64, 64, 64, 64, True),                             # espnet_c, espnet
    ('bnprelu_apply', 262144, 131, 132, 132, 132, True),                         # espnet_c, espnet
    ('bnprelu_apply', 262144, 19, 19, 20, 20, True),                             # espnet
    ('bnprelu_apply', 262144, 38, 40, 40, 40, True),                             # espnet
    ('bnprelu_apply', 262144, 64, 64, 64, 64, True),                             # espnet_c, espnet
    ('bnprelu_apply', 32768, 128, 128, 128, 128, True),                          # espnet_c, espnet
    ('bnprelu_apply', 32768, 19, 20, 20, 20, False),                             # espnet
    ('bnprelu_apply', 32768, 256, 256, 256, 256, True),                          # espnet_c, espnet
    ('bnprelu_apply', 43200, 128, 128, 128, 128, True),                          # espnet_c, espnet
    ('bnprelu_apply', 43200, 19, 20, 20, 20, False),                             # espnet
    ('bnprelu_apply', 43200, 256, 256, 256, 256, True),                          # espnet_c, espnet
    ('bnprelu_apply', 524288, 16, 16, 16, 16, True),                             # espnet_c, espnet
    ('bnprelu_apply', 524288, 19, 20, 20, 20, True),                             # espnet_c, espnet
    ('bnprelu_apply', 65536, 128, 128, 128, 128, True),                          # espnet_c, espnet
    ('bnprelu_apply', 65536, 19, 20, 20, 20, False),                             # espnet
    ('bnprelu_apply', 65536, 256, 256, 256, 256, True),                          # espnet_c, espnet
    ('bnprelu_apply', 691200, 16, 16, 16, 16, True),                             # espnet_c, espnet
    ('bnprelu_apply', 691200, 19, 20, 20, 20, True),                             # espnet_c, espnet
    ('bnprelu_bwd_dx', 172800, 131, 132, 132, 132, True, True),                  # espnet_c, espnet
    ('bnprelu_bwd_dx', 172800, 38, 40, 40, 40, True, True),                      # espnet
    ('bnprelu_bwd_dx', 43200, 19, 20, 20, 20, True, False),                      # espnet
    ('bnprelu_bwd_dx', 43200, 256, 256, 256, 256, True, True),                   # espnet_c, espnet
    ('bnprelu_bwd_dx', 691200, 16, 16, 16, 16, True, True),                      # espnet_c, espnet
    ('bnprelu_bwd_dx', 691200, 19, 20, 20, 20, True, True),                      # espnet_c, espnet
    ('bnprelu_bwd_reduce', 172800, 131, 132, 132, True),                         # espnet_c, espnet
    ('bnprelu_bwd_reduce', 172800, 19, 19, 20, True),                            # espnet
    ('bnprelu_bwd_reduce', 172800, 38, 40, 40, True),                            # espnet
    ('bnprelu_bwd_reduce', 172800, 64, 64, 64, True),                            # espnet_c, espnet
    ('bnprelu_bwd_reduce', 43200, 128, 128, 128, True),                          # espnet_c, espnet
    ('bnprelu_bwd_reduce', 43200, 19, 20, 20, False),                            # espnet
    ('bnprelu_bwd_reduce', 43200, 256, 256, 256, True),                          # espnet_c, espnet
    ('bnprelu_bwd_reduce', 691200, 16, 16, 16, True),                            # espnet_c, espnet
    ('bnprelu_bwd_reduce', 691200, 19, 20, 20, True),                            # espnet_c, espnet
    ('bnprelu_stats', 1048576, 16, 16, True),                                    # mobilenetv2
    ('bnprelu_stats', 1048576, 32, 32, True),                                    # mobilenetv2
    ('bnprelu_stats', 1048576, 96, 96, True),                                    # mobilenetv2
    ('bnprelu_stats', 172800, 131, 132, True),                                   # espnet_c, espnet
    ('bnprelu_stats', 172800, 38, 40, True),                                     # espnet
    ('bnprelu_stats', 262144, 144, 144, True),                                   # mobilenetv2
    ('bnprelu_stats', 262144, 24, 24, True),                                     # mobilenetv2
    ('bnprelu_stats', 43200, 19, 20, True),                                      # espnet
    ('bnprelu_stats', 43200, 256, 256, True),                                    # espnet_c, espnet
    ('bnprelu_stats', 65536, 160, 160, True),                                    # mobilenetv2
    ('bnprelu_stats', 65536, 192, 192, True),                                    # mobilenetv2
    ('bnprelu_stats', 65536, 32, 32, True),                                      # mobilenetv2
    ('bnprelu_stats', 65536, 320, 320, True),                                    # mobilenetv2
    ('bnprelu_stats', 65536, 384, 384, True),                                    # mobilenetv2
    ('bnprelu_stats', 65536, 576, 576, True),                                    # mobilenetv2
    ('bnprelu_stats', 65536, 64, 64, True),                                      # mobilenetv2
    ('bnprelu_stats', 65536, 96, 96, True),                                      # mobilenetv2
    ('bnprelu_stats', 65536, 960, 960, True),                                    # mobilenetv2
    ('bnprelu_stats', 691200, 16, 16, True),                                     # espnet_c, espnet
    ('bnprelu_stats', 691200, 19, 20, True),                                     # espnet_c, espnet
    ('dwconv3x3_dgrad', 8, 144, 128, 256, 1, 1),                                 # mobilenetv2
    ('dwconv3x3_dgrad', 8, 144, 128, 256, 2, 1),                                 # mobilenetv2
    ('dwconv3x3_dgrad', 8, 192, 64, 128, 1, 1),                                  # mobilenetv2
    ('dwconv3x3_dgrad', 8, 32, 256, 512, 1, 1),                                  # mobilenetv2
    ('dwconv3x3_dgrad', 8, 384, 64, 128, 1, 2),                                  # mobilenetv2
    ('dwconv3x3_dgrad', 8, 576, 64, 128, 1, 2),                                  # mobilenetv2
    ('dwconv3x3_dgrad', 8, 96, 256, 512, 2, 1),                                  # mobilenetv2
    ('dwconv3x3_dgrad', 8, 960, 64, 128, 1, 4),                                  # mobilenetv2
    ('dwconv3x3_fwd', 1, 144, 256, 512, 1, 1, False, True),                      # mobilenetv2
    ('dwconv3x3_fwd', 1, 144, 256, 512, 2, 1, False, True),                      # mobilenetv2
    ('dwconv3x3_fwd', 1, 192, 128, 256, 1, 1, False, True),                      # mobilenetv2
    ('dwconv3x3_fwd', 1, 32, 512, 1024, 1, 1, False, True),                      # mobilenetv2
    ('dwconv3x3_fwd', 1, 384, 128, 256, 1, 2, False, True),                      # mobilenetv2
    ('dwconv3x3_fwd', 1, 576, 128, 256, 1, 2, False, True),                      # mobilenetv2
    ('dwconv3x3_fwd', 1, 96, 512, 1024, 2, 1, False, True),                      # mobilenetv2
    ('dwconv3x3_fwd', 1, 960, 128, 256, 1, 4, False, True),                      # mobilenetv2
    ('dwconv3x3_fwd', 2, 144, 256, 512, 1, 1, False, True),                      # mobilenetv2
    ('dwconv3x3_fwd', 2, 144, 256, 512, 2, 1, False, True),                      # mobilenetv2
    ('dwconv3x3_fwd', 2, 192, 128, 256, 1, 1, False, True),                      # mobilenetv2
    ('dwconv3x3_fwd', 2, 32, 512, 1024, 1, 1, False, True),                      # mobilenetv2
    ('dwconv3x3_fwd', 2, 384, 128, 256, 1, 2, False, True),                      # mobilenetv2
    ('dwconv3x3_fwd', 2, 576, 128, 256, 1, 2, False, True),                      # mobilenetv2
    ('dwconv3x3_fwd', 2, 96, 512, 1024, 2, 1, False, True),                      # mobilenetv2
    ('dwconv3x3_fwd', 2, 960, 128, 256, 1, 4, False, True),                      # mobilenetv2
    ('dwconv3x3_fwd', 8, 144, 128, 256, 1, 1, True, True),                       # mobilenetv2
    ('dwconv3x3_fwd', 8, 144, 128, 256, 2, 1, True, True),                       # mobilenetv2
    ('dwconv3x3_fwd', 8, 192, 64, 128, 1, 1, True, True),                        # mobilenetv2
    ('dwconv3x3_fwd', 8, 32, 256, 512, 1, 1, True, True),                        # mobilenetv2
    ('dwconv3x3_fwd', 8, 384, 64, 128, 1, 2, True, True),                        # mobilenetv2
    ('dwconv3x3_fwd', 8, 576, 64, 128, 1, 2, True, True),                        # mobilenetv2
    ('dwconv3x3_fwd', 8, 96, 256, 512, 2, 1, True, True),                        # mobilenetv2
    ('dwconv3x3_fwd', 8, 960, 64, 128, 1, 4, True, True),                        # mobilenetv2
    ('dwconv3x3_wgrad', 8, 144, 128, 256, 1, 1),                                 # mobilenetv2
    ('dwconv3x3_wgrad', 8, 144, 128, 256, 2, 1),                                 # mobilenetv2
    ('dwconv3x3_wgrad', 8, 192, 64, 128, 1, 1),                                  # mobilenetv2
    ('dwconv3x3_wgrad', 8, 32, 256, 512, 1, 1),                                  # mobilenetv2
    ('dwconv3x3_wgrad', 8, 384, 64, 128, 1, 2),                                  # mobilenetv2
    ('dwconv3x3_wgrad', 8, 576, 64, 128, 1, 2),                                  # mobilenetv2
    ('dwconv3x3_wgrad', 8, 96, 256, 512, 2, 1),                                  # mobilenetv2
    ('dwconv3x3_wgrad', 8, 960, 64, 128, 1, 4),                                  # mobilenetv2
    ('esp_bwd_dx', 172800, 16, 12, 64, 64, True, True, False),                   # espnet_c, espnet
    ('esp_bwd_dx', 172800, 16, 12, 64, 64, True, True, True),                    # espnet_c, espnet
    ('esp_bwd_dx', 172800, 7, 3, 19, 20, True, True, False),                     # espnet
    ('esp_bwd_dx', 43200, 28, 25, 128, 128, True, True, False),                  # espnet_c, espnet
    ('esp_bwd_dx', 43200, 28, 25, 128, 128, True, True, True),                   # espnet_c, espnet
    ('esp_combine', 131072, 16, 16, 12, 12, 0, 64, False, False),                # espnet_c, espnet
    ('esp_combine', 131072, 16, 16, 12, 12, 64, 64, False, False),               # espnet_c, espnet
    ('esp_combine', 131072, 7, 8, 3, 4, 0, 19, False, False),                    # espnet
    ('esp_combine', 172800, 16, 16, 12, 12, 0, 64, True, True),                  # espnet_c, espnet
    ('esp_combine', 172800, 16, 16, 12, 12, 64, 64, True, True),                 # espnet_c, espnet
    ('esp_combine', 172800, 7, 8, 3, 4, 0, 19, True, True),                      # espnet
    ('esp_combine', 262144, 16, 16, 12, 12, 0, 64, False, False),                # espnet_c, espnet
    ('esp_combine', 262144, 16, 16, 12, 12, 64, 64, False, False),               # espnet_c, espnet
    ('esp_combine', 262144, 7, 8, 3, 4, 0, 19, False, False),                    # espnet
    ('esp_combine', 32768, 28, 28, 25, 28, 0, 128, False, False),                # espnet_c, espnet
    ('esp_combine', 32768, 28, 28, 25, 28, 128, 128, False, False),              # espnet_c, espnet
    ('esp_combine', 43200, 28, 28, 25, 28, 0, 128, True, True),                  # espnet_c, espnet
    ('esp_combine', 43200, 28, 28, 25, 28, 128, 128, True, True),                # espnet_c, espnet
    ('esp_combine', 65536, 28, 28, 25, 28, 0, 128, False, False),                # espnet_c, espnet
    ('esp_combine', 65536, 28, 28, 25, 28, 128, 128, False, False),              # espnet_c, espnet
    ('resample_adjoint_nhwc', 16, 19, 46, 61, 360, 480, 19),                     # espnet
    ('resample_nhwc', 16, 19, 360, 480, 46, 61, 'nhwc', 20),                     # espnet
    ('resample_nhwc', 16, 19, 46, 61, 360, 480, 'nhwc', 20),                     # espnet
    ('resample_nhwc', 16, 19, 46, 61, 45, 60, 'nhwc', 20),                       # espnet_c
    ('resample_nhwc', 16, 512, 46, 61, 45, 60, 'nhwc', 512),                     # espnet_c, espnet
    ('resample_nhwc', 8, 19, 65, 129, 64, 128, 'nhwc', 20),                      # mobilenetv2
    ('resample_nhwc', 8, 512, 65, 129, 64, 128, 'nhwc', 512),                    # mobilenetv2
])


def test_launch_table_covers_every_student_launch(monkeypatch):
    """Every student kernel call of the three students' steps and eval forwards has its row in STEP_LAUNCHES, so the float64 tests
    below reach every shape those runs launch."""
    from structure_knowledge_distillation_b200 import ops
    for st in STUDENT_STEPS:
        seen = record_launches(monkeypatch, ops, lambda: run_student(*st))
        assert seen, st
        missing = sorted(seen - STEP_LAUNCHES, key=repr)
        assert not missing, (st[0], missing)


# ---------------------------------------------------------------------------------------------- shared machinery
U = 2.0 ** -24                     # unit roundoff of float32
UD = 2.0 ** -53                    # ... of float64
NAN_BITS = 0x7FC0ABCD              # a NaN payload no kernel computes: pitch tails and unwritten outputs keep it
TAIL = 67                          # NaN floats past the last row of every buffer
EPS_ESP, EPS_MB, MOM = 1e-3, 1e-5, 0.1
SMS, THREADS = 132, 256
WORST = {}                         # kernel family -> largest error seen, as a fraction of its bound


@pytest.fixture(scope="module")
def L():
    from structure_knowledge_distillation_b200._cabi import lib
    return lib()


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    print("\nworst error / bound per kernel family:", {k: round(v, 4) for k, v in sorted(WORST.items())})


def _st():
    return torch.cuda.current_stream().cuda_stream


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _buf(P, ld, data=None):
    """A NaN-filled [P][ld] row buffer with TAIL NaNs after it; data [P][C] (C <= ld) written into lanes [0, C)."""
    b = torch.empty(P * ld + TAIL, device="cuda")
    b.view(torch.int32).fill_(NAN_BITS)
    if data is not None:
        b[:P * ld].view(P, ld)[:, :data.shape[1]] = data
    return b


def _nans(*shape):
    t = torch.empty(*shape, device="cuda")
    t.view(torch.int32).fill_(NAN_BITS)
    return t


def _rows(b, P, ld):
    return b[:P * ld].view(P, ld)


def _is_sentinel(t):
    return t.contiguous().view(torch.int32) == NAN_BITS


def _check_pads(b, P, ld, c, cw, what):
    """Lanes [c, cw) exactly 0, lanes [cw, ld) and the tail untouched."""
    r = _rows(b, P, ld)
    if cw > c:
        assert bool((r[:, c:cw] == 0).all()) and not bool(torch.signbit(r[:, c:cw]).any()), (what, "zero pad lanes")
    if ld > cw:
        assert bool(_is_sentinel(r[:, cw:]).all()), (what, "lanes past the written width")
    assert bool(_is_sentinel(b[P * ld:]).all()), (what, "past the last row")


def _same_bits(a, b, what):
    assert torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)), (what, "run to run")


def _within(got, ref, tol, family, what):
    """|got - ref| <= tol elementwise (got float32, ref and tol float64); records the worst fraction of the bound used."""
    assert not bool(torch.isnan(got).any()), (what, "NaN")
    err = (got.double() - ref).abs()
    frac = err / tol.clamp_min(1e-300)
    worst = float(frac.max()) if frac.numel() else 0.0
    WORST[family] = max(WORST.get(family, 0.0), worst)
    assert bool((err <= tol).all()), (what, "worst error / bound", worst, "at", int(frac.argmax()))


def esp_splits(P, C):
    """espnet.cu stat_splits / tile_of: -> (row splits, row lanes per block)."""
    tc = min(C, THREADS)
    chunks = -(-C // tc)
    r = min(-(-4 * SMS // chunks), (P + 31) // 32)
    return max(r, 1), THREADS // tc


def mb_splits(P, C, blocks=4 * SMS):
    """mobilenet.cu splits_of / tile4_of (blocks: 4 * SMs for the statistics and BatchNorm backward, 2 * SMs for the weight gradient)."""
    c4 = C // 4
    tc = min(c4, THREADS)
    chunks = -(-c4 // tc)
    r = min(-(-blocks // chunks), (P + 31) // 32)
    return max(r, 1), THREADS // tc


def _depth(P, splits, tr):
    """Longest chain of double additions a term of a split reduction goes through: its thread's rows, the block's row lanes, the
    splits."""
    return -(-(-(-P // splits)) // tr) + tr + splits


# Per-channel data classes of the reductions, channel c gets class c % len(CLASSES): normal data; post-activation data (half
# zeros); mean 10 / std 0.1; a constant channel sitting on a kink (var = 0, so invstd = 1 / sqrt(eps), and z = b exactly); a 100
# sigma outlier in the first row; every z below 0; every z above 6; integers {m - 1, m, m, m + 1} with exact batch statistics (mean
# m, var 1/2) whose rows at m sit on a kink (z = b exactly) in training as in eval.
CLASSES = ("normal", "post_act", "mean10_std0.1", "const_kink", "outlier_100sd", "z_below_0", "z_above_6", "exact_kink")
KINK_M, KINK_V = 3.0, 0.5


def _classed(P, C, seed, kink6):
    """-> x [P][C], w, b, running mean / var (the eval statistics) and the per-channel class index; kink6: the kink channels
    alternate between z = 0 and z = 6 (ReLU6), else sit at z = 0."""
    g = _gen(seed)
    cls = torch.arange(C, device="cuda") % len(CLASSES)
    x = torch.randn(P, C, device="cuda", generator=g) * 1.5 + 0.3
    x = torch.where(cls == 1, torch.relu(torch.randn(P, C, device="cuda", generator=g)), x)
    x = torch.where(cls == 2, torch.randn(P, C, device="cuda", generator=g) * 0.1 + 10.0, x)
    x = torch.where(cls == 3, torch.full_like(x, KINK_M), x)
    out_row = 0.3 + 100 * 1.5 * torch.sign(torch.randn(C, device="cuda", generator=g))
    x[0] = torch.where(cls == 4, out_row, x[0])
    pattern = torch.tensor([KINK_M - 1, KINK_M, KINK_M, KINK_M + 1], device="cuda").repeat(-(-P // 4))[:P]
    x = torch.where(cls == 7, pattern[:, None].expand(P, C), x)
    w = torch.randn(C, device="cuda", generator=g)
    b = torch.randn(C, device="cuda", generator=g) * 0.5
    kink_b = torch.where((torch.arange(C, device="cuda") // len(CLASSES)) % 2 == 1, 6.0, 0.0) if kink6 else torch.zeros(C, device="cuda")
    b = torch.where((cls == 3) | (cls == 7), kink_b, b)
    w = torch.where((cls == 5) | (cls == 6), 0.1 * torch.sign(w), w)
    b = torch.where(cls == 5, torch.full_like(b, -10.0), torch.where(cls == 6, torch.full_like(b, 16.0), b))
    rm = torch.randn(C, device="cuda", generator=g) * 0.3 + x[: min(P, 64)].mean(0)
    rv = torch.rand(C, device="cuda", generator=g) + 0.5
    kink = (cls == 3) | (cls == 7)
    rm = torch.where(kink, torch.full_like(rm, KINK_M), rm)
    rv = torch.where(kink, torch.full_like(rv, KINK_V), rv)
    return x, w, b, rm, rv, cls


def _stats_tol(xd, P, splits, tr):
    """Bounds of the double-partial statistics rounded once to float32: mean within U |mean| plus the double chains, var likewise
    (s2 / P - mean^2 loses what cancels: the double error is relative to mean(x^2), not to var)."""
    depth = _depth(P, splits, tr) + 2
    m64, v64 = xd.mean(0), xd.var(0, unbiased=False)
    tol_m = U * m64.abs() + depth * UD * xd.abs().mean(0)
    tol_v = U * v64 + 3 * depth * UD * (xd * xd).mean(0)
    return m64, v64, tol_m, tol_v


def _check_stats(mean, var, xd, P, splits, tr, family, what, rm=None, rv=None, rm0=None, rv0=None):
    from oracle import student_kernels_ref as R
    m64, v64, tol_m, tol_v = _stats_tol(xd, P, splits, tr)
    _within(mean, m64, tol_m, family + ":mean", what)
    _within(var, v64, tol_v, family + ":var", what)
    if rm is not None:
        # running statistics: the float32 update (1 - m) r + m batch rounds three times, plus the batch value's own error
        ref_m, ref_v = R.running_update(rm0, rv0, m64, v64, P, MOM)
        f = P / (P - 1) if P > 1 else 1.0
        _within(rm, ref_m, 3 * U * (rm0.double().abs() + MOM * m64.abs()) + MOM * tol_m, family + ":running", what)
        _within(rv, ref_v, 3 * U * (rv0.double().abs() + MOM * f * v64) + MOM * f * (tol_v + U * v64), family + ":running", what)


# ---------------------------------------------------------------------------------------------- ESPNet BatchNorm statistics
SYN_BNPRELU_STATS = [
    ("bnprelu_stats", 1, 19, 20, True),              # one row: var = 0
    ("bnprelu_stats", 21, 131, 132, True),           # fewer than 32 rows: a single split
    ("bnprelu_stats", 100003, 19, 20, True),         # rows not divisible by the split count
    ("bnprelu_stats", 4099, 1, 4, True),             # C = 1
    ("bnprelu_stats", 999, 3, 4, False),             # C = 3
    ("bnprelu_stats", 5003, 257, 260, True),         # a second channel chunk of 1 channel
    ("bnprelu_stats", 3001, 260, 264, True),         # ... of 4 channels
]


def _rows_of(name, extra):
    return sorted([s for s in STEP_LAUNCHES if s[0] == name], key=repr) + extra


@pytest.mark.parametrize("sig", _rows_of("bnprelu_stats", SYN_BNPRELU_STATS), ids=repr)
def test_bnprelu_stats_vs_float64(L, sig):
    _, P, C, ld, running = sig
    x, *_ = _classed(P, C, P + C, False)
    xb = _buf(P, ld, x)
    outs = []
    for _ in range(2):
        st = _nans(2, C)
        rm0 = torch.randn(C, device="cuda", generator=_gen(1)) * 0.1
        rv0 = torch.rand(C, device="cuda", generator=_gen(2)) + 0.5
        rm, rv = rm0.clone(), rv0.clone()
        nbt = torch.zeros(1, dtype=torch.int64, device="cuda")
        ws = torch.empty(L.skd_bnprelu_workspace_doubles(P, C), device="cuda", dtype=torch.float64)
        L.skd_bnprelu_stats(P, C, xb.data_ptr(), ld, MOM, rm.data_ptr() if running else None, rv.data_ptr() if running else None,
                            nbt.data_ptr() if running else None, st[0].data_ptr(), st[1].data_ptr(), ws.data_ptr(), _st())
        outs.append((st, rm, rv, nbt))
    (st, rm, rv, nbt), (st2, rm2, rv2, _) = outs
    for a, b_ in ((st, st2), (rm, rm2), (rv, rv2)):
        _same_bits(a, b_, sig)
    splits, tr = esp_splits(P, C)
    _check_stats(st[0], st[1], x.double(), P, splits, tr, "bnprelu_stats", sig, *((rm, rv, rm0, rv0) if running else ()))
    if running:
        assert int(nbt) == 1
    if P > 1:
        assert bool((st[1][3::len(CLASSES)] == 0).all()), "a constant channel has var exactly 0"
    k = torch.arange(C, device="cuda") % len(CLASSES) == 7
    if P % 4 == 0 and bool(k.any()):
        assert bool((st[0][k] == KINK_M).all() and (st[1][k] == KINK_V).all()), "exact integer statistics"


# ---------------------------------------------------------------------------------------------- BatchNorm + activation backward
def _bn_bwd_checks(kind, x, g, mean, var, w, b, alpha, eps, training, red, dx, splits, tr, family, what):
    """The reduce outputs red = (dweight, dbias, dalpha or None, coef [2][C]) and dx [P][C] against float64 from the same float32
    statistics, with the activation mask of the kernel's own float32 z.  Bounds, per element relative to the magnitudes of its terms:
    z carries six float32 roundings and invstd's three; a double-partial sum carries its chain of double additions and one final
    float32 rounding; dx carries a few roundings per term plus the errors of the two coefficients it subtracts."""
    from oracle import student_kernels_ref as R
    P = x.shape[0]
    z32 = R.z_float32(x, mean, var, w, b, eps)
    ref = R.bn_act_backward(x, g, mean, var, w, b, eps, kind, training, alpha, z32)
    xhat, z, dz, k = ref["xhat"], ref["z"], ref["dz"], ref["k"]
    tol_z = 8 * U * ((xhat * w.double()).abs() + b.double().abs())
    depth = _depth(P, splits, tr) + 2
    dweight, dbias, dalpha, coef = red
    tol_db = (2 * U + depth * UD) * ref["dbias_mag"]
    tol_dw = (8 * U + depth * UD) * ref["dweight_mag"]
    _within(dbias, ref["dbias"], tol_db, family + ":dbias", what)
    _within(dweight, ref["dweight"], tol_dw, family + ":dweight", what)
    if dalpha is not None:
        neg = ~(z32 > 0)
        tol_da = torch.where(neg, tol_z * g.double().abs(), torch.zeros_like(z)).sum(0) + (U + depth * UD) * ref["dalpha_mag"]
        _within(dalpha, ref["dalpha"], tol_da, family + ":dalpha", what)
    tol_c0 = tol_db / P + U * ref["coef"][0].abs()
    tol_c1 = tol_dw / P + U * ref["coef"][1].abs()
    _within(coef[0], ref["coef"][0], tol_c0, family + ":coef", what)
    _within(coef[1], ref["coef"][1], tol_c1, family + ":coef", what)
    if training:
        tol_dx = 14 * U * ref["dx_mag"] + k.abs() * (tol_c0 + xhat.abs() * tol_c1)
    else:
        tol_dx = 6 * U * ref["dx_mag"]
    _within(dx, ref["dx"], tol_dx, family + ":dx", what)
    return z32


def _kink_checks(kind, x, g, w, alpha, mean, var, eps, training, red, dx, cls, what):
    """The kinks pinned exactly: elements with x == mean have z == b in {0, 6}.  ReLU6 passes nothing there (eval: dx exactly 0; a
    channel on a kink throughout: dweight and dbias exactly 0); PReLU takes the slope: eval dx = (alpha g) (w invstd) bit for bit, and
    a channel at z == 0 throughout has dweight and dalpha exactly 0."""
    on = (x == mean[None, :]) & ((cls == 3) | (cls == 7))[None, :]
    if not bool(on.any()):
        return
    const = (cls == 3) & (x == mean[None, :]).all(0)
    if kind == "relu6":
        if not training:
            assert bool((dx[on] == 0).all()), (what, "ReLU6 dx at a kink")
        if bool(const.any()):
            assert bool((red[0][const] == 0).all() and (red[1][const] == 0).all()), (what, "ReLU6 dweight / dbias of a kink channel")
    elif kind == "prelu" and alpha is not None:
        if not training:
            is32 = 1.0 / torch.sqrt(var + eps)
            want = (alpha[None, :] * g) * (w * is32)[None, :]
            assert torch.equal(dx[on], want.expand_as(dx)[on]), (what, "PReLU dx at z = 0")
        if bool(const.any()):
            assert bool((red[0][const] == 0).all() and (red[2][const] == 0).all()), (what, "PReLU dweight / dalpha at z = 0")


def _esp_stats(L, xb, P, C, ld):
    st = _nans(2, C)
    ws = torch.empty(L.skd_bnprelu_workspace_doubles(P, C), device="cuda", dtype=torch.float64)
    L.skd_bnprelu_stats(P, C, xb.data_ptr(), ld, MOM, None, None, None, st[0].data_ptr(), st[1].data_ptr(), ws.data_ptr(), _st())
    return st


def _p(t):
    return None if t is None else t.data_ptr()


# (P, C, ldx, ldd, cw, ldo, alpha, training) of each ESPNet BatchNorm (+ PReLU) launch
def _bnprelu_cases():
    cases = set()
    for s in STEP_LAUNCHES:
        if s[0] == "bnprelu_apply":
            _, P, C, ld, cw, ldo, a = s
            cases.add((P, C, ld, cw, cw, ldo, a, True))
        elif s[0] == "bnprelu_bwd_reduce":
            _, P, C, ld, ldd, a = s
            cases.add((P, C, ld, ldd, (C + 3) // 4 * 4, (C + 3) // 4 * 4, a, True))
        elif s[0] == "bnprelu_bwd_dx":
            _, P, C, ld, ldd, cw, tr, a = s
            cases.add((P, C, ld, ldd, cw, cw, a, tr))
    return sorted(cases) + [
        (1, 19, 20, 20, 20, 24, True, True),             # one row
        (21, 131, 132, 132, 132, 136, True, False),      # a single split; eval
        (100003, 19, 20, 20, 20, 20, True, True),        # rows not divisible by the split count
        (4099, 1, 4, 1, 4, 8, True, True),               # C = 1
        (999, 3, 4, 4, 4, 4, False, False),              # C = 3, plain BatchNorm, eval
        (5003, 257, 260, 257, 260, 264, True, True),     # a second channel chunk of 1 channel
        (3001, 260, 264, 260, 260, 260, True, False),    # ... of 4 channels
        (43200, 256, 256, 256, 256, 256, True, False),   # the level-3 shape with running statistics
        (172800, 19, 20, 20, 20, 20, False, False),
    ]


@pytest.mark.parametrize("case", _bnprelu_cases(), ids=repr)
def test_bnprelu_apply_backward_vs_float64(L, case):
    from oracle import student_kernels_ref as R
    P, C, ld, ldd, cw, ldo, with_alpha, training = case
    x, w, b, rm, rv, cls = _classed(P, C, P * 7 + C, False)
    g = torch.randn(P, C, device="cuda", generator=_gen(P + 1))
    alpha = torch.rand(C, device="cuda", generator=_gen(C)) * 0.45 + 0.05 if with_alpha else None
    xb, gb = _buf(P, ld, x), _buf(P, ldd, g)
    eps = EPS_ESP
    mean, var = _esp_stats(L, xb, P, C, ld) if training else (rm, rv)
    runs = []
    for _ in range(2):
        out = _buf(P, ldo)
        L.skd_bnprelu_apply(P, C, xb.data_ptr(), ld, mean.data_ptr(), var.data_ptr(), w.data_ptr(), b.data_ptr(), _p(alpha), eps,
                            out.data_ptr(), ldo, cw, _st())
        red = _nans(5, C)
        ws = torch.empty(L.skd_bnprelu_workspace_doubles(P, C), device="cuda", dtype=torch.float64)
        L.skd_bnprelu_bwd_reduce(P, C, xb.data_ptr(), ld, gb.data_ptr(), ldd, mean.data_ptr(), var.data_ptr(), w.data_ptr(),
                                 b.data_ptr(), _p(alpha), eps, red[0].data_ptr(), red[1].data_ptr(), _p(red[2] if with_alpha else None),
                                 red[3].data_ptr(), ws.data_ptr(), _st())
        dxb = _buf(P, cw)
        L.skd_bnprelu_bwd_dx(P, C, xb.data_ptr(), ld, gb.data_ptr(), ldd, mean.data_ptr(), var.data_ptr(), w.data_ptr(), b.data_ptr(),
                             _p(alpha), eps, int(training), red[3].data_ptr(), dxb.data_ptr(), cw, cw, _st())
        runs.append((out, red, dxb))
    for a, b_ in zip(*runs):
        _same_bits(a, b_, case)
    out, red, dxb = runs[0]
    _check_pads(out, P, ldo, C, cw, (case, "apply"))
    _check_pads(dxb, P, cw, C, cw, (case, "dx"))
    y = _rows(out, P, ldo)[:, :C]
    # forward: bit for bit the float32 z rounded step by step, then within the float64 bound
    z32 = R.z_float32(x, mean, var, w, b, eps)
    want = torch.where(z32 > 0, z32, alpha * z32) if with_alpha else z32
    _same_bits(y, want, (case, "apply vs float32 z"))
    xhat, z, _ = R.bn_z(x, mean, var, w, b, eps)
    tol_z = 8 * U * ((xhat * w.double()).abs() + b.double().abs())
    y64 = torch.where(z32 > 0, z, alpha.double() * z) if with_alpha else z
    _within(y, y64, tol_z + U * y64.abs(), "bnprelu_apply", case)
    splits, tr = esp_splits(P, C)
    reds = (red[0], red[1], red[2] if with_alpha else None, red[3:5])
    dx = _rows(dxb, P, cw)[:, :C]
    _bn_bwd_checks("prelu", x, g, mean, var, w, b, alpha, eps, training, reds, dx, splits, tr, "bnprelu_bwd", case)
    _kink_checks("prelu", x, g, w, alpha, mean, var, eps, training, reds, dx, cls, case)


# ---------------------------------------------------------------------------------------------- ESP module combine and backward
SYN_ESP_COMBINE = [
    ("esp_combine", 4099, 5, 8, 3, 4, 20, 20, True, True),       # n1 != n, padded pitches, residual
    ("esp_combine", 1, 2, 4, 1, 4, 0, 8, True, True),            # one row
    ("esp_combine", 777, 28, 28, 25, 28, 132, 132, True, False),  # residual pitch wider than C
    ("esp_combine", 3001, 1, 4, 64, 64, 0, 260, True, True),     # C = 257: a second channel chunk of 1 channel
]


@pytest.mark.parametrize("sig", _rows_of("esp_combine", SYN_ESP_COMBINE), ids=repr)
def test_esp_combine_vs_float64(L, sig):
    from oracle import student_kernels_ref as R
    _, P, n1, ld1, n, ldn, ldr, ldo, stats, running = sig
    C = n1 + 4 * n
    g = _gen(P + n1 + n)
    d = [torch.randn(P, k, device="cuda", generator=g) * s for k, s in ((n1, 1.0), (n, 1.0), (n, 0.5), (n, 2.0), (n, 0.25))]
    res = torch.randn(P, C, device="cuda", generator=g) * 3 + 1 if ldr else None
    bufs = [_buf(P, ld1, d[0])] + [_buf(P, ldn, t) for t in d[1:]]
    rb = _buf(P, ldr, res) if ldr else None
    runs = []
    for _ in range(2):
        out = _buf(P, ldo)
        st = _nans(2, C)
        rm0, rv0 = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
        rm, rv = rm0.clone(), rv0.clone()
        ws = torch.empty(L.skd_bnprelu_workspace_doubles(P, C), device="cuda", dtype=torch.float64)
        L.skd_esp_combine(P, n1, n, *[t.data_ptr() for t in bufs[:1]], ld1, *[t.data_ptr() for t in bufs[1:]], ldn, _p(rb), ldr,
                          out.data_ptr(), ldo, MOM, rm.data_ptr() if running else None, rv.data_ptr() if running else None, None,
                          st[0].data_ptr() if stats else None, st[1].data_ptr() if stats else None, ws.data_ptr(), _st())
        runs.append((out, st, rm, rv))
    for a, b_ in zip(*runs):
        _same_bits(a, b_, sig)
    out, st, rm, rv = runs[0]
    _check_pads(out, P, ldo, C, C, sig)
    comb = _rows(out, P, ldo)[:, :C]
    # the additions in the module's order, float32: bit for bit; float64: one rounding per addition
    a1 = d[1]
    a2 = a1 + d[2]
    a3 = a2 + d[3]
    a4 = a3 + d[4]
    want = torch.cat([d[0], a1, a2, a3, a4], 1)
    _same_bits(comb, res + want if ldr else want, (sig, "combine vs float32 order"))
    v64, mag = R.esp_combine(*d, res)
    _within(comb, v64, 4 * U * mag, "esp_combine", sig)
    if stats:
        splits, tr = esp_splits(P, C)
        _check_stats(st[0], st[1], comb.double(), P, splits, tr, "esp_combine_stats", sig,
                     *((rm, rv, torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")) if running else ()))


SYN_ESP_BWD = [
    ("esp_bwd_dx", 4099, 5, 3, 20, 20, True, True, True),        # n1 != n, residual
    ("esp_bwd_dx", 1, 2, 1, 8, 8, True, True, True),             # one row
    ("esp_bwd_dx", 777, 28, 25, 128, 132, False, True, True),    # eval, padded dout
    ("esp_bwd_dx", 3001, 1, 64, 260, 257, True, True, False),    # C = 257
    ("esp_bwd_dx", 43200, 28, 25, 128, 128, False, False, True),  # plain BatchNorm, eval
]


@pytest.mark.parametrize("sig", _rows_of("esp_bwd_dx", SYN_ESP_BWD), ids=repr)
def test_esp_bwd_dx_vs_float64(L, sig):
    """The ESP backward: each channel's BatchNorm + PReLU input gradient is the very value bnprelu_bwd_dx gives (bit for bit), the
    branch gradients its suffix sums added in float32 in the kernel's order (bit for bit), all within the float64 bounds."""
    from oracle import student_kernels_ref as R
    _, P, n1, n, ldx, ldd, training, with_alpha, want_dres = sig
    C = n1 + 4 * n
    x, w, b, rm, rv, cls = _classed(P, C, P + 3 * C, False)
    g = torch.randn(P, C, device="cuda", generator=_gen(P + 5))
    alpha = torch.rand(C, device="cuda", generator=_gen(C + 1)) * 0.45 + 0.05 if with_alpha else None
    xb, gb = _buf(P, ldx, x), _buf(P, ldd, g)
    eps = EPS_ESP
    mean, var = _esp_stats(L, xb, P, C, ldx) if training else (rm, rv)
    red = _nans(5, C)
    ws = torch.empty(L.skd_bnprelu_workspace_doubles(P, C), device="cuda", dtype=torch.float64)
    L.skd_bnprelu_bwd_reduce(P, C, xb.data_ptr(), ldx, gb.data_ptr(), ldd, mean.data_ptr(), var.data_ptr(), w.data_ptr(), b.data_ptr(),
                             _p(alpha), eps, red[0].data_ptr(), red[1].data_ptr(), _p(red[2] if with_alpha else None), red[3].data_ptr(),
                             ws.data_ptr(), _st())
    l1, ln = (n1 + 3) // 4 * 4, (n + 3) // 4 * 4
    runs = []
    for _ in range(2):
        dd = [_buf(P, l1)] + [_buf(P, ln) for _ in range(4)]
        dres = _buf(P, C) if want_dres else None
        L.skd_esp_bwd_dx(P, n1, n, xb.data_ptr(), ldx, gb.data_ptr(), ldd, mean.data_ptr(), var.data_ptr(), w.data_ptr(), b.data_ptr(),
                         _p(alpha), eps, int(training), red[3].data_ptr(), dd[0].data_ptr(), l1, *[t.data_ptr() for t in dd[1:]], ln,
                         _p(dres), C, _st())
        runs.append(dd + ([dres] if want_dres else []))
    for a, b_ in zip(*runs):
        _same_bits(a, b_, sig)
    dd = runs[0][:5]
    _check_pads(dd[0], P, l1, n1, l1, (sig, "dd1"))
    for t in dd[1:]:
        _check_pads(t, P, ln, n, ln, (sig, "dd"))
    dxb = _buf(P, C)
    L.skd_bnprelu_bwd_dx(P, C, xb.data_ptr(), ldx, gb.data_ptr(), ldd, mean.data_ptr(), var.data_ptr(), w.data_ptr(), b.data_ptr(),
                         _p(alpha), eps, int(training), red[3].data_ptr(), dxb.data_ptr(), C, C, _st())
    gk = _rows(dxb, P, C)
    if want_dres:
        _check_pads(runs[0][5], P, C, C, C, (sig, "dres"))
        _same_bits(_rows(runs[0][5], P, C), gk, (sig, "dres vs bnprelu_bwd_dx"))
    sl = [gk[:, n1 + q * n:n1 + (q + 1) * n] for q in range(4)]
    s16 = sl[3]
    s8 = sl[2] + s16
    s4 = sl[1] + s8
    s2 = sl[0] + s4
    got = [_rows(dd[0], P, l1)[:, :n1]] + [_rows(t, P, ln)[:, :n] for t in dd[1:]]
    for a, b_ in zip(got, (gk[:, :n1], s2, s4, s8, s16)):
        _same_bits(a, b_, (sig, "suffix sums vs float32 order"))
    splits, tr = esp_splits(P, C)
    reds = (red[0], red[1], red[2] if with_alpha else None, red[3:5])
    _bn_bwd_checks("prelu", x, g, mean, var, w, b, alpha, eps, training, reds, gk, splits, tr, "esp_bwd", sig)
    _kink_checks("prelu", x, g, w, alpha, mean, var, eps, training, reds, gk, cls, sig)
    # the suffix sums against float64: the float64 slices' sums, each float32 addition one more rounding
    ref = R.bn_act_backward(x, g, mean, var, w, b, eps, "prelu", training, alpha, R.z_float32(x, mean, var, w, b, eps))
    gd = gk.double()
    want64 = R.esp_combine_backward(ref["dx"], n1, n)
    err_in = R.esp_combine_backward((gd - ref["dx"]).abs(), n1, n)       # the slices' own (already bounded) errors, carried along
    mag = R.esp_combine_backward(gd.abs(), n1, n)
    for a, r64, e, m in zip(got, want64, err_in, mag):
        _within(a, r64, e + 3 * U * m + 1e-300, "esp_bwd:suffix", sig)


# ---------------------------------------------------------------------------------------------- MobileNetV2 BatchNorm + ReLU6 / linear
# (P, C, ldx, relu6, residual, training) of each MobileNetV2 BatchNorm launch
def _bnact_cases():
    cases = set()
    for s in STEP_LAUNCHES:
        if s[0] == "bnact_apply":
            cases.add((s[1], s[2], s[3], s[4], s[5] != 0, True))
        elif s[0] in ("bnact_bwd_reduce", "bnact_bwd_dx"):
            cases.add((s[1], s[2], s[3], s[5], False, s[6] if s[0] == "bnact_bwd_dx" else True))
    return sorted(cases) + [
        (1, 32, 32, True, False, True),                  # one row
        (21, 96, 96, True, False, False),                # a single split; eval
        (100003, 24, 24, False, True, True),             # rows not divisible by the split count
        (4099, 4, 4, True, False, True),                 # one channel quad
        (5003, 1028, 1028, True, False, True),           # c4 = 257: a second chunk of one quad
        (3001, 1028, 1028, False, True, False),          # ... linear, residual, eval
        (65536, 960, 960, True, False, False),           # the dilated blocks with running statistics
    ]


@pytest.mark.parametrize("case", _bnact_cases(), ids=repr)
def test_bnact_apply_backward_vs_float64(L, case):
    from oracle import student_kernels_ref as R
    P, C, ld, relu6, with_res, training = case
    kind = "relu6" if relu6 else "linear"
    x, w, b, rm, rv, cls = _classed(P, C, P * 3 + C, relu6)
    g = torch.randn(P, C, device="cuda", generator=_gen(P + 2))
    res = torch.randn(P, C, device="cuda", generator=_gen(P + 3)) if with_res else None
    xb, gb = _buf(P, ld, x), _buf(P, ld, g)
    rb = _buf(P, ld, res) if with_res else None
    eps = EPS_MB
    mean, var = _esp_stats(L, xb, P, C, ld) if training else (rm, rv)
    runs = []
    for _ in range(2):
        out = _buf(P, C)
        L.skd_bnact_apply(P, C, int(relu6), xb.data_ptr(), ld, mean.data_ptr(), var.data_ptr(), w.data_ptr(), b.data_ptr(), eps, _p(rb),
                          ld if with_res else 0, out.data_ptr(), C, _st())
        red = _nans(4, C)
        ws = torch.empty(max(L.skd_mbv2_workspace_doubles(P, C), 1), device="cuda", dtype=torch.float64)
        L.skd_bnact_bwd_reduce(P, C, int(relu6), xb.data_ptr(), ld, gb.data_ptr(), ld, mean.data_ptr(), var.data_ptr(), w.data_ptr(),
                               b.data_ptr(), eps, red[0].data_ptr(), red[1].data_ptr(), red[2].data_ptr(), ws.data_ptr(), _st())
        dxb = _buf(P, C)
        L.skd_bnact_bwd_dx(P, C, int(relu6), xb.data_ptr(), ld, gb.data_ptr(), ld, mean.data_ptr(), var.data_ptr(), w.data_ptr(),
                           b.data_ptr(), eps, int(training), red[2].data_ptr(), dxb.data_ptr(), C, _st())
        runs.append((out, red, dxb))
    for a, b_ in zip(*runs):
        _same_bits(a, b_, case)
    out, red, dxb = runs[0]
    _check_pads(out, P, C, C, C, (case, "apply"))
    _check_pads(dxb, P, C, C, C, (case, "dx"))
    y = _rows(out, P, C)
    z32 = R.z_float32(x, mean, var, w, b, eps)
    want = z32.clamp(0.0, 6.0) if relu6 else (res + z32 if with_res else z32)
    _same_bits(y, want, (case, "apply vs float32 z"))
    xhat, z, _ = R.bn_z(x, mean, var, w, b, eps)
    tol_z = 8 * U * ((xhat * w.double()).abs() + b.double().abs())
    if relu6:
        _within(y, R.relu6(z), tol_z, "bnact_apply", case)
    else:
        y64 = z + res.double() if with_res else z
        _within(y, y64, tol_z + U * (y64.abs() + (res.double().abs() if with_res else 0)), "bnact_apply", case)
    splits, tr = mb_splits(P, C)
    reds = (red[0], red[1], None, red[2:4])
    dx = _rows(dxb, P, C)
    _bn_bwd_checks(kind, x, g, mean, var, w, b, None, eps, training, reds, dx, splits, tr, "bnact_bwd", case)
    _kink_checks(kind, x, g, w, None, mean, var, eps, training, reds, dx, cls, case)


# ---------------------------------------------------------------------------------------------- depthwise 3x3
SYN_DW = [
    (2, 8, 7, 9, 1, 1), (2, 8, 7, 9, 2, 1),           # odd maps
    (1, 12, 1, 37, 2, 1), (3, 4, 33, 1, 2, 2),        # 1 x k and k x 1
    (1, 1028, 5, 6, 1, 1),                            # c4 = 257: a second chunk of one quad
    (2, 16, 9, 11, 2, 4), (1, 4, 3, 3, 1, 8),         # dilation beyond the map
]


def _dw_cases():
    cases = set()
    for s in STEP_LAUNCHES:
        if s[0] == "dwconv3x3_fwd":
            cases.add(("fwd",) + s[1:7] + (s[7],))
        elif s[0] in ("dwconv3x3_dgrad", "dwconv3x3_wgrad"):
            cases.add((s[0][10:],) + s[1:7] + (False,))
    syn = [(k,) + s + (st,) for s in SYN_DW for k, st in (("fwd", True), ("fwd", False), ("dgrad", False), ("wgrad", False))]
    return sorted(cases) + syn


@pytest.mark.parametrize("case", _dw_cases(), ids=repr)
def test_depthwise_vs_float64(L, case):
    from oracle import student_kernels_ref as R
    kind, N, C, H, W, s, d, stats = case
    OH, OW = (H - 1) // s + 1, (W - 1) // s + 1
    g = _gen(N * C + H * W + s + d)
    wt = torch.randn(C, 1, 3, 3, device="cuda", generator=g)
    x = torch.randn(N, H, W, C, device="cuda", generator=g) * 1.5 + 0.3
    dy = torch.randn(N, OH, OW, C, device="cuda", generator=g)
    P_in, P_out = N * H * W, N * OH * OW
    xb, dyb = _buf(P_in, C, x.view(P_in, C)), _buf(P_out, C, dy.view(P_out, C))
    nchw = lambda t, h, w_: t.view(N, h, w_, C).permute(0, 3, 1, 2)                          # noqa: E731
    runs = []
    for _ in range(2):
        if kind == "fwd":
            yb = _buf(P_out, C)
            st = _nans(2, C)
            rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
            ws = torch.empty(max(L.skd_mbv2_workspace_doubles(P_out, C), 1), device="cuda", dtype=torch.float64)
            L.skd_dwconv3x3_fwd(N, H, W, C, s, d, xb.data_ptr(), wt.data_ptr(), yb.data_ptr(), MOM, _p(rm if stats else None),
                                _p(rv if stats else None), None, _p(st[0] if stats else None), _p(st[1] if stats else None),
                                ws.data_ptr(), _st())
            runs.append((yb, st, rm, rv) if stats else (yb,))
        elif kind == "dgrad":
            dxb = _buf(P_in, C)
            L.skd_dwconv3x3_dgrad(N, H, W, C, s, d, dyb.data_ptr(), wt.data_ptr(), dxb.data_ptr(), _st())
            runs.append((dxb,))
        else:
            dwb = _buf(C, 9)
            ws = torch.empty(max(L.skd_mbv2_workspace_doubles(P_out, C), 1), device="cuda", dtype=torch.float64)
            L.skd_dwconv3x3_wgrad(N, H, W, C, s, d, xb.data_ptr(), dyb.data_ptr(), dwb.data_ptr(), ws.data_ptr(), _st())
            runs.append((dwb,))
    for a, b_ in zip(*runs):
        _same_bits(a, b_, case)
    if kind == "fwd":
        yb = runs[0][0]
        _check_pads(yb, P_out, C, C, C, case)
        y = _rows(yb, P_out, C)
        ref, mag = R.dwconv3x3(nchw(x, H, W), wt, s, d)
        # nine fused multiply-adds in a chain: 9 u of the sum of the magnitudes
        _within(y, ref.permute(0, 2, 3, 1).reshape(P_out, C), 9 * U * mag.permute(0, 2, 3, 1).reshape(P_out, C), "dw_fwd", case)
        if stats:
            _, st, rm, rv = runs[0]
            splits, tr = mb_splits(P_out, C)
            _check_stats(st[0], st[1], y.double(), P_out, splits, tr, "dw_fwd_stats", case, rm, rv, torch.zeros(C, device="cuda"),
                         torch.ones(C, device="cuda"))
    elif kind == "dgrad":
        dxb = runs[0][0]
        _check_pads(dxb, P_in, C, C, C, case)
        ref, mag = R.dwconv3x3_dgrad(nchw(dy, OH, OW), wt, (N, C, H, W), s, d)
        _within(_rows(dxb, P_in, C), ref.permute(0, 2, 3, 1).reshape(P_in, C), 9 * U * mag.permute(0, 2, 3, 1).reshape(P_in, C),
                "dw_dgrad", case)
    else:
        dwb = runs[0][0]
        _check_pads(dwb, C, 9, 9, 9, case)
        ref, mag = R.dwconv3x3_wgrad(nchw(x, H, W), nchw(dy, OH, OW), s, d)
        splits, tr = mb_splits(P_out, C, 2 * SMS)
        rpt = -(-(-(-P_out // splits)) // tr)
        # each thread's rows as a float32 chain of fused multiply-adds, the lanes and splits added in double, one final rounding
        tol = (rpt * U + (tr + splits + 2) * UD + U) * mag.view(C, 9)
        _within(_rows(dwb, C, 9), ref.view(C, 9), tol, "dw_wgrad", case)


# ---------------------------------------------------------------------------------------------- average pooling
SYN_POOL = [
    ("avgpool3x3s2", 2, 7, 9, 3, 4, 20),
    ("avgpool3x3s2", 1, 1, 13, 1, 1, 4),
    ("avgpool3x3s2", 3, 11, 1, 5, 8, 5),
    ("avgpool3x3s2", 1, 1, 1, 3, 3, 3),
    ("avgpool3x3s2", 2, 6, 8, 3, 20, 132),
]


@pytest.mark.parametrize("sig", _rows_of("avgpool3x3s2", SYN_POOL), ids=repr)
def test_avgpool3x3s2_vs_float64(L, sig):
    """nn.AvgPool2d(3, 2, 1) into a channel slice of a wider buffer: C lanes written, every other lane of the destination untouched."""
    from oracle import student_kernels_ref as R
    _, N, H, W, C, lds, ldd = sig
    OH, OW = (H + 1) // 2, (W + 1) // 2
    x = torch.rand(N * H * W, C, device="cuda", generator=_gen(H * W + C)) * 255 - 120
    xb = _buf(N * H * W, lds, x)
    runs = []
    for _ in range(2):
        ob = _buf(N * OH * OW, ldd)
        L.skd_avgpool3x3s2(N, H, W, C, xb.data_ptr(), lds, ob.data_ptr(), ldd, _st())
        runs.append(ob)
    _same_bits(runs[0], runs[1], sig)
    P = N * OH * OW
    _check_pads(runs[0], P, ldd, C, C, sig)
    ref, mag = R.avgpool3x3s2(x.view(N, H, W, C).permute(0, 3, 1, 2))
    # up to nine float32 additions and the division
    _within(_rows(runs[0], P, ldd)[:, :C], ref.permute(0, 2, 3, 1).reshape(P, C), 10 * U * mag.permute(0, 2, 3, 1).reshape(P, C),
            "avgpool", sig)


# ---------------------------------------------------------------------------------------------- bilinear resample and its adjoint
SYN_RESAMPLE = [(2, 3, 5, 7, 5, 7), (1, 5, 1, 9, 4, 1), (2, 4, 6, 1, 1, 13), (1, 3, 17, 23, 40, 90), (1, 2, 40, 90, 17, 23),
                (1, 3, 1, 1, 5, 6), (2, 3, 9, 4, 1, 1)]


def _resample_cases():
    cases = set()
    for s in STEP_LAUNCHES:
        if s[0] == "resample_nhwc":
            cases.add(("fwd",) + s[1:7] + (s[8],))
        elif s[0] == "resample_adjoint_nhwc":
            _, n, c, H, W, h, w, cw = s
            cases.add(("adjoint", n, c, h, w, H, W, cw))
    syn = [(k, n, c, h, w, H, W, c + 1) for (n, c, h, w, H, W) in SYN_RESAMPLE for k in ("fwd", "adjoint")]
    return sorted(cases) + syn


@pytest.mark.parametrize("case", _resample_cases(), ids=repr)
def test_resample_vs_float64(L, case):
    """Against the float64 product with the kernels' own float32 taps (pinned: float32 rounding only) and against the float64
    resample itself (the float32 source coordinates move each tap by a few ulps of the map size)."""
    from oracle import student_kernels_ref as R
    kind, N, C, h, w, H, W, ld = case
    g = _gen(h * w + H * W + C)
    shift = 4 * U * max(h, w, H, W) * 2
    if kind == "fwd":
        x = torch.randn(N, h, w, C, device="cuda", generator=g)
        xb = _buf(N * h * w, ld, x.view(-1, C))
        runs = []
        for _ in range(2):
            ob = _buf(N * H * W, C)
            L.skd_resample_bilinear_nhwc(N, C, h, w, xb.data_ptr(), h * w * ld, 1, ld, H, W, ob.data_ptr(), _st())
            runs.append(ob)
        _same_bits(runs[0], runs[1], case)
        _check_pads(runs[0], N * H * W, C, C, C, case)
        got = _rows(runs[0], N * H * W, C).view(N, H, W, C).permute(0, 3, 1, 2)
        xc = x.permute(0, 3, 1, 2)
        ref, mag = R.resample_pinned(xc, H, W)
        _within(got, ref, 5 * U * mag, "resample:pinned", case)
        _within(got, R.resample(xc, H, W), 5 * U * mag + shift * float(x.abs().max()), "resample:float64", case)
    else:
        dout = torch.randn(N, H, W, C, device="cuda", generator=g)
        db = _buf(N * H * W, C, dout.view(-1, C))
        runs = []
        for _ in range(2):
            ob = _buf(N * h * w, ld)
            L.skd_resample_bilinear_adjoint_nhwc(N, C, h, w, db.data_ptr(), H, W, ob.data_ptr(), ld, _st())
            runs.append(ob)
        _same_bits(runs[0], runs[1], case)
        _check_pads(runs[0], N * h * w, ld, C, C, case)
        got = _rows(runs[0], N * h * w, ld)[:, :C].reshape(N, h, w, C).permute(0, 3, 1, 2)
        dc = dout.permute(0, 3, 1, 2)
        ref, mag, chain = R.resample_adjoint_pinned(dc, h, w)
        # each output row's column sum is a float32 chain, then the rows' chain: (columns + rows + 2) u of the magnitudes
        _within(got, ref, (chain + 2) * U * mag, "resample_adjoint:pinned", case)
        xs = torch.zeros(N, C, h, w, device="cuda", dtype=torch.float64, requires_grad=True)
        R.resample(xs, H, W).backward(dc.double())
        _within(got, xs.grad, (chain + 2) * U * mag + shift * float(mag.max()), "resample_adjoint:float64", case)


# ---------------------------------------------------------------------------------------------- launch geometry reached
def test_rows_reach_every_reduction_path():
    """The table's rows and the synthetic ones drive each geometry path of the split reductions and the grid-stride loops."""
    esp = [(P, C) for (P, C, *_r) in _bnprelu_cases()] + [(s[1], s[2]) for s in _rows_of("bnprelu_stats", SYN_BNPRELU_STATS)]
    geo = [(P, C) + esp_splits(P, C) for P, C in esp]
    assert any(sp == 1 for _, _, sp, _ in geo) and any(sp > 100 and P % sp for P, _, sp, _ in geo)
    assert any(C > 256 and C % 256 in (1, 4) for _, C, _, _ in geo)                       # second channel chunk of 1 and 4 channels
    assert any(256 % C for _, C, _, _ in geo if C < 256)                                   # idle threads in a block
    assert any(P * C > SMS * 16 * THREADS * 2 for P, C, _, _ in geo)                       # elementwise grid-stride loops repeat
    mb = [(P, C) for (P, C, *_r) in _bnact_cases()]
    assert any(C // 4 == 257 for _, C in mb) and any(mb_splits(P, C)[0] == 1 for P, C in mb)
    assert any(P % mb_splits(P, C)[0] and mb_splits(P, C)[0] > 100 for P, C in mb)
