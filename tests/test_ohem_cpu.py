"""CPU: the OHEM cross entropy (OhemCrossEntropy2d / CriterionOhemDSN) -- the restatement in tools/ohem_oracle.py against the
golden fixture made by the UNMODIFIED reference classes, the grid rule the CUDA grid-sample kernel implements against scipy,
and the public surface (imports, no CPU fallback, header, NetModel options)."""
import os

import numpy as np
import pytest
import scipy.ndimage as nd
import torch

from tools import ohem_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gold():
    return torch.load(os.path.join(ROOT, "tests", "golden", "ohem.pt"), weights_only=False)


def _rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-12)


@pytest.mark.parametrize("name", sorted(O.OHEM_CASES))
def test_restatement_matches_reference_golden(name):
    G = _gold()["criterion"][name]
    preds, labels = O.ohem_inputs(name)
    loss, thr, kept = O.port_loss(name, preds, labels)
    assert _rel(loss, G["loss"]) <= 1e-6, (float(loss), G["loss"])
    assert np.float32(thr) == np.float32(G["threshold"]) and kept == G["kept"], (thr, G["threshold"], kept, G["kept"])


def test_golden_cases_cover_the_threshold_rule():
    G = _gold()["criterion"]
    assert G["dsn_65x129_512x1024"]["threshold"] == np.float32(0.7)
    assert G["dsn_confident_65x129"]["threshold"] > 0.7
    assert G["dsn_all_kept_64x64"]["threshold"] == 1.0
    assert G["dsn_zero_column_360x480"]["threshold"] > 0.7
    # the golden step drops about half of the valid pixels, so it checks the mask and not just the plain DSN loss
    S = _gold()["step"]
    assert S["threshold"] < 0.7 and 0.3 * S["valid"] < S["kept"] < 0.7 * S["valid"]
    plain = torch.load(os.path.join(ROOT, "tests", "golden", "steps.pt"), weights_only=False)["pi_pa_96x128"]
    assert _rel(S["ce"], plain["ce"]) > 1e-2
    assert os.path.getsize(os.path.join(ROOT, "tests", "golden", "ohem.pt")) < 1 << 20


def test_zero_column_at_360x480_shifts_the_order_statistic():
    """59 * (479 / 59) = 479.00000000000006 > 479: scipy's 'constant' mode reads 0 for the last grid column, probability AND
    label, and those valid zero points are the hardest of the grid."""
    import torch.nn.functional as F
    preds, labels = O.ohem_inputs("dsn_zero_column_360x480")
    prob = torch.softmax(F.interpolate(preds[0], size=(360, 480), mode="bilinear", align_corners=True), 1).numpy()
    pred, glab = O.ohem_grid(prob, labels.numpy(), 8)
    assert pred.shape == (2, 45, 60)
    assert (pred[:, :, -1] == 0).all() and (glab[:, :, -1] == 0).all()
    mk = 100000 // 64
    without = O.ohem_threshold(np.where(np.isfinite(pred[:, :, :-1]), pred[:, :, :-1], np.inf), mk, 0.7)
    assert O.ohem_threshold(pred, mk, 0.7) != without


def test_grid_size_rounds_half_to_even():
    from structure_knowledge_distillation_b200 import ops
    assert O.grid_shape(36, 44, 8) == (4, 6) == ops.ohem_grid_shape(36, 44, 8)
    for H, W, f in ((512, 1024, 8), (360, 480, 8), (97, 131, 4), (37, 45, 3)):
        z = nd.zoom(np.zeros((H, W), np.float32), (1.0 / f, 1.0 / f), order=1)
        assert z.shape == ops.ohem_grid_shape(H, W, f) == O.grid_shape(H, W, f)


# the arithmetic of ohem_grid_kernel (csrc/ohem.cu), written out in numpy
def _coords(n_in, n_out):
    r = (n_in - 1) / (n_out - 1) if n_out > 1 else 1.0
    c = np.arange(n_out, dtype=np.float64) * r
    return c, c > n_in - 1


def _kernel_rule(prob, target, gh, gw):
    H, W = target.shape[-2:]
    cy, oy = _coords(H, gh)
    cx, ox = _coords(W, gw)
    iy = np.minimum(np.floor(cy + 0.5).astype(int), H - 1)
    ix = np.minimum(np.floor(cx + 0.5).astype(int), W - 1)
    lab = target[..., iy[:, None], ix]
    lab[..., oy, :] = 0
    lab[..., :, ox] = 0
    y0 = np.minimum(np.floor(cy).astype(int), H - 1); ty = (cy - y0)[:, None]; y1 = np.minimum(y0 + 1, H - 1)
    x0 = np.minimum(np.floor(cx).astype(int), W - 1); tx = cx - x0; x1 = np.minimum(x0 + 1, W - 1)
    P = prob.astype(np.float64)
    Y0, Y1 = y0[:, None], y1[:, None]
    v = P[..., Y0, x0] * (1 - ty) * (1 - tx)
    v = v + P[..., Y0, x1] * (1 - ty) * tx
    v = v + P[..., Y1, x0] * ty * (1 - tx)
    v = v + P[..., Y1, x1] * ty * tx
    v[..., oy, :] = 0
    v[..., :, ox] = 0
    return v.astype(np.float32), lab


def test_grid_kernel_rule_is_bit_exact_with_scipy_zoom():
    rng = np.random.default_rng(0)
    shapes = [(360, 480, 8), (36, 44, 8), (512, 1024, 8), (97, 131, 4), (64, 64, 8)]
    for _ in range(120):
        f = int(rng.choice([1, 2, 3, 4, 8, 16]))
        shapes.append((int(rng.integers(f, 600)), int(rng.integers(f, 600)), f))
    for H, W, f in shapes:
        prob = rng.random((1, 2, H, W), dtype=np.float32)
        target = rng.integers(0, 19, (1, H, W))
        zp = nd.zoom(prob, (1.0, 1.0, 1.0 / f, 1.0 / f), order=1)
        zt = nd.zoom(target, (1.0, 1.0 / f, 1.0 / f), order=0)
        v, lab = _kernel_rule(prob, target, *zp.shape[-2:])
        assert np.array_equal(v, zp) and np.array_equal(lab, zt), (H, W, f)


def test_criteria_import_and_have_no_cpu_path():
    from structure_knowledge_distillation_b200.utils.criterion import CriterionOhemDSN, OhemCrossEntropy2d
    g = torch.Generator().manual_seed(0)
    labels = torch.randint(0, 19, (1, 16, 16), generator=g)
    with pytest.raises(RuntimeError, match="no CPU path"):
        CriterionOhemDSN()([torch.randn(1, 19, 3, 3), torch.randn(1, 19, 3, 3)], labels)
    with pytest.raises(RuntimeError, match="no CPU path"):
        OhemCrossEntropy2d(factor=4)(torch.randn(1, 19, 16, 16), labels)
    with pytest.raises(AssertionError):
        OhemCrossEntropy2d()(torch.randn(1, 19, 16, 16), labels.float().requires_grad_(True))
    c = CriterionOhemDSN(ignore_index=250, thresh=0.6, min_kept=5000)
    assert (c.ignore_index, c.criterion1.thresh, c.criterion1.min_kept, c.criterion1.factor) == (250, 0.6, 5000, 8)


def test_header_declares_the_ohem_entries():
    from structure_knowledge_distillation_b200 import _cabi
    sig = _cabi.parse_header()
    new = ("skd_ohem_grid_sample", "skd_ohem_threshold_workspace_ints", "skd_ohem_threshold", "skd_ohem_dsn_ce_fwd_train",
           "skd_ohem_dsn_ce_bwd_cols")
    assert all(n in sig for n in new)
    assert len(sig["skd_ohem_dsn_ce_fwd_train"][1]) == 24 and len(sig["skd_ohem_grid_sample"][1]) == 18
    if os.path.exists(_cabi.LIB_PATH):                      # built: the library exports every declared symbol
        import ctypes
        dll = ctypes.CDLL(_cabi.LIB_PATH)
        assert all(hasattr(dll, n) for n in new)


def test_netmodel_ohem_options_default_off():
    from structure_knowledge_distillation_b200.utils.train_options import DEFAULTS, make_args
    assert DEFAULTS["ohem"] is False and DEFAULTS["ohem_thres"] == 0.7 and DEFAULTS["ohem_keep"] == 100000
    a = make_args(ohem=True, ohem_keep=5000)
    assert a.ohem and a.ohem_keep == 5000 and a.ohem_thres == 0.7
