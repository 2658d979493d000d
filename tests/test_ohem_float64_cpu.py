"""CPU: the float64 torch restatement of OhemCrossEntropy2d's threshold grid (tools/ohem_oracle.ohem_grid64), which
tests/test_ohem_float64_gpu.py runs on the GPU as its reference, pinned bit for bit against scipy.ndimage.zoom on float64 arrays
and against ohem_grid (scipy on float32, the restatement that the golden fixture of the unmodified reference pins) over the grid
geometries scipy handles specially."""
import numpy as np
import pytest
import scipy.ndimage as nd
import torch

from tools import ohem_oracle as O

# (H, W, factor): the benchmark's 512 x 1024 at 8 and 16, the zero column of 360 x 480, the half-to-even grid size of 36 x 44, a
# one-point axis (H < 1.5 factor), last grid points that round outside the image (109 at 8, 124 at 16, 30 at 4), every grid point
# on a pixel (99 x 131 at factor 2, factor 1), and plain factor-4 / factor-2 grids
GEOMETRIES = [(512, 1024, 8), (512, 1024, 16), (360, 480, 8), (36, 44, 8), (11, 64, 8), (20, 131, 16), (109, 131, 8),
              (124, 190, 16), (30, 55, 4), (99, 131, 2), (37, 45, 1), (97, 131, 4), (97, 131, 2), (1, 131, 1)]


def _last_point_outside(H, factor):
    gh = O.grid_shape(H, H, factor)[0]
    return gh > 1 and (gh - 1) * ((H - 1) / (gh - 1)) > H - 1


def test_geometries_cover_the_special_cases():
    from structure_knowledge_distillation_b200 import ops
    assert all(O.grid_shape(H, W, f) == ops.ohem_grid_shape(H, W, f) for H, W, f in GEOMETRIES)
    assert O.grid_shape(36, 44, 8) == (4, 6) and O.grid_shape(11, 64, 8)[0] == O.grid_shape(20, 131, 16)[0] == 1
    assert [H for H in range(8, 110) if _last_point_outside(H, 8)] == [109]
    assert _last_point_outside(124, 16) and _last_point_outside(30, 4) and _last_point_outside(480, 8)
    assert all((H - 1) / (O.grid_shape(H, W, 2)[0] - 1) == 2.0 for H, W in ((99, 131), (131, 99)))


@pytest.mark.parametrize("H,W,factor", GEOMETRIES)
def test_grid64_is_scipy_zoom_bit_for_bit(H, W, factor):
    rng = np.random.default_rng(H * 1000 + W + factor)
    C = 3
    prob = rng.random((2, C, H, W))
    target = rng.integers(0, C, (2, H, W))
    target[rng.random((2, H, W)) < 0.1] = 255
    pred, lab = O.ohem_grid64(torch.from_numpy(prob), torch.from_numpy(target), *O.grid_shape(H, W, factor))
    zp = nd.zoom(prob, (1.0, 1.0, 1.0 / factor, 1.0 / factor), order=1)
    zt = nd.zoom(target, (1.0, 1.0 / factor, 1.0 / factor), order=0)
    assert zp.dtype == np.float64 and pred.shape == zp.shape[:1] + zp.shape[2:]
    assert np.array_equal(lab.numpy(), zt)
    valid = zt != 255
    ref = np.where(valid, np.take_along_axis(zp, np.where(valid, zt, 0)[:, None], 1)[:, 0], np.inf)
    assert np.array_equal(pred.numpy(), ref)
    if _last_point_outside(H, factor):                        # the last grid row reads 0: probability and label
        assert (pred.numpy()[:, -1] == 0).all() and (zt[:, -1] == 0).all()


@pytest.mark.parametrize("H,W,factor", GEOMETRIES)
def test_grid64_matches_float32_restatement(H, W, factor):
    g = torch.Generator().manual_seed(H * 7 + W + factor)
    C = 19
    prob = torch.softmax(torch.randn(2, C, H, W, generator=g) * 2, 1)
    target = torch.randint(0, C, (2, H, W), generator=g)
    target[torch.rand(2, H, W, generator=g) < 0.05] = 255
    ref_pred, ref_lab = O.ohem_grid(prob.numpy(), target.numpy(), factor)
    pred, lab = O.ohem_grid64(prob.double(), target, *O.grid_shape(H, W, factor))
    assert np.array_equal(pred.float().numpy(), ref_pred) and np.array_equal(lab.numpy(), ref_lab)


def test_grid64_custom_ignore_index():
    """ignore 0: the outside points (label 0 by mode 'constant') drop out too, and 255 is an ordinary label"""
    rng = np.random.default_rng(5)
    prob = rng.random((1, 2, 109, 131))
    target = rng.integers(0, 2, (1, 109, 131))
    pred, lab = O.ohem_grid64(torch.from_numpy(prob), torch.from_numpy(target), *O.grid_shape(109, 131, 8), ignore_label=0)
    ref, ref_lab = O.ohem_grid(prob, target, 8, ignore_label=0)
    assert np.array_equal(pred.float().numpy(), ref) and torch.isinf(pred[:, -1]).all() and (lab[:, -1] == 0).all()
