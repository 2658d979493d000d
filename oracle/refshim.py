"""Import the UNMODIFIED reference Python on CPU from the checkout named by SKD_REFERENCE_ROOT.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py): used to (re)generate the golden fixtures.  Nothing
the tests, smoke() or bench.py run may call it -- they compare against the stored fixtures.

Two import shims are needed (SURVEY.md §8c):
  * `tensorboardX`  -- utils/utils.py:10 imports SummaryWriter, never calls it
                       on the hot path.
  * `libs`          -- libs/bn.py needs torch.utils.ffi (removed in torch 1.0)
                       and a cffi build of libs/src/bn.cu.  Replaced by
                       `oracle.port.ABN`, a torch restatement of bn.cu math.
Everything else (utils/criterion.py, utils/utils.py, networks/pspnet_combine.py,
networks/sagan_models.py, networks/spectral.py) is imported as shipped.
"""
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("SKD_REFERENCE_ROOT", "")


def reference_available():
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "networks"))


_loaded = {}


def load_reference():
    """Returns a namespace with the reference's modules (criterion, utils, pspnet, sagan, spectral)."""
    if _loaded:
        return _loaded["ns"]
    if not reference_available():
        raise RuntimeError("reference tree not present at %s" % REFERENCE_ROOT)
    from . import port

    tb = types.ModuleType("tensorboardX")
    tb.SummaryWriter = object
    sys.modules.setdefault("tensorboardX", tb)

    libs = types.ModuleType("libs")

    def _abn_factory(num_features, devices=None, eps=1e-5, momentum=0.1, affine=True,
                     activation="leaky_relu", slope=0.01):
        return port.ABN(num_features, eps=eps, momentum=momentum, affine=affine,
                        activation=activation, slope=slope)

    libs.InPlaceABN = _abn_factory
    libs.InPlaceABNSync = _abn_factory
    sys.modules["libs"] = libs

    # The reference uses top-level package names `utils` and `networks`.
    saved = {k: sys.modules.get(k) for k in ("utils", "networks")}
    for k in list(sys.modules):
        if k == "utils" or k.startswith("utils.") or k == "networks" or k.startswith("networks."):
            del sys.modules[k]
    sys.path.insert(0, REFERENCE_ROOT)
    try:
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            import utils.utils as r_utils
            import utils.criterion as r_criterion
            import networks.pspnet_combine as r_pspnet
            import networks.sagan_models as r_sagan
            import networks.spectral as r_spectral
    finally:
        sys.path.remove(REFERENCE_ROOT)
        # leave the reference modules reachable only through the namespace
        for k in list(sys.modules):
            if k == "utils" or k.startswith("utils.") or k == "networks" or k.startswith("networks."):
                del sys.modules[k]
        for k, v in saved.items():
            if v is not None:
                sys.modules[k] = v
    ns = types.SimpleNamespace(utils=r_utils, criterion=r_criterion, pspnet=r_pspnet,
                               sagan=r_sagan, spectral=r_spectral)
    _loaded["ns"] = ns
    return ns
