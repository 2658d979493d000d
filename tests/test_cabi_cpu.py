"""CPU checks of the drop-in boundary: the library loads and exports every symbol include/skd.h declares."""
import ctypes
import os

from structure_knowledge_distillation_b200 import _cabi


def test_header_parses_and_every_symbol_is_exported():
    sigs = _cabi.parse_header()
    assert len(sigs) >= 40
    assert os.path.exists(_cabi.LIB_PATH), "run __graft_entry__.build() first"
    dll = ctypes.CDLL(_cabi.LIB_PATH)
    missing = [n for n in sigs if not hasattr(dll, n)]
    assert not missing, missing


def test_reference_native_abi_names_are_mirrored():
    # libs/src/bn.h:7-19 -> skd_<name> one for one
    sigs = _cabi.parse_header()
    for ref in ("bn_mean_var_cuda", "bn_forward_cuda", "bn_edz_eydz_cuda", "bn_backward_cuda", "leaky_relu_cuda",
                "leaky_relu_backward_cuda", "elu_cuda", "elu_backward_cuda", "elu_inv_cuda"):
        assert "skd_" + ref in sigs
    # same argument list as the reference: (N, C, S, x, mean, var, stream)
    assert len(sigs["skd_bn_mean_var_cuda"][1]) == 7
    assert len(sigs["skd_bn_forward_cuda"][1]) == 12
    assert len(sigs["skd_bn_backward_cuda"][1]) == 15


def test_lib_object_and_version():
    L = _cabi.lib()
    assert L.skd_version() == 90
    assert L.skd_pool_out_size_ceil(256, 3, 2, 1) == 129       # ceil-mode stem max-pool (pspnet_combine.py:130)
    assert L.skd_pool_out_size_ceil(129, 3, 2, 1) == 65
    assert L.skd_abn_num_splits(67080, 512) >= 1
