"""Host-side checks of the exact convolution tier (test_conv_exact_gpu.py): the data rule's sum-of-|terms| premise, the rounding and
sentinel helpers, and the launch inventory's shape."""
import json

import pytest
import torch
import torch.nn.functional as F

from test_conv_exact_gpu import (INVENTORY, KNOBS, LIMIT, PLAN_FIELDS, ROWS, SYNTHETIC, TF32_EXACT, amplitude, bits, check_premise,
                                 conv_ref, exact_round, header_params, inventory_keys, knob_subset, operand, same_bits, sentinel, tf32_rn,
                                 validate)


@pytest.mark.parametrize("terms", [1, 20, 576, 4096 * 9, 3 * 64 * 9, 1 << 20, 4 << 20, 12 << 20])
def test_operand_premise(terms):
    """Two operands drawn for a reduction of `terms` products keep the sum of |terms| at or below 2^22, and stay TF32-exact."""
    g = torch.Generator().manual_seed(terms)
    x, w = operand(terms, (terms,), g, "cpu"), operand(terms, (terms,), g, "cpu")
    assert float(x.abs().max()) <= TF32_EXACT and float(w.abs().max()) <= TF32_EXACT
    assert torch.equal(x, torch.round(x))
    s = float((x.double().abs() * w.double().abs()).sum())
    assert s <= LIMIT
    a = amplitude(terms)
    assert a == 0 or terms * a * a <= LIMIT
    if a >= 2:
        assert float(x.abs().max()) >= 2                                 # the whole range is used, not just +-1
    if terms > LIMIT:
        assert float((x == 0).double().mean()) > 0.3                     # sparse +-1 where even a = 1 is too large


def test_premise_is_checked():
    x = torch.full((1, 1, 3, 3), 2048.0, dtype=torch.float64)
    w = torch.full((1, 1, 3, 3), 2048.0, dtype=torch.float64)
    check_premise(conv_ref(x, w / 16, 1, 0, 1, 1, 1))                    # 9 * 2048 * 128 < 2^22
    with pytest.raises(AssertionError):
        check_premise(conv_ref(x, w, 1, 0, 1, 1, 1))


def test_conv_ref_extent():
    """Output extents past the natural size read zero padding at the far end; smaller ones crop."""
    x = torch.arange(1, 26, dtype=torch.float64).view(1, 1, 5, 5)
    w = torch.ones(1, 1, 3, 3, dtype=torch.float64)
    nat = F.conv2d(x, w, padding=1, stride=2)
    assert torch.equal(conv_ref(x, w, 2, 1, 1, 3, 3), nat)
    big = conv_ref(x, w, 2, 1, 1, 4, 4)
    assert torch.equal(big[:, :, :3, :3], nat) and float(big[0, 0, 3, 3]) == 0.0
    assert torch.equal(conv_ref(x, w, 2, 1, 1, 2, 3), nat[:, :, :2])


def test_exact_round():
    assert torch.equal(exact_round(torch.tensor([1.0 + 1e-9, -3.0 - 5e-7, 2.0 ** 22])), torch.tensor([1.0, -3.0, 2.0 ** 22]))
    with pytest.raises(AssertionError):
        exact_round(torch.tensor([0.5], dtype=torch.float64))


def test_tf32_rn_bits():
    v = torch.tensor([2049.0, 2051.0, 2052.0, 4097.0, 4098.0, 4099.0, -4099.0, 6145.0, 1.0], dtype=torch.float32)
    # 11 significant bits: spacing 2 in [2048, 4096), 4 in [4096, 8192); ties to even
    want = torch.tensor([2048.0, 2052.0, 2052.0, 4096.0, 4096.0, 4100.0, -4100.0, 6144.0, 1.0])
    assert torch.equal(tf32_rn(v), want)
    ints = torch.arange(-TF32_EXACT, TF32_EXACT + 1, dtype=torch.float32)
    assert torch.equal(tf32_rn(ints), ints)                              # every operand value the data rule allows is exact


def test_sentinel_and_bits():
    s = sentinel((4, 3), "cpu")
    assert torch.isnan(s).all()
    assert same_bits(s, s.clone()) and not torch.equal(s, s)              # NaN-safe bit comparison
    a = torch.tensor([0.0]); b = torch.tensor([-0.0])
    assert torch.equal(a, b) and not same_bits(a, b)
    assert bits(torch.tensor([1.0])).item() == 0x3F800000


def test_inventory_well_formed():
    hp = header_params()
    seen = set()
    for e in ROWS:
        assert e["fn"] in hp, e["fn"]
        assert not validate(e), (validate(e), e)
        k = json.dumps({k: v for k, v in e.items() if k != "steps"}, sort_keys=True)
        assert k not in seen, "duplicate row %s" % k
        seen.add(k)
    for e in INVENTORY:
        assert not e.get("synthetic")
        assert set(e["steps"]) <= {"c2", "c4", "espc", "esp", "mnv2", "seg"}
    assert all(e.get("synthetic") and e["steps"] == ("synthetic",) for e in SYNTHETIC)


def test_inventory_covers_every_path():
    """Together the rows must run: 256-row tiles with one and with several N tiles, 128-row tiles with BLOCK_N 32 / 64 / 128, rect
    tiles, split-K, the TMA epilogue, channel chunks outermost, the split-K weight gradient, and every entry point."""
    got = set()
    for e in INVENTORY:
        p = e["plan"]
        if e["fn"] == "skd_conv2d_wgrad_sm100":
            if p[2] > 1:
                got.add("wgrad_splitk")
            got.add("wgrad_bn%d" % p[0])
            continue
        if p is None:
            continue
        d = dict(zip(PLAN_FIELDS, p))
        n_tiles = -(-e["Cout"] // d["bn"])
        if d["rows"] == 256:
            got.add("256_multiN" if n_tiles > 1 else "256_oneN")
        else:
            got.add("128_bn%d" % d["bn"])
        if d["mode"] == 2:
            got.add("rect")
        if d["splits"] > 1:
            got.add("splitk")
        if d["tma_epi"]:
            got.add("tma_epi")
        if d["kc_outer"]:
            got.add("kc_outer")
    need = {"256_multiN", "256_oneN", "128_bn32", "128_bn64", "128_bn128", "rect", "splitk", "tma_epi", "kc_outer", "wgrad_splitk"}
    assert need <= got, need - got
    fns = {e["fn"] for e in ROWS}
    assert fns == set(hp for hp in header_params() if hp in fns) and len(fns) == 12, sorted(fns)
    chain_or_resid = [e for e in INVENTORY if e["fn"] == "skd_conv2d_fwd_sm100" and e.get("residual") and e["caller"] == "dgrad"]
    assert chain_or_resid, "no stride-1 data gradient with a residual"


def test_knob_subset_covers_each_path():
    sub = knob_subset(ROWS)
    classes = {(e["fn"], tuple(e["plan"] or ())) for e in ROWS}
    assert {(e["fn"], tuple(e["plan"] or ())) for e in sub} == classes
    assert len(KNOBS) == 8


def test_inventory_keys_cover_the_logged_forms():
    keys = inventory_keys(INVENTORY)
    kinds = {k[0] for k in keys}
    assert {"fwd", "dgrad", "fwd3x", "split3x", "wgrad", "disc_fwd", "disc_wgrad", "convT_fwd"} <= kinds, kinds
