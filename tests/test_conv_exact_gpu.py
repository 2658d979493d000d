"""Every convolution launch of the training steps, bit for bit against float64 on exact integer data.

Operands are small integers, chosen per launch so that the largest sum of |terms| of any output element stays at or below 2^22 (the
test computes that sum in float64 and asserts it).  Then every product and every fp32 sum is exact in any order, the TF32 operands
are exact (|v| <= 2^11), and split-K partial planes add exactly: every correct tiling, pipeline order and split gives the same
float32 bits, which are the float64 result.  An indexing, halo, pipeline-stage, tile-edge or reduction error shows at the element
where it happens.  Operand rounding is deliberately not tested here (test_pool_layout_float64_gpu.py and the rel-L2 tests do).

INVENTORY lists every distinct convolution launch of one eager step of the benchmark (configurations 2 and 4), the ESPNet-C, ESPNet
and MobileNetV2 distillation steps and the ResNet101 SegModel step, as C entry point + geometry + the plan the host-side dispatch
must choose (skd_conv_fwd_last_plan / skd_conv_wgrad_last_plan).  test_inventory_is_complete fails when a step launches a convolution
the table does not list."""
import ctypes
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

LIMIT = 1 << 22                 # largest sum of |terms| of one output element
TF32_EXACT = 1 << 11            # integers up to this magnitude are exact TF32 values
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "skd.h")

FWD_FNS = ("skd_conv2d_fwd_sm100", "skd_conv2d_fwd_sm100_3xtf32", "skd_conv2d_fwd_sm100_ex", "skd_conv2d_fwd_sm100_splitk",
           "skd_conv2d_fwd_sm100_strided", "skd_conv2d_fwd_sm100_strided_3xtf32")
ALL_FNS = FWD_FNS + ("skd_gemm_nt_sm100", "skd_conv1x1_chain_sm100", "skd_conv2d_wgrad_sm100", "skd_conv2d_fwd_direct",
                     "skd_conv2d_dgrad_direct", "skd_conv2d_wgrad_direct")
PLAN_FIELDS = ("mode", "rows", "bn", "splits", "tma_epi", "kc_outer", "reverse")          # skd_conv_fwd_last_plan
WGRAD_PLAN_FIELDS = ("bn", "linear", "splits")                                            # skd_conv_wgrad_last_plan
ACTS = {0: "none", 1: "leaky_relu", 2: "elu", 3: "relu"}


# ------------------------------------------------------------------------------------------------ helpers (also checked on the CPU)
def header_params(path=HEADER):
    """-> {function: [parameter names]} of include/skd.h (pointer parameters without their '*')."""
    text = re.sub(r"/\*.*?\*/", "", open(path).read(), flags=re.S)
    out = {}
    for name, args in re.findall(r"(skd_\w+)\s*\(([^;{]*)\)\s*;", text, flags=re.S):
        args = " ".join(args.split())
        out[name] = [] if args in ("", "void") else [a.strip().split()[-1].lstrip("*") if len(a.split()) > 1 else a.strip()
                                                     for a in args.split(",")]
    return out


def amplitude(terms, limit=LIMIT):
    """Largest a with terms * a^2 <= limit, capped to the TF32-exact range; 0 when even a = 1 is too large (use sparse_ints)."""
    return min(math.isqrt(limit // max(terms, 1)), TF32_EXACT // 2)


def ints(shape, a, gen, device, density=1.0):
    """Uniform integers in [-a, a] (zeros included) as float32; density < 1 keeps each entry with that probability (else 0)."""
    t = torch.randint(-a, a + 1, shape, generator=gen, device=device).to(torch.float32)
    if density < 1.0:
        t = t * (torch.rand(shape, generator=gen, device=device) < density)
    return t


def operand(terms, shape, gen, device):
    """Integer operand for a reduction of `terms` products of two such operands: dense in [-a, a], or sparse +-1 where a would be 0."""
    a = amplitude(terms)
    if a >= 1:
        return ints(shape, a, gen, device)
    return ints(shape, 1, gen, device, density=math.sqrt(LIMIT / terms) * 1.2)


def exact_round(ref, tol=1e-6):
    """float64 result of an integer computation -> the integer (float64); asserts it is within tol of one."""
    r = torch.round(ref)
    err = float((ref - r).abs().max()) if ref.numel() else 0.0
    assert err <= tol, "float64 reference is not integral (max distance %g)" % err
    return r


def check_premise(abs_sum, limit=LIMIT):
    """abs_sum: float64 sum of |terms| per output element (the same reduction of |operands|)."""
    m = float(abs_sum.max()) if abs_sum.numel() else 0.0
    assert m <= limit, "sum of |terms| %g exceeds %g: fp32 accumulation would not be exact" % (m, limit)
    return m


def sentinel(shape, device):
    return torch.full(shape, float("nan"), device=device, dtype=torch.float32)


def bits(t):
    return t.contiguous().view(torch.int32)


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


def tf32_rn(t):
    """cvt.rn.tf32.f32 restated: round the 13 low mantissa bits away, to nearest, ties to even (finite values)."""
    b = t.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    b = ((b + 0xFFF + ((b >> 13) & 1)) & ~0x1FFF) & 0xFFFFFFFF
    return torch.where(b >= 1 << 31, b - (1 << 32), b).to(torch.int32).view(torch.float32)


def epilogue_ref(raw, scale, shift, residual, act, slope, round_out):
    """The unfused float32 sequence on the exact accumulators raw (float32, channels last): v * scale + shift + residual, act."""
    v = raw.clone()
    if scale is not None:
        v = v * scale
    if shift is not None:
        v = v + shift
    if residual is not None:
        v = v + residual
    if act == 3:
        v = torch.relu(v)
    elif act == 1:
        v = torch.where(v < 0, v * torch.tensor(slope, dtype=torch.float32, device=v.device), v)
    elif act == 2:
        v = torch.where(v < 0, torch.expm1(v), v)
    if round_out:
        v = tf32_rn(v)
    return v


def assert_epilogue(got, want, act, what):
    """bit-exact, except ELU's negative branch: within 1 ulp of float32 expm1."""
    if act == 2:
        neg = want < 0
        d = (bits(got).to(torch.int64) - bits(want).to(torch.int64)).abs()
        assert int(d[~neg].max()) == 0 if (~neg).any() else True, what
        assert int(d[neg].max()) <= 1 if neg.any() else True, (what, int(d.max()))
        return
    if not same_bits(got, want):
        bad = (bits(got) != bits(want)).nonzero()
        raise AssertionError("%s: %d elements differ, first at %s: got %r want %r" % (
            what, bad.shape[0], bad[0].tolist(), float(got[tuple(bad[0])]), float(want[tuple(bad[0])])))


def out_extent(H, W, KH, KW, stride, pad, dil, out_h=0, out_w=0):
    OH = out_h if out_h > 0 else (H + 2 * pad - dil * (KH - 1) - 1) // stride + 1
    OW = out_w if out_w > 0 else (W + 2 * pad - dil * (KW - 1) - 1) // stride + 1
    return OH, OW


def conv_ref(x, w, stride, pad, dil, OH, OW):
    """float64 conv of NCHW x with OIHW w, output cropped / far-end zero padded to OH x OW."""
    KH, KW = w.shape[2], w.shape[3]
    eh = max(0, (OH - 1) * stride + dil * (KH - 1) + 1 - (x.shape[2] + 2 * pad))
    ew = max(0, (OW - 1) * stride + dil * (KW - 1) + 1 - (x.shape[3] + 2 * pad))
    xp = F.pad(x, (pad, pad + ew, pad, pad + eh))
    return F.conv2d(xp, w, stride=stride, dilation=dil)[:, :, :OH, :OW]


def L(fn, steps, plan=None, **geom):
    """One inventory row: C entry point, the steps that launch it, the plan it must take and its arguments by header name (pointer
    arguments as True / False: given or NULL)."""
    return dict(fn=fn, steps=tuple(steps.split()), plan=plan, **geom)


def log_key(e):
    """The CONV_EVENT_LOG key (ops.py / sagan_engine.py) an inventory row's launch is logged under, or None (not logged)."""
    fn, c = e["fn"], e.get("caller", "")
    if fn == "skd_conv2d_fwd_sm100" and c == "dgrad":
        return ("dgrad", e["N"], e["Cin"], e["H"], e["W"], e["Cout"], e["KH"], 1, e["dil"])
    if fn == "skd_conv2d_fwd_sm100":
        return ("fwd", e["N"], e["Cin"], e["H"], e["W"], e["Cout"], e["KH"], e["stride"], e["dil"])
    if fn == "skd_conv2d_fwd_sm100_3xtf32":
        return ("fwd3x", e["N"], e["Cin"], e["H"], e["W"], e["Cout"], e["KH"], e["stride"], e["dil"])
    if fn in ("skd_conv2d_fwd_sm100_ex", "skd_conv2d_fwd_sm100_splitk"):
        return ("disc_fwd", e["N"], e["Cin"], e["H"], e["W"], e["Cout"], e["KH"], e["stride"], e["dil"])
    if fn == "skd_conv2d_wgrad_sm100":
        return ("disc_wgrad" if c == "disc" else "wgrad", e["N"], e["Cin"], e["H"], e["W"], e["Cout"], e["KH"], e["stride"], e["dil"])
    if fn == "skd_conv1x1_chain_sm100":
        return None                     # logged with its image shape rather than P: see chain_matches
    return None


def chain_matches(e, key):
    """A conv1x1_chain log key ("fwd", n, cin3, h, w, cout3, "chain1x1-><cout1>") against a chain inventory row."""
    return (key[0] == "fwd" and isinstance(key[-1], str) and key[-1] == "chain1x1->%d" % e["Cout1"] and key[1] * key[3] * key[4] == e["P"] and
            key[2] == e["Cin3"] and key[5] == e["Cout3"])


def inventory_keys(inv):
    keys = set()
    for e in inv:
        k = log_key(e)
        if k is not None:
            keys.add(k)
        if e["fn"] == "skd_conv2d_fwd_sm100_3xtf32":
            keys.add(("split3x",) + k[1:])               # its lo-part split, logged under the same geometry
        if e["fn"] == "skd_conv2d_fwd_sm100_strided_3xtf32" and e["caller"] == "convT":
            keys.add(("convT_fwd", e["N"], e["Cin"], e["H"], e["W"], e["Cout"] // 2, 2, 2, 1))
    return keys


def validate(e):
    """-> list of problems with one inventory row's geometry for its entry point (empty when well formed)."""
    fn, bad = e["fn"], []
    names = header_params()[fn]
    for k in e:
        if k not in ("fn", "steps", "plan", "caller", "alias", "synthetic") and k not in names:
            bad.append("unknown argument %s" % k)
    if fn in FWD_FNS or fn in ("skd_conv2d_wgrad_sm100", "skd_conv2d_fwd_direct", "skd_conv2d_dgrad_direct", "skd_conv2d_wgrad_direct"):
        OH, OW = out_extent(e["H"], e["W"], e["KH"], e["KW"], e["stride"], e["pad"], e["dil"], e.get("out_h", 0), e.get("out_w", 0))
        if OH <= 0 or OW <= 0:
            bad.append("empty output")
    if fn in FWD_FNS:
        ldx = e["ldx"]
        if e["Cin"] % 4 or ldx % 4 or ldx < e["Cin"]:
            bad.append("Cin / ldx must be whole float4s, ldx >= Cin")
        if "ldy" in e and e["ldy"] < e["Cout"]:
            bad.append("ldy < Cout")
        if e.get("residual") and e["ldr"] < e["Cout"]:
            bad.append("ldr < Cout")
        if not e.get("synthetic") and (e["plan"] is None or len(e["plan"]) != len(PLAN_FIELDS)):
            bad.append("plan")
    if fn == "skd_conv2d_wgrad_sm100":
        if e["Cin"] % 4 or e["Cout"] % 4 or e["ldx"] % 4 or e["ldy"] % 4 or e["ldx"] < e["Cin"] or e["ldy"] < e["Cout"]:
            bad.append("wgrad channel counts / pitches")
        if e["plan"] is None or len(e["plan"]) != len(WGRAD_PLAN_FIELDS):
            bad.append("plan")
    if fn == "skd_conv1x1_chain_sm100":
        if e["Cout3"] % 64 or e["Cout1"] not in (64, 128, 256) or e["Cin3"] % 4:
            bad.append("chain shape")
    if fn == "skd_gemm_nt_sm100" and (e["lda"] < e["K"] or (e.get("D") and e["ldd"] < e["Ncols"])):
        bad.append("gemm pitches")
    if fn in ("skd_conv2d_fwd_direct", "skd_conv2d_dgrad_direct", "skd_conv2d_wgrad_direct") and e["Cin"] % 4 == 0 and e["Cout"] % 4 == 0:
        bad.append("direct SIMT rows are for channel counts that are not multiples of 4")
    if not e["steps"]:
        bad.append("no step")
    return bad
INVENTORY = [
    L('skd_conv1x1_chain_sm100', 'c4 espc esp', None, caller='fwd', Cin3=64, Cout1=64, Cout3=256, P=176176, ldr=256, ldx3=64, ldy1=64, ldy3=256, residual=True, scale1=True, scale3=True, shift1=True, shift3=True, w1=True, w3=True, x3=True, y1=True, y3=True),
    L('skd_conv1x1_chain_sm100', 'c4 espc esp', None, caller='fwd', Cin3=128, Cout1=128, Cout3=512, P=44896, ldr=512, ldx3=128, ldy1=128, ldy3=512, residual=True, scale1=True, scale3=True, shift1=True, shift3=True, w1=True, w3=True, x3=True, y1=True, y3=True),
    L('skd_conv1x1_chain_sm100', 'c2 mnv2', None, caller='fwd', Cin3=64, Cout1=64, Cout3=256, P=265224, ldr=256, ldx3=64, ldy1=64, ldy3=256, residual=True, scale1=True, scale3=True, shift1=True, shift3=True, w1=True, w3=True, x3=True, y1=True, y3=True),
    L('skd_conv1x1_chain_sm100', 'c2 mnv2', None, caller='fwd', Cin3=128, Cout1=128, Cout3=512, P=67080, ldr=512, ldx3=128, ldy1=128, ldy3=512, residual=True, scale1=True, scale3=True, shift1=True, shift3=True, w1=True, w3=True, x3=True, y1=True, y3=True),
    L('skd_conv1x1_chain_sm100', 'c4 espc esp', None, caller='fwd', Cin3=256, Cout1=256, Cout3=1024, P=44896, ldr=1024, ldx3=256, ldy1=256, ldy3=1024, residual=True, scale1=True, scale3=True, shift1=True, shift3=True, w1=True, w3=True, x3=True, y1=True, y3=True),
    L('skd_conv1x1_chain_sm100', 'c2 mnv2', None, caller='fwd', Cin3=256, Cout1=256, Cout3=1024, P=67080, ldr=1024, ldx3=256, ldy1=256, ldy3=1024, residual=True, scale1=True, scale3=True, shift1=True, shift3=True, w1=True, w3=True, x3=True, y1=True, y3=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=320, H=1, KH=1, KW=1, N=8, W=1, act=0, dil=1, ldr=0, ldx=128, ldy=320, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=512, H=1, KH=1, KW=1, N=8, W=1, act=0, dil=1, ldr=0, ldx=128, ldy=512, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=512, H=1, KH=1, KW=1, N=16, W=1, act=0, dil=1, ldr=0, ldx=128, ldy=512, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=320, H=2, KH=1, KW=1, N=8, W=2, act=0, dil=1, ldr=0, ldx=128, ldy=320, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=512, H=2, KH=1, KW=1, N=8, W=2, act=0, dil=1, ldr=0, ldx=128, ldy=512, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=320, H=3, KH=1, KW=1, N=8, W=3, act=0, dil=1, ldr=0, ldx=128, ldy=320, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=512, H=2, KH=1, KW=1, N=16, W=2, act=0, dil=1, ldr=0, ldx=128, ldy=512, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=512, H=3, KH=1, KW=1, N=8, W=3, act=0, dil=1, ldr=0, ldx=128, ldy=512, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=512, Cout=2048, H=1, KH=1, KW=1, N=8, W=1, act=0, dil=1, ldr=0, ldx=512, ldy=2048, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=512, H=3, KH=1, KW=1, N=16, W=3, act=0, dil=1, ldr=0, ldx=128, ldy=512, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=320, H=6, KH=1, KW=1, N=8, W=6, act=0, dil=1, ldr=0, ldx=128, ldy=320, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=512, H=6, KH=1, KW=1, N=8, W=6, act=0, dil=1, ldr=0, ldx=128, ldy=512, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'esp', [1, 128, 32, 1, 1, 0, 0], caller='dgrad', Cin=4, Cout=4, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=2, ldr=4, ldx=4, ldy=4, pad=2, residual=True, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'esp', [1, 128, 32, 1, 1, 0, 0], caller='dgrad', Cin=4, Cout=4, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=4, ldr=4, ldx=4, ldy=4, pad=4, residual=True, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'esp', [1, 128, 32, 1, 1, 0, 0], caller='dgrad', Cin=4, Cout=4, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=8, ldr=4, ldx=4, ldy=4, pad=8, residual=True, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'esp', [1, 128, 32, 1, 1, 0, 0], caller='dgrad', Cin=4, Cout=4, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=16, ldr=4, ldx=4, ldy=4, pad=16, residual=True, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'esp', [0, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=4, Cout=40, H=90, KH=1, KW=1, N=16, W=120, act=0, dil=1, ldr=0, ldx=4, ldy=40, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=512, Cout=2048, H=2, KH=1, KW=1, N=8, W=2, act=0, dil=1, ldr=0, ldx=512, ldy=2048, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=512, H=6, KH=1, KW=1, N=16, W=6, act=0, dil=1, ldr=0, ldx=128, ldy=512, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'esp', [1, 128, 32, 1, 0, 0, 0], caller='dgrad', Cin=8, Cout=4, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=1, ldr=0, ldx=8, ldy=4, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=512, Cout=2048, H=3, KH=1, KW=1, N=8, W=3, act=0, dil=1, ldr=0, ldx=512, ldy=2048, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=20, Cout=128, H=46, KH=1, KW=1, N=16, W=61, act=0, dil=1, ldr=0, ldx=20, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'espc esp', [0, 128, 64, 1, 1, 0, 0], caller='dgrad', Cin=12, Cout=64, H=90, KH=1, KW=1, N=16, W=120, act=0, dil=1, ldr=64, ldx=12, ldy=64, pad=0, residual=True, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'espc esp', [0, 128, 128, 1, 1, 0, 0], caller='dgrad', Cin=28, Cout=128, H=45, KH=1, KW=1, N=16, W=60, act=0, dil=1, ldr=128, ldx=28, ldy=128, pad=0, residual=True, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=20, Cout=128, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldr=0, ldx=20, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=20, Cout=128, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=20, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'espc esp', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=20, Cout=256, H=45, KH=1, KW=1, N=16, W=60, act=0, dil=1, ldr=0, ldx=20, ldy=256, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'espc esp', [1, 128, 32, 1, 1, 0, 0], caller='dgrad', Cin=12, Cout=12, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=2, ldr=12, ldx=12, ldy=12, pad=2, residual=True, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'espc esp', [1, 128, 32, 1, 1, 0, 0], caller='dgrad', Cin=12, Cout=12, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=4, ldr=12, ldx=12, ldy=12, pad=4, residual=True, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'espc esp', [1, 128, 32, 1, 1, 0, 0], caller='dgrad', Cin=12, Cout=12, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=8, ldr=12, ldx=12, ldy=12, pad=8, residual=True, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'espc esp', [1, 128, 32, 1, 1, 0, 0], caller='dgrad', Cin=12, Cout=12, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=16, ldr=12, ldx=12, ldy=12, pad=16, residual=True, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'espc esp', [1, 128, 32, 1, 0, 0, 0], caller='dgrad', Cin=16, Cout=12, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=1, ldr=0, ldx=16, ldy=12, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=32, Cout=144, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldr=0, ldx=32, ldy=144, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=512, Cout=2048, H=6, KH=1, KW=1, N=8, W=6, act=0, dil=1, ldr=0, ldx=512, ldy=2048, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'espc esp', [1, 128, 32, 1, 0, 0, 0], caller='dgrad', Cin=28, Cout=28, H=45, KH=3, KW=3, N=16, W=60, act=0, dil=1, ldr=0, ldx=28, ldy=28, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'espc esp', [1, 128, 32, 1, 1, 0, 0], caller='dgrad', Cin=28, Cout=28, H=45, KH=3, KW=3, N=16, W=60, act=0, dil=2, ldr=28, ldx=28, ldy=28, pad=2, residual=True, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'espc esp', [1, 128, 32, 1, 1, 0, 0], caller='dgrad', Cin=28, Cout=28, H=45, KH=3, KW=3, N=16, W=60, act=0, dil=4, ldr=28, ldx=28, ldy=28, pad=4, residual=True, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'espc esp', [1, 128, 32, 1, 1, 0, 0], caller='dgrad', Cin=28, Cout=28, H=45, KH=3, KW=3, N=16, W=60, act=0, dil=8, ldr=28, ldx=28, ldy=28, pad=8, residual=True, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'espc esp', [1, 128, 32, 1, 1, 0, 0], caller='dgrad', Cin=28, Cout=28, H=45, KH=3, KW=3, N=16, W=60, act=0, dil=16, ldr=28, ldx=28, ldy=28, pad=16, residual=True, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 32, 1, 0, 0, 0], caller='dgrad', Cin=192, Cout=32, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldr=0, ldx=192, ldy=32, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=32, Cout=192, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldr=0, ldx=32, ldy=192, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'esp', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=20, Cout=132, H=90, KH=1, KW=1, N=16, W=120, act=0, dil=1, ldr=0, ldx=20, ldy=132, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 32, 1, 0, 0, 0], caller='dgrad', Cin=16, Cout=32, H=256, KH=1, KW=1, N=8, W=512, act=0, dil=1, ldr=0, ldx=16, ldy=32, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=24, Cout=96, H=128, KH=1, KW=1, N=8, W=256, act=0, dil=1, ldr=0, ldx=24, ldy=96, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=20, Cout=512, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=20, ldy=512, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=64, Cout=192, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldr=0, ldx=64, ldy=192, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 32, 1, 0, 0, 0], caller='dgrad', Cin=144, Cout=24, H=128, KH=1, KW=1, N=8, W=256, act=0, dil=1, ldr=0, ldx=144, ldy=24, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=24, Cout=144, H=128, KH=1, KW=1, N=8, W=256, act=0, dil=1, ldr=0, ldx=24, ldy=144, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=64, Cout=128, H=91, KH=1, KW=1, N=16, W=121, act=0, dil=1, ldr=0, ldx=64, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=256, Cout=128, H=46, KH=1, KW=1, N=16, W=61, act=0, dil=1, ldr=0, ldx=256, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=384, Cout=64, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldr=0, ldx=384, ldy=64, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=64, Cout=384, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldr=0, ldx=64, ldy=384, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 32, 1, 0, 0, 0], caller='dgrad', Cin=96, Cout=16, H=256, KH=1, KW=1, N=8, W=512, act=0, dil=1, ldr=0, ldx=96, ldy=16, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 seg', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=64, Cout=128, H=129, KH=1, KW=1, N=8, W=257, act=0, dil=1, ldr=0, ldx=64, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=256, Cout=128, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=256, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=96, Cout=384, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldr=0, ldx=96, ldy=384, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=576, Cout=96, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldr=0, ldx=576, ldy=96, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=96, Cout=576, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldr=0, ldx=96, ldy=576, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=256, Cout=64, H=129, KH=1, KW=1, N=8, W=257, act=0, dil=1, ldr=0, ldx=256, ldy=64, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=64, Cout=256, H=129, KH=1, KW=1, N=8, W=257, act=0, dil=1, ldr=0, ldx=64, ldy=256, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=512, Cout=128, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=512, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=512, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=128, ldy=512, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'esp', [1, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=20, Cout=40, H=180, KH=3, KW=3, N=16, W=240, act=0, dil=1, ldr=0, ldx=20, ldy=40, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=512, Cout=256, H=46, KH=1, KW=1, N=16, W=61, act=0, dil=1, ldr=0, ldx=512, ldy=256, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=160, Cout=576, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldr=0, ldx=160, ldy=576, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=64, Cout=64, H=91, KH=3, KW=3, N=16, W=121, act=0, dil=1, ldr=0, ldx=64, ldy=64, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=128, H=46, KH=3, KW=3, N=16, W=61, act=0, dil=1, ldr=0, ldx=128, ldy=128, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=96, H=64, KH=3, KW=3, N=8, W=128, act=0, dil=1, ldr=0, ldx=128, ldy=96, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=256, H=129, KH=1, KW=1, N=8, W=257, act=0, dil=1, ldr=0, ldx=128, ldy=256, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=256, Cout=128, H=129, KH=1, KW=1, N=8, W=257, act=0, dil=1, ldr=0, ldx=256, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=512, Cout=256, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=512, ldy=256, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=256, Cout=512, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=256, ldy=512, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 seg', [1, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=64, Cout=64, H=129, KH=3, KW=3, N=8, W=257, act=0, dil=1, ldr=0, ldx=64, ldy=64, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 seg', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=128, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=1, ldr=0, ldx=128, ldy=128, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=960, Cout=160, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldr=0, ldx=960, ldy=160, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=160, Cout=960, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldr=0, ldx=160, ldy=960, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=64, Cout=128, H=91, KH=3, KW=3, N=16, W=121, act=0, dil=1, ldr=0, ldx=64, ldy=128, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=256, H=46, KH=3, KW=3, N=16, W=61, act=0, dil=1, ldr=0, ldx=128, ldy=256, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=256, Cout=128, H=46, KH=3, KW=3, N=16, W=61, act=0, dil=2, ldr=0, ldx=256, ldy=128, pad=2, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=1024, Cout=256, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=1024, ldy=256, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=256, Cout=1024, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=256, ldy=1024, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=64, Cout=128, H=129, KH=3, KW=3, N=8, W=257, act=0, dil=1, ldr=0, ldx=64, ldy=128, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=256, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=1, ldr=0, ldx=128, ldy=256, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=256, Cout=128, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=2, ldr=0, ldx=256, ldy=128, pad=2, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=320, Cout=960, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldr=0, ldx=320, ldy=960, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=64, Cout=64, H=180, KH=3, KW=3, N=16, W=240, act=0, dil=1, ldr=0, ldx=64, ldy=64, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=256, Cout=256, H=46, KH=3, KW=3, N=16, W=61, act=0, dil=2, ldr=0, ldx=256, ldy=256, pad=2, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=512, Cout=1024, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=512, ldy=1024, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=1024, Cout=512, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=1024, ldy=512, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 seg', [1, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=64, Cout=64, H=256, KH=3, KW=3, N=8, W=512, act=0, dil=1, ldr=0, ldx=64, ldy=64, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 seg', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=256, Cout=256, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=2, ldr=0, ldx=256, ldy=256, pad=2, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=64, H=180, KH=3, KW=3, N=16, W=240, act=0, dil=1, ldr=0, ldx=128, ldy=64, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=1024, H=46, KH=3, KW=3, N=16, W=61, act=0, dil=1, ldr=0, ldx=128, ldy=1024, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=512, Cout=256, H=46, KH=3, KW=3, N=16, W=61, act=0, dil=4, ldr=0, ldx=512, ldy=256, pad=4, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=832, H=64, KH=3, KW=3, N=8, W=128, act=0, dil=1, ldr=0, ldx=128, ldy=832, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=2048, Cout=512, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=2048, ldy=512, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=512, Cout=2048, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=512, ldy=2048, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 seg', [1, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=64, H=256, KH=3, KW=3, N=8, W=512, act=0, dil=1, ldr=0, ldx=128, ldy=64, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=1024, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=1, ldr=0, ldx=128, ldy=1024, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=512, Cout=256, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=4, ldr=0, ldx=512, ldy=256, pad=4, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=512, Cout=512, H=46, KH=3, KW=3, N=16, W=61, act=0, dil=4, ldr=0, ldx=512, ldy=512, pad=4, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [0, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=2048, Cout=1024, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=2048, ldy=1024, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 seg', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=512, Cout=512, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=4, ldr=0, ldx=512, ldy=512, pad=4, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=512, Cout=1024, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=1, ldr=0, ldx=512, ldy=1024, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'seg', [1, 256, 128, 1, 0, 0, 0], caller='dgrad', Cin=512, Cout=4096, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=1, ldr=0, ldx=512, ldy=4096, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=320, Cout=128, H=1, KH=1, KW=1, N=8, W=1, act=0, dil=1, ldr=0, ldx=320, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=128, H=1, KH=1, KW=1, N=8, W=1, act=0, dil=1, ldr=0, ldx=512, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=128, H=1, KH=1, KW=1, N=16, W=1, act=0, dil=1, ldr=0, ldx=512, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=320, Cout=128, H=2, KH=1, KW=1, N=8, W=2, act=0, dil=1, ldr=0, ldx=320, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=128, H=2, KH=1, KW=1, N=8, W=2, act=0, dil=1, ldr=0, ldx=512, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=320, Cout=128, H=3, KH=1, KW=1, N=8, W=3, act=0, dil=1, ldr=0, ldx=320, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=128, H=2, KH=1, KW=1, N=16, W=2, act=0, dil=1, ldr=0, ldx=512, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=128, H=3, KH=1, KW=1, N=8, W=3, act=0, dil=1, ldr=0, ldx=512, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=2048, Cout=512, H=1, KH=1, KW=1, N=8, W=1, act=1, dil=1, ldr=0, ldx=2048, ldy=512, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.01, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=128, H=3, KH=1, KW=1, N=16, W=3, act=0, dil=1, ldr=0, ldx=512, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=320, Cout=128, H=6, KH=1, KW=1, N=8, W=6, act=0, dil=1, ldr=0, ldx=320, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=2048, Cout=512, H=1, KH=1, KW=1, N=16, W=1, act=1, dil=1, ldr=0, ldx=2048, ldy=512, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.01, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=128, H=6, KH=1, KW=1, N=8, W=6, act=0, dil=1, ldr=0, ldx=512, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=2048, Cout=512, H=2, KH=1, KW=1, N=8, W=2, act=1, dil=1, ldr=0, ldx=2048, ldy=512, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.01, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=128, H=6, KH=1, KW=1, N=16, W=6, act=0, dil=1, ldr=0, ldx=512, ldy=128, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=2048, Cout=512, H=2, KH=1, KW=1, N=16, W=2, act=1, dil=1, ldr=0, ldx=2048, ldy=512, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.01, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=2048, Cout=512, H=3, KH=1, KW=1, N=8, W=3, act=1, dil=1, ldr=0, ldx=2048, ldy=512, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.01, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=20, H=46, KH=1, KW=1, N=16, W=61, act=0, dil=1, ldr=0, ldx=128, ldy=20, pad=0, residual=False, round_tf32=0, scale=False, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=2048, Cout=512, H=3, KH=1, KW=1, N=16, W=3, act=1, dil=1, ldr=0, ldx=2048, ldy=512, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.01, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=20, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldr=0, ldx=128, ldy=20, pad=0, residual=False, round_tf32=0, scale=False, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=20, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=128, ldy=20, pad=0, residual=False, round_tf32=0, scale=False, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=20, Cout=20, H=90, KH=2, KW=2, N=16, W=120, act=0, dil=1, ldr=0, ldx=20, ldy=20, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=2, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=2048, Cout=512, H=6, KH=1, KW=1, N=8, W=6, act=1, dil=1, ldr=0, ldx=2048, ldy=512, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.01, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=20, H=46, KH=1, KW=1, N=16, W=61, act=0, dil=1, ldr=0, ldx=512, ldy=20, pad=0, residual=False, round_tf32=0, scale=False, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=2048, Cout=512, H=6, KH=1, KW=1, N=16, W=6, act=1, dil=1, ldr=0, ldx=2048, ldy=512, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.01, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2 seg', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=20, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=512, ldy=20, pad=0, residual=False, round_tf32=0, scale=False, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=20, Cout=20, H=180, KH=2, KW=2, N=16, W=240, act=0, dil=1, ldr=0, ldx=20, ldy=20, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=2, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=32, Cout=64, H=180, KH=1, KW=1, N=16, W=240, act=3, dil=1, ldr=0, ldx=32, ldy=64, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=64, H=91, KH=1, KW=1, N=16, W=121, act=3, dil=1, ldr=0, ldx=128, ldy=64, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [0, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=256, H=46, KH=1, KW=1, N=16, W=61, act=0, dil=1, ldr=0, ldx=128, ldy=256, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=32, Cout=64, H=256, KH=1, KW=1, N=8, W=512, act=3, dil=1, ldr=0, ldx=32, ldy=64, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=64, H=129, KH=1, KW=1, N=8, W=257, act=3, dil=1, ldr=0, ldx=128, ldy=64, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [0, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=256, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=128, ldy=256, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 128, 128, 1, 1, 0, 0], caller='fwd', Cin=64, Cout=256, H=91, KH=1, KW=1, N=16, W=121, act=3, dil=1, ldr=256, ldx=64, ldy=256, pad=0, residual=True, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 128, 128, 1, 1, 0, 0], caller='fwd', Cin=128, Cout=512, H=46, KH=1, KW=1, N=16, W=61, act=3, dil=1, ldr=512, ldx=128, ldy=512, pad=0, residual=True, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 128, 128, 1, 1, 0, 0], caller='fwd', Cin=64, Cout=256, H=129, KH=1, KW=1, N=8, W=257, act=3, dil=1, ldr=256, ldx=64, ldy=256, pad=0, residual=True, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 128, 128, 1, 1, 0, 0], caller='fwd', Cin=128, Cout=512, H=65, KH=1, KW=1, N=8, W=129, act=3, dil=1, ldr=512, ldx=128, ldy=512, pad=0, residual=True, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=20, Cout=20, H=360, KH=2, KW=2, N=16, W=480, act=0, dil=1, ldr=0, ldx=20, ldy=20, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=2, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=256, H=91, KH=1, KW=1, N=16, W=121, act=0, dil=1, ldr=0, ldx=128, ldy=256, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=128, H=91, KH=1, KW=1, N=16, W=121, act=3, dil=1, ldr=0, ldx=256, ldy=128, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=256, H=46, KH=1, KW=1, N=16, W=61, act=3, dil=1, ldr=0, ldx=512, ldy=256, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [0, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=512, H=46, KH=1, KW=1, N=16, W=61, act=0, dil=1, ldr=0, ldx=256, ldy=512, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [1, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=64, H=91, KH=3, KW=3, N=16, W=121, act=3, dil=1, ldr=0, ldx=64, ldy=64, pad=1, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=128, H=46, KH=3, KW=3, N=16, W=61, act=3, dil=1, ldr=0, ldx=128, ldy=128, pad=1, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=96, Cout=128, H=64, KH=3, KW=3, N=8, W=128, act=0, dil=1, ldr=0, ldx=96, ldy=128, pad=1, residual=False, round_tf32=0, scale=False, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=256, H=129, KH=1, KW=1, N=8, W=257, act=0, dil=1, ldr=0, ldx=128, ldy=256, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=128, H=129, KH=1, KW=1, N=8, W=257, act=3, dil=1, ldr=0, ldx=256, ldy=128, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=256, H=65, KH=1, KW=1, N=8, W=129, act=3, dil=1, ldr=0, ldx=512, ldy=256, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [0, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=512, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=256, ldy=512, pad=0, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [1, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=64, H=129, KH=3, KW=3, N=8, W=257, act=3, dil=1, ldr=0, ldx=64, ldy=64, pad=1, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=128, H=65, KH=3, KW=3, N=8, W=129, act=3, dil=1, ldr=0, ldx=128, ldy=128, pad=1, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 128, 128, 1, 1, 0, 0], caller='fwd', Cin=256, Cout=1024, H=46, KH=1, KW=1, N=16, W=61, act=3, dil=1, ldr=1024, ldx=256, ldy=1024, pad=0, residual=True, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=256, H=46, KH=3, KW=3, N=16, W=61, act=0, dil=2, ldr=0, ldx=128, ldy=256, pad=2, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=128, H=46, KH=3, KW=3, N=16, W=61, act=0, dil=1, ldr=0, ldx=256, ldy=128, pad=1, residual=False, round_tf32=0, scale=False, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 128, 128, 1, 1, 0, 0], caller='fwd', Cin=256, Cout=1024, H=65, KH=1, KW=1, N=8, W=129, act=3, dil=1, ldr=1024, ldx=256, ldy=1024, pad=0, residual=True, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=256, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=2, ldr=0, ldx=128, ldy=256, pad=2, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=128, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=1, ldr=0, ldx=256, ldy=128, pad=1, residual=False, round_tf32=0, scale=False, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=512, H=91, KH=1, KW=1, N=16, W=121, act=0, dil=1, ldr=0, ldx=256, ldy=512, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=2, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=1024, H=46, KH=1, KW=1, N=16, W=61, act=0, dil=1, ldr=0, ldx=512, ldy=1024, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=1024, Cout=512, H=46, KH=1, KW=1, N=16, W=61, act=3, dil=1, ldr=0, ldx=1024, ldy=512, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [1, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=64, H=180, KH=3, KW=3, N=16, W=240, act=3, dil=1, ldr=0, ldx=64, ldy=64, pad=1, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=128, H=91, KH=3, KW=3, N=16, W=121, act=3, dil=1, ldr=0, ldx=128, ldy=128, pad=1, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=2, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=256, H=46, KH=3, KW=3, N=16, W=61, act=3, dil=2, ldr=0, ldx=256, ldy=256, pad=2, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=256, H=46, KH=3, KW=3, N=16, W=61, act=0, dil=2, ldr=0, ldx=256, ldy=256, pad=2, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=512, H=129, KH=1, KW=1, N=8, W=257, act=0, dil=1, ldr=0, ldx=256, ldy=512, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=2, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=1024, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=512, ldy=1024, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=1024, Cout=512, H=65, KH=1, KW=1, N=8, W=129, act=3, dil=1, ldr=0, ldx=1024, ldy=512, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [1, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=64, H=256, KH=3, KW=3, N=8, W=512, act=3, dil=1, ldr=0, ldx=64, ldy=64, pad=1, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=128, H=129, KH=3, KW=3, N=8, W=257, act=3, dil=1, ldr=0, ldx=128, ldy=128, pad=1, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=2, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=256, H=65, KH=3, KW=3, N=8, W=129, act=3, dil=2, ldr=0, ldx=256, ldy=256, pad=2, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=256, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=2, ldr=0, ldx=256, ldy=256, pad=2, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 128, 128, 1, 1, 0, 0], caller='fwd', Cin=512, Cout=2048, H=46, KH=1, KW=1, N=16, W=61, act=3, dil=1, ldr=2048, ldx=512, ldy=2048, pad=0, residual=True, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=2048, Cout=512, H=46, KH=1, KW=1, N=16, W=61, act=3, dil=1, ldr=0, ldx=2048, ldy=512, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 128, 128, 1, 1, 0, 0], caller='fwd', Cin=512, Cout=2048, H=46, KH=1, KW=1, N=16, W=61, act=3, dil=1, ldr=2048, ldx=512, ldy=4096, pad=0, residual=True, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=128, H=180, KH=3, KW=3, N=16, W=240, act=3, dil=1, ldr=0, ldx=64, ldy=128, pad=1, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=512, H=46, KH=3, KW=3, N=16, W=61, act=0, dil=4, ldr=0, ldx=256, ldy=512, pad=4, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=1024, Cout=128, H=46, KH=3, KW=3, N=16, W=61, act=0, dil=1, ldr=0, ldx=1024, ldy=128, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'mnv2', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=832, Cout=128, H=64, KH=3, KW=3, N=8, W=128, act=0, dil=1, ldr=0, ldx=832, ldy=128, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 128, 128, 1, 1, 0, 0], caller='fwd', Cin=512, Cout=2048, H=65, KH=1, KW=1, N=8, W=129, act=3, dil=1, ldr=2048, ldx=512, ldy=2048, pad=0, residual=True, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=2048, Cout=512, H=65, KH=1, KW=1, N=8, W=129, act=3, dil=1, ldr=0, ldx=2048, ldy=512, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 128, 128, 1, 1, 0, 0], caller='fwd', Cin=512, Cout=2048, H=65, KH=1, KW=1, N=8, W=129, act=3, dil=1, ldr=2048, ldx=512, ldy=4096, pad=0, residual=True, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=128, H=256, KH=3, KW=3, N=8, W=512, act=3, dil=1, ldr=0, ldx=64, ldy=128, pad=1, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=512, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=4, ldr=0, ldx=256, ldy=512, pad=4, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=1024, Cout=128, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=1, ldr=0, ldx=1024, ldy=128, pad=1, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [0, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=1024, Cout=2048, H=46, KH=1, KW=1, N=16, W=61, act=0, dil=1, ldr=0, ldx=1024, ldy=2048, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=512, H=46, KH=3, KW=3, N=16, W=61, act=3, dil=4, ldr=0, ldx=512, ldy=512, pad=4, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=512, H=46, KH=3, KW=3, N=16, W=61, act=0, dil=4, ldr=0, ldx=512, ldy=512, pad=4, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [0, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=1024, Cout=2048, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldr=0, ldx=1024, ldy=2048, pad=0, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=512, H=65, KH=3, KW=3, N=8, W=129, act=3, dil=4, ldr=0, ldx=512, ldy=512, pad=4, residual=False, round_tf32=0, scale=True, shift=True, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=512, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=4, ldr=0, ldx=512, ldy=512, pad=4, residual=False, round_tf32=0, scale=False, shift=False, slope=0.0, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=1024, Cout=512, H=46, KH=3, KW=3, N=16, W=61, act=1, dil=1, ldr=0, ldx=1024, ldy=512, pad=1, residual=False, round_tf32=0, scale=True, shift=True, slope=0.01, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [1, 256, 128, 1, 0, 0, 0], caller='fwd', Cin=1024, Cout=512, H=65, KH=3, KW=3, N=8, W=129, act=1, dil=1, ldr=0, ldx=1024, ldy=512, pad=1, residual=False, round_tf32=0, scale=True, shift=True, slope=0.01, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c4 espc esp', [1, 256, 128, 1, 0, 1, 0], caller='fwd', Cin=4096, Cout=512, H=46, KH=3, KW=3, N=16, W=61, act=1, dil=1, ldr=0, ldx=4096, ldy=512, pad=1, residual=False, round_tf32=0, scale=True, shift=True, slope=0.01, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100', 'c2 mnv2', [1, 256, 128, 1, 0, 1, 0], caller='fwd', Cin=4096, Cout=512, H=65, KH=3, KW=3, N=8, W=129, act=1, dil=1, ldr=0, ldx=4096, ldy=512, pad=1, residual=False, round_tf32=0, scale=True, shift=True, slope=0.01, stride=1, w=True, x=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=2048, Cout=512, H=1, KH=1, KW=1, N=8, W=1, act=0, dil=1, ldx=2048, ldy=512, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=4, Cout=4, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=2, ldx=4, ldy=4, pad=2, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=4, Cout=4, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=4, ldx=4, ldy=4, pad=4, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=4, Cout=4, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=8, ldx=4, ldy=4, pad=8, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=4, Cout=4, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=16, ldx=4, ldy=4, pad=16, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'esp', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=40, Cout=4, H=90, KH=1, KW=1, N=16, W=120, act=0, dil=1, ldx=40, ldy=4, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=2048, Cout=512, H=2, KH=1, KW=1, N=8, W=2, act=0, dil=1, ldx=2048, ldy=512, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=4, Cout=8, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=1, ldx=4, ldy=8, pad=1, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=2048, Cout=512, H=3, KH=1, KW=1, N=8, W=3, act=0, dil=1, ldx=2048, ldy=512, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'espc esp', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=12, H=90, KH=1, KW=1, N=16, W=120, act=0, dil=1, ldx=64, ldy=12, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'espc esp', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=28, H=45, KH=1, KW=1, N=16, W=60, act=0, dil=1, ldx=128, ldy=28, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'espc esp', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=20, H=45, KH=1, KW=1, N=16, W=60, act=0, dil=1, ldx=256, ldy=20, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'espc esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=12, Cout=12, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=2, ldx=12, ldy=12, pad=2, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'espc esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=12, Cout=12, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=4, ldx=12, ldy=12, pad=4, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'espc esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=12, Cout=12, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=8, ldx=12, ldy=12, pad=8, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'espc esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=12, Cout=12, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=16, ldx=12, ldy=12, pad=16, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'espc esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=12, Cout=16, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=1, ldx=12, ldy=16, pad=1, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=144, Cout=32, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldx=144, ldy=32, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=2048, Cout=512, H=6, KH=1, KW=1, N=8, W=6, act=0, dil=1, ldx=2048, ldy=512, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'espc esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=28, Cout=28, H=45, KH=3, KW=3, N=16, W=60, act=0, dil=1, ldx=28, ldy=28, pad=1, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'espc esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=28, Cout=28, H=45, KH=3, KW=3, N=16, W=60, act=0, dil=2, ldx=28, ldy=28, pad=2, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'espc esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=28, Cout=28, H=45, KH=3, KW=3, N=16, W=60, act=0, dil=4, ldx=28, ldy=28, pad=4, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'espc esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=28, Cout=28, H=45, KH=3, KW=3, N=16, W=60, act=0, dil=8, ldx=28, ldy=28, pad=8, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'espc esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=28, Cout=28, H=45, KH=3, KW=3, N=16, W=60, act=0, dil=16, ldx=28, ldy=28, pad=16, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'espc esp', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=32, Cout=16, H=180, KH=1, KW=1, N=16, W=240, act=0, dil=1, ldx=32, ldy=16, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=32, Cout=192, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldx=32, ldy=192, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=192, Cout=32, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldx=192, ldy=32, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'esp', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=132, Cout=20, H=90, KH=1, KW=1, N=16, W=120, act=0, dil=1, ldx=132, ldy=20, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=32, Cout=16, H=256, KH=1, KW=1, N=8, W=512, act=0, dil=1, ldx=32, ldy=16, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=96, Cout=24, H=128, KH=1, KW=1, N=8, W=256, act=0, dil=1, ldx=96, ldy=24, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=192, Cout=64, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldx=192, ldy=64, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=24, Cout=144, H=128, KH=1, KW=1, N=8, W=256, act=0, dil=1, ldx=24, ldy=144, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=144, Cout=24, H=128, KH=1, KW=1, N=8, W=256, act=0, dil=1, ldx=144, ldy=24, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=32, Cout=32, H=256, KH=1, KW=1, N=8, W=512, act=0, dil=1, ldx=32, ldy=32, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c4', [0, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=32, Cout=64, H=180, KH=1, KW=1, N=16, W=240, act=0, dil=1, ldx=32, ldy=64, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c4', [0, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=64, H=91, KH=1, KW=1, N=16, W=121, act=0, dil=1, ldx=128, ldy=64, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c4', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=128, H=91, KH=1, KW=1, N=16, W=121, act=0, dil=1, ldx=64, ldy=128, pad=0, scale=False, shift=False, slope=0.0, stride=2, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'espc esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=20, Cout=12, H=180, KH=3, KW=3, N=16, W=240, act=0, dil=1, ldx=20, ldy=12, pad=1, scale=False, shift=False, slope=0.0, stride=2, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=16, Cout=96, H=256, KH=1, KW=1, N=8, W=512, act=0, dil=1, ldx=16, ldy=96, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=384, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldx=64, ldy=384, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=384, Cout=64, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldx=384, ldy=64, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c2 seg', [0, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=32, Cout=64, H=256, KH=1, KW=1, N=8, W=512, act=0, dil=1, ldx=32, ldy=64, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c2 seg', [0, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=64, H=129, KH=1, KW=1, N=8, W=257, act=0, dil=1, ldx=128, ldy=64, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c2', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=128, H=129, KH=1, KW=1, N=8, W=257, act=0, dil=1, ldx=64, ldy=128, pad=0, scale=False, shift=False, slope=0.0, stride=2, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=384, Cout=96, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldx=384, ldy=96, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=96, Cout=576, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldx=96, ldy=576, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=576, Cout=96, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldx=576, ldy=96, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=256, H=129, KH=1, KW=1, N=8, W=257, act=0, dil=1, ldx=64, ldy=256, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=64, H=129, KH=1, KW=1, N=8, W=257, act=0, dil=1, ldx=256, ldy=64, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=512, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldx=128, ldy=512, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=128, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldx=512, ldy=128, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=40, Cout=20, H=180, KH=3, KW=3, N=16, W=240, act=0, dil=1, ldx=40, ldy=20, pad=1, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'espc esp', [1, 128, 32, 1, 0, 0, 0], caller='fwd', Cin=132, Cout=28, H=90, KH=3, KW=3, N=16, W=120, act=0, dil=1, ldx=132, ldy=28, pad=1, scale=False, shift=False, slope=0.0, stride=2, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=576, Cout=160, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldx=576, ldy=160, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c4', [1, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=64, H=91, KH=3, KW=3, N=16, W=121, act=0, dil=1, ldx=64, ldy=64, pad=1, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c4', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=128, H=46, KH=3, KW=3, N=16, W=61, act=0, dil=1, ldx=128, ldy=128, pad=1, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=256, H=129, KH=1, KW=1, N=8, W=257, act=0, dil=1, ldx=128, ldy=256, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=128, H=129, KH=1, KW=1, N=8, W=257, act=0, dil=1, ldx=256, ldy=128, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=256, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldx=512, ldy=256, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c2 seg', [1, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=64, H=129, KH=3, KW=3, N=8, W=257, act=0, dil=1, ldx=64, ldy=64, pad=1, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c2 seg', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=128, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=1, ldx=128, ldy=128, pad=1, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=160, Cout=960, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldx=160, ldy=960, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=960, Cout=160, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldx=960, ldy=160, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c4', [1, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=64, H=91, KH=3, KW=3, N=16, W=121, act=0, dil=1, ldx=128, ldy=64, pad=1, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c4', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=128, H=91, KH=3, KW=3, N=16, W=121, act=0, dil=1, ldx=64, ldy=128, pad=1, scale=False, shift=False, slope=0.0, stride=2, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=1024, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldx=256, ldy=1024, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=1024, Cout=256, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldx=1024, ldy=256, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c2', [1, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=64, H=129, KH=3, KW=3, N=8, W=257, act=0, dil=1, ldx=128, ldy=64, pad=1, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c2', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=128, H=129, KH=3, KW=3, N=8, W=257, act=0, dil=1, ldx=64, ldy=128, pad=1, scale=False, shift=False, slope=0.0, stride=2, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'mnv2', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=960, Cout=320, H=64, KH=1, KW=1, N=8, W=128, act=0, dil=1, ldx=960, ldy=320, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c4', [1, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=64, H=180, KH=3, KW=3, N=16, W=240, act=0, dil=1, ldx=64, ldy=64, pad=1, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=512, H=129, KH=1, KW=1, N=8, W=257, act=0, dil=1, ldx=256, ldy=512, pad=0, scale=False, shift=False, slope=0.0, stride=2, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=1024, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldx=512, ldy=1024, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=1024, Cout=512, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldx=1024, ldy=512, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c2 seg', [1, 128, 64, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=64, H=256, KH=3, KW=3, N=8, W=512, act=0, dil=1, ldx=64, ldy=64, pad=1, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=128, Cout=128, H=129, KH=3, KW=3, N=8, W=257, act=0, dil=1, ldx=128, ldy=128, pad=1, scale=False, shift=False, slope=0.0, stride=2, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=256, Cout=256, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=2, ldx=256, ldy=256, pad=2, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c4', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=128, H=180, KH=3, KW=3, N=16, W=240, act=0, dil=1, ldx=64, ldy=128, pad=1, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=2048, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldx=512, ldy=2048, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=2048, Cout=512, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldx=2048, ldy=512, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'c2 seg', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=64, Cout=128, H=256, KH=3, KW=3, N=8, W=512, act=0, dil=1, ldx=64, ldy=128, pad=1, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [0, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=1024, Cout=2048, H=65, KH=1, KW=1, N=8, W=129, act=0, dil=1, ldx=1024, ldy=2048, pad=0, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=512, Cout=512, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=4, ldx=512, ldy=512, pad=4, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [1, 128, 128, 1, 0, 0, 0], caller='fwd', Cin=1024, Cout=512, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=1, ldx=1024, ldy=512, pad=1, scale=False, shift=True, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_3xtf32', 'seg', [1, 128, 128, 1, 0, 1, 0], caller='fwd', Cin=4096, Cout=512, H=65, KH=3, KW=3, N=8, W=129, act=0, dil=1, ldx=4096, ldy=512, pad=1, scale=False, shift=False, slope=0.0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 espc esp', [0, 128, 128, 4, 0, 0, 0], caller='disc', Cin=512, Cout=640, H=1, KH=1, KW=1, N=1, W=96, act=0, dil=1, ldr=0, ldx=512, ldy=640, out_h=0, out_w=0, pad=0, residual=False, scale=False, shift=True, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=245760, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 espc esp', [0, 128, 128, 5, 0, 0, 0], caller='disc', Cin=640, Cout=512, H=1, KH=1, KW=1, N=1, W=96, act=0, dil=1, ldr=512, ldx=640, ldy=512, out_h=0, out_w=0, pad=0, residual=True, scale=False, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=245760, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 espc esp', [0, 128, 128, 4, 0, 0, 0], caller='disc', Cin=512, Cout=640, H=1, KH=1, KW=1, N=1, W=96, act=0, dil=1, ldr=0, ldx=512, ldy=640, out_h=0, out_w=0, pad=0, residual=False, scale=False, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=245760, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 espc esp', [0, 128, 128, 2, 0, 0, 0], caller='disc', Cin=256, Cout=320, H=1, KH=1, KW=1, N=1, W=560, act=0, dil=1, ldr=0, ldx=256, ldy=320, out_h=0, out_w=0, pad=0, residual=False, scale=False, shift=True, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=358400, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 espc esp', [0, 128, 128, 2, 0, 0, 0], caller='disc', Cin=320, Cout=256, H=1, KH=1, KW=1, N=1, W=560, act=0, dil=1, ldr=256, ldx=320, ldy=256, out_h=0, out_w=0, pad=0, residual=True, scale=False, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=286720, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 espc esp', [0, 128, 128, 2, 0, 0, 0], caller='disc', Cin=256, Cout=320, H=1, KH=1, KW=1, N=1, W=560, act=0, dil=1, ldr=0, ldx=256, ldy=320, out_h=0, out_w=0, pad=0, residual=False, scale=False, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=358400, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 espc esp', [0, 128, 128, 5, 0, 0, 0], caller='disc', Cin=640, Cout=512, H=1, KH=1, KW=1, N=1, W=192, act=0, dil=1, ldr=512, ldx=640, ldy=512, out_h=0, out_w=0, pad=0, residual=True, scale=False, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=491520, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [0, 128, 128, 2, 0, 0, 0], caller='disc', Cin=256, Cout=320, H=1, KH=1, KW=1, N=1, W=1024, act=0, dil=1, ldr=0, ldx=256, ldy=320, out_h=0, out_w=0, pad=0, residual=False, scale=False, shift=True, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=655360, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [0, 128, 128, 4, 0, 0, 0], caller='disc', Cin=512, Cout=640, H=1, KH=1, KW=1, N=1, W=256, act=0, dil=1, ldr=0, ldx=512, ldy=640, out_h=0, out_w=0, pad=0, residual=False, scale=False, shift=True, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=655360, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [0, 128, 128, 5, 0, 0, 0], caller='disc', Cin=640, Cout=512, H=1, KH=1, KW=1, N=1, W=256, act=0, dil=1, ldr=512, ldx=640, ldy=512, out_h=0, out_w=0, pad=0, residual=True, scale=False, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=655360, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [0, 128, 128, 2, 0, 0, 0], caller='disc', Cin=320, Cout=256, H=1, KH=1, KW=1, N=1, W=1024, act=0, dil=1, ldr=256, ldx=320, ldy=256, out_h=0, out_w=0, pad=0, residual=True, scale=False, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=524288, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [0, 128, 128, 2, 0, 0, 0], caller='disc', Cin=256, Cout=320, H=1, KH=1, KW=1, N=1, W=1024, act=0, dil=1, ldr=0, ldx=256, ldy=320, out_h=0, out_w=0, pad=0, residual=False, scale=False, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=655360, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [0, 128, 128, 4, 0, 0, 0], caller='disc', Cin=512, Cout=640, H=1, KH=1, KW=1, N=1, W=256, act=0, dil=1, ldr=0, ldx=512, ldy=640, out_h=0, out_w=0, pad=0, residual=False, scale=False, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=655360, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 espc esp', [0, 128, 128, 2, 0, 0, 0], caller='disc', Cin=320, Cout=256, H=1, KH=1, KW=1, N=1, W=1120, act=0, dil=1, ldr=256, ldx=320, ldy=256, out_h=0, out_w=0, pad=0, residual=True, scale=False, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=573440, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [0, 128, 128, 5, 0, 0, 0], caller='disc', Cin=640, Cout=512, H=1, KH=1, KW=1, N=1, W=512, act=0, dil=1, ldr=512, ldx=640, ldy=512, out_h=0, out_w=0, pad=0, residual=True, scale=False, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=1310720, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [0, 128, 128, 2, 0, 0, 0], caller='disc', Cin=320, Cout=256, H=1, KH=1, KW=1, N=1, W=2048, act=0, dil=1, ldr=256, ldx=320, ldy=256, out_h=0, out_w=0, pad=0, residual=True, scale=False, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=1048576, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 espc esp', [1, 128, 128, 9, 0, 0, 0], caller='disc', Cin=512, Cout=1024, H=2, KH=3, KW=3, N=16, W=3, act=0, dil=1, ldr=0, ldx=512, ldy=1024, out_h=3, out_w=4, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=1769472, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'espc', [1, 128, 128, 1, 0, 0, 0], caller='disc', Cin=64, Cout=80, H=22, KH=3, KW=3, N=16, W=30, act=0, dil=1, ldr=0, ldx=64, ldy=80, out_h=23, out_w=30, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 esp', [1, 128, 128, 1, 0, 0, 0], caller='disc', Cin=64, Cout=80, H=23, KH=3, KW=3, N=16, W=30, act=0, dil=1, ldr=0, ldx=64, ldy=80, out_h=23, out_w=31, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 espc esp', [1, 128, 128, 6, 0, 0, 0], caller='disc', Cin=256, Cout=512, H=5, KH=3, KW=3, N=16, W=7, act=0, dil=1, ldr=0, ldx=256, ldy=512, out_h=6, out_w=8, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=2359296, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2', [1, 128, 128, 1, 0, 0, 0], caller='disc', Cin=64, Cout=80, H=32, KH=3, KW=3, N=8, W=64, act=0, dil=1, ldr=0, ldx=64, ldy=80, out_h=33, out_w=65, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'mnv2', [1, 128, 128, 1, 0, 0, 0], caller='disc', Cin=64, Cout=80, H=32, KH=3, KW=3, N=8, W=64, act=0, dil=1, ldr=0, ldx=64, ldy=80, out_h=32, out_w=64, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 esp', [1, 128, 128, 3, 0, 0, 0], caller='disc', Cin=128, Cout=256, H=11, KH=3, KW=3, N=16, W=15, act=0, dil=1, ldr=0, ldx=128, ldy=256, out_h=12, out_w=15, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=2211840, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'espc', [1, 128, 128, 4, 0, 0, 0], caller='disc', Cin=128, Cout=256, H=11, KH=3, KW=3, N=16, W=15, act=0, dil=1, ldr=0, ldx=128, ldy=256, out_h=11, out_w=15, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=2703360, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'espc', [1, 128, 64, 1, 0, 0, 0], caller='disc', Cin=20, Cout=64, H=45, KH=4, KW=4, N=16, W=60, act=1, dil=1, ldr=0, ldx=20, ldy=64, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=True, slope=0.1, stride=2, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'espc', [1, 128, 64, 1, 0, 0, 0], caller='disc', Cin=20, Cout=64, H=45, KH=4, KW=4, N=16, W=60, act=0, dil=1, ldr=0, ldx=20, ldy=64, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=2, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 espc esp', [1, 128, 128, 6, 0, 0, 0], caller='disc', Cin=512, Cout=1024, H=2, KH=3, KW=3, N=32, W=3, act=0, dil=1, ldr=0, ldx=512, ldy=1024, out_h=3, out_w=4, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=2359296, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 esp', [1, 128, 64, 1, 0, 0, 0], caller='disc', Cin=20, Cout=64, H=46, KH=4, KW=4, N=16, W=61, act=1, dil=1, ldr=0, ldx=20, ldy=64, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=True, slope=0.1, stride=2, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 esp', [1, 128, 64, 1, 0, 0, 0], caller='disc', Cin=20, Cout=64, H=46, KH=4, KW=4, N=16, W=61, act=0, dil=1, ldr=0, ldx=20, ldy=64, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=2, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'espc', [1, 128, 128, 1, 0, 0, 0], caller='disc', Cin=64, Cout=80, H=22, KH=3, KW=3, N=32, W=30, act=0, dil=1, ldr=0, ldx=64, ldy=80, out_h=23, out_w=30, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 esp', [1, 128, 128, 1, 0, 0, 0], caller='disc', Cin=64, Cout=80, H=23, KH=3, KW=3, N=32, W=30, act=0, dil=1, ldr=0, ldx=64, ldy=80, out_h=23, out_w=31, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 espc esp', [1, 128, 128, 32, 0, 0, 0], caller='disc', Cin=256, Cout=512, H=5, KH=4, KW=4, N=16, W=7, act=1, dil=1, ldr=0, ldx=256, ldy=512, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=True, slope=0.1, stride=2, w=True, w_lo=True, workspace=True, workspace_floats=1572864, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 espc esp', [1, 128, 128, 32, 0, 0, 0], caller='disc', Cin=256, Cout=512, H=5, KH=4, KW=4, N=16, W=7, act=0, dil=1, ldr=0, ldx=256, ldy=512, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=2, w=True, w_lo=True, workspace=True, workspace_floats=1572864, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [1, 128, 128, 9, 0, 0, 0], caller='disc', Cin=512, Cout=1024, H=4, KH=3, KW=3, N=8, W=8, act=0, dil=1, ldr=0, ldx=512, ldy=1024, out_h=4, out_w=8, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=2359296, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [1, 128, 128, 5, 0, 0, 0], caller='disc', Cin=256, Cout=512, H=8, KH=3, KW=3, N=8, W=16, act=0, dil=1, ldr=0, ldx=256, ldy=512, out_h=8, out_w=16, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=2621440, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [1, 128, 128, 3, 0, 0, 0], caller='disc', Cin=128, Cout=256, H=16, KH=3, KW=3, N=8, W=32, act=0, dil=1, ldr=0, ldx=128, ldy=256, out_h=16, out_w=32, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=3145728, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 espc esp', [1, 128, 128, 3, 0, 0, 0], caller='disc', Cin=256, Cout=512, H=5, KH=3, KW=3, N=32, W=7, act=0, dil=1, ldr=0, ldx=256, ldy=512, out_h=6, out_w=8, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=2359296, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'mnv2', [1, 128, 64, 1, 0, 0, 0], caller='disc', Cin=20, Cout=64, H=64, KH=4, KW=4, N=8, W=128, act=1, dil=1, ldr=0, ldx=20, ldy=64, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=True, slope=0.1, stride=2, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'mnv2', [1, 128, 64, 1, 0, 0, 0], caller='disc', Cin=20, Cout=64, H=64, KH=4, KW=4, N=8, W=128, act=0, dil=1, ldr=0, ldx=20, ldy=64, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=2, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2', [1, 128, 64, 1, 0, 0, 0], caller='disc', Cin=20, Cout=64, H=65, KH=4, KW=4, N=8, W=129, act=1, dil=1, ldr=0, ldx=20, ldy=64, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=True, slope=0.1, stride=2, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2', [1, 128, 64, 1, 0, 0, 0], caller='disc', Cin=20, Cout=64, H=65, KH=4, KW=4, N=8, W=129, act=0, dil=1, ldr=0, ldx=20, ldy=64, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=2, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 espc esp', [1, 128, 128, 13, 0, 0, 0], caller='disc', Cin=128, Cout=256, H=11, KH=4, KW=4, N=16, W=15, act=1, dil=1, ldr=0, ldx=128, ldy=256, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=True, slope=0.1, stride=2, w=True, w_lo=True, workspace=True, workspace_floats=1863680, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 espc esp', [1, 128, 128, 13, 0, 0, 0], caller='disc', Cin=128, Cout=256, H=11, KH=4, KW=4, N=16, W=15, act=0, dil=1, ldr=0, ldx=128, ldy=256, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=2, w=True, w_lo=True, workspace=True, workspace_floats=1863680, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'espc', [1, 128, 128, 7, 0, 0, 0], caller='disc', Cin=64, Cout=128, H=22, KH=4, KW=4, N=16, W=30, act=1, dil=1, ldr=0, ldx=64, ldy=128, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=True, slope=0.1, stride=2, w=True, w_lo=True, workspace=True, workspace_floats=2365440, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'espc', [1, 128, 128, 7, 0, 0, 0], caller='disc', Cin=64, Cout=128, H=22, KH=4, KW=4, N=16, W=30, act=0, dil=1, ldr=0, ldx=64, ldy=128, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=2, w=True, w_lo=True, workspace=True, workspace_floats=2365440, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 esp', [1, 128, 128, 7, 0, 0, 0], caller='disc', Cin=64, Cout=128, H=23, KH=4, KW=4, N=16, W=30, act=1, dil=1, ldr=0, ldx=64, ldy=128, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=True, slope=0.1, stride=2, w=True, w_lo=True, workspace=True, workspace_floats=2365440, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 esp', [1, 128, 128, 7, 0, 0, 0], caller='disc', Cin=64, Cout=128, H=23, KH=4, KW=4, N=16, W=30, act=0, dil=1, ldr=0, ldx=64, ldy=128, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=2, w=True, w_lo=True, workspace=True, workspace_floats=2365440, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2', [1, 128, 128, 1, 0, 0, 0], caller='disc', Cin=64, Cout=80, H=32, KH=3, KW=3, N=16, W=64, act=0, dil=1, ldr=0, ldx=64, ldy=80, out_h=33, out_w=65, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'mnv2', [1, 128, 128, 1, 0, 0, 0], caller='disc', Cin=64, Cout=80, H=32, KH=3, KW=3, N=16, W=64, act=0, dil=1, ldr=0, ldx=64, ldy=80, out_h=32, out_w=64, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c4 esp', [1, 128, 128, 1, 0, 0, 0], caller='disc', Cin=128, Cout=256, H=11, KH=3, KW=3, N=32, W=15, act=0, dil=1, ldr=0, ldx=128, ldy=256, out_h=12, out_w=15, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'espc', [1, 128, 128, 1, 0, 0, 0], caller='disc', Cin=128, Cout=256, H=11, KH=3, KW=3, N=32, W=15, act=0, dil=1, ldr=0, ldx=128, ldy=256, out_h=11, out_w=15, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [1, 128, 128, 5, 0, 0, 0], caller='disc', Cin=64, Cout=128, H=32, KH=4, KW=4, N=8, W=64, act=1, dil=1, ldr=0, ldx=64, ldy=128, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=True, slope=0.1, stride=2, w=True, w_lo=True, workspace=True, workspace_floats=2621440, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [1, 128, 128, 8, 0, 0, 0], caller='disc', Cin=128, Cout=256, H=16, KH=4, KW=4, N=8, W=32, act=1, dil=1, ldr=0, ldx=128, ldy=256, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=True, slope=0.1, stride=2, w=True, w_lo=True, workspace=True, workspace_floats=2097152, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [1, 128, 128, 16, 0, 0, 0], caller='disc', Cin=256, Cout=512, H=8, KH=4, KW=4, N=8, W=16, act=1, dil=1, ldr=0, ldx=256, ldy=512, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=True, slope=0.1, stride=2, w=True, w_lo=True, workspace=True, workspace_floats=2097152, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [1, 128, 128, 5, 0, 0, 0], caller='disc', Cin=64, Cout=128, H=32, KH=4, KW=4, N=8, W=64, act=0, dil=1, ldr=0, ldx=64, ldy=128, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=2, w=True, w_lo=True, workspace=True, workspace_floats=2621440, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [1, 128, 128, 8, 0, 0, 0], caller='disc', Cin=128, Cout=256, H=16, KH=4, KW=4, N=8, W=32, act=0, dil=1, ldr=0, ldx=128, ldy=256, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=2, w=True, w_lo=True, workspace=True, workspace_floats=2097152, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [1, 128, 128, 16, 0, 0, 0], caller='disc', Cin=256, Cout=512, H=8, KH=4, KW=4, N=8, W=16, act=0, dil=1, ldr=0, ldx=256, ldy=512, out_h=0, out_w=0, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=2, w=True, w_lo=True, workspace=True, workspace_floats=2097152, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [1, 128, 128, 5, 0, 0, 0], caller='disc', Cin=512, Cout=1024, H=4, KH=3, KW=3, N=16, W=8, act=0, dil=1, ldr=0, ldx=512, ldy=1024, out_h=4, out_w=8, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=2621440, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [1, 128, 128, 3, 0, 0, 0], caller='disc', Cin=256, Cout=512, H=8, KH=3, KW=3, N=16, W=16, act=0, dil=1, ldr=0, ldx=256, ldy=512, out_h=8, out_w=16, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=True, workspace_floats=3145728, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_splitk', 'c2 mnv2', [1, 128, 128, 1, 0, 0, 0], caller='disc', Cin=128, Cout=256, H=16, KH=3, KW=3, N=16, W=32, act=0, dil=1, ldr=0, ldx=128, ldy=256, out_h=16, out_w=32, pad=1, residual=False, scale=True, shift=False, slope=0.0, stride=1, w=True, w_lo=True, workspace=False, workspace_floats=0, x=True, x_lo=True, y=True),
    L('skd_conv2d_fwd_sm100_strided', 'espc esp', [2, 128, 32, 1, 0, 0, 0], caller='dgrad', Cin=12, Cout=20, H=90, KH=1, KW=1, N=16, W=120, dil=1, ldx=12, out_h=90, out_w=120, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=864000, y_pix=40, y_row=9600),
    L('skd_conv2d_fwd_sm100_strided', 'espc esp', [2, 128, 32, 1, 0, 0, 0], caller='dgrad', Cin=12, Cout=20, H=90, KH=1, KW=2, N=16, W=120, dil=1, ldx=12, out_h=90, out_w=120, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=864000, y_pix=40, y_row=9600),
    L('skd_conv2d_fwd_sm100_strided', 'espc esp', [2, 128, 32, 1, 0, 0, 0], caller='dgrad', Cin=12, Cout=20, H=90, KH=2, KW=1, N=16, W=120, dil=1, ldx=12, out_h=90, out_w=120, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=864000, y_pix=40, y_row=9600),
    L('skd_conv2d_fwd_sm100_strided', 'espc esp', [2, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=28, Cout=132, H=45, KH=1, KW=1, N=16, W=60, dil=1, ldx=28, out_h=45, out_w=60, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=1425600, y_pix=264, y_row=31680),
    L('skd_conv2d_fwd_sm100_strided', 'espc esp', [2, 128, 32, 1, 0, 0, 0], caller='dgrad', Cin=12, Cout=20, H=90, KH=2, KW=2, N=16, W=120, dil=1, ldx=12, out_h=90, out_w=120, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=864000, y_pix=40, y_row=9600),
    L('skd_conv2d_fwd_sm100_strided', 'espc esp', [2, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=28, Cout=132, H=45, KH=1, KW=2, N=16, W=60, dil=1, ldx=28, out_h=45, out_w=60, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=1425600, y_pix=264, y_row=31680),
    L('skd_conv2d_fwd_sm100_strided', 'espc esp', [2, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=28, Cout=132, H=45, KH=2, KW=1, N=16, W=60, dil=1, ldx=28, out_h=45, out_w=60, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=1425600, y_pix=264, y_row=31680),
    L('skd_conv2d_fwd_sm100_strided', 'c4', [2, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=64, H=46, KH=1, KW=1, N=16, W=61, dil=1, ldx=128, out_h=46, out_w=61, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=704704, y_pix=128, y_row=15488),
    L('skd_conv2d_fwd_sm100_strided', 'c2', [2, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=64, H=65, KH=1, KW=1, N=8, W=129, dil=1, ldx=128, out_h=65, out_w=129, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=2121792, y_pix=128, y_row=32896),
    L('skd_conv2d_fwd_sm100_strided', 'espc esp', [2, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=28, Cout=132, H=45, KH=2, KW=2, N=16, W=60, dil=1, ldx=28, out_h=45, out_w=60, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=1425600, y_pix=264, y_row=31680),
    L('skd_conv2d_fwd_sm100_strided', 'c4', [2, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=64, H=46, KH=1, KW=2, N=16, W=61, dil=1, ldx=128, out_h=46, out_w=60, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=704704, y_pix=128, y_row=15488),
    L('skd_conv2d_fwd_sm100_strided', 'c4', [2, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=64, H=46, KH=2, KW=1, N=16, W=61, dil=1, ldx=128, out_h=45, out_w=61, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=704704, y_pix=128, y_row=15488),
    L('skd_conv2d_fwd_sm100_strided', 'c2', [2, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=64, H=65, KH=1, KW=2, N=8, W=129, dil=1, ldx=128, out_h=65, out_w=128, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=2121792, y_pix=128, y_row=32896),
    L('skd_conv2d_fwd_sm100_strided', 'c2', [2, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=64, H=65, KH=2, KW=1, N=8, W=129, dil=1, ldx=128, out_h=64, out_w=129, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=2121792, y_pix=128, y_row=32896),
    L('skd_conv2d_fwd_sm100_strided', 'seg', [2, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=128, H=65, KH=1, KW=1, N=8, W=129, dil=1, ldx=128, out_h=65, out_w=129, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=4243584, y_pix=256, y_row=65792),
    L('skd_conv2d_fwd_sm100_strided', 'c4', [2, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=64, H=46, KH=2, KW=2, N=16, W=61, dil=1, ldx=128, out_h=45, out_w=60, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=704704, y_pix=128, y_row=15488),
    L('skd_conv2d_fwd_sm100_strided', 'c2', [2, 128, 64, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=64, H=65, KH=2, KW=2, N=8, W=129, dil=1, ldx=128, out_h=64, out_w=128, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=2121792, y_pix=128, y_row=32896),
    L('skd_conv2d_fwd_sm100_strided', 'seg', [2, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=128, H=65, KH=1, KW=2, N=8, W=129, dil=1, ldx=128, out_h=65, out_w=128, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=4243584, y_pix=256, y_row=65792),
    L('skd_conv2d_fwd_sm100_strided', 'seg', [2, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=128, H=65, KH=2, KW=1, N=8, W=129, dil=1, ldx=128, out_h=64, out_w=129, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=4243584, y_pix=256, y_row=65792),
    L('skd_conv2d_fwd_sm100_strided', 'seg', [2, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=128, Cout=128, H=65, KH=2, KW=2, N=8, W=129, dil=1, ldx=128, out_h=64, out_w=128, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=4243584, y_pix=256, y_row=65792),
    L('skd_conv2d_fwd_sm100_strided', 'seg', [2, 128, 128, 1, 0, 0, 0], caller='dgrad', Cin=512, Cout=256, H=65, KH=1, KW=1, N=8, W=129, dil=1, ldx=512, out_h=65, out_w=129, pad=0, round_tf32=0, stride=1, w=True, x=True, y=True, y_img=8487168, y_pix=512, y_row=131584),
    L('skd_conv2d_fwd_sm100_strided_3xtf32', 'esp', [2, 128, 64, 1, 0, 0, 0], caller='convT', Cin=20, Cout=40, H=45, KH=1, KW=1, N=16, W=60, dil=1, ldx=20, pad=0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True, y_img=216000, y_pix=40, y_row=4800),
    L('skd_conv2d_fwd_sm100_strided_3xtf32', 'esp', [2, 128, 64, 1, 0, 0, 0], caller='convT', Cin=20, Cout=40, H=90, KH=1, KW=1, N=16, W=120, dil=1, ldx=20, pad=0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True, y_img=864000, y_pix=40, y_row=9600),
    L('skd_conv2d_fwd_sm100_strided_3xtf32', 'esp', [2, 128, 64, 1, 0, 0, 0], caller='convT', Cin=20, Cout=40, H=180, KH=1, KW=1, N=16, W=240, dil=1, ldx=20, pad=0, stride=1, w_hi=True, w_lo=True, x_hi=True, x_lo=True, y=True, y_img=3456000, y_pix=40, y_row=19200),
    L('skd_conv2d_wgrad_sm100', 'c4 espc esp', [128, 1, 1], caller='disc', Cin=512, Cout=640, H=2, KH=1, KW=1, N=16, W=3, dil=1, dw=True, dy=True, ldx=512, ldy=640, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4 espc esp', [128, 1, 1], caller='disc', Cin=256, Cout=320, H=5, KH=1, KW=1, N=16, W=7, dil=1, dw=True, dy=True, ldx=256, ldy=320, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4 espc esp', [128, 1, 1], caller='disc', Cin=512, Cout=640, H=2, KH=1, KW=1, N=32, W=3, dil=1, dw=True, dy=True, ldx=512, ldy=640, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 mnv2', [128, 1, 1], caller='disc', Cin=512, Cout=640, H=4, KH=1, KW=1, N=8, W=8, dil=1, dw=True, dy=True, ldx=512, ldy=640, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 mnv2', [128, 1, 2], caller='disc', Cin=256, Cout=320, H=8, KH=1, KW=1, N=8, W=16, dil=1, dw=True, dy=True, ldx=256, ldy=320, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4 espc esp', [128, 1, 2], caller='disc', Cin=256, Cout=320, H=5, KH=1, KW=1, N=32, W=7, dil=1, dw=True, dy=True, ldx=256, ldy=320, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 mnv2', [128, 1, 1], caller='disc', Cin=512, Cout=640, H=4, KH=1, KW=1, N=16, W=8, dil=1, dw=True, dy=True, ldx=512, ldy=640, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 mnv2', [128, 1, 4], caller='disc', Cin=256, Cout=320, H=8, KH=1, KW=1, N=16, W=16, dil=1, dw=True, dy=True, ldx=256, ldy=320, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc', [32, 1, 8], caller='disc', Cin=20, Cout=64, H=45, KH=4, KW=4, N=16, W=60, dil=1, dw=True, dy=True, ldx=20, ldy=64, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4 esp', [32, 1, 8], caller='disc', Cin=20, Cout=64, H=46, KH=4, KW=4, N=16, W=61, dil=1, dw=True, dy=True, ldx=20, ldy=64, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4 espc esp', [128, 1, 1], caller='disc', Cin=256, Cout=512, H=5, KH=4, KW=4, N=16, W=7, dil=1, dw=True, dy=True, ldx=256, ldy=512, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [32, 1, 8], caller='disc', Cin=20, Cout=64, H=64, KH=4, KW=4, N=8, W=128, dil=1, dw=True, dy=True, ldx=20, ldy=64, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2', [32, 1, 8], caller='disc', Cin=20, Cout=64, H=65, KH=4, KW=4, N=8, W=129, dil=1, dw=True, dy=True, ldx=20, ldy=64, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4 espc esp', [128, 1, 1], caller='disc', Cin=128, Cout=256, H=11, KH=4, KW=4, N=16, W=15, dil=1, dw=True, dy=True, ldx=128, ldy=256, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc', [64, 1, 5], caller='disc', Cin=64, Cout=128, H=22, KH=4, KW=4, N=16, W=30, dil=1, dw=True, dy=True, ldx=64, ldy=128, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4 esp', [64, 1, 5], caller='disc', Cin=64, Cout=128, H=23, KH=4, KW=4, N=16, W=30, dil=1, dw=True, dy=True, ldx=64, ldy=128, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc', [32, 1, 33], caller='disc', Cin=20, Cout=64, H=45, KH=4, KW=4, N=32, W=60, dil=1, dw=True, dy=True, ldx=20, ldy=64, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4 esp', [32, 1, 33], caller='disc', Cin=20, Cout=64, H=46, KH=4, KW=4, N=32, W=61, dil=1, dw=True, dy=True, ldx=20, ldy=64, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 mnv2', [128, 1, 1], caller='disc', Cin=256, Cout=512, H=8, KH=4, KW=4, N=8, W=16, dil=1, dw=True, dy=True, ldx=256, ldy=512, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 mnv2', [128, 1, 2], caller='disc', Cin=128, Cout=256, H=16, KH=4, KW=4, N=8, W=32, dil=1, dw=True, dy=True, ldx=128, ldy=256, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 mnv2', [64, 1, 8], caller='disc', Cin=64, Cout=128, H=32, KH=4, KW=4, N=8, W=64, dil=1, dw=True, dy=True, ldx=64, ldy=128, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4 espc esp', [128, 1, 1], caller='disc', Cin=256, Cout=512, H=5, KH=4, KW=4, N=32, W=7, dil=1, dw=True, dy=True, ldx=256, ldy=512, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [32, 1, 8], caller='disc', Cin=20, Cout=64, H=64, KH=4, KW=4, N=16, W=128, dil=1, dw=True, dy=True, ldx=20, ldy=64, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2', [32, 1, 8], caller='disc', Cin=20, Cout=64, H=65, KH=4, KW=4, N=16, W=129, dil=1, dw=True, dy=True, ldx=20, ldy=64, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4 espc esp', [128, 1, 2], caller='disc', Cin=128, Cout=256, H=11, KH=4, KW=4, N=32, W=15, dil=1, dw=True, dy=True, ldx=128, ldy=256, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc', [64, 1, 8], caller='disc', Cin=64, Cout=128, H=22, KH=4, KW=4, N=32, W=30, dil=1, dw=True, dy=True, ldx=64, ldy=128, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4 esp', [64, 1, 8], caller='disc', Cin=64, Cout=128, H=23, KH=4, KW=4, N=32, W=30, dil=1, dw=True, dy=True, ldx=64, ldy=128, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 mnv2', [128, 1, 1], caller='disc', Cin=256, Cout=512, H=8, KH=4, KW=4, N=16, W=16, dil=1, dw=True, dy=True, ldx=256, ldy=512, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 mnv2', [128, 1, 4], caller='disc', Cin=128, Cout=256, H=16, KH=4, KW=4, N=16, W=32, dil=1, dw=True, dy=True, ldx=128, ldy=256, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 mnv2', [64, 1, 8], caller='disc', Cin=64, Cout=128, H=32, KH=4, KW=4, N=16, W=64, dil=1, dw=True, dy=True, ldx=64, ldy=128, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 1], caller='fwd', Cin=320, Cout=128, H=1, KH=1, KW=1, N=8, W=1, dil=1, dw=True, dy=True, ldx=320, ldy=128, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2', [128, 1, 1], caller='fwd', Cin=512, Cout=128, H=1, KH=1, KW=1, N=8, W=1, dil=1, dw=True, dy=True, ldx=512, ldy=128, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [128, 1, 1], caller='fwd', Cin=512, Cout=128, H=1, KH=1, KW=1, N=16, W=1, dil=1, dw=True, dy=True, ldx=512, ldy=128, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 1], caller='fwd', Cin=320, Cout=128, H=2, KH=1, KW=1, N=8, W=2, dil=1, dw=True, dy=True, ldx=320, ldy=128, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2', [128, 1, 1], caller='fwd', Cin=512, Cout=128, H=2, KH=1, KW=1, N=8, W=2, dil=1, dw=True, dy=True, ldx=512, ldy=128, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 1], caller='fwd', Cin=320, Cout=128, H=3, KH=1, KW=1, N=8, W=3, dil=1, dw=True, dy=True, ldx=320, ldy=128, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [128, 1, 1], caller='fwd', Cin=512, Cout=128, H=2, KH=1, KW=1, N=16, W=2, dil=1, dw=True, dy=True, ldx=512, ldy=128, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2', [128, 1, 1], caller='fwd', Cin=512, Cout=128, H=3, KH=1, KW=1, N=8, W=3, dil=1, dw=True, dy=True, ldx=512, ldy=128, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 1], caller='fwd', Cin=2048, Cout=512, H=1, KH=1, KW=1, N=8, W=1, dil=1, dw=True, dy=True, ldx=2048, ldy=512, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [128, 1, 1], caller='fwd', Cin=512, Cout=128, H=3, KH=1, KW=1, N=16, W=3, dil=1, dw=True, dy=True, ldx=512, ldy=128, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 1], caller='fwd', Cin=320, Cout=128, H=6, KH=1, KW=1, N=8, W=6, dil=1, dw=True, dy=True, ldx=320, ldy=128, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2', [128, 1, 1], caller='fwd', Cin=512, Cout=128, H=6, KH=1, KW=1, N=8, W=6, dil=1, dw=True, dy=True, ldx=512, ldy=128, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'esp', [32, 1, 29], caller='fwd', Cin=4, Cout=4, H=90, KH=3, KW=3, N=16, W=120, dil=2, dw=True, dy=True, ldx=4, ldy=4, pad=2, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'esp', [32, 1, 29], caller='fwd', Cin=4, Cout=4, H=90, KH=3, KW=3, N=16, W=120, dil=4, dw=True, dy=True, ldx=4, ldy=4, pad=4, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'esp', [32, 1, 29], caller='fwd', Cin=4, Cout=4, H=90, KH=3, KW=3, N=16, W=120, dil=8, dw=True, dy=True, ldx=4, ldy=4, pad=8, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'esp', [32, 1, 29], caller='fwd', Cin=4, Cout=4, H=90, KH=3, KW=3, N=16, W=120, dil=16, dw=True, dy=True, ldx=4, ldy=4, pad=16, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'esp', [64, 1, 132], caller='fwd', Cin=40, Cout=4, H=90, KH=1, KW=1, N=16, W=120, dil=1, dw=True, dy=True, ldx=40, ldy=4, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 1], caller='fwd', Cin=2048, Cout=512, H=2, KH=1, KW=1, N=8, W=2, dil=1, dw=True, dy=True, ldx=2048, ldy=512, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [128, 1, 1], caller='fwd', Cin=512, Cout=128, H=6, KH=1, KW=1, N=16, W=6, dil=1, dw=True, dy=True, ldx=512, ldy=128, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'esp', [32, 1, 29], caller='fwd', Cin=4, Cout=8, H=90, KH=3, KW=3, N=16, W=120, dil=1, dw=True, dy=True, ldx=4, ldy=8, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 1], caller='fwd', Cin=2048, Cout=512, H=3, KH=1, KW=1, N=8, W=3, dil=1, dw=True, dy=True, ldx=2048, ldy=512, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [128, 1, 83], caller='fwd', Cin=128, Cout=20, H=46, KH=1, KW=1, N=16, W=61, dil=1, dw=True, dy=True, ldx=128, ldy=20, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc esp', [64, 1, 132], caller='fwd', Cin=64, Cout=12, H=90, KH=1, KW=1, N=16, W=120, dil=1, dw=True, dy=True, ldx=64, ldy=12, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc esp', [128, 1, 80], caller='fwd', Cin=128, Cout=28, H=45, KH=1, KW=1, N=16, W=60, dil=1, dw=True, dy=True, ldx=128, ldy=28, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 128], caller='fwd', Cin=128, Cout=20, H=64, KH=1, KW=1, N=8, W=128, dil=1, dw=True, dy=True, ldx=128, ldy=20, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2', [128, 1, 124], caller='fwd', Cin=128, Cout=20, H=65, KH=1, KW=1, N=8, W=129, dil=1, dw=True, dy=True, ldx=128, ldy=20, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc esp', [128, 1, 65], caller='fwd', Cin=256, Cout=20, H=45, KH=1, KW=1, N=16, W=60, dil=1, dw=True, dy=True, ldx=256, ldy=20, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc esp', [32, 1, 29], caller='fwd', Cin=12, Cout=12, H=90, KH=3, KW=3, N=16, W=120, dil=2, dw=True, dy=True, ldx=12, ldy=12, pad=2, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc esp', [32, 1, 29], caller='fwd', Cin=12, Cout=12, H=90, KH=3, KW=3, N=16, W=120, dil=4, dw=True, dy=True, ldx=12, ldy=12, pad=4, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc esp', [32, 1, 29], caller='fwd', Cin=12, Cout=12, H=90, KH=3, KW=3, N=16, W=120, dil=8, dw=True, dy=True, ldx=12, ldy=12, pad=8, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc esp', [32, 1, 29], caller='fwd', Cin=12, Cout=12, H=90, KH=3, KW=3, N=16, W=120, dil=16, dw=True, dy=True, ldx=12, ldy=12, pad=16, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'esp', [32, 1, 33], caller='fwd', Cin=20, Cout=20, H=90, KH=2, KW=2, N=16, W=120, dil=1, dw=True, dy=True, ldx=20, ldy=20, pad=0, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc esp', [32, 1, 29], caller='fwd', Cin=12, Cout=16, H=90, KH=3, KW=3, N=16, W=120, dil=1, dw=True, dy=True, ldx=12, ldy=16, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 63], caller='fwd', Cin=144, Cout=32, H=64, KH=1, KW=1, N=8, W=128, dil=1, dw=True, dy=True, ldx=144, ldy=32, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 1], caller='fwd', Cin=2048, Cout=512, H=6, KH=1, KW=1, N=8, W=6, dil=1, dw=True, dy=True, ldx=2048, ldy=512, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc esp', [32, 1, 29], caller='fwd', Cin=28, Cout=28, H=45, KH=3, KW=3, N=16, W=60, dil=1, dw=True, dy=True, ldx=28, ldy=28, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc esp', [32, 1, 29], caller='fwd', Cin=28, Cout=28, H=45, KH=3, KW=3, N=16, W=60, dil=2, dw=True, dy=True, ldx=28, ldy=28, pad=2, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc esp', [32, 1, 29], caller='fwd', Cin=28, Cout=28, H=45, KH=3, KW=3, N=16, W=60, dil=4, dw=True, dy=True, ldx=28, ldy=28, pad=4, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc esp', [32, 1, 29], caller='fwd', Cin=28, Cout=28, H=45, KH=3, KW=3, N=16, W=60, dil=8, dw=True, dy=True, ldx=28, ldy=28, pad=8, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc esp', [32, 1, 29], caller='fwd', Cin=28, Cout=28, H=45, KH=3, KW=3, N=16, W=60, dil=16, dw=True, dy=True, ldx=28, ldy=28, pad=16, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc esp', [32, 1, 130], caller='fwd', Cin=32, Cout=16, H=180, KH=1, KW=1, N=16, W=240, dil=1, dw=True, dy=True, ldx=32, ldy=16, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [32, 1, 63], caller='fwd', Cin=32, Cout=192, H=64, KH=1, KW=1, N=8, W=128, dil=1, dw=True, dy=True, ldx=32, ldy=192, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 63], caller='fwd', Cin=192, Cout=32, H=64, KH=1, KW=1, N=8, W=128, dil=1, dw=True, dy=True, ldx=192, ldy=32, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'esp', [128, 1, 65], caller='fwd', Cin=132, Cout=20, H=90, KH=1, KW=1, N=16, W=120, dil=1, dw=True, dy=True, ldx=132, ldy=20, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [32, 1, 130], caller='fwd', Cin=32, Cout=16, H=256, KH=1, KW=1, N=8, W=512, dil=1, dw=True, dy=True, ldx=32, ldy=16, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 131], caller='fwd', Cin=96, Cout=24, H=128, KH=1, KW=1, N=8, W=256, dil=1, dw=True, dy=True, ldx=96, ldy=24, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 33], caller='fwd', Cin=512, Cout=20, H=65, KH=1, KW=1, N=8, W=129, dil=1, dw=True, dy=True, ldx=512, ldy=20, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 63], caller='fwd', Cin=192, Cout=64, H=64, KH=1, KW=1, N=8, W=128, dil=1, dw=True, dy=True, ldx=192, ldy=64, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [32, 1, 65], caller='fwd', Cin=24, Cout=144, H=128, KH=1, KW=1, N=8, W=256, dil=1, dw=True, dy=True, ldx=24, ldy=144, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 65], caller='fwd', Cin=144, Cout=24, H=128, KH=1, KW=1, N=8, W=256, dil=1, dw=True, dy=True, ldx=144, ldy=24, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [32, 1, 130], caller='fwd', Cin=32, Cout=32, H=256, KH=1, KW=1, N=8, W=512, dil=1, dw=True, dy=True, ldx=32, ldy=32, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'esp', [32, 1, 33], caller='fwd', Cin=20, Cout=20, H=180, KH=2, KW=2, N=16, W=240, dil=1, dw=True, dy=True, ldx=20, ldy=20, pad=0, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [32, 1, 130], caller='fwd', Cin=32, Cout=64, H=180, KH=1, KW=1, N=16, W=240, dil=1, dw=True, dy=True, ldx=32, ldy=64, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [64, 1, 83], caller='fwd', Cin=64, Cout=128, H=91, KH=1, KW=1, N=16, W=121, dil=1, dw=True, dy=True, ldx=64, ldy=128, pad=0, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [128, 1, 132], caller='fwd', Cin=128, Cout=64, H=91, KH=1, KW=1, N=16, W=121, dil=1, dw=True, dy=True, ldx=128, ldy=64, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [128, 1, 64], caller='fwd', Cin=128, Cout=256, H=46, KH=1, KW=1, N=16, W=61, dil=1, dw=True, dy=True, ldx=128, ldy=256, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc esp', [32, 1, 29], caller='fwd', Cin=20, Cout=12, H=180, KH=3, KW=3, N=16, W=240, dil=1, dw=True, dy=True, ldx=20, ldy=12, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [64, 1, 44], caller='fwd', Cin=64, Cout=384, H=64, KH=1, KW=1, N=8, W=128, dil=1, dw=True, dy=True, ldx=64, ldy=384, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 44], caller='fwd', Cin=384, Cout=64, H=64, KH=1, KW=1, N=8, W=128, dil=1, dw=True, dy=True, ldx=384, ldy=64, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [32, 1, 130], caller='fwd', Cin=16, Cout=96, H=256, KH=1, KW=1, N=8, W=512, dil=1, dw=True, dy=True, ldx=16, ldy=96, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 seg', [32, 1, 130], caller='fwd', Cin=32, Cout=64, H=256, KH=1, KW=1, N=8, W=512, dil=1, dw=True, dy=True, ldx=32, ldy=64, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2', [64, 1, 124], caller='fwd', Cin=64, Cout=128, H=129, KH=1, KW=1, N=8, W=257, dil=1, dw=True, dy=True, ldx=64, ldy=128, pad=0, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 seg', [128, 1, 130], caller='fwd', Cin=128, Cout=64, H=129, KH=1, KW=1, N=8, W=257, dil=1, dw=True, dy=True, ldx=128, ldy=64, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2', [128, 1, 66], caller='fwd', Cin=128, Cout=256, H=65, KH=1, KW=1, N=8, W=129, dil=1, dw=True, dy=True, ldx=128, ldy=256, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 44], caller='fwd', Cin=384, Cout=96, H=64, KH=1, KW=1, N=8, W=128, dil=1, dw=True, dy=True, ldx=384, ldy=96, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 26], caller='fwd', Cin=96, Cout=576, H=64, KH=1, KW=1, N=8, W=128, dil=1, dw=True, dy=True, ldx=96, ldy=576, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 26], caller='fwd', Cin=576, Cout=96, H=64, KH=1, KW=1, N=8, W=128, dil=1, dw=True, dy=True, ldx=576, ldy=96, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [64, 1, 65], caller='fwd', Cin=64, Cout=256, H=129, KH=1, KW=1, N=8, W=257, dil=1, dw=True, dy=True, ldx=64, ldy=256, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 65], caller='fwd', Cin=256, Cout=64, H=129, KH=1, KW=1, N=8, W=257, dil=1, dw=True, dy=True, ldx=256, ldy=64, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 33], caller='fwd', Cin=128, Cout=512, H=65, KH=1, KW=1, N=8, W=129, dil=1, dw=True, dy=True, ldx=128, ldy=512, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 33], caller='fwd', Cin=512, Cout=128, H=65, KH=1, KW=1, N=8, W=129, dil=1, dw=True, dy=True, ldx=512, ldy=128, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'esp', [32, 1, 33], caller='fwd', Cin=20, Cout=20, H=360, KH=2, KW=2, N=16, W=480, dil=1, dw=True, dy=True, ldx=20, ldy=20, pad=0, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'esp', [64, 1, 29], caller='fwd', Cin=40, Cout=20, H=180, KH=3, KW=3, N=16, W=240, dil=1, dw=True, dy=True, ldx=40, ldy=20, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'espc esp', [128, 1, 22], caller='fwd', Cin=132, Cout=28, H=90, KH=3, KW=3, N=16, W=120, dil=1, dw=True, dy=True, ldx=132, ldy=28, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [128, 1, 33], caller='fwd', Cin=256, Cout=512, H=46, KH=1, KW=1, N=16, W=61, dil=1, dw=True, dy=True, ldx=256, ldy=512, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 13], caller='fwd', Cin=576, Cout=160, H=64, KH=1, KW=1, N=8, W=128, dil=1, dw=True, dy=True, ldx=576, ldy=160, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [64, 1, 29], caller='fwd', Cin=64, Cout=64, H=91, KH=3, KW=3, N=16, W=121, dil=1, dw=True, dy=True, ldx=64, ldy=64, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [128, 1, 29], caller='fwd', Cin=128, Cout=128, H=46, KH=3, KW=3, N=16, W=61, dil=1, dw=True, dy=True, ldx=128, ldy=128, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 29], caller='fwd', Cin=96, Cout=128, H=64, KH=3, KW=3, N=8, W=128, dil=1, dw=True, dy=True, ldx=96, ldy=128, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 65], caller='fwd', Cin=256, Cout=128, H=129, KH=1, KW=1, N=8, W=257, dil=1, dw=True, dy=True, ldx=256, ldy=128, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 65], caller='fwd', Cin=128, Cout=256, H=129, KH=1, KW=1, N=8, W=257, dil=1, dw=True, dy=True, ldx=128, ldy=256, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2', [128, 1, 33], caller='fwd', Cin=256, Cout=512, H=65, KH=1, KW=1, N=8, W=129, dil=1, dw=True, dy=True, ldx=256, ldy=512, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 33], caller='fwd', Cin=512, Cout=256, H=65, KH=1, KW=1, N=8, W=129, dil=1, dw=True, dy=True, ldx=512, ldy=256, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 seg', [64, 1, 29], caller='fwd', Cin=64, Cout=64, H=129, KH=3, KW=3, N=8, W=257, dil=1, dw=True, dy=True, ldx=64, ldy=64, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 seg', [128, 1, 29], caller='fwd', Cin=128, Cout=128, H=65, KH=3, KW=3, N=8, W=129, dil=1, dw=True, dy=True, ldx=128, ldy=128, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 33], caller='fwd', Cin=160, Cout=960, H=64, KH=1, KW=1, N=8, W=128, dil=1, dw=True, dy=True, ldx=160, ldy=960, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 33], caller='fwd', Cin=960, Cout=160, H=64, KH=1, KW=1, N=8, W=128, dil=1, dw=True, dy=True, ldx=960, ldy=160, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [64, 1, 29], caller='fwd', Cin=64, Cout=128, H=91, KH=3, KW=3, N=16, W=121, dil=1, dw=True, dy=True, ldx=64, ldy=128, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [128, 1, 29], caller='fwd', Cin=128, Cout=64, H=91, KH=3, KW=3, N=16, W=121, dil=1, dw=True, dy=True, ldx=128, ldy=64, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [128, 1, 22], caller='fwd', Cin=256, Cout=128, H=46, KH=3, KW=3, N=16, W=61, dil=1, dw=True, dy=True, ldx=256, ldy=128, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [128, 1, 22], caller='fwd', Cin=128, Cout=256, H=46, KH=3, KW=3, N=16, W=61, dil=2, dw=True, dy=True, ldx=128, ldy=256, pad=2, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 33], caller='fwd', Cin=256, Cout=1024, H=65, KH=1, KW=1, N=8, W=129, dil=1, dw=True, dy=True, ldx=256, ldy=1024, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 33], caller='fwd', Cin=1024, Cout=256, H=65, KH=1, KW=1, N=8, W=129, dil=1, dw=True, dy=True, ldx=1024, ldy=256, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2', [64, 1, 29], caller='fwd', Cin=64, Cout=128, H=129, KH=3, KW=3, N=8, W=257, dil=1, dw=True, dy=True, ldx=64, ldy=128, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2', [128, 1, 29], caller='fwd', Cin=128, Cout=64, H=129, KH=3, KW=3, N=8, W=257, dil=1, dw=True, dy=True, ldx=128, ldy=64, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2', [128, 1, 22], caller='fwd', Cin=256, Cout=128, H=65, KH=3, KW=3, N=8, W=129, dil=1, dw=True, dy=True, ldx=256, ldy=128, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2', [128, 1, 22], caller='fwd', Cin=128, Cout=256, H=65, KH=3, KW=3, N=8, W=129, dil=2, dw=True, dy=True, ldx=128, ldy=256, pad=2, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 11], caller='fwd', Cin=960, Cout=320, H=64, KH=1, KW=1, N=8, W=128, dil=1, dw=True, dy=True, ldx=960, ldy=320, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [64, 1, 29], caller='fwd', Cin=64, Cout=64, H=180, KH=3, KW=3, N=16, W=240, dil=1, dw=True, dy=True, ldx=64, ldy=64, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [128, 1, 11], caller='fwd', Cin=256, Cout=256, H=46, KH=3, KW=3, N=16, W=61, dil=2, dw=True, dy=True, ldx=256, ldy=256, pad=2, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 33], caller='fwd', Cin=256, Cout=512, H=129, KH=1, KW=1, N=8, W=257, dil=1, dw=True, dy=True, ldx=256, ldy=512, pad=0, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 4], caller='fwd', Cin=1024, Cout=512, H=65, KH=1, KW=1, N=8, W=129, dil=1, dw=True, dy=True, ldx=1024, ldy=512, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 4], caller='fwd', Cin=512, Cout=1024, H=65, KH=1, KW=1, N=8, W=129, dil=1, dw=True, dy=True, ldx=512, ldy=1024, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 seg', [64, 1, 29], caller='fwd', Cin=64, Cout=64, H=256, KH=3, KW=3, N=8, W=512, dil=1, dw=True, dy=True, ldx=64, ldy=64, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 29], caller='fwd', Cin=128, Cout=128, H=129, KH=3, KW=3, N=8, W=257, dil=1, dw=True, dy=True, ldx=128, ldy=128, pad=1, stride=2, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 seg', [128, 1, 11], caller='fwd', Cin=256, Cout=256, H=65, KH=3, KW=3, N=8, W=129, dil=2, dw=True, dy=True, ldx=256, ldy=256, pad=2, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [64, 1, 29], caller='fwd', Cin=64, Cout=128, H=180, KH=3, KW=3, N=16, W=240, dil=1, dw=True, dy=True, ldx=64, ldy=128, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [128, 1, 7], caller='fwd', Cin=1024, Cout=128, H=46, KH=3, KW=3, N=16, W=61, dil=1, dw=True, dy=True, ldx=1024, ldy=128, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [128, 1, 7], caller='fwd', Cin=256, Cout=512, H=46, KH=3, KW=3, N=16, W=61, dil=4, dw=True, dy=True, ldx=256, ldy=512, pad=4, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'mnv2', [128, 1, 2], caller='fwd', Cin=832, Cout=128, H=64, KH=3, KW=3, N=8, W=128, dil=1, dw=True, dy=True, ldx=832, ldy=128, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 2], caller='fwd', Cin=512, Cout=2048, H=65, KH=1, KW=1, N=8, W=129, dil=1, dw=True, dy=True, ldx=512, ldy=2048, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 2], caller='fwd', Cin=2048, Cout=512, H=65, KH=1, KW=1, N=8, W=129, dil=1, dw=True, dy=True, ldx=2048, ldy=512, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 seg', [64, 1, 29], caller='fwd', Cin=64, Cout=128, H=256, KH=3, KW=3, N=8, W=512, dil=1, dw=True, dy=True, ldx=64, ldy=128, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2', [128, 1, 7], caller='fwd', Cin=1024, Cout=128, H=65, KH=3, KW=3, N=8, W=129, dil=1, dw=True, dy=True, ldx=1024, ldy=128, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2', [128, 1, 7], caller='fwd', Cin=256, Cout=512, H=65, KH=3, KW=3, N=8, W=129, dil=4, dw=True, dy=True, ldx=256, ldy=512, pad=4, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c4', [128, 1, 4], caller='fwd', Cin=512, Cout=512, H=46, KH=3, KW=3, N=16, W=61, dil=4, dw=True, dy=True, ldx=512, ldy=512, pad=4, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 1], caller='fwd', Cin=1024, Cout=2048, H=65, KH=1, KW=1, N=8, W=129, dil=1, dw=True, dy=True, ldx=1024, ldy=2048, pad=0, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'c2 seg', [128, 1, 4], caller='fwd', Cin=512, Cout=512, H=65, KH=3, KW=3, N=8, W=129, dil=4, dw=True, dy=True, ldx=512, ldy=512, pad=4, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 2], caller='fwd', Cin=1024, Cout=512, H=65, KH=3, KW=3, N=8, W=129, dil=1, dw=True, dy=True, ldx=1024, ldy=512, pad=1, stride=1, workspace=True, x=True),
    L('skd_conv2d_wgrad_sm100', 'seg', [128, 1, 1], caller='fwd', Cin=4096, Cout=512, H=65, KH=3, KW=3, N=8, W=129, dil=1, dw=True, dy=True, ldx=4096, ldy=512, pad=1, stride=1, workspace=True, x=True),
]

# Entry points and forms no training step launches: each is a synthetic row at a network-like shape.
SYNTHETIC = [
    # the affinity GEMM form with a fused double sum of squares, with and without an output tensor
    L("skd_gemm_nt_sm100", "synthetic", None, synthetic=True, M=2145, Ncols=2145, K=512, A=True, lda=512, B=True, D=True,
      ldd=2148, sumsq=True),
    L("skd_gemm_nt_sm100", "synthetic", None, synthetic=True, M=2145, Ncols=2145, K=512, A=True, lda=516, B=True,
      D=False, ldd=2145, sumsq=True),
    # general forward entry with explicit, distinct hi and lo operands (3xTF32), epilogue scale / shift / residual / leaky ReLU
    L("skd_conv2d_fwd_sm100_ex", "synthetic", None, synthetic=True, N=8, H=33, W=65, Cin=64, Cout=128, KH=3, KW=3,
      stride=1, pad=1, dil=1, x=True, x_lo=True, ldx=64, w=True, w_lo=True, y=True, ldy=136, out_h=0, out_w=0, scale=True, shift=True,
      residual=True, ldr=132, act=1, slope=0.1),
    # ELU epilogue with TF32-rounded output: no step takes it, the epilogue supports it
    L("skd_conv2d_fwd_sm100", "synthetic", None, synthetic=True, N=8, H=65, W=129, Cin=256, Cout=256, KH=3, KW=3,
      stride=1, pad=2, dil=2, x=True, ldx=256, w=True, y=True, ldy=256, scale=True, shift=True, residual=False, ldr=0, act=2, slope=0.0,
      round_tf32=1),
    # direct SIMT kernels, for channel counts that are not multiples of 4
    L("skd_conv2d_fwd_direct", "synthetic", None, synthetic=True, N=8, H=128, W=256, Cin=3, Cout=32, KH=3, KW=3, stride=2, pad=1, dil=1,
      x=True, ldx=3, w=True, y=True, ldy=32, scale=True, shift=True, act=3, slope=0.0),
    L("skd_conv2d_dgrad_direct", "synthetic", None, synthetic=True, N=8, H=65, W=129, Cin=19, Cout=21, KH=3, KW=3, stride=2, pad=1, dil=1,
      dy=True, ldy=21, w=True, dx=True, ldx=19),
    L("skd_conv2d_wgrad_direct", "synthetic", None, synthetic=True, N=8, H=65, W=129, Cin=19, Cout=21, KH=3, KW=3, stride=1, pad=1, dil=1,
      x=True, ldx=20, dy=True, ldy=21, dw=True),
]

# ops.conv2d_dgrad of a stride-2 convolution (one strided launch per input-pixel parity class): the student's stride-2 convolutions
S2_DGRAD = [
    # x shape, Cout, k, pad
    ((8, 64, 129, 257), 128, 3, 1),     # ResNet18 layer2.0.conv1
    ((8, 64, 129, 257), 128, 1, 0),     # ResNet18 layer2.0.downsample
    ((8, 32, 256, 512), 64, 3, 1),      # stem-class shape, even extents
    ((16, 20, 180, 240), 28, 3, 1),     # ESPNet-class shape
]

KNOBS = [("skd_set_conv_tile_m", 1), ("skd_set_conv_tile_m", 2), ("skd_set_conv_im2col", 0), ("skd_set_conv_k_order", 1),
         ("skd_set_conv_k_order", 2), ("skd_set_conv_tile_order", 1), ("skd_set_conv_tile_order", 2), ("skd_set_wgrad_linear", 0)]
KNOB_DEFAULT = {"skd_set_conv_tile_m": 0, "skd_set_conv_im2col": 1, "skd_set_conv_k_order": 0, "skd_set_conv_tile_order": 0,
                "skd_set_wgrad_linear": 1}


def _flop(e):
    if e["fn"] == "skd_conv1x1_chain_sm100":
        return e["P"] * e["Cout3"] * (e["Cin3"] + e["Cout1"])
    if e["fn"] == "skd_gemm_nt_sm100":
        return e["M"] * e["Ncols"] * e["K"]
    return e["N"] * e["H"] * e["W"] * e["Cin"] * e["Cout"] * e["KH"] * e["KW"]


def knob_subset(inv):
    """The cheapest row of every (entry point, plan) class: at least one launch per kernel path."""
    best = {}
    for e in inv:
        k = (e["fn"], tuple(e["plan"] or ()), e["fn"] == "skd_conv2d_fwd_sm100" and bool(e.get("residual")))
        if k not in best or _flop(e) < _flop(best[k]):
            best[k] = e
    return list(best.values())


def _rid(e):
    g = ("%s_%d_%dx%dx%d_%d_k%dx%d_s%d_p%d_d%d" % (e["fn"].replace("skd_", ""), e["N"], e["Cin"], e["H"], e["W"], e["Cout"], e["KH"], e["KW"],
                                                  e["stride"], e["pad"], e["dil"]) if "N" in e else
         "%s_%s" % (e["fn"].replace("skd_", ""), "_".join(str(e[k]) for k in ("P", "Cin3", "Cout3", "Cout1", "M", "Ncols", "K") if k in e)))
    return g + "_" + "-".join(e["steps"])


_IDS = []
for _e in INVENTORY + SYNTHETIC:
    _i, _n = _rid(_e), 1
    while _i in _IDS:
        _n += 1
        _i = "%s#%d" % (_rid(_e), _n)
    _IDS.append(_i)
INV_IDS = dict(zip(range(len(_IDS)), _IDS))


# ------------------------------------------------------------------------------------------------ GPU runners
def _nhwc(t, ld):
    """(N, C, H, W) integer tensor -> channels-last buffer of pitch ld (pitch tail NaN: a read of it poisons the result)."""
    n, c, h, w = t.shape
    buf = sentinel((n, h, w, ld), t.device)
    buf[..., :c] = t.permute(0, 2, 3, 1)
    return buf


def _vec(kind, c, gen, dev):
    if kind == "scale":                                  # powers of two: products stay exact
        return torch.pow(2.0, torch.randint(-1, 2, (c,), generator=gen, device=dev).float())
    return torch.randint(-8, 9, (c,), generator=gen, device=dev).float() / 4        # dyadic shifts


def _plan(L_, wgrad=False):
    o = (ctypes.c_int * (3 if wgrad else 7))()
    (L_.skd_conv_wgrad_last_plan if wgrad else L_.skd_conv_fwd_last_plan)(o)
    return list(o)


def _launch_twice(launch, make_out, check_plan, L_, wgrad=False):
    """Run a launch into two fresh sentinel-filled outputs; -> first output; the two must agree bit for bit."""
    outs = []
    for _ in range(2):
        o = make_out()
        launch(o)
        if check_plan is not None:
            assert _plan(L_, wgrad) == list(check_plan), ("plan", _plan(L_, wgrad), check_plan)
        outs.append(o)
    torch.cuda.synchronize()
    assert same_bits(outs[0], outs[1]), "two runs of the same launch differ"
    return outs[0]


def run_fwd(e, check_plan):
    from structure_knowledge_distillation_b200._cabi import lib
    L_, dev = lib(), "cuda"
    st = torch.cuda.current_stream().cuda_stream
    fn = e["fn"]
    N, H, W, Cin, Cout, KH, KW, s, p, d = (e[k] for k in ("N", "H", "W", "Cin", "Cout", "KH", "KW", "stride", "pad", "dil"))
    OH, OW = out_extent(H, W, KH, KW, s, p, d, e.get("out_h", 0), e.get("out_w", 0))
    three = bool(e.get("x_lo") or e.get("x_hi"))
    gen = torch.Generator(device=dev).manual_seed(Cin * 7 + Cout * 13 + H * 17 + W + KH)
    K = Cin * KH * KW
    terms = 3 * K if three else K
    xs = [operand(terms, (N, Cin, H, W), gen, dev) for _ in range(2 if three else 1)]
    ws = [operand(terms, (Cout, Cin, KH, KW), gen, dev) for _ in range(2 if three else 1)]
    xd, wd = [t.double() for t in xs], [t.double() for t in ws]
    pairs = [(0, 0), (1, 0), (0, 1)] if three else [(0, 0)]
    raw = sum(conv_ref(xd[i], wd[j], s, p, d, OH, OW) for i, j in pairs)
    check_premise(sum(conv_ref(xd[i].abs(), wd[j].abs(), s, p, d, OH, OW) for i, j in pairs))
    raw = exact_round(raw).float().permute(0, 2, 3, 1)                      # [N][OH][OW][Cout], exact in fp32
    ldx = e["ldx"]
    xb = [_nhwc(t, ldx) for t in xs]
    wb = [t.permute(0, 2, 3, 1).contiguous() for t in ws]
    scale = _vec("scale", Cout, gen, dev) if e.get("scale") else None
    shift = _vec("shift", Cout, gen, dev) if e.get("shift") else None
    res = None
    if e.get("residual"):
        res = _nhwc(ints((N, Cout, OH, OW), 8, gen, dev), e["ldr"])
    act, slope, rnd = e.get("act", 0), float(e.get("slope", 0.0)), e.get("round_tf32", 0)
    want = epilogue_ref(raw, scale, shift, None if res is None else res[..., :Cout], act, slope, rnd)
    P_ = lambda t: None if t is None else t.data_ptr()
    strided = "y_pix" in e
    if strided:
        ypix, yrow, yimg = e["y_pix"], e["y_row"], e["y_img"]
        size = (N - 1) * yimg + (OH - 1) * yrow + (OW - 1) * ypix + Cout
        make_out = lambda: sentinel((size,), dev)
        view = lambda o: o.as_strided((N, OH, OW, Cout), (yimg, yrow, ypix, 1))
    else:
        ldy = e["ldy"]
        make_out = lambda: sentinel((N, OH, OW, ldy), dev)
        view = lambda o: o[..., :Cout]
    ws_buf = None
    if fn == "skd_conv2d_fwd_sm100_splitk":
        nws = L_.skd_conv2d_fwd_sm100_splitk_workspace_floats(N, H, W, Cin, Cout, KH, KW, s, p, d, e["out_h"], e["out_w"])
        ws_buf = sentinel((max(nws, 4),), dev) if e.get("workspace") else None
    lo = (lambda l: P_(l[1])) if three else (lambda l: None)

    def launch(y):
        if fn == "skd_conv2d_fwd_sm100":
            L_.skd_conv2d_fwd_sm100(N, H, W, Cin, Cout, KH, KW, s, p, d, P_(xb[0]), ldx, P_(wb[0]), P_(y), ldy, P_(scale), P_(shift), P_(res),
                                    e["ldr"], act, slope, rnd, st)
        elif fn == "skd_conv2d_fwd_sm100_3xtf32":
            L_.skd_conv2d_fwd_sm100_3xtf32(N, H, W, Cin, Cout, KH, KW, s, p, d, P_(xb[0]), P_(xb[1]), ldx, P_(wb[0]), P_(wb[1]), P_(y), ldy,
                                           P_(scale), P_(shift), act, slope, st)
        elif fn == "skd_conv2d_fwd_sm100_ex":
            L_.skd_conv2d_fwd_sm100_ex(N, H, W, Cin, Cout, KH, KW, s, p, d, P_(xb[0]), lo(xb), ldx, P_(wb[0]), lo(wb), P_(y), ldy, e["out_h"],
                                       e["out_w"], P_(scale), P_(shift), P_(res), e["ldr"], act, slope, st)
        elif fn == "skd_conv2d_fwd_sm100_splitk":
            L_.skd_conv2d_fwd_sm100_splitk(N, H, W, Cin, Cout, KH, KW, s, p, d, P_(xb[0]), lo(xb), ldx, P_(wb[0]), lo(wb), P_(y), ldy,
                                           e["out_h"], e["out_w"], P_(scale), P_(shift), P_(res), e["ldr"], act, slope, P_(ws_buf),
                                           0 if ws_buf is None else ws_buf.numel(), st)
        elif fn == "skd_conv2d_fwd_sm100_strided":
            L_.skd_conv2d_fwd_sm100_strided(N, H, W, Cin, Cout, KH, KW, s, p, d, P_(xb[0]), ldx, P_(wb[0]), P_(y), ypix, yrow, yimg,
                                            e["out_h"], e["out_w"], rnd, st)
        else:
            L_.skd_conv2d_fwd_sm100_strided_3xtf32(N, H, W, Cin, Cout, KH, KW, s, p, d, P_(xb[0]), P_(xb[1]), ldx, P_(wb[0]), P_(wb[1]),
                                                   P_(y), ypix, yrow, yimg, st)

    y = _launch_twice(launch, make_out, check_plan, L_)
    got = view(y)
    assert not torch.isnan(got).any(), "output elements left unwritten: %d" % int(torch.isnan(got).sum())
    mask = torch.ones_like(y, dtype=torch.bool)
    view(mask).fill_(False)
    assert torch.isnan(y[mask]).all(), "elements outside the output were written: %d" % int((~torch.isnan(y[mask])).sum())
    assert_epilogue(got, want, act, fn)


def run_chain(e, check_plan):
    """y3 = relu(x3 w3 * scale3 + shift3 + residual), y1 = relu(y3 w1 * scale1 + shift1); y3 is an operand of the second GEMM, so
    its magnitude is kept within the TF32-exact range."""
    from structure_knowledge_distillation_b200._cabi import lib
    L_, dev = lib(), "cuda"
    st = torch.cuda.current_stream().cuda_stream
    P, Cin3, Cout3, Cout1 = e["P"], e["Cin3"], e["Cout3"], e["Cout1"]
    gen = torch.Generator(device=dev).manual_seed(P + Cin3 + Cout1)
    a3 = max(1, math.isqrt((TF32_EXACT - 24) // Cin3))
    x3, w3 = ints((P, Cin3), a3, gen, dev), ints((Cout3, Cin3), a3, gen, dev)
    sc3 = torch.ones(Cout3, device=dev)
    sh3 = torch.randint(-8, 9, (Cout3,), generator=gen, device=dev).float()
    res = ints((P, Cout3), 8, gen, dev)
    raw3 = exact_round(x3.double() @ w3.double().t())
    check_premise(x3.double().abs() @ w3.double().abs().t(), TF32_EXACT - 24)
    y3_ref = torch.relu(raw3.float() * sc3 + sh3 + res)
    assert float(y3_ref.abs().max()) <= TF32_EXACT
    a1 = max(1, amplitude(Cout3 * TF32_EXACT))
    w1 = ints((Cout1, Cout3), a1, gen, dev)
    sc1 = _vec("scale", Cout1, gen, dev)
    sh1 = _vec("shift", Cout1, gen, dev)
    raw1 = exact_round(y3_ref.double() @ w1.double().t())
    check_premise(y3_ref.double() @ w1.double().abs().t())
    y1_ref = torch.relu(raw1.float() * sc1 + sh1)
    xb = sentinel((P, e["ldx3"]), dev); xb[:, :Cin3] = x3
    alias = [tuple(a) for a in e.get("alias", [])]
    rb = sentinel((P, e["ldr"]), dev); rb[:, :Cout3] = res
    outs = []
    for _ in range(2):
        r = rb.clone()
        y3 = r if ("residual", "y3") in alias else sentinel((P, e["ldy3"]), dev)
        y1 = sentinel((P, e["ldy1"]), dev)
        L_.skd_conv1x1_chain_sm100(P, Cin3, Cout3, Cout1, xb.data_ptr(), e["ldx3"], w3.data_ptr(), sc3.data_ptr(), sh3.data_ptr(), r.data_ptr(),
                                   e["ldr"], y3.data_ptr(), e["ldy3"], w1.data_ptr(), sc1.data_ptr(), sh1.data_ptr(), y1.data_ptr(), e["ldy1"], st)
        outs.append((y3, y1))
    torch.cuda.synchronize()
    for i in range(2):
        assert same_bits(outs[0][i], outs[1][i]), "two runs differ"
    y3, y1 = outs[0]
    for t, c, ref, what in ((y3, Cout3, y3_ref, "y3"), (y1, Cout1, y1_ref, "y1")):
        assert not torch.isnan(t[:, :c]).any(), what
        assert torch.isnan(t[:, c:]).all(), what + ": pitch tail written"
        assert_epilogue(t[:, :c], ref, 3, what)


def run_wgrad(e, check_plan):
    """dw[co][kh][kw][ci] = sum over output pixels of dy * x: reductions over up to millions of pixels, so operands are +-1 (sparse
    where even that would pass 2^22)."""
    from structure_knowledge_distillation_b200._cabi import lib
    L_, dev = lib(), "cuda"
    st = torch.cuda.current_stream().cuda_stream
    fn = e["fn"]
    N, H, W, Cin, Cout, KH, KW, s, p, d = (e[k] for k in ("N", "H", "W", "Cin", "Cout", "KH", "KW", "stride", "pad", "dil"))
    OH, OW = out_extent(H, W, KH, KW, s, p, d)
    gen = torch.Generator(device=dev).manual_seed(Cin * 5 + Cout * 3 + H + W * 11)
    terms = N * OH * OW
    x = operand(terms, (N, Cin, H, W), gen, dev)
    dy = operand(terms, (N, Cout, OH, OW), gen, dev)
    ref = torch.nn.grad.conv2d_weight(x.double(), (Cout, Cin, KH, KW), dy.double(), stride=s, padding=p, dilation=d)
    check_premise(torch.nn.grad.conv2d_weight(x.double().abs(), (Cout, Cin, KH, KW), dy.double().abs(), stride=s, padding=p, dilation=d))
    want = exact_round(ref).float().permute(0, 2, 3, 1).contiguous()
    xb, dyb = _nhwc(x, e["ldx"]), _nhwc(dy, e["ldy"])
    wsb = None
    if fn == "skd_conv2d_wgrad_sm100":
        nws = L_.skd_conv2d_wgrad_sm100_workspace_floats(N, H, W, Cin, Cout, KH, KW, s, p, d)
        wsb = sentinel((max(nws, 4),), dev)

    def launch(dw):
        if fn == "skd_conv2d_wgrad_sm100":
            L_.skd_conv2d_wgrad_sm100(N, H, W, Cin, Cout, KH, KW, s, p, d, xb.data_ptr(), e["ldx"], dyb.data_ptr(), e["ldy"], dw.data_ptr(),
                                      wsb.data_ptr(), st)
        else:
            L_.skd_conv2d_wgrad_direct(N, H, W, Cin, Cout, KH, KW, s, p, d, xb.data_ptr(), e["ldx"], dyb.data_ptr(), e["ldy"], dw.data_ptr(), st)

    dw = _launch_twice(launch, lambda: sentinel((Cout, KH, KW, Cin), dev), check_plan, L_, wgrad=True)
    assert not torch.isnan(dw).any()
    assert_epilogue(dw, want, 0, fn)


def run_direct(e, check_plan):
    from structure_knowledge_distillation_b200._cabi import lib
    L_, dev = lib(), "cuda"
    st = torch.cuda.current_stream().cuda_stream
    N, H, W, Cin, Cout, KH, KW, s, p, d = (e[k] for k in ("N", "H", "W", "Cin", "Cout", "KH", "KW", "stride", "pad", "dil"))
    OH, OW = out_extent(H, W, KH, KW, s, p, d)
    gen = torch.Generator(device=dev).manual_seed(Cin + Cout + H)
    K = Cin * KH * KW
    w = operand(K * 4, (Cout, Cin, KH, KW), gen, dev)
    wb = w.permute(0, 2, 3, 1).contiguous()
    if e["fn"] == "skd_conv2d_fwd_direct":
        x = operand(K * 4, (N, Cin, H, W), gen, dev)
        raw = conv_ref(x.double(), w.double(), s, p, d, OH, OW)
        check_premise(conv_ref(x.double().abs(), w.double().abs(), s, p, d, OH, OW))
        sc, sh = _vec("scale", Cout, gen, dev), _vec("shift", Cout, gen, dev)
        want = epilogue_ref(exact_round(raw).float().permute(0, 2, 3, 1), sc, sh, None, e["act"], float(e["slope"]), 0)
        xb = _nhwc(x, e["ldx"])
        y = _launch_twice(lambda y: L_.skd_conv2d_fwd_direct(N, H, W, Cin, Cout, KH, KW, s, p, d, xb.data_ptr(), e["ldx"], wb.data_ptr(),
                                                             y.data_ptr(), e["ldy"], sc.data_ptr(), sh.data_ptr(), e["act"], float(e["slope"]), st),
                          lambda: sentinel((N, OH, OW, e["ldy"]), dev), None, L_)
        assert torch.isnan(y[..., Cout:]).all()
        assert_epilogue(y[..., :Cout], want, e["act"], e["fn"])
    else:
        dy = operand(Cout * KH * KW * 4, (N, Cout, OH, OW), gen, dev)
        ref = torch.nn.grad.conv2d_input((N, Cin, H, W), w.double(), dy.double(), stride=s, padding=p, dilation=d)
        check_premise(torch.nn.grad.conv2d_input((N, Cin, H, W), w.double().abs(), dy.double().abs(), stride=s, padding=p, dilation=d))
        want = exact_round(ref).float().permute(0, 2, 3, 1)
        dyb = _nhwc(dy, e["ldy"])
        dx = _launch_twice(lambda o: L_.skd_conv2d_dgrad_direct(N, H, W, Cin, Cout, KH, KW, s, p, d, dyb.data_ptr(), e["ldy"], wb.data_ptr(),
                                                                o.data_ptr(), e["ldx"], st),
                           lambda: sentinel((N, H, W, e["ldx"]), dev), None, L_)
        assert torch.isnan(dx[..., Cin:]).all()
        assert_epilogue(dx[..., :Cin], want, 0, e["fn"])


def run_gemm(e, check_plan):
    from structure_knowledge_distillation_b200._cabi import lib
    L_, dev = lib(), "cuda"
    st = torch.cuda.current_stream().cuda_stream
    M, Nc, K = e["M"], e["Ncols"], e["K"]
    gen = torch.Generator(device=dev).manual_seed(M + K)
    A, B = ints((M, K), 1, gen, dev), ints((Nc, K), 1, gen, dev)
    ref = exact_round(A.double() @ B.double().t())
    # fp32 squares summed over a row of a tile (up to 32 values) stay exact below 2^24; fp64 across rows and tiles below 2^53
    bound = A.double().abs() @ B.double().abs().t()
    check_premise(bound, 1 << 9)
    assert float((bound ** 2).sum()) < 2.0 ** 53
    want_sq = float((ref ** 2).sum())
    Ab = sentinel((M, e["lda"]), dev); Ab[:, :K] = A
    for _ in range(2):
        sq = torch.zeros(1, dtype=torch.float64, device=dev)
        D = sentinel((M, e["ldd"]), dev) if e["D"] else None
        L_.skd_gemm_nt_sm100(M, Nc, K, Ab.data_ptr(), e["lda"], B.data_ptr(), None if D is None else D.data_ptr(), e["ldd"], sq.data_ptr(), st)
        if check_plan is not None:
            assert _plan(L_) == list(check_plan)
        torch.cuda.synchronize()
        assert float(sq) == want_sq, (float(sq), want_sq)
        if D is not None:
            assert torch.isnan(D[:, Nc:]).all()
            assert_epilogue(D[:, :Nc], ref.float(), 0, "gemm_nt")


def run_row(e, check_plan=True):
    plan = e["plan"] if check_plan else None
    fn = e["fn"]
    if fn in FWD_FNS:
        run_fwd(e, plan)
    elif fn == "skd_conv1x1_chain_sm100":
        run_chain(e, plan)
    elif fn in ("skd_conv2d_wgrad_sm100", "skd_conv2d_wgrad_direct"):
        run_wgrad(e, plan)
    elif fn == "skd_gemm_nt_sm100":
        run_gemm(e, plan)
    else:
        run_direct(e, plan)


ROWS = INVENTORY + SYNTHETIC


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(ROWS)), ids=[INV_IDS[i] for i in range(len(ROWS))])
def test_launch_exact(i):
    run_row(ROWS[i])


@pytest.mark.gpu
@pytest.mark.parametrize("knob", KNOBS, ids=["%s=%d" % k for k in KNOBS])
def test_knob_matrix_exact(knob):
    from structure_knowledge_distillation_b200._cabi import lib
    name, val = knob
    rows = knob_subset(INVENTORY + SYNTHETIC)
    try:
        getattr(lib(), name)(val)
        for e in rows:
            run_row(e, check_plan=False)
    finally:
        getattr(lib(), name)(KNOB_DEFAULT[name])


@pytest.mark.gpu
@pytest.mark.parametrize("case", S2_DGRAD, ids=["%s_%d_k%d" % (c[0], c[1], c[2]) for c in S2_DGRAD])
def test_stride2_dgrad_exact(case):
    """ops.conv2d_dgrad of a stride-2 convolution: four strided launches, one per input-pixel parity class, must cover dx exactly."""
    from structure_knowledge_distillation_b200 import ops
    (N, Cin, H, W), Cout, k, pad = case
    dev = "cuda"
    gen = torch.Generator(device=dev).manual_seed(N + Cin + H + k)
    OH, OW = out_extent(H, W, k, k, 2, pad, 1)
    w = operand(Cout * k * k, (Cout, Cin, k, k), gen, dev)
    dy = operand(Cout * k * k, (N, Cout, OH, OW), gen, dev)
    ref = torch.nn.grad.conv2d_input((N, Cin, H, W), w.double(), dy.double(), stride=2, padding=pad)
    check_premise(torch.nn.grad.conv2d_input((N, Cin, H, W), w.double().abs(), dy.double().abs(), stride=2, padding=pad))
    want = exact_round(ref).float()
    dyb = ops.to_nhwc(dy)
    wb = w.permute(0, 2, 3, 1).contiguous()
    a = ops.conv2d_dgrad(dyb, wb, (N, Cin, H, W), 2, pad, 1)
    b = ops.conv2d_dgrad(dyb, wb, (N, Cin, H, W), 2, pad, 1)
    torch.cuda.synchronize()
    assert same_bits(a, b)
    assert_epilogue(a.permute(0, 2, 3, 1), want.permute(0, 2, 3, 1), 0, "stride-2 dgrad")


STEPS = {
    "c2": ("resnet18", 8, 512, 1024, "net"), "c4": ("resnet18", 16, 360, 480, "net"), "espc": ("espnet_c", 16, 360, 480, "net"),
    "esp": ("espnet", 16, 360, 480, "net"), "mnv2": ("mobilenetv2", 8, 512, 1024, "net"), "seg": ("resnet101", 8, 512, 1024, "seg"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("step", sorted(STEPS))
def test_inventory_is_complete(step):
    """One eager step with every convolution launch logged: each logged launch must be an INVENTORY row of that step."""
    from oracle import port
    from structure_knowledge_distillation_b200 import ops
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.networks.seg_model import SegModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    kind, b, h, w, which = STEPS[step]
    torch.manual_seed(0)
    if which == "net":
        m = NetModel(make_args(batch_size=b, pi=True, pa=True, ho=True, adv_loss_type="wgan-gp", student=kind, cuda_graph=False))
    else:
        m = SegModel(make_args(batch_size=b, seg_model=kind, cuda_graph=False))
    images, labels = port.synthetic_batch(b, h, w, seed=1)
    log = []
    try:
        m.set_input((images, labels, None, None))
        ops.CONV_EVENT_LOG = log
        m.optimize_parameters()
    finally:
        ops.CONV_EVENT_LOG = None
    torch.cuda.synchronize()
    rows = [e for e in INVENTORY if step in e["steps"]]
    keys = inventory_keys(rows)
    chains = [e for e in rows if e["fn"] == "skd_conv1x1_chain_sm100"]
    missing = sorted({r[3] for r in log if r[3] not in keys and not any(chain_matches(e, r[3]) for e in chains)}, key=str)
    assert not missing, "launches missing from INVENTORY: %s" % missing
    del m
    torch.cuda.empty_cache()
