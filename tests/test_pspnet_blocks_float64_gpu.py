"""The ResNet18-PSP student's layer Functions (functions.py: Conv2d, ABN with its fused ReLU / residual / Dropout2d, MaxPool3x3s2,
PspPool, PspAssemble) block by block, and the `frozen` forward of the student and of the ResNet101 teacher stage by stage, against
float64 with the TF32 operands and the inner activation masks pinned (oracle/pspnet_pinned.py).

Training path.  Each block runs the product's modules (networks/pspnet_combine.py) on channel-padded NHWC buffers as ResNet.forward
calls them, with cases.build_models' weights and perturbed BatchNorm, at the geometries of the benchmark step (batch 8 at 512x1024)
and of configuration 4 (batch 16 at 360x480), in train and in eval mode.  The reference is the port module in float64 on the GPU:
every backward convolution pinned, every forward the product runs in TF32 (layer3, layer4, PSP, DSN, head) pinned, the masks of
the ReLUs after the stem's and the BasicBlocks' bn1 and of the PSP stages' and DSN's LeakyReLU taken from the product's own float32
outputs.  A guard counts where those masks disagree with the float64 sign.  The report line of each block gives every error against
the pinned and against the plain float64 reference.

Frozen path.  ResNet._forward_frozen runs unchanged under no_grad (eval-mode ABN folded into the convolution epilogues, layer1-3
bottleneck pairs chained, layer4 writing into the PSP concat buffer); the eval-mode float64 port, every forward convolution pinned,
runs each stage from the product's float32 output of the stage before, so errors do not compound.

Guards record every call signature of these Functions in eager NetModel steps and of the `frozen` path in NetModel's teacher forward
and the evaluation forward of the student, and fail on one the tables here do not make.
"""
import copy
import sys
import time

import pytest
import torch

from test_student_blocks_float64_gpu import _fmt, _nhwc_leaf, _rel, _sub, _worst_channel

pytestmark = pytest.mark.gpu

# ---------------------------------------------------------------------------------------------- bounds
# Worst values over every block, mode and geometry, measured on one H100 80GB HBM3 (700 W), and DESIGN.md "PSPNet blocks against
# float64"; each bound is about 3x its worst value (strict: err < bound).  Forward outputs are float32-grade (3.3e-7) except in blocks
# with a 3x3 convolution whose forward is TF32 (layer3, layer4, PSP, DSN: up to 5.7e-5, "fwd3x3").  Their operands are rounded
# exactly as the reference rounds them (test_tf32_forward_rounds_operands_to_nearest_even, bit for bit); what remains is the
# tensor cores' float32 accumulation over K = 1 152 to 9 216, which truncates: one layer3 3x3 convolution alone is 5.3e-6 from the
# pinned reference, and 1.5e-6 from a model that truncates the float32 sum after every k8 step (the 1x1 head, K = 128: 3.0e-7).
# Train-mode BatchNorm, the ReLUs and the second convolution of a block carry that to the block's output.  Every gradient below
# such a forward inherits it, and the BatchNorm parameters inside a block see their gradient through the next convolution's TF32
# data gradient: affine 2.4e-4, one channel 4.3e-3; input gradients 1.6e-4; convolution weight gradients 3.0e-4, one channel
# 1.7e-3; running statistics 4.4e-6 (the mean, after such a forward).
BOUND = {"fwd": 1e-6, "fwd3x3": 2e-4, "stats": 1.5e-5, "affine": 1e-3, "affine[ch]": 1.5e-2, "dx": 5e-4, "conv": 1e-3, "conv[ch]": 5e-3}
# Every convolution weight gradient and the input gradient of every block with a convolution must be PIN_GAIN times closer to the
# pinned than to the plain float64 reference, and every frozen stage's output likewise.  The exceptions, at 2/3 of the smallest gain
# measured over geometries, modes and class counts (in the comment): gradients reached by the 3x3 TF32 forwards' truncated
# accumulation or summed over few pixels (the PSP stages' 1x1 to 6x6 maps), and the stem's and layer1-2's weight gradients over
# 0.5-1 M pixels of float32 accumulation; the frozen stages all contain 3x3 TF32 forwards (the head alone, 1x1, measures 250x).
# The gains below 2 cannot tell a kernel that truncates its operands from one that rounds them; the operand rounding of every TF32
# forward is checked bit for bit instead (test_tf32_forward_rounds_operands_to_nearest_even), and of the backward by the gains of
# the data gradients (70x and more wherever the forward above them is float32-grade).
PIN_GAIN = 10.0
PIN_GAIN_EXCEPTIONS = {
    ("dsn", "dsn.3.weight"): 4.6,                                      # 7.02
    ("layer1.0", "layer1.0.conv1.weight"): 5.8, ("layer1.0", "layer1.0.conv2.weight"): 4.7,       # 8.74, 7.15
    ("layer1.1", "dx0"): 5.9, ("layer1.1", "layer1.1.conv2.weight"): 4.1,                         # 8.94, 6.19
    ("layer2.0", "dx0"): 5.5, ("layer2.0", "layer2.0.conv1.weight"): 4.8,                         # 8.31, 7.27
    ("layer2.1", "dx0"): 6.0, ("layer2.1", "layer2.1.conv1.weight"): 6.1,                         # 9.09, 9.18
    ("layer3.0", "layer3.0.conv2.weight"): 4.0, ("layer3.0", "layer3.0.downsample.0.weight"): 6.1,  # 6.13, 9.27
    ("layer3.1", "layer3.1.conv2.weight"): 4.0,                                                   # 6.10
    ("layer4.0", "layer4.0.conv2.weight"): 2.9, ("layer4.0", "layer4.0.downsample.0.weight"): 4.7,  # 4.47, 7.09
    ("layer4.1", "layer4.1.conv2.weight"): 2.6,                                                   # 4.03
    ("pspmodule", "dx0"): 2.6, ("pspmodule", "pspmodule.bottleneck.0.weight"): 1.9,               # 3.95, 2.86
    ("pspmodule", "pspmodule.stages.0.1.weight"): 1.8, ("pspmodule", "pspmodule.stages.1.1.weight"): 1.2,  # 2.84, 1.87
    ("pspmodule", "pspmodule.stages.2.1.weight"): 2.2,                                            # 3.32
    ("stem", "conv1.weight"): 2.8, ("stem", "conv2.weight"): 1.6, ("stem", "conv3.weight"): 1.3,  # 4.32, 2.43, 2.01
    ("frozen:resnet101", "x1"): 2.6, ("frozen:resnet101", "x2"): 3.3, ("frozen:resnet101", "x3"): 1.0,   # 4.00, 5.02, 1.53
    ("frozen:resnet101", "x_dsn"): 1.9, ("frozen:resnet101", "x4"): 3.0, ("frozen:resnet101", "feat"): 3.2,  # 2.86, 4.53, 4.87
    ("frozen:resnet18", "x1"): 2.6, ("frozen:resnet18", "x2"): 5.1, ("frozen:resnet18", "x3"): 5.5,      # 3.99, 7.68, 8.28
    ("frozen:resnet18", "x_dsn"): 4.8, ("frozen:resnet18", "x4"): 3.6,                                   # 7.32, 5.44
}
ZERO_BIAS = 2.0               # |d bias_c| < ZERO_BIAS u sum |dz_c| for the DSN convolution's bias in train mode (worst 0.61)
# Pinned-mask disagreements with the float64 sign per activation and call (worst 63, in layer4.1), each at |z| < 5e-5 rms(z) of its
# layer (worst 1.6e-5): the pre-activations carry the 3x3 TF32 forwards' accumulation error above.  A wrong activation flips O(1) of them.
MASK_FLIPS, MASK_FLIP_Z = 200, 5e-5
FROZEN_BOUND = {"fwd": 5e-4, "fwd[ch]": 5e-3}                          # worst 1.7e-4 (ResNet101 x3), one channel 1.6e-3
U = 2.0 ** -24

GEOS = {"b8_512x1024": (8, 512, 1024), "b16_360x480": (16, 360, 480)}
CLASSES = (19, 21, 11)
SMALL = (2, 64, 96)                                                     # the guards' geometry (signatures do not depend on N, H, W)


def _conv_hw(n):
    return (n - 1) // 2 + 1


def _pool_hw(n):
    return -(-(n - 1) // 2) + 1                                         # MaxPool2d(3, 2, 1, ceil_mode=True)


class In:
    """One block input: `c` channels at (h, w); `grad`: it requires grad; `relu`: post-ReLU data (zeros tie in the max-pool)."""

    def __init__(self, c, h, w, grad=True, relu=False):
        self.c, self.h, self.w, self.grad, self.relu = c, h, w, grad, relu


class Block:
    """`prod(net, leaves)` -> the product's outputs; `ref(net64, leaves64)` -> the float64 outputs; `outs`: each output's logical
    width; `mods`: module paths whose parameters and buffers the block owns; `masks`: {pinned activation of the reference: the
    product module whose output gives its mask}; `dropout`: module paths of the Dropout2d whose keep-mask is injected."""

    def __init__(self, geo, classes, name, inputs, prod, ref, outs, mods, masks=None, dropout=(), linear_out=False):
        self.geo, self.classes, self.name, self.inputs, self.prod, self.ref = geo, classes, name, inputs, prod, ref
        self.outs, self.mods, self.masks, self.dropout, self.linear_out = outs, mods, masks or {}, tuple(dropout), linear_out


def blocks(geo, N, H, W):
    from structure_knowledge_distillation_b200 import functions as Fn, ops
    hs, ws = _conv_hw(H), _conv_hw(W)
    hp, wp = _pool_hw(hs), _pool_hw(ws)
    h8, w8 = _conv_hw(hp), _conv_hw(wp)

    def stem(n, L):
        x = ops.pad_channels(L[0], 4)
        x = n.bn1(n.conv1(x), fuse_relu=True)
        x = n.bn2(n.conv2(x), fuse_relu=True)
        return [n.bn3(n.conv3(x), fuse_relu=True)]

    def dsn(n, L):
        bn, drop = n.dsn[1], n.dsn[2]
        return [n.dsn[3](bn(n.dsn[0](L[0]), chan_mul=drop.channel_multiplier(L[0].shape[0], bn.num_features, L[0].device)))]

    def layer(path, cin, h, w):
        return Block(geo, 19, path, [In(cin, h, w)], lambda n, L: [_sub(n, path)(L[0])], lambda r, L: [_sub(r, path)(L[0])],
                     [_sub_out(path)], [path], masks={path + ".act1": path + ".bn1"})

    out = [Block(geo, 19, "stem", [In(3, H, W, grad=False)], stem, lambda r, L: [r.stem(L[0])], [128],
                 ["conv1", "bn1", "conv2", "bn2", "conv3", "bn3"], masks={"act1": "bn1", "act2": "bn2"}),
           Block(geo, 19, "maxpool", [In(128, hs, ws, relu=True)], lambda n, L: [Fn.MaxPool3x3s2.apply(L[0])],
                 lambda r, L: [r.maxpool(L[0])], [128], [], linear_out=True),
           layer("layer1.0", 128, hp, wp), layer("layer1.1", 64, hp, wp), layer("layer2.0", 64, hp, wp), layer("layer2.1", 128, h8, w8),
           layer("layer3.0", 128, h8, w8), layer("layer3.1", 256, h8, w8), layer("layer4.0", 256, h8, w8),
           layer("layer4.1", 512, h8, w8),
           Block(geo, 19, "pspmodule", [In(512, h8, w8)], lambda n, L: [n.pspmodule(L[0])], lambda r, L: [r.pspmodule(L[0])], [128],
                 ["pspmodule"], masks={"pspmodule.stages.%d.2" % i: "pspmodule.stages.%d.2" % i for i in range(4)},
                 dropout=["pspmodule.bottleneck.2"])]
    for c in CLASSES:
        out += [Block(geo, c, "dsn", [In(256, h8, w8)], dsn, lambda r, L: [r.dsn(L[0])], [c], ["dsn"], masks={"dsn.1": "dsn.1"},
                      dropout=["dsn.2"], linear_out=True),
                Block(geo, c, "head", [In(128, h8, w8)], lambda n, L: [n.head(L[0])], lambda r, L: [r.head(L[0])], [c], ["head"],
                      linear_out=True)]
    return out


def _sub_out(path):
    return {"layer1": 64, "layer2": 128, "layer3": 256, "layer4": 512}[path.split(".")[0]]


BLOCKS = [b for g, (N, H, W) in GEOS.items() for b in blocks(g, N, H, W)]
BLOCKS.sort(key=lambda b: CLASSES.index(b.classes))                     # one class count's networks at a time (stable sort)


# ---------------------------------------------------------------------------------------------- networks
_NETS = {}


def nets(classes):
    """-> (product ResNet18-PSP on the GPU, its float32 state, {pinned: float64 port on the GPU}).  pinned=True: backward and the
    product's TF32 forwards pinned; pinned=False: plain float64."""
    if classes not in _NETS:
        from oracle import cases, pspnet_pinned
        from structure_knowledge_distillation_b200.networks.pspnet_combine import BasicBlock, Res_pspnet
        _NETS.clear()
        torch.manual_seed(0)
        ref = cases.build_models(0, with_D=False, classes=classes)[1]
        state = {k: v.clone() for k, v in ref.state_dict().items()}
        prod = Res_pspnet(BasicBlock, [2, 2, 2, 2], classes).cuda()
        prod.load_state_dict(state)
        refs = {p: pspnet_pinned.pin_pspnet(copy.deepcopy(ref).cuda().double(), prod if p else None, pinned=p) for p in (True, False)}
        _NETS[classes] = (prod, state, refs)
    return _NETS[classes]


def _data(blk, N, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for i in blk.inputs:
        d = torch.randn(N, i.c, i.h, i.w, device="cuda", generator=g)
        out.append(d.clamp_min(0) if i.relu else d)
    return out


def _keep_masks(blk, net, N, seed):
    g = torch.Generator().manual_seed(seed)
    return {p: (torch.rand(N, _sub(net, p.rsplit(".", 1)[0])[1].num_features, generator=g) >= 0.1).float().cuda() for p in blk.dropout}


def _inject(net, keep):
    for p, k in keep.items():
        _sub(net, p).injected = k


def _output_gradients(blk, ref, state, data, training, seed):
    """n (standard normal) for a linear output, y n for one that ends in an activation (zero-mean either way; y n vanishes at the
    ReLU's kink), as in test_student_blocks_float64_gpu.  No mask of an earlier run is left set."""
    from oracle import pspnet_pinned
    pspnet_pinned.clear_masks(ref)
    ref.train(training if not blk.linear_out else False)
    with torch.no_grad():
        ys = blk.ref(ref, [d.double() for d in data])
    ref.load_state_dict(state)
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = [torch.randn(y.shape, device="cuda", dtype=torch.float64, generator=g) for y in ys]
    return [(z if blk.linear_out else y * z).float() for y, z in zip(ys, n)]


def _backward(outs, dys, pad):
    torch.autograd.backward(list(outs), [pad(dy, o) for o, dy in zip(outs, dys)])


def _run_product(blk, net, data, training, dys):
    """-> (leaves, outputs, {reference activation: mask from the product's float32 output})."""
    from structure_knowledge_distillation_b200 import ops
    net.train(training)
    got, hooks = {}, []
    for ref_path, prod_path in blk.masks.items():
        hooks.append(_sub(net, prod_path).register_forward_hook(
            lambda m, i, o, k=ref_path: got.__setitem__(k, (o.detach()[:, :m.num_features] > 0).clone())))
    try:
        leaves = [_nhwc_leaf(d, ops.pad4(i.c) if i.c != 3 else 3, i.grad) for d, i in zip(data, blk.inputs)]
        outs = blk.prod(net, leaves)
    finally:
        for h in hooks:
            h.remove()
    _backward(outs, dys, lambda dy, o: ops.pad_channels(dy, o.shape[1]) if o.shape[1] != dy.shape[1] else ops.to_nhwc(dy))
    torch.cuda.synchronize()
    return leaves, outs, got


def _run_ref(blk, ref, data, training, dys, masks):
    from oracle import pspnet_pinned
    acts = pspnet_pinned.pinned_acts(ref)
    pspnet_pinned.clear_masks(ref)
    for k, m in masks.items():
        acts[k].mask = m
    dz = {}

    def keep_dz(m, i, o):
        o.retain_grad()
        dz["o"] = o
    hook = None
    if blk.name == "dsn":                                               # d(dsn[0] out): the scale of the DSN bias's cancellation
        hook = ref.dsn[0].register_forward_hook(keep_dz)
    ref.train(training)
    try:
        leaves = [d.double().requires_grad_(i.grad) for d, i in zip(data, blk.inputs)]
        outs = blk.ref(ref, leaves)
        _backward(outs, dys, lambda dy, o: dy.double())
    finally:
        if hook is not None:
            hook.remove()
    return leaves, outs, {k: acts[k].z for k in masks}, (dz["o"].grad if dz else None)


def _kind(ref_mod, pname):
    """'conv' for the weight of a convolution (all TF32 in the backward), 'affine' for ABN parameters and convolution biases."""
    from oracle import student_pinned
    owner = _sub(ref_mod, pname.rsplit(".", 1)[0]) if "." in pname else ref_mod
    return ("conv" if isinstance(owner, student_pinned.PinnedConv2d) and pname.endswith("weight") else "affine"), 0


def _is_abn(ref_mod, pname):
    from oracle import port
    owner = _sub(ref_mod, pname.rsplit(".", 1)[0]) if "." in pname else ref_mod
    return isinstance(owner, port.ABN)


def run_block(blk, training, seed=0):
    """Runs one block three ways (product, pinned and plain float64); -> (report dict, list of violated checks)."""
    N = GEOS[blk.geo][0]
    prod, state, refs = nets(blk.classes)
    ref_p, ref_u = refs[True], refs[False]
    for net in (prod, ref_p, ref_u):
        net.load_state_dict(state)
        for p in net.parameters():
            p.grad = None
    keep = _keep_masks(blk, prod, N, seed + 7)
    for net in (prod, ref_p, ref_u):
        _inject(net, keep)
    data = _data(blk, N, seed)
    mods_p = [_sub(prod, m) for m in blk.mods]
    before = [{k: v.clone() for k, v in m.state_dict().items()} for m in mods_p]
    dys = _output_gradients(blk, ref_p, state, data, training, seed + 1)
    leaves_p, outs_p, masks = _run_product(blk, prod, data, training, dys)
    leaves_r, outs_r, zs, dz = _run_ref(blk, ref_p, data, training, dys, masks)
    leaves_u, _, _, _ = _run_ref(blk, ref_u, data, training, dys, {})
    _inject(prod, {p: None for p in keep})

    rep, bad = {}, []

    def check(key, err, bound):
        rep[key] = err
        if not err < bound:
            bad.append("%s %.3g >= %.3g" % (key, err, bound))

    def gain(key, e, eu):
        need = PIN_GAIN_EXCEPTIONS.get((blk.name, key), PIN_GAIN)
        rep[key + "_gain"] = eu / max(e, 1e-300)
        if not eu >= need * e:
            bad.append("%s: pinned error %.3g is not %gx below the unpinned %.3g" % (key, e, need, eu))

    # pinned-mask guard: where the product's mask and the float64 sign differ, |z| must be tiny (dropped DSN channels excepted)
    for k, m in masks.items():
        z = zs[k]
        diff = m != (z > 0)
        if blk.dropout and k.startswith("dsn"):
            diff &= keep["dsn.2"].to(diff.device).bool()[:, :, None, None]
        flips = int(diff.sum())
        rep["flips:" + k] = flips
        if flips:
            worst = float(z[diff].abs().max() / z.pow(2).mean().sqrt())
            rep["flipz:" + k] = worst
            if flips > MASK_FLIPS or worst > MASK_FLIP_Z:
                bad.append("%s: %d mask flips, worst |z| %.3g rms" % (k, flips, worst))

    tf32_3x3 = any(getattr(m, "pinned_forward", False) and m.kernel_size != (1, 1) for p in blk.mods for m in _sub(ref_p, p).modules())
    for k, (o, r, c) in enumerate(zip(outs_p, outs_r, blk.outs)):
        check("fwd%d" % k, _rel(o.detach()[:, :c], r.detach()), BOUND["fwd3x3" if tf32_3x3 else "fwd"])
        if not bool(torch.isfinite(o.detach()).all()):
            bad.append("output %d is not finite" % k)
        if o.shape[1] > c and not bool((o.detach()[:, c:] == 0).all()):
            bad.append("output %d pad channels are not 0" % k)
    has_conv = any(_kind(_sub(ref_p, m), n)[0] == "conv" for m in blk.mods for n, _ in _sub(ref_p, m).named_parameters())
    for k, (lp, lr, lu, i) in enumerate(zip(leaves_p, leaves_r, leaves_u, blk.inputs)):
        if not i.grad:
            continue
        if lp.grad is None:
            bad.append("input %d has no gradient" % k)
            continue
        e, eu = _rel(lp.grad[:, :i.c], lr.grad), _rel(lp.grad[:, :i.c], lu.grad)
        rep["dx%d" % k], rep["dx%d_unpinned" % k] = e, eu
        check("dx%d" % k, e, BOUND["dx"])
        if has_conv:
            gain("dx%d" % k, e, eu)
        if lp.grad.shape[1] > i.c and not bool((lp.grad[:, i.c:] == 0).all()):
            bad.append("input %d gradient pad channels are not 0" % k)
    for path, mp, b0 in zip(blk.mods, mods_p, before):
        mr, mu = _sub(ref_p, path), _sub(ref_u, path)
        pr, pu = dict(mr.named_parameters()), dict(mu.named_parameters())
        for name, p in mp.named_parameters():
            key = path + "." + name
            if p.grad is None:
                bad.append("%s has no gradient" % key)
                continue
            if not training and _is_abn(mr, name):                     # the reference's eval quirk: dweight = dbias = 0
                if bool((p.grad != 0).any()) or bool((pr[name].grad != 0).any()):
                    bad.append("%s: eval-mode ABN gradient is not exactly 0" % key)
                continue
            if training and key == "dsn.0.bias":                       # reaches the loss only through train-mode BN: cancels
                scale = U * dz.abs().sum((0, 2, 3))
                r = float((p.grad.double().abs() / scale).max())
                rep[key + "/uSum|dz|"] = r
                if not r < ZERO_BIAS:
                    bad.append("%s: %.3g u sum|dz| >= %g" % (key, r, ZERO_BIAS))
                continue
            kind, dim = _kind(mr, name)
            check(key, _rel(p.grad, pr[name].grad), BOUND[kind])
            check(key + "[ch]", _worst_channel(p.grad, pr[name].grad, dim), BOUND[kind + "[ch]"])
            if kind == "conv":
                rep[key + "_unpinned"] = eu = _rel(p.grad, pu[name].grad)
                gain(key, rep[key], eu)
        br = dict(mr.named_buffers())
        for name, v in mp.named_buffers():
            key = path + "." + name
            if not training:
                if not torch.equal(v, b0[name]):
                    bad.append("%s changed in eval mode" % key)
            elif name.endswith("num_batches_tracked"):
                if int(v) != int(br[name]):
                    bad.append("%s = %d, float64 %d" % (key, int(v), int(br[name])))
            else:
                check(key, _rel(v, br[name]), BOUND["stats"])
    return rep, bad


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("blk", BLOCKS, ids=lambda b: "%s-%d-%s" % (b.geo, b.classes, b.name))
def test_block_matches_pinned_float64(blk, training):
    t0 = time.time()
    rep, bad = run_block(blk, training)
    print("\nBLOCK %s %d %s %s %.1fs %s" % (blk.geo, blk.classes, blk.name, "train" if training else "eval", time.time() - t0,
                                          _fmt(rep)))
    assert not bad, bad


# ---------------------------------------------------------------------------------------------- TF32 operand rounding
# (Cin, Cout, k, stride, pad, dil, bias) of the TF32 forwards: ResNet18's layer3 / layer4 / PSP / DSN / head and ResNet101's
# bottleneck, dilated 3x3 and PSP convolutions; "stem": the small-Cin im2col route of the frozen stem.
TF32_FORWARDS = [(128, 256, 3, 1, 2, 2, False), (256, 256, 3, 1, 2, 2, False), (128, 256, 1, 1, 0, 1, False),
                 (256, 512, 3, 1, 4, 4, False), (512, 512, 3, 1, 4, 4, False), (512, 128, 1, 1, 0, 1, False),
                 (1024, 128, 3, 1, 1, 1, False), (256, 128, 3, 1, 1, 1, True), (128, 19, 1, 1, 0, 1, True),
                 (1024, 256, 1, 1, 0, 1, False), (2048, 512, 1, 1, 0, 1, False), (4096, 512, 3, 1, 1, 1, False), "stem"]


@pytest.mark.parametrize("case", TF32_FORWARDS, ids=repr)
def test_tf32_forward_rounds_operands_to_nearest_even(case):
    """The TF32 forward gives the same bits on raw operands as on operands rounded to TF32 by round-to-nearest-even beforehand
    (pa_pinned.tf32_rn), so the reference's conv(tf32_rn(x), tf32_rn(w)) is exactly what the tensor cores multiply, and it gives other
    bits on operands truncated to TF32.  What remains of the forward error against the pinned reference is the accumulation."""
    from oracle.pa_pinned import tf32_rn
    from structure_knowledge_distillation_b200 import functions as Fn, ops
    g = torch.Generator(device="cuda").manual_seed(11)
    if case == "stem":
        cin, cout, k, s, p, d, bias = 3, 64, 3, 2, 1, 1, False
    else:
        cin, cout, k, s, p, d, bias = case
    x = torch.randn(2, cin, 33, 47, device="cuda", generator=g).clamp_min(0) * 3.0
    w = torch.randn(cout, cin, k, k, device="cuda", generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, device="cuda", generator=g) if bias else None

    def run(xx, ww):
        ww = ww.contiguous(memory_format=torch.channels_last)
        if case == "stem":
            return Fn.conv_forward_small_cin(ops.pad_channels(xx, 4), ww, s, p, d)[0].contiguous()
        return Fn.conv_forward_padded(ops.to_nhwc(xx), ww, b, s, p, d)[0].contiguous()

    def trunc(t):
        return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)
    raw = run(x, w)
    assert torch.equal(raw, run(tf32_rn(x.contiguous()), tf32_rn(w.contiguous())))
    assert not torch.equal(raw, run(trunc(x), trunc(w)))


# ---------------------------------------------------------------------------------------------- the frozen forward, stage by stage
# (network, classes, batch, H, W, mirrored second image): NetModel's teacher at both step geometries, evaluate's student forward of a
# whole 1024x2048 image alone and with its mirror, a 512x512 VOC crop and a 360x480 CamVid image.
FROZEN_CASES = [("resnet101", 19, 8, 512, 1024, False), ("resnet101", 19, 16, 360, 480, False),
                ("resnet18", 19, 1, 1024, 2048, False), ("resnet18", 19, 2, 1024, 2048, True),
                ("resnet18", 21, 1, 512, 512, False), ("resnet18", 11, 1, 360, 480, False)]
STAGES = ("x1", "x2", "x3", "x_dsn", "x4", "feat", "logits")


def frozen_nets(arch, classes):
    """-> (product network, frozen as NetModel / evaluate hold it, {pinned: eval-mode float64 port, every forward pinned or none})."""
    from oracle import cases, pspnet_pinned
    from structure_knowledge_distillation_b200.networks.pspnet_combine import BasicBlock, Bottleneck, Res_pspnet
    torch.manual_seed(0)
    teacher, student, _ = cases.build_models(0, with_D=False, classes=classes)
    ref = teacher if arch == "resnet101" else student
    prod = (Res_pspnet(Bottleneck, [3, 4, 23, 3], classes) if arch == "resnet101" else Res_pspnet(BasicBlock, [2, 2, 2, 2], classes))
    prod.load_state_dict(ref.state_dict())
    prod = prod.cuda().eval()
    if arch == "resnet101":
        for p in prod.parameters():
            p.requires_grad_(False)                                     # NetModel's teacher (folds cached)
    refs = {p: pspnet_pinned.pin_pspnet(copy.deepcopy(ref).cuda().double().eval(), prod if p else None, frozen=True)
            for p in (True, False)}
    return prod, refs


def _image(N, H, W, mirror):
    x = torch.randn(1 if mirror else N, 3, H, W, generator=torch.Generator().manual_seed(3)).cuda() * 40.0
    return torch.cat([x, x.flip(3)]) if mirror else x


def _frozen_stages(r, img, outs):
    """The float64 stages, each from the product's float32 output of the stage before."""
    x, x_dsn, feat, x4, x3, x2, x1 = [o.double() for o in outs]
    return {"x1": r.layer1(r.maxpool(r.stem(img.double()))), "x2": r.layer2(x1), "x3": r.layer3(x2), "x_dsn": r.dsn(x3),
            "x4": r.layer4(x3), "feat": r.pspmodule(x4), "logits": r.head(feat)}


@pytest.mark.parametrize("case", FROZEN_CASES, ids=lambda c: "%s-%d-b%d-%dx%d%s" % (c[:5] + ("-mirror" if c[5] else "",)))
def test_frozen_forward_stages_match_pinned_float64(case):
    arch, classes, N, H, W, mirror = case
    t0 = time.time()
    prod, refs = frozen_nets(arch, classes)
    img = _image(N, H, W, mirror)
    with torch.no_grad():
        outs = prod(img)
        got = dict(zip(("logits", "x_dsn", "feat", "x4", "x3", "x2", "x1"), [o.float() for o in outs]))
        torch.cuda.synchronize()
        rep, bad = {}, []
        want = {p: _frozen_stages(r, img, outs) for p, r in refs.items()}
    for k in STAGES:
        g, w, wu = got[k], want[True][k], want[False][k]
        if not bool(torch.isfinite(g).all()):
            bad.append("%s is not finite" % k)
        e, eu, ch = _rel(g, w), _rel(g, wu), _worst_channel(g, w, 1)
        rep[k], rep[k + "[ch]"], rep[k + "_unpinned"] = e, ch, eu
        if not e < FROZEN_BOUND["fwd"]:
            bad.append("%s %.3g >= %.3g" % (k, e, FROZEN_BOUND["fwd"]))
        if not ch < FROZEN_BOUND["fwd[ch]"]:
            bad.append("%s[ch] %.3g >= %.3g" % (k, ch, FROZEN_BOUND["fwd[ch]"]))
        need = PIN_GAIN_EXCEPTIONS.get(("frozen:" + arch, k), PIN_GAIN)
        if not eu >= need * e:
            bad.append("%s: pinned error %.3g is not %gx below the unpinned %.3g" % (k, e, need, eu))
    print("\nFROZEN %s %d b%d %dx%d%s %.1fs %s" % (arch, classes, N, H, W, " mirror" if mirror else "", time.time() - t0, _fmt(rep)))
    del prod, refs, want, outs
    torch.cuda.empty_cache()
    assert not bad, bad


# ---------------------------------------------------------------------------------------------- completeness guards
LAYER_FNS = ("Conv2d", "ABN", "MaxPool3x3s2", "PspPool", "PspAssemble")
DIRECT = ("skd_conv2d_fwd_direct", "skd_conv2d_dgrad_direct", "skd_conv2d_wgrad_direct")
NET_FILES = ("networks/pspnet_combine.py", "test_pspnet_blocks_float64_gpu.py")


def _pitch(t):
    from structure_knowledge_distillation_b200 import ops
    return ops.nhwc_meta(t)[4]


def _route(x, w, b, precise):
    """The forward route Fn.Conv2d.forward takes."""
    from structure_knowledge_distillation_b200 import functions as Fn
    if Fn._small_cin(w) and b is None and not x.requires_grad:
        return "small-cin 3xtf32" if precise else "small-cin tf32"
    if precise and w.shape[0] % 4 == 0 and w.shape[1] % 4 == 0 and _pitch(x) == x.shape[1]:
        return "3xtf32"
    return "tf32"


def _call_signature(name, a):
    """Channels, pitches, strides, dilations, flags and route of one layer-Function call -- none of N, H, W."""
    if name == "Conv2d":
        x, w, b, stride, pad, dil, precise = (list(a) + [False])[:7]
        return (name, x.shape[1], _pitch(x), tuple(w.shape), stride, pad, dil, b is not None, bool(precise), _route(x, w, b, precise))
    if name == "ABN":
        x, training, act, slope, res, cm = a[0], a[5], a[8], a[9], a[10], a[11]
        return (name, x.shape[1], _pitch(x), bool(training), act, slope, None if res is None else _pitch(res), cm is not None)
    if name == "MaxPool3x3s2":
        return (name, a[0].shape[1], _pitch(a[0]))
    if name == "PspPool":
        return (name, a[0].shape[1], _pitch(a[0]), tuple(a[1]))
    if name == "PspAssemble":
        return (name, a[0].shape[1], _pitch(a[0]), tuple(a[1]), tuple(tuple(s.shape[1:]) for s in a[2:]))
    raise KeyError(name)


def _from_network():
    f = sys._getframe(2)
    while f is not None and ("/torch/" in f.f_code.co_filename or f.f_code.co_filename.endswith(("functions.py", "libs/bn.py"))):
        f = f.f_back
    return f is not None and f.f_code.co_filename.replace("\\", "/").endswith(NET_FILES)


def record_layer_calls(monkeypatch, fn):
    """Run fn() logging the signature of every layer-Function call made from pspnet_combine.py (or the block table), and every direct
    SIMT convolution launched inside such a call's forward or backward; -> (signatures, direct launches)."""
    from structure_knowledge_distillation_b200 import functions as Fn
    from structure_knowledge_distillation_b200._cabi import lib
    seen, direct, active = set(), [], []
    for name in LAYER_FNS:
        cls = getattr(Fn, name)
        fwd, bwd = cls.forward, cls.backward

        def forward(ctx, *args, _fwd=fwd, _name=name):
            ctx._net = _from_network()
            if ctx._net:
                seen.add(_call_signature(_name, args))
                active.append(_name)
            try:
                return _fwd(ctx, *args)
            finally:
                if ctx._net:
                    active.pop()

        def backward(ctx, *grads, _bwd=bwd, _name=name):
            if ctx._net:
                active.append(_name + ".backward")
            try:
                return _bwd(ctx, *grads)
            finally:
                if ctx._net:
                    active.pop()
        monkeypatch.setattr(cls, "forward", staticmethod(forward))
        monkeypatch.setattr(cls, "backward", staticmethod(backward))
    L = lib()
    for name in DIRECT:
        orig = getattr(L, name)

        def launch(*args, _orig=orig, _name=name):
            if active:
                direct.append((active[-1], _name, args[:10]))
            return _orig(*args)
        monkeypatch.setattr(L, name, launch)
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        monkeypatch.undo()
    return seen, direct


def _net_step(batch, h, w, classes):
    from oracle import port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    torch.manual_seed(0)
    m = NetModel(make_args(batch_size=batch, pi=True, pa=True, ho=True, adv_loss_type="wgan-gp", classes_num=classes))
    images, labels = port.synthetic_batch(batch, h, w, seed=1, classes=classes)
    m.set_input((images, labels, None, None))
    m.optimize_parameters()
    torch.cuda.synchronize()
    return m


def test_block_table_covers_every_training_layer_call(monkeypatch):
    """Every layer-Function call from pspnet_combine.py in one eager NetModel step (the benchmark's configuration, configuration 4,
    21 and 11 classes) has a block with the same signature, and none launches a direct SIMT convolution."""
    table = set()
    for blk in blocks("small", *SMALL):
        for training in (True, False):
            def one():
                prod, state, _ = nets(blk.classes)
                prod.load_state_dict(state)
                _inject(prod, _keep_masks(blk, prod, SMALL[0], 0))
                data = _data(blk, SMALL[0], 0)
                prod.train(training)
                from structure_knowledge_distillation_b200 import ops
                leaves = [_nhwc_leaf(d, ops.pad4(i.c) if i.c != 3 else 3, i.grad) for d, i in zip(data, blk.inputs)]
                outs = blk.prod(prod, leaves)
                torch.autograd.backward(outs, [torch.ones_like(o) for o in outs])
                _inject(prod, {p: None for p in blk.dropout})
            s, d = record_layer_calls(monkeypatch, one)
            assert not d, (blk.name, d)
            table |= s
    for batch, h, w, classes in ((8, 512, 1024, 19), (16, 360, 480, 19), (2, 512, 512, 21), (2, 360, 480, 11)):
        holder = []
        seen, direct = record_layer_calls(monkeypatch, lambda: holder.append(_net_step(batch, h, w, classes)))
        del holder
        torch.cuda.empty_cache()
        assert seen, (batch, h, w, classes)
        missing = sorted(seen - table, key=repr)
        assert not missing, ((batch, h, w, classes), missing)
        assert not direct, ((batch, h, w, classes), direct[:8])


def record_frozen_calls(monkeypatch, fn):
    """Run fn() logging the signature of every `frozen`-path call made from pspnet_combine.py: Conv2d.frozen, ops.conv1x1_chain,
    ops.psp_pool_fwd, ops.psp_upsample_fwd, ops.maxpool_fwd."""
    from structure_knowledge_distillation_b200 import ops
    from structure_knowledge_distillation_b200.networks import pspnet_combine as pc
    seen = set()
    frozen = pc.Conv2d.frozen

    def conv_frozen(self, x, scale=None, shift=None, residual=None, act="none", slope=0.0, out=None):
        seen.add(("Conv2d.frozen", x.shape[1], _pitch(x), tuple(self.weight.shape), self.stride, self.padding, self.dilation,
                  self.bias is not None, scale is not None, None if residual is None else _pitch(residual), act, slope,
                  None if out is None else _pitch(out)))
        return frozen(self, x, scale, shift, residual, act, slope, out)
    monkeypatch.setattr(pc.Conv2d, "frozen", conv_frozen)

    def logged(name, sig):
        orig = getattr(ops, name)

        def f(*a, **k):
            if sys._getframe(1).f_code.co_filename.replace("\\", "/").endswith("networks/pspnet_combine.py"):
                seen.add((name,) + sig(*a, **k))
            return orig(*a, **k)
        monkeypatch.setattr(ops, name, f)
    logged("conv1x1_chain", lambda x3, w3, s3, h3, res, w1, *r, **k: (x3.shape[1], _pitch(x3), tuple(w3.shape), _pitch(res),
                                                                       tuple(w1.shape)))
    logged("psp_pool_fwd", lambda x, sizes: (x.shape[1], _pitch(x), tuple(sizes)))
    logged("psp_upsample_fwd", lambda st, s, out, off: (tuple(st.shape[1:]), s, out.shape[1], _pitch(out), off))
    logged("maxpool_fwd", lambda x: (x.shape[1], _pitch(x)))
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        monkeypatch.undo()
    return seen


def test_frozen_table_covers_the_teacher_and_evaluation_forwards(monkeypatch):
    """Every `frozen`-path call signature of NetModel's teacher forward (benchmark configuration, configuration 4) and of evaluate's
    student forward (a 1024x2048 image alone and with its mirror at 19 classes, a 512x512 image at 21 and a 360x480 one at 11) is one
    the frozen stage cases make."""
    from oracle import port
    from structure_knowledge_distillation_b200.networks.evaluate import _scores, zoom_image
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    table = set()
    for arch, classes, N, H, W, mirror in FROZEN_CASES:
        prod, _ = frozen_nets(arch, classes)
        table |= record_frozen_calls(monkeypatch, lambda: _scores(prod, _image(N, H, W, mirror)))
        del prod
    seen = set()
    for batch, h, w, classes in ((8, 512, 1024, 19), (16, 360, 480, 19), (1, 512, 512, 21), (1, 360, 480, 11)):
        torch.manual_seed(0)
        m = NetModel(make_args(batch_size=batch, pi=True, pa=True, ho=False, classes_num=classes))
        if classes == 19:                                               # the teacher at the two step geometries
            images = port.synthetic_batch(batch, h, w, seed=1, classes=classes)[0].cuda()
            with torch.no_grad():
                seen |= record_frozen_calls(monkeypatch, lambda: m.teacher.eval()(images))
        s = m.student.eval()
        image = torch.randn(1, 3, h * 2 if classes == 19 else h, w * 2 if classes == 19 else w,
                            generator=torch.Generator().manual_seed(3)).cuda() * 40.0
        for flip in (False, True):
            seen |= record_frozen_calls(monkeypatch, lambda: _scores(s, zoom_image(image, 1.0, flip)))
        del m, s
        torch.cuda.empty_cache()
    assert seen
    missing = sorted(seen - table, key=repr)
    assert not missing, missing


# ---------------------------------------------------------------------------------------------- the training step's setup
SIDE = ("layer1.0", "layer2.0", "pspmodule", "dsn", "head")


@pytest.mark.parametrize("name", SIDE)
def test_block_bits_with_side_stream_wgrad_and_direct_grads(name, monkeypatch):
    """NetModel's step runs Conv2d with its weight gradients on WgradOverlap's side stream, written straight into FlatSGD's flat
    gradient buffer (direct_grads=True).  A block run that way gives the plain run's outputs and gradients bit for bit; the
    convolutions whose channel counts are multiples of 4 take that route (the downsamples, the PSP stages, the DSN's 3x3), the
    19-class DSN classifier and head do not."""
    from oracle import cases
    from structure_knowledge_distillation_b200 import functions as Fn, ops
    from structure_knowledge_distillation_b200.networks.pspnet_combine import BasicBlock, Res_pspnet
    from structure_knowledge_distillation_b200.optim import FlatSGD
    geo = "b16_360x480"
    blk = next(b for b in BLOCKS if b.geo == geo and b.classes == 19 and b.name == name)
    N = GEOS[geo][0]
    torch.manual_seed(0)
    state = cases.build_models(0, with_D=False, classes=19)[1].state_dict()
    data = _data(blk, N, 5)
    g = torch.Generator(device="cuda").manual_seed(6)
    runs = []
    for overlap in (False, True):
        net = Res_pspnet(BasicBlock, [2, 2, 2, 2], 19).cuda()
        net.load_state_dict(state)
        net.train(True)
        _inject(net, _keep_masks(blk, net, N, 8))
        params = [p for m in blk.mods for p in _sub(net, m).parameters()]
        names = {id(p): m + "." + n for m in blk.mods for n, p in _sub(net, m).named_parameters()}
        written = []
        if overlap:
            opt = FlatSGD(params, lr=0.01, direct_grads=True)
            opt.zero_grad()
            monkeypatch.setattr(Fn, "_grad_written", lambda p, _w=written: _w.append(names[id(p)]))
        leaves = [_nhwc_leaf(d, ops.pad4(i.c), i.grad) for d, i in zip(data, blk.inputs)]
        outs = blk.prod(net, leaves)
        if not runs:
            dys = [torch.randn(o.shape, device="cuda", generator=g) for o in outs]
        if overlap:
            Fn.WgradOverlap.begin()
        try:
            torch.autograd.backward(outs, [ops.pad_channels(d, o.shape[1]) if o.shape[1] != d.shape[1] else ops.to_nhwc(d)
                                           for o, d in zip(outs, dys)])
        finally:
            if overlap:
                Fn.WgradOverlap.end()
                monkeypatch.undo()
        torch.cuda.synchronize()
        if overlap:
            convs = {names[id(p)] for p in params if p.dim() == 4}
            direct = {k for k in written if k in convs}
            want = {names[id(p)] for p in params if p.dim() == 4 and p.shape[0] % 4 == 0 and p.shape[1] % 4 == 0}
            assert direct == want, (sorted(direct), sorted(want))
            assert {"layer1.0.downsample.0.weight", "layer2.0.downsample.0.weight", "dsn.0.weight"} & convs <= direct
            assert all(k in direct for k in convs if ".stages." in k)
            assert not any(k in direct for k in ("dsn.3.weight", "head.weight"))
        runs.append(([o.detach().clone() for o in outs], [lf.grad.clone() for lf in leaves if lf.grad is not None],
                     [p.grad.clone() for p in params], [b.clone() for m in blk.mods for b in _sub(net, m).buffers()]))
    for a, b in zip(*runs):
        for x, y in zip(a, b):
            assert torch.equal(x, y)
