"""Evaluation path and eval/train mode switching on the H100: evaluate_main (networks/evaluate.py:162-206) against a torch
restatement of the reference's numpy pipeline on the same class scores; the student's eval logits after training steps (the
folded BN of a TRAINABLE module must not be cached: ADVICE r1); eval-mode ABN backward (libs/functions.py:144-147)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


class _ToyNet(torch.nn.Module):
    """class scores at 1/8 resolution from plain torch ops: the evaluation kernels are what is under test"""

    def __init__(self, classes):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        self.w = torch.nn.Parameter(torch.randn(classes, 3, 1, 1, generator=g))

    def forward(self, x):
        return [F.conv2d(F.avg_pool2d(x, 8, 8, ceil_mode=True), self.w)]


@torch.no_grad()
def _reference_eval(net, batches, tile, classes, whole):
    conf = np.zeros((classes, classes))
    for image, label, size, _ in batches:
        H, W = image.shape[2:]
        if whole:
            out = F.interpolate(net(image.cuda())[0], size=tile, mode="bilinear", align_corners=True)[0].permute(1, 2, 0).double().cpu().numpy()
        else:
            from math import ceil
            stride = ceil(tile[0] * (1 - 1 / 3))
            rows, cols = int(ceil((H - tile[0]) / stride) + 1), int(ceil((W - tile[1]) / stride) + 1)
            full, cnt = np.zeros((H, W, classes)), np.zeros((H, W, classes))
            for r in range(rows):
                for c in range(cols):
                    x1, y1 = int(c * stride), int(r * stride)
                    x2, y2 = min(x1 + tile[1], W), min(y1 + tile[0], H)
                    x1, y1 = max(int(x2 - tile[1]), 0), max(int(y2 - tile[0]), 0)
                    img = image[:, :, y1:y2, x1:x2]
                    pad = torch.zeros(1, 3, tile[0], tile[1]); pad[:, :, :img.shape[2], :img.shape[3]] = img
                    p = F.interpolate(net(pad.cuda())[0], size=tile, mode="bilinear", align_corners=True)[0].permute(1, 2, 0).double().cpu().numpy()
                    full[y1:y2, x1:x2] += p[:img.shape[2], :img.shape[3]]; cnt[y1:y2, x1:x2] += 1
            out = full / cnt
        pred = np.argmax(out, axis=2)
        gt = label[0].numpy()[:size[0][0], :size[0][1]]
        pred = pred[:size[0][0], :size[0][1]]
        keep = gt != 255
        idx = gt[keep] * classes + pred[keep]
        conf += np.bincount(idx, minlength=classes * classes).reshape(classes, classes)
    pos, res, tp = conf.sum(1), conf.sum(0), np.diag(conf)
    iu = tp / np.maximum(1.0, pos + res - tp)
    return iu.mean(), iu


@pytest.mark.parametrize("whole", [False, True])
def test_evaluate_main_matches_reference_pipeline(whole):
    from structure_knowledge_distillation_b200.networks.evaluate import evaluate_main
    classes = 19
    net = _ToyNet(classes).cuda()
    g = torch.Generator().manual_seed(3)
    batches = []
    for i, (H, W) in enumerate(((1024, 2048), (1024, 2048)) if whole else ((100, 161), (64, 96), (130, 97))):
        image = torch.randn(1, 3, H, W, generator=g)
        label = torch.randint(0, classes, (1, H, W), generator=g)
        label[torch.rand(1, H, W, generator=g) < 0.1] = 255
        size = [np.array([H - (i % 2) * 3, W - (i % 2) * 5, 3])]
        batches.append((image, label, size, ["img%d" % i]))
    tile = (1024, 2048) if whole else (64, 96)
    got = evaluate_main(net, batches, 0, "64,96", classes, whole=whole)
    ref = _reference_eval(net, batches, tile, classes, whole)
    assert abs(got[0] - ref[0]) < 2e-4 and np.abs(got[1] - ref[1]).max() < 2e-3, (got[0], ref[0])     # fp32 ties at tile seams may flip a pixel


def test_student_eval_after_training_steps_is_not_stale():
    """eval -> N train steps -> eval: the second eval must see the updated BN statistics / affine parameters (written through raw
    pointers by the kernels) -- compared with a fresh model that loads the trained state dict."""
    from oracle import port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.networks.pspnet_combine import BasicBlock, Res_pspnet
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    torch.manual_seed(0)
    m = NetModel(make_args(batch_size=2, pi=True, pa=True, ho=False, lr_g=0.05))
    images, labels = port.synthetic_batch(2, 64, 96, seed=1)
    m.set_input((images, labels, None, None))
    x = images.cuda()
    with torch.no_grad():
        e0 = m.student.eval()(x)[0].clone()
    m.student.train()
    for _ in range(3):
        m.optimize_parameters()
    with torch.no_grad():
        e1 = m.student.eval()(x)[0].clone()
    fresh = Res_pspnet(BasicBlock, [2, 2, 2, 2], 19).cuda()
    fresh.load_state_dict(m.student.state_dict())
    with torch.no_grad():
        e2 = fresh.eval()(x)[0]
    assert float((e1 - e0).norm() / e0.norm()) > 1e-3                      # training changed the network ...
    assert float((e1 - e2).norm() / e2.norm()) < 1e-6                      # ... and eval sees exactly the trained state


def test_abn_eval_mode_backward_matches_reference_semantics():
    from oracle import port
    from structure_knowledge_distillation_b200.libs import InPlaceABN
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 32, 7, 9, generator=g)
    ref = port.ABN(32, activation="leaky_relu", slope=0.01).eval()
    with torch.no_grad():
        ref.running_mean.copy_(torch.randn(32, generator=g) * 0.2); ref.running_var.copy_(torch.rand(32, generator=g) + 0.5)
        ref.weight.copy_(torch.randn(32, generator=g)); ref.bias.copy_(torch.randn(32, generator=g) * 0.1)
    mine = InPlaceABN(32).cuda().eval()
    mine.load_state_dict(ref.state_dict())
    xr = x.clone().requires_grad_(True)
    dy = torch.randn(2, 32, 7, 9, generator=g)
    ref(xr).backward(dy)
    xm = x.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    mine(xm).backward(dy.cuda())
    assert float((xm.grad.cpu() - xr.grad).norm() / xr.grad.norm()) < 1e-5
    assert float(mine.weight.grad.abs().max()) == 0.0 and float(mine.bias.grad.abs().max()) == 0.0     # functions.py:144-147 quirk
    assert float(ref.weight.grad.abs().max()) == 0.0
