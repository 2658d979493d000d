"""Cost of 21 classes (PASCAL VOC) against 19 (Cityscapes): the ResNet18 distillation step (batch 8 at 512x512, Pi+Pa+Ho wgan-gp,
CUDA graphs) with the two class counts alternated within one run, the DSN cross entropy (forward + backward, the loss kernels whose
class loop is compiled for 19 and for up to 32 classes) at that shape, and the augmentation kernel on a batch of VOC-sized raw images
(500x375 and 375x500) cropped to 512x512.

    python -m tools.voc_step_bench --steps 20 --warmup 5 --rounds 3

Prints the card name and power limit (read in the same run) and one JSON line.  Random weights and inputs: the rates do not depend
on the values."""
import argparse
import json
import random

import numpy as np
import torch

from tools.espnet_step_bench import _time, card


def step_rate(classes, batch, steps, warmup):
    from oracle import port
    from structure_knowledge_distillation_b200.networks.kd_model import NetModel
    from structure_knowledge_distillation_b200.utils.train_options import make_args
    m = NetModel(make_args(classes_num=classes, batch_size=batch, pi=True, pa=True, ho=True, adv_loss_type="wgan-gp", cuda_graph=True))
    images, labels = port.synthetic_batch(batch, 512, 512, seed=1, classes=classes)
    m.set_input((images, labels, None, None))
    for _ in range(warmup):
        m.optimize_parameters()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        m.optimize_parameters()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    del m
    torch.cuda.empty_cache()
    return batch * 1000.0 / ms, ms


def dsn_ce_ms(classes, batch):
    """CriterionDSN forward + backward on two (batch, classes, 65, 65) NHWC logit maps against 512x512 labels."""
    from structure_knowledge_distillation_b200.utils.criterion import CriterionDSN
    g = torch.Generator(device="cuda").manual_seed(classes)
    xs = [torch.randn(batch, classes, 65, 65, device="cuda", generator=g).contiguous(memory_format=torch.channels_last).requires_grad_(True)
          for _ in range(2)]
    labels = torch.randint(0, classes, (batch, 512, 512), device="cuda", generator=g)
    crit = CriterionDSN()
    return _time(lambda: crit(xs, labels).backward(), 100)


def augment_ms(batch):
    """DeviceAugment (voc=True) on `batch` raw VOC-sized images, VOC scale draws, 512x512 crops."""
    from structure_knowledge_distillation_b200.dataset import VOC_SCALES, DeviceAugment, draw_augmentation
    rng = np.random.default_rng(0)
    shapes = [(375, 500) if i % 2 else (500, 375) for i in range(batch)]
    imgs = [torch.from_numpy(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).cuda() for h, w in shapes]
    labs = [torch.from_numpy(rng.integers(0, 21, (h, w), dtype=np.uint8)).cuda() for h, w in shapes]
    random.seed(0); np.random.seed(0)
    augs = torch.tensor([draw_augmentation(h, w, (512, 512), True, True, VOC_SCALES) for h, w in shapes], dtype=torch.float64)
    aug = DeviceAugment((512, 512), (128, 128, 128), voc=True)
    return _time(lambda: aug(imgs, labs, augs), 200)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=8)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = dict(card=card(), batch=a.batch, shape="512x512", losses="Pi+Pa+Ho wgan-gp", student="resnet18", cuda_graph=True,
               classes19=[], classes21=[])
    for _ in range(a.rounds):
        for c in (19, 21):
            ips, ms = step_rate(c, a.batch, a.steps, a.warmup)
            res["classes%d" % c].append(dict(images_per_s=round(ips, 2), ms_per_step=round(ms, 2)))
    res["dsn_ce_fwd_bwd_ms"] = {str(c): [round(dsn_ce_ms(c, a.batch), 4) for _ in range(3)] for c in (19, 21)}
    res["augment_ms_batch_voc_500x375_to_512x512"] = [round(augment_ms(a.batch), 4) for _ in range(3)]
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
