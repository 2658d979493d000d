"""TEST INFRASTRUCTURE -- generates tests/golden/steps_769.pt: a distillation step of the UNMODIFIED reference at the standard
Cityscapes training crop, 769 x 769, on the CPU, with the ResNet18-PSP student and the PSPNet-101 teacher, pinning oracle/port.py
at that size on the spot.

    SKD_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_large_crop

Case (`LARGE_CROP_CASES`): batch 1, Pi + Pa + Ho wgan-gp.  The logits are 97 x 97, so the discriminator's first self-attention runs
over 144 positions and its second over 36 (the reference's `Discriminator(..., imsize_for_adv=65)` builds l4 at any size and its
attention is a plain bmm).  Same seeds and step order as oracle/make_golden.py's 19-class cases; every stored tensor goes through
`cases.sample_large`, so the fixture stays below 1 MB.  tests/test_large_crop_step_gpu.py checks NetModel against it.
"""
import os
import time

import torch

from . import cases, refshim
from .make_golden import GOLDEN_DIR, step_goldens

LARGE_CROP_CASES = {
    "pi_pa_ho_wgangp_769": dict(batch=1, h=769, w=769, cfg=dict(pi=True, pa=True, ho=True, adv_type="wgan-gp")),
}


def main():
    ref = refshim.load_reference()
    torch.set_num_threads(os.cpu_count())
    t0 = time.time()
    res = step_goldens(ref, LARGE_CROP_CASES, check_port=True)
    res = {name: {k: cases.sample_large(v) if torch.is_tensor(v) else v for k, v in g.items()} for name, g in res.items()}
    out = os.path.join(GOLDEN_DIR, "steps_769.pt")
    torch.save(res, out)
    print("wrote", out, os.path.getsize(out) // 1024, "KB", "%.1fs" % (time.time() - t0))


if __name__ == "__main__":
    main()
