"""The `args` fields NetModel reads (utils/train_options.py:16-83), with the reference's defaults and the values its
launch script sets (run_train_val.sh:8-25).  No argparse side effects (the reference creates log dirs at parse time)."""
import argparse

import torch

DEFAULTS = dict(
    data_set='cityscape', classes_num=19, T_ckpt_path='', S_resume=True, S_ckpt_path='', D_resume=True, D_ckpt_path='',
    batch_size=8, start_epoch=0, epoch_nums=1, parallel='True', input_size='512,512', momentum=0.9, num_steps=40000,
    power=0.9, snapshot_dir='', weight_decay=5e-4, gpu='0', last_step=0, is_student_load_imgnet=False,
    student_pretrain_model_imgnet='None', pi=True, pa=True, ho=True, adv_loss_type='wgan-gp', imsize_for_adv=65,
    adv_conv_dim=64, lambda_gp=10.0, lambda_d=0.1, lambda_pi=10.0, lambda_pa=0.5, pool_scale=0.5, preprocess_GAN_mode=1,
    lr_g=1e-2, lr_d=4e-4, best_mean_IU=0.0, gpu_num=1,
    cuda_graph=False,        # ours: capture the step into CUDA graphs after 3 eager steps (NetModel.enable_cuda_graphs)
    ohem=False, ohem_thres=0.7, ohem_keep=100000,   # ours: CriterionOhemDSN(thresh=ohem_thres, min_kept=ohem_keep) as the CE term
    class_weights=None,      # ours: per-class weights of the task cross entropy (e.g. dataset.class_frequency_weights), not with ohem
    student='resnet18', espnet_p=2, espnet_q=8,     # ours: 'resnet18' (ResNet18-PSP), 'espnet_c' (ESPNet-C with p / q ESP blocks), 'espnet' (ESPNet-C + decoder) or 'mobilenetv2' (dilated MobileNetV2 + PSP head)
    at=False, lambda_at=500.0, mimic=False, lambda_mimic=1.0,   # ours: attention-transfer / MIMIC feature terms; a scalar weight: the PSP features, a list: one per level like lambda_pa
    pa_window=None, pa_dilation=1,   # ours: local pair-wise term, each pooled node against its pa_window x pa_window neighbours at pa_dilation (None: fully connected); scalars or lists like lambda_pa
    cwd=False, lambda_cwd=3.0, lambda_cwd_feat=None, cwd_tau=4.0,   # ours: channel-wise distillation on the logits (lambda_cwd) and on feature levels (lambda_cwd_feat: None, or lambda_at's form), one temperature
    ifv=False, lambda_ifv=200.0)   # ours: intra-class feature variation distillation, lambda_at's form (a scalar: the PSP features); 200 is a starting value, not tuned here


def make_args(**overrides):
    d = dict(DEFAULTS); d.update(overrides)
    ns = argparse.Namespace(**d)
    ns.device = torch.device("cuda")
    return ns
