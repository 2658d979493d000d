"""structure_knowledge_distillation_b200 -- Hopper-native structured-distillation training step.

Drop-in for the hot path of irfanICMLL/structure_knowledge_distillation: `networks.kd_model.NetModel` and the
`utils.criterion` loss classes keep the reference's names and call signatures; underneath, thin
torch.autograd.Functions call hand-written sm_90a CUDA through the C ABI of include/skd.h (libskd_b200.so).
There is no CPU or library fallback: importing an op without the built library raises.
"""
__version__ = "0.1.0"
