"""H100-native BERT-large pretraining hot path (NVIDIA/DeepLearningExamples PyTorch/LanguageModeling/BERT).

Public surface (mirrors the reference's module names):
  modeling    BertConfig, BertForPreTraining, BertModel, ... (same names / parameters / checkpoints)
  lamb        FusedLAMBAMP  (reference lamb_amp_opt.fused_lamb.FusedLAMBAMP)
  schedulers  PolyWarmUpScheduler
  kernels     torch-tensor wrappers over the C ABI in include/dle_b200.h (libdle_b200.so)
"""
__version__ = "0.1.0"
