"""`import modeling` for the UNMODIFIED reference scripts: the H100-native mirror under the reference's module name.

Put this directory on sys.path ahead of the reference tree (tools/run_reference_driver.py does) and
PyTorch/LanguageModeling/BERT/run_pretraining.py drives the sm_90a kernels without an edited line:
  * modeling.BertConfig / BertForPreTraining(config, sequence_output_is_dense=...) / .checkpoint_activations(...) -- same surface;
  * `model.half()` (run_pretraining.py:416-417) selects bfloat16 (modeling.BertPreTrainedModel.half);
  * pass the driver's own `--disable_jit_fusions` (custom autograd Functions are not TorchScript-able, SURVEY.md 8b);
  * `--cuda_graphs` needs a static number of gathered MLM rows, which the reference never passes to the model: this adapter reads
    the driver's own flags (--train_batch_size / --gradient_accumulation_steps / --max_predictions_per_seq) from sys.argv.
"""
import sys

from deeplearningexamples_b200.modeling import *  # noqa: F401,F403
from deeplearningexamples_b200 import modeling as _m
from deeplearningexamples_b200.modeling import (ACT2FN, BertConfig, BertEmbeddings, BertEncoder, BertForPreTraining,  # noqa: F401
                                                BertForQuestionAnswering, BertLayer, BertModel, BertPreTrainedModel, LinearActivation, gelu)


def _driver_flag(name, default):
    argv = sys.argv
    for i, a in enumerate(argv):
        if a == name and i + 1 < len(argv):
            return argv[i + 1]
        if a.startswith(name + "="):
            return a.split("=", 1)[1]
    return default


class BertForPreTraining(_m.BertForPreTraining):          # noqa: F811
    def __init__(self, config, sequence_output_is_dense=False):
        super().__init__(config, sequence_output_is_dense=sequence_output_is_dense)
        if sequence_output_is_dense and "--cuda_graphs" in sys.argv:
            bs = int(_driver_flag("--train_batch_size", 32)) // max(1, int(_driver_flag("--gradient_accumulation_steps", 1)))
            self.cls.static_masked_count = bs * int(_driver_flag("--max_predictions_per_seq", 80))
