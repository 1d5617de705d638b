"""H100-native BERT: the reference's `modeling` interface over hand-written sm_90a kernels.

Mirrors PyTorch/LanguageModeling/BERT/modeling.py of NVIDIA/DeepLearningExamples: the same class names,
constructor and forward signatures, sub-module / parameter names and shapes (= the checkpoint format:
`bert.encoder.layer.{i}.attention.self.{query,key,value}.{weight,bias}`, `...intermediate.dense_act...`),
so reference checkpoints load with load_state_dict and `torch.save(model.state_dict())` round-trips into
the reference's run_squad.py.  What differs is underneath (ops.py / csrc/):

  BertSelfAttention  modeling.py:304-384  -> one packed-QKV wgmma GEMM + fused attention kernel
  BertSelfOutput     modeling.py:387-398  -> GEMM with bias+dropout+residual epilogue + LayerNorm kernel
  BertIntermediate   modeling.py:413-420  -> GEMM with bias+tanh-GELU epilogue
  BertOutput         modeling.py:423-434  -> as BertSelfOutput
  BertEmbeddings     modeling.py:263-301  -> gather+sum+LayerNorm(+dropout) kernel
  BertPreTrainingHeads :577-595           -> row-gather kernel + the same GEMM/LN kernels

The model computes in bf16 (parameters bf16, or fp32 with cached bf16 copies); there is no CPU path --
calling forward with CPU tensors raises.  The model is not TorchScript-able (custom autograd functions):
run the reference driver with its own `--disable_jit_fusions` flag.
"""
import copy
import json
import math
import sys
from collections import OrderedDict

import torch
from torch import nn
from torch.nn import init
from torch.nn.parameter import Parameter
from torch.utils import checkpoint

from . import _lib as L
from . import ops

bf16 = torch.bfloat16


def gelu(x):
    """tanh-approximated GELU (reference modeling.py:121-122)."""
    return torch.nn.functional.gelu(x, approximate="tanh")


def swish(x):
    return x * torch.sigmoid(x)


ACT2FN = {"gelu": gelu, "tanh": torch.tanh, "relu": torch.nn.functional.relu, "swish": swish}
_FUSED_ACTS = {"gelu": "gelu", "tanh": "tanh"}


# ---------------------------------------------------------------------------------------------------
# layout helpers: modules accept [..., H]; kernels see [tokens, H] in *memory* order
# ---------------------------------------------------------------------------------------------------
def _require_cuda(t, what):
    if not t.is_cuda:
        raise L.DleError(f"{what}: expected a CUDA tensor -- the H100 hot path has no CPU fallback")


def _tokens(x):
    """x [d0, d1, H] (or [T, H]) -> (x2d in memory order, restore(y2d) -> tensor shaped like x, transposed_view: bool)."""
    _require_cuda(x, "hidden_states")
    if x.dtype != bf16:
        x = x.to(bf16)
    if x.dim() == 2:
        x2 = x if x.stride(1) == 1 else x.contiguous()
        return x2, (lambda y: y), False
    if x.dim() != 3:
        x = x.reshape(-1, x.shape[-2], x.shape[-1])
    d0, d1, H = x.shape
    if x.is_contiguous():
        return x.view(d0 * d1, H), (lambda y: y.view(d0, d1, y.shape[-1])), False
    xt = x.transpose(0, 1)
    if xt.is_contiguous():      # e.g. the encoder's [S,B,H] view of a [B,S,H] buffer (reference modeling.py:498)
        return xt.reshape(d1 * d0, H), (lambda y: y.view(d1, d0, y.shape[-1]).transpose(0, 1)), True
    xc = x.contiguous()
    return xc.view(d0 * d1, H), (lambda y: y.view(d0, d1, y.shape[-1])), False


def _tokens_like(x, transposed):
    """2-D view of a second tensor in the same token order as the first one."""
    if x.dtype != bf16:
        x = x.to(bf16)
    if x.dim() == 2:
        return x if x.stride(1) == 1 else x.contiguous()
    H = x.shape[-1]
    if transposed:
        return x.transpose(0, 1).contiguous().view(-1, H) if not x.transpose(0, 1).is_contiguous() else x.transpose(0, 1).reshape(-1, H)
    return x.contiguous().view(-1, H)


class LinearActivation(nn.Module):
    """Fused Linear + activation (reference modeling.py:130-166); bias+activation run in the GEMM epilogue."""
    __constants__ = ['bias']

    def __init__(self, in_features, out_features, act='gelu', bias=True):
        super().__init__()
        self.in_features = in_features
        self.out_features = out_features
        assert act in ACT2FN, "Activation function is not found in activation dictionary."
        self.act = act
        self.act_fn = ACT2FN[act]
        self.weight = Parameter(torch.empty(out_features, in_features))
        if bias:
            self.bias = Parameter(torch.empty(out_features))
        else:
            self.register_parameter('bias', None)
        self.reset_parameters()

    def reset_parameters(self):
        init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if self.bias is not None:
            fan_in, _ = init._calculate_fan_in_and_fan_out(self.weight)
            bound = 1 / math.sqrt(fan_in)
            init.uniform_(self.bias, -bound, bound)

    def forward(self, input):
        x2, restore, _ = _tokens(input)
        fused = _FUSED_ACTS.get(self.act)
        y = ops.LinearFn.apply(x2, self.weight, self.bias, fused)
        if fused is None:
            y = self.act_fn(y)
        return restore(y)

    def extra_repr(self):
        return 'in_features={}, out_features={}, bias={}'.format(self.in_features, self.out_features, self.bias is not None)


class BertConfig(object):
    """Configuration of a `BertModel`: an attribute bag that round-trips through JSON.

    Same constructor contract as the reference class (modeling.py:168-261): the first argument is either the vocabulary size (the
    remaining hyper-parameters then come from keyword arguments / defaults) or the path of a JSON file whose keys become attributes.
    `from_dict` / `from_json_file` / `to_dict` / `to_json_string` / `to_json_file` behave as there.
    """
    _DEFAULTS = (("hidden_size", 768), ("num_hidden_layers", 12), ("num_attention_heads", 12), ("intermediate_size", 3072),
                 ("hidden_act", "gelu"), ("hidden_dropout_prob", 0.1), ("attention_probs_dropout_prob", 0.1),
                 ("max_position_embeddings", 512), ("type_vocab_size", 2), ("initializer_range", 0.02),
                 ("output_all_encoded_layers", False))

    def __init__(self, vocab_size_or_config_json_file, **hyper):
        unknown = set(hyper) - {k for k, _ in self._DEFAULTS}
        if unknown:
            raise TypeError("unexpected BertConfig arguments: %s" % sorted(unknown))
        if isinstance(vocab_size_or_config_json_file, str):
            with open(vocab_size_or_config_json_file, "r", encoding="utf-8") as fh:
                self.__dict__.update(json.load(fh))
        elif isinstance(vocab_size_or_config_json_file, int):
            self.vocab_size = vocab_size_or_config_json_file
            for key, default in self._DEFAULTS:
                setattr(self, key, hyper.get(key, default))
        else:
            raise ValueError("First argument must be either a vocabulary size (int)"
                             "or the path to a pretrained model config file (str)")

    @classmethod
    def from_dict(cls, json_object):
        config = cls(vocab_size_or_config_json_file=-1)
        config.__dict__.update(json_object)
        return config

    @classmethod
    def from_json_file(cls, json_file):
        with open(json_file, "r", encoding="utf-8") as fh:
            return cls.from_dict(json.load(fh))

    def to_dict(self):
        return copy.deepcopy(self.__dict__)

    def to_json_string(self):
        return json.dumps(self.to_dict(), indent=2, sort_keys=True) + "\n"

    def to_json_file(self, json_file_path):
        with open(json_file_path, "w", encoding="utf-8") as fh:
            fh.write(self.to_json_string())

    def __repr__(self):
        return self.to_json_string()


class BertEmbeddings(nn.Module):
    """word + position + token-type embeddings, LayerNorm, dropout (reference modeling.py:263-301)."""

    def __init__(self, config):
        super().__init__()
        self.word_embeddings = nn.Embedding(config.vocab_size, config.hidden_size)
        self.position_embeddings = nn.Embedding(config.max_position_embeddings, config.hidden_size)
        self.token_type_embeddings = nn.Embedding(config.type_vocab_size, config.hidden_size)
        self.LayerNorm = nn.LayerNorm(config.hidden_size, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)
        self.distillation = getattr(config, 'distillation', False)
        if self.distillation:
            self.distill_state_dict = OrderedDict()
            self.distill_config = config.distillation_config
        else:
            self.distill_config = {'use_embedding_states': False}
        self._stream_id = ops.new_stream_id()

    def forward(self, input_ids, token_type_ids):
        _require_cuda(input_ids, "input_ids")
        B, S = input_ids.shape
        p = self.dropout.p if self.training else 0.0
        y = ops.EmbeddingLNFn.apply(input_ids, token_type_ids, self.word_embeddings.weight, self.position_embeddings.weight,
                                    self.token_type_embeddings.weight, self.LayerNorm.weight, self.LayerNorm.bias,
                                    p, self.LayerNorm.eps, self._stream_id)
        embeddings = y.view(B, S, -1)
        if self.distillation and self.distill_config["use_embedding_states"]:
            self.distill_state_dict["embedding_states"] = embeddings
        return embeddings


class BertSelfAttention(nn.Module):
    """Multi-head self-attention (reference modeling.py:304-384).  The three nn.Linear parameters keep their
    checkpoint names but live in ONE packed [3H,H] / [3H] storage, so a single GEMM produces q|k|v."""

    def __init__(self, config):
        super().__init__()
        if config.hidden_size % config.num_attention_heads != 0:
            raise ValueError("The hidden size (%d) is not a multiple of the number of attention heads (%d)"
                             % (config.hidden_size, config.num_attention_heads))
        self.num_attention_heads = config.num_attention_heads
        self.attention_head_size = int(config.hidden_size / config.num_attention_heads)
        self.all_head_size = self.num_attention_heads * self.attention_head_size
        self.query = nn.Linear(config.hidden_size, self.all_head_size)
        self.key = nn.Linear(config.hidden_size, self.all_head_size)
        self.value = nn.Linear(config.hidden_size, self.all_head_size)
        self.dropout = nn.Dropout(config.attention_probs_dropout_prob)
        self.distillation = getattr(config, 'distillation', False)
        if self.distillation:
            self.distill_state_dict = OrderedDict()
            self.distill_config = config.distillation_config
        else:
            self.distill_config = {'use_attention_scores': False, 'use_value_states': False}
        self._stream_id = ops.new_stream_id()

    # -- packed parameter storage ------------------------------------------------------------------
    def _packed(self):
        """(w [3H,H], b [3H]) views over the q/k/v parameters' shared storage; repacks if a module conversion
        (.to / .bfloat16 / .float) gave each parameter its own storage again."""
        ws = [self.query.weight, self.key.weight, self.value.weight]
        bs = [self.query.bias, self.key.bias, self.value.bias]
        out = []
        for ps in (ws, bs):
            p0 = ps[0]
            esz, n = p0.element_size(), p0.numel()
            adjacent = all(p.dtype == p0.dtype and p.is_contiguous() for p in ps) and \
                ps[1].data_ptr() == p0.data_ptr() + n * esz and ps[2].data_ptr() == p0.data_ptr() + 2 * n * esz and \
                p0.untyped_storage().nbytes() - p0.storage_offset() * esz >= 3 * n * esz
            if not adjacent:
                with torch.no_grad():
                    packed = torch.cat([p.data.reshape(p0.shape) for p in ps], 0).contiguous()
                    rows = p0.shape[0]
                    for i, p in enumerate(ps):
                        p.data = packed[i * rows:(i + 1) * rows]
            p0 = ps[0]
            shape = (3 * p0.shape[0],) + tuple(p0.shape[1:])
            out.append(p0.data.as_strided(shape, p0.stride()))
        return out[0], out[1]

    def transpose_for_scores(self, x):
        return x.view(x.size(0), x.size(1) * self.num_attention_heads, self.attention_head_size).transpose(0, 1)

    def transpose_key_for_scores(self, x):
        return x.view(x.size(0), x.size(1) * self.num_attention_heads, self.attention_head_size).permute(1, 2, 0)

    def forward(self, hidden_states, attention_mask):
        """hidden_states (seq, bsz, hidden); attention_mask additive, broadcastable [bsz,1,1,seq] or None."""
        if self.attention_head_size != 64:
            raise L.DleError("the fused attention kernel is built for head size 64")
        if self.distillation and (self.distill_config["use_attention_scores"] or self.distill_config["use_value_states"]):
            raise L.DleError("distillation hooks need the materialised score tensor, which the fused kernel never forms")
        S, B, H = hidden_states.shape
        x2, restore, transposed = _tokens(hidden_states)
        seq_first = not transposed
        mask = None
        if attention_mask is not None:
            mask = attention_mask.reshape(B, S).to(torch.float32).contiguous()
        w, b = self._packed()
        p = self.dropout.p if self.training else 0.0
        ctx = ops.SelfAttentionFn.apply(x2, self.query.weight, self.key.weight, self.value.weight, self.query.bias,
                                        self.key.bias, self.value.bias, w, b, mask, B, S, self.num_attention_heads, p,
                                        self._stream_id, seq_first)
        return restore(ctx)


class _DenseDropoutAddLN(nn.Module):
    def __init__(self, in_features, config):
        super().__init__()
        self.dense = nn.Linear(in_features, config.hidden_size)
        self.LayerNorm = nn.LayerNorm(config.hidden_size, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)
        self._stream_id = ops.new_stream_id()

    def forward(self, hidden_states, input_tensor):
        x2, restore, transposed = _tokens(hidden_states)
        r2 = _tokens_like(input_tensor, transposed)
        p = self.dropout.p if self.training else 0.0
        y = ops.DenseDropoutAddLNFn.apply(x2, r2, self.dense.weight, self.dense.bias, self.LayerNorm.weight,
                                          self.LayerNorm.bias, p, self.LayerNorm.eps, self._stream_id)
        return restore(y)


class BertSelfOutput(_DenseDropoutAddLN):
    """LayerNorm(dropout(dense(x)) + input) (reference modeling.py:387-398)."""

    def __init__(self, config):
        super().__init__(config.hidden_size, config)


class BertAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.self = BertSelfAttention(config)
        self.output = BertSelfOutput(config)

    def forward(self, input_tensor, attention_mask):
        self_output = self.self(input_tensor, attention_mask)
        return self.output(self_output, input_tensor)


class BertIntermediate(nn.Module):
    """gelu(dense(x)) (reference modeling.py:413-420)."""

    def __init__(self, config):
        super().__init__()
        self.dense_act = LinearActivation(config.hidden_size, config.intermediate_size, act=config.hidden_act)

    def forward(self, hidden_states):
        return self.dense_act(hidden_states)


class BertOutput(_DenseDropoutAddLN):
    """LayerNorm(dropout(dense(x)) + input) over the FFN width (reference modeling.py:423-434)."""

    def __init__(self, config):
        super().__init__(config.intermediate_size, config)


class BertLayer(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.attention = BertAttention(config)
        self.intermediate = BertIntermediate(config)
        self.output = BertOutput(config)
        self.distillation = getattr(config, 'distillation', False)
        if self.distillation:
            self.distill_state_dict = OrderedDict()
            self.distill_config = config.distillation_config
        else:
            self.distill_config = {'use_hidden_states': False}

    def _fusable(self):
        att = self.attention.self
        return (not self.distillation and not att.distillation and att.attention_head_size == 64
                and self.intermediate.dense_act.act == "gelu" and self.intermediate.dense_act.bias is not None
                and not getattr(self, "force_modular", False))

    def forward(self, hidden_states, attention_mask):
        """hidden_states (seq, bsz, hidden) -> (seq, bsz, hidden).  Default: one hand-differentiated autograd node for
        the whole layer (ops.BertLayerFn); the module-by-module composition below computes the same function."""
        if self._fusable():
            att, so, it, out = self.attention.self, self.attention.output, self.intermediate.dense_act, self.output
            S, B, H = hidden_states.shape
            x2, restore, transposed = _tokens(hidden_states)
            mask = None if attention_mask is None else attention_mask.reshape(B, S).to(torch.float32).contiguous()
            w_qkv, b_qkv = att._packed()
            tr = self.training
            cfg = (B, S, att.num_attention_heads, att.dropout.p if tr else 0.0, so.dropout.p if tr else 0.0, so.LayerNorm.eps,
                   att._stream_id, so._stream_id, out._stream_id, not transposed)
            y = ops.BertLayerFn.apply(x2, mask, att.query.weight, att.key.weight, att.value.weight, att.query.bias, att.key.bias,
                                      att.value.bias, so.dense.weight, so.dense.bias, so.LayerNorm.weight, so.LayerNorm.bias,
                                      it.weight, it.bias, out.dense.weight, out.dense.bias, out.LayerNorm.weight, out.LayerNorm.bias,
                                      w_qkv, b_qkv, cfg)
            return restore(y)
        attention_output = self.attention(hidden_states, attention_mask)
        intermediate_output = self.intermediate(attention_output)
        layer_output = self.output(intermediate_output, attention_output)
        if self.distillation and self.distill_config["use_hidden_states"]:
            self.distill_state_dict["hidden_states"] = layer_output
        return layer_output


class BertEncoder(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.layer = nn.ModuleList([BertLayer(config) for _ in range(config.num_hidden_layers)])
        self.output_all_encoded_layers = config.output_all_encoded_layers
        self._checkpoint_activations = False

    def checkpointed_forward(self, hidden_states, attention_mask):
        """sqrt(L)-chunk activation recomputation (reference modeling.py:471-489).  Unlike the reference branch,
        the layers still receive (seq, bsz, hidden) -- the reference skips that transpose here, a latent quirk."""
        def custom(start, end):
            state = {}

            def custom_forward(*inputs):
                # replay the same dropout seeds when the chunk is recomputed in backward
                saved = None
                if "counter" in state:
                    saved = ops._rng["counter"]
                    ops._rng["counter"] = state["counter"]
                else:
                    state["counter"] = ops._rng["counter"]
                x_ = inputs[0]
                for layer in self.layer[start:end]:
                    x_ = layer(x_, inputs[1])
                if saved is not None:
                    ops._rng["counter"] = saved
                return x_
            return custom_forward

        l, num_layers = 0, len(self.layer)
        chunk_length = math.ceil(math.sqrt(num_layers))
        hidden_states = hidden_states.transpose(0, 1)
        while l < num_layers:
            hidden_states = checkpoint.checkpoint(custom(l, l + chunk_length), hidden_states, attention_mask * 1,
                                                  use_reentrant=False)
            l += chunk_length
        return hidden_states.transpose(0, 1).contiguous()

    def forward(self, hidden_states, attention_mask):
        all_encoder_layers = []
        if self._checkpoint_activations:
            hidden_states = self.checkpointed_forward(hidden_states, attention_mask)
        else:
            # (bsz, seq, hidden) => (seq, bsz, hidden): a VIEW; the kernels read the batch-first memory in place
            hidden_states = hidden_states.transpose(0, 1)
            for layer_module in self.layer:
                hidden_states = layer_module(hidden_states, attention_mask)
                if self.output_all_encoded_layers:
                    all_encoder_layers.append(hidden_states)
            hidden_states = hidden_states.transpose(0, 1).contiguous()     # no copy: already batch-first in memory
        if not self.output_all_encoded_layers or self._checkpoint_activations:
            all_encoder_layers.append(hidden_states)
        return all_encoder_layers


class BertPooler(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense_act = LinearActivation(config.hidden_size, config.hidden_size, act="tanh")

    def forward(self, hidden_states):
        return self.dense_act(hidden_states[:, 0])


class BertPredictionHeadTransform(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense_act = LinearActivation(config.hidden_size, config.hidden_size, act=config.hidden_act)
        self.LayerNorm = nn.LayerNorm(config.hidden_size, eps=1e-12)

    def forward(self, hidden_states):
        hidden_states = self.dense_act(hidden_states)
        x2, restore, _ = _tokens(hidden_states)
        return restore(ops.LayerNormFn.apply(x2, self.LayerNorm.weight, self.LayerNorm.bias, self.LayerNorm.eps))


class BertLMPredictionHead(nn.Module):
    def __init__(self, config, bert_model_embedding_weights):
        super().__init__()
        self.transform = BertPredictionHeadTransform(config)
        # output weights are tied to the input embeddings; output-only bias per token (reference modeling.py:543-549)
        self.decoder = nn.Linear(bert_model_embedding_weights.size(1), bert_model_embedding_weights.size(0), bias=False)
        self.decoder.weight = bert_model_embedding_weights
        self.bias = nn.Parameter(torch.zeros(bert_model_embedding_weights.size(0)))

    def forward(self, hidden_states):
        hidden_states = self.transform(hidden_states)
        x2, restore, _ = _tokens(hidden_states)
        return restore(ops.LinearFn.apply(x2, self.decoder.weight, self.bias, None))


class BertOnlyMLMHead(nn.Module):
    def __init__(self, config, bert_model_embedding_weights):
        super().__init__()
        self.predictions = BertLMPredictionHead(config, bert_model_embedding_weights)

    def forward(self, sequence_output):
        return self.predictions(sequence_output)


class BertOnlyNSPHead(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.seq_relationship = nn.Linear(config.hidden_size, 2)

    def forward(self, pooled_output):
        return self.seq_relationship(pooled_output.to(self.seq_relationship.weight.dtype))


class BertPreTrainingHeads(nn.Module):
    def __init__(self, config, bert_model_embedding_weights, sequence_output_is_dense=False):
        super().__init__()
        self.predictions = BertLMPredictionHead(config, bert_model_embedding_weights)
        self.seq_relationship = nn.Linear(config.hidden_size, 2)
        self.sequence_output_is_dense = sequence_output_is_dense
        # Optional static bound on the number of masked positions per batch (batch * max_predictions_per_seq).  When set, the row
        # indices come from torch.nonzero_static: no device->host sync (the reference's torch.nonzero drains the launch queue once
        # per step) and static shapes for CUDA-graph capture.  Surplus slots hold index -1 = padding: the gather kernel writes a zero
        # row, the scatter in backward skips them and the criterion gives them label -1 (ignored).  A batch with MORE masked positions
        # than the bound would silently lose the excess: that is recorded in `mlm_overflow` (device flag, sticky) and raised by
        # check_mlm_overflow(), which callers invoke at points that already synchronise (logging, checkpoint, end of run).
        self.static_masked_count = None
        self.register_buffer("mlm_overflow", torch.zeros((), dtype=torch.int32), persistent=False)

    def forward(self, sequence_output, pooled_output, masked_lm_labels):
        if self.sequence_output_is_dense:
            # only the masked positions reach the vocabulary GEMM (reference modeling.py:588-591); bit-exact row gather
            flat = sequence_output.reshape(-1, sequence_output.shape[-1])
            if self.static_masked_count:
                is_masked = masked_lm_labels.view(-1) != -1
                idx = torch.nonzero_static(is_masked, size=int(self.static_masked_count), fill_value=-1).squeeze(-1)
                self.mlm_overflow.logical_or_(is_masked.sum() > int(self.static_masked_count))
            else:
                idx = torch.nonzero(masked_lm_labels.view(-1) != -1).squeeze(-1)
            prediction_scores = self.predictions(ops.GatherRowsFn.apply(flat, idx))
        else:
            prediction_scores = self.predictions(sequence_output)
        # the 2-way NSP classifier is a [B,H]x[H,2] product: plain library call
        seq_relationship_score = self.seq_relationship(pooled_output.to(self.seq_relationship.weight.dtype))
        return prediction_scores, seq_relationship_score


    def check_mlm_overflow(self):
        """Host sync.  Raises if any batch so far held more masked positions than `static_masked_count`."""
        if self.static_masked_count and int(self.mlm_overflow.item()) != 0:
            raise L.DleError("a batch held more masked LM positions than static_masked_count=%d: the excess was dropped from the "
                             "loss; raise --max_predictions_per_seq or unset static_masked_count" % int(self.static_masked_count))


class BertPreTrainedModel(nn.Module):
    """Weight initialisation + flags shared by the task models (reference modeling.py:598-636)."""

    def __init__(self, config, *inputs, **kwargs):
        super().__init__()
        if not isinstance(config, BertConfig):
            raise ValueError("Parameter config in `{}(config)` should be an instance of class `BertConfig`.".format(
                self.__class__.__name__))
        self.config = config

    def half(self):
        """16-bit parameters on this path are bf16: the reference driver's `model.half()` (run_pretraining.py:416-417, taken for
        --allreduce_post_accumulation_fp16) therefore selects bfloat16 here, so the unmodified script drives the bf16 kernels.
        fp16 parameters are not supported by the kernels (DESIGN.md, precision policy)."""
        return self.bfloat16()

    def init_bert_weights(self, module):
        if isinstance(module, (nn.Linear, nn.Embedding)):
            module.weight.data.normal_(mean=0.0, std=self.config.initializer_range)
        elif isinstance(module, nn.LayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)
        if isinstance(module, nn.Linear) and module.bias is not None:
            module.bias.data.zero_()

    def checkpoint_activations(self, val):
        def _apply_flag(module):
            if hasattr(module, "_checkpoint_activations"):
                module._checkpoint_activations = val
        self.apply(_apply_flag)

    def enable_apex(self, val):
        def _apply_flag(module):
            if hasattr(module, "apex_enabled"):
                module.apex_enabled = val
        self.apply(_apply_flag)

    # (old name, new name) substrings of checkpoints written before the reference renamed its modules (modeling.py:736-752)
    _LEGACY_KEY_PARTS = (("gamma", "weight"), ("beta", "bias"), ("intermediate.dense.", "intermediate.dense_act."),
                         ("pooler.dense.", "pooler.dense_act."))

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, state_dict=None, cache_dir=None, from_tf=False, distill_config=None,
                        pooler=True, *inputs, **kwargs):
        """Build the model from a local pretrained archive and load its weights: the fine-tuning entry of the reference
        (modeling.py:655-786), same arguments and the same `(model, config)` return value.

        `pretrained_model_name_or_path` is a directory (or a .tar.gz of one) holding `bert_config.json` and `pytorch_model.bin`;
        `state_dict` replaces the weight file when given.  Checkpoint keys are mapped exactly as the reference does (LayerNorm
        gamma/beta -> weight/bias, `intermediate.dense.` / `pooler.dense.` -> `..dense_act.`), a `bert.` prefix is dropped when this
        class has no `bert` attribute (loading a pretraining checkpoint into `BertModel`), missing and unused keys are logged, shape
        mismatches raise.  Not carried over: model names that resolve to downloads (no network: the reference logs an error and
        returns None for an unknown name, and so does this), TensorFlow checkpoints (`from_tf`) and the distillation config
        (out of scope, DESIGN.md section 7) -- both raise NotImplementedError."""
        import logging
        import os
        import shutil
        import tarfile
        import tempfile
        log = logging.getLogger(__name__)
        if from_tf:
            raise NotImplementedError("TensorFlow checkpoints are not supported on this path (DESIGN.md section 7)")
        if distill_config:
            raise NotImplementedError("distillation is out of scope on this path (DESIGN.md section 7)")
        path = str(pretrained_model_name_or_path)
        if not os.path.exists(path):
            log.error("Model name '%s' was not found: pretrained model names need a download and there is no network on this path; "
                      "pass a directory or .tar.gz archive with bert_config.json and pytorch_model.bin", path)
            return None
        tmp = None
        try:
            if os.path.isdir(path):
                root = path
            else:
                tmp = tempfile.mkdtemp(dir=cache_dir)
                with tarfile.open(path, "r:gz") as tar:
                    tar.extractall(tmp, filter="data")
                root = tmp
            config = BertConfig.from_json_file(os.path.join(root, "bert_config.json"))
            model = cls(config, *inputs, **kwargs)
            if state_dict is None:
                state_dict = torch.load(os.path.join(root, "pytorch_model.bin"), map_location="cpu")
        finally:
            if tmp is not None:
                shutil.rmtree(tmp, ignore_errors=True)
        renamed = OrderedDict()
        for key, value in state_dict.items():
            for old, new in cls._LEGACY_KEY_PARTS:
                if old in key:
                    key = key.replace(old, new)          # (the rules are disjoint on real checkpoints; applied cumulatively)
            renamed[key] = value
        if not hasattr(model, "bert") and any(k.startswith("bert.") for k in renamed):
            renamed = OrderedDict((k[len("bert."):], v) for k, v in renamed.items() if k.startswith("bert."))
        result = model.load_state_dict(renamed, strict=False)    # raises RuntimeError on shape mismatches, like the reference
        if result.missing_keys:
            log.info("Weights of %s not initialized from pretrained model: %s", cls.__name__, result.missing_keys)
        if result.unexpected_keys:
            log.info("Weights from pretrained model not used in %s: %s", cls.__name__, result.unexpected_keys)
        return model, config


class BertModel(BertPreTrainedModel):
    """Embeddings + encoder + pooler (reference modeling.py:788-888).
    forward(input_ids, token_type_ids, attention_mask) -> (encoded_layers, pooled_output)."""

    def __init__(self, config):
        super().__init__(config)
        self.distillation = getattr(config, 'distillation', False)
        if self.distillation:
            self.distill_state_dict = OrderedDict()
            self.distill_config = config.distillation_config
        else:
            self.distill_config = {'use_pooler': False, 'use_pred_states': False}
        self.embeddings = BertEmbeddings(config)
        self.encoder = BertEncoder(config)
        if not self.distillation or (self.distill_config["use_pooler"] and self.distill_config["use_pred_states"]):
            self.pooler = BertPooler(config)
        self.apply(self.init_bert_weights)
        self.output_all_encoded_layers = config.output_all_encoded_layers
        self.teacher = False

    def forward(self, input_ids, token_type_ids, attention_mask):
        if attention_mask is None:
            attention_mask = torch.ones_like(input_ids)
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        if self.training:
            ops.advance_step(input_ids.device)      # fresh dropout masks per forward pass, also when this call is a CUDA-graph replay
        # additive mask [B,1,1,S]: 0 where attended, -10000 where masked (reference modeling.py:864-872)
        extended_attention_mask = attention_mask.unsqueeze(1).unsqueeze(2).to(torch.float32)
        extended_attention_mask = (1.0 - extended_attention_mask) * -10000.0
        embedding_output = self.embeddings(input_ids, token_type_ids)
        encoded_layers = self.encoder(embedding_output, extended_attention_mask)
        sequence_output = encoded_layers[-1]
        if not self.distillation or (self.distill_config["use_pooler"] and self.distill_config["use_pred_states"]):
            pooled_output = self.pooler(sequence_output)
        else:
            pooled_output = None
        if not self.output_all_encoded_layers:
            encoded_layers = encoded_layers[-1:]
        if not self.teacher:
            return encoded_layers, pooled_output

    def make_teacher(self):
        self.teacher = True


class BertForPreTraining(BertPreTrainedModel):
    """BERT with the MLM + NSP heads (reference modeling.py:890-958).
    forward(input_ids, token_type_ids, attention_mask, masked_lm_labels) -> (prediction_scores, seq_relationship_score)."""

    def __init__(self, config, sequence_output_is_dense=False):
        super().__init__(config)
        self.bert = BertModel(config)
        self.distillation = getattr(config, 'distillation', False)
        if not self.distillation:
            self.cls = BertPreTrainingHeads(config, self.bert.embeddings.word_embeddings.weight, sequence_output_is_dense)
        self.apply(self.init_bert_weights)

    def forward(self, input_ids, token_type_ids, attention_mask, masked_lm_labels):
        encoded_layers, pooled_output = self.bert(input_ids, token_type_ids, attention_mask)
        if not self.distillation:
            sequence_output = encoded_layers[-1]
            return self.cls(sequence_output, pooled_output, masked_lm_labels)


class BertForQuestionAnswering(BertPreTrainedModel):
    """Span-classification head over the same encoder (reference modeling.py:1301-1371).
    forward(input_ids, token_type_ids, attention_mask) -> (start_logits, end_logits)."""

    def __init__(self, config):
        super().__init__(config)
        self.bert = BertModel(config)
        self.qa_outputs = nn.Linear(config.hidden_size, 2)
        self.apply(self.init_bert_weights)

    def forward(self, input_ids, token_type_ids, attention_mask):
        encoded_layers, _ = self.bert(input_ids, token_type_ids, attention_mask)
        sequence_output = encoded_layers[-1]
        logits = self.qa_outputs(sequence_output.to(self.qa_outputs.weight.dtype))
        start_logits, end_logits = logits.split(1, dim=-1)
        return start_logits.squeeze(-1), end_logits.squeeze(-1)
