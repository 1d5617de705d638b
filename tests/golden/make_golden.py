"""Generate golden vectors by running the UNMODIFIED reference modeling.py (imported from
a reference checkout named by $DLE_REFERENCE_ROOT) on seeded inputs.  Commit the outputs; the tests
themselves never need the reference.

    python tests/golden/make_golden.py

Shims (SURVEY.md 8(c)): stub boto3/botocore (file_utils.py:32-34 imports them), and rebind
modeling.gelu to F.gelu(approximate='tanh') because `approximate=True` (modeling.py:122) only
exists in NGC's patched torch.

Outputs
  bert_tiny_golden.pt : tiny config (H=64, L=2, A=4, I=256, V=512, S=32, B=3, ragged mask):
                        state_dict, batch, per-layer activations, logits, loss, all grads.
  bert_large2_golden.pt : the BENCHMARKED widths (BASELINE configs[1]/[2]: H=1024, A=16, I=4096, V=30528) with 2 encoder
                        layers, B=2, ragged mask, at S=512 and S=128; bf16-representable weights regenerated from the
                        seed by the tests; stored: loss, nsp, strided logits + per-row logsumexp over the full
                        vocabulary, strided sequence output, every gradient norm and strided slices of selected grads.
  bert_base_golden.pt : BASELINE config 1 shape (BERT-base, B=4, S=128, fp32): params are
                        regenerated from seed by oracle.bert_oracle.init_params, so only the
                        loss, logits slices and a few grad norms are stored.
"""
import os
import sys
import types

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.join(os.environ.get("DLE_REFERENCE_ROOT", ""), "PyTorch/LanguageModeling/BERT")
sys.path.insert(0, ROOT)


def import_reference_modeling():
    for name in ("boto3", "botocore", "botocore.exceptions"):
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    sys.modules["botocore.exceptions"].ClientError = Exception
    sys.modules["botocore"].exceptions = sys.modules["botocore.exceptions"]
    sys.path.insert(0, REF)
    import modeling  # the reference's own file
    modeling.gelu = lambda x: F.gelu(x, approximate="tanh")
    modeling.ACT2FN["gelu"] = modeling.gelu
    return modeling


def ref_criterion(scores, nsp, labels, nsl, vocab):
    # run_pretraining.py:85-95 (the driver itself is not importable without CUDA/lddl/dllogger)
    loss_fn = torch.nn.CrossEntropyLoss(ignore_index=-1)
    flat = labels.view(-1)
    mlm = loss_fn(scores.view(-1, vocab), flat[flat != -1].view(-1))
    return mlm + loss_fn(nsp.view(-1, 2), nsl.view(-1))


def run(modeling, cfg, sd, batch, capture_layers):
    from oracle import bert_oracle as O
    config = modeling.BertConfig.from_dict({**cfg, "hidden_dropout_prob": 0.0,
                                            "attention_probs_dropout_prob": 0.0})
    model = modeling.BertForPreTraining(config, sequence_output_is_dense=True)
    full = dict(sd)
    full["cls.predictions.decoder.weight"] = sd["bert.embeddings.word_embeddings.weight"]
    missing, unexpected = model.load_state_dict(full, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    model.train()
    acts = {}
    if capture_layers:
        model.bert.embeddings.register_forward_hook(lambda m, i, o: acts.__setitem__("embeddings", o.detach().clone()))
        for li, layer in enumerate(model.bert.encoder.layer):
            layer.attention.self.register_forward_hook(
                lambda m, i, o, li=li: acts.__setitem__(f"layer{li}.ctx", o.detach().clone()))     # [S,B,H]
            layer.attention.register_forward_hook(
                lambda m, i, o, li=li: acts.__setitem__(f"layer{li}.attn_out", o.detach().clone()))
            layer.intermediate.register_forward_hook(
                lambda m, i, o, li=li: acts.__setitem__(f"layer{li}.inter", o.detach().clone()))
            layer.register_forward_hook(
                lambda m, i, o, li=li: acts.__setitem__(f"layer{li}.out", o.detach().clone()))
    scores, nsp = model(batch["input_ids"], batch["token_type_ids"], batch["attention_mask"], batch["labels"])
    loss = ref_criterion(scores, nsp, batch["labels"], batch["next_sentence_labels"], config.vocab_size)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}
    return dict(scores=scores.detach(), nsp=nsp.detach(), loss=loss.detach(), acts=acts, grads=grads)


SMALL_GRAD_KEYS = ["bert.encoder.layer.0.attention.self.query.weight", "bert.encoder.layer.0.attention.self.value.bias",
                   "bert.encoder.layer.1.intermediate.dense_act.weight", "bert.encoder.layer.1.output.LayerNorm.weight",
                   "bert.encoder.layer.0.attention.output.dense.weight", "bert.embeddings.position_embeddings.weight",
                   "bert.embeddings.LayerNorm.bias", "cls.predictions.transform.dense_act.weight", "bert.pooler.dense_act.weight"]


LARGE_GRAD_KEYS = ["bert.encoder.layer.0.attention.self.query.weight", "bert.encoder.layer.0.attention.self.key.weight",
                   "bert.encoder.layer.0.attention.self.value.bias", "bert.encoder.layer.0.attention.output.dense.weight",
                   "bert.encoder.layer.1.intermediate.dense_act.weight", "bert.encoder.layer.1.intermediate.dense_act.bias",
                   "bert.encoder.layer.1.output.dense.weight", "bert.encoder.layer.1.output.LayerNorm.weight",
                   "bert.embeddings.word_embeddings.weight", "bert.embeddings.position_embeddings.weight",
                   "cls.predictions.transform.dense_act.weight", "cls.predictions.bias", "bert.pooler.dense_act.weight"]


def main():
    from oracle import bert_oracle as O
    modeling = import_reference_modeling()
    torch.manual_seed(0)

    tiny = dict(hidden_size=64, num_hidden_layers=2, num_attention_heads=4, intermediate_size=256,
                vocab_size=512, max_position_embeddings=64, type_vocab_size=2, hidden_act="gelu",
                initializer_range=0.02)
    sd = O.init_params(tiny, seed=7, std=0.2)          # large std so every op is numerically visible
    g = torch.Generator().manual_seed(11)
    for k in sd:                                        # non-trivial LN affine and biases
        if "LayerNorm" in k or k.endswith("bias"):
            sd[k] = sd[k] + 0.1 * torch.randn(sd[k].shape, generator=g)
    batch = O.synthetic_batch(3, 32, tiny["vocab_size"], 5, seed=3, full_mask=False)
    r = run(modeling, tiny, sd, batch, capture_layers=True)
    torch.save(dict(cfg=tiny, state_dict=sd, batch=batch, **r), os.path.join(HERE, "bert_tiny_golden.pt"))
    print("tiny loss", float(r["loss"]))

    # kernel-compatible small config (head size 64, H % 256 == 0, S % 128 == 0).  Weights are bf16-representable
    # (rounded before use) so the bf16 GPU model and the fp32 reference hold identical parameters; they are
    # regenerated from the seed by the tests, only outputs are stored.
    small = dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=1024, vocab_size=1024,
                 max_position_embeddings=128, type_vocab_size=2, hidden_act="gelu", initializer_range=0.02)
    sd = O.bf16_representable_params(small, seed=21)
    batch = O.synthetic_batch(2, 128, small["vocab_size"], 10, seed=5, full_mask=False)
    r = run(modeling, small, sd, batch, capture_layers=True)
    torch.save(dict(cfg=small, param_seed=21, batch_seed=5, loss=r["loss"], scores=r["scores"].half(), nsp=r["nsp"],
                    seq_out=r["acts"]["layer1.out"].transpose(0, 1).contiguous().half(),
                    layer0_ctx=r["acts"]["layer0.ctx"].transpose(0, 1).contiguous().half(),
                    embeddings=r["acts"]["embeddings"].half(),
                    grad_norms={k: v.norm() for k, v in r["grads"].items()},
                    grads={k: r["grads"][k].half() for k in SMALL_GRAD_KEYS}),
               os.path.join(HERE, "bert_small_golden.pt"))
    print("small loss", float(r["loss"]))

    # BERT-large widths, 2 layers (the benchmarked per-layer shapes; 24 layers would only repeat them)
    large2 = dict(O.BERT_LARGE)
    large2.update(num_hidden_layers=2, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    sd = O.bf16_representable_params(large2, seed=77, std=0.04)
    out = dict(cfg=large2, param_seed=77, param_std=0.04, cases={})
    for S, P, bseed in ((512, 80, 13), (128, 20, 17)):
        batch = O.synthetic_batch(2, S, large2["vocab_size"], P, seed=bseed, full_mask=False)
        r = run(modeling, large2, sd, batch, capture_layers=True)
        out["cases"][S] = dict(
            batch_seed=bseed, max_pred=P, loss=r["loss"], nsp=r["nsp"],
            scores_strided=r["scores"][:, ::16].half(), scores_lse=torch.logsumexp(r["scores"], -1),
            scores_absmax=r["scores"].abs().max(),
            seq_out_strided=r["acts"]["layer1.out"].transpose(0, 1).contiguous()[:, :, ::8].half(),
            layer0_ctx_strided=r["acts"]["layer0.ctx"].transpose(0, 1).contiguous()[:, :, ::8].half(),
            grad_norms={k: v.norm() for k, v in r["grads"].items()},
            grads_strided={k: r["grads"][k].reshape(-1)[::(1 if r["grads"][k].numel() <= 4096 else 97)].clone() for k in LARGE_GRAD_KEYS})
        print("large2 S=%d loss" % S, float(r["loss"]))
    torch.save(out, os.path.join(HERE, "bert_large2_golden.pt"))

    base = dict(O.BERT_BASE)
    sd = O.init_params(base, seed=42)
    batch = O.synthetic_batch(4, 128, base["vocab_size"], 20, seed=42, full_mask=True)
    r = run(modeling, base, sd, batch, capture_layers=False)
    keep = ["bert.encoder.layer.0.attention.self.query.weight", "bert.encoder.layer.11.output.dense.weight",
            "bert.embeddings.word_embeddings.weight", "cls.predictions.bias",
            "bert.encoder.layer.5.intermediate.dense_act.bias"]
    torch.save(dict(cfg=base, seed=42, batch_seed=42, loss=r["loss"], scores_slice=r["scores"][:8, :64].clone(),
                    scores_absmean=r["scores"].abs().mean(), nsp=r["nsp"],
                    grad_norms={k: r["grads"][k].norm() for k in keep}),
               os.path.join(HERE, "bert_base_golden.pt"))
    print("base loss", float(r["loss"]))


if __name__ == "__main__":
    main()
