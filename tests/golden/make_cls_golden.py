"""Generate the sequence-classification golden vectors by running the UNMODIFIED reference modeling.py's
BertForSequenceClassification (imported as make_golden.py does, from $DLE_REFERENCE_ROOT) on CPU.  Commit the output; the tests
themselves never need the reference.

    python tests/golden/make_cls_golden.py

Output
  bert_cls_golden.pt : tiny config (H=64, L=2, A=4, I=256, V=512, S=32, B=4, ragged mask), num_labels = 3, dropout off.  The
                       parameters are regenerated from seeds by cls_params() (the tests call it too), so only outputs are stored:
                       the reference's state_dict key list, the batch, the logits, run_glue's loss
                       (CrossEntropyLoss()(logits.view(-1, 3), label_ids.view(-1)), run_glue.py:597,631-634), every gradient's norm
                       (in grad_keys order), the gradients of the head and the pooler in full, and every STRIDE-th element of
                       each other gradient, concatenated in grad_keys order.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

TINY = dict(hidden_size=64, num_hidden_layers=2, num_attention_heads=4, intermediate_size=256, vocab_size=512,
            max_position_embeddings=64, type_vocab_size=2, hidden_act="gelu", initializer_range=0.02)
NUM_LABELS = 3
FULL_GRADS = ("classifier.weight", "classifier.bias", "bert.pooler.dense_act.weight", "bert.pooler.dense_act.bias")
STRIDE = 97                                             # every 97th element of every other gradient


def cls_params(cfg=TINY, num_labels=NUM_LABELS):
    """The golden's state_dict, from seeds: oracle.init_params (std 0.2, every op numerically visible), non-trivial LayerNorm
    affines and biases, and a random classifier."""
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import bert_oracle as O
    sd = {k: v for k, v in O.init_params(cfg, seed=9, std=0.2).items() if k.startswith("bert.")}
    g = torch.Generator().manual_seed(13)
    for k in sd:
        if "LayerNorm" in k or k.endswith("bias"):
            sd[k] = sd[k] + 0.1 * torch.randn(sd[k].shape, generator=g)
    sd["classifier.weight"] = torch.randn(num_labels, cfg["hidden_size"], generator=g) * 0.2
    sd["classifier.bias"] = torch.randn(num_labels, generator=g) * 0.1
    return sd


def cls_batch(cfg=TINY):
    g = torch.Generator().manual_seed(17)
    B, S = 4, 32
    ids = torch.randint(0, cfg["vocab_size"], (B, S), generator=g)
    ids[:, 0] = 101
    lens = torch.tensor([32, 20, 9, 27])
    pos = torch.arange(S).unsqueeze(0)
    am = (pos < lens.unsqueeze(1)).long()
    seg = ((pos >= (lens // 2).unsqueeze(1)) & (am != 0)).long()
    return dict(input_ids=ids, segment_ids=seg, input_mask=am, label_ids=torch.tensor([2, 0, 1, 1]))


def main():
    sys.path.insert(0, HERE)
    from make_golden import import_reference_modeling
    modeling = import_reference_modeling()
    torch.manual_seed(0)
    config = modeling.BertConfig.from_dict({**TINY, "hidden_dropout_prob": 0.0, "attention_probs_dropout_prob": 0.0})
    model = modeling.BertForSequenceClassification(config, num_labels=NUM_LABELS)
    keys = list(model.state_dict().keys())
    missing, unexpected = model.load_state_dict(cls_params(), strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    b = cls_batch()
    model.train()
    logits = model(b["input_ids"], b["segment_ids"], b["input_mask"])
    loss = torch.nn.CrossEntropyLoss()(logits.view(-1, NUM_LABELS), b["label_ids"].view(-1))
    loss.backward()
    grads = {k: p.grad.detach() for k, p in model.named_parameters() if p.grad is not None}
    torch.save(dict(num_labels=NUM_LABELS, state_dict_keys=keys, batch=b, logits=logits.detach(), loss=loss.detach(),
                    grad_keys=list(grads), grad_norms=torch.stack([v.norm() for v in grads.values()]),
                    grads={k: v.clone() for k, v in grads.items() if k in FULL_GRADS},
                    grads_strided=torch.cat([v.reshape(-1)[::STRIDE] for k, v in grads.items() if k not in FULL_GRADS])),
               os.path.join(HERE, "bert_cls_golden.pt"))
    print("cls loss", float(loss.detach()), "keys", len(keys), "grads", len(grads))


if __name__ == "__main__":
    main()
