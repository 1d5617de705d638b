"""Generate the multiple-choice golden vectors by running the UNMODIFIED reference modeling.py's BertForMultipleChoice (imported as
make_golden.py does, from $DLE_REFERENCE_ROOT) on CPU.  Commit the output; the tests themselves never need the reference.

    python tests/golden/make_mc_golden.py

Output
  bert_mc_golden.pt : tiny config (H=64, L=2, A=4, I=256, V=512), 3 examples x 4 choices x S=32 with ragged masks, num_choices = 4,
                      dropout off.  The parameters are regenerated from seeds by mc_params() (make_cls_golden.cls_params with a
                      [1, H] classifier; the tests call it too), so only outputs are stored: the reference's state_dict key list, the
                      batch, reshaped_logits [3, 4], the loss model(..., labels) returns (run_swag.py:468), every gradient's norm (in
                      grad_keys order), the gradients of the head and the pooler in full, and every STRIDE-th element of each other
                      gradient, concatenated in grad_keys order.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_cls_golden import FULL_GRADS, STRIDE, TINY, cls_params  # noqa: E402

NUM_CHOICES = 4
N, S = 3, 32


def mc_params(cfg=TINY):
    """The golden's state_dict, from seeds: make_cls_golden's parameters with one output row in the classifier."""
    return cls_params(cfg, num_labels=1)


def mc_batch(cfg=TINY):
    g = torch.Generator().manual_seed(23)
    ids = torch.randint(0, cfg["vocab_size"], (N, NUM_CHOICES, S), generator=g)
    ids[:, :, 0] = 101
    lens = torch.tensor([[32, 20, 9, 27], [14, 30, 5, 18], [25, 25, 12, 31]])
    pos = torch.arange(S).view(1, 1, S)
    am = (pos < lens.unsqueeze(-1)).long()
    seg = ((pos >= (lens // 2).unsqueeze(-1)) & (am != 0)).long()
    return dict(input_ids=ids, segment_ids=seg, input_mask=am, label_ids=torch.tensor([2, 0, 3]))


def main():
    from make_golden import import_reference_modeling
    modeling = import_reference_modeling()
    torch.manual_seed(0)
    config = modeling.BertConfig.from_dict({**TINY, "hidden_dropout_prob": 0.0, "attention_probs_dropout_prob": 0.0})
    model = modeling.BertForMultipleChoice(config, num_choices=NUM_CHOICES)
    keys = list(model.state_dict().keys())
    missing, unexpected = model.load_state_dict(mc_params(), strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    b = mc_batch()
    model.train()
    with torch.no_grad():
        logits = model(b["input_ids"], b["segment_ids"], b["input_mask"])
    loss = model(b["input_ids"], b["segment_ids"], b["input_mask"], b["label_ids"])
    loss.backward()
    grads = {k: p.grad.detach() for k, p in model.named_parameters() if p.grad is not None}
    torch.save(dict(num_choices=NUM_CHOICES, state_dict_keys=keys, batch=b, logits=logits.detach(), loss=loss.detach(),
                    grad_keys=list(grads), grad_norms=torch.stack([v.norm() for v in grads.values()]),
                    grads={k: v.clone() for k, v in grads.items() if k in FULL_GRADS},
                    grads_strided=torch.cat([v.reshape(-1)[::STRIDE] for k, v in grads.items() if k not in FULL_GRADS])),
               os.path.join(HERE, "bert_mc_golden.pt"))
    print("mc loss", float(loss.detach()), "logits", tuple(logits.shape), "keys", len(keys), "grads", len(grads))


if __name__ == "__main__":
    main()
