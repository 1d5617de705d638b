"""Sequence packing on the host: several pretraining samples per S-token row (BertPreTrainedModel.pack_sequences).

The packed batch format (the one BertModel.forward reads in packed mode; dle_segment_table is its device-side reader):

  * input_ids, token_type_ids, labels: int64 [B, S].  Each sample keeps its own [CLS], token types and MLM labels (-1 = none).
  * attention_mask: int64 [B, S], the sample number of each token: the tokens of a row's j-th sample hold j (1 <= j <= k), samples are
    contiguous and in increasing order, and the row's padding tail holds 0 and comes last.  k = max_per_row is a static setting.
  * next_sentence_labels: int64 [B, k], -1 in slots that hold no sample.

Shapes are those of an unpacked batch (plus k NSP slots per row), so a packed step keeps the padded step's static shapes and can be
captured into a CUDA graph.  The packer places each sample whole (first-fit decreasing over a pool of samples), so a row holds at most
S tokens, at most k samples and at most `max_pred` MLM labels: the static bound of B * max_pred masked rows holds as for unpacked rows.

The packed SQuAD format (BertForQuestionAnswering.pack_sequences(k, per_sample_logits=True); the keys squad.squad_training_step
reads):

  * input_ids, segment_ids: int64 [B, S].  Each feature keeps its own [CLS] question [SEP] context [SEP] tokens and segment ids.
  * input_mask: int64 [B, S], sample numbers 1..k and 0 on the tail, exactly as attention_mask above.
  * start_positions, end_positions: int64 [B*k].  Slot b*k + j-1 holds sample j of row b; a position counts from the sample's first
    token.  An empty slot, and an answer outside the feature, hold S: the loss's ignore_index (run_squad.py:1073-1079).
  * feature_index (a host attribute of the PackedBatch, numpy int64 [B*k]): the index of the SQuAD feature in each slot, -1 when the
    slot is empty.  Evaluation maps the [B*k, S] logits back to their features through it.

The packed GLUE format (BertForSequenceClassification.pack_sequences(k); the keys glue.glue_training_step reads, run_glue.py's batch):

  * input_ids, segment_ids: int64 [B, S].  Each example keeps its own [CLS] a [SEP] b [SEP] tokens and segment ids.
  * input_mask: int64 [B, S], sample numbers 1..k and 0 on the tail, exactly as attention_mask above.
  * label_ids: int64 [B*k].  Slot b*k + j-1 holds sample j of row b; an empty slot holds -100, the default ignore_index of the
    reference's CrossEntropyLoss (run_glue.py:597), so its loss line runs unchanged and averages over the real samples.
  * example_index (a host attribute of the PackedBatch, numpy int64 [B*k]): the index of the example in each slot, -1 when the slot
    is empty.  Evaluation maps the [B*k, num_labels] logits back to their examples through it.

The packed SWAG format (BertForMultipleChoice.pack_sequences(k), k a multiple of the number of choices C; the keys
swag.swag_training_step reads).  The unpacked source is run_swag.py's batch (select_field, :237-245, :548-552): input_ids, input_mask,
segment_ids [N, C, S_choice], each choice a right-padded [CLS] context [SEP] ending [SEP] row, and label_ids [N].  The unit of packing
is the example, never a single choice: a row holds at most k/C whole examples, each choice keeping its own tokens and segment ids and
the choices in their order (the label indexes them).

  * input_ids, segment_ids: int64 [B, S].
  * input_mask: int64 [B, S].  Choice c of the row's m-th example holds sample number m*C + c + 1; the tail holds 0.  Every sample
    number is a slot of attention_mask above, so the pooled output is [B*k, H] and slot b*k + m*C + c is choice c of that example.
  * label_ids: int64 [B*k/C].  Group b*(k/C) + m holds the label of the m-th example of row b, -100 when the group is empty.  The
    reference's view(-1, C) of the [B*k, 1] logits therefore lines every group of C scores up with its label.
  * example_index (a host attribute of the PackedBatch, numpy int64 [B*k/C]): the index of the example in each group, -1 when the
    group is empty.
"""
import numpy as np
import torch

KEYS = ("input_ids", "token_type_ids", "attention_mask", "labels", "next_sentence_labels")


class Sample:
    """One pretraining sample: ids, token types and MLM labels of its real tokens (1-D int64 numpy arrays) and its NSP label."""
    __slots__ = ("input_ids", "token_type_ids", "labels", "next_sentence_label", "n_labels")

    def __init__(self, input_ids, token_type_ids, labels, next_sentence_label):
        self.input_ids, self.token_type_ids, self.labels = input_ids, token_type_ids, labels
        self.next_sentence_label = int(next_sentence_label)
        self.n_labels = int((labels != -1).sum())

    def __len__(self):
        return len(self.input_ids)


class SquadSample:
    """One SQuAD feature: ids and segment ids of its real tokens (1-D int64 numpy arrays), its answer's start and end relative to its
    first token (S or more: no answer in this feature, ignored by the loss) and the index of the feature in its source stream."""
    __slots__ = ("input_ids", "segment_ids", "start_position", "end_position", "feature_index")
    n_labels = 0                                         # no MLM labels: pack()'s label bound never binds

    def __init__(self, input_ids, segment_ids, start_position, end_position, feature_index):
        self.input_ids, self.segment_ids = input_ids, segment_ids
        self.start_position, self.end_position = int(start_position), int(end_position)
        self.feature_index = int(feature_index)

    def __len__(self):
        return len(self.input_ids)


class GlueSample:
    """One GLUE example: ids and segment ids of its real tokens (1-D int64 numpy arrays), its label and the index of the example in
    its source stream."""
    __slots__ = ("input_ids", "segment_ids", "label", "example_index")
    n_labels = 0                                         # no MLM labels: pack()'s label bound never binds

    def __init__(self, input_ids, segment_ids, label, example_index):
        self.input_ids, self.segment_ids = input_ids, segment_ids
        self.label, self.example_index = int(label), int(example_index)

    def __len__(self):
        return len(self.input_ids)


class SwagSample:
    """One SWAG example: per choice, the ids and segment ids of its real tokens (tuples of C 1-D int64 numpy arrays, in choice order),
    its label and the index of the example in its source stream.  Its length is the sum of its choices' lengths."""
    __slots__ = ("input_ids", "segment_ids", "label", "example_index")
    n_labels = 0                                         # no MLM labels: pack()'s label bound never binds

    def __init__(self, input_ids, segment_ids, label, example_index):
        self.input_ids, self.segment_ids = tuple(input_ids), tuple(segment_ids)
        self.label, self.example_index = int(label), int(example_index)

    def __len__(self):
        return sum(len(c) for c in self.input_ids)


class PackedBatch(dict):
    """A packed batch: the tensors as dict items, and `num_samples`, the number of samples it holds (a host int; a SWAG batch counts
    examples).  A SQuAD batch also carries `feature_index`, a GLUE or SWAG batch `example_index` (see the module docstring)."""

    def __init__(self, tensors, num_samples):
        super().__init__(tensors)
        self.num_samples = int(num_samples)


def split_samples(batch, max_pred=None):
    """The samples of an unpacked lddl-format batch (0/1 attention_mask, next_sentence_labels [B]): the tokens whose mask is 1, in
    order, one sample per row; a row without such a token holds no sample.  Raises ValueError for a sample with more than `max_pred`
    MLM labels, which no packed row could take."""
    ids, tt, am, lab, nsl = (batch[k].cpu().numpy() for k in KEYS)
    if am.min(initial=0) < 0 or am.max(initial=0) > 1:
        raise ValueError("split_samples takes an unpacked batch: attention_mask must hold only 0 and 1")
    out = []
    for b in range(ids.shape[0]):
        keep = am[b] != 0
        if not keep.any():
            continue
        s = Sample(ids[b][keep], tt[b][keep], lab[b][keep], nsl[b])
        if max_pred is not None and s.n_labels > max_pred:
            raise ValueError(f"a sample holds {s.n_labels} MLM labels, more than max_predictions_per_seq = {max_pred}")
        out.append(s)
    return out


def pack(samples, B, S, k, max_pred):
    """First-fit decreasing: (rows, unplaced).  rows: at most B lists of sample indices, each row within S tokens, k samples and
    max_pred labels; a row's samples in the order they were placed.  unplaced: the indices that found no room, in increasing order.
    Ties in length go to the earlier sample, so the result is a function of the list alone."""
    order = sorted(range(len(samples)), key=lambda i: (-len(samples[i]), i))
    rows, used = [], []                                  # used[r] = [tokens, samples, labels]
    unplaced = []
    for i in order:
        n, nl = len(samples[i]), samples[i].n_labels
        if n > S or nl > max_pred:
            raise ValueError(f"a sample of {n} tokens and {nl} labels does not fit a row of {S} tokens and {max_pred} labels")
        for r, u in enumerate(used):
            if u[0] + n <= S and u[1] < k and u[2] + nl <= max_pred:
                rows[r].append(i)
                u[0] += n; u[1] += 1; u[2] += nl
                break
        else:
            if len(rows) < B:
                rows.append([i])
                used.append([n, 1, nl])
            else:
                unplaced.append(i)
    return rows, sorted(unplaced)


def to_batch(samples, rows, B, S, k, pin=False):
    """The packed batch (PackedBatch of CPU int64 tensors) with rows[r] in row r; rows past len(rows) hold no sample."""
    ids = np.zeros((B, S), np.int64)
    tt = np.zeros((B, S), np.int64)
    am = np.zeros((B, S), np.int64)
    lab = np.full((B, S), -1, np.int64)
    nsl = np.full((B, k), -1, np.int64)
    count = 0
    for r, members in enumerate(rows):
        off = 0
        for j, i in enumerate(members, 1):
            s = samples[i]
            n = len(s)
            ids[r, off:off + n] = s.input_ids
            tt[r, off:off + n] = s.token_type_ids
            lab[r, off:off + n] = s.labels
            am[r, off:off + n] = j
            nsl[r, j - 1] = s.next_sentence_label
            off += n
            count += 1
    t = {key: torch.from_numpy(v) for key, v in zip(KEYS, (ids, tt, am, lab, nsl))}
    if pin:
        t = {key: v.pin_memory() for key, v in t.items()}
    return PackedBatch(t, count)


def unpack(batch):
    """The samples of a packed batch, row by row and in sample order (the inverse of to_batch)."""
    ids, tt, am, lab, nsl = (batch[key].cpu().numpy() for key in KEYS)
    out = []
    for r in range(ids.shape[0]):
        for j in range(1, nsl.shape[1] + 1):
            sel = am[r] == j
            if sel.any():
                out.append(Sample(ids[r][sel], tt[r][sel], lab[r][sel], nsl[r, j - 1]))
    return out


SQUAD_KEYS = ("input_ids", "segment_ids", "input_mask", "start_positions", "end_positions")


def split_squad_samples(batch, first_feature_index=0):
    """The features of an unpacked SQuAD batch (0/1 input_mask, right-padded rows, start/end_positions [B]): the tokens whose mask is
    1, one feature per row, feature index first_feature_index + row; a row without such a token holds no feature."""
    ids, seg, am, sp, ep = (batch[key].cpu().numpy() for key in SQUAD_KEYS)
    if am.min(initial=0) < 0 or am.max(initial=0) > 1:
        raise ValueError("split_squad_samples takes an unpacked batch: input_mask must hold only 0 and 1")
    out = []
    for b in range(ids.shape[0]):
        keep = am[b] != 0
        if keep.any():
            out.append(SquadSample(ids[b][keep], seg[b][keep], sp[b], ep[b], first_feature_index + b))
    return out


def to_squad_batch(samples, rows, B, S, k, pin=False):
    """The packed SQuAD batch (PackedBatch of CPU int64 tensors, with feature_index) with rows[r] in row r.  A position of S or more
    becomes S (ignored, as the reference's clamp makes it); a position inside [len, S) points into a padded row's padding, which a
    packed sample does not have: ValueError."""
    ids = np.zeros((B, S), np.int64)
    seg = np.zeros((B, S), np.int64)
    am = np.zeros((B, S), np.int64)
    pos = np.full((2, B * k), S, np.int64)
    fi = np.full(B * k, -1, np.int64)
    count = 0
    for r, members in enumerate(rows):
        off = 0
        for j, i in enumerate(members, 1):
            s = samples[i]
            n = len(s)
            for c, p in enumerate((s.start_position, s.end_position)):
                if n <= p < S:
                    raise ValueError(f"feature {s.feature_index}: answer position {p} lies in the padding of its row (length {n}, "
                                     f"S = {S}); only positions < {n} or >= {S} (ignored) have a meaning per sample")
                pos[c, r * k + j - 1] = min(p, S)
            ids[r, off:off + n] = s.input_ids
            seg[r, off:off + n] = s.segment_ids
            am[r, off:off + n] = j
            fi[r * k + j - 1] = s.feature_index
            off += n
            count += 1
    t = {key: torch.from_numpy(v) for key, v in zip(SQUAD_KEYS, (ids, seg, am, pos[0], pos[1]))}
    if pin:
        t = {key: v.pin_memory() for key, v in t.items()}
    batch = PackedBatch(t, count)
    batch.feature_index = fi
    return batch


def unpack_squad(batch):
    """The features of a packed SQuAD batch in slot order (the inverse of to_squad_batch, with positions past the sample as S)."""
    ids, seg, am, sp, ep = (batch[key].cpu().numpy() for key in SQUAD_KEYS)
    k = sp.shape[0] // ids.shape[0]
    out = []
    for r in range(ids.shape[0]):
        for j in range(1, k + 1):
            sel = am[r] == j
            if sel.any():
                slot = r * k + j - 1
                out.append(SquadSample(ids[r][sel], seg[r][sel], sp[slot], ep[slot], batch.feature_index[slot]))
    return out


GLUE_KEYS = ("input_ids", "segment_ids", "input_mask", "label_ids")
GLUE_IGNORE = -100                                       # CrossEntropyLoss's default ignore_index


def split_glue_samples(batch, first_example_index=0):
    """The examples of an unpacked GLUE batch (0/1 input_mask, right-padded rows, label_ids [B]): the tokens whose mask is 1, one
    example per row, example index first_example_index + row; a row without such a token holds no example."""
    ids, seg, am, lab = (batch[key].cpu().numpy() for key in GLUE_KEYS)
    if am.min(initial=0) < 0 or am.max(initial=0) > 1:
        raise ValueError("split_glue_samples takes an unpacked batch: input_mask must hold only 0 and 1")
    out = []
    for b in range(ids.shape[0]):
        keep = am[b] != 0
        if keep.any():
            out.append(GlueSample(ids[b][keep], seg[b][keep], lab[b], first_example_index + b))
    return out


def to_glue_batch(samples, rows, B, S, k, pin=False):
    """The packed GLUE batch (PackedBatch of CPU int64 tensors, with example_index) with rows[r] in row r; rows past len(rows) and
    slots past a row's samples are empty (label -100, example index -1).  ValueError when a row exceeds S tokens or k samples."""
    ids = np.zeros((B, S), np.int64)
    seg = np.zeros((B, S), np.int64)
    am = np.zeros((B, S), np.int64)
    lab = np.full(B * k, GLUE_IGNORE, np.int64)
    ei = np.full(B * k, -1, np.int64)
    if len(rows) > B:
        raise ValueError(f"{len(rows)} rows do not fit a batch of {B}")
    count = 0
    for r, members in enumerate(rows):
        n_row = sum(len(samples[i]) for i in members)
        if n_row > S or len(members) > k:
            raise ValueError(f"row {r}: {len(members)} samples of {n_row} tokens do not fit a row of {k} samples and {S} tokens")
        off = 0
        for j, i in enumerate(members, 1):
            s = samples[i]
            n = len(s)
            ids[r, off:off + n] = s.input_ids
            seg[r, off:off + n] = s.segment_ids
            am[r, off:off + n] = j
            lab[r * k + j - 1] = s.label
            ei[r * k + j - 1] = s.example_index
            off += n
            count += 1
    t = {key: torch.from_numpy(v) for key, v in zip(GLUE_KEYS, (ids, seg, am, lab))}
    if pin:
        t = {key: v.pin_memory() for key, v in t.items()}
    batch = PackedBatch(t, count)
    batch.example_index = ei
    return batch


def unpack_glue(batch):
    """The examples of a packed GLUE batch in slot order (the inverse of to_glue_batch)."""
    ids, seg, am, lab = (batch[key].cpu().numpy() for key in GLUE_KEYS)
    k = lab.shape[0] // ids.shape[0]
    out = []
    for r in range(ids.shape[0]):
        for j in range(1, k + 1):
            sel = am[r] == j
            if sel.any():
                slot = r * k + j - 1
                out.append(GlueSample(ids[r][sel], seg[r][sel], lab[slot], batch.example_index[slot]))
    return out


SWAG_KEYS = ("input_ids", "input_mask", "segment_ids", "label_ids")


def _check_choices(k, num_choices):
    if num_choices < 1 or k < 1 or k % num_choices != 0:
        raise ValueError(f"max_per_row must be a positive multiple of num_choices = {num_choices}, got {k}")


def split_swag_samples(batch, first_example_index=0):
    """The examples of an unpacked SWAG batch (input_ids, input_mask, segment_ids [N, C, S_choice] with right-padded 0/1 masks,
    label_ids [N]): per choice the tokens whose mask is 1, example index first_example_index + n.  An example none of whose choices
    holds a token holds no example; one with some empty choices raises ValueError (its scores would not line up with its label)."""
    ids, am, seg, lab = (batch[key].cpu().numpy() for key in SWAG_KEYS)
    if am.ndim != 3:
        raise ValueError(f"split_swag_samples takes [N, C, S] tensors, got input_mask of shape {tuple(am.shape)}")
    if am.min(initial=0) < 0 or am.max(initial=0) > 1:
        raise ValueError("split_swag_samples takes an unpacked batch: input_mask must hold only 0 and 1")
    out = []
    for n in range(ids.shape[0]):
        keep = am[n] != 0
        has = keep.any(-1)
        if not has.any():
            continue
        if not has.all():
            raise ValueError(f"example {first_example_index + n}: choices {np.nonzero(~has)[0].tolist()} hold no token")
        out.append(SwagSample([ids[n, c][keep[c]] for c in range(ids.shape[1])], [seg[n, c][keep[c]] for c in range(ids.shape[1])],
                              lab[n], first_example_index + n))
    return out


def to_swag_batch(samples, rows, B, S, k, num_choices, pin=False):
    """The packed SWAG batch (PackedBatch of CPU int64 tensors, with example_index) with the examples rows[r] in row r; rows past
    len(rows) and groups past a row's examples are empty (label -100, example index -1).  ValueError when k is not a positive multiple
    of num_choices, or a row exceeds S tokens or k/num_choices examples, or an example does not hold num_choices choices."""
    _check_choices(k, num_choices)
    C, E = num_choices, k // num_choices
    ids = np.zeros((B, S), np.int64)
    seg = np.zeros((B, S), np.int64)
    am = np.zeros((B, S), np.int64)
    lab = np.full(B * E, GLUE_IGNORE, np.int64)
    ei = np.full(B * E, -1, np.int64)
    if len(rows) > B:
        raise ValueError(f"{len(rows)} rows do not fit a batch of {B}")
    count = 0
    for r, members in enumerate(rows):
        n_row = sum(len(samples[i]) for i in members)
        if n_row > S or len(members) > E:
            raise ValueError(f"row {r}: {len(members)} examples of {n_row} tokens do not fit a row of {E} examples and {S} tokens")
        off = 0
        for m, i in enumerate(members):
            s = samples[i]
            if len(s.input_ids) != C:
                raise ValueError(f"example {s.example_index} holds {len(s.input_ids)} choices, not {C}")
            for c in range(C):
                n = len(s.input_ids[c])
                ids[r, off:off + n] = s.input_ids[c]
                seg[r, off:off + n] = s.segment_ids[c]
                am[r, off:off + n] = m * C + c + 1
                off += n
            lab[r * E + m] = s.label
            ei[r * E + m] = s.example_index
            count += 1
    t = {key: torch.from_numpy(v) for key, v in zip(SWAG_KEYS, (ids, am, seg, lab))}
    if pin:
        t = {key: v.pin_memory() for key, v in t.items()}
    batch = PackedBatch(t, count)
    batch.example_index = ei
    return batch


def unpack_swag(batch, num_choices):
    """The examples of a packed SWAG batch in group order (the inverse of to_swag_batch)."""
    ids, am, seg, lab = (batch[key].cpu().numpy() for key in SWAG_KEYS)
    C, E = num_choices, lab.shape[0] // ids.shape[0]
    out = []
    for r in range(ids.shape[0]):
        for m in range(E):
            sels = [am[r] == m * C + c + 1 for c in range(C)]
            if any(sel.any() for sel in sels):
                g = r * E + m
                out.append(SwagSample([ids[r][sel] for sel in sels], [seg[r][sel] for sel in sels], lab[g], batch.example_index[g]))
    return out


def token_fill(batch):
    """Share of the batch's B*S token slots that hold a sample token."""
    am = batch["input_mask"] if "input_mask" in batch else batch["attention_mask"]
    return float((am != 0).sum()) / am.numel()


class PackedLoader:
    """Packs the batches of any loader of unpacked lddl-format batches (five int64 tensors, 0/1 attention_mask) into PackedBatches of
    exactly `batch_size` rows.  Samples are drawn into a pool until it holds `pool_rows` * batch_size * seq_len tokens (or the source
    ends), packed first-fit decreasing, and what finds no room carries over to the next batch.  When the source ends the pool is
    packed out, so the last batches may hold rows without samples.  Deterministic for a deterministic source.

    squad=True packs unpacked SQuAD batches (SQUAD_KEYS, 0/1 input_mask) into the packed SQuAD format instead; max_pred is unused
    then, and feature indices count the source's rows from 0.  glue=True does the same for unpacked GLUE batches (GLUE_KEYS) and
    the packed GLUE format, with example indices counting the source's rows from 0.  swag=True packs unpacked SWAG batches
    (SWAG_KEYS, [N, C, S_choice]) into the packed SWAG format: whole examples of num_choices choices, at most max_per_row /
    num_choices of them per row (max_per_row counts sample slots and must be a multiple of num_choices)."""

    def __init__(self, source, batch_size, seq_len, max_per_row, max_pred=0, pool_rows=2, pin=False, squad=False, glue=False,
                 swag=False, num_choices=4):
        if max_per_row < 1:
            raise ValueError(f"max_per_row must be >= 1, got {max_per_row}")
        if squad + glue + swag > 1:
            raise ValueError("PackedLoader packs one format: pass one of squad=True, glue=True or swag=True")
        if swag:
            _check_choices(max_per_row, num_choices)
        self.source, self.B, self.S, self.k, self.P = source, batch_size, seq_len, max_per_row, max_pred
        self.pool_tokens, self.pin, self.squad, self.glue = pool_rows * batch_size * seq_len, pin, squad, glue
        self.swag, self.C = swag, num_choices

    def __iter__(self):
        pool, it, done = [], iter(self.source), False
        rows_seen = 0
        while True:
            tokens = sum(len(s) for s in pool)
            while not done and tokens < self.pool_tokens:
                try:
                    batch = next(it)
                except StopIteration:
                    done = True
                    break
                if self.squad or self.glue or self.swag:
                    split = split_squad_samples if self.squad else split_glue_samples if self.glue else split_swag_samples
                    new = split(batch, rows_seen)
                    rows_seen += batch["input_ids"].shape[0]
                else:
                    new = split_samples(batch, self.P)
                pool += new
                tokens += sum(len(s) for s in new)
            if not pool:
                return
            if self.swag:
                rows, unplaced = pack(pool, self.B, self.S, self.k // self.C, self.P)
                yield to_swag_batch(pool, rows, self.B, self.S, self.k, self.C, self.pin)
            else:
                rows, unplaced = pack(pool, self.B, self.S, self.k, self.P)
                fmt = to_squad_batch if self.squad else to_glue_batch if self.glue else to_batch
                yield fmt(pool, rows, self.B, self.S, self.k, self.pin)
            pool = [pool[i] for i in unplaced]


def synthetic_varlen_batch(B, S, vocab, max_pred, seed=42, round_to=1, mlm_fraction=0.15, pin=False):
    """An unpacked lddl-format batch of right-padded samples: lengths ~ U{S/4..S} rounded up to `round_to` (capped at S), [CLS] first,
    token type 1 on the second half of each sample, MLM labels on round(mlm_fraction * length) real tokens after [CLS] (at least one,
    at most max_pred), random NSP labels."""
    g = torch.Generator().manual_seed(seed)
    lens = ((torch.randint(S // 4, S + 1, (B,), generator=g) + round_to - 1) // round_to * round_to).clamp(max=S)
    ids = torch.randint(0, min(vocab, 30522), (B, S), generator=g, dtype=torch.int64)
    ids[:, 0] = 101
    pos = torch.arange(S).unsqueeze(0)
    am = (pos < lens.unsqueeze(1)).to(torch.int64)
    tt = ((pos >= (lens // 2).unsqueeze(1)) & (am != 0)).to(torch.int64)
    labels = torch.full((B, S), -1, dtype=torch.int64)
    for b in range(B):
        n = int(lens[b])
        n_lab = min(max_pred, max(1, round(mlm_fraction * n)), n - 1)
        where = 1 + torch.randperm(n - 1, generator=g)[:n_lab]
        labels[b, where] = torch.randint(0, min(vocab, 30522), (n_lab,), generator=g)
    nsl = torch.randint(0, 2, (B,), generator=g, dtype=torch.int64)
    batch = {"input_ids": ids, "token_type_ids": tt, "attention_mask": am, "labels": labels, "next_sentence_labels": nsl}
    if pin:
        batch = {k: v.pin_memory() for k, v in batch.items()}
    return batch
