"""CPU checks of the reference-facing shims: the unmodified reference driver imports over both arms, the lddl stand-in yields the
batch format the driver consumes (run_pretraining.py:520-521,603-609) with LDDL-style sequence binning from memory and from parquet,
the dllogger stand-in writes the records the driver logs."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
THIRD = os.path.join(ROOT, "shims", "thirdparty")
sys.path.insert(0, ROOT)
from oracle.build_ref import REF_BERT as REF  # noqa: E402


@pytest.fixture()
def third_on_path():
    sys.path.insert(0, THIRD)
    yield
    sys.path.remove(THIRD)
    for m in [m for m in sys.modules if m.split(".")[0] in ("lddl", "dllogger")]:
        del sys.modules[m]


@pytest.mark.parametrize("arm", ["ours", "reference"])
def test_unmodified_reference_driver_imports_and_parses_its_flags(arm):
    if not os.path.exists(os.path.join(REF, "run_pretraining.py")):
        pytest.skip("no reference checkout")
    if arm == "reference":
        from oracle import build_ref
        if build_ref.built_path() is None:
            pytest.skip("oracle/_ref not built")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_reference_driver.py"), "--arm", arm, "--", "--help"],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "--allreduce_post_accumulation_fp16" in r.stdout and "--cuda_graphs" in r.stdout


def test_lddl_stand_in_batches_are_binned_and_well_formed(third_on_path):
    import lddl.torch as lt
    loader = lt.get_bert_pretrain_data_loader("synthetic?seq_len=512&max_pred=80&samples=512&bin_size=64", local_rank=0,
                                              data_loader_kwargs={"batch_size": 4, "num_workers": 0, "pin_memory": False}, base_seed=7)
    assert len(loader) == 512 // 4
    seen = set()
    for i, b in enumerate(loader):
        assert set(b) == {"input_ids", "token_type_ids", "attention_mask", "labels", "next_sentence_labels"}
        S = b["input_ids"].shape[1]
        assert all(v.dtype == torch.int64 for v in b.values()) and b["next_sentence_labels"].shape == (4,)
        assert S % 64 == 0 and S <= 512
        lens = b["attention_mask"].sum(1)
        assert (lens > S - 64).all() and (lens <= S).all()                      # every sequence belongs to this batch's length bin
        assert (b["input_ids"][:, 0] == 101).all()
        n_masked = (b["labels"] != -1).sum(1)
        assert (n_masked >= 1).all() and (n_masked <= 80).all()
        assert ((b["labels"] != -1) <= (b["attention_mask"] == 1)).all()         # masked positions lie inside the sequence
        seen.add(S)
        if i >= 40:
            break
    assert len(seen) >= 3
    # every rank draws the same bin sequence (same shapes per step under DDP), different samples
    a = lt.get_bert_pretrain_data_loader("synthetic?seq_len=512&samples=512&bin_size=64", local_rank=0, data_loader_kwargs={"batch_size": 4}, base_seed=7)
    os.environ["RANK"], os.environ["WORLD_SIZE"] = "1", "2"
    try:
        c = lt.get_bert_pretrain_data_loader("synthetic?seq_len=512&samples=512&bin_size=64", local_rank=1, data_loader_kwargs={"batch_size": 4}, base_seed=7)
    finally:
        del os.environ["RANK"], os.environ["WORLD_SIZE"]
    sa = [b["input_ids"].shape[1] for _, b in zip(range(8), a)]
    sc = [b["input_ids"].shape[1] for _, b in zip(range(8), c)]
    assert sa == sc
    assert not torch.equal(next(iter(a))["input_ids"], next(iter(c))["input_ids"])


def test_lddl_stand_in_reads_parquet_shards(third_on_path, tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import make_synthetic_lddl as mk
    finally:
        sys.path.remove(os.path.join(ROOT, "tools"))
    out = str(tmp_path / "ds")
    mk.main(["--out", out, "--samples", "256", "--seq-len", "256", "--bin-size", "64", "--max-pred", "38", "--shards", "2"])
    assert os.path.exists(os.path.join(out, "meta.json"))
    import lddl.torch as lt
    loader = lt.get_bert_pretrain_data_loader(out, local_rank=0, data_loader_kwargs={"batch_size": 8, "pin_memory": False}, base_seed=3)
    b = next(iter(loader))
    assert b["input_ids"].shape[0] == 8 and b["input_ids"].shape[1] in (64, 128, 192, 256)
    assert (b["labels"] != -1).sum() > 0 and b["token_type_ids"].max() == 1


def test_dllogger_stand_in_records(third_on_path, tmp_path):
    import dllogger
    f = str(tmp_path / "log.json")
    dllogger.init(backends=[dllogger.JSONStreamBackend(verbosity=dllogger.Verbosity.VERBOSE, filename=f),
                            dllogger.StdOutBackend(verbosity=dllogger.Verbosity.VERBOSE, step_format=lambda s: str(s))])
    dllogger.metadata("training_sequences_per_second", {"unit": "sequences/s"})
    dllogger.log(step=(0, 3), data={"average_loss": 1.5})
    dllogger.log(step=tuple(), data={"training_sequences_per_second": 10.0})
    dllogger.flush()
    recs = [json.loads(l[5:]) for l in open(f) if l.startswith("DLLL ")]
    assert recs[0]["type"] == "METADATA" and recs[1]["step"] == [0, 3] and recs[2]["data"]["training_sequences_per_second"] == 10.0
