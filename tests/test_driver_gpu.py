"""GPU: the driver mirror end to end on a small config -- train, checkpoint in the reference format, resume, phase-2 reset."""
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

CFG = dict(attention_probs_dropout_prob=0.1, hidden_act="gelu", hidden_dropout_prob=0.1, hidden_size=256, initializer_range=0.02,
           intermediate_size=1024, max_position_embeddings=128, num_attention_heads=4, num_hidden_layers=2, type_vocab_size=2, vocab_size=1021)


def _run(tmp_path, extra):
    from deeplearningexamples_b200 import run_pretraining as rp
    cfg = tmp_path / "cfg.json"
    cfg.write_text(json.dumps(CFG))
    argv = ["--config_file", str(cfg), "--output_dir", str(tmp_path / "out"), "--input_dir", "synthetic", "--do_train", "--fp16",
            "--allreduce_post_accumulation", "--allreduce_post_accumulation_fp16", "--train_batch_size", "4", "--max_seq_length", "128",
            "--max_predictions_per_seq", "10", "--learning_rate", "2e-3", "--warmup_proportion", "0.1", "--json-summary",
            str(tmp_path / "log.json"), "--disable_jit_fusions", "--init_loss_scale", "1024"] + extra
    return rp.main(argv)


def test_train_checkpoint_resume_and_phase2(tmp_path):
    args, t_raw, model_step, skip, final_loss, _ = _run(tmp_path, ["--max_steps", "8", "--num_steps_per_checkpoint", "4"])
    out = tmp_path / "out"
    assert model_step == 8 and final_loss == final_loss
    assert sorted(os.listdir(out)) == ["ckpt_4.pt", "ckpt_8.pt"]
    ck = torch.load(out / "ckpt_8.pt", weights_only=False)
    assert set(ck) == {"model", "optimizer", "grad_scaler", "epoch"}                      # run_pretraining.py:500-503
    assert "bert.encoder.layer.1.attention.self.value.bias" in ck["model"] and "cls.predictions.decoder.weight" in ck["model"]
    assert ck["model"]["bert.embeddings.word_embeddings.weight"].shape == (1024, 256)   # vocab padded to a multiple of 8 (:383-384)
    pg = ck["optimizer"]["param_groups"]
    assert pg[0]["step"].item() == 8 and pg[0]["step"].dtype == torch.int32 and pg[0]["lr"].dtype == torch.float32
    st = ck["optimizer"]["state"]
    assert all(v["exp_avg"].dtype == torch.float32 and v["exp_avg_sq"].dtype == torch.float32 for v in st.values())
    # resume: continues from step 8 to 12, keeps the newest checkpoints
    args2, *_ = _run(tmp_path, ["--max_steps", "12", "--num_steps_per_checkpoint", "4", "--resume_from_checkpoint"])
    assert args2.resume_step == 8
    ck12 = torch.load(out / "ckpt_12.pt", weights_only=False)
    assert ck12["optimizer"]["param_groups"][0]["step"].item() == 12
    assert not torch.equal(ck12["model"]["bert.encoder.layer.0.output.dense.weight"], ck["model"]["bert.encoder.layer.0.output.dense.weight"])
    # phase 2 from the phase-1 checkpoint: optimizer step and lr restart, file names are offset by phase1_end_step (:442-445,:496-499)
    args3, *_ = _run(tmp_path, ["--max_steps", "3", "--phase2", "--resume_from_checkpoint", "--phase1_end_step", "12",
                                "--learning_rate", "1e-3", "--skip_checkpoint"])
    assert args3.resume_step == 12
    lines = [json.loads(l) for l in open(tmp_path / "log.json")]
    assert any("final_loss" in l["data"] for l in lines)


def test_gradient_accumulation_matches_reference_batch_split(tmp_path):
    """train_batch_size is divided by the accumulation steps (:363); 2 micro-steps of 2 == 1 optimizer step."""
    args, t_raw, model_step, *_ = _run(tmp_path, ["--max_steps", "3", "--gradient_accumulation_steps", "2", "--skip_checkpoint"])
    assert args.train_batch_size == 2 and model_step == 6


def test_gradient_accumulation_under_cuda_graphs(tmp_path):
    """The same batch split with --cuda_graphs: the micro-steps replay the accumulation graph, every second step the full-step graph.
    The capture's 14 warm-ups take optimizer steps, so the schedule runs past them (--max_steps 100); the run stops after 3 steps."""
    args, t_raw, model_step, skip, final_loss, _ = _run(tmp_path, ["--max_steps", "100", "--steps_this_run", "3", "--cuda_graphs",
                                                                   "--gradient_accumulation_steps", "2", "--skip_checkpoint"])
    assert args.train_batch_size == 2 and model_step == 6
    assert 0.0 < final_loss < 12.0
