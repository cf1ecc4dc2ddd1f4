"""Dataset-level predict / validate on the H100: `evaluation.predict` against `predict_step` batch by batch and against
the C oracle's brute-force fp64 ranking, batch-size and token-budget invariance, `B200PremiseRetriever.load` of a
Lightning checkpoint against `load_hf` of the same weights, and `predict_cli` end to end."""
import json
import os
import pickle

import numpy as np
import pytest
import torch

from oracle import c_oracle
from reprover_b200 import synth
from reprover_b200.corpus import Corpus
from reprover_b200.evaluation import load_examples, predict, predict_step, validate
from reprover_b200.retriever import B200PremiseRetriever

pytestmark = pytest.mark.gpu
MAX_LEN = 256
K = 10


@pytest.fixture(scope="module")
def setup(tmp_path_factory, cuda_device):
    tmp = tmp_path_factory.mktemp("predict")
    data = synth.write_leandojo_dataset(str(tmp / "ds"), n_files=6, premises_per_file=40, theorems=(10, 5, 5),
                                        min_accessible=K, seed=17)
    cfg = synth.tiny_config(num_layers=2)
    sd = synth.random_t5_state_dict(cfg, seed=23)
    hf_dir = tmp / "hf"
    synth.save_hf_checkpoint(str(hf_dir), cfg, sd)
    ckpt = tmp / "retriever.ckpt"      # what the reference's ModelCheckpoint writes
    torch.save({"epoch": 1, "global_step": 10, "state_dict": {f"encoder.{k}": v for k, v in sd.items()},
                "hyper_parameters": {"model_name": str(hf_dir), "lr": 1e-4, "warmup_steps": 2000,
                                     "max_seq_len": MAX_LEN, "num_retrieved": K}}, ckpt)
    corpus = Corpus(os.path.join(data, "../corpus.jsonl"))
    retr = B200PremiseRetriever.load_hf(str(hf_dir), MAX_LEN, cuda_device)
    retr.num_retrieved = K
    retr.load_corpus(corpus)
    examples = load_examples(data, corpus)
    preds = predict(retr, examples, batch_size=8)
    return dict(tmp=tmp, data=data, hf_dir=hf_dir, ckpt=ckpt, corpus=corpus, retr=retr, examples=examples, preds=preds)


def _same_records(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert list(g) == list(w)
        for key in w:
            assert g[key] == w[key], key
        assert all(type(s) is float for s in g["scores"])


def test_predict_equals_predict_step_and_the_oracle_ranking(setup):
    r, examples, preds = setup["retr"], setup["examples"], setup["preds"]
    assert len(preds) == len(examples) > 40
    # predict_step encodes through retrieve_batch, which puts a batch of few tokens on the encoder's latency tiles
    # (other rounding); predict never does, so the comparison runs with that path off
    saved = r.state_latency_tokens
    r.state_latency_tokens = 0
    try:
        want = []
        for lo in range(0, len(examples), 8):
            part = examples[lo:lo + 8]
            want += predict_step(r, {key: [ex[key] for ex in part] for key in part[0]})
    finally:
        r.state_latency_tokens = saved
    _same_records(preds, want)
    # every ranking is the brute-force fp64 ranking of the engine's own embeddings under the reference's
    # accessibility walk (score desc, index asc)
    corpus = r.corpus
    q = r.encode_texts([ex["context"].serialize() for ex in examples])
    words = np.stack([corpus.accessible_mask_words(ex["context"].path, ex["context"].theorem_pos) for ex in examples])
    ws, wi, wc = c_oracle.sim_topk(c_oracle.bf16_bits(q), c_oracle.bf16_bits(r.corpus_embeddings), K, words)
    assert np.all(wc == K)
    index_of = {id(p): i for i, p in enumerate(corpus.all_premises)}
    got_i = np.array([[index_of[id(p)] for p in rec["retrieved_premises"]] for rec in preds])
    assert np.array_equal(got_i, wi)
    assert np.array_equal(np.array([rec["scores"] for rec in preds], dtype=np.float32), ws.astype(np.float32))
    assert any(rec["all_pos_premises"] for rec in preds) and any(not rec["all_pos_premises"] for rec in preds)


def test_batch_size_and_token_budget_invariance(setup):
    r, examples = setup["retr"], setup["examples"]
    base = pickle.dumps(setup["preds"])
    saved = r.encoder.max_tokens_per_call
    try:
        for budget, batch_size in ((saved, 3), (saved, 64), (MAX_LEN, 8), (700, 5)):
            r.encoder.max_tokens_per_call = budget
            assert pickle.dumps(predict(r, examples, batch_size=batch_size)) == base, (budget, batch_size)
    finally:
        r.encoder.max_tokens_per_call = saved


def test_load_checkpoint_equals_load_hf(setup, cuda_device):
    r = setup["retr"]
    r2 = B200PremiseRetriever.load(str(setup["ckpt"]), cuda_device, freeze=True)
    assert r2.max_seq_len == MAX_LEN and r2.num_retrieved == K and r2.model_name == str(setup["hf_dir"])
    r2.load_corpus(setup["corpus"])
    r2.reindex_corpus(batch_size=32)
    assert torch.equal(r2.corpus_embeddings, r.corpus_embeddings)
    _same_records(predict(r2, setup["examples"], batch_size=16), setup["preds"])


def test_cli_end_to_end(setup, tmp_path, capsys):
    from reprover_b200 import predict_cli
    from reprover_b200.compat import load_reference_predictions
    from tests.test_predict_cpu import _restated_eval

    cfg = tmp_path / "cli.yaml"
    cfg.write_text(f"seed_everything: 3407\ntrainer:\n  accelerator: gpu\n  devices: 1\n"
                   f"model:\n  model_name: google/byt5-small\n  num_retrieved: {K}\n"
                   f"data:\n  data_path: {setup['data']}\n  corpus_path: {os.path.join(setup['data'], '../corpus.jsonl')}\n"
                   f"  eval_batch_size: 8\n  max_seq_len: {MAX_LEN}\n")
    out = tmp_path / "predictions.pickle"
    predict_cli.main(["predict", "--config", str(cfg), "--ckpt_path", str(setup["ckpt"]), "--output-path", str(out)])
    with pytest.raises((ModuleNotFoundError, AttributeError)):      # the reference's classes, not this package's
        pickle.loads(out.read_bytes())
    got = load_reference_predictions(str(out))
    _same_records(got, setup["preds"])
    # what retrieval/evaluate.py reads: unique (file_path, full_name, start, tactic_idx) keys, positives, rankings
    preds_map = {(p["file_path"], p["full_name"], tuple(p["start"]), p["tactic_idx"]): p for p in got}
    assert len(preds_map) == len(got)
    for split in ("train", "val", "test"):
        with open(os.path.join(setup["data"], f"{split}.json")) as fh:
            r1, r10, mrr = _restated_eval(json.load(fh), preds_map)
        assert 0 <= r1 <= r10 <= 100 and 0 <= mrr <= 1
    capsys.readouterr()
    metrics = predict_cli.main(["validate", "--config", str(cfg), "--hf-ckpt", str(setup["hf_dir"]),
                                "--data.eval_batch_size", "3"])
    printed = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    want = validate(setup["retr"], load_examples(setup["data"], setup["corpus"], ("val",)), batch_size=8)
    assert printed == metrics == want
    assert set(want) == {f"Recall@{j}_val" for j in range(1, K + 1)} | {"MRR", "num_with_premises"}
