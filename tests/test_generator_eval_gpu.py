"""The generator's validation path on the H100: `evaluate` (one prefill for the loss and the search) against
`__call__` + `generate` bit for bit, its errors, `generator_eval.validate` against a restatement of the reference's
`validation_step` loop fed the engine's own per-batch outputs, `load` of a Lightning checkpoint against `from_hf_dir`
of the converted directory, and `predict_cli predict` -> `generator_cli validate` end to end."""
import ctypes as C
import json
import os

import pytest
import torch

from reprover_b200 import _native, synth
from reprover_b200.generator import T5GeneratorEngine

pytestmark = pytest.mark.gpu
EOS = 1
CFG = dict(synth.tiny_config(2), num_decoder_layers=2, decoder_start_token_id=0)


@pytest.fixture(scope="module")
def gen(cuda_device):
    sd = synth.random_t5_seq2seq_state_dict(CFG, seed=51)
    engine = T5GeneratorEngine(CFG, sd, cuda_device)
    yield sd, engine
    engine.close()


def _batch(in_lens, out_lens, seed):
    g = torch.Generator().manual_seed(seed)
    B = len(in_lens)
    ids = torch.zeros(B, max(in_lens), dtype=torch.int64)
    mask = torch.zeros_like(ids)
    labels = torch.full((B, max(out_lens)), -100, dtype=torch.int64)
    for i, (n, m) in enumerate(zip(in_lens, out_lens)):
        ids[i, :n] = torch.randint(3, CFG["vocab_size"], (n,), generator=g)
        ids[i, n - 1] = EOS
        mask[i, :n] = 1
        labels[i, :m] = torch.randint(3, CFG["vocab_size"], (m,), generator=g)
        labels[i, m - 1] = EOS
    return ids, mask, labels


def _bits_equal(a, b):
    assert a.dtype == b.dtype and a.shape == b.shape
    if a.is_floating_point():   # bits, so that NaN equals NaN
        a, b = a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8)
    assert torch.equal(a, b)


@pytest.mark.parametrize("nb,n_ret", [(1, 1), (4, 3), (8, 5)])
@pytest.mark.parametrize("masked", [True, False])
def test_evaluate_equals_call_and_generate(gen, nb, n_ret, masked):
    _, engine = gen
    if masked:
        ids, mask, labels = _batch([300, 7, 129, 64], [20, 1, 33, 9], seed=nb)
    else:
        ids, _, labels = _batch([96, 96, 96], [5, 17, 12], seed=nb + 100)
        mask = None
    kw = dict(max_length=40, num_beams=nb, num_return_sequences=n_ret, length_penalty=1.0, do_sample=False,
              early_stopping=False, output_scores=True, return_dict_in_generate=True)
    loss_out, gen_out = engine.evaluate(ids, mask, labels, return_logits=True, **kw)
    steps = engine.last_steps
    want_loss = engine(ids, mask, labels)
    want_gen = engine.generate(ids, mask, **kw)
    traced, trace = engine.generate(ids, mask, _trace_steps=1, **kw)
    for got, want in zip(loss_out, want_loss):
        _bits_equal(got, want)
    _bits_equal(gen_out.sequences, want_gen.sequences)
    _bits_equal(traced.sequences, want_gen.sequences)
    if nb > 1:
        _bits_equal(gen_out.sequences_scores, want_gen.sequences_scores)
    else:
        assert gen_out.sequences_scores is None and want_gen.sequences_scores is None
    assert steps == trace["steps"] > 0
    # the plain call shape returns the sequences tensor, as `generate` does
    plain_loss, plain = engine.evaluate(ids, mask, labels, max_length=40, num_beams=nb, num_return_sequences=n_ret)
    assert plain_loss.logits is None
    _bits_equal(plain_loss.loss, want_loss.loss)
    _bits_equal(plain, engine.generate(ids, mask, max_length=40, num_beams=nb, num_return_sequences=n_ret))


def test_evaluate_errors(gen):
    _, engine = gen
    ids, mask, labels = _batch([50, 20], [6, 4], seed=3)
    bad = labels.clone()
    bad[1, 0] = CFG["vocab_size"]
    with pytest.raises(_native.RpxError, match="labels must be -100"):
        engine.evaluate(ids, mask, bad, max_length=10)
    bad[1, 0] = -5
    with pytest.raises(_native.RpxError, match="labels must be -100"):
        engine.evaluate(ids, mask, bad, max_length=10)
    with pytest.raises(NotImplementedError, match="do_sample"):
        engine.evaluate(ids, mask, labels, max_length=10, do_sample=True)
    # a workspace one byte short
    lib, dev = engine.lib, engine.device
    B, L_in, L_out, nb, ML = 2, ids.shape[1], labels.shape[1], 4, 10
    need = lib.rpx_seq2seq_evaluate_workspace_bytes(engine._handle, engine.encoder._handle, B, L_in, L_out, nb, ML)
    assert need > 0
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    d_ids, d_mask, d_lab = (t.to(dev).contiguous() for t in (ids, mask, labels))
    seq_lp = torch.empty(B, dtype=torch.float64, device=dev)
    seq_n = torch.empty(B, dtype=torch.int32, device=dev)
    seqs = torch.empty(B * nb, ML, dtype=torch.int64, device=dev)
    scores = torch.empty(B * nb, dtype=torch.float32, device=dev)
    out_len, steps = C.c_int32(0), C.c_int32(0)

    def call(nbytes):
        return lib.rpx_seq2seq_evaluate(engine._handle, engine.encoder._handle, d_ids.data_ptr(), d_mask.data_ptr(),
                                        B, L_in, d_lab.data_ptr(), L_out, None, seq_lp.data_ptr(), seq_n.data_ptr(),
                                        nb, nb, ML, 1.0, EOS, seqs.data_ptr(), scores.data_ptr(), C.byref(out_len),
                                        C.byref(steps), ws.data_ptr(), nbytes, torch.cuda.current_stream().cuda_stream)

    assert call(need - 1) == _native.RPX_ERR_WORKSPACE
    assert call(need) == _native.RPX_OK
    assert out_len.value >= 2


# ---------------------------------------------------------------------------------------------- dataset level
MAX_INP, MAX_OUP = 300, 64


def _reference_validation(engine, examples, batch_size, nb):
    """The reference's `validation_step` loop and Lightning's epoch-end reduction, restated over the engine's
    `__call__` and `generate` and HF's `ByT5Tokenizer.batch_decode`."""
    from transformers import ByT5Tokenizer

    from reprover_b200.corpus import remove_marks
    from reprover_b200.generator_eval import collate

    tok = ByT5Tokenizer()
    loss_sum, size_sum, correct, total = 0.0, 0, [0] * nb, 0
    for lo in range(0, len(examples), batch_size):
        batch = collate(examples[lo:lo + batch_size], MAX_INP, MAX_OUP)
        loss = engine(batch["state_ids"], batch["state_mask"], batch["tactic_ids"]).loss
        output = engine.generate(batch["state_ids"], batch["state_mask"], max_length=MAX_OUP, num_beams=nb,
                                 do_sample=False, num_return_sequences=nb, early_stopping=False)
        text = tok.batch_decode(output.cpu(), skip_special_tokens=True)
        bs = batch["state_ids"].size(0)
        preds = [text[i * nb:(i + 1) * nb] for i in range(bs)]
        loss_sum += float(loss) * bs
        size_sum += bs
        for k in range(1, nb + 1):
            for p, gt in zip(preds, batch["tactic"]):
                correct[k - 1] += remove_marks(gt) in [remove_marks(x) for x in p][:k]
        total += bs
    return {"loss_val": loss_sum / size_sum, **{f"top{k}_acc_val": correct[k - 1] / total for k in range(1, nb + 1)}}


def _plant_tactics(engine, data_path, nb):
    """Rewrites val.json so that some tactics are, with marks, the engine's j-th prediction for their state (j
    cycling over the beams and a miss), which makes every top-k accuracy a nontrivial count."""
    from reprover_b200.generator_eval import collate, load_examples, validation_step

    path = os.path.join(data_path, "val.json")
    examples = load_examples(path)
    preds = []
    for lo in range(0, len(examples), 8):
        preds += validation_step(engine, collate(examples[lo:lo + 8], MAX_INP, MAX_OUP), nb, MAX_OUP)[1]
    with open(path) as fh:
        thms = json.load(fh)
    i = 0
    for thm in thms:
        for tac in thm["traced_tactics"]:
            j = i % (nb + 1)
            if j < nb and preds[i][j]:
                tac["tactic"] = f"<a>{preds[i][j][:3]}</a>{preds[i][j][3:]}"
            i += 1
    with open(path, "w") as fh:
        json.dump(thms, fh)


@pytest.fixture(scope="module")
def dataset(tmp_path_factory, gen):
    tmp = tmp_path_factory.mktemp("genval")
    data = synth.write_leandojo_dataset(str(tmp / "ds"), n_files=4, premises_per_file=20, theorems=(4, 9, 2),
                                        state_len=(16, 250), premise_len=(16, 120), min_accessible=10, seed=29)
    _plant_tactics(gen[1], data, 2)
    return tmp, data


def test_validate_equals_the_reference_loop(gen, dataset):
    from reprover_b200.generator_eval import load_examples, validate

    _, engine = gen
    _, data = dataset
    examples = load_examples(os.path.join(data, "val.json"))
    assert len(examples) % 6 != 0          # a partial last batch
    got = validate(engine, examples, batch_size=6, num_beams=2, max_inp_seq_len=MAX_INP, max_oup_seq_len=MAX_OUP)
    want = _reference_validation(engine, examples, 6, 2)
    assert got == want
    assert 0 < got["top1_acc_val"] < got["top2_acc_val"] < 1


def _generator_ckpt(tmp, sd, retriever_sd):
    """What the reference's ModelCheckpoint writes for a generator trained with `ret_ckpt_path`."""
    path = tmp / "generator.ckpt"
    state = {f"generator.{k}": v for k, v in sd.items()}
    state.update({f"retriever.encoder.{k}": v for k, v in retriever_sd.items()})
    torch.save({"epoch": 2, "global_step": 40, "state_dict": state,
                "hyper_parameters": {"model_name": "not-cached/byt5-nowhere", "lr": 5e-4, "warmup_steps": 2000,
                                     "num_beams": 3, "length_penalty": 0.0, "eval_num_retrieved": 100,
                                     "eval_num_workers": 1, "eval_num_gpus": 1, "eval_num_theorems": 0,
                                     "max_inp_seq_len": 999, "max_oup_seq_len": 999, "ret_ckpt_path": "r.ckpt"}},
               path)
    return path


def test_load_equals_from_hf_dir_of_the_converted_directory(gen, tmp_path, cuda_device):
    from reprover_b200 import convert_cli

    sd, _ = gen
    ckpt = _generator_ckpt(tmp_path, sd, synth.random_t5_state_dict(synth.tiny_config(1), seed=5))
    loaded = T5GeneratorEngine.load(str(ckpt), cuda_device)
    assert loaded.hparams["num_beams"] == 3 and loaded.hparams["max_oup_seq_len"] == 999
    convert_cli.main(["generator", "--src", str(ckpt), "--dst", str(tmp_path / "hf")])
    hf = T5GeneratorEngine.from_hf_dir(str(tmp_path / "hf"), cuda_device)
    ids, mask, labels = _batch([80, 31], [12, 6], seed=8)
    a = loaded.evaluate(ids, mask, labels, return_logits=True, max_length=24, num_beams=4, num_return_sequences=4,
                        output_scores=True, return_dict_in_generate=True)
    b = hf.evaluate(ids, mask, labels, return_logits=True, max_length=24, num_beams=4, num_return_sequences=4,
                    output_scores=True, return_dict_in_generate=True)
    for x, y in zip(a[0], b[0]):
        _bits_equal(x, y)
    for x, y in zip(a[1], b[1]):
        _bits_equal(x, y)
    loaded.close()
    hf.close()


@pytest.mark.parametrize("native_layout", [False, True])
def test_predict_then_validate_end_to_end(gen, dataset, tmp_path, capsys, native_layout):
    from reprover_b200 import generator_cli, predict_cli
    from reprover_b200.generator_eval import load_examples, load_predictions, validate

    sd, engine = gen
    tmp, data = dataset
    corpus = os.path.join(data, "../corpus.jsonl")
    ret_sd = synth.random_t5_state_dict(synth.tiny_config(1), seed=5)
    ret_ckpt = tmp_path / "retriever.ckpt"
    torch.save({"state_dict": {f"encoder.{k}": v for k, v in ret_sd.items()},
                "hyper_parameters": {"model_name": "not-cached/byt5-nowhere", "max_seq_len": 256,
                                     "num_retrieved": 10}}, ret_ckpt)
    preds_path = tmp_path / "predictions.pickle"
    predict_cli.main(["predict", "--ckpt_path", str(ret_ckpt), "--data.data_path", data, "--data.corpus_path", corpus,
                      "--data.eval_batch_size", "8", "--output-path", str(preds_path)]
                     + (["--native-layout"] if native_layout else []))
    cfg = tmp_path / "cli.yaml"
    cfg.write_text(f"seed_everything: 3407\ntrainer:\n  devices: 1\nmodel:\n  model_name: google/byt5-small\n"
                   f"  num_beams: 2\n  eval_num_theorems: 250\n  ret_ckpt_path: null\n"
                   f"data:\n  data_path: {data}\n  corpus_path: {corpus}\n  preds_path: null\n  eval_batch_size: 4\n"
                   f"  max_inp_seq_len: {MAX_INP}\n  max_oup_seq_len: {MAX_OUP}\n  p_drop: 0.5\n")
    ckpt = _generator_ckpt(tmp_path, sd, ret_sd)
    capsys.readouterr()
    metrics = generator_cli.main(["validate", "--config", str(cfg), "--ckpt_path", str(ckpt),
                                  "--data.preds_path", str(preds_path)])
    printed = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    preds = load_predictions(str(preds_path))
    examples = load_examples(os.path.join(data, "val.json"), preds, MAX_INP)
    assert any(len(ex["state"].encode()) > 250 for ex in examples)    # premises were prepended
    want = validate(engine, examples, batch_size=4, num_beams=2, max_inp_seq_len=MAX_INP, max_oup_seq_len=MAX_OUP)
    assert printed == metrics == want
    assert set(want) == {"loss_val", "top1_acc_val", "top2_acc_val"}
