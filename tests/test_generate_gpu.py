"""Generation on the H100: the decode self-attention kernel against the float64 reference of
tests/decode_attention_ref.py (with exact cases), the traced step log-probs against HF and the engine's own forward,
the search bookkeeping against tests/beam_ref.py fed the same log-probs (exact), batch invariance, errors and bounds."""
import pytest
import torch

from reprover_b200 import _native, synth
from reprover_b200.generator import T5GeneratorEngine
from tests import beam_ref
from tests import decode_attention_ref as DA
from tests import seq2seq_ref as S

pytestmark = pytest.mark.gpu
H = 6
INNER = H * 64
EOS = 1


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _decode(lib, case, dev, lin=True):
    ML, R, _ = case.cache.shape
    cache = case.cache.to(dev).bfloat16().contiguous()
    lin_d = case.lin.to(dev).int().contiguous() if lin else None
    lut = case.lut.to(dev).contiguous()
    out = torch.full((R + 1, INNER), float("nan"), dtype=torch.bfloat16, device=dev)
    _native.check(lib.rpx_debug_decode_attention(cache.data_ptr(), None if lin_d is None else lin_d.data_ptr(),
                                                 lut.data_ptr(), out.data_ptr(), case.t, R, ML, H, case.md, _stream()))
    torch.cuda.synchronize()
    assert bool(out[R].isnan().all()), "wrote past the last row"
    return out[:R]


@pytest.mark.parametrize("t,R", [(0, 1), (1, 8), (63, 64), (64, 128), (65, 8), (127, 64), (128, 1), (129, 128),
                                 (511, 64), (2047, 8)])
def test_decode_attention_against_float64(rpx_lib, cuda_device, t, R):
    case = DA.random_case(t, R, H=H, ML=t + 2, seed=1000 * t + R)
    out = _decode(rpx_lib, case, cuda_device)
    assert DA.check(out, case) == 0


def test_decode_attention_one_hot_routing(rpx_lib, cuda_device):
    """One hot row per launch: its query meets a huge q.k (256 per head) at one position of its own lineage, so that
    key's softmax weight is 1 and every other weight underflows to 0 (exp(-250)); the output is the slot lin routes
    to, bit for bit.  Every row of the case is checked."""
    t, R = 70, 8
    base = DA.random_case(t, R, H=H, ML=t + 2, seed=3)
    base.cache[..., :2 * INNER] = 0.0
    g = torch.Generator().manual_seed(4)
    checked = 0
    for r in range(R):
        case = DA.Case(base.cache.clone(), base.lin, base.lut, base.t, base.H, base.md)
        p = int(torch.randint(0, t + 1, (1,), generator=g))
        slot = int(case.lin[r, p])
        case.cache[t, r, :INNER] = 1.0                   # q of row r
        case.cache[p, slot, INNER:2 * INNER] = 4.0       # k at position p of row r's lineage
        out = _decode(rpx_lib, case, cuda_device)
        assert torch.equal(out[r].float().cpu(), case.cache[p, slot, 2 * INNER:].bfloat16().float()), (r, p, slot)
        checked += 1
    assert checked == R


def test_decode_attention_bias_readback(rpx_lib, cuda_device):
    """q = k = 0: the weights are softmax over p of lut[h][p - t]; one-hot values read them back across every
    unidirectional bucket (t = 700 > max distance 128)."""
    t, R = 700, 2
    case = DA.random_case(t, R, H=H, ML=t + 1, seed=5)
    case.cache.zero_()
    for p in range(t + 1):
        for s in range(R):
            for h in range(H):
                case.cache[p, s, 2 * INNER + 64 * h + p % 64] = 1.0
    out = _decode(rpx_lib, case, cuda_device)
    assert DA.check(out, case) == 0


def test_decode_attention_ignores_off_lineage_slots(rpx_lib, cuda_device):
    """A slot no row's lineage reaches, given a huge score and value, leaves every output bit-identical."""
    t, R = 100, 8
    case = DA.random_case(t, R, H=H, ML=t + 2, seed=6)
    base = _decode(rpx_lib, case, cuda_device)
    used = {(p, int(case.lin[r, p])) for r in range(R) for p in range(t + 1)}
    free = [(p, s) for p in range(t + 1) for s in range(R) if (p, s) not in used]
    assert free
    for p, s in free[:4]:
        case.cache[p, s, INNER:2 * INNER] = 30.0
        case.cache[p, s, 2 * INNER:] = 1e4
    out = _decode(rpx_lib, case, cuda_device)
    assert torch.equal(out.view(torch.int16), base.view(torch.int16))


# ---------------------------------------------------------------------------------------------- whole search
def _engine(cfg, seed):
    sd = synth.random_t5_seq2seq_state_dict(cfg, seed=seed)
    return sd, T5GeneratorEngine(cfg, sd, torch.device("cuda:0"))


def _states(cfg, lens, seed):
    g = torch.Generator().manual_seed(seed)
    L = max(lens)
    ids = torch.zeros(len(lens), L, dtype=torch.int64)
    mask = torch.zeros(len(lens), L, dtype=torch.int64)
    for i, n in enumerate(lens):
        ids[i, :n] = torch.randint(3, cfg["vocab_size"], (n,), generator=g)
        ids[i, n - 1] = EOS
        mask[i, :n] = 1
    return ids, mask


def _prefixes(trace, R, start=0):
    """The engine's prefixes [R, t + 1] at every traced step, rebuilt from the parents and tokens it recorded."""
    out = [torch.full((R, 1), start, dtype=torch.int64)]
    par, tok = trace["parents"].long().cpu(), trace["tokens"].long().cpu()
    for t in range(trace["steps"] - 1):
        p = par[t].clamp_min(0)
        out.append(torch.cat([out[-1][p], tok[t].clamp_min(0)[:, None]], 1))
    return out


def _replay(trace, R, nb):
    """beam_ref's step function: the engine's traced step scores, after checking that beam_ref asks for the prefixes
    the engine ran (rows of states whose search had ended are not traced; they get zeros, which cannot change a
    finished set)."""
    pre = _prefixes(trace, R)
    scores = trace["scores"].cpu()

    def step(t, prefixes):
        s = scores[t].clone()
        live = ~s.isnan().any(-1)
        assert torch.equal(prefixes[live], pre[t][live]), f"step {t}: beam_ref asks for other prefixes"
        s[~live] = 0.0
        return s

    return step


def _bookkeeping(gen, ids, mask, nb, n_ret, max_length, lp):
    out, trace = gen.generate(ids, mask, num_beams=nb, num_return_sequences=n_ret, max_length=max_length,
                              length_penalty=lp, output_scores=True, return_dict_in_generate=True,
                              _trace_steps=max_length)
    B = ids.shape[0]
    R = B * nb
    step = _replay(trace, R, nb)
    if nb == 1:
        want = beam_ref.greedy(step, B, max_length, EOS, 0, 0)
        assert torch.equal(out.sequences.cpu(), want)
        assert out.sequences_scores is None
    else:
        want, want_scores = beam_ref.beam_search(step, B, nb, n_ret, max_length, lp, EOS, 0, 0)
        assert torch.equal(out.sequences.cpu(), want)
        assert torch.equal(out.sequences_scores.cpu(), want_scores)
    return out, trace


@pytest.fixture(scope="module")
def tiny_gen():
    cfg = dict(synth.tiny_config(2), num_decoder_layers=2, decoder_start_token_id=0)
    sd, gen = _engine(cfg, 41)
    yield cfg, sd, gen
    gen.close()


@pytest.mark.parametrize("nb,n_ret,lp", [(1, 1, 1.0), (4, 4, 0.0), (4, 2, 1.0), (8, 3, -0.5)])
def test_bookkeeping_exact_tiny(cuda_device, tiny_gen, nb, n_ret, lp):
    cfg, _, gen = tiny_gen
    ids, mask = _states(cfg, [40, 7, 300], seed=nb)
    _bookkeeping(gen, ids, mask, nb, n_ret, 48, lp)


def test_bookkeeping_exact_full_geometry_prover_shape(cuda_device):
    cfg = dict(synth.BYT5_SMALL, decoder_start_token_id=0)
    sd, gen = _engine(cfg, 43)
    ids, mask = _states(cfg, [2300], seed=44)
    out, trace = _bookkeeping(gen, ids, mask, 64, 64, 512, 0.0)
    assert out.sequences.shape[0] == 64
    gen.close()


@pytest.fixture
def fp32_matmul():
    """HF's fp32 reference without TF32 matmuls, restored afterwards."""
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


def test_step_numerics_against_hf_and_the_engine_forward(tmp_path, cuda_device, tiny_gen, fp32_matmul):
    """Traced step log-probs against HF fp32 teacher-forced on the same prefixes: no worse than HF bf16 (floor 0.05);
    against the engine's own rpx_seq2seq_forward on those prefixes: within 0.02."""
    from transformers import T5ForConditionalGeneration

    cfg, sd, gen = tiny_gen
    ids, mask = _states(cfg, [40, 7, 300], seed=9)
    nb = 4
    _, trace = gen.generate(ids, mask, num_beams=nb, num_return_sequences=nb, max_length=40, length_penalty=1.0,
                            return_dict_in_generate=True, output_scores=True, _trace_steps=40)
    pre = _prefixes(trace, ids.shape[0] * nb)
    synth.save_hf_checkpoint(str(tmp_path), cfg, sd)
    enc_ids, enc_mask = ids.repeat_interleave(nb, 0).cuda(), mask.repeat_interleave(nb, 0).cuda()
    errs = {}
    for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        m = T5ForConditionalGeneration.from_pretrained(str(tmp_path), torch_dtype=dt).cuda().eval()
        res = []
        for t in (0, 5, 20, 38):
            with torch.no_grad():
                lg = m(input_ids=enc_ids, attention_mask=enc_mask, decoder_input_ids=pre[t].cuda()).logits[:, -1]
            res.append(torch.log_softmax(lg.float(), -1))
        errs[name] = res
        del m
    e_eng = e_bf = 0.0
    for i, t in enumerate((0, 5, 20, 38)):
        got = trace["scores"][t]
        live = ~got.isnan().any(-1)
        e_eng = max(e_eng, float((got[live] - errs["fp32"][i][live]).abs().max()))
        e_bf = max(e_bf, float((errs["bf16"][i][live] - errs["fp32"][i][live]).abs().max()))
    assert e_eng <= max(e_bf, 0.05), (e_eng, e_bf)
    # the engine's teacher-forced forward on the step-38 prefixes: the last position's log-prob of each next token
    t = 38
    tok = trace["tokens"][t].long().cpu()
    labels = torch.cat([pre[t][:, 1:], tok[:, None]], 1)
    fwd = gen(input_ids=enc_ids, attention_mask=enc_mask, labels=labels.cuda())
    lp_fwd = torch.log_softmax(fwd.logits[:, -1].double(), -1)
    got = trace["scores"][t].double()
    live = ~got.isnan().any(-1)
    assert float((got[live] - lp_fwd[live]).abs().max()) <= 0.02


def _gen_lengths(seqs: torch.Tensor) -> torch.Tensor:
    """Generated tokens per row of [N, L_out] sequences: through the first EOS, else the whole row."""
    body = seqs[:, 1:]
    n = torch.full((seqs.shape[0],), body.shape[1], dtype=torch.int64)
    for r in range(seqs.shape[0]):
        e = (body[r] == EOS).nonzero()
        if len(e):
            n[r] = int(e[0]) + 1
    return n


def _widen(seqs: torch.Tensor, L: int, fill: int) -> torch.Tensor:
    out = torch.full((seqs.shape[0], L), fill, dtype=seqs.dtype)
    out[:, :seqs.shape[1]] = seqs
    return out


@pytest.fixture(scope="module")
def bf16_exact_gen():
    """The tiny geometry with every weight rounded to bf16, so HF's fp32 model and the engine hold the same weights
    and the measured error is the engine's arithmetic alone."""
    cfg = dict(synth.tiny_config(2), num_decoder_layers=2, decoder_start_token_id=0)
    sd = {k: v.bfloat16().float() for k, v in synth.random_t5_seq2seq_state_dict(cfg, seed=45).items()}
    gen = T5GeneratorEngine(cfg, sd, torch.device("cuda:0"))
    yield cfg, sd, gen
    gen.close()


@pytest.mark.parametrize("nb,lp,max_length", [(1, 1.0, 6), (2, 0.0, 3), (2, 1.0, 3)])
def test_end_to_end_against_hf_generate(tmp_path, cuda_device, bf16_exact_gen, fp32_matmul, nb, lp, max_length):
    """The engine's generate against HF `generate` in fp32 on the GPU, for the states whose search HF decided by a
    clear margin.  The engine's per-step error `err` is measured here: its step-0 scores against HF's (the same
    prefixes) and its last traced step against HF fp32 teacher-forced on the engine's prefixes.  Each state's
    smallest decision margin comes from replaying HF's own step scores through tests/beam_ref.py (which must
    reproduce HF's sequences).  States whose margin exceeds 2 err must match HF's sequences exactly and its scores
    within 2 err per summed log-prob; at least half the states must be checkable.  Every returned score times
    len ** lp must equal the sequence's float64 teacher-forced log-likelihood (tests/seq2seq_ref.py) within
    2 err per token + 1e-4."""
    cfg, sd, gen = bf16_exact_gen
    lens = [40, 7, 300, 64, 1, 129, 17, 200, 90, 33, 2, 250, 65, 128, 12, 180, 5, 77, 310, 21, 99, 140, 3, 56]
    B = len(lens)
    ids, mask = _states(cfg, lens, seed=20 + nb + int(lp))
    out, trace = gen.generate(ids, mask, num_beams=nb, num_return_sequences=nb, max_length=max_length,
                              length_penalty=lp, output_scores=True, return_dict_in_generate=True,
                              _trace_steps=max_length)
    synth.save_hf_checkpoint(str(tmp_path), cfg, sd)
    m = S.hf_model_from_dir(str(tmp_path)).cuda()
    with torch.no_grad():
        hf = m.generate(input_ids=ids.cuda(), attention_mask=mask.cuda(), num_beams=nb, num_return_sequences=nb,
                        max_length=max_length, length_penalty=lp, do_sample=False, early_stopping=False,
                        output_scores=True, return_dict_in_generate=True)
    hf_scores = [x.float().cpu() for x in hf.scores]
    R = B * nb
    pre = _prefixes(trace, R)
    err = float((trace["scores"][0].cpu() - hf_scores[0]).abs().max())
    tl = trace["steps"] - 1
    enc_ids, enc_mask = ids.repeat_interleave(nb, 0).cuda(), mask.repeat_interleave(nb, 0).cuda()
    with torch.no_grad():
        lg = m(input_ids=enc_ids, attention_mask=enc_mask, decoder_input_ids=pre[tl].cuda()).logits[:, -1].float()
    want = torch.log_softmax(lg, -1) if nb > 1 else lg
    got = trace["scores"][tl]
    live = ~got.isnan().any(-1)
    err = max(err, float((got[live] - want[live]).abs().max()))
    del m
    st = beam_ref.SearchStats()
    step = lambda t, prefixes: hf_scores[t]  # noqa: E731
    if nb == 1:
        replay = beam_ref.greedy(step, B, max_length, EOS, 0, 0, stats=st)
    else:
        replay, _ = beam_ref.beam_search(step, B, nb, nb, max_length, lp, EOS, 0, 0, stats=st)
    hf_seqs = hf.sequences.cpu()
    assert torch.equal(replay, hf_seqs), "the restatement does not reproduce HF's search from HF's own scores"
    checkable = [b for b in range(B) if st.margins[b] > 2 * err]
    assert len(checkable) >= B / 2, (err, st.margins)
    fill = 0 if nb == 1 else EOS
    eng_seqs = out.sequences.cpu()
    L = max(eng_seqs.shape[1], hf_seqs.shape[1])
    eng_w, hf_w = _widen(eng_seqs, L, fill), _widen(hf_seqs, L, fill)
    for b in checkable:
        rows = slice(b * nb, (b + 1) * nb)
        assert torch.equal(eng_w[rows], hf_w[rows]), (b, st.margins[b], err)
    if nb == 1:
        assert out.sequences_scores is None
        return
    n_gen = _gen_lengths(eng_seqs).double()
    got_sc = out.sequences_scores.cpu().double()
    for b in checkable:
        rows = slice(b * nb, (b + 1) * nb)
        tol = 2 * err * n_gen[rows] ** (1 - lp) + 1e-5
        assert bool(((got_sc[rows] - hf.sequences_scores.cpu().double()[rows]).abs() <= tol).all()), b
    labels = eng_seqs[:, 1:].clone()
    for r in range(labels.shape[0]):
        labels[r, int(n_gen[r]):] = S.IGNORE
    ll = S.forward(cfg, sd, ids.repeat_interleave(nb, 0), mask.repeat_interleave(nb, 0), labels)["sequence_log_probs"]
    dev = (got_sc * n_gen ** lp - ll).abs()
    assert bool((dev <= 2 * err * n_gen + 1e-4).all()), (float(dev.max()), err)


def test_batch_invariance(cuda_device, tiny_gen):
    cfg, _, gen = tiny_gen
    lens = [300, 17, 2300, 64, 65, 1, 128, 900]
    ids, mask = _states(cfg, lens, seed=12)
    for nb, n_ret in ((1, 1), (4, 4)):
        big = gen.generate(ids, mask, num_beams=nb, num_return_sequences=n_ret, max_length=40, length_penalty=1.0,
                           output_scores=True, return_dict_in_generate=True)
        for b in (0, 2, 5):
            one = gen.generate(ids[b:b + 1, :lens[b]], mask[b:b + 1, :lens[b]], num_beams=nb, num_return_sequences=n_ret,
                               max_length=40, length_penalty=1.0, output_scores=True, return_dict_in_generate=True)
            rows = slice(b * n_ret, (b + 1) * n_ret)
            L = one.sequences.shape[1]
            assert torch.equal(one.sequences, big.sequences[rows, :L]), (nb, b)
            fill = 0 if nb == 1 else EOS
            assert bool((big.sequences[rows, L:] == fill).all())
            if nb > 1:
                assert torch.equal(one.sequences_scores, big.sequences_scores[rows]), (nb, b)


def test_errors_and_bounds(cuda_device, tiny_gen):
    cfg, _, gen = tiny_gen
    lib = gen.lib
    ids, mask = _states(cfg, [30, 20], seed=14)
    bad = ids.clone()
    bad[1, 3] = cfg["vocab_size"]
    with pytest.raises(_native.RpxError) as ei:
        gen.generate(bad, mask, num_beams=2, max_length=5)
    assert ei.value.code == _native.RPX_ERR_INVALID
    bm = mask.clone()
    bm[0, 0] = 0
    with pytest.raises(_native.RpxError) as ei:
        gen.generate(ids, bm, num_beams=2, max_length=5)
    assert ei.value.code == _native.RPX_ERR_MASK
    for kw in ({"do_sample": True}, {"no_repeat_ngram_size": 2}, {"max_new_tokens": 4}, {"early_stopping": True}):
        with pytest.raises(NotImplementedError):
            gen.generate(ids, mask, num_beams=2, **kw)
    with pytest.raises(ValueError):
        gen.generate(ids, mask, num_beams=2, num_return_sequences=3)
    with pytest.raises(NotImplementedError, match="pad_token_id"):
        gen.generate(ids, mask, num_beams=2, pad_token_id=5)
    # HF's `model.to(device).eval()`, as the reference's HuggingFaceGenerator.initialize calls it
    assert gen.to(cuda_device).eval() is gen and gen.to("cuda") is gen
    with pytest.raises(ValueError):
        gen.to("cpu")
    B, L_in, nb, n_ret, ML = 2, ids.shape[1], 4, 3, 12
    d_ids, d_mask = ids.cuda(), mask.cuda()
    need = lib.rpx_seq2seq_generate_workspace_bytes(gen._handle, gen.encoder._handle, B, L_in, nb, ML)
    assert need > 0
    import ctypes as C

    seqs = torch.full((B * n_ret * ML + 64,), -7, dtype=torch.int64, device=cuda_device)
    scores = torch.full((B * n_ret + 8,), float("nan"), device=cuda_device)
    out_len, steps = C.c_int32(0), C.c_int32(0)
    ws = torch.empty(need, dtype=torch.uint8, device=cuda_device)
    rc = lib.rpx_seq2seq_generate(gen._handle, gen.encoder._handle, d_ids.data_ptr(), d_mask.data_ptr(), B, L_in, nb,
                                  n_ret, ML, 1.0, EOS, seqs.data_ptr(), scores.data_ptr(), C.byref(out_len),
                                  C.byref(steps), None, ws.data_ptr(), need - 256, _stream())
    assert rc == _native.RPX_ERR_WORKSPACE
    for bad_args in ((nb, nb + 1, ML), (nb, n_ret, 1), (cfg["vocab_size"], 1, ML), (129, 1, ML)):
        rc = lib.rpx_seq2seq_generate(gen._handle, gen.encoder._handle, d_ids.data_ptr(), d_mask.data_ptr(), B, L_in,
                                      bad_args[0], bad_args[1], bad_args[2], 1.0, EOS, seqs.data_ptr(),
                                      scores.data_ptr(), C.byref(out_len), C.byref(steps), None, ws.data_ptr(), need,
                                      _stream())
        assert rc == _native.RPX_ERR_INVALID, bad_args
    _native.check(lib.rpx_seq2seq_generate(gen._handle, gen.encoder._handle, d_ids.data_ptr(), d_mask.data_ptr(), B,
                                           L_in, nb, n_ret, ML, 1.0, EOS, seqs.data_ptr(), scores.data_ptr(),
                                           C.byref(out_len), C.byref(steps), None, ws.data_ptr(), need, _stream()))
    torch.cuda.synchronize()
    assert bool((seqs[B * n_ret * ML:] == -7).all()) and bool((seqs[:B * n_ret * ML] >= 0).all())
    assert bool(scores[B * n_ret:].isnan().all()) and not bool(scores[:B * n_ret].isnan().any())
    assert 2 <= out_len.value <= ML and 1 <= steps.value <= ML - 1
    ref = gen.generate(ids, mask, num_beams=nb, num_return_sequences=n_ret, max_length=ML, length_penalty=1.0,
                       output_scores=True, return_dict_in_generate=True)
    assert torch.equal(seqs[:B * n_ret * ML].view(B * n_ret, ML)[:, :out_len.value], ref.sequences)
    assert torch.equal(scores[:B * n_ret], ref.sequences_scores)
