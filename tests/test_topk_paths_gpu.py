"""The three top-k paths behind `rpx_index_topk` — tensor core (any Q), HBM-streaming (Q <= 2) and
exact fp64 — each pinned through the C ABI against the C oracle (`oracle/rpx_oracle.c`): indices and
fp64 scores bit-exact under (score desc, index asc).  Includes the inputs the fp32 fast paths cannot
rank by themselves (near-ties far below fp32 accumulation noise): the exactness guard must hand those
queries to the exact pass, and the guard's epsilon must dominate the observed fp32 error."""
import numpy as np
import pytest
import torch

from oracle import c_oracle
from reprover_b200 import _native, synth
from reprover_b200.retrieval_ops import IndexHandle, sim_topk, topk_merge, topk_merge_packed

pytestmark = pytest.mark.gpu

MMA, STREAM, EXACT, AUTO = _native.RPX_TOPK_FORCE_MMA, _native.RPX_TOPK_FORCE_STREAM, _native.RPX_TOPK_FORCE_EXACT, 0


def _unit(n, d, seed, dev):
    return synth.random_unit_rows(n, d, seed, dev)


def _pack_mask(m):
    nq, n = m.shape
    words = np.zeros((nq, (n + 31) // 32 * 32), dtype=bool)
    words[:, :n] = m
    return np.packbits(words.reshape(nq, -1, 8), axis=2, bitorder="little").reshape(nq, -1).view("<u4").copy()


def _check(Q, E, k, flags, mask_words=None, idx_offset=0):
    handle = E if isinstance(E, IndexHandle) else IndexHandle(E)
    dev_mask = None if mask_words is None else torch.from_numpy(mask_words.view(np.int32)).to(Q.device)
    s32, idx, cnt, s64, packed = sim_topk(Q, handle, k, access_mask=dev_mask, idx_offset=idx_offset, want_scores64=True,
                                          want_packed=True, flags=flags)
    torch.cuda.synchronize()
    ws, wi, wc = c_oracle.sim_topk(c_oracle.bf16_bits(Q), c_oracle.bf16_bits(handle.embeddings), k, mask_words, idx_offset)
    gi, gs, gc = idx.cpu().numpy(), s64.cpu().numpy(), cnt.cpu().numpy()
    assert np.array_equal(gc, wc), (gc[:8], wc[:8])
    bad = np.argwhere(gi != wi)
    assert bad.size == 0, f"{len(bad)} index mismatches, first at {bad[:5].tolist()}: got {gi[tuple(bad[0])]} want {wi[tuple(bad[0])]}"
    assert np.array_equal(gs, ws)
    assert np.array_equal(s32.cpu().numpy(), ws.astype(np.float32))
    # the packed records are the same results, interleaved (fp64 bits, index)
    assert torch.equal(packed[..., 0].contiguous().view(torch.float64), s64) and torch.equal(packed[..., 1], idx)
    return handle


@pytest.mark.parametrize("nq", [1, 2])
@pytest.mark.parametrize("n,d,k", [(50_000, 1472, 100), (1000, 128, 10), (37, 64, 100), (20_001, 256, 200), (7, 1472, 3)])
def test_streaming_path_matches_oracle(rpx_lib, cuda_device, nq, n, d, k):
    h = _check(_unit(nq, d, 100 + nq, cuda_device), _unit(n, d, 200 + n % 97, cuda_device), k, STREAM, idx_offset=123_456)
    st = h.stats()
    assert st["n_exact"] == 0, st                   # ordinary data never needs the exact pass ...
    assert st["max_err"] <= 0.25 * st["max_eps"], st  # ... and the guard's bound is far above the observed error


def test_streaming_path_with_access_mask_skips_hidden_rows(rpx_lib, cuda_device):
    nq, n, d, k = 4, 30_000, 1472, 100
    rng = np.random.default_rng(1)
    m = np.zeros((nq, n), dtype=bool)
    for q in range(nq):   # accessibility = a few contiguous file ranges + a prefix of one file (common.py:280-289)
        for _ in range(5):
            a = int(rng.integers(0, n - 3000))
            m[q, a:a + int(rng.integers(100, 3000))] = True
    m[3, :] = False
    m[3, [0, 1, 29_999]] = True   # fewer than k accessible: count 3
    words = _pack_mask(m)
    Q, E = _unit(nq, d, 1, cuda_device), _unit(n, d, 2, cuda_device)
    _check(Q[:2], E, k, STREAM, mask_words=words[:2])
    _check(Q[2:], E, k, STREAM, mask_words=words[2:])   # holds the row with 3 accessible premises
    _check(Q[:1], E, k, STREAM, mask_words=words[:1])
    _check(Q, E, k, MMA, mask_words=words)


def test_streaming_path_refuses_three_queries(rpx_lib, cuda_device):
    Q, E = _unit(3, 256, 13, cuda_device), _unit(1000, 256, 14, cuda_device)
    with pytest.raises(_native.RpxError) as err:
        sim_topk(Q, E, 10, flags=STREAM)
    assert err.value.code == _native.RPX_ERR_UNSUPPORTED


def test_streaming_path_full_size_like_the_provers_call(rpx_lib, cuda_device):
    """BASELINE-sized index (200k x 1472), ONE state, k = 100, a realistic access mask (imports = long runs
    of files, plus a prefix of the own file): the shape `retrieve()` runs at (retrieval/model.py:338-375)."""
    n, d, k = 200_000, 1472, 100
    E, Q = _unit(n, d, 61, cuda_device), _unit(1, d, 62, cuda_device)
    m = np.zeros((1, n), dtype=bool)
    m[0, : 150_000] = True          # everything imported ...
    m[0, 40_000:55_000] = False     # ... except a few files that are not
    m[0, 150_000:150_037] = True    # premises of the own file before the theorem
    h = _check(Q, E, k, AUTO, mask_words=_pack_mask(m))
    assert h.stats()["n_exact"] == 0
    _check(Q, h, k, AUTO)           # and without a mask, through the same handle


@pytest.mark.parametrize("flags,nq", [(MMA, 1), (MMA, 4), (MMA, 130), (EXACT, 3), (AUTO, 5)])
def test_forced_paths_agree_with_oracle(rpx_lib, cuda_device, flags, nq):
    _check(_unit(nq, 1472, 7, cuda_device), _unit(9001, 1472, 8, cuda_device), 100, flags)


@pytest.mark.parametrize("k", [201, 500, 1024])
def test_large_k_goes_through_the_exact_pass(rpx_lib, cuda_device, k):
    h = _check(_unit(3, 256, 9, cuda_device), _unit(3000, 256, 10, cuda_device), k, AUTO)
    assert h.stats()["n_exact"] == 3
    _check(_unit(2, 128, 11, cuda_device), _unit(40, 128, 12, cuda_device), k, AUTO)   # k > n: count = n


def _near_ties(n, d, seed, dev):
    """One unit vector + a +-1-ulp (bf16) perturbation of ONE coordinate per row: fp64 score gaps of
    ~1e-9..1e-6, at or below the fp32 accumulation noise of either fast path."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    u = torch.nn.functional.normalize(torch.randn(d, generator=g), dim=0).to(torch.bfloat16)
    bits = u.view(torch.int16).to(torch.int32)
    rows = bits.repeat(n, 1)
    col = torch.randint(0, d, (n,), generator=g)
    delta = torch.randint(0, 2, (n,), generator=g) * 2 - 1
    rows[torch.arange(n), col] += delta.to(torch.int32)
    return rows.to(torch.int16).view(torch.bfloat16).to(dev)


@pytest.mark.parametrize("flags,nq", [(STREAM, 1), (STREAM, 2), (MMA, 5), (MMA, 130)])
@pytest.mark.parametrize("masked", [False, True])
def test_near_ties_below_fp32_noise_are_ranked_exactly(rpx_lib, cuda_device, flags, nq, masked):
    n, d, k = 5000, 1472, 100
    E = _near_ties(n, d, 3, cuda_device)
    Q = _unit(nq, d, 4, cuda_device)
    words = None
    if masked:
        rng = np.random.default_rng(5)
        words = _pack_mask(rng.random((nq, n)) < 0.6)
    h = _check(Q, E, k, flags, mask_words=words)
    st = h.stats()
    print("guard stats", flags, nq, masked, st)
    if flags == MMA:
        assert st["n_exact"] == nq, st   # every query was flagged by its guard and recomputed exactly
    else:
        pass  # the streaming path ranks its candidates by exact fp64 scores and may prove these queries by itself


def test_near_tie_cluster_inside_a_large_corpus(rpx_lib, cuda_device):
    """A cluster of 300 near-duplicates that straddles the k-th place of an ordinary 60k corpus."""
    d, k = 1472, 100
    E = _unit(60_000, d, 21, cuda_device)
    q = _unit(1, d, 22, cuda_device)
    cluster = _near_ties(300, d, 23, cuda_device).float()
    # aim the cluster at the query so that its scores sit around rank ~50..350
    s = (E.float() @ q.float().t()).flatten().sort(descending=True).values
    target = float(s[60])
    base = torch.nn.functional.normalize(cluster[0], dim=0)
    qn = torch.nn.functional.normalize(q.float()[0], dim=0)
    ortho = torch.nn.functional.normalize(base - (base @ qn) * qn, dim=0)
    c = target / float(q.float().norm())
    mix = c * qn + (1 - c * c) ** 0.5 * ortho
    rows = (cluster - cluster[0] + mix).to(torch.bfloat16)
    pos = torch.randperm(60_000, generator=torch.Generator().manual_seed(1))[:300].to(cuda_device)
    E[pos] = rows
    for flags, Q in ((STREAM, q), (MMA, torch.cat([q, _unit(4, d, 24, cuda_device)]))):
        _check(Q, E.clone(), k, flags)


def test_bit_identical_copies_at_the_kth_place(rpx_lib, cuda_device):
    """400 copies of one row whose score sits at about rank 60 of a 20k corpus, k = 100: the k-th place is a tie
    of bit-identical scores, cut by index.  More ties than the streaming kernel's ranking buffer holds, so it
    hands the query to the exact pass, which cuts the tie on the indices."""
    n, d, k = 20_000, 1472, 100
    E = _unit(n, d, 51, cuda_device)
    Q = _unit(5, d, 52, cuda_device)
    s = (E.float() @ Q[0].float()).sort(descending=True)
    pos = torch.randperm(n, generator=torch.Generator().manual_seed(53))[:400].to(cuda_device)
    E[pos] = E[s.indices[60]].clone()
    for flags, nq in ((STREAM, 1), (STREAM, 2), (MMA, 5), (EXACT, 5)):
        _check(Q[:nq], E.clone(), k, flags)


def test_handle_follows_in_place_updates_of_the_index(rpx_lib, cuda_device):
    E = _unit(4000, 256, 31, cuda_device)
    Q = _unit(2, 256, 32, cuda_device)
    a = sim_topk(Q, E, 10)[1].clone()
    E[a[0, 0]] = 0   # in-place edit bumps the tensor version -> a fresh handle (new row-norm bound, same storage)
    b = sim_topk(Q, E, 10)[1]
    assert a[0, 0] not in b[0].tolist()
    ws, wi, wc = c_oracle.sim_topk(c_oracle.bf16_bits(Q), c_oracle.bf16_bits(E), 10)
    assert np.array_equal(b.cpu().numpy(), wi)


def test_merge_packed_equals_merge(rpx_lib, cuda_device):
    nq, d, k, R = 70, 256, 100, 4
    Q = _unit(nq, d, 19, cuda_device)
    shards = [_unit(3000 + 17 * r, d, 20 + r, cuda_device) for r in range(R)]
    offs = np.concatenate([[0], np.cumsum([s.shape[0] for s in shards])])
    parts = [sim_topk(Q, shards[r], k, idx_offset=int(offs[r]), want_scores64=True, want_packed=True) for r in range(R)]
    a = topk_merge(torch.stack([p[3] for p in parts]), torch.stack([p[1] for p in parts]))
    b = topk_merge_packed(torch.stack([p[4] for p in parts]).contiguous())
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    one = sim_topk(Q, torch.cat(shards), k, want_scores64=True)
    assert torch.equal(one[1], b[1]) and torch.equal(one[3], b[3])


def test_one_shot_abi_form_matches_handle_form(rpx_lib, cuda_device):
    """rpx_sim_topk (no handle: state in the workspace, norm pass per call) == rpx_index_topk."""
    import ctypes as C

    Q, E, k = _unit(3, 128, 41, cuda_device), _unit(2500, 128, 42, cuda_device), 20
    want = sim_topk(Q, E, k, want_scores64=True)
    need = rpx_lib.rpx_sim_topk_workspace_bytes(E.shape[0], 128, 3, k)
    ws = torch.empty(need, dtype=torch.uint8, device=cuda_device)
    s = torch.empty(3, k, dtype=torch.float32, device=cuda_device)
    s64 = torch.empty(3, k, dtype=torch.float64, device=cuda_device)
    i = torch.empty(3, k, dtype=torch.int64, device=cuda_device)
    c = torch.empty(3, dtype=torch.int32, device=cuda_device)
    _native.check(rpx_lib.rpx_sim_topk(Q.data_ptr(), 3, E.data_ptr(), E.shape[0], 128, k, None, 0, s.data_ptr(), s64.data_ptr(),
                                       i.data_ptr(), c.data_ptr(), 0, ws.data_ptr(), ws.numel(),
                                       torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert torch.equal(i, want[1]) and torch.equal(s64, want[3]) and torch.equal(s, want[0]) and torch.equal(c, want[2])
