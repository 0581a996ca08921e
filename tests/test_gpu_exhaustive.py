"""Exhaustive exact search (K7 + selection): every document scored against every query.

GPU tests are marked; the last two tests are the CPU tier (argument checks and the no-CPU-path error)."""

from __future__ import annotations

import ctypes

import pytest
import torch
from util import build_oracle_index, make_docs, make_queries, oracle_exact_scores, ranking_consistent, to_index_tensors

from oracle import plaid_oracle as po

SENTINEL = -10000.0


def _device_index(oidx, device, ivf: bool = True):
    from fast_plaid_b200.engine import DeviceIndex, IndexTensors

    t = to_index_tensors(oidx)
    if not ivf:
        t = IndexTensors(t.nbits, t.centroids, t.bucket_weights, t.doc_lengths, t.doc_codes, t.doc_residuals, None, None)
    return DeviceIndex(t, device)


def _oracle_all(oidx, queries: torch.Tensor) -> torch.Tensor:
    n = int(oidx.doc_lengths.shape[0])
    return torch.stack([oracle_exact_scores(oidx, queries[b], list(range(n))) for b in range(queries.shape[0])])


def _oracle_maxima(oidx, query: torch.Tensor) -> torch.Tensor:
    """The reference's fp16 per-query-token maxima of every document, [N, Q] (colbert_score_reduce before its sum)."""
    sel = torch.arange(int(oidx.doc_lengths.shape[0]), dtype=torch.int64)
    codes, lens = po.ragged_lookup(oidx.doc_codes, oidx.doc_offsets, oidx.doc_lengths, sel)
    res, _ = po.ragged_lookup(oidx.doc_residuals, oidx.doc_offsets, oidx.doc_lengths, sel)
    emb = po.decompress_residuals(res, oidx.bucket_weights, oidx.byte_reversed_bits_map,
                                  oidx.bucket_weight_indices_lookup, codes, oidx.centroids, oidx.dim, oidx.nbits)
    padded, mask = po.direct_pad_sequences(emb, lens, 0.0)
    ts = padded.matmul(query.half().unsqueeze(0).transpose(-2, -1))
    return ts.masked_fill(~mask.unsqueeze(-1).expand(ts.shape), -9999.0).max(dim=1).values


def _assert_scores_match(got: torch.Tensor, oidx, queries: torch.Tensor, what: str, didx) -> None:
    """Every score within 1e-3 relative of the reference.  Bit-identity is checked where each rounding happens:

    * the fp16 maxima: a one-token query scores exactly its fp16 maximum, so running every query token as its own
      query gives the kernel's maxima; fewer than 5 % may differ from the reference's (the CPU matmul and the tensor
      cores can round a dot product differently);
    * the sum: every score must be the exactly rounded sum of the kernel's own maxima, bit for bit;
    * the scores themselves: fewer than 5 % not bit-identical to the reference's fp32 running sum, up to Q = 100.
      At Q = 256 one differing maximum in 256 is enough to change a score, and that bound does not hold (see the
      first point for the bound that does)."""
    B, Q, D = queries.shape
    ref = _oracle_all(oidx, queries)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    tol = 1e-3 * ref.abs().clamp_min(1.0)
    bad = (got - ref).abs() > tol
    assert not bad.any(), f"{what}: {int(bad.sum())} scores off by more than 1e-3 relative, e.g. " \
                          f"{got[bad][:3].tolist()} vs {ref[bad][:3].tolist()}"
    maxima = didx.exhaustive_scores(queries.reshape(B * Q, 1, D).half().to(didx.device)).cpu()
    maxima = maxima.view(B, Q, -1).transpose(1, 2)  # [B, N, Q]
    ref_maxima = torch.stack([_oracle_maxima(oidx, queries[b]).float() for b in range(B)])
    flips = int((maxima != ref_maxima).sum())
    assert flips < 0.05 * ref_maxima.numel(), f"{what}: {flips}/{ref_maxima.numel()} fp16 maxima differ"
    assert torch.equal(got, maxima.double().sum(-1).float()), f"{what}: a score is not the exact sum of its maxima"
    if Q <= 100:
        differ = int((got != ref).sum())
        assert differ < 0.05 * ref.numel(), f"{what}: {differ}/{ref.numel()} scores are not bit-identical"


def _index_with_empty_and_long_docs(dim: int = 128, nbits: int = 4):
    """40 ragged documents, three 2000-token ones (longer than any tile) and one document without tokens."""
    docs = make_docs(40, 1, 40, dim=dim, seed=71) + make_docs(3, 2000, 2000, dim=dim, seed=72) \
        + make_docs(20, 1, 40, dim=dim, seed=73)
    oidx, _ = build_oracle_index(docs, nbits=nbits)
    empty_at = 17
    lens = oidx.doc_lengths.clone()
    lens = torch.cat([lens[:empty_at], torch.zeros(1, dtype=lens.dtype), lens[empty_at:]])
    o2 = po.OracleIndex(oidx.nbits, oidx.centroids, oidx.bucket_weights, None, None, oidx.doc_codes,
                        oidx.doc_residuals, lens)
    return o2, empty_at, docs


CONFIGS = [  # (dim, nbits, Q)
    (128, 4, 1), (128, 4, 20), (128, 4, 32), (128, 4, 64), (128, 4, 100), (128, 4, 256),
    (128, 2, 32), (64, 4, 32), (64, 2, 32), (64, 2, 100),
]


@pytest.mark.gpu
@pytest.mark.parametrize("dim,nbits,Q", CONFIGS)
def test_every_score_matches_the_oracle(dim, nbits, Q, cuda_device):
    docs = make_docs(150, 1, 40, dim=dim, seed=61 + Q)
    oidx, _ = build_oracle_index(docs, nbits=nbits)
    didx = _device_index(oidx, cuda_device)
    queries = make_queries(3, Q, dim=dim, seed=62 + Q, docs=docs)
    got = didx.exhaustive_scores(queries.half().to(cuda_device)).cpu()
    _assert_scores_match(got, oidx, queries, f"dim={dim} nbits={nbits} Q={Q}", didx)


@pytest.mark.gpu
@pytest.mark.parametrize("dim,nbits,Q", [(128, 4, 32), (128, 4, 100), (64, 2, 64)])
def test_empty_and_long_documents(dim, nbits, Q, cuda_device):
    oidx, empty_at, _ = _index_with_empty_and_long_docs(dim, nbits)
    didx = _device_index(oidx, cuda_device, ivf=False)
    queries = make_queries(4, Q, dim=dim, seed=74)
    got = didx.exhaustive_scores(queries.half().to(cuda_device)).cpu()
    assert torch.all(got[:, empty_at] == Q * SENTINEL)
    _assert_scores_match(got, oidx, queries, f"empty/long dim={dim} nbits={nbits} Q={Q}", didx)


@pytest.mark.gpu
@pytest.mark.parametrize("dim,nbits", [(128, 4), (64, 2)])
def test_chunks_of_many_documents(dim, nbits, cuda_device, monkeypatch):
    """Chunks of several documents: ragged lengths that start and end inside tiles and cross them, empty documents
    between, at the start and at the end of chunks, one document longer than two tiles.  Every chunk size gives
    every score of the oracle, and the same bytes."""
    lens = torch.randint(1, 121, (150,), generator=torch.Generator().manual_seed(151)).tolist()
    lens[40] = 700
    docs = []
    g = torch.Generator().manual_seed(152)
    for n in lens:
        docs.append(torch.nn.functional.normalize(torch.randn(n, dim, generator=g), dim=-1))
    oidx, _ = build_oracle_index(docs, nbits=nbits)
    empty = [0, 5, 6, 7, 31, 32, 63, 64, 100]  # positions after insertion; 5-7 consecutive
    lens_t = oidx.doc_lengths.tolist()
    for p in empty:
        lens_t.insert(p, 0)
    oidx = po.OracleIndex(oidx.nbits, oidx.centroids, oidx.bucket_weights, None, None, oidx.doc_codes,
                          oidx.doc_residuals, torch.tensor(lens_t, dtype=oidx.doc_lengths.dtype))
    didx = _device_index(oidx, cuda_device, ivf=False)
    queries = make_queries(3, 32, dim=dim, seed=153, docs=docs)
    q16 = queries.half().to(cuda_device)
    first = None
    for dpc in (32, 13, 4, 2, 1):
        monkeypatch.setenv("FPB_K7_DOCS_PER_CHUNK", str(dpc))
        got = didx.exhaustive_scores(q16).cpu()
        assert torch.all(got[:, empty] == 32 * SENTINEL)
        if first is None:
            _assert_scores_match(got, oidx, queries, f"chunks of {dpc} documents", didx)
            first = got
        else:
            assert torch.equal(got, first), f"chunks of {dpc} documents change the scores"


def _canonical(scores: torch.Tensor, k: int):
    """Stable sort by (-score, id): the (score desc, id asc) order."""
    n = scores.shape[0]
    order = sorted(range(n), key=lambda d: (-float(scores[d]), d))[:k]
    return order, [float(scores[d]) for d in order]


def _check_canonical_ranking(docs, copies, query_docs, device, tied_top: bool) -> None:
    """search_exhaustive at several k against the canonical sort of the exhaustive scores; `copies` are the indices
    of copies of document 3.  tied_top: also assert that the copies hold the top score of every query, more than
    2048 of them tied."""
    oidx, _ = build_oracle_index(docs)
    didx = _device_index(oidx, device)
    n = len(docs)
    queries = make_queries(5, 32, seed=82, docs=query_docs).half().to(device)
    scores = didx.exhaustive_scores(queries).cpu()
    assert torch.equal(scores[:, copies], scores[:, [3]].expand(-1, len(copies)))
    if tied_top:
        top = scores.max(dim=1, keepdim=True).values
        assert torch.equal(scores[:, [3]], top), "the copied document does not hold the top score"
        assert torch.all((scores == top).sum(dim=1) > 2048)
    for k in (1, 10, 124, n, 300, 4096):
        ids, sc, counts = (t.cpu() for t in didx.search_exhaustive(queries, k))
        assert ids.shape == (5, k) and sc.shape == (5, k)
        for b in range(5):
            exp_ids, exp_sc = _canonical(scores[b], k)
            m = min(k, n)
            assert int(counts[b]) == m
            assert ids[b, :m].tolist() == exp_ids, f"n={n} k={k} query {b}"
            assert sc[b, :m].tolist() == exp_sc
            assert torch.all(ids[b, m:] == -1) and torch.all(sc[b, m:] == float("-inf"))


@pytest.mark.gpu
def test_ranking_is_the_canonical_sort_with_ties(cuda_device):
    base = make_docs(120, 5, 30, seed=81)
    docs = base + [base[i].clone() for i in (3, 3, 50, 77, 119)]  # duplicated documents: exact ties
    _check_canonical_ranking(docs, [120, 121], docs, cuda_device, tied_top=False)
    # more than 2048 copies of document 3, and queries drawn from it: the copies tie at the top of every query, so for
    # every k <= 2048 the k-th best score lies in a value bucket of more than 2048 scores, more than k3b_select's
    # bucket fast path orders, and the radix passes must select the smallest ids among the copies
    docs = base + [base[3].clone() for _ in range(2100)]
    _check_canonical_ranking(docs, list(range(120, len(docs))), [base[3]], cuda_device, tied_top=True)


@pytest.mark.gpu
def test_exact_top_k_dominates_the_approximate_search(cuda_device):
    from fast_plaid_b200.engine import DeviceIndex

    docs = make_docs(1500, 10, 60, seed=91)
    oidx, _ = build_oracle_index(docs)
    didx = _device_index(oidx, cuda_device)
    queries = make_queries(8, 32, seed=92, docs=docs).half().to(cuda_device)
    k = 20
    ids, sc, counts = (t.cpu() for t in didx.search(queries, DeviceIndex.make_params(k, 64, 2)))
    eids, esc, ecounts = (t.cpu() for t in didx.search_exhaustive(queries, k))
    every = didx.exhaustive_scores(queries).cpu()
    assert torch.all(ecounts == k)
    for b in range(queries.shape[0]):
        for i in range(int(counts[b])):
            d, s = int(ids[b, i]), float(sc[b, i])
            ex = float(every[b, d])
            assert abs(ex - s) <= 1e-3 * max(1.0, abs(ex)), f"query {b} doc {d}: search {s} vs exhaustive {ex}"
            assert float(esc[b, i]) >= s - 1e-3 * max(1.0, abs(s)), f"query {b} rank {i}"


@pytest.mark.gpu
def test_compress_only_index_is_searchable_exhaustively(tmp_path, cuda_device):
    from fast_plaid_b200 import search
    from fast_plaid_b200.index import store

    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device=cuda_device)
    docs = make_docs(200, 5, 50, seed=101)
    fp.create(docs, kmeans_niters=2, compress_only=True)
    queries = make_queries(4, 32, seed=102, docs=docs)
    with pytest.raises(ValueError, match="compress_only"):
        fp.search(queries, top_k=5)
    res = fp.search_exhaustive(queries, top_k=10)
    data = store.read_index(path)
    assert data.ivf is None
    oidx = po.OracleIndex(data.nbits, data.centroids, data.bucket_weights, None, None, data.doc_codes,
                          data.doc_residuals, data.doc_lengths)
    ref = _oracle_all(oidx, queries)
    for b in range(4):
        assert len(res[b]) == 10
        ok, why = ranking_consistent([d for d, _ in res[b]], [s for _, s in res[b]],
                                     dict(enumerate(ref[b].tolist())), 1e-3)
        assert ok, why
        best = float(ref[b].max())
        assert abs(res[b][0][1] - best) <= 1e-3 * max(1.0, abs(best))
    fp.close()


@pytest.mark.gpu
def test_chunked_batch_and_repeated_calls_are_byte_identical(cuda_device):
    oidx, _, docs = _index_with_empty_and_long_docs()
    didx = _device_index(oidx, cuda_device, ivf=False)
    queries = make_queries(13, 48, seed=111).half().to(cuda_device)
    ids, sc, counts = didx.search_exhaustive(queries, 15)
    small = didx.exhaustive_workspace_bytes(3, 48, 15)  # about three queries per call
    ids2, sc2, counts2 = didx.search_exhaustive(queries, 15, budget_bytes=small)
    assert torch.equal(ids, ids2) and torch.equal(sc, sc2) and torch.equal(counts, counts2)
    a = didx.exhaustive_scores(queries)
    b = didx.exhaustive_scores(queries)
    parts = torch.cat([didx.exhaustive_scores(queries[s : s + 4]) for s in range(0, 13, 4)])
    assert torch.equal(a, b) and torch.equal(a, parts)
    ids3, sc3, counts3 = didx.search_exhaustive(queries, 15)
    assert torch.equal(ids, ids3) and torch.equal(sc, sc3) and torch.equal(counts, counts3)


def _fastplaid_index(tmp_path, device):
    from fast_plaid_b200 import search

    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device=device)
    docs = make_docs(250, 5, 60, seed=121)
    fp.create(docs, kmeans_niters=2)
    return path, fp, docs


@pytest.mark.gpu
def test_fastplaid_surface(tmp_path, cuda_device):
    path, fp, docs = _fastplaid_index(tmp_path, cuda_device)
    queries = make_queries(6, 32, seed=122, docs=docs)
    res = fp.search_exhaustive(queries, top_k=12)  # fp32 host input: the same fp16 cast as search
    res_dev = fp.search_exhaustive(queries.to(cuda_device).half(), top_k=12)
    assert res == res_dev
    for r in res:
        assert len(r) == 12 and all(isinstance(d, int) and isinstance(s, float) for d, s in r)
        assert len({d for d, _ in r}) == 12
        assert all(r[i][1] >= r[i + 1][1] for i in range(11))
    # list of queries of different lengths: zero-padded like `search`
    lst = [queries[0][:20], queries[1], queries[2][:7]]
    res_list = fp.search_exhaustive(lst, top_k=5)
    padded = torch.zeros(3, 32, 128)
    padded[0, :20], padded[1], padded[2, :7] = queries[0][:20], queries[1], queries[2][:7]
    assert res_list == fp.search_exhaustive(padded, top_k=5)
    assert res_list[1] == res[1][:5]
    with pytest.raises(ValueError):
        fp.search_exhaustive(queries[0], top_k=5)
    fp.close()


@pytest.mark.gpu
def test_two_devices_equal_one(tmp_path, cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from fast_plaid_b200 import search

    path, fp, docs = _fastplaid_index(tmp_path, cuda_device)
    queries = make_queries(7, 32, seed=131, docs=docs)
    one = fp.search_exhaustive(queries, top_k=10)
    fp.close()
    fp2 = search.FastPlaid(path, device=["cuda:0", "cuda:1"])
    assert fp2.search_exhaustive(queries, top_k=10) == one
    fp2.close()


def test_workspace_query_refuses_bad_arguments():
    from fast_plaid_b200.engine import FPB_ERR_INVALID, FPB_ERR_UNSUPPORTED, load_library

    lib = load_library()
    out = ctypes.c_size_t()
    assert lib.fpb_exhaustive_workspace_bytes(None, 4, 32, 10, ctypes.byref(out)) == FPB_ERR_INVALID
    assert b"NULL index" in lib.fpb_last_error()
    assert lib.fpb_exhaustive_workspace_bytes(None, 4, 32, 5000, ctypes.byref(out)) == FPB_ERR_UNSUPPORTED
    assert b"top_k=5000" in lib.fpb_last_error()
    assert lib.fpb_exhaustive_workspace_bytes(None, 4, 300, 10, ctypes.byref(out)) == FPB_ERR_UNSUPPORTED
    assert lib.fpb_exhaustive_scores(None, None, 4, 32, None, 0, None, None) == FPB_ERR_INVALID
    assert lib.fpb_search_exhaustive(None, None, 4, 32, 0, None, 0, None, None, None, None) == FPB_ERR_INVALID


def test_search_exhaustive_on_cpu_device_fails_loudly(tmp_path):
    from fast_plaid_b200 import search
    from fast_plaid_b200.engine import EngineUnavailableError

    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device="cpu")
    fp.create(make_docs(30, 5, 30, seed=141), kmeans_niters=2)
    with pytest.raises(EngineUnavailableError, match="no CPU search path"):
        fp.search_exhaustive(torch.randn(2, 8, 128), top_k=5)
    fp_sharded = search.FastPlaid.__new__(search.FastPlaid)
    fp_sharded.shard = (0, 2)
    with pytest.raises(NotImplementedError, match="document-sharded"):
        search.FastPlaid.search_exhaustive(fp_sharded, torch.randn(2, 8, 128))
