"""GPU parity tests: the CUDA engine (through the C ABI) against the CPU oracle.

What is bit-exact and what is toleranced (DESIGN.md "Parity contract"):
  * index / integer stages (probe cells, candidate ids, pruning, ranking) are compared
    exactly, under the canonical tie rule, on the GPU's own fp16 score table S;
  * the two fp32-accumulated dot products (S and the MaxSim token scores) and the fp32 norm
    may differ from ATen's CPU kernels by the accumulation order, i.e. by one fp16 ulp on a
    small fraction of entries -- the tests bound both the size (<= 1 ulp) and the fraction;
  * final scores: within 1e-3 relative (the tolerance BASELINE.json states).
"""

from __future__ import annotations

import pytest
import torch

from util import (build_oracle_index, fp16_ulp_diff, make_docs, make_queries, oracle_exact_scores,
                  oracle_token_matrix, ranking_consistent, to_index_tensors)

from oracle import plaid_oracle as po

pytestmark = pytest.mark.gpu

CONFIGS = {
    # name: (n_docs, min_len, max_len, dim, nbits, B, Q, top_k, n_full, n_probe, noisy_queries)
    "base": (1000, 30, 100, 128, 4, 8, 32, 10, 256, 8, True),
    "cfg1_shape": (400, 300, 300, 128, 4, 10, 50, 10, 4096, 8, False),
    "ragged_short": (600, 1, 40, 128, 4, 6, 32, 20, 128, 4, True),
    "nbits2": (500, 20, 80, 128, 2, 4, 32, 10, 256, 8, True),
    "dim64": (500, 20, 80, 64, 4, 4, 20, 10, 256, 8, True),
    "probe1": (500, 20, 80, 128, 4, 4, 16, 5, 64, 1, True),
    "q64": (300, 50, 120, 128, 4, 3, 64, 10, 256, 16, True),
    "q100": (300, 10, 90, 128, 4, 2, 100, 10, 256, 8, True),
    # every (dim, nbits) at query lengths past 32, up to the 256-token limit (Qp = 256: generic K5, K1 v1, and the
    # approximate stage with 32 lanes per S row)
    "q129": (300, 20, 90, 128, 4, 2, 129, 10, 256, 8, True),
    "q256": (300, 20, 90, 128, 4, 2, 256, 10, 256, 8, True),
    "nbits2_q100": (300, 20, 80, 128, 2, 2, 100, 10, 256, 8, True),
    "dim64_q64": (300, 20, 80, 64, 4, 3, 64, 10, 256, 8, True),
    "dim64_nbits2": (400, 20, 80, 64, 2, 3, 32, 10, 256, 8, True),
    "dim64_nbits2_q256": (300, 20, 80, 64, 2, 2, 256, 10, 256, 8, True),
}

_cache: dict = {}


def _setup(name: str, device: str):
    if name in _cache:
        return _cache[name]
    from fast_plaid_b200.engine import DeviceIndex

    n_docs, lo, hi, dim, nbits, B, Q, top_k, n_full, n_probe, noisy = CONFIGS[name]
    docs = make_docs(n_docs, lo, hi, dim=dim, seed=1234)
    oidx, _ = build_oracle_index(docs, nbits=nbits)
    didx = DeviceIndex(to_index_tensors(oidx), device)
    queries = make_queries(B, Q, dim=dim, seed=4321, docs=docs if noisy else None)
    params = DeviceIndex.make_params(top_k, n_full, n_probe)
    q16 = queries.to(torch.float16)
    # `stages`: approximate stage with every candidate scored exactly (FPB_FLAG_APPROX_EXACT_ALL), so that
    # off_approx can be compared entry by entry; the default (pruned two-pass) and the one-pass (DIRECT) runs
    # are compared with it in test_two_pass_approx_equals_scoring_every_candidate
    from fast_plaid_b200.engine import FPB_FLAG_APPROX_EXACT_ALL

    stages = _snapshot(didx.run_stages(q16.to(device), DeviceIndex.with_flags(params, FPB_FLAG_APPROX_EXACT_ALL)))
    torch.cuda.synchronize()
    _cache[name] = (oidx, didx, queries, params, stages)
    return _cache[name]


def _snapshot(st: dict) -> dict:
    """run_stages returns views of the (shared, reused) workspace: keep copies."""
    return {k: (v.clone() if isinstance(v, torch.Tensor) and k != "workspace" else v) for k, v in st.items()
            if k != "workspace"}


@pytest.mark.parametrize("name", list(CONFIGS))
def test_centroid_scores(name, cuda_device):
    oidx, didx, queries, params, st = _setup(name, cuda_device)
    Q = queries.shape[1]
    S_gpu = st["S"][:, :, :Q].cpu()
    bad = 0
    total = 0
    for b in range(queries.shape[0]):
        S_ref = oidx.centroids.matmul(queries[b].half().t())  # search.rs:491
        d = fp16_ulp_diff(S_gpu[b], S_ref)
        assert int(d.max()) <= 1, f"query {b}: S differs by {int(d.max())} fp16 ulps"
        bad += int((d > 0).sum())
        total += d.numel()
    assert bad / total < 2e-3, f"{bad}/{total} S entries differ by one ulp"
    # padded query columns are exactly zero
    if st["S"].shape[2] > Q:
        assert float(st["S"][:, :, Q:].abs().max()) == 0.0


@pytest.mark.parametrize("name", list(CONFIGS))
def test_integer_stages_bit_exact_given_S(name, cuda_device):
    """probe cells, candidates, approx scores and the pruned list must equal the canonical
    oracle exactly when it is fed the GPU's own S."""
    oidx, didx, queries, params, st = _setup(name, cuda_device)
    B, Q = queries.shape[0], queries.shape[1]
    n_inexact = 0
    for b in range(B):
        S_b = st["S"][b, :, :Q].cpu().contiguous()
        ref = po.search_one(queries[b], oidx, params.n_ivf_probe, 2000, params.n_full_scores, params.top_k,
                            ties="canonical", return_stages=True, inject={"S": S_b})
        cells_gpu = torch.unique(st["cells"][b].cpu().flatten().long())
        cells_gpu = cells_gpu[cells_gpu >= 0]
        assert torch.equal(cells_gpu, ref["cells"]), f"query {b}: probed cells differ"
        n = int(st["n_cand"][b])
        cand_gpu = st["cand"][b, :n].cpu().long()
        assert torch.equal(cand_gpu, ref["candidates"]), f"query {b}: candidate ids differ"
        approx_gpu = st["approx"][b, :n].cpu()
        if not torch.equal(approx_gpu, ref["approx"]):
            # fp32 sums of fp16 values: exact unless a partial sum needs > 24 bits (the summation order of
            # ATen's vectorised sum is not the kernel's).  The pruned list is then checked against the oracle
            # fed the GPU's own approximate scores.
            rel = ((approx_gpu - ref["approx"]).abs() / ref["approx"].abs().clamp_min(1.0)).max()
            assert float(rel) < 1e-6, f"query {b}: approx scores differ by {float(rel)}"
            n_inexact += 1
            ref = po.search_one(queries[b], oidx, params.n_ivf_probe, 2000, params.n_full_scores, params.top_k,
                                ties="canonical", return_stages=True, inject={"S": S_b, "approx": approx_gpu})
        r = int(st["n_rerank"][b])
        rer_gpu = st["rerank"][b, :r].cpu().long()
        assert r == ref["rerank"].shape[0]
        # canonical order of the pruned list is (approx desc, id asc) when pruning happened,
        # id order otherwise -- compare as the oracle produced it
        assert torch.equal(rer_gpu, ref["rerank"]), f"query {b}: pruned list differs"
    assert n_inexact <= B // 2


@pytest.mark.parametrize("name", list(CONFIGS))
def test_two_pass_approx_equals_scoring_every_candidate(name, cuda_device):
    """The default approximate stage (bound pass over the rows of high centroids + exact pass over the
    unresolved candidates that can reach the pruning threshold) must give the same pruned list, the same
    approximate scores on it, and the same final result as scoring every candidate (EXACT_ALL and the
    one-pass DIRECT alternative); what it leaves in off_approx for the other candidates is an upper bound
    strictly below the threshold."""
    from fast_plaid_b200.engine import FPB_FLAG_APPROX_DIRECT, FPB_FLAG_APPROX_TWO_PASS, DeviceIndex

    oidx, didx, queries, params, st = _setup(name, cuda_device)
    q16 = queries.half().to(cuda_device)
    direct = _snapshot(didx.run_stages(q16, DeviceIndex.with_flags(params, FPB_FLAG_APPROX_DIRECT)))
    # (without a flag the library would score an index this small in one pass)
    pruned = _snapshot(didx.run_stages(q16, DeviceIndex.with_flags(params, FPB_FLAG_APPROX_TWO_PASS)))
    torch.cuda.synchronize()
    B = queries.shape[0]
    R = st["layout"].R
    for b in range(B):
        n = int(st["n_cand"][b])
        exact_all = st["approx"][b, :n]
        assert torch.equal(direct["approx"][b, :n], exact_all), f"query {b}: one-pass and two-pass(all) scores differ"
        ub = pruned["approx"][b, :n]
        lb = pruned["approx_lb"][b, :n]
        T = float(pruned["thresh"][b])
        assert bool((ub >= exact_all).all()), f"query {b}: an entry of off_approx is below the exact score"
        refined = torch.zeros(n, dtype=torch.bool, device=ub.device)
        refined[pruned["refine"][b, : int(pruned["n_refine"][b])].long()] = True
        resolved = lb == ub  # set by the bound pass; refined entries were overwritten with the exact score
        known = refined | resolved
        assert torch.equal(ub[known], exact_all[known]), f"query {b}: a resolved/refined score is not the exact one"
        assert bool((ub[~known] < T).all()), f"query {b}: an unrefined upper bound reaches the threshold {T}"
        if n > R:  # at least R candidates are at or above the threshold
            assert int((exact_all >= T).sum()) >= R
        for other in (direct, pruned):
            r = int(st["n_rerank"][b])
            assert int(other["n_rerank"][b]) == r
            assert torch.equal(other["rerank"][b, :r], st["rerank"][b, :r]), f"query {b}: pruned lists differ"
            assert torch.equal(other["rerank_approx"][b, :r], st["rerank_approx"][b, :r])
            assert torch.equal(other["exact"][b, :r], st["exact"][b, :r])
        assert torch.equal(pruned["ids"][b], st["ids"][b]) and torch.equal(pruned["scores"][b], st["scores"][b])
        assert torch.equal(direct["ids"][b], st["ids"][b]) and torch.equal(direct["scores"][b], st["scores"][b])


@pytest.mark.parametrize("name", list(CONFIGS))
def test_exact_scores(name, cuda_device):
    oidx, didx, queries, params, st = _setup(name, cuda_device)
    B, Q = queries.shape[0], queries.shape[1]
    flips = 0
    total = 0
    for b in range(B):
        r = int(st["n_rerank"][b])
        rer = st["rerank"][b, :r].cpu().long()
        if r == 0:
            continue
        # oracle exact scores of exactly the documents the GPU re-ranked
        ref = oracle_exact_scores(oidx, queries[b], rer.tolist())
        got = st["exact"][b, :r].cpu()
        rel = (got - ref).abs() / ref.abs().clamp_min(1.0)
        assert float(rel.max()) < 1e-3, f"query {b}: exact score off by {float(rel.max())} relative"
        flips += int((got != ref).sum())
        total += r
    # fp16-faithful arithmetic: the vast majority of scores are bit-identical
    assert flips / max(total, 1) < 0.05, f"{flips}/{total} exact scores not bit-identical"


@pytest.mark.parametrize("name", list(CONFIGS))
def test_end_to_end_against_reference_ties(name, cuda_device):
    """Whole pipeline through fpb_search_batch vs the op-for-op oracle (torch tie order)."""
    oidx, didx, queries, params, st = _setup(name, cuda_device)
    ids, scores, counts = didx.search(queries.half().to(cuda_device), params)
    torch.cuda.synchronize()
    ids, scores, counts = ids.cpu(), scores.cpu(), counts.cpu()
    # the staged run and the one-call run agree bit for bit
    assert torch.equal(ids, st["ids"].cpu()) and torch.equal(counts, st["counts"].cpu())
    strict = 0
    outside = 0
    for b in range(queries.shape[0]):
        ref = po.search_one(queries[b], oidx, params.n_ivf_probe, 2000, params.n_full_scores, 10**9,
                            ties="torch", return_stages=True)
        n = int(counts[b])
        assert n == min(params.top_k, len(ref["ids"]))
        score_of = dict(zip(ref["ids"], ref["scores"]))
        n_ref = len(score_of)
        ok, why = ranking_consistent(ids[b, :n].tolist(), scores[b, :n].tolist(), score_of, 1e-3,
                                     fallback=lambda d, b=b: float(oracle_exact_scores(oidx, queries[b], [d])[0]))
        assert ok, f"query {b}: {why}"
        outside += len(score_of) - n_ref
        strict += int(ids[b, :n].tolist() == ref["ids"][:n])
        assert (ids[b, n:] == -1).all()
    # informational: how often the id lists are identical outright
    print(f"[{name}] strict id-list equality on {strict}/{queries.shape[0]} queries; "
          f"{outside} returned docs outside the reference's re-ranked set (topk-boundary ties)")
    assert outside <= max(1, queries.shape[0] // 4)


def test_host_path_matches_device_path(cuda_device):
    oidx, didx, queries, params, st = _setup("base", cuda_device)
    h_ids, h_scores, h_counts = didx.search_host(queries, params)  # fp32 host queries
    assert torch.equal(h_ids, st["ids"].cpu())
    assert torch.equal(h_counts, st["counts"].cpu())
    assert torch.equal(h_scores, st["scores"].cpu())


def test_same_query_twice_is_deterministic(cuda_device):
    oidx, didx, queries, params, st = _setup("base", cuda_device)
    a = didx.search(queries.half().to(cuda_device), params)
    b = didx.search(queries.half().to(cuda_device), params)
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_top_k_larger_than_index(cuda_device):
    """tests/test.py:880-886 of the reference: fewer than top_k results, never more than N."""
    from fast_plaid_b200.engine import DeviceIndex

    oidx, didx, queries, _, _ = _setup("probe1", cuda_device)
    params = DeviceIndex.make_params(2000, 4096, 8)
    ids, scores, counts = didx.search(queries.half().to(cuda_device), params)
    torch.cuda.synchronize()
    assert int(counts.max()) <= oidx.doc_lengths.shape[0]
    for b in range(queries.shape[0]):
        n = int(counts[b])
        s = scores[b, :n].cpu()
        assert bool((s[:-1] >= s[1:]).all())  # tests/test.py:939-954 sorted descending
        assert len(set(ids[b, :n].tolist())) == n


def test_reconstruct_matches_oracle(cuda_device):
    oidx, didx, queries, params, st = _setup("base", cuda_device)
    docs = [0, 5, 17, 999]
    got = didx.reconstruct(docs)
    torch.cuda.synchronize()
    bad = 0
    tot = 0
    for d, g in zip(docs, got):
        sel = torch.tensor([d])
        codes, _ = po.ragged_lookup(oidx.doc_codes, oidx.doc_offsets, oidx.doc_lengths, sel)
        res, _ = po.ragged_lookup(oidx.doc_residuals, oidx.doc_offsets, oidx.doc_lengths, sel)
        ref = po.decompress_residuals(res, oidx.bucket_weights, oidx.byte_reversed_bits_map,
                                      oidx.bucket_weight_indices_lookup, codes, oidx.centroids, oidx.dim, oidx.nbits)
        dlt = fp16_ulp_diff(g.cpu(), ref)
        assert int(dlt.max()) <= 1
        bad += int((dlt > 0).sum())
        tot += dlt.numel()
    assert bad / tot < 5e-3


@pytest.mark.parametrize("name", ["base", "ragged_short", "q64", "nbits2", "dim64"])
def test_token_score_matrices_match_the_oracle(name, cuda_device):
    """fpb_token_scores (search.rs:668-686) against the oracle's token matrices for the documents the engine
    returns: every entry within one fp16 ulp, almost all identical (the two sides accumulate the 128 products
    of a dot product in different orders), and max-over-tokens / sum-over-query-tokens of the GPU matrix equals
    the score the search returned (tests/test.py:175-197 asserts 0.1; here 1e-3)."""
    oidx, didx, queries, params, st = _setup(name, cuda_device)
    B, Q = queries.shape[0], queries.shape[1]
    q16 = queries.half().to(cuda_device)
    pairs = [(b, int(d)) for b in range(B) for d in st["ids"][b, : int(st["counts"][b])].tolist()]
    mats = didx.token_scores(q16, torch.tensor([p[0] for p in pairs], dtype=torch.int32),
                             torch.tensor([p[1] for p in pairs], dtype=torch.int32)).cpu()
    torch.cuda.synchronize()
    bad = tot = far = 0
    for k, (b, d) in enumerate(pairs):
        ref = oracle_token_matrix(oidx, queries[b], d)  # [Q, len]
        n = ref.shape[1]
        got = mats[k, :n, :].transpose(0, 1)
        dlt = fp16_ulp_diff(got, ref)
        # One fp16 ulp -- except for dot products that cancel to almost zero, where an ulp shrinks to 6e-8 while the
        # noise stays absolute: summing 128 fp32 products in a different order (~1e-5), and, for a token whose fp16
        # norm lands one ulp away, the re-rounding of each of its 128 normalised elements (up to 128 * 2^-11 * |term|,
        # a few 1e-4 at worst).  Such entries must stay within 1e-3 absolute and be rare; they never decide a MaxSim
        # (the maximum over tokens is nowhere near zero).
        off = dlt > 1
        assert float((got.float() - ref.float()).abs()[off].max() if bool(off.any()) else 0.0) <= 1e-3, \
            f"pair {k}: token scores differ by {int(dlt.max())} fp16 ulps"
        far += int(off.sum())
        bad += int((dlt > 0).sum())
        tot += dlt.numel()
        assert float(mats[k, n:, :].abs().max() if mats.shape[1] > n else 0.0) == 0.0  # rows past the document stay zero
        rank = st["ids"][b, : int(st["counts"][b])].tolist().index(d)
        manual = float(got.float().max(dim=1).values.sum())
        assert abs(manual - float(st["scores"][b, rank])) <= 1e-3 * max(1.0, abs(manual))
    assert bad / max(tot, 1) < 5e-3, f"{bad}/{tot} token scores differ by one ulp"
    assert far / max(tot, 1) < 1e-3, f"{far}/{tot} token scores differ by more than one ulp"


def test_compress_only_index_refuses_search(cuda_device):
    """tests/test.py:748-761 of the reference."""
    from fast_plaid_b200.engine import DeviceIndex, IndexTensors

    oidx, _, queries, params, _ = _setup("probe1", cuda_device)
    t = to_index_tensors(oidx)
    t = IndexTensors(t.nbits, t.centroids, t.bucket_weights, t.doc_lengths, t.doc_codes, t.doc_residuals, None, None)
    d = DeviceIndex(t, cuda_device)
    with pytest.raises(ValueError, match="compress_only"):
        d.search(queries.half().to(cuda_device), params)


@pytest.mark.parametrize("name", ["base", "dim64", "ragged_short"])
def test_subset_search_matches_oracle(name, cuda_device):
    """`subset=` (search.rs:494-517, :544-547): restricted probing + candidate intersection."""
    oidx, didx, queries, params, st = _setup(name, cuda_device)
    B, Q = queries.shape[0], queries.shape[1]
    n_docs = int(oidx.doc_lengths.shape[0])
    g = torch.Generator().manual_seed(5)
    subsets = []
    for b in range(B):
        kind = b % 5
        if kind == 0:
            sub = torch.randperm(n_docs, generator=g)[: max(1, n_docs // 10)].tolist()
        elif kind == 1:
            sub = [int(torch.randint(0, n_docs, (1,), generator=g))]
        elif kind == 2:
            sub = []
        elif kind == 3:
            sub = list(range(n_docs))
        else:
            sub = torch.randint(0, n_docs, (50,), generator=g).tolist() * 2  # duplicates
        subsets.append(sub)
    stg = didx.run_stages(queries.half().to(cuda_device), params, subset=subsets)
    torch.cuda.synchronize()
    for b in range(B):
        S_b = stg["S"][b, :, :Q].cpu().contiguous()
        ref = po.search_one(queries[b], oidx, params.n_ivf_probe, 2000, params.n_full_scores, params.top_k,
                            subset=torch.tensor(subsets[b], dtype=torch.int64), ties="canonical", return_stages=True,
                            inject={"S": S_b})
        cells = torch.unique(stg["cells"][b].cpu().flatten().long())
        assert torch.equal(cells[cells >= 0], ref["cells"]), f"query {b}: probed cells differ"
        n = int(stg["n_cand"][b])
        assert torch.equal(stg["cand"][b, :n].cpu().long(), ref["candidates"]), f"query {b}: candidates differ"
        cnt = int(stg["counts"][b])
        got = stg["ids"][b, :cnt].cpu().tolist()
        assert set(got) <= set(subsets[b])  # tests/test.py:409-411
        assert cnt == min(params.top_k, len(ref["ids"]))
        if cnt:
            sc = dict(zip(ref["ids"], ref["scores"]))
            ok, why = ranking_consistent(got, stg["scores"][b, :cnt].cpu().tolist(), sc, 1e-3,
                                         fallback=lambda d, b=b: float(oracle_exact_scores(oidx, queries[b], [d])[0]))
            assert ok, why
    # the one-call entry point agrees with the staged run
    ids, scores, counts = didx.search(queries.half().to(cuda_device), params, subset=subsets)
    torch.cuda.synchronize()
    assert torch.equal(ids, stg["ids"]) and torch.equal(counts, stg["counts"])


# ---- edge cases the reference's tests exercise (tests/test.py) plus size extremes ----------------
def _search_vs_oracle(oidx, didx, queries, params, device, tol=1e-3):
    ids, scores, counts = didx.search(queries.half().to(device), params)
    torch.cuda.synchronize()
    ids, scores, counts = ids.cpu(), scores.cpu(), counts.cpu()
    for b in range(queries.shape[0]):
        ref = po.search_one(queries[b], oidx, params.n_ivf_probe, 2000, params.n_full_scores, 10**9, ties="torch",
                            return_stages=True)
        n = int(counts[b])
        assert n == min(params.top_k, len(ref["ids"])), (n, len(ref["ids"]))
        ok, why = ranking_consistent(ids[b, :n].tolist(), scores[b, :n].tolist(), dict(zip(ref["ids"], ref["scores"])), tol,
                                     fallback=lambda d, b=b: float(oracle_exact_scores(oidx, queries[b], [d])[0]))
        assert ok, f"query {b}: {why}"
    return ids, scores, counts


def test_unnormalised_randn_inputs_like_the_reference_tests(cuda_device):
    """tests/test.py feeds raw torch.randn documents and queries (norm ~ 11), dim 128 and 64."""
    from fast_plaid_b200.engine import DeviceIndex

    for dim in (128, 64):
        docs = make_docs(150, 20, 60, dim=dim, seed=3, normalize=False)
        oidx, _ = build_oracle_index(docs, kmeans_niters=2)
        g = torch.Generator().manual_seed(4)
        queries = torch.randn(3, 30, dim, generator=g)
        didx = DeviceIndex(to_index_tensors(oidx), cuda_device)
        for n_probe in (2, 16):  # tests/test.py:897-906
            _search_vs_oracle(oidx, didx, queries, DeviceIndex.make_params(10, 4096, n_probe), cuda_device, tol=2e-3)


def test_tiny_index_and_single_token_query(cuda_device):
    """K < 128 (one partial centroid tile), B = 1, Q = 1 (padded to 16 internally)."""
    from fast_plaid_b200.engine import DeviceIndex

    docs = make_docs(12, 3, 6, seed=8)
    oidx, _ = build_oracle_index(docs, kmeans_niters=2)
    assert oidx.centroids.shape[0] < 128
    didx = DeviceIndex(to_index_tensors(oidx), cuda_device)
    q = make_queries(1, 1, seed=9, docs=docs)
    ids, scores, counts = _search_vs_oracle(oidx, didx, q, DeviceIndex.make_params(5, 4096, 8), cuda_device)
    assert 0 < int(counts[0]) <= 5


def test_large_rerank_budget_and_top_k(cuda_device):
    """n_full_scores = 16384 -> 4096 re-ranked documents (the supported maximum), top_k = 3000."""
    from fast_plaid_b200.engine import DeviceIndex

    oidx, didx, queries, _, _ = _setup("base", cuda_device)
    params = DeviceIndex.make_params(3000, 16384, 8)
    ids, scores, counts = _search_vs_oracle(oidx, didx, queries[:2], params, cuda_device)
    assert int(counts.max()) <= 1000  # the index holds 1000 documents
    with pytest.raises(ValueError):
        didx.search(queries[:1].half().to(cuda_device), DeviceIndex.make_params(10, 4 * 4097, 8))


def test_empty_document_gets_the_reference_score(cuda_device):
    """A zero-token document scores Q * fp16(-9999) = Q * -10000 (search.rs:395) and never wins."""
    from fast_plaid_b200.engine import DeviceIndex, IndexTensors

    docs = make_docs(60, 5, 20, seed=12)
    oidx, _ = build_oracle_index(docs, kmeans_niters=2)
    lens = oidx.doc_lengths.clone()
    lens[8] += lens[7]
    lens[7] = 0  # document 7 becomes empty; its tokens now belong to document 8
    o2 = po.OracleIndex(oidx.nbits, oidx.centroids, oidx.bucket_weights, oidx.ivf, oidx.ivf_lengths, oidx.doc_codes,
                        oidx.doc_residuals, lens)
    t = to_index_tensors(o2)
    didx = DeviceIndex(t, cuda_device)
    q = make_queries(2, 8, seed=13, docs=docs)
    params = DeviceIndex.make_params(60, 4096, 8)
    ids, scores, counts = didx.search(q.half().to(cuda_device), params)
    torch.cuda.synchronize()
    for b in range(2):
        got = dict(zip(ids[b, : int(counts[b])].tolist(), scores[b, : int(counts[b])].tolist()))
        if 7 in got:  # it is a candidate only through the IVF entries of its former tokens
            assert got[7] == 8 * -10000.0
            assert ids[b, int(counts[b]) - 1] == 7
    emb = didx.reconstruct([7, 8])
    assert emb[0].shape[0] == 0 and emb[1].shape[0] == int(lens[8])


def test_select_fallback_path_with_all_equal_scores(cuda_device):
    """An all-zero query gives S == 0 everywhere, so every candidate has the same approximate score: the value
    range is empty, the bucket fast path of k3b_select declines and the radix passes must pick, by the canonical
    rule, the n_full_scores/4 smallest candidate ids.  The exact scores are all 0 too: ids come back ascending."""
    from fast_plaid_b200.engine import DeviceIndex

    oidx, didx, _, _, _ = _setup("base", cuda_device)
    q = torch.zeros(2, 32, 128, dtype=torch.float16, device=cuda_device)
    from fast_plaid_b200.engine import FPB_FLAG_APPROX_TWO_PASS

    # R = 16 documents re-ranked, far fewer than the candidates; two-pass stage: tau = 0 = every score, all resolved
    params = DeviceIndex.with_flags(DeviceIndex.make_params(16, 64, 8), FPB_FLAG_APPROX_TWO_PASS)
    st = didx.run_stages(q, params)
    torch.cuda.synchronize()
    for b in range(2):
        n = int(st["n_cand"][b])
        assert n > 16
        assert bool((st["approx"][b, :n] == 0).all())
        cand = st["cand"][b, :n].cpu()
        assert torch.equal(st["rerank"][b, :16].cpu(), cand[:16])  # candidates are in ascending id order
        ids = st["ids"][b, : int(st["counts"][b])].cpu()
        assert torch.equal(ids, torch.sort(ids).values) and int(st["counts"][b]) == 16
        assert bool((st["scores"][b, :16] == 0).all())
