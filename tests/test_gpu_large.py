"""Larger-scale GPU checks on a synthetic 200k-document index (BASELINE-shaped: 128-dim, nbits=4,
batch of 64 x 32-token queries, top_k=100): size-independent properties for the whole batch, an
oracle cross-check on a sample of queries, and sharded == unsharded at this size."""

from __future__ import annotations

import pytest
import torch

from util import oracle_exact_scores, ranking_consistent

from oracle import plaid_oracle as po

pytestmark = pytest.mark.gpu

N_DOCS, DOC_LEN, B, Q, TOP_K = 200_000, 128, 64, 32, 100


@pytest.fixture(scope="module")
def big(cuda_device):
    from fast_plaid_b200.engine import DeviceIndex
    from fast_plaid_b200.index.synthetic import synthetic_index

    data, _ = synthetic_index(N_DOCS, DOC_LEN, device=cuda_device, seed=77, ragged=True)
    didx = DeviceIndex(data, cuda_device)
    g = torch.Generator().manual_seed(78)
    docs = torch.randint(0, N_DOCS, (B,), generator=g).tolist()
    embs = didx.reconstruct(docs)
    qs = []
    for e in embs:
        e = e.float().cpu()
        rows = torch.randint(0, e.shape[0], (Q,), generator=g)
        qs.append(torch.nn.functional.normalize(e[rows] + 0.1 * torch.randn(Q, 128, generator=g), dim=-1))
    queries = torch.stack(qs)
    params = DeviceIndex.make_params(TOP_K, 4096, 8)
    return data, didx, queries, params, docs


def test_batch_properties(big, cuda_device):
    data, didx, queries, params, src_docs = big
    q16 = queries.half().to(cuda_device)
    ids, scores, counts = didx.search(q16, params)
    ids2, scores2, counts2 = didx.search(q16, params)
    torch.cuda.synchronize()
    assert torch.equal(ids, ids2) and torch.equal(scores, scores2)  # idempotent / deterministic
    ids, scores, counts = ids.cpu(), scores.cpu(), counts.cpu()
    assert bool((counts == TOP_K).all())
    assert bool((scores[:, :-1] >= scores[:, 1:]).all())  # sorted descending
    for b in range(B):
        row = ids[b].tolist()
        assert len(set(row)) == TOP_K and min(row) >= 0 and max(row) < N_DOCS
        # a query made of noisy copies of a document's tokens finds that document first
        assert row[0] == src_docs[b]
    # each query alone returns what it returned inside the batch (no cross-query leakage)
    for b in (0, 17, 63):
        i1, s1, c1 = didx.search(q16[b : b + 1], params)
        torch.cuda.synchronize()
        assert torch.equal(i1[0].cpu(), ids[b]) and torch.equal(s1[0].cpu(), scores[b])
    # host path == device path
    h = didx.search_host(queries, params)
    assert torch.equal(h[0], ids) and torch.equal(h[1], scores)


def test_sample_against_oracle(big, cuda_device):
    data, didx, queries, params, _ = big
    lens = (didx.doc_offsets[1:] - didx.doc_offsets[:-1]).cpu()
    ivf_len = (didx.ivf_offsets[1:] - didx.ivf_offsets[:-1]).cpu()
    oidx = po.OracleIndex(nbits=4, centroids=didx.centroids.cpu(), bucket_weights=didx.bucket_weights.cpu(),
                          ivf=didx.ivf_pids.cpu().long(), ivf_lengths=ivf_len, doc_codes=didx.doc_codes.cpu().long(),
                          doc_residuals=didx.doc_residuals.cpu(), doc_lengths=lens)
    from fast_plaid_b200.engine import FPB_FLAG_APPROX_EXACT_ALL, FPB_FLAG_APPROX_TWO_PASS, DeviceIndex

    # pruned two-pass approximate stage first (views of the shared workspace: copy what is compared)
    dflt = didx.run_stages(queries[:3].half().to(cuda_device), DeviceIndex.with_flags(params, FPB_FLAG_APPROX_TWO_PASS))
    torch.cuda.synchronize()
    d_rerank, d_ids, d_scores = dflt["rerank"].clone(), dflt["ids"].clone(), dflt["scores"].clone()
    d_ub, d_nref = dflt["approx"].clone(), dflt["n_refine"].clone()
    st = didx.run_stages(queries[:3].half().to(cuda_device), DeviceIndex.with_flags(params, FPB_FLAG_APPROX_EXACT_ALL))
    torch.cuda.synchronize()
    for b in range(3):
        n = int(st["n_cand"][b])
        # pruned two-pass == every candidate scored exactly: same pruned list and result, upper bounds elsewhere
        assert torch.equal(d_rerank[b], st["rerank"][b]) and torch.equal(d_ids[b], st["ids"][b])
        assert torch.equal(d_scores[b], st["scores"][b])
        assert bool((d_ub[b, :n] >= st["approx"][b, :n]).all())
        assert int(d_nref[b]) < n // 2, f"query {b}: the exact pass re-scored {int(d_nref[b])} of {n} candidates"
    for b in range(3):
        # integer stages bit-exact given the GPU's S (canonical ties), at 50k+ candidates per query
        S_b = st["S"][b, :, :Q].cpu().contiguous()
        ref = po.search_one(queries[b], oidx, 8, 2000, 4096, TOP_K, ties="canonical", return_stages=True, inject={"S": S_b})
        n = int(st["n_cand"][b])
        assert n > 10_000
        assert torch.equal(st["cand"][b, :n].cpu().long(), ref["candidates"])
        assert torch.equal(st["approx"][b, :n].cpu(), ref["approx"])
        r = int(st["n_rerank"][b])
        assert torch.equal(st["rerank"][b, :r].cpu().long(), ref["rerank"])
        cnt = int(st["counts"][b])
        ok, why = ranking_consistent(st["ids"][b, :cnt].cpu().tolist(), st["scores"][b, :cnt].cpu().tolist(),
                                     dict(zip(ref["rerank"].tolist(), ref["exact"].tolist())), 1e-3,
                                     fallback=lambda d, b=b: float(oracle_exact_scores(oidx, queries[b], [d])[0]))
        assert ok, why


def test_sharded_equals_unsharded_at_size(big, cuda_device):
    from fast_plaid_b200.engine import DeviceIndex, shard_tensors

    data, didx, queries, params, _ = big
    q16 = queries[:16].half().to(cuda_device)
    ids, scores, counts = didx.search(q16, params)
    world = 4
    shards = []
    for r in range(world):
        sh, base = shard_tensors(data, r, world)
        shards.append(DeviceIndex(sh, cuda_device, doc_id_base=base))
    all_keys = torch.stack([d.shard_approx_keys(q16, params) for d in shards])
    recs = torch.stack([d.shard_exact_records(all_keys, r, Q, params) for r, d in enumerate(shards)])
    i2, s2, c2 = didx.merge_records(recs, TOP_K)
    torch.cuda.synchronize()
    assert torch.equal(i2, ids) and torch.equal(s2, scores) and torch.equal(c2, counts)


def test_cfg2_built_by_create_searches_like_the_oracle(tmp_path, cuda_device):
    """BASELINE config 2 end to end through the public surface: 100k documents x 300 tokens built by
    FastPlaid.create() on the GPU (k-means on the sm_90a assign/update kernels, streaming chunk encode, K = 65536),
    loaded by the direct-to-device loader, searched with B = 64, Q = 32, top_k = 100.  For 8 queries every integer
    stage must equal the canonical oracle given the GPU's own S -- probed cells, candidates, approximate scores
    (or the pruned list from the GPU's approximate scores when a fp32 sum rounds differently), pruned list -- and
    the returned ranking must be a 1e-3-valid ranking of the oracle's exact scores."""
    import time

    from fast_plaid_b200 import search
    from fast_plaid_b200.engine import FPB_FLAG_APPROX_EXACT_ALL, DeviceIndex
    from fast_plaid_b200.index import store
    from fast_plaid_b200.index.synthetic import SyntheticDocuments

    n_docs, doc_len, B, Q, top_k = 100_000, 300, 64, 32, 100
    docs = SyntheticDocuments(n_docs, doc_len, device=cuda_device, seed=11, clusters=8192)
    path = str(tmp_path / "cfg2")
    fp = search.FastPlaid(path, device=cuda_device)
    t0 = time.time()
    fp.create(docs, kmeans_niters=4, seed=42)
    t_create = time.time() - t0
    meta = store.read_metadata(path)
    assert meta["num_documents"] == n_docs and meta["num_embeddings"] == n_docs * doc_len
    assert meta["num_partitions"] == 65536
    # queries: noisy copies of document tokens
    g = torch.Generator().manual_seed(5)
    src = torch.randint(0, n_docs, (B,), generator=g).tolist()
    queries = torch.stack([torch.nn.functional.normalize(
        docs[d].float().cpu()[torch.randint(0, doc_len, (Q,), generator=g)] + 0.05 * torch.randn(Q, 128, generator=g), dim=-1)
        for d in sorted(src)])
    t0 = time.time()
    res = fp.search(queries, top_k=top_k)
    t_search = time.time() - t0
    assert len(res) == B and all(len(r) == top_k for r in res)
    print(f"[cfg2] create() {t_create:.1f} s, first search of 64 queries {t_search * 1e3:.1f} ms")
    # the source document is found (tests/test.py relevance idea: queries are copies of its tokens)
    hits = sum(int(d == r[0][0]) for d, r in zip(sorted(src), res))
    assert hits >= B // 2, hits
    # oracle on the directory the builder wrote
    data = store.read_index(path)
    oidx = po.OracleIndex(data.nbits, data.centroids, data.bucket_weights, data.ivf, data.ivf_lengths.long(),
                          data.doc_codes, data.doc_residuals, data.doc_lengths)
    didx = fp.indices[cuda_device]
    params = DeviceIndex.make_params(top_k, 4096, 8)
    nq = 8
    st = didx.run_stages(queries[:nq].half().to(cuda_device), DeviceIndex.with_flags(params, FPB_FLAG_APPROX_EXACT_ALL))
    torch.cuda.synchronize()
    for b in range(nq):
        S_b = st["S"][b, :, :Q].cpu().contiguous()
        ref = po.search_one(queries[b], oidx, 8, 2000, 4096, top_k, ties="canonical", return_stages=True, inject={"S": S_b})
        cells = torch.unique(st["cells"][b].cpu().flatten().long())
        assert torch.equal(cells[cells >= 0], ref["cells"]), f"query {b}: probed cells differ"
        n = int(st["n_cand"][b])
        assert n > 30_000
        assert torch.equal(st["cand"][b, :n].cpu().long(), ref["candidates"]), f"query {b}: candidates differ"
        approx = st["approx"][b, :n].cpu()
        if not torch.equal(approx, ref["approx"]):
            assert float(((approx - ref["approx"]).abs() / ref["approx"].abs().clamp_min(1.0)).max()) < 1e-6
            ref = po.search_one(queries[b], oidx, 8, 2000, 4096, top_k, ties="canonical", return_stages=True,
                                inject={"S": S_b, "approx": approx})
        r = int(st["n_rerank"][b])
        assert torch.equal(st["rerank"][b, :r].cpu().long(), ref["rerank"]), f"query {b}: pruned list differs"
        ok, why = ranking_consistent([d for d, _ in res[b]], [s for _, s in res[b]],
                                     dict(zip(ref["rerank"].tolist(), ref["exact"].tolist())), 1e-3)
        assert ok, f"query {b}: {why}"
    fp.close()
