"""GPU tests through the public surface: FastPlaid create/search/update/delete on a CUDA
device, the committed golden fixtures, and the sharded path (two shards on one GPU)."""

from __future__ import annotations

import glob
import os

import pytest
import torch

from util import (build_oracle_index, make_docs, make_queries, oracle_exact_scores, ranking_consistent,
                  to_index_tensors)

from oracle import plaid_oracle as po

pytestmark = pytest.mark.gpu

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "small_*.pt")))


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_engine_reproduces_golden_fixtures(path, cuda_device):
    """Committed vectors (minted by the oracle, tests/golden/make_golden.py): integer stages
    exactly, scores to 1e-3 relative, ranking consistent."""
    from fast_plaid_b200.engine import DeviceIndex, IndexTensors

    blob = torch.load(path, weights_only=False)
    ix, m = blob["index"], blob["meta"]
    didx = DeviceIndex(IndexTensors(ix["nbits"], ix["centroids"], ix["bucket_weights"], ix["doc_lengths"],
                                    ix["doc_codes"], ix["doc_residuals"], ix["ivf"], ix["ivf_lengths"]), cuda_device)
    params = DeviceIndex.make_params(m["top_k"], m["n_full"], m["n_probe"])
    st = didx.run_stages(blob["queries"].to(cuda_device), params)
    torch.cuda.synchronize()
    n_strict = 0
    for b, exp in enumerate(blob["expected"]):
        cells = torch.unique(st["cells"][b].cpu().flatten().long())
        n = int(st["n_cand"][b])
        r = int(st["n_rerank"][b])
        n_ids = int(st["counts"][b])
        got_ids = st["ids"][b, :n_ids].cpu().tolist()
        got_sc = st["scores"][b, :n_ids].cpu().tolist()
        # S can differ from the CPU by one fp16 ulp on ~1e-4 of its entries, which may move a
        # boundary cell / candidate; anything that does not match exactly must still be a valid
        # ranking of the oracle's scores
        exact_match = (torch.equal(cells[cells >= 0], exp["cells"]) and
                       torch.equal(st["cand"][b, :n].cpu().long(), exp["candidates"]) and
                       torch.equal(st["rerank"][b, :r].cpu().long(), exp["rerank"]))
        n_strict += int(exact_match and got_ids == exp["ids"])
        if exact_match:
            assert torch.allclose(st["exact"][b, :r].cpu(), exp["exact"], rtol=1e-3, atol=1e-3)
        score_of = dict(zip(exp["ids"], exp["scores"]))
        oix = po.OracleIndex(ix["nbits"], ix["centroids"], ix["bucket_weights"], ix["ivf"].long(),
                             ix["ivf_lengths"].long(), ix["doc_codes"].long(), ix["doc_residuals"], ix["doc_lengths"].long())
        ok, why = ranking_consistent(got_ids, got_sc, score_of, 1e-3,
                                     fallback=lambda d, b=b: float(oracle_exact_scores(oix, blob["queries"][b].float(), [d])[0]))
        assert ok, why
    assert n_strict >= len(blob["expected"]) - 1, f"only {n_strict} queries matched the golden vectors exactly"


def test_fastplaid_surface_on_gpu(tmp_path, cuda_device):
    """create -> search -> update -> delete -> get_embeddings through the FastPlaid class, on
    the same structural checks as the reference's tests (tests/test.py:31-104, 202-389)."""
    from fast_plaid_b200 import search
    from fast_plaid_b200.index import store

    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device=cuda_device)
    docs = make_docs(300, 20, 80, seed=11)
    fp.create(docs, kmeans_niters=4)
    queries = make_queries(10, 30, seed=12, docs=docs)
    res = fp.search(queries, top_k=10)
    assert len(res) == 10 and all(len(r) == 10 for r in res)  # tests/test.py:44-49
    assert all(isinstance(d, int) and isinstance(s, float) for r in res for d, s in r)
    # the same directory, searched by the oracle
    data = store.read_index(path)
    oidx = po.OracleIndex(data.nbits, data.centroids, data.bucket_weights, data.ivf, data.ivf_lengths.long(),
                          data.doc_codes, data.doc_residuals, data.doc_lengths)
    for b in range(10):
        ref = po.search_one(queries[b], oidx, top_k=10**9, return_stages=True)
        ok, why = ranking_consistent([d for d, _ in res[b]], [s for _, s in res[b]], dict(zip(ref["ids"], ref["scores"])), 1e-3,
                                     fallback=lambda d, b=b: float(oracle_exact_scores(oidx, queries[b], [d])[0]))
        assert ok, why
    # list-of-tensors input is zero padded like the reference (fast_plaid.py:772-780)
    res_list = fp.search([queries[0][:20], queries[1]], top_k=5)
    assert len(res_list) == 2 and all(len(r) == 5 for r in res_list)
    # subset filtering through the public surface (tests/test.py:409-435): single list and per-query lists
    sub = list(range(0, 300, 3))
    r_sub = fp.search(queries[:4], top_k=5, subset=sub)
    assert all(d in set(sub) for r in r_sub for d, _ in r) and all(len(r) == 5 for r in r_sub)
    r_sub2 = fp.search(queries[:2], top_k=5, subset=[[1, 2, 3], [10]])
    assert [len(r) for r in r_sub2] == [3, 1] and r_sub2[1][0][0] == 10
    # top_k beyond the index size (tests/test.py:880-886)
    big = fp.search(queries[:2], top_k=1000)
    assert all(0 < len(r) <= 300 for r in big)
    # update then delete keep ids in range (tests/test.py:218-238, 363-368)
    fp.update(make_docs(50, 20, 80, seed=13))
    res = fp.search(queries, top_k=10)
    assert all(0 <= d < 350 for r in res for d, _ in r)
    fp.delete(list(range(0, 100)))
    res = fp.search(queries, top_k=10)
    assert all(0 <= d < 250 for r in res for d, _ in r)
    # get_embeddings returns unit-norm rows of the right length
    embs = fp.get_embeddings([0, 7])
    lens = store.read_index(path).doc_lengths
    assert [e.shape[0] for e in embs] == [int(lens[0]), int(lens[7])]
    assert torch.allclose(embs[0].float().norm(dim=-1), torch.ones(embs[0].shape[0]), atol=2e-3)
    # token-score matrices (tests/test.py:109-197)
    ts = fp.search_token_scores(queries[:2], top_k=3)
    plain = fp.search(queries[:2], top_k=3)
    for rq, rp in zip(ts, plain):
        assert [d for d, _, _ in rq] == [d for d, _ in rp]
        for d, s, m in rq:
            assert m.shape == (30, int(store.read_index(path).doc_lengths[d]))
            assert abs(float(m.float().max(dim=1).values.sum()) - s) < 0.1
    # non-3D tensor -> ValueError (search.rs:234-239)
    with pytest.raises(ValueError):
        fp.search(queries[0], top_k=5)
    fp.close()


def test_two_shards_on_one_gpu_equal_the_unsharded_search(cuda_device):
    """fpb_search_shard x2 + fpb_merge_shards == fpb_search_batch, bit for bit."""
    from fast_plaid_b200.engine import DeviceIndex, shard_tensors

    docs = make_docs(900, 10, 60, seed=21)
    oidx, _ = build_oracle_index(docs)
    t = to_index_tensors(oidx)
    whole = DeviceIndex(t, cuda_device)
    queries = make_queries(6, 32, seed=22, docs=docs).half().to(cuda_device)
    for n_full, top_k in ((64, 10), (4096, 50)):
        params = DeviceIndex.make_params(top_k, n_full, 8)
        ids, scores, counts = whole.search(queries, params)
        for world in (2, 3):
            recs = []
            for r in range(world):
                sh, base = shard_tensors(t, r, world)
                d = DeviceIndex(sh, cuda_device, doc_id_base=base)
                recs.append(d.search_records(queries, params))
            gathered = torch.stack(recs)
            i2, s2, c2 = whole.merge_records(gathered, top_k)
            torch.cuda.synchronize()
            assert torch.equal(c2, counts)
            assert torch.equal(i2, ids), f"world={world} n_full={n_full}"
            assert torch.equal(s2, scores)
            # two-step variant: keys -> global threshold -> exact scores of the survivors only
            shards = [DeviceIndex(*shard_tensors(t, r, world)[:1], cuda_device, doc_id_base=shard_tensors(t, r, world)[1])
                      for r in range(world)]
            all_keys = torch.stack([d.shard_approx_keys(queries, params) for d in shards])
            recs2 = [d.shard_exact_records(all_keys, r, int(queries.shape[1]), params) for r, d in enumerate(shards)]
            n_scored = sum(int((rec.view(torch.int64).view(rec.shape[0], rec.shape[1], 2)[:, :, 1] >= 0).sum()) for rec in recs2)
            i3, s3, c3 = whole.merge_records(torch.stack(recs2), top_k)
            torch.cuda.synchronize()
            assert torch.equal(i3, ids) and torch.equal(s3, scores) and torch.equal(c3, counts)
            assert n_scored <= queries.shape[0] * (n_full // 4)  # exact-scored docs: at most R per query in total


def test_one_rank_communicator_runs_the_sharded_c_path(cuda_device):
    """fpb_comm_create with one rank + fpb_search_batch_sharded(_host): the whole exchange path (keys ->
    ncclAllGather -> threshold -> MaxSim -> records -> ncclAllGather -> merge) on a single GPU, equal to
    fpb_search_batch; also through FastPlaid(shard=(0, 1)).  Ragged batch: 5 queries."""
    from fast_plaid_b200.engine import DeviceIndex, ShardComm
    from fast_plaid_b200.search.fast_plaid import FastPlaid

    docs = make_docs(500, 10, 60, seed=41)
    oidx, _ = build_oracle_index(docs)
    didx = DeviceIndex(to_index_tensors(oidx), cuda_device)
    queries = make_queries(5, 32, seed=42, docs=docs)
    q16 = queries.half().to(cuda_device)
    comm = ShardComm(1, 0, ShardComm.new_unique_id(), cuda_device)
    assert didx._lib.fpb_comm_nccl_version() > 0
    for n_full, top_k in ((64, 10), (4096, 40)):
        params = DeviceIndex.make_params(top_k, n_full, 8)
        ids, scores, counts = didx.search(q16, params)
        i2, s2, c2 = didx.search_sharded(comm, 1, q16, params)
        torch.cuda.synchronize()
        assert torch.equal(i2, ids) and torch.equal(s2, scores) and torch.equal(c2, counts)
        h = didx.search_sharded_host(comm, 1, queries, params)
        assert torch.equal(h[0], ids.cpu()) and torch.equal(h[1], scores.cpu()) and torch.equal(h[2], counts.cpu())
    with pytest.raises(ValueError):
        didx.search_sharded(comm, 2, q16, params)  # 2 query groups do not divide 1 rank
    comm.close()
    fp = FastPlaid.from_device_index(didx, shard=(0, 1))
    plain = FastPlaid.from_device_index(didx)
    assert fp.search(queries, top_k=10) == plain.search(queries, top_k=10)
    # token-score matrices through the sharded surface (the owning rank computes, search.rs:668-686)
    a_ts = fp.search_token_scores(queries, top_k=4)
    b_ts = plain.search_token_scores(queries, top_k=4)
    for ra, rb in zip(a_ts, b_ts):
        assert [(d, s_) for d, s_, _ in ra] == [(d, s_) for d, s_, _ in rb]
        assert all(torch.equal(ma, mb) for (_, _, ma), (_, _, mb) in zip(ra, rb))
    fp.close()


def test_adaptive_approx_mode_switches_without_changing_results(cuda_device):
    """The host path re-examines, every few calls, how much the exact pass of the two-pass approximate stage had to
    re-score and holds the one-pass mode when that is high; both modes must return the same bytes."""
    from fast_plaid_b200.engine import DeviceIndex

    docs = make_docs(800, 10, 60, seed=51)
    oidx, _ = build_oracle_index(docs)
    didx = DeviceIndex(to_index_tensors(oidx), cuda_device)
    queries = make_queries(6, 32, seed=52, docs=docs)
    params = DeviceIndex.make_params(10, 256, 8)
    base = didx.search_host(queries, params)
    # (an index this small is scored in one pass anyway; the mechanism is what is under test: the probe sees
    # n_refine / n_cand = 0 > -1 and holds the explicit one-pass flag)
    didx.APPROX_PROBE_EVERY, didx.APPROX_DIRECT_ABOVE, didx.APPROX_HOLD_CALLS = 1, -1.0, 3  # force the switch
    assert not didx._approx_direct
    r1 = didx.search_host(queries, params)  # two-pass call that trips the switch
    assert didx._approx_direct
    for _ in range(3):  # held one-pass calls
        r = didx.search_host(queries, params)
        assert all(torch.equal(x, y) for x, y in zip(r, base))
    assert not didx._approx_direct  # probing the two-pass mode again
    assert all(torch.equal(x, y) for x, y in zip(r1, base))


def test_sharded_subset_search_equals_the_unsharded_subset_search(cuda_device):
    """subset= with documents sharded: the centroid bitmaps of the shards are OR-ed (the all-gather is
    emulated by stacking, all shards live on one device) and the result must equal the single-index
    subset search bit for bit, including a subset that lives entirely in one shard and an empty one."""
    from fast_plaid_b200.engine import FPB_FLAG_SUBSET, DeviceIndex, shard_tensors

    docs = make_docs(900, 10, 60, seed=31)
    oidx, _ = build_oracle_index(docs)
    t = to_index_tensors(oidx)
    whole = DeviceIndex(t, cuda_device)
    queries = make_queries(5, 32, seed=32, docs=docs).half().to(cuda_device)
    g = torch.Generator().manual_seed(33)
    subset = [torch.randperm(900, generator=g)[:300].tolist(),
              list(range(0, 200)),                      # only in the first shard(s)
              [],                                       # empty: no result
              torch.randperm(900, generator=g)[:40].tolist(),
              list(range(880, 900)) + [5, 5, 7]]        # duplicates, both ends
    for n_full, top_k in ((64, 10), (4096, 50)):
        params = DeviceIndex.make_params(top_k, n_full, 8)
        ids, scores, counts = whole.search(queries, params, subset=subset)
        for world in (2, 3):
            shards = []
            for r in range(world):
                sh, base = shard_tensors(t, r, world)
                shards.append(DeviceIndex(sh, cuda_device, doc_id_base=base))
            ps = DeviceIndex.with_flags(params, FPB_FLAG_SUBSET)
            Q = int(queries.shape[1])
            cbs = torch.stack([d.shard_subset_begin(queries, ps, subset) for d in shards])
            all_keys = torch.stack([d.shard_subset_keys(cbs, Q, ps) for d in shards])
            recs = [d.shard_exact_records(all_keys, r, Q, ps) for r, d in enumerate(shards)]
            i2, s2, c2 = whole.merge_records(torch.stack(recs), top_k)
            torch.cuda.synchronize()
            assert torch.equal(c2, counts), (world, n_full, c2.tolist(), counts.tolist())
            assert int(c2[2]) == 0
            for b in range(queries.shape[0]):
                n = int(counts[b])
                assert torch.equal(i2[b, :n], ids[b, :n]) and torch.equal(s2[b, :n], scores[b, :n]), (world, n_full, b)
                assert set(i2[b, :n].tolist()) <= set(subset[b])


def test_chunked_pinned_upload_equals_the_direct_copy(cuda_device, monkeypatch):
    """Loader fast path: arrays above the threshold stream through two pinned staging buffers with the
    int64 -> int32 narrowing done while copying into pinned memory; contents must equal `.to()`."""
    from fast_plaid_b200 import engine

    g = torch.Generator().manual_seed(3)
    codes = torch.randint(0, 2**31 - 1, (100_003,), generator=g, dtype=torch.int64)
    res = torch.randint(0, 256, (50_001, 64), generator=g, dtype=torch.uint8)
    monkeypatch.setattr(engine, "UPLOAD_DIRECT_BYTES", 1024)
    monkeypatch.setattr(engine, "UPLOAD_CHUNK_BYTES", 37 * 1024)  # many chunks, ragged last chunk
    dev = torch.device(cuda_device)
    a = engine.upload_narrow(codes, dev, torch.int32)
    b = engine.upload_narrow(res, dev, torch.uint8)
    assert a.dtype == torch.int32 and torch.equal(a.cpu(), codes.to(torch.int32))
    assert b.dtype == torch.uint8 and torch.equal(b.cpu(), res)
    # a whole index built through the chunked path searches identically
    docs = make_docs(300, 10, 40, seed=5)
    oidx, _ = build_oracle_index(docs)
    t = to_index_tensors(oidx)
    q = make_queries(3, 32, seed=6, docs=docs).half().to(cuda_device)
    p = engine.DeviceIndex.make_params(10, 128, 8)
    chunked = engine.DeviceIndex(t, cuda_device)
    monkeypatch.setattr(engine, "UPLOAD_DIRECT_BYTES", 1 << 40)
    direct = engine.DeviceIndex(t, cuda_device)
    r1, r2 = chunked.search(q, p), direct.search(q, p)
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(r1, r2))
