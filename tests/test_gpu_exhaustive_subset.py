"""Exhaustive exact search over document subsets (fpb_search_exhaustive_subset, K7 walking per-list documents).

The contract: query b gets the top_k of the SET of valid documents of its subset by (score desc, id asc), each score
bit-identical to the full scan's score of the same document.  GPU tests are marked; the last tests are the CPU tier
(the grouping of subsets into lists, argument checks, the document-sharded refusal)."""

from __future__ import annotations

import ctypes
import random

import pytest
import torch
from test_gpu_exhaustive import CONFIGS, _device_index, _index_with_empty_and_long_docs
from util import build_oracle_index, make_docs, make_queries

SENTINEL = -10000.0


def _invalid(n: int) -> list[int]:
    return [-1, n, n + 5, 2**31 - 1]


def _messy(docs: list[int], n: int, rng: random.Random, invalid: bool = True) -> list[int]:
    """`docs` unsorted, with duplicates and (invalid=True) the ids -1, N, N + 5 and 2^31 - 1 mixed in."""
    out = list(docs) + [rng.choice(docs) for _ in range(len(docs) // 3 + 1)] if docs else []
    if invalid:
        out += _invalid(n)
    rng.shuffle(out)
    return out


def _check_against_full_scan(ids, sc, counts, every, subsets, k, n) -> None:
    """Row b is the canonical top k of the valid set of subsets[b], scores bit-identical to the full scan's."""
    for b, sub in enumerate(subsets):
        members = sorted({d for d in sub if 0 <= d < n})
        exp = _canonical_subset(every[b], members, k)
        m = len(exp)
        assert int(counts[b]) == m == min(k, len(members)), f"query {b}: count {int(counts[b])} vs {m}"
        assert ids[b, :m].tolist() == exp, f"query {b} k={k}: ids are not the canonical sort of the set"
        got = sc[b, :m]
        ref = every[b, torch.tensor(exp, dtype=torch.int64)] if m else got
        assert torch.equal(got, ref), f"query {b} k={k}: a score is not the full scan's bit for bit"
        assert torch.all(ids[b, m:] == -1) and torch.all(sc[b, m:] == float("-inf"))


def _canonical_subset(scores: torch.Tensor, members: list[int], k: int) -> list[int]:
    return sorted(members, key=lambda d: (-float(scores[d]), d))[:k]


@pytest.mark.gpu
@pytest.mark.parametrize("dim,nbits,Q", CONFIGS)
def test_scores_are_the_full_scans_bit_for_bit(dim, nbits, Q, cuda_device):
    """Per-query lists of 0, 1, 7, 33, 100 entries and all N documents, unsorted, with duplicates and invalid ids, on
    a ragged index with an empty document and 2000-token documents."""
    oidx, empty_at, _ = _index_with_empty_and_long_docs(dim, nbits)
    didx = _device_index(oidx, cuda_device, ivf=False)
    n = didx.num_documents
    rng = random.Random(1000 + Q)
    subsets = [[]]
    for length in (1, 7, 33, 100):
        subsets.append(_messy([rng.randrange(n) for _ in range(length)], n, rng, invalid=length >= 7))
    subsets.append(_messy(list(range(n)), n, rng))
    q16 = make_queries(len(subsets), Q, dim=dim, seed=2000 + Q).half().to(cuda_device)
    every = didx.exhaustive_scores(q16).cpu()
    assert torch.all(every[:, empty_at] == Q * SENTINEL)
    for k in (n + 5, 1, 5, 20):
        ids, sc, counts = (t.cpu() for t in didx.search_exhaustive(q16, k, subset=subsets))
        assert ids.shape == (len(subsets), k)
        _check_against_full_scan(ids, sc, counts, every, subsets, k, n)
        if k > n:  # the empty document scores Q x -10000 and ranks last
            assert int(ids[-1, n - 1]) == empty_at and float(sc[-1, n - 1]) == Q * SENTINEL
    assert int(counts[0]) == 0


@pytest.mark.gpu
def test_grouping_does_not_change_the_bytes(cuda_device):
    """One broadcast list, the same contents as distinct lists, and interleaved sharing (queries 0, 2, 4 share list A,
    1 and 3 list B) all give the bytes of every query searched alone.  Q = 48 with 5 queries: the rows of one list
    cross a 128-row stage boundary."""
    oidx, _, _ = _index_with_empty_and_long_docs()
    didx = _device_index(oidx, cuda_device, ivf=False)
    n = didx.num_documents
    rng = random.Random(7)
    q16 = make_queries(5, 48, seed=301).half().to(cuda_device)
    a = _messy(rng.sample(range(n), 40), n, rng)
    b = _messy(rng.sample(range(n), 9), n, rng)
    k = 30

    def alone(subsets):
        rows = [didx.search_exhaustive(q16[i : i + 1], k, subset=[subsets[i]]) for i in range(5)]
        return tuple(torch.cat([r[j] for r in rows]).cpu() for j in range(3))

    def same(x, y):
        return all(torch.equal(u.cpu(), v.cpu()) for u, v in zip(x, y))

    ref = alone([a] * 5)
    assert same(didx.search_exhaustive(q16, k, subset=[a] * 5), ref)
    assert same(didx.search_exhaustive(q16, k, subset=[list(a) for _ in range(5)]), ref)
    shared = [a, b, a, b, a]
    ref_shared = alone(shared)
    assert same(didx.search_exhaustive(q16, k, subset=shared), ref_shared)
    assert same(didx.search_exhaustive(q16, k, subset=[list(x) for x in shared]), ref_shared)
    every = didx.exhaustive_scores(q16).cpu()
    _check_against_full_scan(*ref_shared, every, shared, k, n)
    # a shard's index (doc_id_base > 0): global ids in, global ids out
    base = 1000
    from fast_plaid_b200.engine import DeviceIndex
    from util import to_index_tensors

    shard = DeviceIndex(to_index_tensors(oidx), cuda_device, doc_id_base=base)
    ids, sc, counts = (t.cpu() for t in shard.search_exhaustive(q16, k, subset=[[d + base for d in x] for x in shared]))
    # the valid ids shifted by base stay valid, every other id stays outside the index
    for bi, sub in enumerate(shared):
        members = sorted({d for d in sub if 0 <= d < n})
        exp = _canonical_subset(every[bi], members, k)
        assert ids[bi, : len(exp)].tolist() == [d + base for d in exp]
        assert torch.equal(sc[bi, : len(exp)], ref_shared[1][bi, : len(exp)])


@pytest.mark.gpu
def test_ties_go_to_the_smallest_ids(cuda_device):
    base = make_docs(120, 5, 30, seed=81)
    rng = random.Random(11)
    # duplicated documents (exact ties) inside subsets
    docs = base + [base[i].clone() for i in (3, 3, 50, 77, 119)]
    didx = _device_index(build_oracle_index(docs)[0], cuda_device)
    n = len(docs)
    q16 = make_queries(4, 32, seed=82, docs=docs).half().to(cuda_device)
    every = didx.exhaustive_scores(q16).cpu()
    subsets = [_messy([3, 120, 121, 50, 122, 77, 123, 119, 124, 10, 11], n, rng) for _ in range(4)]
    for k in (1, 3, 6, 20):
        ids, sc, counts = (t.cpu() for t in didx.search_exhaustive(q16, k, subset=subsets))
        _check_against_full_scan(ids, sc, counts, every, subsets, k, n)
    # more than 2048 copies of document 3, tied at the top of every query, inside one unsorted subset: k3b_select's
    # radix passes must pick the smallest ids among them
    docs = base + [base[3].clone() for _ in range(2100)]
    didx = _device_index(build_oracle_index(docs)[0], cuda_device)
    n = len(docs)
    q16 = make_queries(3, 32, seed=83, docs=[base[3]]).half().to(cuda_device)
    every = didx.exhaustive_scores(q16).cpu()
    top = every.max(dim=1, keepdim=True).values
    assert torch.all((every == top).sum(dim=1) > 2048)
    sub = _messy([3] + list(range(120, n)) + list(range(0, 120, 7)), n, rng)
    for k in (1, 10, 124, 2048, 4096):
        ids, sc, counts = (t.cpu() for t in didx.search_exhaustive(q16, k, subset=[sub] * 3))
        _check_against_full_scan(ids, sc, counts, every, [sub] * 3, k, n)


@pytest.mark.gpu
def test_chunk_size_batch_split_and_repeats_give_the_same_bytes(cuda_device, monkeypatch):
    oidx, _, _ = _index_with_empty_and_long_docs()
    didx = _device_index(oidx, cuda_device, ivf=False)
    n = didx.num_documents
    rng = random.Random(21)
    shared = _messy(rng.sample(range(n), 30), n, rng)
    subsets = [shared if i % 3 == 0 else _messy(rng.sample(range(n), 5 + 4 * i), n, rng) for i in range(13)]
    q16 = make_queries(13, 48, seed=111).half().to(cuda_device)
    k = 15
    first = None
    for dpc in (32, 13, 4, 2, 1):
        monkeypatch.setenv("FPB_K7_DOCS_PER_CHUNK", str(dpc))
        got = tuple(t.cpu() for t in didx.search_exhaustive(q16, k, subset=subsets))
        if first is None:
            _check_against_full_scan(*got, didx.exhaustive_scores(q16).cpu(), subsets, k, n)
            first = got
        else:
            assert all(torch.equal(x, y) for x, y in zip(got, first)), f"chunks of {dpc} documents change the result"
    monkeypatch.delenv("FPB_K7_DOCS_PER_CHUNK")
    max_len = max(len(s) for s in subsets)
    small = didx.exhaustive_subset_workspace_bytes(3, 48, k, 3, max_len)  # about three queries per call
    split = tuple(t.cpu() for t in didx.search_exhaustive(q16, k, budget_bytes=small, subset=subsets))
    assert all(torch.equal(x, y) for x, y in zip(split, first))
    for _ in range(2):
        again = tuple(t.cpu() for t in didx.search_exhaustive(q16, k, subset=subsets))
        assert all(torch.equal(x, y) for x, y in zip(again, first))


def _fastplaid_index(tmp_path, device, **kw):
    from fast_plaid_b200 import search

    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device=device)
    docs = make_docs(250, 5, 60, seed=121)
    fp.create(docs, kmeans_niters=2, **kw)
    return path, fp, docs


def _filtered(full: list[tuple[int, float]], subset) -> list[tuple[int, float]]:
    keep = set(subset)
    return [(d, s) for d, s in full if d in keep]


@pytest.mark.gpu
def test_fastplaid_surface(tmp_path, cuda_device):
    from fast_plaid_b200 import filtering

    meta = [{"lang": "en" if i % 3 else "fr"} for i in range(250)]
    path, fp, docs = _fastplaid_index(tmp_path, cuda_device, metadata=meta)
    queries = make_queries(6, 32, seed=122, docs=docs)
    full = fp.search_exhaustive(queries, top_k=250)
    assert fp.search_exhaustive(queries, top_k=12, subset=None) == fp.search_exhaustive(queries, top_k=12)
    assert fp.search_exhaustive(queries, top_k=12, subset=[]) == fp.search_exhaustive(queries, top_k=12)
    # one id
    res = fp.search_exhaustive(queries, top_k=5, subset=17)
    assert res == [_filtered(f, [17]) for f in full]
    # one list for every query: the result of a metadata filter
    fr = filtering.where(path, "lang = ?", ("fr",))
    assert len(fr) == 84
    res = fp.search_exhaustive(queries, top_k=100, subset=fr)
    assert res == [_filtered(f, fr) for f in full]
    # one list per query, k below and above the subset size
    rng = random.Random(5)
    per = [rng.sample(range(250), 3 + 11 * b) for b in range(6)]
    res = fp.search_exhaustive(queries, top_k=60, subset=per)
    assert res == [_filtered(f, s) for f, s in zip(full, per)]
    res = fp.search_exhaustive(queries, top_k=4, subset=per)
    assert res == [_filtered(f, s)[:4] for f, s in zip(full, per)]
    # fp32 host and fp16 device queries
    assert fp.search_exhaustive(queries.to(cuda_device).half(), top_k=60, subset=per) == \
        fp.search_exhaustive(queries, top_k=60, subset=per)
    with pytest.raises(ValueError, match="Subset length"):
        fp.search_exhaustive(queries, top_k=5, subset=per[:5])
    fp.close()


@pytest.mark.gpu
def test_compress_only_index(tmp_path, cuda_device):
    path, fp, docs = _fastplaid_index(tmp_path, cuda_device, compress_only=True)
    queries = make_queries(4, 32, seed=131, docs=docs)
    full = fp.search_exhaustive(queries, top_k=250)
    sub = list(range(0, 250, 4))
    assert fp.search_exhaustive(queries, top_k=100, subset=sub) == [_filtered(f, sub) for f in full]
    fp.close()


@pytest.mark.gpu
def test_two_devices_equal_one(tmp_path, cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from fast_plaid_b200 import search

    path, fp, docs = _fastplaid_index(tmp_path, cuda_device)
    queries = make_queries(7, 32, seed=141, docs=docs)
    per = [list(range(b, 250, 7)) for b in range(7)]
    one = fp.search_exhaustive(queries, top_k=10, subset=per)
    fp.close()
    fp2 = search.FastPlaid(path, device=["cuda:0", "cuda:1"])
    assert fp2.search_exhaustive(queries, top_k=10, subset=per) == one
    fp2.close()


def test_grouping_of_subsets_into_lists():
    from fast_plaid_b200.engine import group_subsets

    ids = [5, 3, 9]
    lists, qlist = group_subsets([ids] * 4)  # the broadcast form: one object
    assert lists == [ids] and qlist == [0, 0, 0, 0]
    lists, qlist = group_subsets([[1, 2], [1, 2], [3]])  # equal contents
    assert lists == [[1, 2], [3]] and qlist == [0, 0, 1]
    lists, qlist = group_subsets([[1, 2], [], [3], []])  # an empty list is a list of its own
    assert lists == [[1, 2], [], [3]] and qlist == [0, 1, 2, 1]
    lists, qlist = group_subsets([[2, 1], [1, 2]])  # order matters to the grouping, not to the result
    assert qlist == [0, 1]


def test_c_abi_refuses_bad_arguments():
    from fast_plaid_b200.engine import FPB_ERR_INVALID, FPB_ERR_UNSUPPORTED, load_library

    lib = load_library()
    h = (ctypes.c_int32 * 4)(0, 0, 0, 0)

    def call(B=4, Q=32, top_k=10, n_lists=1, h_list=h):
        return lib.fpb_search_exhaustive_subset(None, None, B, Q, top_k, None, None, n_lists, 8, h_list, None, 0,
                                                None, None, None, None)

    assert call(top_k=0) == FPB_ERR_INVALID
    assert b"top_k=0 must be >= 1" in lib.fpb_last_error()
    assert call(top_k=5000) == FPB_ERR_UNSUPPORTED
    assert b"top_k=5000" in lib.fpb_last_error()
    assert call(Q=300) == FPB_ERR_UNSUPPORTED
    assert b"Q=300" in lib.fpb_last_error()
    assert call(n_lists=0) == FPB_ERR_INVALID
    assert b"n_lists=0" in lib.fpb_last_error()
    assert call(h_list=None) == FPB_ERR_INVALID
    assert b"NULL h_query_list" in lib.fpb_last_error()
    bad = (ctypes.c_int32 * 4)(0, 1, 2, 3)
    assert call(n_lists=3, h_list=bad) == FPB_ERR_INVALID
    assert b"h_query_list[3]=3 is not in [0, n_lists=3)" in lib.fpb_last_error()
    assert call() == FPB_ERR_INVALID  # every argument above is fine: the index is checked last
    assert b"NULL index" in lib.fpb_last_error()
    out = ctypes.c_size_t()
    assert lib.fpb_exhaustive_subset_workspace_bytes(None, 4, 32, 10, 0, 8, ctypes.byref(out)) == FPB_ERR_INVALID
    assert lib.fpb_exhaustive_subset_workspace_bytes(None, 4, 32, 10, 1, 8, ctypes.byref(out)) == FPB_ERR_INVALID
    assert b"NULL index" in lib.fpb_last_error()


def test_document_sharded_index_is_still_refused():
    from fast_plaid_b200 import search

    fp_sharded = search.FastPlaid.__new__(search.FastPlaid)
    fp_sharded.shard = (0, 2)
    with pytest.raises(NotImplementedError, match="document-sharded"):
        search.FastPlaid.search_exhaustive(fp_sharded, torch.randn(2, 8, 128), subset=[1, 2])
