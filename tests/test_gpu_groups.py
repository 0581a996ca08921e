"""Grouped results (`group_by=`, fpb_index_with_groups): each query gets at most one document per group, the group's
best under the canonical order (score desc, then id asc), ranked in that order, with the ungrouped scores bit for bit.

- Exact search equals the host collapse of the canonical ranking of `exhaustive_scores` (restricted to the subset).
- `search` equals the host collapse of the ungrouped search with top_k = n_full_scores // 4, cut to top_k.
GPU tests are marked; the argument checks at the end run without a GPU."""

from __future__ import annotations

import ctypes
import random

import numpy as np
import pytest
import torch
from test_gpu_exhaustive import _device_index, _index_with_empty_and_long_docs
from util import build_oracle_index, make_docs, make_queries, oracle_exact_scores

from fast_plaid_b200 import engine
from fast_plaid_b200.engine import Groups

CODECS = [(128, 4), (128, 2), (64, 4), (64, 2), (128, 1)]


def _canonical(scores: torch.Tensor, members) -> list[int]:
    """Members (all documents when None) by (score desc, id asc)."""
    s = scores.double().numpy()
    ids = np.arange(s.shape[0]) if members is None else np.asarray(sorted(members), dtype=np.int64)
    if ids.size == 0:
        return []
    order = np.lexsort((ids, -s[ids]))
    return ids[order].tolist()


def _collapse(ranked: list[int], groups, k: int) -> list[int]:
    out, seen = [], set()
    for d in ranked:
        g = int(groups[d])
        if g not in seen:
            seen.add(g)
            out.append(d)
            if len(out) == k:
                break
    return out


def _check_rows(ids, sc, counts, every, groups, k, members=None) -> None:
    """Row b is the collapse of the canonical ranking of row b of `every` (restricted to members[b])."""
    for b in range(ids.shape[0]):
        exp = _collapse(_canonical(every[b], None if members is None else members[b]), groups, k)
        m = len(exp)
        assert int(counts[b]) == m, f"query {b} k={k}: count {int(counts[b])}, expected {m}"
        assert ids[b, :m].tolist() == exp, f"query {b} k={k}: not the host collapse of the canonical ranking"
        ref = every[b, torch.tensor(exp, dtype=torch.int64)] if m else sc[b, :0]
        assert torch.equal(sc[b, :m], ref), f"query {b} k={k}: a score is not the ungrouped one"
        assert torch.all(ids[b, m:] == -1) and torch.all(sc[b, m:] == float("-inf"))


def _group_maps(n: int, seed: int = 5) -> dict[str, torch.Tensor]:
    rng = random.Random(seed)
    return {
        "singletons": torch.arange(n, dtype=torch.int64),
        "one": torch.full((n,), 7, dtype=torch.int64),
        "runs10": torch.arange(n, dtype=torch.int64) // 10,
        "random": torch.tensor([rng.randint(1, 1000) for _ in range(n)], dtype=torch.int64),
        "sparse": torch.tensor([(1 << 62) + rng.randrange(0, 1 << 40, 1 << 30) for _ in range(n)], dtype=torch.int64),
        "pairs_i32": (torch.arange(n, dtype=torch.int32) * 7919 % 13),
    }


@pytest.mark.gpu
@pytest.mark.parametrize("dim,nbits", CODECS)
def test_exact_is_the_collapse_of_the_canonical_ranking(dim, nbits, cuda_device):
    """Every group map and top_k 1, 10, more than the groups and 4096, on a ragged index with an empty document
    and 2000-token documents."""
    oidx, empty_at, _ = _index_with_empty_and_long_docs(dim, nbits)
    didx = _device_index(oidx, cuda_device, ivf=False)
    n = didx.num_documents
    q16 = make_queries(4, 32, dim=dim, seed=300 + dim + nbits).half().to(cuda_device)
    every = didx.exhaustive_scores(q16).cpu()
    for name, g in _group_maps(n).items():
        groups = Groups.from_tensor(g, n, cuda_device)
        inv = groups.ids.cpu()
        for k in (1, 10, groups.n_groups + 5, 4096):
            ids, sc, counts = (t.cpu() for t in didx.search_exhaustive(q16, k, groups=groups))
            _check_rows(ids, sc, counts, every, inv, k)
            if name == "singletons":
                plain = [t.cpu() for t in didx.search_exhaustive(q16, k)]
                assert torch.equal(ids, plain[0]) and torch.equal(sc, plain[1]) and torch.equal(counts, plain[2])
        if name == "one":
            assert torch.equal(counts, torch.ones_like(counts))
    # the empty document alone in its group is still a group present
    g = torch.zeros(n, dtype=torch.int64)
    g[empty_at] = 1
    ids, sc, counts = (t.cpu() for t in didx.search_exhaustive(q16, 5, groups=Groups.from_tensor(g, n, cuda_device)))
    assert torch.all(counts == 2) and torch.all(ids[:, 1] == empty_at)


@pytest.mark.gpu
def test_exact_ties(cuda_device):
    """Duplicated documents score the same: in one group the smaller id represents it, in different groups both
    are kept, the smaller id first."""
    docs = make_docs(30, 3, 30, seed=91)
    docs = docs + [d.clone() for d in docs[:12]]
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    n = didx.num_documents
    q16 = make_queries(3, 32, seed=92, docs=docs).half().to(cuda_device)
    every = didx.exhaustive_scores(q16).cpu()
    assert torch.equal(every[:, :12], every[:, 30:42])
    same = torch.arange(n) % 30
    for g in (same, torch.arange(n), torch.arange(n) % 4):
        groups = Groups.from_tensor(g, n, cuda_device)
        for k in (1, 5, 40):
            ids, sc, counts = (t.cpu() for t in didx.search_exhaustive(q16, k, groups=groups))
            _check_rows(ids, sc, counts, every, groups.ids.cpu(), k)
    ids, _, _ = didx.search_exhaustive(q16, 40, groups=Groups.from_tensor(same, n, cuda_device))
    assert int(ids.max()) < 30  # every copy loses its tie to the original


@pytest.mark.gpu
def test_exact_against_the_oracle(cuda_device):
    docs = make_docs(60, 1, 40, seed=93)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    n = didx.num_documents
    queries = make_queries(2, 32, seed=94, docs=docs)
    g = torch.arange(n) // 6
    ids, sc, counts = (t.cpu() for t in didx.search_exhaustive(queries.half().to(cuda_device), 20,
                                                                 groups=Groups.from_tensor(g, n, cuda_device)))
    for b in range(2):
        ref = oracle_exact_scores(oidx, queries[b], list(range(n))).float()
        assert int(counts[b]) == 10
        got = ids[b, :10].tolist()
        assert sorted(int(g[d]) for d in got) == list(range(10))
        assert torch.allclose(sc[b, :10], ref[got], rtol=1e-3, atol=1e-2)
        for d in got:  # each is its group's best up to the oracle's rounding
            members = (g == g[d]).nonzero().flatten()
            assert float(ref[d]) >= float(ref[members].max()) - 1e-2


def _fastplaid(didx):
    from fast_plaid_b200.search import fast_plaid as fpmod

    return fpmod.FastPlaid.from_device_index(didx)


def _subset_forms(n: int, B: int, rng: random.Random):
    shared = sorted(rng.sample(range(n), n // 2))
    rows = [sorted(rng.sample(range(n), rng.randint(0, n // 3))) for _ in range(B)]
    width = max(len(r) for r in rows)
    padded = torch.full((B, width), -1, dtype=torch.int64)
    for b, r in enumerate(rows):
        padded[b, :len(r)] = torch.tensor(r, dtype=torch.int64)
    mask = torch.zeros(n, dtype=torch.bool)
    mask[shared] = True
    masks = torch.zeros((B, n), dtype=torch.bool)
    for b, r in enumerate(rows):
        masks[b, r] = True
    return [
        (shared, [shared] * B),
        (rows, rows),
        (torch.tensor(shared), [shared] * B),
        (padded, rows),
        (mask, [shared] * B),
        (masks, rows),
    ]


def _as_rows(res, k: int):
    ids = torch.full((len(res), k), -1, dtype=torch.int64)
    sc = torch.full((len(res), k), float("-inf"), dtype=torch.float32)
    counts = torch.zeros(len(res), dtype=torch.int32)
    for b, r in enumerate(res):
        counts[b] = len(r)
        for i, (d, s) in enumerate(r):
            ids[b, i], sc[b, i] = d, s
    return ids, sc, counts


@pytest.mark.gpu
def test_exact_with_every_subset_form(cuda_device):
    docs = make_docs(120, 1, 30, seed=95)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    n, B = didx.num_documents, 4
    fp = _fastplaid(didx)
    q = make_queries(B, 32, seed=96, docs=docs)
    every = didx.exhaustive_scores(q.half().to(cuda_device)).cpu()
    g = torch.tensor([random.Random(97).randint(0, 30) for _ in range(n)])
    inv = torch.unique(g, return_inverse=True)[1]
    for form, members in _subset_forms(n, B, random.Random(98)):
        for k in (1, 10, 40):
            res = fp.search_exhaustive(q.to(cuda_device), top_k=k, subset=form, group_by=g.to(cuda_device))
            ids, sc, counts = _as_rows(res, k)
            _check_rows(ids, sc, counts, every, inv, k, members=members)


def _host_collapse(res, groups: torch.Tensor, k: int):
    """Each row of (doc, score) pairs with every group's first pair kept, cut to k."""
    out = []
    for row in res:
        seen, kept = set(), []
        for d, s in row:
            if int(groups[d]) not in seen:
                seen.add(int(groups[d]))
                kept.append((d, s))
        out.append(kept[:k])
    return out


@pytest.mark.gpu
def test_approximate_is_the_collapse_of_the_rerank_list(cuda_device):
    """search(top_k=k, group_by=g, n_full_scores=n) == collapse(search(top_k=max(n // 4, 1), n_full_scores=n))[:k]
    for n 4 .. 16384, n_ivf_probe 8 and 64, every subset form, device and host (fp32 CPU) queries."""
    docs = make_docs(400, 4, 40, seed=99)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    n_docs, B = didx.num_documents, 3
    fp = _fastplaid(didx)
    q = make_queries(B, 32, seed=100, docs=docs)
    g = torch.arange(n_docs) // 5
    forms = [(None, None)] + _subset_forms(n_docs, B, random.Random(101))
    for n_full in (4, 40, 1000, 16384):
        R = max(n_full // 4, 1)
        for probe in (8, 64):
            for form, _ in forms:
                for queries in (q.to(cuda_device), q) if form is None else (q.to(cuda_device),):
                    base = fp.search(queries, top_k=R, n_full_scores=n_full, n_ivf_probe=probe, subset=form)
                    for k in (1, 10):
                        got = fp.search(queries, top_k=k, n_full_scores=n_full, n_ivf_probe=probe, subset=form,
                                        group_by=g)
                        assert got == _host_collapse(base, g, k), (n_full, probe, k, type(form))


@pytest.mark.gpu
def test_results_do_not_depend_on_the_split(cuda_device, monkeypatch):
    oidx, _, _ = _index_with_empty_and_long_docs(128, 4)
    didx = _device_index(oidx, cuda_device)
    n = didx.num_documents
    q16 = make_queries(9, 32, seed=102).half().to(cuda_device)
    groups = Groups.from_tensor(torch.arange(n) // 3, n, cuda_device)
    ref = [t.cpu() for t in didx.search_exhaustive(q16, 10, groups=groups)]
    small = didx.exhaustive_workspace_bytes(2, 32, 10)
    got = [t.cpu() for t in didx.search_exhaustive(q16, 10, budget_bytes=small, groups=groups)]
    assert all(torch.equal(a, b) for a, b in zip(ref, got))
    rows = torch.randint(-1, n, (9, 30), generator=torch.Generator().manual_seed(1)).to(cuda_device)
    ref_rows = [t.cpu() for t in didx.search_exhaustive(q16, 10, subset=rows, groups=groups)]
    for dpc in ("1", "32"):
        monkeypatch.setenv("FPB_K7_DOCS_PER_CHUNK", dpc)
        got = [t.cpu() for t in didx.search_exhaustive(q16, 10, groups=groups)]
        assert all(torch.equal(a, b) for a, b in zip(ref, got)), dpc
        got = [t.cpu() for t in didx.search_exhaustive(q16, 10, subset=rows, groups=groups)]
        assert all(torch.equal(a, b) for a, b in zip(ref_rows, got)), dpc


@pytest.mark.gpu
def test_token_scores_follow_the_grouped_results(cuda_device):
    docs = make_docs(200, 4, 30, seed=103)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    fp = _fastplaid(didx)
    q = make_queries(2, 32, seed=104, docs=docs).to(cuda_device)
    g = torch.arange(didx.num_documents) // 4
    grouped = fp.search(q, top_k=8, group_by=g)
    full = fp.search_token_scores(q, top_k=8, group_by=g)
    assert [[(d, s) for d, s, _ in r] for r in full] == grouped
    plain = {(b, d): m for b, r in enumerate(fp.search_token_scores(q, top_k=1000)) for d, _, m in r}
    for b, r in enumerate(full):
        for d, _, m in r:
            assert torch.equal(m, plain[(b, d)])


@pytest.mark.gpu
def test_a_map_of_the_old_length_is_refused_after_update_and_delete(cuda_device):
    docs = make_docs(50, 2, 20, seed=105)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    n = didx.num_documents
    old = Groups.from_tensor(torch.arange(n), n, cuda_device)
    q16 = make_queries(1, 32, seed=106).half().to(cuda_device)
    o0, o1 = int(didx.doc_offsets[0]), int(didx.doc_offsets[1])
    grown = didx.append(didx.doc_codes[o0:o1].cpu(), didx.doc_residuals[o0:o1].cpu(), torch.tensor([o1 - o0]))
    smaller = didx.delete([3])
    for idx in (grown, smaller):
        with pytest.raises(ValueError):
            idx.search_exhaustive(q16, 5, groups=old)
        with pytest.raises(ValueError):
            Groups.check(torch.arange(n), idx.num_documents)
        ok = Groups.from_tensor(torch.arange(idx.num_documents), idx.num_documents, cuda_device)
        assert int(idx.search_exhaustive(q16, 5, groups=ok)[2][0]) == 5


@pytest.mark.gpu
def test_grouped_handles_are_refused_by_the_sharded_entry_points(cuda_device):
    docs = make_docs(20, 2, 10, seed=107)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    lib = engine.load_library()
    gids = torch.zeros(didx.num_documents, dtype=torch.int32, device=cuda_device)
    h = ctypes.c_void_p()
    assert lib.fpb_index_with_groups(ctypes.byref(h), didx._handle, gids.data_ptr(), 1) == engine.FPB_OK
    try:
        assert lib.fpb_search_shard(h, None, 1, 1, None, None, 0, None, None) == engine.FPB_ERR_UNSUPPORTED
        assert lib.fpb_shard_approx_keys(h, None, 1, 1, None, None, 0, None, None) == engine.FPB_ERR_UNSUPPORTED
        assert lib.fpb_stage_records(h, 1, 1, None, None, 0, None, None) == engine.FPB_ERR_UNSUPPORTED
        assert lib.fpb_stage_keys(h, 1, 1, None, None, 0, None, None) == engine.FPB_ERR_UNSUPPORTED
        assert lib.fpb_shard_exhaustive_records(h, None, 1, 1, 1, None, 0, None, None) == engine.FPB_ERR_UNSUPPORTED
        assert lib.fpb_search_exhaustive_sharded(h, None, 1, None, 1, 1, 1, None, 0, None, 0, None, None, None,
                                                 None) == engine.FPB_ERR_UNSUPPORTED
        assert b"groups" in lib.fpb_last_error()
    finally:
        lib.fpb_index_destroy(h)


# ---- no GPU needed ---------------------------------------------------------------------------------------------


def test_group_maps_are_checked():
    Groups.check(torch.tensor([0, 5, 2**62], dtype=torch.int64), 3)
    Groups.check(torch.tensor([1, 1, 0], dtype=torch.int32), 3)
    bad = [
        torch.tensor([0, 1], dtype=torch.int64),  # wrong length
        torch.tensor([0.0, 1.0, 2.0]),
        torch.tensor([True, False, True]),
        torch.zeros((3, 1), dtype=torch.int64),
        torch.tensor([0, -1, 2]),
        [0, 1, 2],
    ]
    for g in bad:
        with pytest.raises(ValueError):
            Groups.check(g, 3)


def test_with_groups_refuses_bad_arguments():
    lib = engine.load_library()
    fake = torch.zeros(64, dtype=torch.uint8)  # never dereferenced: the checks come first
    gids = torch.zeros(4, dtype=torch.int32)
    h = ctypes.c_void_p()
    assert lib.fpb_index_with_groups(None, fake.data_ptr(), gids.data_ptr(), 1) == engine.FPB_ERR_INVALID
    assert lib.fpb_index_with_groups(ctypes.byref(h), None, gids.data_ptr(), 1) == engine.FPB_ERR_INVALID
    assert lib.fpb_index_with_groups(ctypes.byref(h), fake.data_ptr(), None, 1) == engine.FPB_ERR_INVALID
    for n_groups in (0, -1, 2**31):
        assert lib.fpb_index_with_groups(ctypes.byref(h), fake.data_ptr(), gids.data_ptr(), n_groups) \
            == engine.FPB_ERR_INVALID
        assert b"n_groups" in lib.fpb_last_error()
    assert h.value is None


def test_sharded_group_by_is_refused_before_any_exchange():
    from fast_plaid_b200.search import fast_plaid as fpmod

    fp = object.__new__(fpmod.FastPlaid)
    fp.shard = (0, 2)
    fp._comm = None
    g = torch.zeros(4, dtype=torch.int64)
    with pytest.raises(NotImplementedError):
        fp.search(torch.zeros((1, 4, 128)), group_by=g)
    with pytest.raises(NotImplementedError):
        fp.search_exhaustive(torch.zeros((1, 4, 128)), group_by=g)
    assert fp._comm is None
