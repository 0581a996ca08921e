"""Up to m documents per group (`group_by=` with `max_per_group=`, fpb_index_with_groups_max): walking the canonical
ranking (score desc, then id asc), a document is kept when fewer than m documents of its group were kept before it;
the first top_k kept documents come back with the ungrouped scores bit for bit.

- Exact search equals the rule applied on the host to the ungrouped full ranking (search_exhaustive, top_k = N).
- `search` equals the rule applied to the ungrouped search with top_k = n_full_scores // 4, cut to top_k.
GPU tests are marked; the argument checks at the end run without a GPU."""

from __future__ import annotations

import ctypes
import random

import numpy as np
import pytest
import torch
from test_gpu_exhaustive import _device_index, _index_with_empty_and_long_docs
from test_gpu_groups import _as_rows, _fastplaid, _subset_forms
from util import build_oracle_index, make_docs, make_queries

from fast_plaid_b200 import engine
from fast_plaid_b200.engine import Groups

CODECS = [(128, 4), (128, 2), (64, 4), (64, 2), (128, 1)]
LIMITS = (1, 2, 3, 7, 64)


def _limit(ranked, groups, m: int, k: int) -> list:
    """The first k entries of `ranked` (documents, or (document, score) pairs) of which fewer than m of the same
    group come before."""
    out, kept = [], {}
    for e in ranked:
        g = int(groups[e[0] if isinstance(e, tuple) else e])
        if kept.get(g, 0) < m:
            kept[g] = kept.get(g, 0) + 1
            out.append(e)
            if len(out) == k:
                break
    return out


def _check_rows(got, full, groups, m: int, k: int, members=None) -> None:
    """Row b of `got` (ids, scores, counts) is the rule applied to row b of the ungrouped full ranking `full`
    (restricted to members[b]), with the full ranking's scores bit for bit."""
    ids, sc, counts = got
    f_ids, f_sc, f_counts = full
    for b in range(ids.shape[0]):
        ranked = f_ids[b, : int(f_counts[b])].tolist()
        if members is not None:
            keep = set(members[b])
            ranked = [d for d in ranked if d in keep]
        exp = _limit(ranked, groups, m, k)
        n = len(exp)
        assert int(counts[b]) == n, f"query {b} m={m} k={k}: count {int(counts[b])}, expected {n}"
        assert ids[b, :n].tolist() == exp, f"query {b} m={m} k={k}: not the rule applied to the full ranking"
        pos = {d: i for i, d in enumerate(f_ids[b, : int(f_counts[b])].tolist())}
        ref = f_sc[b, torch.tensor([pos[d] for d in exp], dtype=torch.int64)] if n else sc[b, :0]
        assert torch.equal(sc[b, :n], ref), f"query {b} m={m} k={k}: a score is not the ungrouped one"
        assert torch.all(ids[b, n:] == -1) and torch.all(sc[b, n:] == float("-inf"))
        assert torch.all(sc[b, 1:n] <= sc[b, : max(n - 1, 0)]), f"query {b} m={m} k={k}: scores not non-increasing"


def _group_maps(n: int, seed: int = 15) -> dict[str, torch.Tensor]:
    rng = random.Random(seed)
    return {
        "singletons": torch.arange(n, dtype=torch.int64),
        "one": torch.full((n,), 3, dtype=torch.int64),
        "runs10": torch.arange(n, dtype=torch.int64) // 10,
        "random10": torch.tensor([rng.randint(0, max(n // 10, 1)) for _ in range(n)], dtype=torch.int64),
        "sparse": torch.tensor([(1 << 62) + rng.randrange(0, 1 << 40, 1 << 33) for _ in range(n)], dtype=torch.int64),
        "i32": (torch.arange(n, dtype=torch.int32) * 7919 % 13),
    }


def _admissible(groups: torch.Tensor, m: int) -> int:
    return int(torch.clamp(torch.bincount(groups.long()), max=m).sum())


def _exact_sweep(didx, q16, device) -> None:
    n = didx.num_documents
    full = [t.cpu() for t in didx.search_exhaustive(q16, n)]
    assert torch.all(full[2] == n)  # the whole canonical ranking
    for name, g in _group_maps(n).items():
        for m in LIMITS:
            groups = Groups.from_tensor(g, n, device, m)
            inv = groups.ids.cpu()
            largest = int(torch.bincount(inv.long()).max())
            for k in (1, 10, _admissible(inv, m) + 5, 4096):
                got = [t.cpu() for t in didx.search_exhaustive(q16, k, groups=groups)]
                _check_rows(got, full, inv, m, k)
                if m >= largest:  # no group is cut: the ungrouped bytes
                    plain = [t.cpu() for t in didx.search_exhaustive(q16, k)]
                    assert all(torch.equal(a, b) for a, b in zip(got, plain)), (name, m, k)


@pytest.mark.gpu
@pytest.mark.parametrize("dim,nbits", CODECS)
def test_exact_is_the_rule_applied_to_the_full_ranking(dim, nbits, cuda_device):
    """Every group map, m in {1, 2, 3, 7, 64} and top_k 1, 10, more than the admissible documents and 4096, on a
    ragged index with an empty document and 2000-token documents."""
    oidx, _, _ = _index_with_empty_and_long_docs(dim, nbits)
    didx = _device_index(oidx, cuda_device, ivf=False)
    _exact_sweep(didx, make_queries(4, 32, dim=dim, seed=400 + dim + nbits).half().to(cuda_device), cuda_device)


@pytest.mark.gpu
def test_exact_on_a_larger_index(cuda_device):
    """3000 documents: the keys of the m rounds in the accumulator region and after it, and wide selections."""
    docs = make_docs(3000, 1, 12, seed=410)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    _exact_sweep(didx, make_queries(3, 32, seed=411, docs=docs).half().to(cuda_device), cuda_device)


class _OneDocumentEntry:
    """The library with fpb_index_with_groups_max answered by fpb_index_with_groups: the one-per-group handle."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def fpb_index_with_groups_max(self, out, ix, ids, n_groups, m):
        assert m == 1
        return self._lib.fpb_index_with_groups(out, ix, ids, n_groups)


@pytest.mark.gpu
def test_one_per_group_is_the_bytes_of_the_one_document_handle(cuda_device, monkeypatch):
    docs = make_docs(300, 2, 30, seed=412)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    n = didx.num_documents
    q16 = make_queries(5, 32, seed=413, docs=docs).half().to(cuda_device)
    groups = Groups.from_tensor(torch.arange(n) // 7, n, cuda_device, 1)
    params = didx.make_params(10, 256, 16)
    new = [[t.cpu() for t in didx.search_exhaustive(q16, k, groups=groups)] for k in (1, 30)]
    new.append([t.cpu() for t in didx.search(q16, params, groups=groups)])
    monkeypatch.setattr(didx, "_lib", _OneDocumentEntry(didx._lib))
    old = [[t.cpu() for t in didx.search_exhaustive(q16, k, groups=groups)] for k in (1, 30)]
    old.append([t.cpu() for t in didx.search(q16, params, groups=groups)])
    for a, b in zip(new, old):
        assert all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.gpu
def test_exact_ties(cuda_device):
    """Duplicated documents score the same, inside one group and across groups: the smaller id comes first."""
    docs = make_docs(30, 3, 30, seed=414)
    docs = docs + [d.clone() for d in docs[:12]] + [d.clone() for d in docs[:6]]
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    n = didx.num_documents
    q16 = make_queries(3, 32, seed=415, docs=docs).half().to(cuda_device)
    full = [t.cpu() for t in didx.search_exhaustive(q16, n)]
    for g in (torch.arange(n) % 30, torch.arange(n), torch.arange(n) % 4, torch.arange(n) // 20):
        for m in (2, 3):
            groups = Groups.from_tensor(g, n, cuda_device, m)
            for k in (1, 5, 40, n):
                got = [t.cpu() for t in didx.search_exhaustive(q16, k, groups=groups)]
                _check_rows(got, full, groups.ids.cpu(), m, k)


@pytest.mark.gpu
def test_exact_with_every_subset_form(cuda_device):
    docs = make_docs(120, 1, 30, seed=416)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    n, B = didx.num_documents, 4
    fp = _fastplaid(didx)
    q = make_queries(B, 32, seed=417, docs=docs)
    full = [t.cpu() for t in didx.search_exhaustive(q.half().to(cuda_device), n)]
    g = torch.tensor([random.Random(418).randint(0, 12) for _ in range(n)])
    inv = torch.unique(g, return_inverse=True)[1]
    for form, members in _subset_forms(n, B, random.Random(419)):
        for m in (2, 5):
            for k in (1, 10, 40):
                res = fp.search_exhaustive(q.to(cuda_device), top_k=k, subset=form, group_by=g.to(cuda_device),
                                           max_per_group=m)
                _check_rows(_as_rows(res, k), full, inv, m, k, members=members)


@pytest.mark.gpu
def test_results_do_not_depend_on_the_split(cuda_device, monkeypatch):
    oidx, _, _ = _index_with_empty_and_long_docs(128, 4)
    didx = _device_index(oidx, cuda_device)
    n = didx.num_documents
    q16 = make_queries(9, 32, seed=420).half().to(cuda_device)
    for m in (2, 7):
        groups = Groups.from_tensor(torch.arange(n) // 9, n, cuda_device, m)
        ref = [t.cpu() for t in didx.search_exhaustive(q16, 10, groups=groups)]
        small = didx.exhaustive_workspace_bytes(2, 32, 10)
        got = [t.cpu() for t in didx.search_exhaustive(q16, 10, budget_bytes=small, groups=groups)]
        assert all(torch.equal(a, b) for a, b in zip(ref, got))
        rows = torch.randint(-1, n, (9, 40), generator=torch.Generator().manual_seed(m)).to(cuda_device)
        ref_rows = [t.cpu() for t in didx.search_exhaustive(q16, 10, subset=rows, groups=groups)]
        for dpc in ("1", "32"):
            monkeypatch.setenv("FPB_K7_DOCS_PER_CHUNK", dpc)
            got = [t.cpu() for t in didx.search_exhaustive(q16, 10, groups=groups)]
            assert all(torch.equal(a, b) for a, b in zip(ref, got)), (m, dpc)
            got = [t.cpu() for t in didx.search_exhaustive(q16, 10, subset=rows, groups=groups)]
            assert all(torch.equal(a, b) for a, b in zip(ref_rows, got)), (m, dpc)
        monkeypatch.delenv("FPB_K7_DOCS_PER_CHUNK")


@pytest.mark.gpu
def test_workspace_grows_for_the_rounds(cuda_device):
    docs = make_docs(50, 1, 10, seed=421)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    n = didx.num_documents
    sizes = []
    for m in (1, 64):
        with didx._grouped(Groups.from_tensor(torch.arange(n), n, cuda_device, m)):
            sizes.append(didx.exhaustive_workspace_bytes(4, 32, 10))
    assert sizes[1] >= sizes[0] + 4 * 63 * n * 8


@pytest.mark.gpu
def test_approximate_is_the_rule_applied_to_the_rerank_list(cuda_device):
    """search(top_k=k, group_by=g, max_per_group=m, n_full_scores=n) == rule(search(top_k=max(n // 4, 1)))[:k] for
    n 4 .. 16384, n_ivf_probe 8 and 64, device and host (fp32 CPU) queries and a shared subset."""
    docs = make_docs(400, 4, 40, seed=422)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    n_docs, B = didx.num_documents, 3
    fp = _fastplaid(didx)
    q = make_queries(B, 32, seed=423, docs=docs)
    g = torch.arange(n_docs) // 5
    shared = sorted(random.Random(424).sample(range(n_docs), n_docs // 2))
    forms = [None, shared, torch.tensor(shared)]
    for n_full in (4, 40, 1000, 16384):
        R = max(n_full // 4, 1)
        for probe in (8, 64):
            for form in forms:
                for queries in (q.to(cuda_device), q) if form is None else (q.to(cuda_device),):
                    base = fp.search(queries, top_k=R, n_full_scores=n_full, n_ivf_probe=probe, subset=form)
                    for m in (2, 3):
                        for k in (1, 10):
                            got = fp.search(queries, top_k=k, n_full_scores=n_full, n_ivf_probe=probe, subset=form,
                                            group_by=g, max_per_group=m)
                            assert got == [_limit(row, g, m, k) for row in base], (n_full, probe, m, k, type(form))


@pytest.mark.gpu
def test_token_scores_follow_the_grouped_results(cuda_device):
    docs = make_docs(200, 4, 30, seed=425)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    fp = _fastplaid(didx)
    q = make_queries(2, 32, seed=426, docs=docs).to(cuda_device)
    g = torch.arange(didx.num_documents) // 4
    grouped = fp.search(q, top_k=8, group_by=g, max_per_group=2)
    full = fp.search_token_scores(q, top_k=8, group_by=g, max_per_group=2)
    assert [[(d, s) for d, s, _ in r] for r in full] == grouped
    plain = {(b, d): mat for b, r in enumerate(fp.search_token_scores(q, top_k=1000)) for d, _, mat in r}
    for b, r in enumerate(full):
        for d, _, mat in r:
            assert torch.equal(mat, plain[(b, d)])


@pytest.mark.gpu
def test_limited_handles_are_refused_by_the_sharded_entry_points(cuda_device):
    docs = make_docs(20, 2, 10, seed=427)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    lib = engine.load_library()
    gids = torch.zeros(didx.num_documents, dtype=torch.int32, device=cuda_device)
    h = ctypes.c_void_p()
    assert lib.fpb_index_with_groups_max(ctypes.byref(h), didx._handle, gids.data_ptr(), 1, 3) == engine.FPB_OK
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


def test_the_host_rule():
    groups = [0, 0, 1, 0, 1, 2]
    assert _limit(list(range(6)), groups, 1, 10) == [0, 2, 5]
    assert _limit(list(range(6)), groups, 2, 10) == [0, 1, 2, 4, 5]
    assert _limit(list(range(6)), groups, 2, 3) == [0, 1, 2]
    assert _limit([(d, 1.0) for d in range(6)], groups, 3, 10) == [(d, 1.0) for d in range(6)]


def test_max_per_group_is_checked_before_any_index_load():
    from fast_plaid_b200.search import fast_plaid as fpmod

    fp = object.__new__(fpmod.FastPlaid)  # no index: a check that comes later would fail differently
    q = torch.zeros((1, 4, 128))
    g = torch.zeros(4, dtype=torch.int64)
    for m in (0, -1, 65, True, 2.0, "2", np.int64(2), None):
        for call in (fp.search, fp.search_exhaustive, fp.search_token_scores):
            with pytest.raises(ValueError, match="max_per_group"):
                call(q, group_by=g, max_per_group=m)
    for call in (fp.search, fp.search_exhaustive, fp.search_token_scores):
        with pytest.raises(ValueError, match="group_by"):
            call(q, max_per_group=2)
    Groups.check_max_per_group(1, None)
    Groups.check_max_per_group(64, g)
    fp.shard = (0, 2)
    fp._comm = None
    for call in (fp.search, fp.search_exhaustive):
        with pytest.raises(NotImplementedError):
            call(q, group_by=g, max_per_group=2)
    assert fp._comm is None


def test_with_groups_max_refuses_bad_arguments():
    lib = engine.load_library()
    fake = torch.zeros(64, dtype=torch.uint8)  # never dereferenced: the checks come first
    gids = torch.zeros(4, dtype=torch.int32)
    h = ctypes.c_void_p()
    assert lib.fpb_index_with_groups_max(None, fake.data_ptr(), gids.data_ptr(), 1, 2) == engine.FPB_ERR_INVALID
    assert lib.fpb_index_with_groups_max(ctypes.byref(h), None, gids.data_ptr(), 1, 2) == engine.FPB_ERR_INVALID
    assert lib.fpb_index_with_groups_max(ctypes.byref(h), fake.data_ptr(), None, 1, 2) == engine.FPB_ERR_INVALID
    for n_groups in (0, -1, 2**31):
        assert lib.fpb_index_with_groups_max(ctypes.byref(h), fake.data_ptr(), gids.data_ptr(), n_groups, 2) \
            == engine.FPB_ERR_INVALID
        assert b"n_groups" in lib.fpb_last_error()
    for m in (0, -1, 65, 2**31 - 1):
        assert lib.fpb_index_with_groups_max(ctypes.byref(h), fake.data_ptr(), gids.data_ptr(), 1, m) \
            == engine.FPB_ERR_INVALID
        assert b"max_per_group" in lib.fpb_last_error()
    assert h.value is None
