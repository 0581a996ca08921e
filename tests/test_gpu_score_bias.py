"""Biased scores (`score_bias=`, fpb_index_with_bias): document d is ranked and returned with s'_d = fp32(s_d + b_d).

- Exact search equals the unbiased `exhaustive_scores` plus the bias added in numpy float32, sorted by (score desc,
  id asc), restricted to the subset, with the group rule applied to that biased ranking.
- `search` equals the unbiased search with top_k = n_full_scores // 4, its scores biased on the host, re-sorted,
  grouped, cut to top_k.
GPU tests are marked; the argument checks at the end run without a GPU."""

from __future__ import annotations

import ctypes
import os
import random

import numpy as np
import pytest
import torch
from test_gpu_exhaustive import _device_index, _index_with_empty_and_long_docs
from test_gpu_exhaustive_sharded import _spawn
from test_gpu_groups import _subset_forms
from util import build_oracle_index, make_docs, make_queries, to_index_tensors

from fast_plaid_b200 import engine
from fast_plaid_b200.engine import FPB_FLAG_APPROX_TWO_PASS, DeviceIndex, Groups, ScoreBias

CODECS = [(128, 4), (128, 2), (64, 4), (64, 2), (128, 1)]
FLT_MAX = float(np.finfo(np.float32).max)


def _biased(scores, bias) -> np.ndarray:
    """fp32(s + b): one IEEE fp32 addition, rounded to nearest."""
    return np.asarray(scores, dtype=np.float32) + np.asarray(bias, dtype=np.float32)


def _rule(ranked: list[int], groups, m: int, k: int) -> list[int]:
    """The group rule over a ranking: a document is kept when fewer than m of its group were kept before it."""
    out, kept = [], {}
    for d in ranked:
        g = None if groups is None else int(groups[d])
        if g is not None:
            if kept.get(g, 0) >= m:
                continue
            kept[g] = kept.get(g, 0) + 1
        out.append(d)
        if len(out) == k:
            break
    return out


def _canonical(ids: np.ndarray, s: np.ndarray) -> list[int]:
    """ids by (s desc, id asc); s holds fp32 values (ties stay ties, -0.0 equals 0.0)."""
    if ids.size == 0:
        return []
    return ids[np.lexsort((ids, -s.astype(np.float64)))].tolist()


def _check_exact(ids, sc, counts, every, bias, k, members=None, groups=None, m=1) -> None:
    """Row b is the biased canonical ranking of row b of `every` (restricted to members[b]), under the group rule."""
    for b in range(ids.shape[0]):
        row = _biased(every[b].numpy(), bias)
        cand = np.arange(row.shape[0]) if members is None else np.asarray(sorted(set(members[b])), dtype=np.int64)
        exp = _rule(_canonical(cand, row[cand]), groups, m, k)
        n = len(exp)
        assert int(counts[b]) == n, f"query {b} k={k}: count {int(counts[b])}, expected {n}"
        assert ids[b, :n].tolist() == exp, f"query {b} k={k}: not the biased canonical ranking"
        got = sc[b, :n].numpy()
        assert got.tobytes() == row[exp].tobytes(), f"query {b} k={k}: a score is not fp32(s + b)"
        assert torch.all(ids[b, n:] == -1) and torch.all(sc[b, n:] == float("-inf"))


def _rerank(base, bias, k, groups=None, m=1):
    """The approximate contract on FastPlaid results: each row of the unbiased search at top_k = n_full_scores // 4,
    its scores biased, re-sorted by (score desc, id asc), the group rule, cut to k."""
    out = []
    for row in base:
        d = np.asarray([x for x, _ in row], dtype=np.int64)
        s = _biased(np.asarray([y for _, y in row], dtype=np.float32), np.asarray(bias, dtype=np.float32)[d])
        by = dict(zip(d.tolist(), s.tolist()))
        out.append([(x, by[x]) for x in _rule(_canonical(d, s), groups, m, k)])
    return out


def _rows_to_lists(ids, sc, counts):
    return [[(int(ids[b, i]), float(sc[b, i])) for i in range(int(counts[b]))] for b in range(ids.shape[0])]


def _fastplaid(didx, **kw):
    from fast_plaid_b200.search.fast_plaid import FastPlaid

    return FastPlaid.from_device_index(didx, **kw)


def _random_bias(n: int, seed: int, scale: float = 4.0) -> torch.Tensor:
    return (torch.rand(n, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) - 0.5) * scale


# ---- exhaustive search ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dim,nbits", CODECS)
def test_exact_is_the_biased_canonical_ranking(dim, nbits, cuda_device):
    """Every codec, on a ragged index with an empty document and 2000-token documents: the biased score table of
    fpb_exhaustive_scores, and the top k of the full scan for k 1, 10 and 4096, with and without groups."""
    oidx, _, _ = _index_with_empty_and_long_docs(dim, nbits)
    didx = _device_index(oidx, cuda_device, ivf=False)
    n = didx.num_documents
    q16 = make_queries(4, 32, dim=dim, seed=700 + dim + nbits).half().to(cuda_device)
    every = didx.exhaustive_scores(q16).cpu()
    b64 = _random_bias(n, 701)
    bias = ScoreBias.from_tensor(b64, n, cuda_device)
    b32 = b64.to(torch.float32).numpy()
    with didx._biased(bias):
        table = didx.exhaustive_scores(q16).cpu()
    assert table.numpy().tobytes() == _biased(every.numpy(), b32).tobytes()
    for k in (1, 10, 4096):
        ids, sc, counts = (t.cpu() for t in didx.search_exhaustive(q16, k, bias=bias))
        _check_exact(ids, sc, counts, every, b32, k)
    g = torch.arange(n) // 4
    for m in (1, 3):
        groups = Groups.from_tensor(g, n, cuda_device, m)
        ids, sc, counts = (t.cpu() for t in didx.search_exhaustive(q16, 10, groups=groups, bias=bias))
        _check_exact(ids, sc, counts, every, b32, 10, groups=g, m=m)


@pytest.mark.gpu
def test_exact_with_every_subset_form_and_groups(cuda_device):
    """FastPlaid.search_exhaustive: the id list, list of lists, [L], [B, L] padded with -1, [N] and [B, N] masks,
    each without groups and with group_by at m = 1 and m = 3; the bias on the CPU and on the GPU, fp64 and fp16."""
    docs = make_docs(150, 1, 30, seed=702)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    n, B = didx.num_documents, 4
    fp = _fastplaid(didx)
    q = make_queries(B, 32, seed=703, docs=docs)
    every = didx.exhaustive_scores(q.half().to(cuda_device)).cpu()
    g = torch.tensor([random.Random(704).randint(0, 30) for _ in range(n)])
    forms = [(None, None)] + _subset_forms(n, B, random.Random(705))
    for bias in (_random_bias(n, 706), _random_bias(n, 707).half().to(cuda_device)):
        b32 = bias.cpu().to(torch.float32).numpy()
        for form, members in forms:
            for kw, groups, m in ((dict(), None, 1), (dict(group_by=g), g, 1), (dict(group_by=g, max_per_group=3), g, 3)):
                for k in (1, 10, 40):
                    res = fp.search_exhaustive(q.to(cuda_device), top_k=k, subset=form, score_bias=bias, **kw)
                    ids = torch.full((B, k), -1, dtype=torch.int64)
                    sc = torch.full((B, k), float("-inf"), dtype=torch.float32)
                    counts = torch.tensor([len(r) for r in res], dtype=torch.int32)
                    for b, r in enumerate(res):
                        for i, (d, s) in enumerate(r):
                            ids[b, i], sc[b, i] = d, s
                    _check_exact(ids, sc, counts, every, b32, k, members=members, groups=groups, m=m)


@pytest.mark.gpu
def test_exact_adversarial_biases(cuda_device):
    """Exact fp32 ties made by the bias, +-1e30 (the order follows the bias, then the id), FLT_MAX on several
    documents, an empty document lifted to the top, and an all-zero bias (the unbiased ids and score values)."""
    oidx, empty_at, _ = _index_with_empty_and_long_docs(128, 4)
    didx = _device_index(oidx, cuda_device, ivf=False)
    n = didx.num_documents
    q16 = make_queries(3, 32, seed=708).half().to(cuda_device)
    every = didx.exhaustive_scores(q16).cpu()
    rng = random.Random(709)
    signs = torch.tensor([rng.choice((-1.0, 1.0)) for _ in range(n)], dtype=torch.float64)
    flt_max = torch.zeros(n, dtype=torch.float64)
    flt_max[[3, 9, 40, 41]] = FLT_MAX
    lift = torch.zeros(n, dtype=torch.float64)
    lift[empty_at] = 1e6
    cases = {
        "ties": torch.full((n,), float(1 << 24), dtype=torch.float64),  # the sums land on multiples of 2: ties
        "1e30": signs * 1e30,
        "flt_max": flt_max,
        "lift_empty": lift,
        "zero": torch.zeros(n, dtype=torch.float64),
    }
    for name, bvals in cases.items():
        bias = ScoreBias.from_tensor(bvals, n, cuda_device)
        b32 = bvals.to(torch.float32).numpy()
        for k in (1, 10, n):
            ids, sc, counts = (t.cpu() for t in didx.search_exhaustive(q16, k, bias=bias))
            _check_exact(ids, sc, counts, every, b32, k)
            if name == "1e30":
                up = [d for d in range(n) if signs[d] > 0]
                assert ids[0, : min(k, len(up))].tolist() == up[:k]  # ties at 1e30 fall back to the id
            if name == "flt_max" and k >= 4:
                assert ids[:, :4].tolist() == [[3, 9, 40, 41]] * 3 and torch.all(sc[:, :4] == FLT_MAX)
            if name == "lift_empty":
                assert torch.all(ids[:, 0] == empty_at)
                assert torch.all(sc[:, 0] == np.float32(32 * -10000.0) + np.float32(1e6))
            if name == "zero":
                plain = [t.cpu() for t in didx.search_exhaustive(q16, k)]
                assert torch.equal(ids, plain[0]) and torch.equal(counts, plain[2])
                assert torch.all(sc == plain[1])
        if name == "ties":
            ids, _, _ = (t.cpu() for t in didx.search_exhaustive(q16, n, bias=bias))
            s = _biased(every.numpy(), b32)
            assert any(len(set(r.tolist())) < n for r in s), "the bias made no tie"


@pytest.mark.gpu
def test_exact_does_not_depend_on_the_split(cuda_device, monkeypatch):
    oidx, _, _ = _index_with_empty_and_long_docs(128, 4)
    didx = _device_index(oidx, cuda_device)
    n = didx.num_documents
    q16 = make_queries(9, 32, seed=710).half().to(cuda_device)
    bias = ScoreBias.from_tensor(_random_bias(n, 711), n, cuda_device)
    ref = [t.cpu() for t in didx.search_exhaustive(q16, 10, bias=bias)]
    small = didx.exhaustive_workspace_bytes(2, 32, 10)
    got = [t.cpu() for t in didx.search_exhaustive(q16, 10, budget_bytes=small, bias=bias)]
    assert all(torch.equal(a, b) for a, b in zip(ref, got))
    for dpc in ("1", "32"):
        monkeypatch.setenv("FPB_K7_DOCS_PER_CHUNK", dpc)
        got = [t.cpu() for t in didx.search_exhaustive(q16, 10, bias=bias)]
        assert all(torch.equal(a, b) for a, b in zip(ref, got)), dpc


@pytest.mark.gpu
def test_derived_handles_compose_in_either_order(cuda_device):
    oidx, _, _ = _index_with_empty_and_long_docs(128, 4)
    didx = _device_index(oidx, cuda_device)
    n = didx.num_documents
    q16 = make_queries(3, 32, seed=712).half().to(cuda_device)
    bias = ScoreBias.from_tensor(_random_bias(n, 713), n, cuda_device)
    groups = Groups.from_tensor(torch.arange(n) // 3, n, cuda_device, 2)
    with didx._grouped(groups), didx._biased(bias):
        a = [t.cpu() for t in didx.search_exhaustive(q16, 10)]
    with didx._biased(bias), didx._grouped(groups):
        b = [t.cpu() for t in didx.search_exhaustive(q16, 10)]
    c = [t.cpu() for t in didx.search_exhaustive(q16, 10, groups=groups, bias=bias)]
    assert all(torch.equal(x, y) and torch.equal(x, z) for x, y, z in zip(a, b, c))
    every = didx.exhaustive_scores(q16).cpu()
    _check_exact(*a, every, bias.values.cpu().numpy(), 10, groups=torch.arange(n) // 3, m=2)


# ---- approximate search --------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("Q", [32, 64, 100, 256])
def test_search_is_the_biased_rerank_list(Q, cuda_device):
    """Q = 32 runs K5 v4, 64 and 100 v5, 256 the generic kernel (dim 128, nbits 4): every subset form, device and
    host fp32 queries, with and without groups, n_full_scores 40 and 1000."""
    docs = make_docs(400, 4, 40, seed=714)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    n, B = didx.num_documents, 3
    fp = _fastplaid(didx)
    q = make_queries(B, Q, seed=715 + Q, docs=docs)
    g = torch.arange(n) // 5
    bias = _random_bias(n, 716, scale=8.0)
    forms = [(None, None)] + _subset_forms(n, B, random.Random(717))
    for n_full in (40, 1000):
        R = n_full // 4
        for form, _ in forms:
            for queries in (q.to(cuda_device), q) if form is None else (q.to(cuda_device),):
                base = fp.search(queries, top_k=R, n_full_scores=n_full, subset=form)
                for k in (1, 10):
                    got = fp.search(queries, top_k=k, n_full_scores=n_full, subset=form, score_bias=bias)
                    assert got == _rerank(base, bias, k), (n_full, k, type(form))
                    got = fp.search(queries, top_k=k, n_full_scores=n_full, subset=form, score_bias=bias,
                                    group_by=g, max_per_group=2)
                    assert got == _rerank(base, bias, k, g, 2), (n_full, k, type(form), "grouped")


@pytest.mark.gpu
@pytest.mark.parametrize("dim,nbits,k5", [(128, 4, "v1"), (128, 2, None), (64, 4, None), (64, 2, None), (128, 1, None)])
def test_search_generic_kernel_and_other_codecs(dim, nbits, k5, cuda_device, monkeypatch):
    if k5:
        monkeypatch.setenv("FPB_K5", k5)
    docs = make_docs(300, 4, 40, dim=dim, seed=718)
    oidx, _ = build_oracle_index(docs, nbits=nbits)
    didx = _device_index(oidx, cuda_device)
    fp = _fastplaid(didx)
    q = make_queries(3, 32, dim=dim, seed=719, docs=docs)
    bias = _random_bias(didx.num_documents, 720, scale=8.0)
    base = fp.search(q.to(cuda_device), top_k=64, n_full_scores=256)
    for k in (1, 10, 64):
        assert fp.search(q.to(cuda_device), top_k=k, n_full_scores=256, score_bias=bias) == _rerank(base, bias, k)
    # the token matrices stay the raw similarities; the scores and the order are the biased ones
    full = fp.search_token_scores(q.to(cuda_device), top_k=10, n_full_scores=256, score_bias=bias)
    assert [[(d, s) for d, s, _ in r] for r in full] == _rerank(base, bias, 10)
    plain = {(b, d): m for b, r in enumerate(fp.search_token_scores(q.to(cuda_device), top_k=64, n_full_scores=256))
             for d, _, m in r}
    for b, r in enumerate(full):
        for d, _, m in r:
            assert torch.equal(m, plain[(b, d)])


@pytest.mark.gpu
def test_search_in_both_approximate_modes(cuda_device):
    """The one-pass and the two-pass candidate stages, through DeviceIndex.search and search_host."""
    docs = make_docs(500, 4, 40, seed=721)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    n = didx.num_documents
    q = make_queries(4, 32, seed=722, docs=docs)
    q16 = q.half().to(cuda_device)
    b64 = _random_bias(n, 723, scale=8.0)
    bias = ScoreBias.from_tensor(b64, n, cuda_device)
    for flags in (0, FPB_FLAG_APPROX_TWO_PASS):
        base_p = DeviceIndex.with_flags(DeviceIndex.make_params(128, 512, 16), flags)
        p = DeviceIndex.with_flags(DeviceIndex.make_params(10, 512, 16), flags)
        base = _rows_to_lists(*(t.cpu() for t in didx.search(q16, base_p)))
        exp = _rerank(base, b64, 10)
        assert _rows_to_lists(*(t.cpu() for t in didx.search(q16, p, bias=bias))) == exp, flags
        assert _rows_to_lists(*(t.cpu() for t in didx.search_host(q, p, bias=bias))) == exp, flags


@pytest.mark.gpu
def test_search_adversarial_biases(cuda_device):
    docs = make_docs(300, 4, 40, seed=724)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    n = didx.num_documents
    fp = _fastplaid(didx)
    q = make_queries(3, 32, seed=725, docs=docs).to(cuda_device)
    base = fp.search(q, top_k=256, n_full_scores=1024)
    rng = random.Random(726)
    flt_max = torch.zeros(n, dtype=torch.float64)
    flt_max[[1, 2, 50]] = FLT_MAX
    for bvals in (torch.full((n,), float(1 << 24), dtype=torch.float64),
                  torch.tensor([rng.choice((-1e30, 1e30)) for _ in range(n)], dtype=torch.float64),
                  flt_max, torch.zeros(n, dtype=torch.float64)):
        for k in (1, 10, 256):
            assert fp.search(q, top_k=k, n_full_scores=1024, score_bias=bvals) == _rerank(base, bvals, k)
    assert fp.search(q, top_k=10, n_full_scores=1024, score_bias=torch.zeros(n)) == [r[:10] for r in base]


# ---- shards and growth -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_one_rank_shard_equals_unsharded(cuda_device):
    """FastPlaid(shard=(0, 1)): search (device and host queries, a subset), search_exhaustive and search_token_scores,
    with and without group_by, give the unsharded biased bytes."""
    docs = make_docs(500, 4, 40, seed=727)
    oidx, _ = build_oracle_index(docs)
    didx = DeviceIndex(to_index_tensors(oidx), cuda_device)
    q = make_queries(5, 32, seed=728, docs=docs)
    fp = _fastplaid(didx, shard=(0, 1))
    plain = _fastplaid(didx)
    n = didx.num_documents
    bias = _random_bias(n, 729, scale=8.0)
    g = torch.arange(n) * 7 // 40
    sub = sorted(random.Random(730).sample(range(n), 200))
    for kw in (dict(), dict(group_by=g), dict(group_by=g, max_per_group=3)):
        for queries in (q, q.to(cuda_device)):
            assert fp.search(queries, top_k=10, n_full_scores=512, score_bias=bias, **kw) \
                == plain.search(queries, top_k=10, n_full_scores=512, score_bias=bias, **kw)
        assert fp.search(q.to(cuda_device), top_k=10, n_full_scores=512, subset=sub, score_bias=bias, **kw) \
            == plain.search(q.to(cuda_device), top_k=10, n_full_scores=512, subset=sub, score_bias=bias, **kw)
        assert fp.search_exhaustive(q, top_k=20, score_bias=bias, **kw) \
            == plain.search_exhaustive(q, top_k=20, score_bias=bias, **kw)
    a = fp.search_token_scores(q, top_k=5, n_full_scores=512, score_bias=bias)
    b = plain.search_token_scores(q, top_k=5, n_full_scores=512, score_bias=bias)
    assert [[(d, s) for d, s, _ in r] for r in a] == [[(d, s) for d, s, _ in r] for r in b]
    assert all(torch.equal(x[2], y[2]) for ra, rb in zip(a, b) for x, y in zip(ra, rb))
    fp.close()  # the communicator and the index go now, not whenever the collector finds them


@pytest.mark.gpu
def test_a_bias_of_the_old_length_is_refused_after_update_and_delete(cuda_device):
    docs = make_docs(50, 2, 20, seed=731)
    oidx, _ = build_oracle_index(docs, nbits=4)
    didx = _device_index(oidx, cuda_device)
    n = didx.num_documents
    old = ScoreBias.from_tensor(torch.zeros(n), n, cuda_device)
    q16 = make_queries(1, 32, seed=732).half().to(cuda_device)
    o0, o1 = int(didx.doc_offsets[0]), int(didx.doc_offsets[1])
    grown = didx.append(didx.doc_codes[o0:o1].cpu(), didx.doc_residuals[o0:o1].cpu(), torch.tensor([o1 - o0]))
    smaller = didx.delete([3])
    lib = engine.load_library()
    for idx in (grown, smaller):
        with pytest.raises(ValueError):
            idx.search_exhaustive(q16, 5, bias=old)
        with pytest.raises(ValueError):
            ScoreBias.check(torch.zeros(n), idx.num_documents)
        h = ctypes.c_void_p()
        assert lib.fpb_index_with_bias(ctypes.byref(h), idx._handle, old.values.data_ptr(), n) \
            == engine.FPB_ERR_INVALID
        assert h.value is None
        m = idx.num_documents
        lift = torch.zeros(m)
        lift[m - 1] = 1e6
        ok = ScoreBias.from_tensor(lift, m, cuda_device)
        ids, _, counts = idx.search_exhaustive(q16, 5, bias=ok)
        assert int(counts[0]) == 5 and int(ids[0, 0]) == m - 1


def _nccl_worker(rank: int, world: int, port: int, out):
    import sys

    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import torch.distributed as dist
    from util import build_oracle_index, make_docs, make_queries, to_index_tensors

    from fast_plaid_b200.engine import DeviceIndex, shard_grid, shard_tensors
    from fast_plaid_b200.search.fast_plaid import FastPlaid

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    torch.set_num_threads(4)
    dev = f"cuda:{rank}"
    docs = make_docs(700, 10, 60, seed=733)
    oidx, _ = build_oracle_index(docs)
    t = to_index_tensors(oidx)
    queries = make_queries(5, 32, seed=734, docs=docs)
    bias = (torch.rand(700, generator=torch.Generator().manual_seed(735)) - 0.5) * 8.0
    g = torch.arange(700, dtype=torch.int64) * 7 // 50
    plain = FastPlaid.from_device_index(DeviceIndex(t, dev))
    failed = []
    for kw in (dict(score_bias=bias), dict(score_bias=bias, group_by=g, max_per_group=2)):
        ref_s = plain.search(queries, top_k=10, n_full_scores=512, **kw)
        ref_e = plain.search_exhaustive(queries, top_k=20, **kw)
        for n_groups in [q for q in (1, 2, 4) if world % q == 0]:
            _, d_shard, n_shards = shard_grid(rank, world, n_groups)
            sh, base = shard_tensors(t, d_shard, n_shards)
            fp = FastPlaid.from_device_index(DeviceIndex(sh, dev, doc_id_base=base), shard=(rank, world),
                                             query_groups=n_groups)
            if fp.search(queries, top_k=10, n_full_scores=512, **kw) != ref_s:
                failed.append(f"search {list(kw)} groups={n_groups}")
            if fp.search(queries.to(dev), top_k=10, n_full_scores=512, **kw) != ref_s:
                failed.append(f"search (device queries) {list(kw)} groups={n_groups}")
            if fp.search_exhaustive(queries, top_k=20, **kw) != ref_e:
                failed.append(f"search_exhaustive {list(kw)} groups={n_groups}")
            fp.close()
    flag = torch.tensor([0 if failed else 1], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        out.put((int(flag.item()), failed))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("world", [2, 4])
def test_nccl_biased_sharded_equals_unsharded(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    ok, failed = _spawn(_nccl_worker, world, 900)
    assert ok == 1, failed


@pytest.mark.gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_several_devices_in_one_process():
    from fast_plaid_b200.search.fast_plaid import FastPlaid

    docs = make_docs(300, 4, 40, seed=736)
    oidx, _ = build_oracle_index(docs)
    t = to_index_tensors(oidx)
    one = FastPlaid.from_device_index(DeviceIndex(t, "cuda:0"))
    two = FastPlaid.from_device_index(DeviceIndex(t, "cuda:0"))
    two.devices = ["cuda:0", "cuda:1"]  # replicas, the query list split across them
    two.indices["cuda:1"] = DeviceIndex(t, "cuda:1")
    q = make_queries(6, 32, seed=737, docs=docs)
    bias = _random_bias(300, 738)
    assert two.search(q, top_k=10, score_bias=bias) == one.search(q, top_k=10, score_bias=bias)
    assert two.search_exhaustive(q, top_k=10, score_bias=bias) == one.search_exhaustive(q, top_k=10, score_bias=bias)


# ---- no GPU needed ---------------------------------------------------------------------------------------------
def test_biases_are_checked():
    ScoreBias.check(torch.tensor([0.0, -1.5, FLT_MAX]), 3)
    ScoreBias.check(torch.tensor([0.0, 1.0, 2.0], dtype=torch.float16), 3)
    ScoreBias.check(torch.tensor([0.0, 1.0, 2.0], dtype=torch.bfloat16), None)
    bad = [
        [0.0, 1.0, 2.0],  # not a tensor
        np.zeros(3, dtype=np.float32),
        torch.tensor([0, 1, 2]),
        torch.tensor([True, False, True]),
        torch.zeros(3, dtype=torch.complex64),
        torch.zeros((3, 1)),
        torch.zeros(()),
        torch.zeros(2),  # wrong length
        torch.tensor([0.0, float("nan"), 1.0]),
        torch.tensor([0.0, float("inf"), 1.0]),
        torch.tensor([0.0, float("-inf"), 1.0]),
        torch.tensor([0.0, 1e39, 1.0], dtype=torch.float64),  # infinite in fp32
    ]
    for b in bad:
        with pytest.raises(ValueError):
            ScoreBias.check(b, 3)
    with pytest.raises(ValueError):
        ScoreBias.for_shard(torch.zeros(5), 3, 3, "cpu")  # does not cover the shard
    with pytest.raises(ValueError):
        ScoreBias.for_shard(torch.tensor([0.0] * 5 + [float("nan")]), 0, 3, "cpu")  # checked whole, on every rank
    assert torch.equal(ScoreBias.for_shard(torch.arange(6, dtype=torch.float64), 2, 3, "cpu").values,
                       torch.tensor([2.0, 3.0, 4.0]))


def test_with_bias_refuses_bad_arguments():
    lib = engine.load_library()
    fake = torch.zeros(4096, dtype=torch.uint8)  # a handle of 0 documents, never dereferenced past its fields
    vals = torch.zeros(4, dtype=torch.float32)
    h = ctypes.c_void_p()
    assert lib.fpb_index_with_bias(None, fake.data_ptr(), vals.data_ptr(), 0) == engine.FPB_ERR_INVALID
    assert lib.fpb_index_with_bias(ctypes.byref(h), None, vals.data_ptr(), 0) == engine.FPB_ERR_INVALID
    assert lib.fpb_index_with_bias(ctypes.byref(h), fake.data_ptr(), None, 0) == engine.FPB_ERR_INVALID
    for n in (1, 4, -1):
        assert lib.fpb_index_with_bias(ctypes.byref(h), fake.data_ptr(), vals.data_ptr(), n) == engine.FPB_ERR_INVALID
        assert b"entries" in lib.fpb_last_error()
    assert h.value is None


def test_fastplaid_refuses_a_bad_bias_before_any_exchange():
    from fast_plaid_b200.search import fast_plaid as fpmod

    fp = object.__new__(fpmod.FastPlaid)
    fp.shard = (0, 2)
    fp._comm = None
    q = torch.zeros((1, 4, 128))
    for call in (fp.search, fp.search_exhaustive, fp.search_token_scores):
        with pytest.raises(ValueError):
            call(q, score_bias=torch.tensor([0.0, float("nan")]))
        with pytest.raises(ValueError):
            call(q, score_bias=torch.zeros(2, dtype=torch.int64))
        with pytest.raises(NotImplementedError):  # several ranks need a process group
            call(q, score_bias=torch.zeros(2))
    assert fp._comm is None
