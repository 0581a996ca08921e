"""Grouped results on document-sharded indexes (`group_by=` / `max_per_group=` with `shard=`,
fpb_index_with_shard_groups and fpb_merge_shards_grouped): the bytes the same call returns on one GPU holding the
whole index with the same group map, at every shard count.

- Exact search: each shard's top_k under the rule (its local map), merged and ruled again with the whole index's map.
- Approximate search: the ungrouped shard steps, then the grouped merge of the R globally kept records.
The unmarked tests run without a GPU: the argument behind the exact merge (as a property test in plain Python), the
C-ABI refusals and the refusals of the Python surface.  The NCCL tests need 2 or 4 GPUs and are skipped below that."""

from __future__ import annotations

import ctypes
import os
import random

import pytest
import torch
from test_gpu_exhaustive_sharded import _shards, _spawn
from test_gpu_group_limit import _admissible, _group_maps, _limit
from test_gpu_groups import _subset_forms
from util import build_oracle_index, make_docs, make_queries, to_index_tensors

from fast_plaid_b200 import engine
from fast_plaid_b200.engine import DeviceIndex, Groups

CODECS = [(128, 4), (128, 2), (64, 4), (64, 2), (128, 1)]
LIMITS = (1, 2, 3, 7, 64)
MERGE_MAX = 16384


def _equal(a, b) -> bool:
    return all(torch.equal(x.cpu(), y.cpu()) for x, y in zip(a, b))


def _maps(n: int, world: int) -> dict[str, torch.Tensor]:
    """The maps of the single-GPU tests, plus runs that straddle every shard boundary and groups spread over every
    shard (document d in group d % 7)."""
    out = _group_maps(n)
    out["straddle"] = (torch.arange(n, dtype=torch.int64) + n // (2 * world)) // max(n // world, 1)
    out["spread"] = torch.arange(n, dtype=torch.int64) % 7
    return out


def _for_shards(parts, g: torch.Tensor, m: int) -> list[Groups]:
    return [Groups.for_shard(g, p.doc_id_base, p.num_documents, p.device, m) for p in parts]


def _exact_stepwise(parts, q16, k: int, groups: list[Groups]):
    recs = torch.stack([p.shard_exhaustive_records(q16, k, g) for p, g in zip(parts, groups)])
    return parts[0].merge_records(recs, k, groups[0], n_keep=len(parts) * k)


# ---- CPU: the argument behind the exact merge -------------------------------------------------------------------------
def _ranking(items):
    """(id, score) pairs in the canonical order: score desc, then id asc."""
    return sorted(items, key=lambda e: (-e[1], e[0]))


def test_per_shard_top_k_under_the_rule_merges_to_the_global_rule():
    """For random scores (with ties), maps and contiguous shard splits: the rule applied to the union of every
    shard's first top_k kept documents, cut to top_k, is the rule applied to the whole ranking, cut to top_k."""
    rng = random.Random(2024)
    for trial in range(300):
        n = rng.randint(1, 60)
        scores = [float(rng.randint(0, 12)) for _ in range(n)]  # few values: many ties
        groups = [rng.randint(0, rng.randint(0, 8)) for _ in range(n)]
        world = rng.randint(1, min(n, 6))
        cuts = sorted(rng.sample(range(1, n), world - 1)) if world > 1 else []
        bounds = list(zip([0] + cuts, cuts + [n]))
        m = LIMITS[trial % len(LIMITS)]
        admissible = sum(min(m, groups.count(g)) for g in set(groups))
        for k in range(1, admissible + 3):
            whole = _limit(_ranking([(d, scores[d]) for d in range(n)]), groups, m, k)
            union = []
            for lo, hi in bounds:
                union += _limit(_ranking([(d, scores[d]) for d in range(lo, hi)]), groups, m, k)
            assert _limit(_ranking(union), groups, m, k) == whole, (trial, m, k, bounds)


# ---- CPU: refusals ----------------------------------------------------------------------------------------------------
def test_c_abi_refusals():
    lib = engine.load_library()
    fake = torch.zeros(4096, dtype=torch.uint8)  # a zeroed host "handle" (doc_id_base 0, no documents), never launched
    gids = torch.zeros(4, dtype=torch.int32)
    h = ctypes.c_void_p()
    F, G, INV = fake.data_ptr(), gids.data_ptr(), engine.FPB_ERR_INVALID
    with_shard = lib.fpb_index_with_shard_groups
    assert with_shard(None, F, G, 1, 1, G, 4) == INV
    assert with_shard(ctypes.byref(h), None, G, 1, 1, G, 4) == INV
    assert with_shard(ctypes.byref(h), F, None, 1, 1, G, 4) == INV
    assert with_shard(ctypes.byref(h), F, G, 1, 1, None, 4) == INV
    for n_groups in (0, -1, 2**31):
        assert with_shard(ctypes.byref(h), F, G, n_groups, 1, G, 4) == INV
        assert b"n_groups" in lib.fpb_last_error()
    for m in (0, -1, 65):
        assert with_shard(ctypes.byref(h), F, G, 1, m, G, 4) == INV
        assert b"max_per_group" in lib.fpb_last_error()
    for n_total in (0, -1, 2**31):
        assert with_shard(ctypes.byref(h), F, G, 1, 1, G, n_total) == INV
        assert b"n_total_docs" in lib.fpb_last_error()
    assert h.value is None

    merge = lib.fpb_merge_shards_grouped
    rec = torch.zeros(64, dtype=torch.uint8).data_ptr()  # never dereferenced: the checks come first
    out = torch.zeros(64, dtype=torch.uint8).data_ptr()
    assert merge(None, 2, 1, 4, 4, 3, G, 4, 1, out, out, out, None) == INV
    assert merge(rec, 2, 1, 4, 4, 3, None, 4, 1, out, out, out, None) == INV
    for bad_out in ((None, out, out), (out, None, out), (out, out, None)):
        assert merge(rec, 2, 1, 4, 4, 3, G, 4, 1, *bad_out, None) == INV
    for n_total in (0, -1, 2**31):
        assert merge(rec, 2, 1, 4, 4, 3, G, n_total, 1, out, out, out, None) == INV
        assert b"n_total_docs" in lib.fpb_last_error()
    for m in (0, -1, 65):
        assert merge(rec, 2, 1, 4, 4, 3, G, 4, m, out, out, out, None) == INV
        assert b"max_per_group" in lib.fpb_last_error()
    for n_keep in (0, -1, 9):
        assert merge(rec, 2, 1, 4, n_keep, 3, G, 4, 1, out, out, out, None) == INV
        assert b"n_keep" in lib.fpb_last_error()
    for n_shards, B, R, k in ((0, 1, 4, 3), (2, 0, 4, 3), (2, 1, 0, 3), (2, 1, 4, 0)):
        assert merge(rec, n_shards, B, R, 1, k, G, 4, 1, out, out, out, None) == INV
    # the merge limit: n_shards * R <= 16384 records per query
    assert merge(rec, 5, 1, 4096, 4096, 10, G, 4, 1, out, out, out, None) == engine.FPB_ERR_UNSUPPORTED
    assert b"16384" in lib.fpb_last_error()


def test_python_refusals():
    from fast_plaid_b200.search import fast_plaid as fpmod

    # several ranks without a process group: refused before any index load or communicator
    fp = object.__new__(fpmod.FastPlaid)
    fp.shard = (1, 3)
    fp._comm = None
    q = torch.zeros((1, 4, 128))
    g = torch.zeros(9, dtype=torch.int64)
    for call in (fp.search, fp.search_exhaustive, fp.search_token_scores):
        with pytest.raises(NotImplementedError, match="process group"):
            call(q, group_by=g, max_per_group=2)
    assert fp._comm is None
    # the map must cover the whole index: a shard's slice is refused
    with pytest.raises(ValueError, match="whole index"):
        Groups.for_shard(torch.zeros(5, dtype=torch.int64), 5, 5, "cpu")
    with pytest.raises(ValueError):
        Groups.for_shard(torch.tensor([0, -1, 2, 3]), 0, 2, "cpu")
    with pytest.raises(ValueError, match="max_per_group"):
        Groups.for_shard(torch.zeros(4, dtype=torch.int64), 0, 2, "cpu", 65)


def test_device_form_of_a_sharded_map():
    g = torch.tensor([7, 7, 2**62, 3, 7, 3], dtype=torch.int64)
    s = Groups.for_shard(g, 2, 3, "cpu", 2)
    assert s.ids.tolist() == [2, 0, 1] and s.n_groups == 3 and s.max_per_group == 2
    assert s.global_ids.dtype == torch.int32 and s.global_ids.tolist() == [1, 1, 2, 0, 1, 0]


# ---- one GPU, step-wise -------------------------------------------------------------------------------------------
def _exact_sweep(t, q16, device, worlds, maps_of=_maps, limits=LIMITS) -> None:
    whole = DeviceIndex(t, device)
    N = whole.num_documents
    for world in worlds:
        parts = _shards(t, world, device)
        for name, g in maps_of(N, world).items():
            for m in limits:
                one = Groups.from_tensor(g, N, device, m)
                per = _for_shards(parts, g, m)
                for k in sorted({1, 10, _admissible(one.ids.cpu(), m) + 5, min(4096, MERGE_MAX // world)}):
                    ref = whole.search_exhaustive(q16, k, groups=one)
                    got = _exact_stepwise(parts, q16, k, per)
                    assert _equal(got, ref), f"world={world} map={name} m={m} top_k={k}"
        for p in parts:
            p.close()
    whole.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dim,nbits", CODECS)
def test_exact_stepwise_equals_the_whole_index(dim, nbits, cuda_device):
    """Every codec on 150 documents at 2, 3 and 5 shards: the shards' grouped records merged by the grouped merge
    equal the unsharded grouped search_exhaustive, for every map, m in {1, 2, 3, 7, 64} and top_k 1, 10, more than
    the admissible documents and the merge limit's largest."""
    docs = make_docs(150, 1, 40, dim=dim, seed=500 + dim + nbits)
    oidx, _ = build_oracle_index(docs, nbits=nbits)
    q16 = make_queries(3, 32, dim=dim, seed=501, docs=docs).half().to(cuda_device)
    _exact_sweep(to_index_tensors(oidx), q16, cuda_device, (2, 3, 5))


@pytest.mark.gpu
def test_exact_stepwise_on_a_larger_index(cuda_device):
    """3000 documents: wide per-shard selections and merges of up to 16384 records."""
    docs = make_docs(3000, 1, 12, seed=510)
    oidx, _ = build_oracle_index(docs, nbits=4)
    q16 = make_queries(3, 32, seed=511, docs=docs).half().to(cuda_device)
    _exact_sweep(to_index_tensors(oidx), q16, cuda_device, (2, 3, 5), limits=(1, 3, 64))


@pytest.mark.gpu
def test_exact_ties_across_shards(cuda_device):
    """Copies of a document in other shards score alike: the smaller global id ranks first, and whether the copies
    share a group or not, the merge equals the whole index."""
    docs = make_docs(60, 5, 30, seed=520)
    for src, dst in ((3, 25), (3, 47), (10, 55), (10, 30)):  # shards at world 3: [0, 20), [20, 40), [40, 60)
        docs[dst] = docs[src].clone()
    oidx, _ = build_oracle_index(docs)
    t = to_index_tensors(oidx)
    whole = DeviceIndex(t, cuda_device)
    q16 = torch.cat([make_queries(2, 32, seed=521, docs=[docs[3]]),
                     make_queries(2, 32, seed=522, docs=[docs[10]])]).half().to(cuda_device)
    parts = _shards(t, 3, cuda_device)
    copies = torch.arange(60, dtype=torch.int64)
    copies[[25, 47]] = 3
    copies[[30, 55]] = 10
    for g in (copies, torch.arange(60) % 2, torch.arange(60)):
        for m in (1, 2, 3):
            for k in (1, 3, 8, 60):
                ref = whole.search_exhaustive(q16, k, groups=Groups.from_tensor(g, 60, cuda_device, m))
                got = _exact_stepwise(parts, q16, k, _for_shards(parts, g, m))
                assert _equal(got, ref), (m, k)
    ids = whole.search_exhaustive(q16, 8, groups=Groups.from_tensor(torch.arange(60), 60, cuda_device))[0].cpu()
    for b, group in enumerate(([3, 25, 47], [3, 25, 47], [10, 30, 55], [10, 30, 55])):
        pos = [ids[b].tolist().index(d) for d in group]
        assert pos == sorted(pos), f"query {b}: the tied copies are not in id order"


def _approx_stepwise(parts, q16, params, groups: Groups, subset=None):
    Q = int(q16.shape[1])
    if subset is None:
        keys = torch.stack([p.shard_approx_keys(q16, params) for p in parts])
    else:
        from fast_plaid_b200.search import fast_plaid as fpmod

        params = DeviceIndex.with_flags(params, engine.FPB_FLAG_SUBSET)
        if isinstance(subset, torch.Tensor):
            cbs = torch.stack([p.shard_subset_begin(q16, params, filter=fpmod._SubsetTensor(subset).to_filter(
                p, q16.shape[0])) for p in parts])
        else:
            cbs = torch.stack([p.shard_subset_begin(q16, params, subset) for p in parts])
        keys = torch.stack([p.shard_subset_keys(cbs, Q, params) for p in parts])
    recs = torch.stack([p.shard_exact_records(keys, r, Q, params) for r, p in enumerate(parts)])
    return parts[0].merge_records(recs, params.top_k, groups)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3, 5])
def test_approximate_stepwise_equals_the_whole_index(world, cuda_device):
    """The ungrouped shard steps, then the grouped merge: the unsharded grouped `search`, for n_full_scores from 4 to
    the merge limit's largest at this world, n_ivf_probe 8 and 64, and m in {1, 3, 64}."""
    docs = make_docs(1200, 5, 40, seed=530 + world)
    oidx, _ = build_oracle_index(docs, nbits=4)
    t = to_index_tensors(oidx)
    whole = DeviceIndex(t, cuda_device)
    N = whole.num_documents
    parts = _shards(t, world, cuda_device)
    q16 = make_queries(4, 32, seed=531, docs=docs).half().to(cuda_device)
    maps = _maps(N, world)
    for n_full in (4, 64, 1024, 4 * min(4096, MERGE_MAX // world)):
        for probe in (8, 64):
            params = DeviceIndex.make_params(10, n_full, probe)
            for name in ("straddle", "spread", "random10", "singletons"):
                for m in (1, 3, 64):
                    g = maps[name]
                    ref = whole.search(q16, params, groups=Groups.from_tensor(g, N, cuda_device, m))
                    got = _approx_stepwise(parts, q16, params, _for_shards(parts, g, m)[0])
                    assert _equal(got, ref), f"world={world} n_full={n_full} probe={probe} map={name} m={m}"
    # every subset form through the fpb_shard_subset_* / filter steps
    rng = random.Random(world)
    params = DeviceIndex.make_params(10, 256, 16)
    g = maps["straddle"]
    for m in (1, 2):
        one = Groups.from_tensor(g, N, cuda_device, m)
        for form, lists in _subset_forms(N, 4, rng):
            ref = whole.search(q16, DeviceIndex.with_flags(params, engine.FPB_FLAG_SUBSET), subset=lists, groups=one)
            step_form = form if isinstance(form, torch.Tensor) else lists  # the list steps take one list per query
            got = _approx_stepwise(parts, q16, params, _for_shards(parts, g, m)[0], subset=step_form)
            assert _equal(got, ref), f"world={world} m={m} subset form {type(form).__name__}"
    for p in parts:
        p.close()
    whole.close()


@pytest.mark.gpu
def test_shard_grouped_handles_are_accepted_where_they_merge_only(cuda_device):
    """A shard-grouped handle is refused by the single-GPU and step-wise entry points; a plain grouped handle stays
    refused by the sharded ones; a total below the shard's range is refused."""
    docs = make_docs(20, 2, 10, seed=540)
    oidx, _ = build_oracle_index(docs, nbits=4)
    t = to_index_tensors(oidx)
    sh, base = engine.shard_tensors(t, 1, 2)
    part = DeviceIndex(sh, cuda_device, doc_id_base=base)
    lib = engine.load_library()
    gids = torch.zeros(20, dtype=torch.int32, device=cuda_device)
    h = ctypes.c_void_p()
    assert lib.fpb_index_with_shard_groups(ctypes.byref(h), part._handle, gids.data_ptr(), 1, 2, gids.data_ptr(),
                                           base + part.num_documents - 1) == engine.FPB_ERR_INVALID
    assert lib.fpb_index_with_shard_groups(ctypes.byref(h), part._handle, gids.data_ptr(), 1, 2, gids.data_ptr(),
                                           20) == engine.FPB_OK
    fake = torch.zeros(256, dtype=torch.uint8, device=cuda_device).data_ptr()
    params = DeviceIndex.make_params(10, 64, 8)
    U = engine.FPB_ERR_UNSUPPORTED
    try:
        assert lib.fpb_search_batch(h, fake, 1, 1, ctypes.byref(params), fake, 256, fake, fake, fake, None) == U
        assert lib.fpb_stage_rank(h, 1, 1, ctypes.byref(params), fake, 256, fake, fake, fake, None) == U
        assert lib.fpb_search_exhaustive(h, fake, 1, 1, 1, fake, 256, fake, fake, fake, None) == U
        assert lib.fpb_exhaustive_scores(h, fake, 1, 1, fake, 256, fake, None) == U
        assert b"shard-grouped" in lib.fpb_last_error()
        assert lib.fpb_shard_approx_keys(h, fake, 1, 1, ctypes.byref(params), fake, 256, fake, None) == U
        assert lib.fpb_stage_records(h, 1, 1, ctypes.byref(params), fake, 256, fake, None) == U
        assert lib.fpb_stage_keys(h, 1, 1, ctypes.byref(params), fake, 256, fake, None) == U
        ws = ctypes.c_size_t()
        assert lib.fpb_exhaustive_workspace_bytes(h, 2, 32, 10, ctypes.byref(ws)) == engine.FPB_OK
        plain = part.exhaustive_workspace_bytes(2, 32, 10)
        assert ws.value >= plain + 2 * 10 * 8
    finally:
        lib.fpb_index_destroy(h)
    part.close()


# ---- one GPU, one-rank communicator ----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_one_rank_fastplaid_equals_unsharded(cuda_device):
    """FastPlaid(shard=(0, 1)): search (device and host queries), search_exhaustive (one step and several) and
    search_token_scores with group_by / max_per_group give the unsharded FastPlaid's result."""
    from fast_plaid_b200.search.fast_plaid import FastPlaid

    docs = make_docs(500, 10, 60, seed=550)
    oidx, _ = build_oracle_index(docs)
    didx = DeviceIndex(to_index_tensors(oidx), cuda_device)
    queries = make_queries(5, 32, seed=551, docs=docs)
    fp = FastPlaid.from_device_index(didx, shard=(0, 1))
    plain = FastPlaid.from_device_index(didx)
    rng = random.Random(552)
    g = torch.tensor([rng.randint(0, 50) for _ in range(500)], dtype=torch.int64)
    for gb in (g, g.to(cuda_device)):
        for m in (1, 4):
            kw = dict(group_by=gb, max_per_group=m)
            for q in (queries, queries.to(cuda_device)):
                assert fp.search(q, top_k=10, n_full_scores=256, **kw) == plain.search(q, top_k=10,
                                                                                      n_full_scores=256, **kw)
            assert fp.search(queries, top_k=10, subset=list(range(0, 500, 3)), **kw) == plain.search(
                queries, top_k=10, subset=list(range(0, 500, 3)), **kw)
            for k in (10, 300):
                assert fp.search_exhaustive(queries, top_k=k, **kw) == plain.search_exhaustive(queries, top_k=k, **kw)
            tok = fp.search_token_scores(queries, top_k=5, **kw)
            ref = plain.search_token_scores(queries, top_k=5, **kw)
            assert [[(d, s) for d, s, _ in r] for r in tok] == [[(d, s) for d, s, _ in r] for r in ref]
            assert all(torch.equal(a[2], b[2]) for ra, rb in zip(tok, ref) for a, b in zip(ra, rb))
    # a budget of about two queries' grouped workspace: several collective calls, the same result
    groups = Groups.for_shard(g, 0, 500, cuda_device, 4)
    budget = didx.exhaustive_workspace_bytes(2, 32, 10) + 2 * 10 * 8
    assert didx.exhaustive_sharded_step(1, 5, 32, 10, budget, groups) < 5
    assert fp._search_exhaustive_sharded(didx, queries, 10, budget_bytes=budget, group_by=g, max_per_group=4) == \
        plain.search_exhaustive(queries, top_k=10, group_by=g, max_per_group=4)
    # the map must cover the whole index
    with pytest.raises(ValueError, match="documents"):
        fp.search(queries, top_k=10, group_by=g[:499])
    fp.close()


@pytest.mark.gpu
def test_a_shard_map_of_shard_length_is_refused(cuda_device):
    """A rank holding documents [base, base + n) of a larger index takes the map of the whole index only."""
    from fast_plaid_b200.search.fast_plaid import FastPlaid

    docs = make_docs(40, 2, 10, seed=560)
    oidx, _ = build_oracle_index(docs)
    sh, base = engine.shard_tensors(to_index_tensors(oidx), 1, 2)
    part = DeviceIndex(sh, cuda_device, doc_id_base=base)
    fp = FastPlaid.from_device_index(part, shard=(0, 1))
    q = make_queries(1, 8, seed=561, docs=docs)
    for call in (fp.search, fp.search_exhaustive):
        with pytest.raises(ValueError, match="documents"):
            call(q, top_k=5, group_by=torch.zeros(part.num_documents, dtype=torch.int64))
    fp.close()


# ---- NCCL: 2 and 4 ranks, one process per GPU ----------------------------------------------------------------------
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
    docs = make_docs(700, 10, 60, seed=570)
    oidx, _ = build_oracle_index(docs)
    t = to_index_tensors(oidx)
    queries = make_queries(5, 32, seed=571, docs=docs)  # B = 5: ragged over 2 and 4 query groups
    g = torch.arange(700, dtype=torch.int64) * 7 // 50
    plain = FastPlaid.from_device_index(DeviceIndex(t, dev))
    failed = []
    for m in (1, 3):
        kw = dict(group_by=g, max_per_group=m)
        ref_s = plain.search(queries, top_k=10, n_full_scores=512, **kw)
        ref_e = plain.search_exhaustive(queries, top_k=20, **kw)
        for n_groups in [q for q in (1, 2, 4) if world % q == 0]:
            _, d_shard, n_shards = shard_grid(rank, world, n_groups)
            sh, base = shard_tensors(t, d_shard, n_shards)
            fp = FastPlaid.from_device_index(DeviceIndex(sh, dev, doc_id_base=base), shard=(rank, world),
                                             query_groups=n_groups)
            if fp.search(queries, top_k=10, n_full_scores=512, **kw) != ref_s:
                failed.append(f"search m={m} groups={n_groups}")
            if fp.search(queries.to(dev), top_k=10, n_full_scores=512, **kw) != ref_s:
                failed.append(f"search (device queries) m={m} groups={n_groups}")
            if fp.search_exhaustive(queries, top_k=20, **kw) != ref_e:
                failed.append(f"search_exhaustive m={m} groups={n_groups}")
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
def test_nccl_grouped_sharded_equals_unsharded(world):
    """Every query-group grid the world allows: grouped search (host and device queries) and search_exhaustive
    through FastPlaid(shard=..., query_groups=G) equal the unsharded grouped calls."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    ok, failed = _spawn(_nccl_worker, world, 900)
    assert ok == 1, failed
