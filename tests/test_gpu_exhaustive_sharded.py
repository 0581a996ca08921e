"""Exhaustive exact search on document-sharded indexes: fpb_shard_exhaustive_records + fpb_merge_shards (step-wise),
fpb_search_exhaustive_sharded (one call, the all-gather issued below the C ABI) and FastPlaid(shard=...).

The contract: the bytes search_exhaustive returns on one GPU holding the whole index -- ids, scores and counts -- at
every shard count and query-group grid.  GPU tests are marked; the NCCL cases need 2 or 4 GPUs and are skipped
below that.  The unmarked tests at the end run without a GPU: the C-ABI refusals, the merge limit of the FastPlaid
surface, the ranks' agreement on the batch step (over gloo) and the sharded refusals."""

from __future__ import annotations

import ctypes
import os
import socket

import numpy as np
import pytest
import torch
from util import build_oracle_index, make_docs, make_queries, to_index_tensors

from fast_plaid_b200.engine import DeviceIndex, shard_tensors

CODECS = [(128, 4), (128, 2), (64, 4), (64, 2), (128, 1)]


def _range_tensors(t, lo: int, hi: int):
    """Documents [lo, hi) of index tensors `t`, without an IVF (the exhaustive search reads none): shards of any
    size, where shard_tensors makes them differ by one document at most."""
    from fast_plaid_b200.engine import IndexTensors

    lens = t.doc_lengths.to(torch.int64)
    offs = torch.cat([torch.zeros(1, dtype=torch.int64), lens.cumsum(0)])
    t0, t1 = int(offs[lo]), int(offs[hi])
    return IndexTensors(t.nbits, t.centroids, t.bucket_weights, lens[lo:hi], t.doc_codes[t0:t1],
                        t.doc_residuals[t0:t1], None, None)


def _shards(t, world: int, device) -> list:
    out = []
    for r in range(world):
        sh, base = shard_tensors(t, r, world)
        out.append(DeviceIndex(sh, device, doc_id_base=base))
    return out


def _check_records(rec: torch.Tensor, part, k: int) -> None:
    """One shard's records: global ids of its own range, approx == exact, padding (-inf, -inf, -1) after the
    min(k, local documents) selected ones."""
    r = rec.cpu().contiguous()
    f = r.view(torch.float32)  # [B, k, 4]: approx, exact, id (two words)
    ids = r.view(torch.int64)[..., 1]
    n = min(k, part.num_documents)
    lo, hi = part.doc_id_base, part.doc_id_base + part.num_documents
    assert bool(((ids[:, :n] >= lo) & (ids[:, :n] < hi)).all()), "a record does not carry a global id of its shard"
    assert torch.equal(f[:, :n, 0], f[:, :n, 1]), "a record's approximate score is not its exact one"
    assert bool((ids[:, n:] == -1).all()), "a padding record's id is not -1"
    assert bool((f[:, n:, :2] == float("-inf")).all()), "a padding record's scores are not -inf"


def _top_ks(world: int, n_total: int, n_shard_max: int) -> list[int]:
    # 1, 10, more than one shard holds, more than the index holds, and 4096 or the merge limit's largest
    return [1, 10, n_shard_max + 1, n_total + 7, min(4096, 16384 // world)]


def _equal(a, b) -> bool:
    return all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.gpu
@pytest.mark.parametrize("dim,nbits", CODECS)
def test_stepwise_shards_merge_to_the_whole_index(dim, nbits, cuda_device):
    """2, 3 and 5 shards of one index on one GPU: every shard's records, stacked as an all-gather leaves them and
    merged with R = top_k, give the unsharded search_exhaustive's bytes.  Q 1, 32, 100 and 256; top_k up to 4096
    (the merge limit's largest at 5 shards), with shards of fewer documents than top_k."""
    docs = make_docs(150, 1, 40, dim=dim, seed=200 + dim + nbits)
    oidx, _ = build_oracle_index(docs, nbits=nbits)
    t = to_index_tensors(oidx)
    whole = DeviceIndex(t, cuda_device)
    N = whole.num_documents
    for world in (2, 3, 5):
        parts = _shards(t, world, cuda_device)
        assert sum(p.num_documents for p in parts) == N
        for Q in (1, 32, 100, 256):
            q16 = make_queries(3, Q, dim=dim, seed=300 + Q, docs=docs).half().to(cuda_device)
            for k in _top_ks(world, N, max(p.num_documents for p in parts)):
                ref = whole.search_exhaustive(q16, k)
                recs = [p.shard_exhaustive_records(q16, k) for p in parts]
                for p, rec in zip(parts, recs):
                    _check_records(rec, p, k)
                got = parts[0].merge_records(torch.stack(recs), k)
                torch.cuda.synchronize()
                assert _equal(got, ref), f"dim={dim} nbits={nbits} world={world} Q={Q} top_k={k}"
                assert bool((got[2] == min(k, N)).all())
        for p in parts:
            p.close()
    whole.close()


@pytest.mark.gpu
def test_ties_across_shards_rank_the_smaller_global_id_first(cuda_device):
    """Copies of a document planted in other shards score the same: the merged ranking must put the smaller global
    id first, as the canonical order of the whole index's exhaustive scores does."""
    docs = make_docs(60, 5, 30, seed=311)
    for src, dst in ((3, 25), (3, 47), (10, 55), (10, 30)):  # shards at world 3: [0, 20), [20, 40), [40, 60)
        docs[dst] = docs[src].clone()
    oidx, _ = build_oracle_index(docs)
    t = to_index_tensors(oidx)
    whole = DeviceIndex(t, cuda_device)
    queries = torch.cat([make_queries(2, 32, seed=312, docs=[docs[3]]),
                         make_queries(2, 32, seed=313, docs=[docs[10]])])
    q16 = queries.half().to(cuda_device)
    every = whole.exhaustive_scores(q16).cpu().numpy()
    parts = _shards(t, 3, cuda_device)
    k = 8
    ids, scores, counts = (x.cpu() for x in parts[0].merge_records(
        torch.stack([p.shard_exhaustive_records(q16, k) for p in parts]), k))
    for b, group in enumerate(([3, 25, 47], [3, 25, 47], [10, 30, 55], [10, 30, 55])):
        row = every[b]
        assert len({float(row[d]) for d in group}) == 1, "the planted copies do not score alike"
        order = np.lexsort((np.arange(row.shape[0]), -row))[:k]
        assert ids[b].tolist() == order.tolist(), f"query {b}: {ids[b].tolist()} vs {order.tolist()}"
        assert torch.equal(scores[b], torch.from_numpy(row[order])), f"query {b}: scores"
        pos = [ids[b].tolist().index(d) for d in group]
        assert pos == sorted(pos) and pos[-1] - pos[0] == 2, f"query {b}: the tied copies are not adjacent in id order"
    for p in parts:
        p.close()
    whole.close()


@pytest.mark.gpu
def test_one_rank_communicator(cuda_device):
    """fpb_search_exhaustive_sharded over a one-rank communicator equals fpb_search_exhaustive on a ragged batch of
    5 queries, in one call and in several; so does FastPlaid(shard=(0, 1)).search_exhaustive.  Two query groups on
    one rank are refused."""
    from fast_plaid_b200.engine import ShardComm
    from fast_plaid_b200.search.fast_plaid import FastPlaid

    docs = make_docs(500, 10, 60, seed=41)
    oidx, _ = build_oracle_index(docs)
    didx = DeviceIndex(to_index_tensors(oidx), cuda_device)
    queries = make_queries(5, 32, seed=42, docs=docs)
    q16 = queries.half().to(cuda_device)
    comm = ShardComm(1, 0, ShardComm.new_unique_id(), cuda_device)
    for k in (1, 10, 100, 600, 4096):
        ref = didx.search_exhaustive(q16, k)
        for step in (None, 2):
            got = didx.search_exhaustive_sharded(comm, 1, q16, k, step=step)
            torch.cuda.synchronize()
            assert _equal(got, ref), f"top_k={k} step={step}"
    with pytest.raises(ValueError, match="2 query groups do not divide 1 ranks"):
        didx.search_exhaustive_sharded(comm, 2, q16, 10)
    with pytest.raises(ValueError, match="top_k=4097"):
        didx.search_exhaustive_sharded(comm, 1, q16, 4097)
    comm.close()
    fp = FastPlaid.from_device_index(didx, shard=(0, 1))
    plain = FastPlaid.from_device_index(didx)
    for k in (10, 600):
        assert fp.search_exhaustive(queries, top_k=k) == plain.search_exhaustive(queries, top_k=k)
    # a budget of about two queries' workspace: several collective calls
    budget = didx.exhaustive_workspace_bytes(2, 32, 10)
    assert didx.exhaustive_sharded_step(1, 5, 32, 10, budget) < 5
    assert fp._search_exhaustive_sharded(didx, queries, 10, budget_bytes=budget) == plain.search_exhaustive(queries,
                                                                                                             top_k=10)
    with pytest.raises(NotImplementedError, match="document-sharded"):
        fp.search_exhaustive(queries, top_k=10, subset=[1, 2])
    groups = FastPlaid.from_device_index(didx, shard=(0, 1), query_groups=2)
    with pytest.raises(ValueError, match="query groups do not divide"):
        groups.search_exhaustive(queries, top_k=10)
    fp.close()


@pytest.mark.gpu
def test_compress_only_index_opened_sharded(tmp_path, cuda_device):
    """A compress_only index (no IVF: exhaustive search is its only search) opened with shard=(0, 1)."""
    from fast_plaid_b200 import search

    docs = make_docs(300, 5, 40, seed=121)
    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device=cuda_device)
    fp.create(docs, kmeans_niters=2, compress_only=True)
    queries = make_queries(4, 32, seed=122, docs=docs)
    ref = fp.search_exhaustive(queries, top_k=20)
    sharded = search.FastPlaid(path, device=cuda_device, shard=(0, 1))
    try:
        assert not sharded.indices[cuda_device].has_ivf
        assert sharded.search_exhaustive(queries, top_k=20) == ref
        assert sharded.search_exhaustive(queries, top_k=400) == fp.search_exhaustive(queries, top_k=400)
    finally:
        sharded.close()
        fp.close()


# ---- NCCL: 2 and 4 ranks, one process per GPU ----------------------------------------------------------------------
def _free_port() -> int:
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _nccl_worker(rank: int, world: int, port: int, out):
    import sys

    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import torch.distributed as dist
    from util import build_oracle_index, make_docs, make_queries, to_index_tensors

    from fast_plaid_b200.engine import DeviceIndex, ShardComm, shard_grid, shard_tensors
    from fast_plaid_b200.search.fast_plaid import FastPlaid, _results_to_lists

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    torch.set_num_threads(4)
    dev = f"cuda:{rank}"
    docs = make_docs(700, 10, 60, seed=31)
    oidx, _ = build_oracle_index(docs)
    t = to_index_tensors(oidx)
    queries = make_queries(5, 32, seed=32, docs=docs)  # B = 5: ragged over 2 and 4 query groups
    q16 = queries.half().to(dev)
    whole = DeviceIndex(t, dev)
    comm = ShardComm.from_process_group(dev)
    failed = []
    for k in (10, 100):
        ref = whole.search_exhaustive(q16, k)
        ref_lists = _results_to_lists(*(x.cpu() for x in ref))
        for n_groups in [g for g in (1, 2, 4) if world % g == 0]:
            _, d_shard, n_shards = shard_grid(rank, world, n_groups)
            sh, base = shard_tensors(t, d_shard, n_shards)
            part = DeviceIndex(sh, dev, doc_id_base=base)
            got = part.search_exhaustive_sharded(comm, n_groups, q16, k)
            torch.cuda.synchronize()
            if not _equal(got, ref):
                failed.append(f"one call, top_k={k} groups={n_groups}")
            fp = FastPlaid.from_device_index(part, shard=(rank, world), query_groups=n_groups)
            if fp.search_exhaustive(queries, top_k=k) != ref_lists:
                failed.append(f"FastPlaid, top_k={k} groups={n_groups}")
            fp.close()
        # shards of very different sizes and a budget of two queries' workspace on the smallest: the ranks' own steps
        # differ, and every rank must still make the same calls and return the unsharded result
        cuts = [round(700 * (r / world) ** 2) for r in range(world + 1)]
        part = DeviceIndex(_range_tensors(t, cuts[rank], cuts[rank + 1]), dev, doc_id_base=cuts[rank])
        budget = torch.tensor([part.exhaustive_workspace_bytes(2, 32, k)], dtype=torch.int64, device=dev)
        dist.all_reduce(budget, op=dist.ReduceOp.MIN)
        steps = torch.tensor([part.exhaustive_sharded_step(1, 5, 32, k, int(budget))] * 2, device=dev)
        dist.all_reduce(steps[:1], op=dist.ReduceOp.MIN)
        dist.all_reduce(steps[1:], op=dist.ReduceOp.MAX)
        if int(steps[0]) == int(steps[1]):
            failed.append(f"top_k={k}: the ranks' own steps do not differ ({steps.tolist()})")
        fp = FastPlaid.from_device_index(part, shard=(rank, world))
        if fp._search_exhaustive_sharded(part, queries, k, budget_bytes=int(budget)) != ref_lists:
            failed.append(f"budget {int(budget)}, top_k={k}")
        fp.close()
    comm.close()
    flag = torch.tensor([0 if failed else 1], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        out.put((int(flag.item()), failed))
    dist.barrier()
    dist.destroy_process_group()


def _spawn(target, world: int, timeout: float):
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = q.get(timeout=timeout)
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0
    finally:
        for p in procs:  # a rank that did not finish is not left behind
            if p.is_alive():
                p.kill()
                p.join()
    return res


@pytest.mark.gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("world", [2, 4])
def test_nccl_sharded_exhaustive_equals_unsharded(world):
    """Every grid of query groups x document shards the world allows, through the one-call path and through
    FastPlaid(shard=..., query_groups=G), on a batch of 5; and a budget that splits the batch while the shards'
    sizes differ, so that each rank alone would choose a different step."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    ok, failed = _spawn(_nccl_worker, world, 900)
    assert ok == 1, failed


# ---- CPU tier --------------------------------------------------------------------------------------------------------
def test_c_abi_refuses_bad_arguments():
    """The shapes first, then the pointers, before any CUDA call."""
    from fast_plaid_b200.engine import FPB_ERR_INVALID, FPB_ERR_UNSUPPORTED, load_library

    lib = load_library()

    def call(G=1, B=4, Q=32, top_k=10):
        return lib.fpb_search_exhaustive_sharded(None, None, G, None, B, Q, top_k, None, 0, None, 0, None, None,
                                                 None, None)

    assert call(top_k=0) == FPB_ERR_INVALID
    assert b"top_k=0 must be >= 1" in lib.fpb_last_error()
    assert call(top_k=4097) == FPB_ERR_UNSUPPORTED
    assert b"top_k=4097" in lib.fpb_last_error()
    assert call(Q=257) == FPB_ERR_UNSUPPORTED
    assert b"Q=257" in lib.fpb_last_error()
    assert call(B=0) == FPB_ERR_INVALID
    assert call(G=0) == FPB_ERR_INVALID  # no query-group count divides the ranks unless it is at least 1
    assert b"n_query_groups=0" in lib.fpb_last_error()
    assert call() == FPB_ERR_INVALID  # every shape above is fine: NULL index and communicator
    assert b"NULL argument" in lib.fpb_last_error()

    def records(B=4, Q=32, top_k=10):
        return lib.fpb_shard_exhaustive_records(None, None, B, Q, top_k, None, 0, None, None)

    assert records(top_k=0) == FPB_ERR_INVALID
    assert records(top_k=4097) == FPB_ERR_UNSUPPORTED
    assert records(Q=257) == FPB_ERR_UNSUPPORTED
    assert records() == FPB_ERR_INVALID
    assert b"NULL index" in lib.fpb_last_error()


def test_sharded_exhaustive_merge_limit():
    """n_shards * top_k <= 16384: top_k 2048 on 8 shards reaches the communicator, 2049 raises ValueError before it
    exists; 4 shards (2 query groups of 8 ranks) take 4096."""
    from fast_plaid_b200.engine import check_exhaustive_merge_records
    from fast_plaid_b200.search.fast_plaid import FastPlaid

    for n_shards, k in ((1, 4096), (4, 4096), (8, 2048), (16, 1024), (3, 5461)):
        check_exhaustive_merge_records(n_shards, k)
    for n_shards, k in ((8, 2049), (5, 4096), (16, 1025), (16385, 1)):
        with pytest.raises(ValueError, match="exceed the 16384"):
            check_exhaustive_merge_records(n_shards, k)

    class Reached(Exception):
        pass

    def shard_comm(idx):
        raise Reached

    fp = FastPlaid.__new__(FastPlaid)
    fp.shard = (0, 8)  # 8 ranks
    fp._shard_comm = shard_comm
    q = torch.zeros(1, 4, 128)
    for groups, k, error in ((1, 2048, Reached), (1, 2049, ValueError), (2, 4096, Reached), (2, 4097, ValueError),
                             (3, 10, ValueError)):
        fp.query_groups = groups  # 8 / groups document shards; 3 groups do not divide 8 ranks
        with pytest.raises(error):
            fp._search_exhaustive_sharded(None, q, k)


class _CpuShard:
    """The workspace arithmetic of a shard, without a GPU: `per_query` bytes per query on top of a fixed part."""

    device = torch.device("cpu")

    def __init__(self, per_query: int) -> None:
        self.per_query = per_query

    def exhaustive_workspace_bytes(self, B: int, Q: int, top_k: int) -> int:
        return 4096 + B * self.per_query

    _exhaustive_step = DeviceIndex._exhaustive_step
    exhaustive_sharded_step = DeviceIndex.exhaustive_sharded_step


def _gloo_worker(rank: int, world: int, port: int, out):
    import sys

    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import torch.distributed as dist

    from fast_plaid_b200.search.fast_plaid import FastPlaid

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    fp = FastPlaid.__new__(FastPlaid)
    fp.shard, fp.query_groups = (rank, world), 1
    shard = _CpuShard(1000 + rank)  # rank 1 holds a little more per query
    budget = 4096 + 10 * 1000  # rank 0 fits 10 queries per call, rank 1 only 9
    own = shard.exhaustive_sharded_step(1, 64, 32, 10, budget)
    agreed = fp._exhaustive_sharded_step(shard, 64, 32, 10, budget)
    both = [None] * world
    dist.all_gather_object(both, (own, agreed))
    if rank == 0:
        out.put(both)
    dist.barrier()
    dist.destroy_process_group()


def test_ranks_agree_on_the_step_over_gloo():
    """Two ranks whose workspace crosses the budget at different batch sizes choose the same step, the smaller."""
    both = _spawn(_gloo_worker, 2, 300)
    assert [own for own, _ in both] == [10, 9]
    assert [agreed for _, agreed in both] == [9, 9]


def test_sharded_refusals_come_before_the_index_is_touched(tmp_path):
    """subset= on a document-sharded index stays refused, in every form `search` accepts; several ranks without a
    torch.distributed process group (through which the communicator is made and the step agreed) are refused; one
    rank needs no process group and goes on to the search itself (here: the CPU device's refusal)."""
    from fast_plaid_b200 import search
    from fast_plaid_b200.engine import EngineUnavailableError

    bare = search.FastPlaid.__new__(search.FastPlaid)
    bare.shard = (0, 2)
    q = torch.randn(2, 8, 128)
    for subset in (7, [1, 2], [[1], [2]]):
        with pytest.raises(NotImplementedError, match="subset= on a document-sharded index"):
            search.FastPlaid.search_exhaustive(bare, q, subset=subset)
    path = str(tmp_path / "idx")
    search.FastPlaid(path, device="cpu").create(make_docs(30, 5, 30, seed=141), kmeans_niters=2)
    two = search.FastPlaid(path, device="cpu", shard=(1, 2))
    for subset in (None, []):
        with pytest.raises(NotImplementedError, match="document-sharded index of 2 ranks needs an initialised"):
            two.search_exhaustive(q, top_k=5, subset=subset)
    one = search.FastPlaid(path, device="cpu", shard=(0, 1))
    with pytest.raises(EngineUnavailableError, match="no CPU search path"):
        one.search_exhaustive(q, top_k=5)
