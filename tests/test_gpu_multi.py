"""Multi-GPU tests of the document-sharded path over NCCL (skipped with fewer than 2 GPUs): the step-wise
exchange (fpb_search_shard / fpb_shard_* + all_gather_into_tensor + fpb_merge_shards) and the one-call
fpb_search_batch_sharded (ncclAllGather issued below the C ABI, every query-group x document-shard grid) must
equal the unsharded fpb_search_batch bit for bit on every rank.  The one-rank form of the C path runs on a
single GPU in tests/test_gpu_api.py."""

from __future__ import annotations

import os
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port() -> int:
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank: int, world: int, port: int, out):
    import sys

    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import torch.distributed as dist
    from util import build_oracle_index, make_docs, make_queries, to_index_tensors

    from fast_plaid_b200.engine import FPB_FLAG_SUBSET, DeviceIndex, shard_tensors

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    torch.set_num_threads(4)
    dev = f"cuda:{rank}"
    docs = make_docs(700, 10, 60, seed=31)
    oidx, _ = build_oracle_index(docs)
    t = to_index_tensors(oidx)
    queries = make_queries(5, 32, seed=32, docs=docs).half().to(dev)
    whole = DeviceIndex(t, dev)
    sh, base = shard_tensors(t, rank, world)
    mine = DeviceIndex(sh, dev, doc_id_base=base)
    ok = True
    for n_full, top_k in ((64, 10), (4096, 40)):
        params = DeviceIndex.make_params(top_k, n_full, 8)
        ids, scores, counts = whole.search(queries, params)
        rec = mine.search_records(queries, params)
        gathered = torch.empty((world,) + tuple(rec.shape), dtype=torch.uint8, device=dev)
        dist.all_gather_into_tensor(gathered.view(-1), rec.view(-1))
        i2, s2, c2 = mine.merge_records(gathered, top_k)
        torch.cuda.synchronize()
        ok = ok and torch.equal(i2, ids) and torch.equal(s2, scores) and torch.equal(c2, counts)
        # two-step variant
        keys = mine.shard_approx_keys(queries, params)
        all_keys = torch.empty((world,) + tuple(keys.shape), dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(all_keys.view(-1), keys.view(-1))
        rec2 = mine.shard_exact_records(all_keys, rank, int(queries.shape[1]), params)
        dist.all_gather_into_tensor(gathered.view(-1), rec2.view(-1))
        i3, s3, c3 = mine.merge_records(gathered, top_k)
        torch.cuda.synchronize()
        ok = ok and torch.equal(i3, ids) and torch.equal(s3, scores) and torch.equal(c3, counts)
        # subset search: the shards' centroid bitmaps are all-gathered and OR-ed (search.rs:494-517)
        g = torch.Generator().manual_seed(5)
        subset = [torch.randperm(700, generator=g)[:200].tolist() for _ in range(queries.shape[0])]
        subset[1] = list(range(0, 100))  # lives in shard 0 only
        i4, s4, c4 = whole.search(queries, params, subset=subset)
        ps = DeviceIndex.with_flags(params, FPB_FLAG_SUBSET)
        cb = mine.shard_subset_begin(queries, ps, subset)
        all_cb = torch.empty((world,) + tuple(cb.shape), dtype=torch.int32, device=dev)
        dist.all_gather_into_tensor(all_cb.view(-1), cb.view(-1))
        keys = mine.shard_subset_keys(all_cb, int(queries.shape[1]), ps)
        dist.all_gather_into_tensor(all_keys.view(-1), keys.view(-1))
        rec3 = mine.shard_exact_records(all_keys, rank, int(queries.shape[1]), ps)
        dist.all_gather_into_tensor(gathered.view(-1), rec3.view(-1))
        i5, s5, c5 = mine.merge_records(gathered, top_k)
        torch.cuda.synchronize()
        ok = ok and torch.equal(c5, c4)
        for b in range(queries.shape[0]):
            n = int(c4[b])
            ok = ok and torch.equal(i5[b, :n], i4[b, :n]) and torch.equal(s5[b, :n], s4[b, :n])
        # the same exchange below the C ABI: one call, both ncclAllGather issued inside (csrc/comm.cu), on every
        # grid of query groups x document shards the world allows
        from fast_plaid_b200.engine import ShardComm, shard_grid

        if "comm" not in locals():
            comm = ShardComm.from_process_group(dev)
        for n_groups in [g for g in (1, 2, 4) if world % g == 0]:
            _, d_shard, n_shards = shard_grid(rank, world, n_groups)
            sh_g, base_g = shard_tensors(t, d_shard, n_shards)
            part = DeviceIndex(sh_g, dev, doc_id_base=base_g)
            i6, s6, c6 = part.search_sharded(comm, n_groups, queries, params)
            torch.cuda.synchronize()
            ok = ok and torch.equal(i6, ids) and torch.equal(s6, scores) and torch.equal(c6, counts)
            h = part.search_sharded_host(comm, n_groups, queries.float().cpu(), params)
            ok = ok and torch.equal(h[0], ids.cpu()) and torch.equal(h[1], scores.cpu())
    # the FastPlaid surface in sharded mode: search and search_token_scores (matrices computed by the owning rank)
    from fast_plaid_b200.search.fast_plaid import FastPlaid

    fp_sh = FastPlaid.from_device_index(mine, shard=(rank, world))
    fp_w = FastPlaid.from_device_index(whole)
    qh = queries.float().cpu()
    ok = ok and fp_sh.search(qh, top_k=7) == fp_w.search(qh, top_k=7)
    ts_a, ts_b = fp_sh.search_token_scores(qh, top_k=4), fp_w.search_token_scores(qh, top_k=4)
    for ra, rb in zip(ts_a, ts_b):
        ok = ok and [(d, s_) for d, s_, _ in ra] == [(d, s_) for d, s_, _ in rb]
        ok = ok and all(torch.equal(ma, mb) for (_, _, ma), (_, _, mb) in zip(ra, rb))
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        out.put(int(flag.item()))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("world", [2, 4])
def test_nccl_sharded_search_equals_unsharded(world):
    import torch.multiprocessing as mp

    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = q.get(timeout=600)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert res == 1


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_replicated_devices_in_one_process_equal_a_single_device(tmp_path):
    """The reference's own multi-GPU mode (fast_plaid.py:893-928): one process, the index replicated on every device
    of the list, the query list split across one thread per device.  Every kernel's shared-memory opt-in must hold
    on the second device too (cudaFuncSetAttribute is per device)."""
    import sys

    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from util import make_docs, make_queries

    from fast_plaid_b200 import search

    docs = make_docs(400, 20, 80, seed=61)
    queries = make_queries(9, 32, seed=62, docs=docs)
    one = search.FastPlaid(str(tmp_path / "idx"), device="cuda:0")
    one.create(docs, kmeans_niters=2)
    ref = one.search(queries, top_k=10)
    ref_ts = one.search_token_scores(queries[:3], top_k=3)
    one.close()
    both = search.FastPlaid(str(tmp_path / "idx"), device=["cuda:0", "cuda:1"])
    got = both.search(queries, top_k=10)
    assert got == ref
    sub = both.search(queries, top_k=5, subset=list(range(0, 400, 2)))
    assert all(d % 2 == 0 for r in sub for d, _ in r)
    ts = both.search_token_scores(queries[:3], top_k=3)
    for ra, rb in zip(ts, ref_ts):
        assert [(d, s_) for d, s_, _ in ra] == [(d, s_) for d, s_, _ in rb]
        assert all(torch.equal(ma, mb) for (_, _, ma), (_, _, mb) in zip(ra, rb))
    both.close()
