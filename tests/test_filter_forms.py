"""Host side of the `subset=` tensor forms (no GPU): their checks, the split of a batch over several devices, and the
document count a mask must cover on a document-sharded index of several ranks (one all-reduce over the process
group; here gloo with two processes)."""

from __future__ import annotations

import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from fast_plaid_b200.search import fast_plaid as fpmod
from fast_plaid_b200.search.fast_plaid import FastPlaid, _split_subset, _SubsetTensor


def test_subset_forms_are_checked_and_classified():
    s = FastPlaid._subset_tensor
    n = lambda: 10  # noqa: E731
    assert s(None, 3, n) is None and s([], 3, n) is None and s([[1], [2], [3]], 3, n) is None
    assert torch.equal(s(7, 3, n).data, torch.tensor([7])) and not s(7, 3, n).per_query
    assert torch.equal(s([4, 2], 3, n).data, torch.tensor([4, 2]))
    assert s(torch.zeros(3, 5, dtype=torch.int32), 3, n).per_query
    assert s(torch.zeros(10, dtype=torch.bool), 3, n).data.dtype == torch.bool
    with pytest.raises(ValueError, match="float64"):
        s(torch.zeros(2, dtype=torch.float64), 3, n)
    with pytest.raises(ValueError, match=r"\[9\].*10 documents"):
        s(torch.zeros(9, dtype=torch.bool), 3, n)
    with pytest.raises(ValueError, match="Subset length must match number of queries"):
        s(torch.zeros(2, 10, dtype=torch.bool), 3, n)
    with pytest.raises(ValueError, match=r"\[3, 1, 1\]"):
        s(torch.zeros(3, 1, 1, dtype=torch.int64), 3, n)


def test_split_over_devices():
    """Shared forms go whole to every device, per-query forms by rows, lists by slices: 7 queries over 2 devices."""
    shared = _SubsetTensor(torch.arange(5))
    assert [x is shared for x in _split_subset(shared, 4, 2)] == [True, True]
    rows = _SubsetTensor(torch.arange(14).reshape(7, 2))
    parts = _split_subset(rows, 4, 2)
    assert torch.equal(parts[0].data, rows.data[:4]) and torch.equal(parts[1].data, rows.data[4:])
    mask = _SubsetTensor(torch.eye(7, dtype=torch.bool))
    assert [p.data.shape[0] for p in _split_subset(mask, 4, 2)] == [4, 3]
    assert _split_subset([[i] for i in range(7)], 4, 2) == [[[0], [1], [2], [3]], [[4], [5], [6]]]
    assert _split_subset(None, 4, 2) == [None, None]


def _free_port() -> int:
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank: int, world: int, port: int, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ends = [150, 300]  # rank r holds global ids [150 r, ends[r])
    out.put((rank, fpmod._sharded_num_documents(ends[rank], "cpu")))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_document_count_is_the_largest_range_end():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert got == {0: 300, 1: 300}
