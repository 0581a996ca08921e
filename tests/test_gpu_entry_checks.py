"""Every DeviceIndex method that hands queries or all-gathered arrays to the C ABI checks them first: the kernels
read exactly B x Q x dim fp16 queries, and gathered arrays of the workspace layout's trailing sizes.  A mismatch
raises ValueError before anything is launched.  Each bad input here is larger than what the kernels read (fp32,
wider rows, longer trailing sizes), so a missing check would still read inside the buffer."""

from __future__ import annotations

import types

import pytest
import torch

from util import build_oracle_index, make_docs, make_queries, to_index_tensors

pytestmark = pytest.mark.gpu

B, Q = 3, 16


@pytest.fixture(scope="module")
def env(cuda_device):
    from fast_plaid_b200.engine import DeviceIndex, ShardComm

    docs = make_docs(300, 10, 40, seed=61)
    oidx, _ = build_oracle_index(docs)
    tensors = to_index_tensors(oidx)
    didx = DeviceIndex(tensors, cuda_device)
    comm = ShardComm(1, 0, ShardComm.new_unique_id(), cuda_device)
    queries = make_queries(B, Q, seed=62, docs=docs)
    yield types.SimpleNamespace(tensors=tensors, didx=didx, comm=comm, host=queries,
                                q16=queries.half().to(cuda_device), params=DeviceIndex.make_params(5, 64, 8))
    comm.close()
    didx.close()


def _device_call(name: str, env, q: torch.Tensor):
    from fast_plaid_b200.engine import FPB_FLAG_SUBSET, DeviceIndex

    d, p = env.didx, env.params
    one = torch.zeros(1, dtype=torch.int32)
    calls = {
        "search": lambda: d.search(q, p),
        "search_records": lambda: d.search_records(q, p),
        "search_sharded": lambda: d.search_sharded(env.comm, 1, q, p),
        "shard_approx_keys": lambda: d.shard_approx_keys(q, p),
        "shard_subset_begin": lambda: d.shard_subset_begin(q, DeviceIndex.with_flags(p, FPB_FLAG_SUBSET),
                                                           [[0, 1, 2]] * q.shape[0]),
        "run_stages": lambda: d.run_stages(q, p),
        "stage_fn": lambda: d.stage_fn("centroid_scores", q, p)(),
        "token_scores": lambda: d.token_scores(q, one, one),
        "exhaustive_scores": lambda: d.exhaustive_scores(q),
        "search_exhaustive": lambda: d.search_exhaustive(q, 5),
    }
    out = calls[name]()
    torch.cuda.synchronize()
    return out


DEVICE_METHODS = ["search", "search_records", "search_sharded", "shard_approx_keys", "shard_subset_begin",
                  "run_stages", "stage_fn", "token_scores", "exhaustive_scores", "search_exhaustive"]


@pytest.mark.parametrize("name", DEVICE_METHODS)
def test_device_query_methods_refuse_fp32_and_too_wide_queries(env, name):
    _device_call(name, env, env.q16)  # the well-formed call runs
    with pytest.raises(ValueError, match="fp16 queries"):
        _device_call(name, env, env.q16.float())
    wide = torch.zeros(B, Q, 2 * env.didx.dim, dtype=torch.float16, device=env.q16.device)
    with pytest.raises(ValueError, match="query dim"):
        _device_call(name, env, wide)


@pytest.mark.parametrize("name", ["search_host", "search_sharded_host"])
def test_host_query_methods_refuse_too_wide_queries(env, name):
    d, p = env.didx, env.params
    call = (lambda q: d.search_host(q, p)) if name == "search_host" else (
        lambda q: d.search_sharded_host(env.comm, 1, q, p))
    call(env.host)
    with pytest.raises(ValueError, match="query dim"):
        call(torch.zeros(B, Q, 2 * d.dim))


def test_gathered_inputs_must_match_the_layout(env):
    from fast_plaid_b200.engine import FPB_FLAG_SUBSET, DeviceIndex

    d, p, dev = env.didx, env.params, env.q16.device
    ps = DeviceIndex.with_flags(p, FPB_FLAG_SUBSET)
    _, lay = d.workspace(B, Q, ps)
    cb = torch.zeros((1, B, lay.cbitmap_words + 1), dtype=torch.int32, device=dev)
    with pytest.raises(ValueError, match="gathered"):
        d.shard_subset_keys(cb, Q, ps)
    keys = torch.zeros((1, B, lay.R + 1), dtype=torch.int64, device=dev)
    with pytest.raises(ValueError, match="gathered"):
        d.shard_exact_records(keys, 0, Q, p)
    recs = torch.full((1, B, lay.R, 17), 0xFF, dtype=torch.uint8, device=dev)
    with pytest.raises(ValueError, match="gathered"):
        d.merge_records(recs, p.top_k)
    # the shapes the layout asks for pass
    keys = d.shard_subset_keys(cb[:, :, :-1], Q, ps)
    rec = d.shard_exact_records(keys.unsqueeze(0), 0, Q, ps)
    d.merge_records(rec.unsqueeze(0), p.top_k)
    torch.cuda.synchronize()


def test_sharded_fastplaid_refuses_too_wide_cuda_queries(env):
    from fast_plaid_b200.engine import DeviceIndex
    from fast_plaid_b200.search.fast_plaid import FastPlaid

    fp = FastPlaid.from_device_index(DeviceIndex(env.tensors, env.q16.device), shard=(0, 1))
    try:
        with pytest.raises(ValueError, match="query dim"):
            fp.search(torch.zeros(B, Q, 2 * env.didx.dim, device=env.q16.device), top_k=5)
    finally:
        fp.close()
