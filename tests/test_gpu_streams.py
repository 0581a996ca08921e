"""The stream and thread contract of every entry point (include/fastplaid_b200.h): each runs on the caller's stream,
the `_host` ones synchronise that stream, and one fpb_index serves several host threads at once, each with its own
stream and workspace.  The memory a DeviceIndex caches across calls (workspace, scratch, pinned staging, the tensors
kept alive for the stream) must stay valid for every stream that still uses it.

Each scenario makes its ordering deterministic with a hold: a ~200 ms sleep kernel enqueued on a non-blocking side
stream, so the work queued behind it cannot have run when the host issues the next operation.  The reference of every
check is the serial run, the same call on the default stream, synchronised; the other suites hold that run to the
float64 and oracle references.  Comparisons are byte-exact (floats as their int32 bit patterns).  Every scenario runs
once, and all memory it touches stays allocated in PyTorch's caching allocator: a wrong order gives wrong bytes."""

from __future__ import annotations

import ast
import contextlib
import ctypes
import gc
import os
import random
import threading

import pytest
import torch
from util import build_oracle_index, make_docs, make_queries, to_index_tensors

from fast_plaid_b200 import engine
from fast_plaid_b200.engine import (
    FPB_FLAG_APPROX_DIRECT, FPB_FLAG_APPROX_TWO_PASS, FPB_FLAG_SUBSET, DeviceIndex, Filter, Groups, ShardComm,
    encode_tokens, kmeans_assign, kmeans_update, shard_tensors,
)

CODECS = [(128, 4), (128, 2), (64, 4), (64, 2), (128, 1)]
N_DOCS, B, Q, K = 400, 6, 32, 10
HOLD_MS = 200.0  # long enough that a host hiccup does not outlast it
PARAMS = DeviceIndex.make_params(K, 64, 8)


# ---- the hold -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="session")
def hold(cuda_device):
    """hold(stream, ms): enqueue a sleep of about `ms` on `stream`.  The SM clock is measured, not assumed."""
    side = torch.cuda.Stream(cuda_device)

    def timed(cycles: int) -> float:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(side):
            a.record()
            torch.cuda._sleep(cycles)
            b.record()
        b.synchronize()
        return a.elapsed_time(b)

    timed(1000)  # module load
    probe = 20_000_000
    per_ms = max(probe / max(timed(probe), 1e-3) for _ in range(3))  # the fastest clock seen: holds are not shorter
    took = timed(int(per_ms * HOLD_MS))
    assert took >= HOLD_MS / 2, f"a hold of {HOLD_MS} ms took {took:.1f} ms: every check below would be vacuous"

    def _hold(stream: torch.cuda.Stream, ms: float = HOLD_MS) -> None:
        with torch.cuda.stream(stream):
            torch.cuda._sleep(int(per_ms * ms))

    return _hold


@contextlib.contextmanager
def _no_collection():
    """No garbage collection while a scenario times a call against a hold: an index collected then would synchronise
    the device in its finaliser (DeviceIndex.close) and make an asynchronous call look blocking."""
    gc.collect()
    gc.disable()
    try:
        yield
    finally:
        gc.enable()


# ---- byte comparison ----------------------------------------------------------------------------------------------
def _bits(x):
    if isinstance(x, torch.Tensor):
        t = x.detach().cpu().contiguous()
        return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16) if t.dtype == torch.float16 else t
    if isinstance(x, (tuple, list)):
        return [_bits(y) for y in x]
    return x


def _same(a, b) -> bool:
    a, b = _bits(a), _bits(b)
    if isinstance(a, torch.Tensor) or isinstance(b, torch.Tensor):
        return (isinstance(a, torch.Tensor) and isinstance(b, torch.Tensor) and a.dtype == b.dtype
                and a.shape == b.shape and torch.equal(a, b))
    if isinstance(a, list) and isinstance(b, list):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


# ---- the indexes --------------------------------------------------------------------------------------------------
class _Ctx:
    """One codec's index, its shards, queries and inputs, built on first use."""

    def __init__(self, dim: int, nbits: int, device: str) -> None:
        self.dim, self.nbits, self.device = dim, nbits, device
        self.docs = make_docs(N_DOCS, 4, 40, dim=dim, seed=100 + dim + nbits)
        oidx, _ = build_oracle_index(self.docs, nbits=nbits, kmeans_niters=2)
        self.tensors = to_index_tensors(oidx)
        self.didx = DeviceIndex(self.tensors, device)
        self.queries = make_queries(B, Q, dim=dim, seed=7, docs=self.docs)  # host fp32
        self.decoy_queries = make_queries(B, Q, dim=dim, seed=8, docs=self.docs)
        self.q = self.queries.half().to(device)
        self.qd = self.decoy_queries.half().to(device)
        rng = random.Random(dim * 10 + nbits)
        self.sets = [sorted(rng.sample(range(N_DOCS), rng.randrange(20, 200))) for _ in range(B)]
        self.decoy_sets = [sorted(rng.sample(range(N_DOCS), rng.randrange(20, 200))) for _ in range(B)]
        self.shards: dict[int, list[DeviceIndex]] = {}
        self._comm = None

    def shard_indexes(self, world: int) -> list[DeviceIndex]:
        if world not in self.shards:
            parts = [shard_tensors(self.tensors, r, world) for r in range(world)]
            self.shards[world] = [DeviceIndex(t, self.device, doc_id_base=base) for t, base in parts]
        return self.shards[world]

    @property
    def comm(self) -> ShardComm:
        if self._comm is None:
            self._comm = ShardComm(1, 0, ShardComm.new_unique_id(), self.device)
        return self._comm

    def close(self) -> None:
        if self._comm is not None:
            self._comm.close()


@pytest.fixture(scope="module")
def ctx_of(cuda_device):
    made: dict[tuple, _Ctx] = {}

    def get(codec) -> _Ctx:
        if codec not in made:
            made[codec] = _Ctx(*codec, cuda_device)
        return made[codec]

    yield get
    for c in made.values():
        c.close()


def _padded(sets: list[list[int]]) -> torch.Tensor:
    L = max(len(s) for s in sets)
    return torch.tensor([s + [-1] * (L - len(s)) for s in sets], dtype=torch.int64)


def _mask(ids: list[int], n: int) -> torch.Tensor:
    m = torch.zeros(n, dtype=torch.bool)
    m[torch.tensor(ids, dtype=torch.int64)] = True
    return m


def _group_ids(c: _Ctx, mult: int) -> torch.Tensor:
    """A dense group map of 37 groups (device int32)."""
    return Groups.from_tensor((torch.arange(N_DOCS) * mult) % 37, N_DOCS, c.device).ids


# ---- the entry points ---------------------------------------------------------------------------------------------
# Each builder returns (fn, real inputs, decoy inputs): fn(*inputs) calls the entry point on the current stream.
# BLOCKS: the entry points whose Python wrapper waits for the stream before it returns, and the line that does.
def _search(flags: int = 0):
    def build(c):
        p = DeviceIndex.with_flags(PARAMS, flags)
        return (lambda q: c.didx.search(q, p)), [c.q], [c.qd]
    return build


def _search_subset(c):
    return (lambda q: c.didx.search(q, PARAMS, subset=c.sets)), [c.q], [c.qd]


def _search_filter_ids(c):
    bm = Filter.from_ids(_padded(c.sets).to(c.device), N_DOCS, c.device, B).bitmap
    bd = Filter.from_ids(_padded(c.decoy_sets).to(c.device), N_DOCS, c.device, B).bitmap
    return (lambda q, m: c.didx.search(q, PARAMS, filter=Filter(m, list(range(B)), N_DOCS))), [c.q, bm], [c.qd, bd]


def _search_filter_mask(c):
    bm = Filter.from_mask(_mask(c.sets[0], N_DOCS).to(c.device), c.device, B).bitmap
    bd = Filter.from_mask(_mask(c.decoy_sets[0], N_DOCS).to(c.device), c.device, B).bitmap
    return (lambda q, m: c.didx.search(q, PARAMS, filter=Filter(m, [0] * B, N_DOCS))), [c.q, bm], [c.qd, bd]


def _search_groups(m: int):
    def build(c):
        return ((lambda q, g: c.didx.search(q, PARAMS, groups=Groups(g, 37, m))),
                [c.q, _group_ids(c, 1)], [c.qd, _group_ids(c, 7)])
    return build


def _exhaustive(c):
    return (lambda q: c.didx.search_exhaustive(q, K)), [c.q], [c.qd]


def _exhaustive_subset(c):
    return (lambda q: c.didx.search_exhaustive(q, K, subset=c.sets)), [c.q], [c.qd]


def _exhaustive_rows(c):
    rows = _padded(c.sets).to(c.device)
    L = rows.shape[1]
    decoy = torch.tensor([(s + [-1] * L)[:L] for s in c.decoy_sets], dtype=torch.int64, device=c.device)
    return (lambda q, r: c.didx.search_exhaustive(q, K, subset=r)), [c.q, rows], [c.qd, decoy]


def _exhaustive_filter(c):
    fn, real, decoy = _search_filter_ids(c)
    return ((lambda q, m: c.didx.search_exhaustive(q, K, filter=Filter(m, list(range(B)), N_DOCS))), real, decoy)


def _exhaustive_groups(c):
    return ((lambda q, g: c.didx.search_exhaustive(q, K, groups=Groups(g, 37, 3))),
            [c.q, _group_ids(c, 1)], [c.qd, _group_ids(c, 7)])


def _exhaustive_split(c):
    budget = c.didx.exhaustive_workspace_bytes(1, Q, K)  # the smallest call's workspace: the batch is split
    assert c.didx._exhaustive_step(B, Q, K, budget) < B
    return (lambda q: c.didx.search_exhaustive(q, K, budget_bytes=budget)), [c.q], [c.qd]


def _exhaustive_scores(c):
    return (lambda q: c.didx.exhaustive_scores(q)), [c.q], [c.qd]


def _search_records(c):
    return (lambda q: c.didx.search_records(q, PARAMS)), [c.q], [c.qd]


def _stepwise(world: int):
    def build(c):
        shards = c.shard_indexes(world)

        def fn(q):
            keys = torch.stack([d.shard_approx_keys(q, PARAMS) for d in shards])
            recs = torch.stack([d.shard_exact_records(keys, r, Q, PARAMS) for r, d in enumerate(shards)])
            return c.didx.merge_records(recs, K)
        return fn, [c.q], [c.qd]
    return build


def _stepwise_filter(c):
    shards = c.shard_indexes(2)
    ps = DeviceIndex.with_flags(PARAMS, FPB_FLAG_SUBSET)
    _, real, decoy = _search_filter_ids(c)

    def fn(q, m):
        f = Filter(m, list(range(B)), N_DOCS)
        cbs = torch.stack([d.shard_subset_begin(q, ps, filter=f) for d in shards])
        keys = torch.stack([d.shard_subset_keys(cbs, Q, ps) for d in shards])
        recs = torch.stack([d.shard_exact_records(keys, r, Q, ps) for r, d in enumerate(shards)])
        return c.didx.merge_records(recs, K)
    return fn, real, decoy


def _stepwise_exhaustive(c):
    shards = c.shard_indexes(2)
    return ((lambda q: c.didx.merge_records(torch.stack([d.shard_exhaustive_records(q, K) for d in shards]), K)),
            [c.q], [c.qd])


def _sharded(c):
    return (lambda q: c.didx.search_sharded(c.comm, 1, q, PARAMS)), [c.q], [c.qd]


def _exhaustive_sharded(c):
    return (lambda q: c.didx.search_exhaustive_sharded(c.comm, 1, q, K)), [c.q], [c.qd]


def _token_scores(c):
    qo = torch.tensor([0, 1, 2, 3, 4, 5, 0, 5], dtype=torch.int32, device=c.device)
    di = torch.tensor([3, 50, 120, 7, 399, 211, 64, 0], dtype=torch.int32, device=c.device)
    dd = torch.tensor([8, 9, 10, 11, 12, 13, 14, 15], dtype=torch.int32, device=c.device)
    return (lambda q, o, d: c.didx.token_scores(q, o, d)), [c.q, qo, di], [c.qd, qo, dd]


def _reconstruct(c):
    return (lambda: c.didx.reconstruct([5, 399, 0, 77])), [], []


def _from_ids(c):
    real = _padded(c.sets).to(c.device)
    decoy = torch.flip(real, (0,)).contiguous()
    return (lambda ids: Filter.from_ids(ids, N_DOCS, c.device, B).bitmap), [real], [decoy]


def _from_mask(c):
    real = torch.stack([_mask(s, N_DOCS) for s in c.sets]).to(c.device)
    return (lambda m: Filter.from_mask(m, c.device, B).bitmap), [real], [torch.flip(real, (0,)).contiguous()]


def _tokens(c, seed: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.nn.functional.normalize(torch.randn(256, c.dim, generator=g), dim=-1).half().to(c.device)


def _encode(c):
    cutoffs = torch.linspace(-0.04, 0.04, 2**c.nbits - 1, device=c.device)
    return ((lambda t: encode_tokens(t, c.didx.centroids, cutoffs, c.nbits)), [_tokens(c, 1)], [_tokens(c, 2)])


def _kmeans_assign(c):
    return (lambda p: kmeans_assign(p, c.didx.centroids)), [_tokens(c, 1)], [_tokens(c, 2)]


def _kmeans_update(c):
    cent = c.didx.centroids[:16].clone()
    pts, other = _tokens(c, 1), _tokens(c, 2)
    a, b = kmeans_assign(pts, cent), kmeans_assign(other, cent)

    def fn(p, asg, cen):
        cen = cen.clone()  # updated in place
        counts, shift = kmeans_update(p, asg, cen)
        return counts, shift, cen
    return fn, [pts, a, cent], [other, b, cent.flip(0).contiguous()]


# name -> (builder, the engine functions it reaches, codecs, why it blocks or None)
_SUBSET_CSR = "engine.py DeviceIndex._subset_csr: `.to(self.device)` of the pageable host lists waits for the stream"
ENTRIES = {
    "search": (_search(), ["DeviceIndex.search"], CODECS, None),
    "search-subset": (_search_subset, ["DeviceIndex.search"], CODECS, _SUBSET_CSR),
    "search-filter-ids": (_search_filter_ids, ["DeviceIndex.search"], CODECS, None),
    "search-filter-mask": (_search_filter_mask, ["DeviceIndex.search"], CODECS, None),
    "search-groups-1": (_search_groups(1), ["DeviceIndex.search"], CODECS, None),
    "search-groups-3": (_search_groups(3), ["DeviceIndex.search"], CODECS, None),
    "search-two-pass": (_search(FPB_FLAG_APPROX_TWO_PASS), ["DeviceIndex.search"], CODECS, None),
    "search-direct": (_search(FPB_FLAG_APPROX_DIRECT), ["DeviceIndex.search"], CODECS, None),
    "search_records": (_search_records, ["DeviceIndex.search_records"], CODECS, None),
    "stepwise-2": (_stepwise(2), ["DeviceIndex.shard_approx_keys", "DeviceIndex.shard_exact_records",
                                  "DeviceIndex.merge_records"], CODECS, None),
    "stepwise-4": (_stepwise(4), ["DeviceIndex.shard_approx_keys", "DeviceIndex.shard_exact_records",
                                  "DeviceIndex.merge_records"], CODECS, None),
    "stepwise-filter": (_stepwise_filter, ["DeviceIndex.shard_subset_begin", "DeviceIndex.shard_subset_keys",
                                           "DeviceIndex.shard_exact_records", "DeviceIndex.merge_records"],
                        CODECS, None),
    "stepwise-exhaustive": (_stepwise_exhaustive, ["DeviceIndex.shard_exhaustive_records",
                                                   "DeviceIndex.merge_records"], CODECS, None),
    "search_sharded": (_sharded, ["DeviceIndex.search_sharded"], CODECS, None),
    "search_exhaustive_sharded": (_exhaustive_sharded, ["DeviceIndex.search_exhaustive_sharded"], CODECS, None),
    "exhaustive": (_exhaustive, ["DeviceIndex.search_exhaustive"], CODECS, None),
    "exhaustive-subset": (_exhaustive_subset, ["DeviceIndex._search_exhaustive_subset"], CODECS, _SUBSET_CSR),
    "exhaustive-rows": (_exhaustive_rows, ["DeviceIndex._search_exhaustive_id_rows"], CODECS, None),
    "exhaustive-filter": (_exhaustive_filter, ["DeviceIndex._search_exhaustive_filter"], CODECS,
                          "engine.py DeviceIndex._search_exhaustive_filter: `int(self.filter_counts(filter).max())` "
                          "sizes the workspace from the device"),
    "exhaustive-groups": (_exhaustive_groups, ["DeviceIndex.search_exhaustive"], CODECS, None),
    "exhaustive-split": (_exhaustive_split, ["DeviceIndex.search_exhaustive"], CODECS, None),
    "exhaustive_scores": (_exhaustive_scores, ["DeviceIndex.exhaustive_scores"], CODECS, None),
    "token_scores": (_token_scores, ["DeviceIndex.token_scores"], CODECS, None),
    "reconstruct": (_reconstruct, ["DeviceIndex.reconstruct"], CODECS,
                    "engine.py DeviceIndex.reconstruct: `self.doc_offsets.cpu()` reads the document lengths"),
    "Filter.from_ids": (_from_ids, ["Filter.from_ids"], CODECS[:1], None),
    "Filter.from_mask": (_from_mask, ["Filter.from_mask"], CODECS[:1], None),
    "encode_tokens": (_encode, ["encode_tokens"], CODECS[:1], None),
    "kmeans_assign": (_kmeans_assign, ["kmeans_assign"], CODECS[:1], None),
    "kmeans_update": (_kmeans_update, ["kmeans_update"], CODECS[:1],
                      "engine.py kmeans_update: `torch.bincount` on the device reads the largest assignment"),
}
# the `_host` entry points, tested by test_host_calls_synchronise_the_callers_stream
HOST_ENTRIES = {"search_host": ["DeviceIndex.search_host"], "search_sharded_host": ["DeviceIndex.search_sharded_host"]}
# engine functions that pass a stream to the library without a test here, and why
EXEMPT = {
    "DeviceIndex.append": "synchronises the stream before fpb_index_append (index construction, test_gpu_append.py)",
    "DeviceIndex.delete": "synchronises the stream before fpb_index_create (index construction, test_gpu_delete.py)",
    "DeviceIndex.run_stages": "stage-level access for the kernel tests; its stream order is tested by "
                              "test_one_device_index_shared_by_two_threads",
    "DeviceIndex.stage_fn": "stage launcher of the roofline bench, which times it on one stream",
}

_PAIRS = [(name, codec) for name, (_, _, codecs, _) in ENTRIES.items() for codec in codecs]


def _on_held_stream(hold, fn, real: list, decoy: list, device: str):
    """fn on a held side stream, its inputs holding `decoy` until the stream copies `real` over them after the hold.
    Returns (outputs, whether the call returned while the stream was still held)."""
    bufs = [d.clone() for d in decoy]
    torch.cuda.synchronize(device)
    s = torch.cuda.Stream(device)
    with _no_collection():
        hold(s)
        held = torch.cuda.Event()
        held.record(s)
        with torch.cuda.stream(s):
            for b, r in zip(bufs, real):
                b.copy_(r)
            out = fn(*bufs)
        returned_held = not held.query()
    torch.cuda.synchronize(device)
    return out, returned_held


@pytest.mark.gpu
@pytest.mark.parametrize("name,codec", _PAIRS, ids=[f"{n}-d{d}n{b}" for n, (d, b) in _PAIRS])
def test_entry_point_runs_on_the_callers_stream(name, codec, ctx_of, hold, cuda_device):
    """Every stage runs on the caller's stream, after the inputs that stream wrote: anything launched on another
    stream, or before its inputs exist, reads the decoy.  The asynchronous ones return while the stream is held."""
    c = ctx_of(codec)
    build, _, _, blocks = ENTRIES[name]
    fn, real, decoy = build(c)
    ref = fn(*real)
    torch.cuda.synchronize()
    if real:
        assert not _same(fn(*decoy), ref), f"{name}: the decoy input gives the same bytes, the check is vacuous"
        torch.cuda.synchronize()
    got, returned_held = _on_held_stream(hold, fn, real, decoy, cuda_device)
    assert _same(got, ref), f"{name}: the held-stream call differs from the serial call"
    if blocks is None:
        assert returned_held, f"{name}: returned only after the hold had ended"
    else:
        assert not returned_held, f"{name}: returned while the stream was held; it no longer blocks ({blocks})"


@pytest.mark.gpu
@pytest.mark.parametrize("codec", CODECS, ids=[f"d{d}n{n}" for d, n in CODECS])
@pytest.mark.parametrize("name", list(HOST_ENTRIES))
def test_host_calls_synchronise_the_callers_stream(name, codec, ctx_of, hold, cuda_device):
    """With the caller's stream held, a `_host` call returns the right host tensors without a further synchronise:
    it waited for that stream, not the legacy one.  The pinned result buffers hold a decoy batch's results before."""
    c = ctx_of(codec)
    if name == "search_host":
        def fn(x):
            return c.didx.search_host(x, PARAMS)
    else:
        def fn(x):
            return c.didx.search_sharded_host(c.comm, 1, x, PARAMS)
    ref = fn(c.queries)
    decoy = fn(c.decoy_queries)
    assert not _same(decoy, ref)
    s = torch.cuda.Stream(cuda_device)
    hold(s)
    with torch.cuda.stream(s):
        got = fn(c.queries)
        assert _same(got, ref), f"{name}: host results read before the caller's stream finished"
        assert torch.cuda.current_stream().query()
    torch.cuda.synchronize()


# ---- concurrent calls ---------------------------------------------------------------------------------------------
def _run_threads(targets) -> None:
    errors: list[BaseException] = []

    def wrap(t):
        try:
            t()
        except BaseException as e:  # noqa: BLE001  (re-raised on the main thread)
            errors.append(e)
    threads = [threading.Thread(target=wrap, args=(t,)) for t in targets]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    if errors:
        raise errors[0]


@pytest.mark.gpu
@pytest.mark.parametrize("mix", [False, True], ids=["search", "mixed"])
@pytest.mark.parametrize("n_threads", [2, 4])
def test_one_fpb_index_serves_threads_with_their_own_workspaces(n_threads, mix, ctx_of, hold, cuda_device):
    """The header's sentence as written: several host threads search one fpb_index at once, each on its own
    non-blocking stream with its own workspace (fpb_search_batch, fpb_search_exhaustive, fpb_token_scores)."""
    c = ctx_of(CODECS[0])
    didx, lib = c.didx, c.didx._lib
    kinds = [("search", "exhaustive", "token")[i % 3] if mix else "search" for i in range(n_threads)]
    qs = [make_queries(B, Q, dim=c.dim, seed=200 + i, docs=c.docs).half().to(cuda_device) for i in range(n_threads)]
    qo = torch.arange(B, dtype=torch.int32, device=cuda_device).repeat(2)
    di = torch.arange(0, 2 * B * 30, 30, dtype=torch.int32, device=cuda_device)

    def setup(kind):
        if kind == "search":
            ws = torch.empty(didx.layout(B, Q, PARAMS).total_bytes, dtype=torch.uint8, device=cuda_device)
        elif kind == "exhaustive":
            ws = torch.empty(didx.exhaustive_workspace_bytes(B, Q, K), dtype=torch.uint8, device=cuda_device)
        else:
            ws = None
        if kind == "token":
            out = [torch.zeros((2 * B, didx.max_doc_len, Q), dtype=torch.float16, device=cuda_device)]
        else:
            out = [torch.full((B, K), -7, dtype=torch.int64, device=cuda_device),
                   torch.full((B, K), -7.0, dtype=torch.float32, device=cuda_device),
                   torch.full((B,), -7, dtype=torch.int32, device=cuda_device)]
        return ws, out

    def call(kind, q, ws, out, st: int) -> None:
        if kind == "search":
            rc = lib.fpb_search_batch(didx._handle, q.data_ptr(), B, Q, ctypes.byref(PARAMS), ws.data_ptr(),
                                      ws.numel(), *(t.data_ptr() for t in out), st)
        elif kind == "exhaustive":
            rc = lib.fpb_search_exhaustive(didx._handle, q.data_ptr(), B, Q, K, ws.data_ptr(), ws.numel(),
                                           *(t.data_ptr() for t in out), st)
        else:
            rc = lib.fpb_token_scores(didx._handle, q.data_ptr(), Q, qo.data_ptr(), di.data_ptr(), 2 * B,
                                      didx.max_doc_len, out[0].data_ptr(), st)
        assert rc == 0, lib.fpb_last_error()

    refs = []
    for kind, q in zip(kinds, qs):
        ws, out = setup(kind)
        call(kind, q, ws, out, torch.cuda.current_stream().cuda_stream)
        refs.append(out)
    torch.cuda.synchronize()
    states = [setup(kind) for kind in kinds]
    streams = [torch.cuda.Stream(cuda_device) for _ in kinds]
    torch.cuda.synchronize()
    barrier = threading.Barrier(n_threads)

    def worker(i):
        def run():
            barrier.wait()
            hold(streams[i])
            call(kinds[i], qs[i], *states[i], streams[i].cuda_stream)
        return run
    _run_threads([worker(i) for i in range(n_threads)])
    torch.cuda.synchronize()
    for i, (ref, (_, out)) in enumerate(zip(refs, states)):
        assert _same(out, ref), f"thread {i} ({kinds[i]}) differs from its serial run"


def _views(r: dict) -> list:
    """The workspace state a `run_stages` call leaves, per query: candidate and re-rank counts, re-ranked ids and
    their exact scores."""
    n = r["n_rerank"].cpu()
    return [r["n_cand"], n, r["ids"], r["scores"], r["counts"]] + [
        r["rerank"][b, : int(n[b])] for b in range(n.shape[0])] + [r["exact"][b, : int(n[b])] for b in range(n.shape[0])]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["search", "search_exhaustive", "search_records", "run_stages"])
def test_one_device_index_shared_by_two_threads(kind, ctx_of, hold, cuda_device):
    """Thread A searches X on a held stream; thread B, as soon as A's call returns, searches Y on an unheld stream
    with the same DeviceIndex and so the same workspace.  B's call must be ordered after A's: both equal their serial
    runs, and the workspace a `run_stages` of B leaves holds Y's state, not X's."""
    c = ctx_of(CODECS[0])
    didx = c.didx
    calls = {
        "search": lambda q: didx.search(q, PARAMS),
        "search_exhaustive": lambda q: didx.search_exhaustive(q, K),
        "search_records": lambda q: didx.search_records(q, PARAMS),
        "run_stages": lambda q: didx.run_stages(q, PARAMS),
    }
    a_call, b_call = calls["search" if kind == "run_stages" else kind], calls[kind]
    x, y = c.q, c.qd
    ref_a = _bits(a_call(x))
    ref_b = b_call(y)
    ref_b = _bits(_views(ref_b) if kind == "run_stages" else ref_b)
    torch.cuda.synchronize()
    sa, sb = torch.cuda.Stream(cuda_device), torch.cuda.Stream(cuda_device)
    a_returned = threading.Event()
    out: dict = {}

    def thread_a():
        hold(sa)
        out["a_held"] = torch.cuda.Event()
        out["a_held"].record(sa)
        with torch.cuda.stream(sa):
            out["a"] = a_call(x)
        a_returned.set()

    def thread_b():
        a_returned.wait()
        with torch.cuda.stream(sb):
            out["b"] = b_call(y)
        out["a_pending"] = not out["a_held"].query()

    with _no_collection():
        _run_threads([thread_a, thread_b])
    torch.cuda.synchronize()
    assert out["a_pending"], "thread B's call returned after A's hold had ended: no overlap was tested"
    assert _same(out["a"], ref_a), "thread A's result differs from its serial run"
    got_b = _views(out["b"]) if kind == "run_stages" else out["b"]
    assert _same(got_b, ref_b), "thread B's result differs from its serial run"


@pytest.mark.gpu
def test_fastplaid_search_from_two_threads(ctx_of, hold, cuda_device):
    """FastPlaid.search on one FastPlaid from two threads, each inside its own stream: the serial lists."""
    from fast_plaid_b200.search.fast_plaid import FastPlaid

    c = ctx_of(CODECS[0])
    fp = FastPlaid.from_device_index(c.didx)
    xs = [c.queries, c.decoy_queries]
    refs = [fp.search(x, top_k=K) for x in xs]
    assert refs[0] != refs[1]
    got: list = [None, None]
    streams = [torch.cuda.Stream(cuda_device) for _ in xs]
    barrier = threading.Barrier(2)

    def worker(i):
        def run():
            barrier.wait()
            hold(streams[i])
            with torch.cuda.stream(streams[i]):
                got[i] = fp.search(xs[i], top_k=K)
        return run
    _run_threads([worker(0), worker(1)])
    torch.cuda.synchronize()
    assert got == refs


# ---- memory a DeviceIndex caches across calls -------------------------------------------------------------------
def _block_at(ptr: int) -> dict:
    """The caching allocator's block that starts at `ptr` (its size and state)."""
    for seg in torch.cuda.memory_snapshot():
        addr = seg["address"]
        for blk in seg["blocks"]:
            if addr == ptr:
                return blk
            addr += blk["size"]
    raise AssertionError(f"no allocator block starts at {ptr:#x}")


def _reuse_check(old_ptr: int, nbytes: int, check_results, device: str, tries: int = 32) -> None:
    """A cached block of `nbytes` at `old_ptr`, which work queued on a held stream still uses, has just been dropped.
    Either the allocator withholds it until that stream is done (its state is not "inactive"), or it is free at once:
    then the caller allocates that size on the default stream, with no other allocation in between, until it is given
    that block (other free blocks of the size may come first; each stays allocated), and fills it; the fill must
    survive the held stream's work.  Then `check_results()` compares the held stream's results with serial."""
    blk = _block_at(old_ptr)
    if blk["state"] == "inactive":
        mine = []
        while len(mine) < tries and (not mine or mine[-1].data_ptr() != old_ptr):
            mine.append(torch.empty(nbytes, dtype=torch.uint8, device=device))
            mine[-1].fill_(0x5A)
        if mine[-1].data_ptr() != old_ptr:
            pytest.skip(f"the allocator gave the caller {tries} other blocks: the scenario proves nothing")
        torch.cuda.synchronize(device)
        assert bool((mine[-1] == 0x5A).all()), "the caller's tensor was overwritten by work queued on the held stream"
    else:
        assert blk["state"] != "active_allocated", "the dropped buffer is still referenced: nothing was dropped"
        torch.cuda.synchronize(device)
    check_results()


@pytest.mark.gpu
@pytest.mark.parametrize("grow_on", ["same", "other"])
@pytest.mark.parametrize("kind", ["search", "search_records", "search_exhaustive"])
def test_workspace_growth_keeps_the_old_buffer_for_the_held_stream(kind, grow_on, ctx_of, hold, cuda_device):
    """The workspace is allocated on the default stream.  On held stream S a search uses it; a larger batch (on S, or
    on another stream) then grows it and drops the old one.  The caller's next allocation of the old size on the
    default stream must not be handed memory S has yet to use."""
    c = ctx_of(CODECS[0])
    didx = DeviceIndex(c.tensors, cuda_device)
    big = make_queries(4 * B, Q, dim=c.dim, seed=9, docs=c.docs).half().to(cuda_device)
    call = {"search": lambda q: didx.search(q, PARAMS), "search_records": lambda q: didx.search_records(q, PARAMS),
            "search_exhaustive": lambda q: didx.search_exhaustive(q, K)}[kind]
    other = DeviceIndex(c.tensors, cuda_device)
    ocall = {"search": lambda q: other.search(q, PARAMS), "search_records": lambda q: other.search_records(q, PARAMS),
             "search_exhaustive": lambda q: other.search_exhaustive(q, K)}[kind]
    ref_small, ref_big = _bits(ocall(c.q)), _bits(ocall(big))
    call(c.q)
    torch.cuda.synchronize()
    old_ptr, nbytes = didx._buf.data_ptr(), didx._buf.numel()
    s, s2 = torch.cuda.Stream(cuda_device), torch.cuda.Stream(cuda_device)
    hold(s)
    with torch.cuda.stream(s):
        small = call(c.q)
    with torch.cuda.stream(s if grow_on == "same" else s2):
        grown = call(big)
    assert didx._buf.numel() > nbytes

    def check():
        assert _same(small, ref_small), "the search on the held stream differs from serial"
        assert _same(grown, ref_big), "the growing search differs from serial"
    _reuse_check(old_ptr, nbytes, check, cuda_device)


@pytest.mark.gpu
def test_sharded_scratch_growth_keeps_the_old_scratch_for_the_held_stream(ctx_of, hold, cuda_device):
    """The same for the scratch of the sharded exhaustive search (`_scratch`)."""
    c = ctx_of(CODECS[0])
    didx = DeviceIndex(c.tensors, cuda_device)
    k_small, k_big = 200, 400
    comm = c.comm
    ref_small = _bits(c.didx.search_exhaustive_sharded(comm, 1, c.q, k_small))
    ref_big = _bits(c.didx.search_exhaustive_sharded(comm, 1, c.q, k_big))
    didx.search_exhaustive_sharded(comm, 1, c.q, k_small)
    torch.cuda.synchronize()
    old_ptr, nbytes = didx._scratch.data_ptr(), didx._scratch.numel()
    s = torch.cuda.Stream(cuda_device)
    hold(s)
    with torch.cuda.stream(s):
        small = didx.search_exhaustive_sharded(comm, 1, c.q, k_small)
        grown = didx.search_exhaustive_sharded(comm, 1, c.q, k_big)
    assert didx._scratch.numel() > nbytes

    def check():
        assert _same(small, ref_small) and _same(grown, ref_big)
    _reuse_check(old_ptr, nbytes, check, cuda_device)


@pytest.mark.gpu
@pytest.mark.parametrize("second", ["default", "third"])
def test_a_filter_kept_alive_outlives_the_held_stream(second, ctx_of, hold, cuda_device):
    """A filter built on the default stream is searched on held stream S and then dropped by the caller; a second
    filtered search (on the default stream, or a third stream) releases what the first call kept alive.  The caller's
    next allocation of the filter's size on the default stream must not change what S reads."""
    c = ctx_of(CODECS[0])
    didx = DeviceIndex(c.tensors, cuda_device)
    n_bits = 12_000_000 + 7 * 32  # a bitmap of 1.5 MB: its own block of the allocator's large pool
    ids1 = torch.tensor(c.sets[0], dtype=torch.int64, device=cuda_device)
    ids2 = torch.tensor(c.sets[1], dtype=torch.int64, device=cuda_device)
    f2 = Filter.from_ids(ids2, n_bits, cuda_device, B)
    ref1 = _bits(didx.search(c.q, PARAMS, filter=Filter.from_ids(ids1, n_bits, cuda_device, B)))
    ref2 = _bits(didx.search(c.qd, PARAMS, filter=f2))
    f1 = Filter.from_ids(ids1, n_bits, cuda_device, B)
    torch.cuda.synchronize()
    old_ptr, nbytes = f1.bitmap.data_ptr(), f1.bitmap.numel() * 4
    s, s3 = torch.cuda.Stream(cuda_device), torch.cuda.Stream(cuda_device)
    hold(s)
    with torch.cuda.stream(s):
        r1 = didx.search(c.q, PARAMS, filter=f1)
    del f1
    with torch.cuda.stream(torch.cuda.default_stream(cuda_device) if second == "default" else s3):
        r2 = didx.search(c.qd, PARAMS, filter=f2)

    def check():
        assert _same(r1, ref1), "the search on the held stream read a filter the caller's tensor overwrote"
        assert _same(r2, ref2)
    _reuse_check(old_ptr, nbytes, check, cuda_device)


@pytest.mark.gpu
@pytest.mark.parametrize("then", ["stage_queries", "search_host"])
def test_staged_queries_are_not_overwritten_before_their_copy(then, ctx_of, hold, cuda_device):
    """stage_queries writes a cached pinned buffer and queues its copy to the device.  On a held stream, a second
    staging of the same shape (or a search_host, which writes the same buffer) must not change what the first copy
    reads: the first batch gives its own results."""
    c = ctx_of(CODECS[0])
    didx = DeviceIndex(c.tensors, cuda_device)
    ref_x = _bits(didx.search(didx.stage_queries(c.queries, K), PARAMS))
    ref_y = _bits(didx.search(didx.stage_queries(c.decoy_queries, K), PARAMS))
    torch.cuda.synchronize()
    s = torch.cuda.Stream(cuda_device)
    hold(s)
    with torch.cuda.stream(s):
        rx = didx.search(didx.stage_queries(c.queries, K), PARAMS)
        if then == "stage_queries":
            ry = didx.search(didx.stage_queries(c.decoy_queries, K), PARAMS)
        else:
            ry = didx.search_host(c.decoy_queries, PARAMS)
    torch.cuda.synchronize()
    assert _same(rx, ref_x), "the first staged batch was overwritten before its copy to the device"
    assert _same(ry, ref_y)


# ---- reach, without a GPU -----------------------------------------------------------------------------------------
def _stream_users() -> set[str]:
    """Every function of engine.py (methods as Class.name) that calls the library (`fpb_*`) and reads the current
    stream (`self._stream()` or `current_stream(...)`)."""
    path = os.path.join(os.path.dirname(engine.__file__), "engine.py")
    tree = ast.parse(open(path, encoding="utf-8").read())
    found: set[str] = set()

    def visit(node, prefix: str) -> None:
        for child in ast.iter_child_nodes(node):
            if isinstance(child, ast.ClassDef):
                visit(child, child.name + ".")
            elif isinstance(child, (ast.FunctionDef, ast.AsyncFunctionDef)):
                called = {n.func.attr for n in ast.walk(child)
                          if isinstance(n, ast.Call) and isinstance(n.func, ast.Attribute)}
                if called & {"_stream", "current_stream"} and any(a.startswith("fpb_") for a in called):
                    found.add(prefix + child.name)
    visit(tree, "")
    return found


def test_every_stream_entry_point_has_a_stream_test():
    """A new engine function that hands the caller's stream to the library fails here until it has a held-stream
    test in ENTRIES / HOST_ENTRIES or a reason in EXEMPT."""
    covered = {f for _, reached, _, _ in ENTRIES.values() for f in reached}
    covered |= {f for reached in HOST_ENTRIES.values() for f in reached}
    users = _stream_users()
    assert users, "no engine function reads the stream: the parse found nothing"
    missing = sorted(users - covered - set(EXEMPT))
    assert not missing, f"engine functions that pass the caller's stream with no stream test: {missing}"
    stale = sorted((covered | set(EXEMPT)) - users)
    assert not stale, f"listed here but no longer reading the stream in engine.py: {stale}"
