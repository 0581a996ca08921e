"""Wide probes: `n_ivf_probe` from 33 to 4096.

Above 32 cells per query token the probe (K1b) selects block-wide and the candidate pass (K2) drops repeated cells with
a per-query centroid bitmap (kernels.h, DESIGN §7 "Wide probes").  These tests hold the wide path to the same contract as the narrow
one:

  probe          injected S and tile maxima (the adversarial tables of test_gpu_selection.py), against a canonical
                 sort, with and without a subset; n past the number of tiles and past K
  stages         cells, candidates, approximate scores, re-rank list and exact scores against the oracle given S, at
                 every codec, on a ragged batch, with and without a subset
  FastPlaid      `search` against the oracle (also filtered), a (0, 1) shard, and n = 4096 on a small index against
                 `search_exhaustive`
  nesting        the candidates at n are contained in those at n + 1
  range          [1, 4096]
  n <= 32        the same kernels as before
"""

from __future__ import annotations

import re

import numpy as np
import pytest
import torch

from util import (build_oracle_index, make_docs, make_queries, oracle_exact_scores, ranking_consistent,
                  to_index_tensors)

from oracle import plaid_oracle as po

pytestmark = pytest.mark.gpu


def _canon(values: np.ndarray, ids: np.ndarray) -> np.ndarray:
    """Positions in canonical order: larger value first, then smaller id (-0 == +0 under the comparison)."""
    return np.lexsort((ids, -np.asarray(values, dtype=np.float64)))


# ---- the probe on injected tables -----------------------------------------------------------------------------------
PROBE_KINDS = ("shared n-th", "all equal", "all negative", "-0/+0")
WIDE_N = [33, 64, 100, 1000, 4096]
_cache: dict = {}


def _probe_tables(K: int, Q: int, rng) -> np.ndarray:
    """[4, K, Q] fp16, one table per PROBE_KINDS entry, drawn per column: few distinct values (the n-th score is
    shared by centroids of many tiles), one value, negative values only, and mostly -0 / +0."""
    out = np.empty((4, K, Q), dtype=np.float16)
    for q in range(Q):
        col = rng.integers(-4, 3, K) / 4
        hot = rng.permutation(K)[:204]
        col[hot[:4]] = 2.0
        col[hot[4:]] = 1.0
        out[0, :, q] = col
        out[1, :, q] = rng.integers(-4, 5) / 8
        out[2, :, q] = -(rng.integers(1, 65, K) / 16)
        col = rng.choice(np.array([-0.0, 0.0, -0.5], dtype=np.float16), K, p=[0.45, 0.45, 0.1])
        col[rng.permutation(K)[:3]] = 0.5
        out[3, :, q] = col
    return out


def _probe_index(K: int):
    """500 documents of 8 tokens with random codes: the subset of all documents touches most of the K centroids."""
    if ("probe", K) not in _cache:
        from fast_plaid_b200.engine import DeviceIndex, IndexTensors

        rng = np.random.default_rng(K)
        g = torch.Generator().manual_seed(K)
        N, L = 500, 8
        codes = rng.integers(0, K, N * L)
        lengths = np.full(N, L)
        cent = torch.nn.functional.normalize(torch.randn(K, 128, generator=g), dim=-1).half()
        bw = torch.sort(torch.randn(4, generator=g) * 0.03).values.half()
        res = torch.randint(0, 256, (N * L, 32), generator=g).to(torch.uint8)
        pairs = np.unique(codes * N + np.repeat(np.arange(N), L))
        t = IndexTensors(2, cent, bw, torch.from_numpy(lengths), torch.from_numpy(codes), res,
                         torch.from_numpy(pairs % N), torch.from_numpy(np.bincount(pairs // N, minlength=K)))
        _cache[("probe", K)] = (t, DeviceIndex(t, "cuda:0"))
    return _cache[("probe", K)]


def _inject_S(st: dict, S_np: np.ndarray) -> None:
    """S[:, :, :Q] = S_np, padded columns zero (as K1 writes them), tmax = the column maxima of every 128-row tile."""
    S = st["S"]
    B, K, Qp = S.shape
    S.zero_()
    S[:, :, : S_np.shape[2]].copy_(torch.from_numpy(np.ascontiguousarray(S_np, dtype=np.float16)))
    n_tiles = st["layout"].n_tiles
    pad = torch.full((B, n_tiles * 128 - K, Qp), float("-inf"), dtype=torch.float16, device=S.device)
    st["tmax"].copy_(torch.cat([S, pad], 1).view(B, n_tiles, 128, Qp).amax(2).transpose(1, 2))


@pytest.mark.parametrize("n_probe", WIDE_N)
@pytest.mark.parametrize("K", [1000, 2048, 5000])
def test_probe_canonical_top_n(K, n_probe, cuda_device):
    """Per (query, token) the min(n, K) best centroids in rank order, then -1: K = 1000 and 5000 have a partial last
    tile, n = 1000 and 4096 exceed the number of tiles, and n = 4096 exceeds K."""
    from fast_plaid_b200.engine import DeviceIndex

    t, didx = _probe_index(K)
    params = DeviceIndex.make_params(10, 64, n_probe)
    for Q in (1, 20, 32, 256):
        S_np = _probe_tables(K, Q, np.random.default_rng(1000 * K + 10 * n_probe + Q))
        q16 = torch.zeros((4, Q, 128), dtype=torch.float16, device=cuda_device)
        st = didx.run_stages(q16, params, upto="centroid_scores")
        _inject_S(st, S_np)
        didx.stage_fn("probe", q16, params)()
        torch.cuda.synchronize()
        cells = st["cells"].cpu().numpy()
        m = min(n_probe, K)
        for b, kind in enumerate(PROBE_KINDS):
            for q in range(Q):
                want = _canon(S_np[b, :, q], np.arange(K))[:m]
                assert np.array_equal(cells[b, q, :m], want) and (cells[b, q, m:] == -1).all(), \
                    f"K={K} n={n_probe} Q={Q} {kind}: token {q}: cells {cells[b, q, :40]} != {want[:40]}"


@pytest.mark.parametrize("n_probe", WIDE_N)
@pytest.mark.parametrize("K", [1000, 2048, 5000])
def test_probe_subset_canonical_top_n(K, n_probe, cuda_device):
    """The subset probe: the min(n, #centroids of the subset's documents) best of those centroids, then -1, for
    subsets of a few documents, one document, and all of them."""
    from fast_plaid_b200.engine import FPB_FLAG_SUBSET, DeviceIndex

    t, didx = _probe_index(K)
    rng = np.random.default_rng(7 * K + n_probe)
    subset = [sorted(rng.choice(500, 10, replace=False).tolist()), [int(rng.integers(500))],
              sorted(rng.choice(500, 120, replace=False).tolist()), list(range(500))]
    params = DeviceIndex.make_params(10, 64, n_probe)
    codes, offs = t.doc_codes.numpy(), np.concatenate([[0], np.cumsum(t.doc_lengths.numpy())])
    for Q in (1, 20, 32, 256):
        S_np = _probe_tables(K, Q, rng)
        q16 = torch.zeros((4, Q, 128), dtype=torch.float16, device=cuda_device)
        st = didx.run_stages(q16, params, upto="subset", subset=subset)
        _inject_S(st, S_np)
        didx.stage_fn("probe", q16, DeviceIndex.with_flags(params, FPB_FLAG_SUBSET))()
        torch.cuda.synchronize()
        cells = st["cells"].cpu().numpy()
        for b, kind in enumerate(PROBE_KINDS):
            cset = np.unique(np.concatenate([codes[offs[d] : offs[d + 1]] for d in subset[b]]))
            n = min(n_probe, len(cset))
            for q in range(Q):
                want = cset[_canon(S_np[b, cset, q], cset)[:n]]
                assert np.array_equal(cells[b, q, :n], want) and (cells[b, q, n:] == -1).all(), \
                    f"K={K} n={n_probe} Q={Q} {kind}: token {q}: cells {cells[b, q, :40]} != {want[:40]}"


# ---- every stage against the oracle given S -------------------------------------------------------------------------
CODECS = [(128, 4), (64, 2), (128, 1)]
B_PARITY, Q_PARITY = 4, 32
QUERY_LENS = [32, 20, 7, 1]  # the rest of each row is zero, as FastPlaid pads a ragged list


def _parity_index(dim: int, nbits: int):
    if ("parity", dim, nbits) not in _cache:
        from fast_plaid_b200.engine import DeviceIndex

        docs = make_docs(500, 20, 80, dim=dim, seed=1234)
        oidx, _ = build_oracle_index(docs, nbits=nbits)
        didx = DeviceIndex(to_index_tensors(oidx), "cuda:0")
        queries = make_queries(B_PARITY, Q_PARITY, dim=dim, seed=4321, docs=docs)
        for b, n in enumerate(QUERY_LENS):
            queries[b, n:] = 0
        _cache[("parity", dim, nbits)] = (oidx, didx, queries)
    return _cache[("parity", dim, nbits)]


def _subsets(n_docs: int) -> list[list[int]]:
    g = torch.Generator().manual_seed(5)
    return [torch.randperm(n_docs, generator=g)[: n_docs // 10].tolist(), [int(torch.randint(0, n_docs, (1,), generator=g))],
            list(range(n_docs)), torch.randint(0, n_docs, (50,), generator=g).tolist() * 2]


@pytest.mark.parametrize("with_subset", [False, True])
@pytest.mark.parametrize("n_probe", [48, 256, 4096])
@pytest.mark.parametrize("dim,nbits", CODECS)
def test_stages_match_the_oracle(dim, nbits, n_probe, with_subset, cuda_device):
    """Given the GPU's own S: probe cells, candidates and the re-rank list exactly, approximate scores exactly (or
    within fp32 summation order); exact scores within 1e-3 relative, almost all bit-identical."""
    from fast_plaid_b200.engine import FPB_FLAG_APPROX_EXACT_ALL, DeviceIndex

    oidx, didx, queries = _parity_index(dim, nbits)
    params = DeviceIndex.make_params(10, 256, n_probe)
    subsets = _subsets(int(oidx.doc_lengths.shape[0])) if with_subset else None
    st = didx.run_stages(queries.half().to(cuda_device), DeviceIndex.with_flags(params, FPB_FLAG_APPROX_EXACT_ALL),
                         subset=subsets)
    torch.cuda.synchronize()
    assert st["layout"].n_probe == n_probe
    flips = total = 0
    for b in range(B_PARITY):
        S_b = st["S"][b, :, :Q_PARITY].cpu().contiguous()
        kw = dict(ties="canonical", return_stages=True, inject={"S": S_b})
        if with_subset:
            kw["subset"] = torch.tensor(subsets[b], dtype=torch.int64)
        ref = po.search_one(queries[b], oidx, n_probe, 2000, params.n_full_scores, params.top_k, **kw)
        cells = torch.unique(st["cells"][b].cpu().flatten().long())
        assert torch.equal(cells[cells >= 0], ref["cells"]), f"query {b}: probed cells differ"
        n = int(st["n_cand"][b])
        assert torch.equal(st["cand"][b, :n].cpu().long(), ref["candidates"]), f"query {b}: candidates differ"
        if n == 0:
            continue
        approx = st["approx"][b, :n].cpu()
        if not torch.equal(approx, ref["approx"]):
            rel = ((approx - ref["approx"]).abs() / ref["approx"].abs().clamp_min(1.0)).max()
            assert float(rel) < 1e-6, f"query {b}: approx scores differ by {float(rel)}"
            kw["inject"] = {"S": S_b, "approx": approx}
            ref = po.search_one(queries[b], oidx, n_probe, 2000, params.n_full_scores, params.top_k, **kw)
        r = int(st["n_rerank"][b])
        rer = st["rerank"][b, :r].cpu().long()
        assert torch.equal(rer, ref["rerank"]), f"query {b}: re-rank list differs"
        oracle_exact = oracle_exact_scores(oidx, queries[b], rer.tolist())
        got = st["exact"][b, :r].cpu()
        rel = (got - oracle_exact).abs() / oracle_exact.abs().clamp_min(1.0)
        assert float(rel.max()) < 1e-3, f"query {b}: exact scores off by {float(rel.max())} relative"
        flips += int((got != oracle_exact).sum())
        total += r
    assert flips / max(total, 1) < 0.05, f"{flips}/{total} exact scores not bit-identical"


@pytest.mark.parametrize("n", [32, 100])
def test_candidates_nest(n, cuda_device):
    """For one S, every candidate at n is a candidate at n + 1 (across the switch to the wide kernels at 32 -> 33)."""
    from fast_plaid_b200.engine import DeviceIndex

    oidx, didx, queries = _parity_index(128, 4)
    q16 = queries.half().to(cuda_device)
    got = []
    for m in (n, n + 1):
        st = didx.run_stages(q16, DeviceIndex.make_params(10, 256, m), upto="candidates")
        torch.cuda.synchronize()
        got.append([set(st["cand"][b, : int(st["n_cand"][b])].tolist()) for b in range(B_PARITY)])
        S = st["S"].clone()
        if m == n:
            S0 = S
    assert torch.equal(S0, S)
    for b in range(B_PARITY):
        assert got[0][b] <= got[1][b], f"query {b}: a candidate at n={n} is missing at n={n + 1}"


def test_probing_every_cell_is_exhaustive(cuda_device):
    """K <= 4096 and N <= 4096: n_ivf_probe = 4096 makes every document a candidate and n_full_scores = 4 N re-ranks
    all of them, so `search` ranks as `search_exhaustive` does, up to the last bit of a score."""
    from fast_plaid_b200.engine import DeviceIndex

    oidx, didx, queries = _parity_index(128, 4)
    N = int(oidx.doc_lengths.shape[0])
    assert didx.num_centroids <= 4096 and N <= 4096
    q16 = queries.half().to(cuda_device)
    ids, scores, counts = (x.cpu() for x in didx.search(q16, DeviceIndex.make_params(100, 4 * N, 4096)))
    e_ids, e_scores, e_counts = (x.cpu() for x in didx.search_exhaustive(q16, N))
    for b in range(B_PARITY):
        assert int(counts[b]) == 100 and int(e_counts[b]) == N
        every = dict(zip(e_ids[b].tolist(), e_scores[b].tolist()))
        ok, why = ranking_consistent(ids[b].tolist(), scores[b].tolist(), every, 1e-3)
        assert ok, f"query {b}: {why}"
        assert abs(float(scores[b, 0]) - float(e_scores[b, 0])) <= 1e-3 * max(1.0, abs(float(e_scores[b, 0])))


# ---- FastPlaid --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fastplaid_index(tmp_path_factory):
    from fast_plaid_b200 import search
    from fast_plaid_b200.index import store

    path = str(tmp_path_factory.mktemp("wide") / "idx")
    docs = make_docs(400, 20, 80, seed=11)
    fp = search.FastPlaid(path, device="cuda:0")
    fp.create(docs, kmeans_niters=4, nbits=4)
    data = store.read_index(path)
    oidx = po.OracleIndex(data.nbits, data.centroids, data.bucket_weights, data.ivf, data.ivf_lengths.long(),
                          data.doc_codes, data.doc_residuals, data.doc_lengths)
    queries = make_queries(6, 30, seed=12, docs=docs)
    yield fp, oidx, queries
    fp.close()


@pytest.mark.parametrize("n_probe", [64, 512])
def test_fastplaid_search_against_the_oracle(fastplaid_index, n_probe, cuda_device):
    fp, oidx, queries = fastplaid_index
    sub = list(range(0, 400, 7))
    for subset in (None, sub):
        res = fp.search(queries, top_k=10, n_ivf_probe=n_probe, subset=subset)
        for b in range(len(res)):
            s = None if subset is None else torch.tensor(subset, dtype=torch.int64)
            ref = po.search_one(queries[b], oidx, n_ivf_probe=n_probe, top_k=10**9, subset=s, return_stages=True)
            assert len(res[b]) == min(10, len(ref["ids"]))
            if subset is not None:
                assert {d for d, _ in res[b]} <= set(subset)
            ok, why = ranking_consistent([d for d, _ in res[b]], [s for _, s in res[b]],
                                         dict(zip(ref["ids"], ref["scores"])), 1e-3,
                                         fallback=lambda d, b=b: float(oracle_exact_scores(oidx, queries[b], [d])[0]))
            assert ok, f"n={n_probe} subset={subset is not None} query {b}: {why}"


def test_sharded_search_equals_unsharded(fastplaid_index, cuda_device):
    from fast_plaid_b200 import search
    from fast_plaid_b200.engine import DeviceIndex

    fp, oidx, queries = fastplaid_index
    sharded = search.FastPlaid.from_device_index(DeviceIndex(to_index_tensors(oidx), cuda_device), shard=(0, 1))
    try:
        for subset in (None, list(range(0, 400, 3))):
            whole = fp.search(queries, top_k=10, n_ivf_probe=256, subset=subset)
            assert sharded.search(queries, top_k=10, n_ivf_probe=256, subset=subset) == whole
    finally:
        sharded.close()


# ---- the range and the narrow path ------------------------------------------------------------------------------------
def test_range(cuda_device):
    from fast_plaid_b200.engine import DeviceIndex

    oidx, didx, queries = _parity_index(128, 4)
    assert didx.layout(4, 32, DeviceIndex.make_params(10, 256, 4096)).n_probe == 4096
    for n in (0, 4097):
        with pytest.raises(ValueError, match=re.escape("[1,4096]")):
            didx.layout(4, 32, DeviceIndex.make_params(10, 256, n))


def _kernel_names(keys) -> set[str]:
    """The *_kernel functions named in profiler keys, demangled ("(anonymous namespace)::k2_mark_kernel(int const*,
    ...)") or not ("_ZN12_GLOBAL__N_114k2_mark_kernelEPKi...").  The profiler also lists runtime activity (memsets,
    copies, lazy loading); every kernel of the library is a *_kernel function."""
    names = set()
    for key in keys:
        names.update(re.findall(r"(?<![A-Za-z0-9_])([A-Za-z]\w*_kernel)(?![A-Za-z0-9_])", key))
        for m in re.finditer(r"(?<![0-9])([0-9]+)", key):  # Itanium mangling: <length><identifier>
            ident = key[m.end() : m.end() + int(m.group(1))]
            if ident.endswith("_kernel") and re.fullmatch(r"[A-Za-z_]\w*", ident):
                names.add(ident)
    return names


MARKER = "spin_kernel"  # torch.cuda._sleep's kernel


def _kernel_runs(fns) -> list[set[str]]:
    """The library kernels each of `fns` launches.  All calls are profiled in one torch.profiler session, each between
    two torch.cuda._sleep marker kernels on the same stream, and the kernels are told apart by their start times.

    A first session, whose events are not used, runs the same calls: after a long run of other GPU work (the whole
    suite) the first profiler session has listed no device event at all while the next ones listed every kernel.
    Within one session the markers also keep any event delivered late from an earlier session out of every call's
    set."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    def run():
        torch.cuda.synchronize()
        for fn in fns:
            torch.cuda._sleep(1000)
            fn()
            torch.cuda.synchronize()
        torch.cuda._sleep(1000)
        torch.cuda.synchronize()

    with profile(activities=[ProfilerActivity.CUDA]):
        run()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
    kernels = sorted((e.time_range.start, e.name) for e in prof.events() if e.device_type == DeviceType.CUDA)
    marks = [i for i, (_, name) in enumerate(kernels) if MARKER in _kernel_names([name])]
    assert len(marks) == len(fns) + 1, f"{len(marks)} markers among the device events {[k for _, k in kernels]}"
    return [_kernel_names(name for _, name in kernels[a + 1 : b]) for a, b in zip(marks, marks[1:])]


def test_narrow_probe_runs_the_narrow_kernels(cuda_device):
    """n <= 32 launches the warp-list probe and the slot-scanning candidate pass, nothing else changes; n = 33 swaps
    exactly those two for the wide kernels."""
    from fast_plaid_b200.engine import DeviceIndex

    oidx, didx, queries = _parity_index(128, 4)
    q16 = queries.half().to(cuda_device)
    for subset in (None, _subsets(int(oidx.doc_lengths.shape[0]))):
        ns = (8, 32, 33)
        runs = _kernel_runs([lambda n=n: didx.search(q16, DeviceIndex.make_params(10, 256, n), subset=subset)
                             for n in ns])
        got = dict(zip(ns, runs))
        probe = "k1b_probe_kernel" if subset is None else "k1b_probe_subset_kernel"
        wide = "k1b_probe_wide_kernel" if subset is None else "k1b_probe_subset_wide_kernel"
        assert got[8] == got[32]
        assert {probe, "k2_mark_kernel"} <= got[32] and not any("wide" in k for k in got[32]), got[32]
        assert got[33] == (got[32] - {probe, "k2_mark_kernel"}) | {wide, "k2_mark_wide_kernel"}, got[33]
