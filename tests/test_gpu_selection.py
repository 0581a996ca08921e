"""The selection kernels and the two-pass approximate stage on adversarial scores, against a canonical sort.

Every stage that keeps "the best few" orders by one rule (csrc/select.cuh, DESIGN §2): larger value first, then smaller
id, with -0 equal to +0.  The reference here is a plain numpy sort by that rule, `np.lexsort((ids, -values))`, and
every comparison is exact.  Each kernel is driven on its own, on inputs the test writes into the workspace (the pattern
of `_maxsim` in test_gpu_kernels.py: `run_stages(..., upto=...)` pads the queries and lays out the workspace,
`views()` gives the buffers to overwrite, `stage_fn(name, ...)()` launches one stage):

  k1b_probe (+ subset)   injected S and tile maxima: few distinct values with the n-th score shared across tiles,
                         all equal, all negative, -0/+0
  k3b_select             injected candidates and scores: the threshold bucket of the fast path holding exactly
                         2048 keys (fast) and 2049 (radix fallback) with ties straddling the cut, a dense cluster
                         with an outlier, two values, -0/+0, +-inf, +-3e38, subnormals; n in {0, R-1, R, R+1, many,
                         cand_cap} for R from 1 to 4096
  k6_rank                injected exact scores with ties, every top_k around n and past next_pow2(R)
  apply_threshold        a local list and gathered keys with ties across shards, fewer than R keys, R = 4096
  k6_merge               hand-made records with padding inside a shard's block and ties, every n_shards * R up to
                         16384 (and the refusal above it)

Then the approximate stage on adversarial centroid-score tables (multiples of 1/8 in [-4, 4], so every fp32 sum is
exact): bit for bit against the oracle, the same pruned list and ranking in every mode and at every FPB_K3_LAMBDA, and
`tau` against the estimator it documents.

Scores are never NaN here: no NaN reaches a selection (select.cuh).  Injected tables stay above the padding sentinel
-10000, where every maximum starts.
"""

from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch

import util
from oracle import plaid_oracle as po

pytestmark = pytest.mark.gpu


# ---- the canonical rule and the 64-bit key --------------------------------------------------------------------------
def _canon(values: np.ndarray, ids: np.ndarray) -> np.ndarray:
    """Positions in canonical order: larger value first, then smaller id (-0 == +0 under the comparison)."""
    return np.lexsort((ids, -np.asarray(values, dtype=np.float64)))


def _f32_key(v: np.ndarray) -> np.ndarray:
    u = np.asarray(v, dtype=np.float32).view(np.uint32).copy()
    u[(u << np.uint32(1)) == 0] = 0  # -0 -> +0
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint64)


def _rank_key(v: np.ndarray, ids: np.ndarray) -> np.ndarray:
    return (_f32_key(v) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - np.asarray(ids).astype(np.uint64))


# ---- indexes with chosen codes --------------------------------------------------------------------------------------
def _tensors(lengths, codes, K: int, dim: int = 128, nbits: int = 2, seed: int = 0):
    """IndexTensors with the given codes, random residuals and the IVF lists the codes imply."""
    from fast_plaid_b200.engine import IndexTensors

    g = torch.Generator().manual_seed(seed)
    lengths = np.asarray(lengths, dtype=np.int64)
    codes = np.asarray(codes, dtype=np.int64)
    N = len(lengths)
    cent = torch.nn.functional.normalize(torch.randn(K, dim, generator=g), dim=-1).half()
    bw = torch.sort(torch.randn(2 ** nbits, generator=g) * 0.03).values.half()
    res = torch.randint(0, 256, (len(codes), dim * nbits // 8), generator=g).to(torch.uint8)
    pairs = np.unique(codes * N + np.repeat(np.arange(N), lengths))
    ivf_lengths = np.bincount(pairs // N, minlength=K)
    return IndexTensors(nbits, cent, bw, torch.from_numpy(lengths), torch.from_numpy(codes), res,
                        torch.from_numpy(pairs % N), torch.from_numpy(ivf_lengths))


def _oracle_index(t) -> po.OracleIndex:
    return po.OracleIndex(t.nbits, t.centroids, t.bucket_weights, t.ivf, t.ivf_lengths, t.doc_codes, t.doc_residuals,
                          t.doc_lengths)


_cache: dict = {}


def _device_index(key, make, doc_id_base: int = 0):
    if key not in _cache:
        from fast_plaid_b200.engine import DeviceIndex

        t = make()
        _cache[key] = (t, DeviceIndex(t, "cuda:0", doc_id_base=doc_id_base))
    return _cache[key]


def _one_token_index(N: int, doc_id_base: int = 0):
    """N one-token documents (codes i % 16): the selection stages only need ids below N."""
    return _device_index(("one-token", N, doc_id_base),
                         lambda: _tensors(np.ones(N), np.arange(N) % 16, 16), doc_id_base)


# ---- driving single stages ------------------------------------------------------------------------------------------
def _zero_queries(B: int, Q: int) -> torch.Tensor:
    return torch.zeros((B, Q, 128), dtype=torch.float16, device="cuda:0")


def _inject_S(st: dict, S_np: np.ndarray) -> None:
    """S[:, :, :Q] = S_np, padded columns zero (as K1 writes them), tmax = the exact column maxima of every 128-row
    tile over the real rows."""
    S = st["S"]
    B, K, Qp = S.shape
    S.zero_()
    S[:, :, : S_np.shape[2]].copy_(torch.from_numpy(np.ascontiguousarray(S_np, dtype=np.float16)))
    n_tiles = st["layout"].n_tiles
    pad = torch.full((B, n_tiles * 128 - K, Qp), float("-inf"), dtype=torch.float16, device=S.device)
    st["tmax"].copy_(torch.cat([S, pad], 1).view(B, n_tiles, 128, Qp).amax(2).transpose(1, 2))


def _rank(didx, q16: torch.Tensor, params):
    """fpb_stage_rank alone on the cached workspace: (ids, scores, counts)."""
    from fast_plaid_b200.engine import _check

    B, Q, _ = q16.shape
    k = params.top_k
    buf, _ = didx.workspace(B, Q, params)
    ids = torch.empty((B, k), dtype=torch.int64, device=didx.device)
    scores = torch.empty((B, k), dtype=torch.float32, device=didx.device)
    counts = torch.empty((B,), dtype=torch.int32, device=didx.device)
    _check(didx._lib.fpb_stage_rank(didx._handle, B, Q, ctypes.byref(params), buf.data_ptr(), buf.numel(),
                                    ids.data_ptr(), scores.data_ptr(), counts.data_ptr(), didx._stream()))
    torch.cuda.synchronize()
    return ids.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy()


# =====================================================================================================================
# k1b_probe
# =====================================================================================================================
PROBE_KINDS = ("shared n-th", "all equal", "all negative", "-0/+0")


def _probe_tables(K: int, Q: int, rng) -> np.ndarray:
    """[4, K, Q] fp16, one table per PROBE_KINDS entry, drawn per column."""
    out = np.empty((4, K, Q), dtype=np.float16)
    for q in range(Q):
        # few distinct values; 4 centroids at 2.0 and 200 at 1.0 spread over every tile: the n-th best of n = 1 is a
        # 4-way tie, of n = 8 and 32 a 200-way tie
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
    def make():
        rng = np.random.default_rng(K)
        return _tensors(np.full(50, 4), rng.integers(0, K, 200), K)

    return _device_index(("probe", K), make)


@pytest.mark.parametrize("n_probe", [1, 8, 32])
@pytest.mark.parametrize("K", [1000, 2048])
def test_probe_canonical_top_n(K, n_probe, cuda_device):
    """Per (query, token) the n best centroids in rank order, with the tile pruning of pass 1 on tables where the
    n-th score is shared by centroids of many tiles (K = 1000: a partial last tile)."""
    from fast_plaid_b200.engine import DeviceIndex

    t, didx = _probe_index(K)
    params = DeviceIndex.make_params(10, 64, n_probe)
    for Q in (1, 20, 32):
        S_np = _probe_tables(K, Q, np.random.default_rng(1000 * K + 10 * n_probe + Q))
        q16 = _zero_queries(4, Q)
        st = didx.run_stages(q16, params, upto="centroid_scores")
        _inject_S(st, S_np)
        didx.stage_fn("probe", q16, params)()
        torch.cuda.synchronize()
        cells = st["cells"].cpu().numpy()
        for b, kind in enumerate(PROBE_KINDS):
            for q in range(Q):
                want = _canon(S_np[b, :, q], np.arange(K))[:n_probe]
                assert np.array_equal(cells[b, q], want), \
                    f"K={K} n={n_probe} Q={Q} {kind}: token {q}: cells {cells[b, q]} != {want}"


@pytest.mark.parametrize("n_probe", [1, 8, 32])
@pytest.mark.parametrize("K", [1000, 2048])
def test_probe_subset_canonical_top_n(K, n_probe, cuda_device):
    """The subset probe: the n = min(n_probe, #centroids of the subset's documents) best of those centroids, -1
    after them; S is overwritten after the subset stage built the centroid list."""
    from fast_plaid_b200.engine import FPB_FLAG_SUBSET, DeviceIndex

    t, didx = _probe_index(K)
    rng = np.random.default_rng(7 * K + n_probe)
    subset = [sorted(rng.choice(50, 10, replace=False).tolist()), [int(rng.integers(50))],
              sorted(rng.choice(50, 12, replace=False).tolist()), list(range(50))]
    params = DeviceIndex.make_params(10, 64, n_probe)
    Q = 20
    S_np = _probe_tables(K, Q, rng)
    q16 = _zero_queries(4, Q)
    st = didx.run_stages(q16, params, upto="subset", subset=subset)
    _inject_S(st, S_np)
    didx.stage_fn("probe", q16, DeviceIndex.with_flags(params, FPB_FLAG_SUBSET))()
    torch.cuda.synchronize()
    cells = st["cells"].cpu().numpy()
    codes, offs = t.doc_codes.numpy(), np.concatenate([[0], np.cumsum(t.doc_lengths.numpy())])
    for b, kind in enumerate(PROBE_KINDS):
        cset = np.unique(np.concatenate([codes[offs[d] : offs[d + 1]] for d in subset[b]]))
        n = min(n_probe, len(cset))
        for q in range(Q):
            want = cset[_canon(S_np[b, cset, q], cset)[:n]]
            assert np.array_equal(cells[b, q, :n], want) and (cells[b, q, n:] == -1).all(), \
                f"K={K} n={n_probe} {kind}: token {q}: cells {cells[b, q]} != {want}"


# =====================================================================================================================
# k3b_select
# =====================================================================================================================
SELECT_N = 300_000  # cand_cap of the selection index


def _bucket_row(R: int, m: int, rng) -> np.ndarray:
    """min 0 and max 2047, so the fast path's scale is exactly 1 and a value's bucket is its floor.  Bucket 1000 holds
    m keys (three values, a third each) and is the threshold bucket: 1 + R // 2 values lie above it (the max and
    values in [1001, 2046]), so R - 1 - R // 2 of its keys are taken and the cut falls inside a run of equal values."""
    above = 1 + (R // 2 if R >= 3 else 0)
    vals = np.concatenate([
        [2047.0], rng.integers(1001 * 8, 2046 * 8, above - 1) / 8,
        1000 + np.array([1, 4, 7])[np.arange(m) % 3] / 8,
        [0.0], rng.integers(8, 999 * 8, 3000) / 8,
    ]).astype(np.float32)
    return rng.permutation(vals)


def _select_rows(R: int, rng) -> list[tuple[str, np.ndarray]]:
    many = 20_000
    rows = [(f"uniform n={n}", (rng.random(n) * 100).astype(np.float32)) for n in (0, R - 1, R, R + 1, 50_000)]
    rows.append(("n=cand_cap, ties", (rng.integers(-500, 500, SELECT_N) / 8).astype(np.float32)))
    if R >= 2:
        rows += [("threshold bucket of 2048 keys (fast path)", _bucket_row(R, 2048, rng)),
                 ("threshold bucket of 2049 keys (radix path)", _bucket_row(R, 2049, rng))]
    cluster = (1 + rng.integers(0, 64, many) * 2.0 ** -20).astype(np.float32)
    cluster[rng.integers(many)] = 1e6
    f32 = lambda *v: np.array(v, dtype=np.float32)  # noqa: E731
    inf = (rng.normal(size=5000) * 3).astype(np.float32)
    inf[rng.permutation(5000)[:40]] = np.repeat(f32(np.inf, -np.inf), 20)
    rows += [
        ("dense cluster and one outlier", cluster),
        ("two values", rng.choice(f32(0.5, 1.5), 5000, p=[0.7, 0.3])),
        ("mixed sign, -0/+0", rng.choice(f32(-1.0, -0.0, 0.0, 0.5), 5000, p=[0.3, 0.3, 0.3, 0.1])),
        ("+-inf", inf),
        ("+-3e38 (range overflows)", rng.choice(f32(-3e38, -1e38, 0.0, 1e38, 3e38), 5000)),
        ("near 3e38 (range < 3e38)", rng.choice(np.linspace(1e38, 3.2e38, 20).astype(np.float32), 5000)),
        ("subnormals", (rng.integers(-50, 50, 5000) * 2.0 ** -149).astype(np.float32)),
    ]
    return rows


@pytest.mark.parametrize("R", [1, 2, 3, 1000, 1024, 1025, 4096])
def test_select_canonical_top_r(R, cuda_device):
    """K3b: the R best candidates by (score desc, candidate index asc) -- doc id order, the candidates ascending and
    non-contiguous -- with their scores, in rank order; when n <= R, the list in candidate order.  Slots past n_cand
    hold NaN and -1, so a read past the row's candidates shows."""
    from fast_plaid_b200.engine import DeviceIndex

    t, didx = _one_token_index(SELECT_N)
    rng = np.random.default_rng(R)
    rows = _select_rows(R, rng)
    B = len(rows)
    params = DeviceIndex.make_params(10, 4 * R, 1)
    q16 = _zero_queries(B, 1)
    st = didx.run_stages(q16, params, upto="centroid_scores")
    cap = st["layout"].cand_cap
    assert st["layout"].R == R and cap == SELECT_N
    approx = np.full((B, cap), np.nan, dtype=np.float32)
    cand = np.full((B, cap), -1, dtype=np.int32)
    for b, (_, v) in enumerate(rows):
        approx[b, : len(v)] = v
        cand[b, : len(v)] = np.arange(cap) if len(v) == cap else np.sort(rng.choice(cap, len(v), replace=False))
    st["approx"].copy_(torch.from_numpy(approx))
    st["cand"].copy_(torch.from_numpy(cand))
    st["n_cand"].copy_(torch.tensor([len(v) for _, v in rows], dtype=torch.int32))
    didx.stage_fn("select", q16, params)()
    torch.cuda.synchronize()
    n_rr, rr, ra = (st[k].cpu().numpy() for k in ("n_rerank", "rerank", "rerank_approx"))
    for b, (name, v) in enumerate(rows):
        n = len(v)
        take = np.arange(n) if n <= R else _canon(v, np.arange(n))[:R]
        r = len(take)
        assert n_rr[b] == r, f"R={R} {name}: n_rerank {n_rr[b]} != {r}"
        assert np.array_equal(rr[b, :r], cand[b, take]), f"R={R} {name}: pruned list differs"
        assert np.array_equal(ra[b, :r].view(np.uint32), v[take].view(np.uint32)), f"R={R} {name}: scores differ"


# =====================================================================================================================
# k6_rank
# =====================================================================================================================
@pytest.mark.parametrize("R", [1, 37, 1024, 4096])
def test_rank_canonical_order(R, cuda_device):
    """K6 on an index with doc_id_base != 0: (exact desc, id asc), ids offset by the base, then -1 / -inf up to
    top_k; counts = min(top_k, n_rerank).  Exact scores tie heavily (and mix -0 and +0); n_rerank in {R, R - 1, 0,
    1, R // 2}; top_k in {1, n - 1, n, n + 5, past next_pow2(R)}."""
    from fast_plaid_b200.engine import DeviceIndex

    base = 1000
    N = 5000
    t, didx = _one_token_index(N, doc_id_base=base)
    rng = np.random.default_rng(R)
    n_rr = np.array([R, R - 1, 0, 1, R // 2])
    B = len(n_rr)
    rerank = np.stack([rng.choice(N, R, replace=False) for _ in range(B)]).astype(np.int32)
    exact = (rng.integers(-6, 7, (B, R)) / 4).astype(np.float32)
    exact[4] = rng.choice(np.array([-0.0, 0.0, -0.25], dtype=np.float32), R)
    for b in range(B):  # never read
        rerank[b, n_rr[b]:] = -1
        exact[b, n_rr[b]:] = np.nan
    p2 = 1 << (R - 1).bit_length()
    for top_k in sorted({1, max(R - 1, 1), R, R + 5, 2 * p2 + 1}):
        params = DeviceIndex.make_params(top_k, 4 * R, 1)
        q16 = _zero_queries(B, 1)
        st = didx.run_stages(q16, params, upto="centroid_scores")
        st["rerank"].copy_(torch.from_numpy(rerank))
        st["exact"].copy_(torch.from_numpy(exact))
        st["n_rerank"].copy_(torch.from_numpy(n_rr.astype(np.int32)))
        ids, scores, counts = _rank(didx, q16, params)
        for b in range(B):
            n = int(n_rr[b])
            order = _canon(exact[b, :n], rerank[b, :n])
            cnt = min(top_k, n)
            want_ids = np.full(top_k, -1, dtype=np.int64)
            want_sc = np.full(top_k, -np.inf, dtype=np.float32)
            want_ids[:cnt] = base + rerank[b, order[:cnt]]
            want_sc[:cnt] = exact[b, order[:cnt]]
            what = f"R={R} top_k={top_k} n={n}"
            assert counts[b] == cnt, f"{what}: count {counts[b]} != {cnt}"
            assert np.array_equal(ids[b], want_ids), f"{what}: ids differ"
            assert np.array_equal(scores[b], want_sc), f"{what}: scores differ"


# =====================================================================================================================
# apply_threshold
# =====================================================================================================================
@pytest.mark.parametrize("R", [37, 1000, 4096])
@pytest.mark.parametrize("n_shards", [1, 2, 3, 4])
def test_apply_threshold_keeps_entries_at_or_above_the_global_rth_key(n_shards, R, cuda_device):
    """The shard threshold through DeviceIndex.shard_exact_records: from gathered keys [n_shards, B, R] (key 0 =
    padding) the R-th best key T of the query; this shard's list keeps, in its original order, the entries whose key
    is >= T (T = 0 when the shards hold fewer than R keys: everything is kept).  Rows: approximate scores tied across
    shards, fewer than R keys in total, a local list shorter than R, distinct scores.  R = 4096 fills the kernel's
    four entries per thread exactly."""
    from fast_plaid_b200.engine import DeviceIndex

    N = 5000
    t, didx = _one_token_index(N)
    rank = n_shards // 2
    rng = np.random.default_rng(10 * R + n_shards)
    B = 4
    keys = np.zeros((n_shards, B, R), dtype=np.uint64)
    local_ids = np.full((B, R), -1, dtype=np.int32)
    local_ap = np.full((B, R), np.nan, dtype=np.float32)
    n_old = np.zeros(B, dtype=np.int32)
    for b in range(B):
        for s in range(n_shards):
            n = {0: R, 1: R // (n_shards + 1), 2: R if s != rank else R // 3 + 1, 3: R}[b]
            ap = ((rng.integers(0, 8, n) / 4) if b in (0, 2) else rng.normal(size=n)).astype(np.float32)
            ids = rng.choice(N, n, replace=False)
            keys[s, b, :n] = _rank_key(ap, s * 100_000 + ids)  # global ids: shard s holds [s * 100000, ...)
            if s == rank:
                n_old[b] = n
                local_ids[b, :n] = ids
                local_ap[b, :n] = ap
    params = DeviceIndex.make_params(10, 4 * R, 1)
    q16 = _zero_queries(B, 1)
    st = didx.run_stages(q16, params, upto="centroid_scores")
    st["rerank"].copy_(torch.from_numpy(local_ids))
    st["rerank_approx"].copy_(torch.from_numpy(local_ap))
    st["n_rerank"].copy_(torch.from_numpy(n_old))
    all_keys = torch.from_numpy(keys.view(np.int64)).to(cuda_device)
    didx.shard_exact_records(all_keys, rank, 1, params)
    torch.cuda.synchronize()
    buf, lay = didx.workspace(B, 1, params)
    v = didx.views(buf, lay)
    n_new, rr, ra = (v[k].cpu().numpy() for k in ("n_rerank", "rerank", "rerank_approx"))
    for b in range(B):
        T = np.sort(keys[:, b].ravel())[::-1][R - 1]
        mine = keys[rank, b, : n_old[b]]
        keep = np.flatnonzero((mine != 0) & (mine >= T))
        what = f"n_shards={n_shards} R={R} row {b}"
        assert n_new[b] == len(keep), f"{what}: {n_new[b]} entries kept, expected {len(keep)}"
        assert np.array_equal(rr[b, : len(keep)], local_ids[b, keep]), f"{what}: kept ids differ"
        assert np.array_equal(ra[b, : len(keep)], local_ap[b, keep]), f"{what}: kept scores differ"


# =====================================================================================================================
# k6_merge
# =====================================================================================================================
REC = np.dtype([("approx", "<f4"), ("exact", "<f4"), ("doc_id", "<i8")])


@pytest.mark.parametrize("n_shards,R", [(1, 1), (1, 4096), (2, 3), (2, 4096), (3, 1000), (3, 4096), (4, 1024),
                                        (4, 4096), (5, 3000), (8, 1), (8, 1000), (8, 2048)])
def test_merge_equals_host_rule(n_shards, R, cuda_device):
    """fpb_merge_shards on hand-made records: the R best by (approx desc, id asc), ordered by (exact desc, id asc).
    Padding records (id -1, approx -inf) sit inside the shards' blocks; approximate and exact scores tie across
    shards.  Row 1 holds fewer than R valid records.  4 x 4096 and 8 x 2048 are the largest merges."""
    t, didx = _one_token_index(5000)
    rng = np.random.default_rng(n_shards * 10_000 + R)
    B = 3
    rec = np.zeros((n_shards, B, R), dtype=REC)
    rec["approx"] = rng.integers(0, 6, rec.shape) / 2
    rec["exact"] = rng.integers(0, 6, rec.shape) / 2
    rec["doc_id"] = np.arange(n_shards)[:, None, None] * 1_000_000 + np.stack(
        [np.stack([rng.permutation(R) for _ in range(B)]) for _ in range(n_shards)])
    pad = np.zeros(rec.shape, dtype=bool)
    pad[:, 1] = rng.random((n_shards, R)) < 0.9
    pad[:, 2] = rng.random((n_shards, R)) < 0.2
    rec["approx"][pad] = -np.inf
    rec["exact"][pad] = -np.inf
    rec["doc_id"][pad] = -1
    top_k = R + 3
    ids, scores, counts = didx.merge_records(torch.from_numpy(rec.view(np.uint8).reshape(n_shards, B, R, 16))
                                             .to(cuda_device), top_k)
    ids, scores, counts = ids.cpu().numpy(), scores.cpu().numpy(), counts.cpu().numpy()
    for b in range(B):
        valid = rec[:, b][rec[:, b]["doc_id"] >= 0]
        want = util.merge_records_host([(float(r["approx"]), float(r["exact"]), int(r["doc_id"])) for r in valid], R,
                                       top_k)
        cnt = len(want)
        assert counts[b] == cnt, f"{n_shards}x{R} row {b}: count {counts[b]} != {cnt}"
        assert ids[b, :cnt].tolist() == [d for d, _ in want], f"{n_shards}x{R} row {b}: ids differ"
        assert scores[b, :cnt].tolist() == [s for _, s in want], f"{n_shards}x{R} row {b}: scores differ"
        assert (ids[b, cnt:] == -1).all() and (scores[b, cnt:] == -np.inf).all(), f"{n_shards}x{R} row {b}: tail"


def test_merge_refuses_more_than_16384_records_per_query(cuda_device):
    from fast_plaid_b200.engine import FPB_ERR_UNSUPPORTED, MERGE_MAX_RECORDS

    t, didx = _one_token_index(5000)
    n_shards, B, R = 8, 1, 4096
    assert n_shards * R > MERGE_MAX_RECORDS
    rec = torch.zeros((n_shards, B, R, 16), dtype=torch.uint8, device=cuda_device)
    out = [torch.empty((B, 10), dtype=torch.int64, device=cuda_device),
           torch.empty((B, 10), dtype=torch.float32, device=cuda_device),
           torch.empty((B,), dtype=torch.int32, device=cuda_device)]
    rc = didx._lib.fpb_merge_shards(rec.data_ptr(), n_shards, B, R, 10, *(o.data_ptr() for o in out),
                                    didx._stream())
    assert rc == FPB_ERR_UNSUPPORTED
    assert "exceed" in didx._lib.fpb_last_error().decode()
    with pytest.raises(ValueError, match="8\\*4096 records per query exceed the 16384"):
        didx.merge_records(rec, 10)


# =====================================================================================================================
# The approximate stage on adversarial S, against the oracle
# =====================================================================================================================
APPROX_K = 1024
RESERVED = [tile * 128 + 127 for tile in range(APPROX_K // 128)]  # one unused centroid per tile (the redo table)
EMPTY = list(range(900, 932))  # unused: a query that probes only these has no candidate
TOP_CODES = [10, 300, 520, 700, 1000]  # the codes of document 0 and of no other document
APPROX_N = 600
N_PROBE = 16
N_FULL = 400  # R = 100
TABLES = ("quantized", "one column constant", "all negative", "-0/+0", "one document far above", "redo",
          "no candidate")


def _approx_index():
    def make():
        rng = np.random.default_rng(5)
        lengths = rng.integers(1, 41, APPROX_N)
        lengths[0] = len(TOP_CODES)
        usable = np.setdiff1d(np.arange(APPROX_K), RESERVED + EMPTY + TOP_CODES)
        codes = np.concatenate([TOP_CODES, rng.choice(usable, int(lengths[1:].sum()))])
        return _tensors(lengths, codes, APPROX_K, seed=5)

    t, didx = _device_index("approx", make)
    if "oracle" not in _cache:
        _cache["oracle"] = _oracle_index(t)
    return t, didx, _cache["oracle"]


def _approx_tables(Q: int, rng) -> np.ndarray:
    """[7, K, Q] fp16 multiples of 1/8 in [-4, 4], one per TABLES entry."""
    K = APPROX_K
    q8 = lambda lo, hi: rng.integers(lo, hi + 1, (K, Q)) / 8  # noqa: E731  multiples of 1/8 in [lo/8, hi/8]
    out = np.stack([q8(-8, 8) for _ in TABLES])
    out[1, :, 0] = 0.5
    out[2] = -q8(1, 32)
    out[3] = rng.choice([-0.0, 0.0, -0.125, 0.125, 0.25], (K, Q), p=[0.35, 0.35, 0.1, 0.1, 0.1])
    out[4, TOP_CODES] = 4.0
    out[5, RESERVED] = 4.0  # every tile's maximum: the tau floor is above every value a document can sample
    out[6, EMPTY] = 4.0  # the N_PROBE best centroids of every token have empty IVF lists
    return out.astype(np.float16)


def _approx_run(didx, q16, params, S_np, subset=None) -> dict:
    """Centroid scores (+ subset), then S and tmax overwritten, then probe .. maxsim stage by stage and the rank;
    copies of every intermediate."""
    from fast_plaid_b200.engine import FPB_FLAG_SUBSET, DeviceIndex

    st = didx.run_stages(q16, params, upto="subset" if subset else "centroid_scores", subset=subset)
    if subset:
        params = DeviceIndex.with_flags(params, FPB_FLAG_SUBSET)
    _inject_S(st, S_np)
    for name in ("probe", "candidates", "approx", "select", "maxsim"):
        didx.stage_fn(name, q16, params)()
    ids, scores, counts = _rank(didx, q16, params)
    out = {k: v.cpu().clone() for k, v in st.items() if isinstance(v, torch.Tensor) and k != "workspace"}
    out.update(ids=ids, scores=scores, counts=counts, R=st["layout"].R)
    return out


def _tau_reference(t, S_b: np.ndarray, cand: np.ndarray, Qp: int, lam: float) -> np.ndarray:
    """k3_tau's estimator: the sample is candidates cand[j * n / ns], j < ns = min(n, 64), with every token's row;
    per column the want-th largest sampled value counted with multiplicity, want = max(1, rint(lam * ns)); -inf when
    fewer values were sampled, +inf on padded columns."""
    n = len(cand)
    ns = min(n, 64)
    want = max(1, int(np.rint(np.float32(lam) * np.float32(ns))))
    offs = np.concatenate([[0], np.cumsum(t.doc_lengths.numpy())])
    codes = t.doc_codes.numpy()
    docs = [int(cand[j * n // ns]) for j in range(ns)]
    rows = np.concatenate([codes[offs[d] : offs[d + 1]] for d in docs]) if docs else np.zeros(0, dtype=np.int64)
    Q = S_b.shape[1]
    tau = np.full(Qp, np.inf)
    for q in range(Q):
        vals = np.sort(S_b[rows, q].astype(np.float64))[::-1]
        tau[q] = vals[want - 1] if len(vals) >= want else -np.inf
    return tau


@pytest.mark.parametrize("Q,with_subset", [(20, False), (32, False), (100, False), (256, False), (32, True)])
def test_approx_stage_on_adversarial_tables(Q, with_subset, cuda_device, monkeypatch):
    """Seven tables (TABLES), one per query of the batch, at Qp = 32, 128, 256 (full and padded query tiles):
      1. EXACT_ALL against the oracle fed the same S: cells, candidates, approximate scores, the pruned list and its
         scores bit for bit, the final ranking consistent with the oracle's exact scores;
      2. DIRECT, TWO_PASS and EXACT_ALL at FPB_K3_LAMBDA in {0.5, 2, 8, 64}: the same pruned list, scores, ids and
         ranking everywhere; every two-pass run keeps ub >= exact, resolved or refined entries exact, unrefined upper
         bounds below T and at least R candidates at or above T;
      3. tau at FPB_K3_LAMBDA = 2 equal to its estimator (_tau_reference), the redo table included."""
    from fast_plaid_b200.engine import (FPB_FLAG_APPROX_DIRECT, FPB_FLAG_APPROX_EXACT_ALL, FPB_FLAG_APPROX_TWO_PASS,
                                        DeviceIndex)

    t, didx, oidx = _approx_index()
    rng = np.random.default_rng(Q + 1000 * with_subset)
    B = len(TABLES)
    S_np = _approx_tables(Q, rng)
    queries = torch.nn.functional.normalize(torch.randn(B, Q, 128, generator=torch.Generator().manual_seed(Q)), dim=-1)
    q16 = queries.half().to(cuda_device)
    subset = [sorted(rng.choice(APPROX_N, 150, replace=False).tolist()) for _ in range(B)] if with_subset else None
    params = DeviceIndex.make_params(N_FULL // 4, N_FULL, N_PROBE)

    runs = {}
    for lam in ("0.5", "2", "8", "64"):
        monkeypatch.setenv("FPB_K3_LAMBDA", lam)
        for mode, flag in (("exact_all", FPB_FLAG_APPROX_EXACT_ALL), ("two_pass", FPB_FLAG_APPROX_TWO_PASS)):
            runs[mode, lam] = _approx_run(didx, q16, DeviceIndex.with_flags(params, flag), S_np, subset)
    runs["direct", None] = _approx_run(didx, q16, DeviceIndex.with_flags(params, FPB_FLAG_APPROX_DIRECT), S_np, subset)
    ref_run = runs["exact_all", "2"]
    R = ref_run["R"]
    Qp = ref_run["S"].shape[2]

    for b, table in enumerate(TABLES):
        what = f"Q={Q}{' subset' if subset else ''} {table}"
        # ---- 1. against the oracle ----
        ref = po.search_one(queries[b], oidx, N_PROBE, 2000, N_FULL, 10**9,
                            subset=torch.tensor(subset[b]) if subset else None, ties="canonical", return_stages=True,
                            inject={"S": torch.from_numpy(S_np[b])})
        cells = ref_run["cells"][b].long()
        if subset:
            cells = torch.unique(cells[cells >= 0])
            assert torch.equal(cells, ref["cells"]), f"{what}: probed cells differ"
        else:
            assert torch.equal(cells.flatten(), ref["probe_cells"]), f"{what}: probed cells differ"
        n = int(ref_run["n_cand"][b])
        assert torch.equal(ref_run["cand"][b, :n].long(), ref["candidates"]), f"{what}: candidates differ"
        if table == "no candidate" and not subset:
            assert n == 0
        if n == 0:
            assert int(ref_run["n_rerank"][b]) == 0 and int(ref_run["counts"][b]) == 0, f"{what}: results without candidates"
        else:
            assert torch.equal(ref_run["approx"][b, :n], ref["approx"]), f"{what}: approximate scores differ"
            r = int(ref_run["n_rerank"][b])
            assert r == len(ref["rerank"]) and torch.equal(ref_run["rerank"][b, :r].long(), ref["rerank"]), \
                f"{what}: pruned list differs"
            approx_of = dict(zip(ref["candidates"].tolist(), ref["approx"].tolist()))
            assert ref_run["rerank_approx"][b, :r].tolist() == [approx_of[d] for d in ref["rerank"].tolist()], \
                f"{what}: scores of the pruned list differ"
            cnt = int(ref_run["counts"][b])
            assert cnt == min(params.top_k, r)
            ok, msg = util.ranking_consistent(ref_run["ids"][b, :cnt].tolist(), ref_run["scores"][b, :cnt].tolist(),
                                              dict(zip(ref["rerank"].tolist(), ref["exact"].tolist())), 1e-3)
            assert ok, f"{what}: {msg}"
        # ---- 2. every mode and lambda ----
        exact_all = ref_run["approx"][b, :n]
        r = int(ref_run["n_rerank"][b])
        for (mode, lam), run in runs.items():
            how = f"{what} {mode} lambda={lam}"
            assert torch.equal(run["cand"][b, :n], ref_run["cand"][b, :n]), f"{how}: candidates differ"
            assert int(run["n_rerank"][b]) == r, f"{how}: n_rerank differs"
            assert torch.equal(run["rerank"][b, :r], ref_run["rerank"][b, :r]), f"{how}: pruned list differs"
            assert torch.equal(run["rerank_approx"][b, :r], ref_run["rerank_approx"][b, :r]), f"{how}: scores differ"
            assert np.array_equal(run["ids"][b], ref_run["ids"][b]), f"{how}: ids differ"
            assert np.array_equal(run["scores"][b], ref_run["scores"][b]), f"{how}: final scores differ"
            if mode != "two_pass":
                assert torch.equal(run["approx"][b, :n], exact_all), f"{how}: approximate scores differ"
                continue
            ub, lb = run["approx"][b, :n], run["approx_lb"][b, :n]
            T = float(run["thresh"][b])
            assert bool((ub >= exact_all).all()), f"{how}: an upper bound is below the exact score"
            refined = torch.zeros(n, dtype=torch.bool)
            refined[run["refine"][b, : int(run["n_refine"][b])].long()] = True
            known = refined | (lb == ub)
            assert torch.equal(ub[known], exact_all[known]), f"{how}: a resolved or refined score is not exact"
            assert bool((ub[~known] < T).all()), f"{how}: an unrefined upper bound reaches T = {T}"
            if n > R:
                assert int((exact_all >= T).sum()) >= R, f"{how}: fewer than R candidates at or above T = {T}"
        # ---- 3. tau ----
        cand = ref_run["cand"][b, :n].numpy()
        want = _tau_reference(t, S_np[b], cand, Qp, 2.0)
        for mode in ("exact_all", "two_pass"):
            tau = runs[mode, "2"]["tau"][b].double().numpy()
            assert np.array_equal(tau, want), f"{what} {mode}: tau {tau[:Q]} != estimator {want[:Q]}"
