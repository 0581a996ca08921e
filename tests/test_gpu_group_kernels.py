"""The grouping kernels (csrc/groups.cu) on adversarial scores and group maps, against a canonical sort.

The rule: walking the canonical order (larger value first, then smaller id, -0 equal to +0; the key
`(f32_key(v) << 32) | (0xffffffff - id)` of test_gpu_selection.py), an entry is kept when its group is in
[0, n_groups) and fewer than m entries of its group were kept before it; the first top_k kept come back, then -1 / -inf.
The reference is that rule in numpy (`_rule`), and every comparison is exact: ids, scores as uint32 bit patterns,
counts and the tails.  Each kernel is driven on injected inputs:

  group_max + group_select  fpb_stage_group_rank (rank_groups of exact search) on scores written here: value rows with
                            the selection's threshold bucket holding 2048 keys (fast path) and 2049 (radix), all equal,
                            two values, a dense cluster with an outlier, -0/+0, +-inf, +-1.6e38 (range >= 3e38) and
                            +-1.4e38, subnormals, values one ulp apart; group maps of one group, one document per
                            group, alternating, period 3, runs across the 8-entry runs and 256-entry warps of
                            group_max, descending ids, ids outside [0, n_groups), n_groups far above the documents;
                            m in {1, 2, 3, 7, 64}; full-scan rows and list rows of n in {0, 1, cols - 1, cols}
  k6_rank_grouped           fpb_stage_rank on a grouped handle, exact / rerank / n_rerank injected, R up to 4096
  k6_merge_grouped          DeviceIndex.merge_records(groups=, n_keep=) on hand-made records up to 16384 per query

and the public exact search is checked to give the same bytes as the stage entry on the same scores.  A list row is
poisoned past n[b] with valid documents scoring +inf, so a read past the row's end changes the result instead of
faulting.  No NaN: none reaches a selection (select.cuh).  The argument checks of fpb_stage_group_rank run without a
GPU."""

from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch
from test_gpu_exhaustive import _device_index
from test_gpu_selection import REC, _canon, _one_token_index, _rank, _rank_key, _zero_queries
from util import build_oracle_index, make_docs, make_queries

from fast_plaid_b200 import engine
from fast_plaid_b200.engine import Groups

LIMITS = (1, 2, 3, 7, 64)
F32 = np.float32


# ---- the rule ---------------------------------------------------------------------------------------------------------
def _rule(values, ids, groups, n_groups: int, m: int, top_k: int | None = None):
    """(ids, scores) of the first top_k entries kept by the rule, in canonical order; scores with -0 written as +0."""
    values = np.asarray(values, dtype=F32)
    ids = np.asarray(ids, dtype=np.int64)
    groups = np.asarray(groups, dtype=np.int64)
    ok = (groups >= 0) & (groups < n_groups)
    v, d, g = values[ok], ids[ok], groups[ok]
    order = _canon(v, d)
    gs = g[order]
    by_group = np.argsort(gs, kind="stable")  # each group's entries, in canonical order
    sg = gs[by_group]
    start = np.r_[True, sg[1:] != sg[:-1]] if len(sg) else np.zeros(0, dtype=bool)
    first = np.maximum.accumulate(np.where(start, np.arange(len(sg)), 0)) if len(sg) else np.zeros(0, dtype=np.int64)
    place = np.empty(len(sg), dtype=np.int64)
    place[by_group] = np.arange(len(sg)) - first  # rank of each sorted entry within its group
    keep = order[place < m][:top_k]
    sc = v[keep].copy()
    sc[sc == 0] = 0.0
    return d[keep], sc


def _expect(got, want_ids, want_sc, top_k: int, what: str) -> None:
    """Row (ids, scores, count) of a kernel against the rule's entries, then -1 / -inf up to top_k."""
    ids, sc, count = got
    n = len(want_ids)
    wi = np.full(top_k, -1, dtype=np.int64)
    ws = np.full(top_k, -np.inf, dtype=F32)
    wi[:n] = want_ids
    ws[:n] = want_sc
    assert int(count) == n, f"{what}: count {int(count)} != {n}"
    assert np.array_equal(ids, wi), f"{what}: ids differ at {np.flatnonzero(ids != wi)[:8]}"
    assert np.array_equal(np.asarray(sc, dtype=F32).view(np.uint32), ws.view(np.uint32)), \
        f"{what}: scores differ at {np.flatnonzero(np.asarray(sc, dtype=F32).view(np.uint32) != ws.view(np.uint32))[:8]}"


def _threshold_bucket(values, top_k: int):
    """group_select's bucket search over the values of a row's non-empty keys, computed in fp32 as the device does
    (IEEE sub, mul and div, truncation): the number of keys in the threshold bucket, or None when the search does not
    run (at most top_k keys, or a range of 0 or >= 3e38)."""
    v = np.asarray(values, dtype=F32)
    if len(v) <= top_k:
        return None
    mn, mx = v.min(), v.max()
    span = F32(mx - mn)
    if not (span > 0 and span < F32(3.0e38)):
        return None
    scale = F32(2047) / span
    with np.errstate(over="ignore", invalid="ignore"):
        x = (v - mn) * scale
    bk = np.clip(np.nan_to_num(np.trunc(x), nan=0.0, posinf=2047), 0, 2047).astype(np.int64)
    hist = np.bincount(bk, minlength=2048)
    at_or_above = np.cumsum(hist[::-1])[::-1]  # count(bucket >= t)
    t = int(np.flatnonzero(at_or_above >= top_k).max())
    return int(hist[t])


def _ks(n_kept) -> list[int]:
    """top_k 1, n_kept - 1, n_kept, n_kept + 1 (every row's n_kept) and 4096, within [1, 4096]."""
    ks = {1, 4096}
    for nk in n_kept:
        ks |= {nk - 1, nk, nk + 1}
    return sorted(k for k in ks if 1 <= k <= 4096)


# ---- fpb_stage_group_rank ---------------------------------------------------------------------------------------------
def _out(B: int, k: int, device):
    return (torch.empty((B, k), dtype=torch.int64, device=device), torch.empty((B, k), dtype=torch.float32, device=device),
            torch.empty((B,), dtype=torch.int32, device=device))


def _group_rank(didx, groups: Groups, scores: np.ndarray, cand, n, top_k: int):
    """fpb_stage_group_rank on the handle of `groups`: rows of `scores` [B, cols], cand [B, cols] / n [B] or None."""
    dev = didx.device
    B, cols = scores.shape
    s = torch.from_numpy(np.ascontiguousarray(scores, dtype=F32)).to(dev)
    c = None if cand is None else torch.from_numpy(np.ascontiguousarray(cand, dtype=np.int32)).to(dev)
    nn = None if n is None else torch.from_numpy(np.asarray(n, dtype=np.int32)).to(dev)
    gk = torch.empty(B * groups.max_per_group * groups.n_groups, dtype=torch.int64, device=dev)
    ids, sc, counts = _out(B, top_k, dev)
    with didx._grouped(groups):
        engine._check(didx._lib.fpb_stage_group_rank(
            didx._handle, s.data_ptr(), None if c is None else c.data_ptr(), None if nn is None else nn.data_ptr(),
            cols, B, top_k, gk.data_ptr(), gk.numel() * 8, ids.data_ptr(), sc.data_ptr(), counts.data_ptr(),
            didx._stream()))
    torch.cuda.synchronize()
    return ids.cpu().numpy(), sc.cpu().numpy(), counts.cpu().numpy()


def _groups(gmap: np.ndarray, n_groups: int, m: int, device) -> Groups:
    """Groups built directly (Groups.from_tensor refuses negative ids): ids outside [0, n_groups) are kept."""
    return Groups(ids=torch.from_numpy(np.ascontiguousarray(gmap, dtype=np.int32)).to(device), n_groups=n_groups,
                  max_per_group=m)


# =====================================================================================================================
# group_max + group_select
# =====================================================================================================================
STAGE_N = 8192  # documents of the stage index
STAGE_BASE = 1000  # its doc_id_base: every output id is offset by it
COLS = 2601  # row length: 325 runs of 8 and a partial one, ten 256-entry warps and a part


def _value_rows(cols: int, rng) -> list[tuple[str, np.ndarray]]:
    """One row of scores per kind, none NaN."""
    f32 = lambda *v: np.array(v, dtype=F32)  # noqa: E731
    inf = (rng.normal(size=cols) * 3).astype(F32)
    inf[rng.permutation(cols)[: cols // 8]] = rng.choice(f32(np.inf, -np.inf), cols // 8)
    cluster = (1 + rng.integers(0, 64, cols) * 2.0 ** -20).astype(F32)
    cluster[rng.integers(cols)] = 1e6
    return [
        ("distinct", (rng.normal(size=cols) * 10).astype(F32)),
        ("all equal", np.full(cols, 0.75, dtype=F32)),
        ("two values", rng.choice(f32(0.5, 1.5), cols, p=[0.7, 0.3])),
        ("dense cluster and one outlier", cluster),
        ("mixed sign, -0/+0", rng.choice(f32(-1.0, -0.0, 0.0, 0.5), cols, p=[0.3, 0.3, 0.3, 0.1])),
        ("+-inf", inf),
        ("+-1.6e38 (range >= 3e38)", rng.choice(f32(-1.6e38, -1e38, 0.0, 1e38, 1.6e38), cols)),
        ("+-1.4e38 (range < 3e38)", rng.choice(np.linspace(-1.4e38, 1.4e38, 15).astype(F32), cols)),
        ("subnormals", (rng.integers(-50, 50, cols) * 2.0 ** -149).astype(F32)),
        ("one ulp apart", (F32(1.0).view(np.uint32) + rng.integers(-40, 40, cols).astype(np.uint32)).view(F32)),
    ]


def _out_of_range(g: np.ndarray, n_groups: int, rng) -> np.ndarray:
    """About 10 % of the ids replaced by -1, n_groups, n_groups + x or INT32_MAX."""
    g = g.copy()
    bad = rng.random(len(g)) < 0.1
    g[bad] = rng.choice(np.array([-1, n_groups, n_groups + 977, 2**31 - 1], dtype=np.int64), int(bad.sum()))
    return g


def _map(name: str, m: int, rng) -> tuple[np.ndarray, int]:
    """Group map of the stage index's documents: (group of every document, n_groups)."""
    N = STAGE_N
    p = np.arange(N, dtype=np.int64)
    if name == "one group":
        return np.zeros(N, dtype=np.int64), 1
    if name == "one document per group":
        return p, N
    if name == "alternating":
        return p % 2, 2
    if name == "period 3":
        return p % 3, 3
    if name.startswith("runs of "):
        r = int(name.split()[-1])
        return p // r, -(-N // r)
    if name == "descending":
        return (N - 1 - p) // 5, -(-N // 5)
    if name == "random, 10% outside [0, n_groups)":
        G = N // 6
        return _out_of_range(rng.integers(0, G, N), G, rng), G
    if name == "n_groups far above the documents":
        return p * 7 + 3, 7 * N + 11  # 7N + 11 is odd: m * n_groups is never a multiple of 1024
    if name == "sizes m - 1, m, m + 1":
        sizes = np.resize(np.array([max(m - 1, 1), m, m + 1]), N)
        return np.repeat(np.arange(N), sizes)[:N], N
    raise KeyError(name)


MAPS = ["one group", "one document per group", "alternating", "period 3", "runs of 7", "runs of 8", "runs of 9",
        "runs of 31", "runs of 32", "runs of 33", "runs of 257", "descending", "random, 10% outside [0, n_groups)",
        "n_groups far above the documents", "sizes m - 1, m, m + 1"]


def _list_rows(B: int, cols: int, valid_docs: np.ndarray, rng):
    """cand [B, cols] and n [B]: n[b] cycles through 0, 1, cols - 1, cols; even rows walk a contiguous id range from
    an offset that is not a multiple of 8 (runs keep their shape, shifted across the 8-entry boundaries), odd rows a
    random set in random order.  Past n[b]: documents of a valid group (poison, scored +inf by the caller)."""
    n = np.array([(0, 1, cols - 1, cols)[b % 4] for b in range(B)], dtype=np.int32)
    cand = np.empty((B, cols), dtype=np.int32)
    for b in range(B):
        cand[b] = 3 + 411 * b + np.arange(cols) if b % 2 == 0 else rng.choice(STAGE_N, cols, replace=False)
        cand[b, n[b]:] = rng.choice(valid_docs, cols - n[b])
    assert cand.min() >= 0 and cand.max() < STAGE_N
    return cand, n


@pytest.mark.gpu
@pytest.mark.parametrize("map_name", MAPS)
def test_group_rank_on_adversarial_rows(map_name, cuda_device):
    """fpb_stage_group_rank against the rule, for every m in {1, 2, 3, 7, 64}, on rows of every value kind
    (_value_rows), full-scan rows (cand and n NULL) and list rows (n in {0, 1, cols - 1, cols}), top_k 1, n_kept - 1,
    n_kept, n_kept + 1 and 4096, on an index whose doc_id_base is 1000."""
    t, didx = _one_token_index(STAGE_N, doc_id_base=STAGE_BASE)
    rng = np.random.default_rng(MAPS.index(map_name))
    for m in LIMITS:
        gmap, n_groups = _map(map_name, m, rng)
        if map_name == "n_groups far above the documents":
            assert (m * n_groups) % 1024 != 0 and n_groups > 7 * STAGE_N
        groups = _groups(gmap, n_groups, m, cuda_device)
        valid_docs = np.flatnonzero((gmap >= 0) & (gmap < n_groups))
        rows = _value_rows(COLS, rng)
        names = [nm for nm, _ in rows]
        vals = np.stack([v for _, v in rows])
        B = len(rows)
        cand, n = _list_rows(B, COLS, valid_docs, rng)
        list_vals = vals.copy()
        for b in range(B):
            list_vals[b, n[b]:] = np.inf  # poison: a read past n[b] ranks a +inf document first
        full_docs = np.broadcast_to(np.arange(COLS), (B, COLS))
        for form, sc, cd, nn, docs, lens in (("full scan", vals, None, None, full_docs, [COLS] * B),
                                              ("list", list_vals, cand, n, cand, n)):
            want = [_rule(sc[b, : lens[b]], docs[b, : lens[b]], gmap[docs[b, : lens[b]]], n_groups, m)
                    for b in range(B)]
            for k in _ks({len(w[0]) for w in want}):
                got = _group_rank(didx, groups, sc, cd, nn, k)
                for b in range(B):
                    what = f"{map_name} m={m} {form} n={lens[b]} top_k={k} {names[b]}"
                    _expect((got[0][b], got[1][b], got[2][b]), STAGE_BASE + want[b][0][:k], want[b][1][:k], k, what)


def _bucket_values(top_k: int, count: int, rng) -> np.ndarray:
    """Values whose min is 0 and max 2047, so the bucket scale is exactly 1 and a value's bucket is its floor.  Bucket
    1000 holds `count` values (1000 + 1/8, 4/8, 7/8, a third each), and top_k - min(top_k - 1, 1000) values lie above
    it: the threshold bucket is 1000, and the cut falls inside a run of equal values."""
    above = max(1, top_k - 1000)
    return rng.permutation(np.concatenate([
        [2047.0], rng.integers(1001 * 8, 2046 * 8, above - 1) / 8, 1000 + np.array([1, 4, 7])[np.arange(count) % 3] / 8,
        [0.0], rng.integers(8, 999 * 8, 500) / 8,
    ]).astype(F32))


@pytest.mark.gpu
@pytest.mark.parametrize("count", [2048, 2049])
def test_group_rank_threshold_bucket_of_2048_and_2049_keys(count, cuda_device):
    """group_select with its threshold bucket holding exactly 2048 keys (the fast path's capacity) and 2049 (the radix
    passes), ties straddling the cut, at top_k 3, 1500 and 4096.  Every group holds at most m documents, so every key
    is kept; documents of groups outside [0, n_groups) score +inf.  Full-scan and list rows."""
    t, didx = _one_token_index(STAGE_N, doc_id_base=STAGE_BASE)
    rng = np.random.default_rng(count)
    p = np.arange(STAGE_N)
    for label, m, gmap, n_groups in (("one document per group", 1, p, STAGE_N), ("runs of 2", 2, p // 2, STAGE_N),
                                     ("runs of 7", 7, p // 7, STAGE_N),
                                     ("runs of 64, 10% outside", 64, _out_of_range(p // 64, STAGE_N // 64, rng),
                                      STAGE_N // 64)):
        groups = _groups(gmap, n_groups, m, cuda_device)
        ok = (gmap >= 0) & (gmap < n_groups)
        for top_k in (3, 1500, 4096):
            B = 2
            kept = [_bucket_values(top_k, count, rng) for _ in range(B)]
            L = len(kept[0])
            # full scan: documents 0 .. cols - 1, the first L valid ones carrying the values
            cols = int(np.flatnonzero(np.cumsum(ok) == L)[0]) + 1
            full = np.full((B, cols), np.inf, dtype=F32)
            for b in range(B):
                full[b, ok[:cols]] = kept[b]
            # list rows: documents in a random order up to the L-th valid one, then poison
            perm = [rng.permutation(STAGE_N) for _ in range(B)]
            pos = [np.flatnonzero(ok[pm])[:L] for pm in perm]
            n = np.array([ps[-1] + 1 for ps in pos], dtype=np.int32)
            lcols = int(n.max()) + 40
            cand = np.stack([pm[:lcols] for pm in perm]).astype(np.int32)
            lst = np.full((B, lcols), np.inf, dtype=F32)
            for b in range(B):
                lst[b, pos[b]] = kept[b]
                cand[b, n[b]:] = rng.choice(np.flatnonzero(ok), lcols - n[b])
            for form, sc, cd, nn, docs, lens in (("full scan", full, None, None, np.broadcast_to(p[:cols], (B, cols)),
                                                  [cols] * B), ("list", lst, cand, n, cand, n)):
                got = _group_rank(didx, groups, sc, cd, nn, top_k)
                for b in range(B):
                    what = f"{label} top_k={top_k} {form} row {b}"
                    d = docs[b, : lens[b]]
                    assert _threshold_bucket(sc[b, : lens[b]][ok[d]], top_k) == count, what
                    want = _rule(sc[b, : lens[b]], d, gmap[d], n_groups, m, top_k)
                    assert len(want[0]) == top_k
                    _expect((got[0][b], got[1][b], got[2][b]), STAGE_BASE + want[0], want[1], top_k, what)


# =====================================================================================================================
# k6_rank_grouped
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("R", [1, 3, 1024, 1025, 4096])
def test_rank_grouped_equals_the_rule(R, cuda_device):
    """fpb_stage_rank on a grouped handle (k6_rank_grouped_kernel, ONE at m = 1, the general instance at m in {2, 7,
    64}) against the rule over the injected re-ranked list: n_rerank in {R, R - 1, 0, 1, R // 2}, heavy ties, -0/+0,
    +-inf, re-ranked documents of groups outside [0, n_groups); top_k 1, n_kept - 1, n_kept, n_kept + 1, past R and
    past next_pow2(R).  Slots past n_rerank hold valid documents scoring +inf."""
    from fast_plaid_b200.engine import DeviceIndex

    base, N = 1000, 5000
    t, didx = _one_token_index(N, doc_id_base=base)
    rng = np.random.default_rng(R)
    n_rr = np.array([R, max(R - 1, 0), 0, 1, R // 2], dtype=np.int32)
    B = len(n_rr)
    f32 = lambda *v: np.array(v, dtype=F32)  # noqa: E731
    exact = np.stack([
        (rng.integers(-6, 7, R) / 4).astype(F32),
        rng.choice(f32(-0.0, 0.0, -0.25, 0.25), R),
        rng.normal(size=R).astype(F32),
        rng.choice(f32(np.inf, -np.inf, 1.0), R),
        rng.choice(f32(np.inf, -np.inf, -0.0, 0.0, 2.0), R),
    ])
    rerank = np.stack([rng.choice(N, R, replace=False) for _ in range(B)]).astype(np.int32)
    G = max(R // 4, 1)
    p = np.arange(N)
    maps = [("random, 10% outside [0, n_groups)", _out_of_range(rng.integers(0, G, N), G, rng), G),
            ("one group", np.zeros(N, dtype=np.int64), 1), ("runs of 3", p // 3, -(-N // 3))]
    p2 = 1 << max(R - 1, 0).bit_length()
    for label, gmap, n_groups in maps:
        ok = (gmap >= 0) & (gmap < n_groups)
        rr, ex = rerank.copy(), exact.copy()
        for b in range(B):  # never read
            rr[b, n_rr[b]:] = rng.choice(np.flatnonzero(ok), R - n_rr[b])
            ex[b, n_rr[b]:] = np.inf
        for m in (1, 2, 7, 64):
            groups = _groups(gmap, n_groups, m, cuda_device)
            want = [_rule(ex[b, : n_rr[b]], rr[b, : n_rr[b]], gmap[rr[b, : n_rr[b]]], n_groups, m) for b in range(B)]
            ks = {1, R + 5, 2 * p2 + 1}
            for nk in (len(w[0]) for w in want[:2]):
                ks |= {nk - 1, nk, nk + 1}
            for k in sorted(x for x in ks if 1 <= x <= 4096 * 2 + 1):
                params = DeviceIndex.make_params(k, 4 * R, 1)
                q16 = _zero_queries(B, 1)
                st = didx.run_stages(q16, params, upto="centroid_scores")
                assert st["layout"].R == R
                st["rerank"].copy_(torch.from_numpy(rr))
                st["exact"].copy_(torch.from_numpy(ex))
                st["n_rerank"].copy_(torch.from_numpy(n_rr))
                with didx._grouped(groups):
                    ids, scores, counts = _rank(didx, q16, params)
                for b in range(B):
                    what = f"R={R} {label} m={m} top_k={k} n={n_rr[b]}"
                    _expect((ids[b], scores[b], counts[b]), base + want[b][0][:k], want[b][1][:k], k, what)


# =====================================================================================================================
# k6_merge_grouped
# =====================================================================================================================
def _merge_grouped_host(rec: np.ndarray, gl: np.ndarray, m: int, n_keep: int, top_k: int):
    """The grouped merge rule over one query's records: the n_keep best by (approx desc, id asc) among the non-padding
    ones (id >= 0), of which a record whose id is >= len(gl) or whose group is -1 takes its slot and is then dropped;
    the rest ranked by (exact desc, id asc) under the rule."""
    r = rec[rec["doc_id"] >= 0]
    r = r[_canon(r["approx"], r["doc_id"])[:n_keep]]
    d = r["doc_id"]
    g = np.where(d < len(gl), gl[np.minimum(d, len(gl) - 1)], -1)
    return _rule(r["exact"], d, g, 2**31, m, top_k)


@pytest.mark.gpu
@pytest.mark.parametrize("n_shards,R", [(1, 1), (2, 3), (3, 1000), (5, 3000), (4, 4096), (8, 2048)])
def test_merge_grouped_equals_the_host_rule(n_shards, R, cuda_device):
    """fpb_merge_shards_grouped on hand-made records: n_keep in {1, R, total - 1, total} (the prune and the no-prune
    paths), m in {1, 2, 64}, top_k 1, 37 and R + 3.  Padding records sit inside the shards' blocks (row 1 mostly
    padding); approximate and exact scores tie across shards; in row 2, records whose id is >= n_total_docs or whose
    group is -1 have the best approximate scores.  4 x 4096 and 8 x 2048 are the largest merges."""
    t, didx = _one_token_index(5000)
    rng = np.random.default_rng(n_shards * 10_000 + R)
    B, total = 3, n_shards * R
    n_total = total + 5
    rec = np.zeros((n_shards, B, R), dtype=REC)
    rec["approx"] = rng.integers(0, 6, rec.shape) / 2
    rec["exact"] = rng.choice(np.array([-0.0, 0.0, 0.5, 1.0, 1.5, -1.0], dtype=F32), rec.shape)
    rec["doc_id"] = np.arange(n_shards)[:, None, None] * R + np.stack(
        [np.stack([rng.permutation(R) for _ in range(B)]) for _ in range(n_shards)])
    G = max(total // 7, 1)
    gl = rng.integers(0, G, n_total).astype(np.int32)
    pad = np.zeros(rec.shape, dtype=bool)
    pad[:, 1] = rng.random((n_shards, R)) < 0.9
    pad[:, 2] = rng.random((n_shards, R)) < 0.2
    rec["approx"][pad] = -np.inf
    rec["exact"][pad] = -np.inf
    rec["doc_id"][pad] = -1
    live = np.argwhere(~pad[:, 2])
    bad = live[rng.permutation(len(live))[: max(2, total // 50)]]
    for j, (s, i) in enumerate(bad):
        rec["approx"][s, 2, i] = 10.0
        if j % 2 == 0:
            rec["doc_id"][s, 2, i] = n_total + j  # outside the group map: its group is never read
        else:
            gl[rec["doc_id"][s, 2, i]] = -1
    rec_t = torch.from_numpy(rec.view(np.uint8).reshape(n_shards, B, R, 16)).to(cuda_device)
    gl_t = torch.from_numpy(gl).to(cuda_device)
    for m in (1, 2, 64):
        groups = Groups(ids=gl_t, n_groups=G, max_per_group=m, global_ids=gl_t)
        for n_keep in sorted({1, R, max(total - 1, 1), total}):
            for top_k in (1, 37, R + 3):
                got = [x.cpu().numpy() for x in didx.merge_records(rec_t, top_k, groups, n_keep=n_keep)]
                for b in range(B):
                    want = _merge_grouped_host(rec[:, b].ravel(), gl, m, n_keep, top_k)
                    what = f"{n_shards}x{R} m={m} n_keep={n_keep} top_k={top_k} row {b}"
                    _expect((got[0][b], got[1][b], got[2][b]), want[0], want[1], top_k, what)


# =====================================================================================================================
# The public exact search gives the stage entry's bytes
# =====================================================================================================================
N_BASE, N_COPIES = 400, 2049

_real: dict = {}


def _real_index(device):
    """N_BASE random documents, then N_COPIES copies of one more document (equal scores for every query), and
    queries drawn from that document, so the copies score above every base document."""
    if "didx" not in _real:
        docs = make_docs(N_BASE, 4, 16, seed=500)
        copy = make_docs(1, 12, 12, seed=501)[0]
        docs = docs + [copy.clone() for _ in range(N_COPIES)]
        oidx, _ = build_oracle_index(docs, nbits=4)
        _real["didx"] = _device_index(oidx, device)
        _real["q16"] = make_queries(3, 32, seed=502, docs=[copy]).half().to(device)
    return _real["didx"], _real["q16"]


def _real_map(m: int, tied: int, rng) -> np.ndarray:
    """Base documents in ~150 groups, every copy in a group of its own, except that the first m + 1 copies share
    one when `tied` is 2048: m of them are kept, so `tied` copies reach the selection."""
    g = np.concatenate([rng.integers(0, 150, N_BASE), 150 + np.arange(N_COPIES)])
    if tied == N_COPIES - 1:
        g[N_BASE : N_BASE + m + 1] = 150
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("tied", [2048, 2049])
def test_public_exact_search_is_the_stage_bytes(tied, cuda_device):
    """search_exhaustive(groups=) == fpb_stage_group_rank on exhaustive_scores of the same queries == the rule, at
    m = 1 (the group keys inside the accumulator region) and m = 64 (after it), with top_k 1000: the threshold bucket
    of the selection is the one of the tied copies, holding `tied` keys (2048: the fast path; 2049: the radix passes).
    Then with per-query subsets (the list walk: cand and n), of different lengths, each holding every copy."""
    didx, q16 = _real_index(cuda_device)
    N = didx.num_documents
    every = didx.exhaustive_scores(q16).cpu().numpy()
    B = every.shape[0]
    rng = np.random.default_rng(tied)
    subsets = [sorted(set(rng.choice(N_BASE, 50 + 100 * b, replace=False).tolist())
                      | set(range(N_BASE, N))) for b in range(B)]
    for m in (1, 64):
        g_user = _real_map(m, tied, rng)
        groups = Groups.from_tensor(torch.from_numpy(g_user), N, cuda_device, m)
        gmap = groups.ids.cpu().numpy().astype(np.int64)
        n_groups = groups.n_groups
        assert (m * n_groups <= N) == (m == 1)  # m = 1: keys in the accumulator region; m = 64: after it
        for top_k in (1000, 4096):
            pub = [x.cpu().numpy() for x in didx.search_exhaustive(q16, top_k, groups=groups)]
            stage = _group_rank(didx, groups, every, None, None, top_k)
            for b in range(B):
                what = f"tied={tied} m={m} top_k={top_k} query {b}"
                kept, _ = _rule(every[b], np.arange(N), gmap, n_groups, m)
                if top_k == 1000:
                    assert _threshold_bucket(every[b][kept], top_k) == tied, what
                want = _rule(every[b], np.arange(N), gmap, n_groups, m, top_k)
                _expect((stage[0][b], stage[1][b], stage[2][b]), want[0], want[1], top_k, f"{what}: stage")
                _expect((pub[0][b], pub[1][b], pub[2][b]), want[0], want[1], top_k, f"{what}: search_exhaustive")
            # the list walk
            pub = [x.cpu().numpy() for x in didx.search_exhaustive(q16, top_k, subset=subsets, groups=groups)]
            cols = max(len(s) for s in subsets)
            cand = np.empty((B, cols), dtype=np.int32)
            sc = np.full((B, cols), np.inf, dtype=F32)
            n = np.array([len(s) for s in subsets], dtype=np.int32)
            for b, s in enumerate(subsets):
                cand[b, : n[b]] = s
                cand[b, n[b]:] = s[: cols - n[b]]  # poison: valid documents at +inf
                sc[b, : n[b]] = every[b, s]
            stage = _group_rank(didx, groups, sc, cand, n, top_k)
            for b, s in enumerate(subsets):
                what = f"tied={tied} m={m} top_k={top_k} query {b} subset of {len(s)}"
                want = _rule(every[b, s], np.asarray(s), gmap[s], n_groups, m, top_k)
                _expect((stage[0][b], stage[1][b], stage[2][b]), want[0], want[1], top_k, f"{what}: stage")
                _expect((pub[0][b], pub[1][b], pub[2][b]), want[0], want[1], top_k, f"{what}: search_exhaustive")


# =====================================================================================================================
# No GPU needed
# =====================================================================================================================
def test_the_host_rule():
    v = np.array([1.0, 2.0, 2.0, -0.0, 0.0, 3.0], dtype=F32)
    ids = np.array([5, 4, 3, 2, 1, 0])
    g = np.array([0, 0, 1, 1, -1, 7])
    d, s = _rule(v, ids, g, 2, 1)
    assert d.tolist() == [3, 4] and s.tolist() == [2.0, 2.0]
    d, s = _rule(v, ids, g, 2, 2)
    assert d.tolist() == [3, 4, 5, 2] and s.view(np.uint32).tolist() == np.array([2, 2, 1, 0], F32).view(np.uint32).tolist()
    assert _rule(v, ids, g, 8, 1, 2)[0].tolist() == [0, 3]
    assert _rule(v[:0], ids[:0], g[:0], 8, 3)[0].size == 0
    keys = _rank_key(v, ids)
    assert np.array_equal(np.argsort(keys, kind="stable")[::-1][:3], _canon(v, ids)[:3])
    assert _threshold_bucket(np.array([0.0, 2047.0, 1000.5, 1000.25], F32), 2) == 2
    assert _threshold_bucket(np.ones(5, F32), 2) is None
    assert _threshold_bucket(np.array([-1.6e38, 1.6e38, 0.0], F32), 1) is None


def test_stage_group_rank_refuses_bad_arguments():
    """Every refusal of fpb_stage_group_rank comes before any CUDA call: host bytes stand in for the index (a zeroed
    handle without groups) and for every device buffer, which a refused call never touches."""
    lib = engine.load_library()
    fake = torch.zeros(4096, dtype=torch.uint8)  # an index with N = 0, no groups
    gids = torch.zeros(4, dtype=torch.int32)
    buf = torch.zeros(1 << 16, dtype=torch.uint8)
    grouped, sharded = ctypes.c_void_p(), ctypes.c_void_p()
    assert lib.fpb_index_with_groups_max(ctypes.byref(grouped), fake.data_ptr(), gids.data_ptr(), 3, 2) == engine.FPB_OK
    assert lib.fpb_index_with_shard_groups(ctypes.byref(sharded), fake.data_ptr(), gids.data_ptr(), 3, 2,
                                           gids.data_ptr(), 4) == engine.FPB_OK
    P = buf.data_ptr()

    def call(ix=grouped, scores=P, cand=None, n=None, cols=16, B=2, top_k=10, gkeys=P, nbytes=2 * 2 * 3 * 8,
             ids=P, sc=P, counts=P):
        return lib.fpb_stage_group_rank(ix, scores, cand, n, cols, B, top_k, gkeys, nbytes, ids, sc, counts, None)

    def refused(rc, code, text: bytes):
        assert rc == code, (rc, lib.fpb_last_error())
        assert text in lib.fpb_last_error(), lib.fpb_last_error()

    try:
        refused(call(ix=None), engine.FPB_ERR_INVALID, b"needs an index handle with groups")
        refused(call(ix=fake.data_ptr()), engine.FPB_ERR_INVALID, b"needs an index handle with groups")
        refused(call(ix=sharded), engine.FPB_ERR_UNSUPPORTED, b"shard-grouped")
        for kw in ("scores", "gkeys", "ids", "sc", "counts"):
            refused(call(**{kw: None}), engine.FPB_ERR_INVALID, b"NULL score, key or output pointer")
        for B, cols in ((0, 16), (-1, 16), (2, 0), (2, -5)):
            refused(call(B=B, cols=cols), engine.FPB_ERR_INVALID, b"must be >= 1")
        for k in (0, -1, 4097):
            refused(call(top_k=k), engine.FPB_ERR_INVALID, b"top_k=%d must be in [1, 4096]" % k)
        refused(call(nbytes=2 * 2 * 3 * 8 - 1), engine.FPB_ERR_WORKSPACE, b"key scratch too small")
        refused(call(B=3), engine.FPB_ERR_WORKSPACE, b"key scratch too small")
        # the size check does not overflow: 2^31 - 1 queries of 64 * (2^31 - 1) keys
        big = ctypes.c_void_p()
        assert lib.fpb_index_with_groups_max(ctypes.byref(big), fake.data_ptr(), gids.data_ptr(), 2**31 - 1,
                                             64) == engine.FPB_OK
        try:
            refused(call(ix=big, B=2**31 - 1, nbytes=2**63), engine.FPB_ERR_WORKSPACE, b"key scratch too small")
        finally:
            lib.fpb_index_destroy(big)
    finally:
        lib.fpb_index_destroy(grouped)
        lib.fpb_index_destroy(sharded)
