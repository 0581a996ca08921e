"""The exhaustive-search kernel (K7: full scan and list walk), `reconstruct` / `get_embeddings` and the token matrices
against the float64 reference of test_gpu_kernels.py (imported, not copied), at every codec.

Each of these kernels has a rounding contract that can be checked exactly:

  K7             score = RN_fp32( sum_q fp16 max_t (e_hat[t] . q) ), the sum exact in fixed point: every score is the
                 fp32 rounding of the exact sum of the kernel's own fp16 maxima (each obtained by a one-token query),
                 and each maximum lies in the float64 bracket of test_gpu_kernels.py;
  reconstruct    e_hat = fp16( fp32(e) / fp32(n) ), n the engine's norm table: the reference's e_hat bit for bit.
                 div_rn's remainder step does not show in it: for every fp16 e with |e| < 4 and every fp16 n in
                 [0.5, 2), fp16(RN32(e * RN32(1/n))) already equals fp16(RN32(e / n)) (checked exhaustively);
  token_scores   fp16 of the fp32 fma chain over k = 0 .. D-1 in index order (k5_token_scores_kernel): a product of
                 two fp16 values is exact in fp32, so numpy replays the chain in float32 bit for bit (`fma_chain`).
                 Every entry is also checked against the float64 bracket, which holds whatever the order of the sum.

K7 decodes 256-token tiles made of the 8-token passes of a chunk of consecutive documents, keeps the maxima of a
document that crosses a tile in a carry array and runs one 128-column block for a tile of 16 passes or fewer.
`k7_tiles` rebuilds its tile table, and the queries plant maxima on the first and last token of every tile, on the
first and last token of every document and on the tokens just outside each document.

The last tests run without a GPU: they check the two reference helpers and the reach of the length set."""

from __future__ import annotations

import dataclasses

import numpy as np
import pytest
import torch

import test_gpu_kernels as gk

gpu = pytest.mark.gpu
CODECS = [(128, 4), (128, 2), (64, 4), (64, 2), (128, 1)]
K7_DPC = (1, 4, 13, 32)  # FPB_K7_DOCS_PER_CHUNK: one document, a few, a prime number and a whole warp's worth
# gk.LENGTHS, then lengths around one tile (248 .. 257 tokens) and two (512, 513), two 2000-token documents whose
# middle tiles read and write the carry array, and empty documents at the start and the end of chunks of 4, 13 and
# 32 documents (positions 23 / 24, 25 / 26, 31 / 32, 38, and the last document)
K7_LENGTHS = gk.LENGTHS + (248, 8, 256, 0, 0, 0, 0, 257, 512, 513, 1, 0, 0, 7, 2000, 8, 9, 256, 0, 255, 257, 0)
# (Q, B): B * ceil16(Q) query rows fill one 128-row A stage exactly, or spill one 16-row group into the next stage
# (its second warpgroup has no live rows), or span three and six stages
K7_CELLS = [(1, 8), (1, 9), (16, 8), (17, 4), (32, 4), (33, 3), (64, 2), (65, 2), (100, 3), (128, 1), (129, 1),
            (256, 3)]
TS_Q = (1, 17, 33, 129, 256)


# ---- reference helpers -----------------------------------------------------------------------------------------------
def k7_tiles(lengths, dpc: int) -> list[tuple[tuple[int, int], tuple[int, int], int]]:
    """K7's tile table at `dpc` documents per chunk: a chunk is dpc consecutive documents, document d has
    ceil(len_d / 8) passes of 8 tokens (a partial pass repeats its last token), and tile t of a chunk is passes
    32t .. 32t + 31 of the chunk's passes in document order.  Per tile: (document, token) of its first token, of
    its last token, and its number of passes."""
    out = []
    for c0 in range(0, len(lengths), dpc):
        passes = [(d, 8 * k) for d in range(c0, min(c0 + dpc, len(lengths))) for k in range(-(-int(lengths[d]) // 8))]
        for p0 in range(0, len(passes), 32):
            tile = passes[p0 : p0 + 32]
            (d0, t0), (d1, t1) = tile[0], tile[-1]
            out.append(((d0, t0), (d1, min(t1 + 7, int(lengths[d1]) - 1)), len(tile)))
    return out


def fma_chain(e: np.ndarray, q: np.ndarray) -> np.ndarray:
    """float32 [T, Q]: e[t] . q[j] as k5_token_scores_kernel sums it, acc = fmaf(e[t, k], q[j, k], acc) for k = 0 ..
    D-1 from acc = +0.  e and q hold fp16 values, so each product is exact in float32 and the float32 addition
    rounds once, as the fma does."""
    e32, q32 = np.asarray(e, np.float32), np.asarray(q, np.float32)
    assert (e32.astype(np.float16) == e32).all() and (q32.astype(np.float16) == q32).all(), "fp16 values only"
    acc = np.zeros((e32.shape[0], q32.shape[0]), np.float32)
    for k in range(e32.shape[1]):
        acc += np.outer(e32[:, k], q32[:, k])
    return acc


# ---- the index and the queries ---------------------------------------------------------------------------------------
def _with_ivf(t):
    """The synthetic index with its inverted lists (every document under each of its codes), so that FastPlaid can
    search it."""
    lens = t.doc_lengths.numpy()
    doc = np.repeat(np.arange(len(lens)), lens)
    pairs = np.unique(np.stack([t.doc_codes.numpy(), doc], 1), axis=0)  # sorted by code, then document
    K = int(t.centroids.shape[0])
    return dataclasses.replace(t, ivf=torch.from_numpy(pairs[:, 1].copy()),
                               ivf_lengths=torch.bincount(torch.from_numpy(pairs[:, 0].copy()), minlength=K))


_cache: dict = {}


def _kindex(dim: int, nbits: int):
    if (dim, nbits) not in _cache:
        from fast_plaid_b200.engine import DeviceIndex

        t = _with_ivf(gk._synthetic(dim, nbits, K7_LENGTHS))
        didx = DeviceIndex(t, "cuda:0")
        _cache[dim, nbits] = (t, didx, gk._Ref(t, didx))
    return _cache[dim, nbits]


def _pool(ref) -> np.ndarray:
    """e_hat of the first and last token of every tile at every pinned chunk size, of the first and last token of
    every document and of the tokens just outside it."""
    toks = set()
    for dpc in K7_DPC:
        for (d0, t0), (d1, t1), _ in k7_tiles(ref.lens, dpc):
            toks |= {int(ref.off[d0]) + t0, int(ref.off[d1]) + t1}
    for d in range(len(ref.lens)):
        o0, o1 = int(ref.off[d]), int(ref.off[d + 1])
        if o1 > o0:
            toks |= {o0, o1 - 1} | ({o0 - 1} if o0 > 0 else set()) | ({o1} if o1 < ref.E else set())
    return ref.ehat[sorted(toks)]


def _queries(ref, Q: int, B: int) -> np.ndarray:
    """B queries of Q planted rows.  With B >= 3 query 1 has zero rows (all of them at Q = 1); with B >= 2 the last
    query is negated, its rows tilted toward the centroids' shared direction first (query 5 of
    test_gpu_kernels.test_maxsim_stage), so that every one of its maxima is negative."""
    pool = _pool(ref)
    q = np.stack([pool[(7 * Q + b * Q + np.arange(Q)) % len(pool)] for b in range(B)])
    if B >= 3:
        q[1, ::2] = 0.0
    if B >= 2:
        u = ref.ehat.mean(0)
        v = q[-1] + u / np.linalg.norm(u)
        q[-1] = -gk._f16(v / np.linalg.norm(v, axis=1, keepdims=True))
        _, _, ms = ref.maxima(q[-1])
        assert (ms[ref.lens > 0] < 0).all(), "the negated query should have a negative maximum everywhere"
    return q


def _bits(x: np.ndarray) -> np.ndarray:
    return x.view(np.uint16 if x.dtype == np.float16 else np.uint32)


# ---- K7 --------------------------------------------------------------------------------------------------------------
def _one_token_maxima(didx, q16: torch.Tensor) -> np.ndarray:
    """[B, N, Q]: the kernel's fp16 maxima, each query row run as a query of its own."""
    B, Q, D = q16.shape
    return didx.exhaustive_scores(q16.reshape(B * Q, 1, D)).cpu().numpy().reshape(B, Q, -1).transpose(0, 2, 1)


def _check_k7(ref, q: np.ndarray, scores: np.ndarray, maxima: np.ndarray, what: str) -> tuple[int, int]:
    """Every score of a non-empty document inside the bracket of its float64 maxima plus the fp32 rounding of their
    sum, every empty one Q fp16(-9999); every maximum inside its bracket, fewer than 1 % of them off m*; every score
    the fp32 rounding of the exact sum of its maxima.  Returns (maxima off m*, maxima)."""
    B, Q, _ = q.shape
    empty = ref.lens == 0
    differ = 0
    for b in range(B):
        lo, hi, ms = ref.maxima(q[b])
        assert (scores[b, empty] == np.float32(Q * gk.SENTINEL)).all(), f"{what}: query {b}: an empty document"
        slack = Q * 2.0 ** -24 * np.abs(ms[~empty]).sum(1)
        s = scores[b, ~empty].astype(np.float64)
        bad = ~((lo[~empty].sum(1) - slack <= s) & (s <= hi[~empty].sum(1) + slack))
        if bad.any():
            d = int(np.flatnonzero(~empty)[np.flatnonzero(bad)[0]])
            raise AssertionError(f"{what}: query {b}: {int(bad.sum())} scores outside their bracket, e.g. document "
                                 f"{d} ({ref.lens[d]} tokens): {scores[b, d]!r}, reference {ms[d].sum()!r}")
        m = maxima[b, ~empty].astype(np.float64)
        bad = ~((lo[~empty] <= m) & (m <= hi[~empty]))
        if bad.any():
            i, j = np.argwhere(bad)[0]
            d = int(np.flatnonzero(~empty)[i])
            raise AssertionError(f"{what}: query {b}: {int(bad.sum())} maxima outside their bracket, e.g. document "
                                 f"{d} ({ref.lens[d]} tokens), row {j}: {m[i, j]!r}, reference {ms[d, j]!r}")
        differ += int((m != ms[~empty]).sum())
    total = B * Q * int((~empty).sum())
    assert differ < 0.01 * total, f"{what}: {differ}/{total} maxima differ from m*"
    exact = maxima.astype(np.float64).sum(-1).astype(np.float32)  # a sum of <= 256 fp16 values is exact in float64
    assert np.array_equal(_bits(scores), _bits(exact)), f"{what}: a score is not the fp32 sum of the kernel's maxima"
    return differ, total


@gpu
@pytest.mark.parametrize("Q,B", K7_CELLS)
@pytest.mark.parametrize("dim,nbits", CODECS)
def test_exhaustive_scores_against_float64(dim, nbits, Q, B, cuda_device, monkeypatch):
    """Every document of the boundary index at 1, 4, 13 and 32 documents per chunk: the float64 bracket, the exact
    sum of the kernel's maxima, and the same bytes at every chunk size."""
    t, didx, ref = _kindex(dim, nbits)
    q = _queries(ref, Q, B)
    q16 = torch.from_numpy(q).half().to(cuda_device)
    outs = {}
    for dpc in K7_DPC:
        monkeypatch.setenv("FPB_K7_DOCS_PER_CHUNK", str(dpc))
        outs[dpc] = didx.exhaustive_scores(q16).cpu().numpy()
    monkeypatch.delenv("FPB_K7_DOCS_PER_CHUNK")
    what = f"({dim},{nbits}) Q={Q} B={B}"
    differ, total = _check_k7(ref, q, outs[1], _one_token_maxima(didx, q16), what)
    print(f"{what}: {differ}/{total} K7 maxima differ from m*")
    for dpc, s in outs.items():
        assert np.array_equal(_bits(s), _bits(outs[1])), f"{what}: {dpc} documents per chunk change the scores"


@gpu
@pytest.mark.parametrize("Q", [1, 17, 33])
@pytest.mark.parametrize("dim,nbits", CODECS)
def test_list_walk_returns_the_full_scan_scores(dim, nbits, Q, cuda_device, monkeypatch):
    """search_exhaustive(subset=...) on the boundary index: one list searched by queries 0, 2 and 3 (every document,
    shuffled, with repeats) and three lists of one query each (the documents around the chunk boundaries, the
    2000-token document alone, a random sample with the empty documents).  Each list's rows start on a 64-row
    boundary, so at these Q some lists start in the middle of an A stage.  Every ranking is the full scan's
    (score desc, id asc), every score its float64-checked full-scan score bit for bit, at every chunk size."""
    t, didx, ref = _kindex(dim, nbits)
    N, B = len(ref.lens), 6
    q = _queries(ref, Q, B)
    q16 = torch.from_numpy(q).half().to(cuda_device)
    every = didx.exhaustive_scores(q16).cpu().numpy()
    what = f"({dim},{nbits}) Q={Q} list walk"
    _check_k7(ref, q, every, _one_token_maxima(didx, q16), what)
    rng = np.random.default_rng(Q)
    shared = rng.permutation(np.concatenate([np.arange(N), rng.integers(0, N, 9)])).tolist()
    empties = np.flatnonzero(ref.lens == 0).tolist()
    sample = rng.permutation(rng.integers(0, N, 15).tolist() + empties).tolist()
    subset = [shared, list(range(N - 1, 19, -1)), list(shared), list(shared), [17], sample]
    for dpc in K7_DPC:
        monkeypatch.setenv("FPB_K7_DOCS_PER_CHUNK", str(dpc))
        ids, scores, counts = (x.cpu().numpy() for x in didx.search_exhaustive(q16, N, subset=subset))
        for b in range(B):
            members = sorted(set(subset[b]))
            want = sorted(members, key=lambda d: (-float(every[b, d]), d))
            n = int(counts[b])
            assert n == len(members) and ids[b, :n].tolist() == want, f"{what}, {dpc} per chunk: query {b}'s ranking"
            assert np.array_equal(_bits(scores[b, :n]), _bits(every[b, want])), \
                f"{what}, {dpc} per chunk: query {b}'s scores differ from the full scan"


# ---- reconstruct and get_embeddings ---------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dim,nbits", CODECS)
def test_reconstruct_is_bit_exact(dim, nbits, cuda_device, tmp_path):
    """Every document, the empty ones ([0, D]), duplicate and unsorted ids, and more ids than the kernel's grid
    (sm_count * 8 CTAs) so that its grid-stride loop runs more than once: e_hat bit for bit.  FastPlaid's
    get_embeddings returns the same tensors on the host; [] gives [] and an id outside the index is refused."""
    from fast_plaid_b200 import search

    t, didx, ref = _kindex(dim, nbits)
    N = len(ref.lens)
    n_sm = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    rng = np.random.default_rng(dim * 8 + nbits)
    empties = np.flatnonzero(ref.lens == 0).tolist()
    e16 = ref.ehat.astype(np.float16)
    cases = [list(range(N)), empties, [N - 1, 3, 3, 0, 17, 17, 2, N - 1, 34, 0, empties[0]],
             rng.integers(0, N, n_sm * 8 + 37).tolist()]
    for ids in cases:
        got = didx.reconstruct(ids)
        assert len(got) == len(ids)
        for i, (d, g) in enumerate(zip(ids, got)):
            o0, o1 = int(ref.off[d]), int(ref.off[d + 1])
            assert g.dtype == torch.float16 and tuple(g.shape) == (o1 - o0, dim), (d, tuple(g.shape))
        flat = torch.cat(got).cpu().numpy()
        want = np.concatenate([e16[int(ref.off[d]) : int(ref.off[d + 1])] for d in ids])
        bad = np.argwhere(_bits(flat) != _bits(want))
        assert bad.shape[0] == 0, f"{len(ids)} ids: {bad.shape[0]} elements differ from e_hat, first (row, col) " \
                                  f"{bad[0].tolist()}: {flat[tuple(bad[0])]!r} vs {want[tuple(bad[0])]!r}"
    assert didx.reconstruct([]) == []
    for ids in ([N], [-1], [0, N]):
        with pytest.raises(ValueError, match="out of range"):
            didx.reconstruct(ids)
    fp = search.FastPlaid.from_device_index(didx, index_dir=str(tmp_path))
    ids = cases[2]
    for g, h in zip(didx.reconstruct(ids), fp.get_embeddings(ids)):
        assert h.device.type == "cpu" and torch.equal(h, g.cpu())
    assert fp.get_embeddings([]) == []


# ---- token matrices --------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("Q", TS_Q)
@pytest.mark.parametrize("dim,nbits", CODECS)
def test_token_scores_are_the_fma_chain(dim, nbits, Q, cuda_device):
    """Every (query, document) pair of three queries, then repeats up to 1 200 pairs at Q <= 33 (more than the
    kernel's grid), in shuffled order: each entry the fp16 of the fp32 fma chain bit for bit and inside the float64
    bracket, rows past the document's length and every row of an empty document exactly zero.  The index's
    documents run up to 2000 tokens, far past one token step of the kernel (128 / lanes per token)."""
    t, didx, ref = _kindex(dim, nbits)
    N, B = len(ref.lens), 3
    q = _queries(ref, Q, B)
    q16 = torch.from_numpy(q).half().to(cuda_device)
    rng = np.random.default_rng(Q)
    n = 1200 if Q <= 33 else B * N
    pairs = np.concatenate([np.stack(np.meshgrid(np.arange(B), np.arange(N), indexing="ij"), -1).reshape(-1, 2),
                            np.stack([rng.integers(0, B, n - B * N), rng.integers(0, N, n - B * N)], 1)])
    pairs = rng.permutation(pairs)
    mats = didx.token_scores(q16, torch.from_numpy(pairs[:, 0].astype(np.int32)),
                             torch.from_numpy(pairs[:, 1].astype(np.int32))).cpu().numpy()
    assert mats.shape == (n, int(ref.lens.max()), Q)
    chain = [fma_chain(ref.ehat, q[b]).astype(np.float16) for b in range(B)]  # [E, Q]: every token of the index
    ts = [gk._f16(ref.ehat @ q[b].T) for b in range(B)]
    tol = [gk._tol(ts[b], np.abs(ref.ehat) @ np.abs(q[b]).T, dim) for b in range(B)]
    what = f"({dim},{nbits}) Q={Q}"
    for k, (b, d) in enumerate(pairs):
        o0, o1 = int(ref.off[d]), int(ref.off[d + 1])
        got = mats[k, : o1 - o0]
        assert not _bits(mats[k, o1 - o0 :]).any(), f"{what}: pair {k} (document {d}): a row past its length"
        bad = np.argwhere(_bits(got) != _bits(chain[b][o0:o1]))
        assert bad.shape[0] == 0, f"{what}: pair {k} (query {b}, document {d}): {bad.shape[0]} entries are not the " \
                                  f"fma chain, first (token, row) {bad[0].tolist()}"
        err = np.abs(got.astype(np.float64) - ts[b][o0:o1])
        assert (err <= tol[b][o0:o1]).all(), f"{what}: pair {k}: an entry off t* by {err.max()}"


@gpu
@pytest.mark.parametrize("dim,nbits", CODECS)
def test_search_token_scores(dim, nbits, cuda_device, tmp_path):
    """FastPlaid.search_token_scores: every matrix is token_scores of its (query, document) pair, the result equals
    the one of a shard of one (shard=(0, 1)) byte for byte, and every row's maximum lies in the float64 bracket of
    that row's m*."""
    from fast_plaid_b200 import search
    from fast_plaid_b200.engine import DeviceIndex

    t, didx, ref = _kindex(dim, nbits)
    Q, B = 33, 3
    q = _queries(ref, Q, B)
    queries = torch.from_numpy(q).float()
    plain = search.FastPlaid.from_device_index(didx, index_dir=str(tmp_path / "plain"))
    sharded = search.FastPlaid.from_device_index(DeviceIndex(t, cuda_device), index_dir=str(tmp_path / "shard"),
                                                 shard=(0, 1))
    res = plain.search_token_scores(queries, top_k=10, show_progress=False)
    res_s = sharded.search_token_scores(queries, top_k=10, show_progress=False)
    sharded.close()
    assert len(res) == len(res_s) == B
    q16 = queries.half().to(cuda_device)
    for b in range(B):
        assert len(res[b]) == len(res_s[b]) > 0, f"query {b}"
        lo, hi, _ = ref.maxima(q[b])
        docs = [d for d, _, _ in res[b]]
        want = didx.token_scores(q16, torch.full((len(docs),), b, dtype=torch.int32),
                                 torch.tensor(docs, dtype=torch.int32)).cpu()
        for k, ((d, s, m), (d2, s2, m2)) in enumerate(zip(res[b], res_s[b])):
            assert (d, s) == (d2, s2) and torch.equal(m, m2), f"query {b}, rank {k}: the shard of one differs"
            L = int(ref.lens[d])
            assert tuple(m.shape) == (Q, L) and L > 0
            assert torch.equal(m, want[k, :L].transpose(0, 1)), f"query {b}, document {d}: not its token matrix"
            row_max = m.double().amax(1).numpy()
            assert ((lo[d] <= row_max) & (row_max <= hi[d])).all(), f"query {b}, document {d}: a row maximum"


# ---- without a GPU: the reference helpers and the reach of the length set --------------------------------------------
def test_tile_table_on_hand_worked_chunks():
    # 5 tokens (one partial pass), an empty document, then a 300-token one in a chunk of its own: 32 passes + 6
    assert k7_tiles((5, 0, 300), 2) == [((0, 0), (0, 4), 1), ((2, 0), (2, 255), 32), ((2, 256), (2, 299), 6)]
    # exactly one tile, then a one-token document
    assert k7_tiles((256, 1), 1) == [((0, 0), (0, 255), 32), ((1, 0), (1, 0), 1)]
    # empty documents around two that share a tile: 2 + 32 passes, the second document crossing into tile 1
    assert k7_tiles((0, 9, 0, 255), 4) == [((1, 0), (3, 239), 32), ((3, 240), (3, 254), 2)]
    # a chunk of empty documents has no tile
    assert k7_tiles((0, 0, 3), 2) == [((2, 0), (2, 2), 1)]


def test_k7_length_set_reaches_every_tile_case():
    """Over the pinned chunk sizes, the index has tiles of 16 passes or fewer (one MMA block) and of more, documents
    that end exactly on a tile's end after a carry (the `pfx + np == p0 + 32` flush edge) and after another document
    of the same tile, chunks of <= 16, 17 .. 32 and more than 32 passes, and empty documents first and last in
    chunks.  The query cells fill, overfill by one 16-row group, and span three or more 128-row A stages."""
    lens = K7_LENGTHS
    small = big = end_carry = end_shared = 0
    totals = set()
    first_empty = last_empty = 0
    for dpc in K7_DPC:
        for (d0, t0), (d1, t1), n in k7_tiles(lens, dpc):
            small += n <= 16
            big += n > 16
            if n == 32 and t1 == lens[d1] - 1:
                end_carry += d0 == d1 and t0 > 0
                end_shared += d0 != d1
        for c0 in range(0, len(lens), dpc):
            chunk = lens[c0 : c0 + dpc]
            p = sum(-(-x // 8) for x in chunk)
            totals.add(0 if p == 0 else 1 if p <= 16 else 2 if p <= 32 else 3)
            first_empty += dpc > 1 and chunk[0] == 0
            last_empty += dpc > 1 and chunk[-1] == 0
    assert small and big and end_carry and end_shared and first_empty and last_empty
    assert {1, 2, 3} <= totals
    assert {0, 1, 7, 8, 9, 248, 255, 256, 257, 512, 513, 2000} <= set(lens)
    rows = {B * -(-Q // 16) * 16 for Q, B in K7_CELLS}
    assert 128 in rows and 144 in rows and max(rows) >= 3 * 128
    assert {Q for Q, _ in K7_CELLS} == set(gk.K5_Q)


def test_fma_chain_is_the_rounded_dot_product_when_every_partial_sum_is_exact():
    rng = np.random.default_rng(5)
    e = rng.integers(-16, 17, (40, 128)) / 16.0  # multiples of 2^-4 up to 1, and of 2^-6 up to 1: every partial
    q = rng.integers(-64, 65, (7, 128)) / 64.0   # sum a multiple of 2^-10 below 2^7, exact in 24 bits
    partial = np.cumsum(e[:, None, :] * q[None, :, :], -1)
    assert (partial.astype(np.float32) == partial).all()
    dot = e @ q.T
    got = fma_chain(e, q)
    assert got.dtype == np.float32 and np.array_equal(got, dot.astype(np.float32))
    assert np.array_equal(got.astype(np.float16), dot.astype(np.float16))


def test_fma_chain_differs_from_a_pairwise_sum():
    """2^24 + 1 + 1 - 2^24: the chain loses both ones (2^24 + 1 rounds to 2^24), a pairwise sum keeps one, the
    reversed chain keeps both (the exact sum)."""
    e = np.array([[4096.0, 1.0, 1.0, -4096.0]])
    q = np.array([[4096.0, 1.0, 1.0, 4096.0]])
    assert fma_chain(e, q)[0, 0] == 0.0
    terms = (e * q)[0].astype(np.float32)
    assert (terms[0] + terms[1]) + (terms[2] + terms[3]) == np.float32(1.0)
    assert fma_chain(e[:, ::-1], q[:, ::-1])[0, 0] == 2.0 == (e @ q.T)[0, 0]
