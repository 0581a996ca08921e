"""Every centroid-score and MaxSim kernel variant against a float64 reference, at every padded query length.

The engine picks its kernel by (dim, nbits), by the padded query length Qp (16 .. 256) and by the longest document:
K1 v2 (wgmma) or K1 v1 (mma.sync) for the centroid scores S; K5 v4, K5 v5 or the generic K5 for the re-rank MaxSim.
`FPB_K1=v1` and `FPB_K5=v1` pin the alternatives, `FPB_K5_DOCS_PER_CHUNK` pins v5's chunk size; all three are read at
every launch, so the tests switch them with monkeypatch.

The reference reproduces the rounding points of the reference implementation and does everything else in float64:

  e   = fp16(w + c)                   bucket index from the oracle's integer unpacking of the packed bytes
  n*  = fp16(sqrt(sum e^2))           the norm table the engine derives at load
  ê   = fp16(fp32(e / n))             n = the engine's own norm table; a float64 quotient of two fp16 numbers rounded
                                      to fp32 is the correctly rounded fp32 quotient, so ê is bit-identical to the
                                      kernels' (IEEE division, then one rounding to fp16)
  t*  = fp16(ê . q)                   token score, dot product in float64
  S*  = fp16(C . q)                   centroid score, dot product in float64

A kernel result x is accepted against x* when |x - x*| <= ulp16(x*) + D 2^-23 sum_k |a_k b_k|: one fp16 step for a
rounding that lands on the other side of a boundary, plus a bound on fp32 accumulation noise when a dot product nearly
cancels.  A maximum over tokens is then bracketed by [max_t (t* - tol), max_t (t* + tol)] (rounding is monotone), and
a score sum_q m_q by the sums of those brackets plus Q 2^-24 sum_q |m*_q| for its fp32 running sum.  Fewer than 1 % of
the results of a cell may differ from x* at all: a kernel that rounds toward zero stays within one ulp everywhere and
is caught by that count, not by the bound.
"""

from __future__ import annotations

import os
import subprocess

import numpy as np
import pytest
import torch

import util  # noqa: F401  (puts the repository root on sys.path)
from oracle import plaid_oracle as po

pytestmark = pytest.mark.gpu

SENTINEL = -10000.0  # fp16(-9999): the score of a query token against an empty document (search.rs:395)
# token positions where a kernel's passes (8 tokens), tiles (64 / 128 tokens) and v5's pass table (2048 passes)
# start and end; the last token of every document is added per document
BOUNDARY = (0, 7, 8, 63, 64, 127, 128, 8191, 8192, 16383, 16384)
# the re-rank test index: empty documents, every length around a pass and tile boundary, one long document; the
# first and the last document are ordinary ones
LENGTHS = (5, 129, 0, 1, 2, 7, 8, 9, 15, 16, 17, 63, 64, 65, 127, 128, 300, 2000, 0, 12)
K5_Q = (1, 16, 17, 32, 33, 64, 65, 100, 128, 129, 256)
SHAPES = [(128, 4), (128, 2), (64, 4), (64, 2)]
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "fast_plaid_b200", "csrc")


# ---- float64 reference ----------------------------------------------------------------------------------------------
def _f16(x) -> np.ndarray:
    """Round to fp16 (numpy rounds float64 and float32 to nearest-even directly) and widen back to float64."""
    return np.asarray(x).astype(np.float16).astype(np.float64)


def _ulp16(x: np.ndarray) -> np.ndarray:
    """Spacing of fp16 at |x|: 2^(e-10) in the binade [2^e, 2^(e+1)), 2^-24 below the normal range."""
    _, e = np.frexp(np.maximum(np.abs(x), 2.0 ** -14))
    return np.ldexp(1.0, e - 11)


def _tol(ref: np.ndarray, absdot: np.ndarray, dim: int) -> np.ndarray:
    return _ulp16(ref) + dim * 2.0 ** -23 * absdot


class _Ref:
    """Decoded tokens of an index, in float64, with the engine's rounding points."""

    def __init__(self, t, didx):
        self.dim = int(t.centroids.shape[1])
        rev, lut = po.codec_luts(t.nbits)
        res = t.doc_residuals.long()
        bucket = lut[rev[res].long()]  # [E, D*nbits/8, 8/nbits] bucket index of every element
        E = res.shape[0]
        w = t.bucket_weights.half().double()[bucket].reshape(E, self.dim).numpy()
        c = t.centroids.half().double()[t.doc_codes.long()].numpy()
        e = _f16(w + c)
        self.sq = (e * e).sum(1)
        self.norm = _f16(np.sqrt(self.sq))
        n = didx.token_norms[:E].cpu().double().numpy()
        self.ehat = _f16((e / n[:, None]).astype(np.float32))
        self.lens = t.doc_lengths.long().numpy()
        self.off = np.concatenate([[0], np.cumsum(self.lens)])
        self.E = E

    def _segmax(self, x: np.ndarray) -> np.ndarray:
        out = np.full((len(self.lens), x.shape[1]), np.nan)
        ne = self.lens > 0
        out[ne] = np.maximum.reduceat(x, self.off[:-1][ne], axis=0)
        return out

    def maxima(self, q: np.ndarray):
        """Per document and query row: the bracket [lo, hi] of the kernel's fp16 maximum over tokens, and m*."""
        ts = _f16(self.ehat @ q.T)
        tol = _tol(ts, np.abs(self.ehat) @ np.abs(q).T, self.dim)
        return self._segmax(ts - tol), self._segmax(ts + tol), self._segmax(ts)

    def probe_rows(self, doc_ids) -> np.ndarray:
        """Query rows that plant maxima: ê of each listed document's token at a boundary position, and ê of the tokens
        just outside it (first token of the next document, last of the previous), which score about 0.5 against it
        (the index's centroids share a direction) and 1 against themselves: a read past a document shows up as an
        error of about 0.5."""
        rows = []
        for d in doc_ids:
            o0, o1 = int(self.off[d]), int(self.off[d + 1])
            if o1 == o0:
                continue
            for p in sorted({p for p in BOUNDARY if p < o1 - o0} | {o1 - o0 - 1}):
                rows.append(self.ehat[o0 + p])
            if o1 < self.E:
                rows.append(self.ehat[o1])
            if o0 > 0:
                rows.append(self.ehat[o0 - 1])
        return np.stack(rows)


def _synthetic(dim: int, nbits: int, lengths, K: int = 300, seed: int = 0):
    """An index with random codes and packed residuals.  The centroids share one direction, so every pair of decoded
    tokens has a dot product near 0.5 and a token scores about 1 against itself: a planted maximum stands out, and a
    negated query has a negative maximum against every document."""
    from fast_plaid_b200.engine import IndexTensors

    g = torch.Generator().manual_seed(seed)
    u = torch.nn.functional.normalize(torch.randn(dim, generator=g), dim=0)
    cent = torch.nn.functional.normalize(u + torch.randn(K, dim, generator=g) / dim ** 0.5, dim=-1).half()
    bw = torch.sort(torch.randn(2 ** nbits, generator=g) * 0.03).values.half()
    E = int(sum(lengths))
    codes = torch.randint(0, K, (E,), generator=g)
    res = torch.randint(0, 256, (E, dim * nbits // 8), generator=g).to(torch.uint8)
    return IndexTensors(nbits, cent, bw, torch.tensor(lengths, dtype=torch.int64), codes, res, None, None)


_cache: dict = {}


def _index(dim: int, nbits: int, lengths=LENGTHS, K: int = 300):
    key = (dim, nbits, tuple(lengths), K)
    if key not in _cache:
        from fast_plaid_b200.engine import DeviceIndex

        t = _synthetic(dim, nbits, lengths, K)
        didx = DeviceIndex(t, "cuda:0")
        _cache[key] = (t, didx, _Ref(t, didx))
    return _cache[key]


# ---- driving the MaxSim stage directly --------------------------------------------------------------------------------
def _maxsim(didx, q: np.ndarray, rerank: np.ndarray, n_rerank: np.ndarray) -> np.ndarray:
    """Pad the queries (centroid-score stage), write a hand-made re-rank list into the workspace, fill `exact` with
    NaN and launch the MaxSim stage alone."""
    from fast_plaid_b200.engine import DeviceIndex

    R = rerank.shape[1]
    q16 = torch.from_numpy(q).half().to(didx.device)  # exact: every row holds fp16 values
    params = DeviceIndex.make_params(10, 4 * R, 8)
    st = didx.run_stages(q16, params, upto="centroid_scores")
    assert st["layout"].R == R
    st["rerank"].copy_(torch.from_numpy(rerank.astype(np.int32)))
    st["n_rerank"].copy_(torch.from_numpy(n_rerank.astype(np.int32)))
    st["exact"].fill_(float("nan"))
    didx.stage_fn("maxsim", q16, params)()
    torch.cuda.synchronize()
    return st["exact"].cpu().numpy().copy()


def _check_scores(ref: _Ref, q: np.ndarray, rerank: np.ndarray, n_rerank: np.ndarray, exact: np.ndarray, what: str):
    B, Q, _ = q.shape
    for b in range(B):
        nr = int(n_rerank[b])
        assert np.isnan(exact[b, nr:]).all(), f"{what}: query {b}: a slot past n_rerank={nr} was written"
        lo, hi, ms = ref.maxima(q[b])
        slack = Q * 2.0 ** -24 * np.abs(ms).sum(1)
        docs = rerank[b, :nr]
        s = exact[b, :nr].astype(np.float64)
        empty = ref.lens[docs] == 0
        assert (s[empty] == np.float32(Q * SENTINEL)).all(), f"{what}: query {b}: an empty document's score"
        lo_s, hi_s = lo.sum(1)[docs] - slack[docs], hi.sum(1)[docs] + slack[docs]
        bad = ~empty & ~((lo_s <= s) & (s <= hi_s))
        if bad.any():
            r = int(np.flatnonzero(bad)[0])
            d = int(docs[r])
            raise AssertionError(f"{what}: query {b}, slot {r} (document {d}, {ref.lens[d]} tokens): score {s[r]!r} "
                                 f"outside [{lo_s[r]!r}, {hi_s[r]!r}], reference {ms[d].sum()!r}")
        for d in np.unique(docs):
            same = exact[b, :nr][docs == d]
            assert (same.view(np.int32) == same[0].view(np.int32)).all(), f"{what}: query {b}: copies of {d} differ"


def _rerank_lists(n_docs: int, B: int, R: int, seed: int) -> np.ndarray:
    """Per query a shuffled list of every document with the rest of the R slots taken by repeats (so one document is
    listed twice at least)."""
    rng = np.random.default_rng(seed)
    out = np.empty((B, R), dtype=np.int64)
    for b in range(B):
        base = np.concatenate([np.arange(n_docs), rng.integers(0, n_docs, R - n_docs)])
        out[b] = rng.permutation(base)
    return out


def _planted_queries(ref: _Ref, B: int, Q: int) -> np.ndarray:
    pool = ref.probe_rows(range(len(ref.lens)))
    q = np.stack([pool[(b * Q + np.arange(Q)) % len(pool)] for b in range(B)])
    return q


# ---- the norm table --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim,nbits", SHAPES)
def test_token_norm_table(dim, nbits, cuda_device):
    t, didx, ref = _index(dim, nbits)
    got = didx.token_norms[: ref.E].cpu().double().numpy()
    tol = _tol(ref.norm, ref.sq, dim)
    assert (np.abs(got - ref.norm) <= tol).all(), f"norm off by {np.abs(got - ref.norm).max()}"
    assert (got != ref.norm).mean() < 0.01, f"{int((got != ref.norm).sum())}/{ref.E} norms differ from n*"


# ---- centroid scores --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["default", "v1"])
@pytest.mark.parametrize("Q", [1, 16, 17, 32, 33, 64, 100, 128, 129, 256])
@pytest.mark.parametrize("dim", [64, 128])
def test_centroid_scores(dim, Q, variant, cuda_device, monkeypatch):
    """S against S*, for K in {37, 128, 1000} (one partial tile, one whole tile, a partial last tile) and B in
    {1, 3, 7} (odd batches: v1's split of the batch over the grid, v2's partial token tiles).  `tmax` must be the
    exact maximum of the same run's S over the rows < K of each 128-row tile, and padded columns exactly 0.  The 1 %
    count is taken over all K and B of the (dim, Q, variant) cell."""
    from fast_plaid_b200.engine import DeviceIndex

    if variant == "v1":
        monkeypatch.setenv("FPB_K1", "v1")
    else:
        monkeypatch.delenv("FPB_K1", raising=False)
    g = torch.Generator().manual_seed(100 + Q)
    qs = torch.nn.functional.normalize(torch.randn(7, Q, dim, generator=g), dim=-1).half()
    params = DeviceIndex.make_params(10, 64, 8)
    differ = total = 0
    for K in (37, 128, 1000):
        t, didx, _ = _index(dim, 4, lengths=(4, 4), K=K)
        C = t.centroids.half().double().numpy()
        q64 = qs.double().numpy()
        S_ref = _f16(np.einsum("kd,bqd->bkq", C, q64))
        tol = _tol(S_ref, np.einsum("kd,bqd->bkq", np.abs(C), np.abs(q64)), dim)
        for B in (1, 3, 7):
            st = didx.run_stages(qs[:B].to(cuda_device), params, upto="centroid_scores")
            torch.cuda.synchronize()
            S = st["S"]
            Qp, n_tiles = S.shape[2], st["layout"].n_tiles
            if Qp > Q:
                assert float(S[:, :, Q:].abs().max()) == 0.0, "padded columns are not zero"
            pad = torch.full((B, n_tiles * 128 - K, Qp), float("-inf"), dtype=torch.float16, device=S.device)
            tmax_ref = torch.cat([S, pad], 1).view(B, n_tiles, 128, Qp).amax(2).transpose(1, 2)
            assert torch.equal(st["tmax"], tmax_ref), f"K={K} B={B}: tile maxima are not the maxima of S"
            got = S[:, :, :Q].double().cpu().numpy()
            err = np.abs(got - S_ref[:B])
            assert (err <= tol[:B]).all(), f"K={K} B={B}: S off by {err.max()} (tolerance {tol[:B].flat[err.argmax()]})"
            differ += int((got != S_ref[:B]).sum())
            total += got.size
    assert differ / total < 0.01, f"{differ}/{total} S entries differ from S*"


# ---- the MaxSim stage, every variant ----------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["default", "v1"])
@pytest.mark.parametrize("Q", K5_Q)
@pytest.mark.parametrize("dim,nbits", SHAPES)
def test_maxsim_stage(dim, nbits, Q, variant, cuda_device, monkeypatch):
    """Hand-made re-rank lists (every document, empty ones, the first and the last, one listed twice; n_rerank = R, 0,
    1, odd, R - 1, R) and queries with planted maxima at pass and tile boundaries.  Query 3 has zero rows.  Query 5 is
    negated, its rows tilted toward the centroids' shared direction first, so that every maximum is negative."""
    if variant == "v1":
        monkeypatch.setenv("FPB_K5", "v1")
    else:
        monkeypatch.delenv("FPB_K5", raising=False)
    t, didx, ref = _index(dim, nbits)
    N = len(LENGTHS)
    R = N + 1
    B = 6
    rerank = _rerank_lists(N, B, R, seed=Q)
    n_rerank = np.array([R, 0, 1, 13, R - 1, R])
    q = _planted_queries(ref, B, Q)
    q[3, 2::5] = 0.0
    u = ref.ehat.mean(0)
    v = q[5] + u / np.linalg.norm(u)
    q[5] = -_f16(v / np.linalg.norm(v, axis=1, keepdims=True))
    _, _, ms = ref.maxima(q[5])
    assert (ms[ref.lens > 0] < 0).all(), "the negated query should have a negative maximum everywhere"
    exact = _maxsim(didx, q, rerank, n_rerank)
    _check_scores(ref, q, rerank, n_rerank, exact, f"({dim},{nbits}) Q={Q} {variant}")


@pytest.mark.parametrize("variant", ["default", "v1"])
@pytest.mark.parametrize("Q", [1, 17, 32, 33, 64, 128, 256])
@pytest.mark.parametrize("dim,nbits", SHAPES)
def test_one_hot_maxima(dim, nbits, Q, variant, cuda_device, monkeypatch):
    """Query b has one nonzero row, p = b, so its score is one fp16 maximum exactly (a zero row contributes exactly
    0): B = Q queries put the nonzero row on every row, including the first and the last and rows 64-127, which v5
    computes as its second m-tile.  Each maximum must lie in its bracket, and fewer than 1 % may differ from m*."""
    if variant == "v1":
        monkeypatch.setenv("FPB_K5", "v1")
    else:
        monkeypatch.delenv("FPB_K5", raising=False)
    t, didx, ref = _index(dim, nbits)
    N = len(LENGTHS)
    R = N + 1
    rerank = _rerank_lists(N, Q, R, seed=1000 + Q)
    pool = ref.probe_rows(range(N))
    rows = pool[np.arange(Q) * 7 % len(pool)]
    q = np.zeros((Q, Q, dim))
    q[np.arange(Q), np.arange(Q)] = rows
    exact = _maxsim(didx, q, rerank, np.full(Q, R))
    lo, hi, ms = ref.maxima(rows)  # [N, Q]: column b is the maximum of query b's nonzero row
    cols = np.broadcast_to(np.arange(Q)[:, None], rerank.shape)
    empty = ref.lens[rerank] == 0
    s = exact.astype(np.float64)
    assert (s[empty] == np.float32(Q * SENTINEL)).all()
    lo_, hi_, m_ = lo[rerank, cols][~empty], hi[rerank, cols][~empty], ms[rerank, cols][~empty]
    s = s[~empty]
    bad = ~((lo_ <= s) & (s <= hi_))
    assert not bad.any(), f"{int(bad.sum())} maxima outside their bracket, e.g. {s[bad][0]!r} vs {m_[bad][0]!r}"
    assert (_f16(s) == s).all(), "a one-hot score is not a single fp16 value"
    assert (s != m_).mean() < 0.01, f"{int((s != m_).sum())}/{s.size} maxima differ from m*"


# ---- K5 v5: chunk sizes and the pass-table limit ----------------------------------------------------------------------
SHORT = (5, 129, 0, 1, 2, 7, 8, 9, 15, 16, 17, 63, 64, 65, 127, 128, 300, 0, 12)


@pytest.mark.parametrize("Q", [33, 64, 128])
def test_v5_chunk_size_does_not_change_scores(Q, cuda_device, monkeypatch):
    """Every FPB_K5_DOCS_PER_CHUNK gives the same bytes (K7 asserts the same rule for FPB_K7_DOCS_PER_CHUNK in
    test_gpu_exhaustive.py).  n_rerank values are not multiples of the chunk sizes, so chunks end mid-list; the longest
    document has 38 passes, so 32 documents fit v5's pass table."""
    monkeypatch.delenv("FPB_K5", raising=False)
    t, didx, ref = _index(128, 4, lengths=SHORT)
    N = len(SHORT)
    R = 45
    rerank = _rerank_lists(N, 4, R, seed=7 + Q)
    n_rerank = np.array([R, 37, 13, 7])
    q = _planted_queries(ref, 4, Q)
    outs = {}
    for dpc in (1, 2, 4, 8, 16, 32):
        monkeypatch.setenv("FPB_K5_DOCS_PER_CHUNK", str(dpc))
        outs[dpc] = _maxsim(didx, q, rerank, n_rerank)
    _check_scores(ref, q, rerank, n_rerank, outs[1], f"v5 Q={Q}")
    for dpc, ex in outs.items():
        assert np.array_equal(ex.view(np.int32), outs[1].view(np.int32)), f"{dpc} documents per chunk change scores"


@pytest.mark.parametrize("long_len", [16384, 16385])
def test_v5_pass_table_limit(long_len, cuda_device, monkeypatch):
    """A 16 384-token document is exactly v5's 2048 passes (one document per chunk); at 16 385 tokens the index falls
    back to the generic kernel.  Both against the reference."""
    monkeypatch.delenv("FPB_K5", raising=False)
    monkeypatch.delenv("FPB_K5_DOCS_PER_CHUNK", raising=False)
    lengths = (3, long_len, 9, 200)
    t, didx, ref = _index(128, 4, lengths=lengths)
    rerank = np.array([[1, 0, 3, 2, 1], [3, 1, 2, 0, 0]])
    n_rerank = np.array([5, 4])
    q = _planted_queries(ref, 2, 64)
    exact = _maxsim(didx, q, rerank, n_rerank)
    _check_scores(ref, q, rerank, n_rerank, exact, f"{long_len}-token document")


# ---- which kernel runs ------------------------------------------------------------------------------------------------
def _kernels(fn) -> str:
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return " ".join(e.key for e in prof.key_averages())


@pytest.mark.parametrize("dim,nbits,Q,lengths,pin,kernel", [
    (128, 4, 16, LENGTHS, None, "k5_maxsim_v4_kernel"),
    (128, 4, 32, LENGTHS, None, "k5_maxsim_v4_kernel"),
    (128, 4, 64, LENGTHS, None, "k5_maxsim_v5_kernel"),
    (128, 4, 128, LENGTHS, None, "k5_maxsim_v5_kernel"),
    (128, 4, 256, LENGTHS, None, "k5_maxsim_kernel"),
    (128, 4, 32, LENGTHS, "v1", "k5_maxsim_kernel"),
    (128, 4, 64, (3, 16384, 9), None, "k5_maxsim_v5_kernel"),
    (128, 4, 64, (3, 16385, 9), None, "k5_maxsim_kernel"),
    (128, 2, 64, LENGTHS, None, "k5_maxsim_kernel"),
    (64, 2, 32, LENGTHS, None, "k5_maxsim_kernel"),
    (128, 1, 16, LENGTHS, None, "k5_maxsim_kernel"),
    (128, 1, 64, LENGTHS, None, "k5_maxsim_kernel"),
    (128, 1, 128, LENGTHS, None, "k5_maxsim_kernel"),
    (128, 4, 32, LENGTHS, "", "k5_maxsim_v4_kernel"),  # only FPB_K5=v1 pins
])
def test_maxsim_dispatch(dim, nbits, Q, lengths, pin, kernel, cuda_device, monkeypatch):
    """The cells above reach the kernel they are meant to test."""
    if pin is not None:
        monkeypatch.setenv("FPB_K5", pin)
    else:
        monkeypatch.delenv("FPB_K5", raising=False)
    t, didx, ref = _index(dim, nbits, lengths=lengths)
    N = len(lengths)
    rerank = _rerank_lists(N, 1, N, seed=0)
    q = _planted_queries(ref, 1, Q)
    names = _kernels(lambda: _maxsim(didx, q, rerank, np.array([N])))
    others = {"k5_maxsim_kernel", "k5_maxsim_v4_kernel", "k5_maxsim_v5_kernel"} - {kernel}
    assert kernel in names and not any(o in names for o in others), names


@pytest.mark.parametrize("dim,Q,pin,kernel", [
    (128, 32, None, "k1_centroid_v2_kernel"),
    (128, 128, None, "k1_centroid_v2_kernel"),
    (128, 256, None, "k1_centroid_scores_kernel"),
    (128, 32, "v1", "k1_centroid_scores_kernel"),
    (64, 64, None, "k1_centroid_scores_kernel"),
    (128, 32, "", "k1_centroid_v2_kernel"),  # only FPB_K1=v1 pins
])
def test_centroid_scores_dispatch(dim, Q, pin, kernel, cuda_device, monkeypatch):
    from fast_plaid_b200.engine import DeviceIndex

    if pin is not None:
        monkeypatch.setenv("FPB_K1", pin)
    else:
        monkeypatch.delenv("FPB_K1", raising=False)
    t, didx, _ = _index(dim, 4, lengths=(4, 4), K=1000)
    q = torch.randn(3, Q, dim, device=cuda_device).half()
    names = _kernels(lambda: didx.run_stages(q, DeviceIndex.make_params(10, 64, 8), upto="centroid_scores"))
    other = ({"k1_centroid_v2_kernel", "k1_centroid_scores_kernel"} - {kernel}).pop()
    assert kernel in names and other not in names, names


# ---- limits and the decoder's reciprocal -------------------------------------------------------------------------------
def test_query_length_limit(cuda_device):
    from fast_plaid_b200.engine import DeviceIndex

    t, didx, _ = _index(128, 4, lengths=(4, 4), K=128)
    params = DeviceIndex.make_params(10, 64, 8)
    didx.run_stages(torch.zeros(1, 256, 128, dtype=torch.float16, device=cuda_device), params, upto="centroid_scores")
    with pytest.raises(ValueError, match="more than 256 tokens are not supported"):
        didx.run_stages(torch.zeros(1, 257, 128, dtype=torch.float16, device=cuda_device), params,
                        upto="centroid_scores")


def test_branch_free_reciprocal_is_correctly_rounded(cuda_device):
    """v4 and v5 divide by a token's norm with decode.cuh's rcp_rn_normal, whose result the final division corrects so
    well that an error in it almost never reaches a decoded element.  So it is checked on its own: equal to the IEEE
    reciprocal on every positive normal fp16 value (build() compiles tools/check_sqrt_rcp.cu)."""
    exe = os.path.join(CSRC, "build", "check_sqrt_rcp")
    assert os.path.exists(exe), f"{exe} is missing: run build()"
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "rcp mismatches 0 " in out.stdout, out.stdout + out.stderr
