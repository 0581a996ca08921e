"""The exact pass of the two-pass approximate stage, and the one-pass mode that shares its kernel, at every work-queue
granule: the scores and the refine list do not depend on how the documents are dealt to the warps.

The exact pass takes its documents in chunks of g consecutive entries of a query's refine list (of its candidates in
the one-pass mode: 64), one chunk per CTA.  For the refine lists g is chosen on the device from the list lengths; FPB_K3_EXACT_DOCS_PER_CHUNK
pins it (a multiple of the 8 warps of a CTA, up to 64) and is read at every launch.  The refine list is built by a cluster of CTAs per query; its order is free,
its set and the threshold T are not.  Checked here at every pin:
  * the threshold T equals the two-level bucket rule computed on the host from the same lower bounds, bit for bit;
  * the refined set is exactly {unresolved (lb < ub) and ub >= T}, with lb and ub recomputed on the host from S, tau
    and the high-centroid bitmap (the exact pass overwrites ub of the refined entries; lb, and ub of the others, must
    match the device bit for bit), n_refine its size;
  * the approximate scores of the refined candidates equal the scores of EXACT_ALL (every candidate scored), and every
    approximate score, n_refine, T and the refined set are byte-identical to the unpinned run;
on batches whose queries have refine lists of length 0, 1, 2, R and more, and a batch where one query holds all the work
and the others none (empty subsets); and the one-pass mode against EXACT_ALL at every pin.
"""

from __future__ import annotations

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N_FULL = 64  # R = n_full_scores / 4 = 16
PINS = (None, 8, 16, 24, 40, 64)
SEL_BINS = 2048

_cache: dict = {}


def _index():
    """600 documents of 20..60 random codes over K = 256 centroids; document 1's codes are the first 20 of document
    0's 40 distinct codes, so in a query of these two candidates document 0 holds every column's maximum: it resolves
    in the bound pass and document 1 does not (a refine list of length 1)."""
    if "didx" not in _cache:
        from fast_plaid_b200.engine import DeviceIndex, IndexTensors

        K, N, dim, nbits = 256, 600, 128, 2
        rng = np.random.default_rng(21)
        lengths = rng.integers(20, 61, N)
        lengths[0], lengths[1] = 40, 20
        first = rng.choice(K, 40, replace=False)
        codes = np.concatenate([first, first[:20], rng.integers(0, K, int(lengths[2:].sum()))]).astype(np.int64)
        g = torch.Generator().manual_seed(21)
        cent = torch.nn.functional.normalize(torch.randn(K, dim, generator=g), dim=-1).half()
        bw = torch.sort(torch.randn(2 ** nbits, generator=g) * 0.03).values.half()
        res = torch.randint(0, 256, (len(codes), dim * nbits // 8), generator=g).to(torch.uint8)
        pairs = np.unique(codes * N + np.repeat(np.arange(N), lengths))
        t = IndexTensors(nbits, cent, bw, torch.from_numpy(lengths), torch.from_numpy(codes), res,
                         torch.from_numpy(pairs % N), torch.from_numpy(np.bincount(pairs // N, minlength=K)))
        _cache["didx"] = DeviceIndex(t, "cuda:0")
        _cache["N"] = N
        offs = np.concatenate([[0], np.cumsum(lengths)])
        _cache["doc_codes"] = [codes[offs[d]:offs[d + 1]] for d in range(N)]
    return _cache["didx"], _cache["N"]


def _col_sum(cols: np.ndarray, Q: int) -> np.float32:
    """K3Cols::sum: each group of 8 columns summed in order in fp32 (padded columns skipped), then the groups combined
    by the xor butterfly of the lanes that hold them."""
    lanes = len(cols) // 8
    vals = []
    for lane in range(lanes):
        s = np.float32(0)
        for q in range(8 * lane, 8 * lane + 8):
            if q < Q:
                s = np.float32(s + np.float32(cols[q]))
        vals.append(s)
    off = 1
    while off < lanes:
        vals = [np.float32(vals[lane] + vals[lane ^ off]) for lane in range(lanes)]
        off <<= 1
    return vals[0]


def _bounds(st: dict, b: int, Q: int) -> tuple[np.ndarray, np.ndarray]:
    """The bound pass's lb and ub of query b's candidates from its S, tau and high-centroid bitmap: per column the
    maximum over the rows whose bit is set (from the padding sentinel), then raised to tau for ub."""
    S = st["S"][b].numpy()
    tau = st["tau"][b].numpy()
    words = st["hibits"][b].numpy().view(np.uint32)
    n = int(st["n_cand"][b])
    lb, ub = np.zeros(n, np.float32), np.zeros(n, np.float32)
    for i, d in enumerate(st["cand"][b, :n].tolist()):
        c = _cache["doc_codes"][d]
        rows = c[((words[c >> 5] >> (c & 31).astype(np.uint32)) & 1) == 1]
        m = np.full(S.shape[1], np.float16(-10000.0))
        if len(rows):
            m = np.maximum(m, S[rows].max(0))
        lb[i] = _col_sum(m, Q)
        ub[i] = _col_sum(np.maximum(m, tau), Q)
    return lb, ub


def _bucket(v: np.ndarray, lo: np.float32, scale: np.float32) -> np.ndarray:
    """value_bucket (select.cuh) in fp32: truncation of (v - lo) * scale, clamped to the buckets."""
    x = (v - lo).astype(np.float32) * scale
    return np.clip(np.trunc(x.astype(np.float32)), 0, SEL_BINS - 1).astype(np.int64)


def _find(b: np.ndarray, need: int) -> tuple[int, int]:
    """The bucket t with count(> t) < need <= count(>= t), and need - count(> t)."""
    ge = np.cumsum(np.bincount(b, minlength=SEL_BINS)[::-1])[::-1]  # ge[t] = count(>= t)
    t = int(np.nonzero(ge >= need)[0].max())
    above = int(ge[t + 1]) if t + 1 < SEL_BINS else 0
    return t, need - above


def _threshold(lb: np.ndarray, n_dec: int) -> np.float32:
    """T of k3_refine_list: the smallest lower bound of the upper set of two levels of 2048 linear buckets that holds
    at least n_dec of them; -inf when nothing is pruned."""
    lb = lb.astype(np.float32)
    if len(lb) <= n_dec:
        return np.float32(-np.inf)
    mn, mx = np.float32(lb.min()), np.float32(lb.max())
    rng = np.float32(mx - mn)
    if rng == 0:
        return mn
    if not rng < np.float32(3.0e38):
        return np.float32(-np.inf)
    scale1 = np.float32(np.float32(SEL_BINS - 1) / rng)
    b1 = _bucket(lb, mn, scale1)
    t1, need1 = _find(b1, n_dec)
    lo1 = np.float32(mn + np.float32(np.float32(t1) / scale1))
    scale2 = np.float32(np.float32(SEL_BINS - 1) * scale1)
    b2 = _bucket(lb, lo1, scale2)
    t2, _ = _find(b2[b1 == t1], need1)
    sel = (b1 > t1) | ((b1 == t1) & (b2 >= t2))
    return np.float32(lb[sel].min())


def _run(didx, q16, params, subset, pin, monkeypatch) -> dict:
    if pin is None:
        monkeypatch.delenv("FPB_K3_EXACT_DOCS_PER_CHUNK", raising=False)
    else:
        monkeypatch.setenv("FPB_K3_EXACT_DOCS_PER_CHUNK", str(pin))
    st = didx.run_stages(q16, params, upto="approx", subset=subset)
    torch.cuda.synchronize()
    return {k: v.cpu().clone() for k, v in st.items() if isinstance(v, torch.Tensor) and k != "workspace"}


def _batches(N: int, rng) -> dict[str, list[list[int]]]:
    """Subsets per query: sizes around R = 16 (lists of 0, 1, R and more entries; [0, 1] refines one) and one query
    holding all."""
    every = list(range(N))
    sizes = [0, 1, 2, 16, 17, 40, 300, N]
    return {
        "mixed": [sorted(rng.choice(N, s, replace=False).tolist()) for s in sizes] + [[0, 1]],
        "one query holds all": [every] + [[] for _ in range(5)],
    }


@pytest.mark.parametrize("lam", ["0.5", "2"])
def test_exact_pass_and_refine_list_at_every_granule(lam, cuda_device, monkeypatch):
    """At FPB_K3_LAMBDA = 0.5 almost no candidate resolves in the bound pass, so a query of n <= R candidates refines
    all n of them (lists of length 0, 2 and R; the one-candidate query resolves, and of documents 0 and 1 only 1 is
    refined: a list of length 1); at 2 the lists are the bench's mix of pruned and refined."""
    from fast_plaid_b200.engine import FPB_FLAG_APPROX_EXACT_ALL, FPB_FLAG_APPROX_TWO_PASS, DeviceIndex

    didx, N = _index()
    monkeypatch.setenv("FPB_K3_LAMBDA", lam)
    rng = np.random.default_rng(3)
    params = DeviceIndex.make_params(N_FULL // 4, N_FULL, 8)
    two = DeviceIndex.with_flags(params, FPB_FLAG_APPROX_TWO_PASS)
    every = DeviceIndex.with_flags(params, FPB_FLAG_APPROX_EXACT_ALL)
    lengths_seen = set()
    for name, subset in _batches(N, rng).items():
        B = len(subset)
        q16 = torch.nn.functional.normalize(
            torch.randn(B, 32, 128, generator=torch.Generator().manual_seed(B)), dim=-1).half().to(cuda_device)
        ref = _run(didx, q16, every, subset, None, monkeypatch)
        runs = {pin: _run(didx, q16, two, subset, pin, monkeypatch) for pin in PINS}
        base = runs[None]
        R = N_FULL // 4
        for b in range(B):
            n = int(base["n_cand"][b])
            exact = ref["approx"][b, :n]
            ub, lb = base["approx"][b, :n], base["approx_lb"][b, :n]
            T = _threshold(lb.numpy(), R)
            what = f"{name} query {b} (n = {n}) lambda={lam}"
            assert base["thresh"][b].numpy().view(np.int32) == T.view(np.int32), \
                f"{what}: T = {float(base['thresh'][b])}, host rule {float(T)}"
            # after the exact pass a refined entry holds its exact score, not its upper bound: the bounds are
            # recomputed on the host (lb must match the device's bit for bit, and so must ub wherever it was kept)
            lb_h, ub_h = _bounds(base, b, 32)
            assert np.array_equal(lb_h.view(np.int32), lb.numpy().view(np.int32)), f"{what}: host lower bounds"
            want = np.nonzero((lb_h < ub_h) & (ub_h >= T))[0]
            nr = int(base["n_refine"][b])
            got = np.sort(base["refine"][b, :nr].numpy())
            assert nr == len(want) and np.array_equal(got, want), f"{what}: refined set differs from the rule"
            kept = np.setdiff1d(np.arange(n), want)
            assert np.array_equal(ub_h[kept].view(np.int32), ub.numpy()[kept].view(np.int32)), f"{what}: upper bounds"
            lengths_seen.add(nr)
            assert torch.equal(ub[want].view(torch.int32), exact[want].view(torch.int32)), \
                f"{what}: a refined score differs from EXACT_ALL"
            for pin, run in runs.items():
                how = f"{what} pin={pin}"
                assert torch.equal(run["approx"][b, :n].view(torch.int32), ub.view(torch.int32)), f"{how}: scores"
                assert int(run["n_refine"][b]) == nr, f"{how}: n_refine"
                assert torch.equal(run["thresh"][b:b + 1].view(torch.int32), base["thresh"][b:b + 1].view(torch.int32)), \
                    f"{how}: T"
                assert np.array_equal(np.sort(run["refine"][b, :nr].numpy()), got), f"{how}: refined set"
    assert 0 in lengths_seen and len(lengths_seen) >= 3, sorted(lengths_seen)
    if lam == "0.5":
        assert {1, 2, R} <= lengths_seen, sorted(lengths_seen)


def test_one_pass_mode_at_every_granule(cuda_device, monkeypatch):
    """The one-pass mode (every candidate through the exact kernel, no list, fixed 64-document chunks that the pin does
    not change) equals EXACT_ALL with the pin set or not."""
    from fast_plaid_b200.engine import FPB_FLAG_APPROX_DIRECT, FPB_FLAG_APPROX_EXACT_ALL, DeviceIndex

    didx, N = _index()
    monkeypatch.delenv("FPB_K3_LAMBDA", raising=False)
    rng = np.random.default_rng(4)
    params = DeviceIndex.make_params(N_FULL // 4, N_FULL, 8)
    for name, subset in _batches(N, rng).items():
        B = len(subset)
        q16 = torch.nn.functional.normalize(
            torch.randn(B, 32, 128, generator=torch.Generator().manual_seed(B + 1)), dim=-1).half().to(cuda_device)
        ref = _run(didx, q16, DeviceIndex.with_flags(params, FPB_FLAG_APPROX_EXACT_ALL), subset, None, monkeypatch)
        for pin in PINS:
            run = _run(didx, q16, DeviceIndex.with_flags(params, FPB_FLAG_APPROX_DIRECT), subset, pin, monkeypatch)
            for b in range(B):
                n = int(ref["n_cand"][b])
                assert int(run["n_cand"][b]) == n
                assert torch.equal(run["approx"][b, :n].view(torch.int32), ref["approx"][b, :n].view(torch.int32)), \
                    f"{name} query {b} pin={pin}: one-pass scores differ from EXACT_ALL"
                assert int(run["n_refine"][b]) == 0
