"""Every kernel past the 32-bit offsets: residual rows beyond 2 GiB and 4 GiB, and a score table beyond 2^31 elements.

At dim 128, nbits 4 a token's packed residuals are 64 bytes, so residual byte 2^31 is token 2^25 and byte 2^32 is
token 2^26.  The kernels form these offsets as `tok * PD`, `row * 64`, `src * vec_per_row` and so on; a product
narrowed to 32 bits reads the wrong rows past the first 2 GiB.  The large index here holds 2^26 + 200 000 tokens
(4.3 GB of residuals): about 65 000 filler documents of 1 024 tokens on centroids around -u, and about 30 probe
documents on a disjoint block of centroids around +u, planted at exact token positions (`_plan`): at offset 0, ending
and starting exactly at 2^25 and 2^26, straddling them (300 tokens from 7 before, 129 tokens from 3 before, so
that an 8-token pass crosses the boundary, 2 000 tokens from 1 000 before), 1-token documents on either side of
2^26, empty documents next to each boundary, and the last document of the index.  One layout cannot hold all of
these at once, so the large fixture is built once per layout (`LAYOUTS`), one at a time.

The small index has the same centroid table and bucket weights and holds only the probe documents, in the same
order, with its own inverted file.  Queries are ê rows of the probe documents (test_gpu_kernels._Ref.probe_rows),
which score every probe centroid far above every filler centroid: with n_ivf_probe <= 256 every probed cell is a
probe cell and every candidate a probe document (each test asserts it).  Small-index ids map to large-index ids in
increasing order, so integer stages and tie orders carry over, and the contract is: mapped ids, same bytes.  The
small index is further held to the float64 references of test_gpu_kernels.py, test_gpu_exact_kernels.py and
test_gpu_exact_schedule.py (imported, not copied).

After `delete` (one filler before 2^25: every later document moves 1 024 tokens down across both boundaries; a
block of fillers larger than 2^25 tokens: documents read above 4 GiB are written below 2 GiB) and `append` (copies
of the probe documents land past 4 GiB, so the growable buffers commit past it) the same checks run again.

The score table: K = 2^20 centroids, B = 40 queries of Q = 64 (Qp = 64) make S 40 * 2^20 * 64 = 2.7e9 elements, so
the last eight queries' rows lie wholly past element 2^31.  At this K the high-centroid bitmap (hb_words * 4 =
128 KiB) does not fit the bound pass's shared memory and FPB_FLAG_APPROX_TWO_PASS falls back to one pass.

The large fixtures check `torch.cuda.mem_get_info` against what they need and skip with both numbers when it falls
short; each prints the free memory it saw, its build time and the peak device memory in use (torch's allocator plus
the growable buffers, which torch does not count).  The last tests run without a GPU: they check the arithmetic of
the layouts, of the deletes and of the score table."""

from __future__ import annotations

import dataclasses
import gc
import time

import numpy as np
import pytest
import torch

import test_gpu_exact_kernels as ek
import test_gpu_kernels as gk
from test_gpu_exact_kernels import fma_chain
from test_gpu_exact_schedule import _col_sum
from test_gpu_kernels import _check_scores, _maxsim, _Ref

gpu = pytest.mark.gpu

DIM, NBITS, PD = 128, 4, 64
B1, B2 = 1 << 25, 1 << 26  # the tokens at residual bytes 2^31 and 2^32
E_END = B2 + 200_000  # tokens of the large index
FILL = 1024  # filler length (the first filler of a gap takes the remainder)
K_F, K_P = 4096, 256  # filler centroids [0, K_F), probe centroids [K_F, K_F + K_P)
GiB = 1 << 30

# A layout is a list of clusters (anchor, before, after): the probe documents `before` end exactly at token
# `anchor`, the documents `after` start there.  Every layout starts with gk.LENGTHS at offset 0 (the control group)
# and ends with TAIL, whose last document is the last of the index.
LAYOUTS = {
    "edges": [(B1, (0, 300, 0), (129, 0)), (B2, (0, 300, 1, 0), (1, 129, 0))],
    "straddle": [(B1 - 7, (0,), (300, 0)), (B2 - 7, (0,), (300, 0))],
    "pass": [(B1 - 3, (0,), (129, 0)), (B2 - 3, (0,), (129, 0))],
    "long": [(B1 - 1000, (0,), (2000, 0)), (B2 - 1000, (0,), (2000, 0))],
}
TAIL = (0, 65, 7, 5)
SEARCH_Q = (16, 32, 64, 256)
MAXSIM_Q = (16, 32, 64, 128, 256)


# ---- the layouts (host arithmetic) -----------------------------------------------------------------------------------
@dataclasses.dataclass
class Plan:
    lengths: np.ndarray  # [N] every document of the large index
    probe: np.ndarray  # [n] large-index ids of the probe documents, increasing
    off: np.ndarray  # [N + 1] token offsets

    @property
    def probe_lens(self) -> np.ndarray:
        return self.lengths[self.probe]


def _plan(name: str) -> Plan:
    clusters = [(0, (), gk.LENGTHS)] + LAYOUTS[name] + [(E_END, TAIL, ())]
    lengths, probe, cur = [], [], 0
    for anchor, before, after in clusters:
        start = anchor - sum(before)
        gap = start - cur
        assert gap >= 0, (name, anchor)
        r = gap % FILL
        lengths += ([r] if r else []) + [FILL] * (gap // FILL)
        probe += range(len(lengths), len(lengths) + len(before) + len(after))
        lengths += list(before) + list(after)
        cur = start + sum(before) + sum(after)
    assert cur == E_END
    lengths = np.array(lengths, np.int64)
    return Plan(lengths, np.array(probe, np.int64), np.concatenate([[0], np.cumsum(lengths)]))


def _deletes(plan: Plan) -> dict[str, np.ndarray]:
    """The fillers each delete drops.  "one": the last filler before 2^25's cluster (1 024 tokens).  "block": every
    filler before 2^25's cluster, then fillers after it until more than 2^25 + 8 192 tokens are dropped, so that every
    document that ended past 2^26 - 1 000 + 2 000 before now ends below 2^25."""
    is_probe = np.zeros(len(plan.lengths), bool)
    is_probe[plan.probe] = True
    fill = np.flatnonzero(~is_probe)
    first = plan.probe[len(gk.LENGTHS)]  # the first document of 2^25's cluster
    before = fill[fill < first]
    after = fill[fill > first]
    need = B1 + 8192 - int(plan.lengths[before].sum())
    n_after = int(np.searchsorted(np.cumsum(plan.lengths[after]), need, side="right")) + 1
    return {"one": before[-1:], "block": np.concatenate([before, after[:n_after]])}


def _remap(ids: np.ndarray, dropped: np.ndarray) -> np.ndarray:
    """The ids of kept documents after a delete of `dropped` (sorted): each moves down by the dropped ids below it."""
    return ids - np.searchsorted(dropped, ids)


# ---- the fixtures ----------------------------------------------------------------------------------------------------
_live: list[dict] = []  # the large fixture alive now, released before another is built


def _release() -> None:
    for holder in _live:
        for v in holder.values():
            if hasattr(v, "close"):
                v.close()
        holder.clear()
    _live.clear()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _start(need: int, what: str) -> int:
    _release()
    free, total = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"{what} needs {need / GiB:.1f} GiB of free device memory, {free / GiB:.1f} GiB are free")
    torch.cuda.reset_peak_memory_stats()
    return free


class _Peak:
    """Device memory in use above the fixture's start: sampled at every check (torch's own peak misses the growable
    buffers, which map their memory outside the allocator)."""

    def __init__(self, free0: int) -> None:
        self.free0, self.used = free0, 0

    def sample(self) -> None:
        torch.cuda.synchronize()
        self.used = max(self.used, self.free0 - torch.cuda.mem_get_info()[0])

    def report(self, what: str) -> str:
        self.sample()
        return (f"{what}: free at start {self.free0 / GiB:.2f} GiB, peak in use {self.used / GiB:.2f} GiB, torch "
                f"max_memory_allocated {torch.cuda.max_memory_allocated() / GiB:.2f} GiB")


def _small_tensors(lengths, seed: int):
    """The codec shared by both indexes and the probe documents alone: filler centroids around -u, probe centroids
    around +u, probe codes in [K_F, K_F + K_P)."""
    from fast_plaid_b200.engine import IndexTensors

    g = torch.Generator().manual_seed(seed)
    u = torch.nn.functional.normalize(torch.randn(DIM, generator=g), dim=0)
    cf = torch.nn.functional.normalize(-u + torch.randn(K_F, DIM, generator=g) / DIM ** 0.5, dim=-1)
    cp = torch.nn.functional.normalize(u + torch.randn(K_P, DIM, generator=g) / DIM ** 0.5, dim=-1)
    cent = torch.cat([cf, cp]).half()
    bw = torch.sort(torch.randn(2 ** NBITS, generator=g) * 0.03).values.half()
    E = int(sum(lengths))
    codes = torch.randint(K_F, K_F + K_P, (E,), generator=g)
    res = torch.randint(0, 256, (E, PD), generator=g).to(torch.uint8)
    t = IndexTensors(NBITS, cent, bw, torch.tensor(np.asarray(lengths), dtype=torch.int64), codes, res, None, None)
    return ek._with_ivf(t)


def _large(plan: Plan, small, dev: str, seed: int):
    """The large index, built on the device in growable buffers (so that `append` grows it in place): random filler
    codes and residuals, the probe documents' rows copied in at their planned offsets, and its inverted file."""
    from fast_plaid_b200.engine import DeviceIndex, GrowableArrays, IndexTensors

    N, E = len(plan.lengths), int(plan.off[-1])
    arrays = GrowableArrays(torch.device(dev), PD)
    v = arrays.views(N, E)
    g = torch.Generator(device=dev).manual_seed(seed)
    v["codes"].random_(0, K_F, generator=g)
    v["residuals"].random_(0, 256, generator=g)
    pos = torch.from_numpy(np.concatenate([np.arange(plan.off[d], plan.off[d + 1]) for d in plan.probe])).to(dev)
    v["codes"].index_copy_(0, pos, small.doc_codes.to(dev, torch.int32))
    v["residuals"].index_copy_(0, pos, small.doc_residuals.to(dev))
    lens = torch.from_numpy(plan.lengths)
    key = v["codes"].long() * N + torch.repeat_interleave(torch.arange(N, device=dev), lens.to(dev))
    key = torch.unique(key)  # (code, document) pairs, sorted by code, then document
    ivf, ivf_lengths = (key % N).int(), torch.bincount(key // N, minlength=K_F + K_P)
    del key, pos
    t = IndexTensors(NBITS, small.centroids, small.bucket_weights, lens, v["codes"], v["residuals"], ivf, ivf_lengths,
                     growable=arrays)
    didx = DeviceIndex(t, dev)
    del t, ivf, ivf_lengths, v
    return didx


@pytest.fixture(scope="module", params=list(LAYOUTS))
def big(request, cuda_device):
    """Per layout: the small and the large index, the small one's float64 reference and the id map.  Needs about
    11 GiB (the large index's 4.7 GB of per-token arrays, its walk layout and inverted file, and a delete's second
    copy)."""
    from fast_plaid_b200.engine import DeviceIndex

    name = request.param
    free0 = _start(12 * GiB, f"the large index ({name})")
    t0 = time.time()
    plan = _plan(name)
    small_t = _small_tensors(plan.probe_lens, seed=31)
    small = DeviceIndex(small_t, cuda_device)
    ref = _Ref(small_t, small)
    n = len(plan.probe)
    pool = ref.probe_rows(range(n))
    C = small_t.centroids.double().numpy()
    lo, hi = (pool @ C[K_F:].T).min(), (pool @ C[:K_F].T).max()
    assert lo > hi + 0.1, f"a filler centroid scores {hi} and a probe centroid {lo}: a filler cell could be probed"
    large = _large(plan, small_t, cuda_device, seed=32)
    holder = {"small": small, "large": large}
    _live.append(holder)
    peak = _Peak(free0)
    peak.sample()
    offs = large.doc_offsets.cpu().numpy()
    assert np.array_equal(offs, plan.off), f"{name}: the probe documents are not at their planned offsets"
    assert large.max_doc_len == small.max_doc_len == 2000
    print(f"\n[{name}] {len(plan.lengths)} documents, {large.num_tokens} tokens, built in {time.time() - t0:.1f} s")
    del large  # only `holder` may hold it: `_release` frees it before the next fixture is built
    yield dict(name=name, plan=plan, small_t=small_t, small=small, ref=ref, holder=holder, peak=peak, dev=cuda_device)
    print(peak.report(f"[{name}]"))
    _release()


# ---- the checks (shared by the base index, the deletes and the append) -----------------------------------------------
def _b16(x: torch.Tensor | np.ndarray) -> np.ndarray:
    x = x.cpu().numpy() if isinstance(x, torch.Tensor) else x
    return x.view({2: np.uint16, 4: np.uint32, 8: np.uint64, 1: np.uint8}[x.dtype.itemsize])


def _queries(fx, B: int, Q: int) -> np.ndarray:
    return gk._planted_queries(fx["ref"], B, Q)


def _check_load(fx, large, ids: np.ndarray, what: str) -> None:
    """Token norms and walk windows of every probe document equal the small index's; the small index's norms lie in
    the float64 bracket of n* (test_gpu_kernels.test_token_norm_table)."""
    small, ref = fx["small"], fx["ref"]
    s_off, l_off = small.doc_offsets.cpu().numpy(), large.doc_offsets.cpu().numpy()
    assert np.array_equal(np.diff(l_off)[ids], np.diff(s_off)), f"{what}: document lengths"
    s_norm, l_norm = _b16(small.token_norms[: small.num_tokens]), _b16(large.token_norms[: large.num_tokens])
    for i, d in enumerate(ids):
        assert np.array_equal(l_norm[l_off[d]: l_off[d + 1]], s_norm[s_off[i]: s_off[i + 1]]), \
            f"{what}: token norms of probe document {i} (tokens {l_off[d]} .. {l_off[d + 1]})"
    got = small.token_norms[: ref.E].cpu().double().numpy()
    assert (np.abs(got - ref.norm) <= gk._tol(ref.norm, ref.sq, DIM)).all(), "small index: a norm off n*"
    assert (got != ref.norm).mean() < 0.01
    s_codes, s_win = (x.cpu().numpy() for x in small.walk_layout())
    l_codes, l_win = large.walk_layout()
    l_win = l_win.cpu().numpy()
    for i, d in enumerate(ids):
        w = l_codes[int(l_win[d]): int(l_win[d + 1])].cpu().numpy()
        assert np.array_equal(w, s_codes[s_win[i]: s_win[i + 1]]), f"{what}: walk windows of probe document {i}"
    del l_codes
    fx["peak"].sample()


def _check_reconstruct(fx, large, ids: np.ndarray, what: str) -> None:
    small, ref = fx["small"], fx["ref"]
    n = len(ids)
    order = list(range(n)) + [n - 1, 0, n // 2]
    got = torch.cat(large.reconstruct([int(ids[i]) for i in order])).cpu().numpy()
    want = torch.cat(small.reconstruct(order)).cpu().numpy()
    assert np.array_equal(_b16(got), _b16(want)), f"{what}: reconstruct differs from the small index"
    e16 = ref.ehat.astype(np.float16)
    flat = np.concatenate([e16[int(ref.off[i]): int(ref.off[i + 1])] for i in order])
    assert np.array_equal(_b16(want), _b16(flat)), "small index: reconstruct is not e_hat"


def _check_token_scores(fx, large, ids: np.ndarray, what: str) -> None:
    small, ref = fx["small"], fx["ref"]
    n, B, Q = len(ids), 2, 33
    q = _queries(fx, B, Q)
    q16 = torch.from_numpy(q).half().to(fx["dev"])
    qo = torch.arange(B, dtype=torch.int32).repeat_interleave(n)
    docs = torch.arange(n, dtype=torch.int32).repeat(B)
    want = small.token_scores(q16, qo, docs).cpu().numpy()
    got = large.token_scores(q16, qo, torch.from_numpy(ids[docs.numpy()].astype(np.int32))).cpu().numpy()
    assert got.shape == want.shape and np.array_equal(_b16(got), _b16(want)), f"{what}: token matrices differ"
    for b in range(B):
        chain = fma_chain(ref.ehat, q[b]).astype(np.float16)
        for i in range(n):
            o0, o1 = int(ref.off[i]), int(ref.off[i + 1])
            k = b * n + i
            assert np.array_equal(_b16(want[k, : o1 - o0]), _b16(chain[o0:o1])), \
                f"small index: query {b}, document {i}: not the fma chain"
            assert not _b16(want[k, o1 - o0:]).any()


def _stage_copy(st: dict) -> dict:
    return {k: v.cpu().clone() for k, v in st.items() if isinstance(v, torch.Tensor) and k != "workspace"}


def _run(didx, q16, params, **kw) -> dict:
    st = didx.run_stages(q16, params, **kw)
    torch.cuda.synchronize()
    return _stage_copy(st)


def _compare_stages(s: dict, g: dict, ids: np.ndarray, what: str, two_pass: bool, direct: bool) -> None:
    """Every stage array of the large index's run `g` equals the small index's `s` after mapping ids; every cell is a
    probe cell and every candidate a probe document."""
    B = s["n_cand"].shape[0]
    probe = set(ids.tolist())
    m = lambda x: ids[x.numpy().astype(np.int64)]  # noqa: E731
    for b in range(B):
        w = f"{what}: query {b}"
        cells = g["cells"][b].numpy()
        assert (cells[cells >= 0] >= K_F).all() and (cells >= 0).any(), f"{w}: a filler cell was probed"
        assert torch.equal(g["cells"][b], s["cells"][b]), f"{w}: cells"
        n = int(s["n_cand"][b])
        assert n > 0 and int(g["n_cand"][b]) == n, f"{w}: n_cand {int(g['n_cand'][b])} vs {n}"
        assert set(g["cand"][b, :n].tolist()) <= probe, f"{w}: a filler is a candidate"
        assert np.array_equal(g["cand"][b, :n].numpy(), m(s["cand"][b, :n])), f"{w}: cand"
        assert np.array_equal(_b16(g["approx"][b, :n]), _b16(s["approx"][b, :n])), f"{w}: approx"
        if two_pass:
            assert np.array_equal(_b16(g["approx_lb"][b, :n]), _b16(s["approx_lb"][b, :n])), f"{w}: approx_lb"
            assert np.array_equal(_b16(g["thresh"][b]), _b16(s["thresh"][b])), f"{w}: thresh"
        assert int(g["n_refine"][b]) == int(s["n_refine"][b]), f"{w}: n_refine"
        if direct:
            assert int(s["n_refine"][b]) == 0
        r = int(s["n_rerank"][b])
        assert int(g["n_rerank"][b]) == r and r > 0, f"{w}: n_rerank"
        assert np.array_equal(g["rerank"][b, :r].numpy(), m(s["rerank"][b, :r])), f"{w}: rerank"
        for k in ("rerank_approx", "exact"):
            assert np.array_equal(_b16(g[k][b, :r]), _b16(s[k][b, :r])), f"{w}: {k}"
        c = int(s["counts"][b])
        assert int(g["counts"][b]) == c and c > 0, f"{w}: counts"
        assert np.array_equal(g["ids"][b, :c].numpy(), m(s["ids"][b, :c])), f"{w}: ids"
        assert np.array_equal(_b16(g["scores"][b, :c]), _b16(s["scores"][b, :c])), f"{w}: scores"


def _check_approx_ref(fx, s: dict, Q: int, what: str) -> None:
    """Where every candidate is scored in full (one pass, EXACT_ALL), its approximate score is K3Cols::sum
    (test_gpu_exact_schedule._col_sum) of the column maxima of its codes' S rows, bit for bit, from the run's own S."""
    t, off = fx["small_t"], fx["ref"].off
    codes = t.doc_codes.numpy()
    for b in range(s["n_cand"].shape[0]):
        S = s["S"][b].numpy()
        n = int(s["n_cand"][b])
        want = np.array([_col_sum(S[codes[off[d]: off[d + 1]]].max(0), Q) for d in s["cand"][b, :n].tolist()])
        assert np.array_equal(_b16(want.astype(np.float32)), _b16(s["approx"][b, :n])), f"{what}: query {b}"


FLAGS = ("APPROX_DIRECT", "APPROX_TWO_PASS", "APPROX_EXACT_ALL")


def _check_search(fx, large, ids: np.ndarray, what: str, Qs=SEARCH_Q, flags=FLAGS) -> None:
    from fast_plaid_b200 import engine
    from fast_plaid_b200.engine import DeviceIndex

    small = fx["small"]
    for Q in Qs:
        q16 = torch.from_numpy(_queries(fx, 4, Q)).half().to(fx["dev"])
        for f in flags:
            params = DeviceIndex.make_params(10, 64, 32, flags=getattr(engine, "FPB_FLAG_" + f))
            s = _run(small, q16, params)
            g = _run(large, q16, params)
            fx["peak"].sample()
            if f != "APPROX_TWO_PASS":
                _check_approx_ref(fx, s, Q, f"small index Q={Q} {f}")
            _compare_stages(s, g, ids, f"{what} Q={Q} {f}", two_pass=f != "APPROX_DIRECT", direct=f == "APPROX_DIRECT")


def _check_exhaustive(fx, large, ids: np.ndarray, what: str) -> None:
    small = fx["small"]
    n = len(ids)
    for Q in (16, 64):
        q16 = torch.from_numpy(_queries(fx, 3, Q)).half().to(fx["dev"])
        want = small.exhaustive_scores(q16).cpu().numpy()
        got = large.exhaustive_scores(q16)[:, torch.from_numpy(ids).to(fx["dev"])].cpu().numpy()
        fx["peak"].sample()
        assert np.array_equal(_b16(got), _b16(want)), f"{what} Q={Q}: exhaustive scores of the probe documents"
        si, ss, sc = (x.cpu().numpy() for x in small.search_exhaustive(q16, n, subset=[list(range(n))] * 3))
        gi, gs, gc_ = (x.cpu().numpy() for x in large.search_exhaustive(q16, n, subset=[ids.tolist()] * 3))
        assert np.array_equal(gc_, sc) and (sc == n).all(), f"{what} Q={Q}: list-walk counts"
        assert np.array_equal(gi, ids[si]), f"{what} Q={Q}: list-walk ranking"
        assert np.array_equal(_b16(gs), _b16(ss)), f"{what} Q={Q}: list-walk scores"


# ---- the large residual index ----------------------------------------------------------------------------------------
@gpu
def test_load(big):
    _check_load(big, big["holder"]["large"], big["plan"].probe, big["name"])


@gpu
def test_reconstruct_and_get_embeddings(big, tmp_path):
    from fast_plaid_b200 import search

    large, ids = big["holder"]["large"], big["plan"].probe
    _check_reconstruct(big, large, ids, big["name"])
    fp = search.FastPlaid.from_device_index(large, index_dir=str(tmp_path))
    sel = [int(ids[-1]), int(ids[0]), int(ids[len(ids) // 2])]
    for g, h in zip(large.reconstruct(sel), fp.get_embeddings(sel)):
        assert h.device.type == "cpu" and torch.equal(h, g.cpu())


@gpu
def test_token_scores(big, tmp_path):
    """token_scores, then search_token_scores through FastPlaid on both indexes (B = 2 keeps both below the size
    at which the library picks the two-pass approximate stage by itself)."""
    from fast_plaid_b200 import search

    large, ids = big["holder"]["large"], big["plan"].probe
    _check_token_scores(big, large, ids, big["name"])
    queries = torch.from_numpy(_queries(big, 2, 33)).float()
    res_s = search.FastPlaid.from_device_index(big["small"], index_dir=str(tmp_path / "s")).search_token_scores(
        queries, top_k=10, show_progress=False)
    res_l = search.FastPlaid.from_device_index(large, index_dir=str(tmp_path / "l")).search_token_scores(
        queries, top_k=10, show_progress=False)
    for b in range(2):
        assert len(res_s[b]) == len(res_l[b]) > 0
        for (d, s, mat), (d2, s2, mat2) in zip(res_s[b], res_l[b]):
            assert d2 == int(ids[d]) and s2 == s and torch.equal(mat, mat2), f"query {b}, document {d}"


@gpu
@pytest.mark.parametrize("variant", ["default", "v1"])
def test_maxsim_stage(big, variant, monkeypatch):
    """Re-rank lists naming every probe document and repeats, at Q = 16 .. 256 (K5 v4, v5 and the generic kernel;
    FPB_K5=v1 pins the generic one): the large index's scores equal the small index's bit for bit, and lie in the
    float64 bracket."""
    if variant == "v1":
        monkeypatch.setenv("FPB_K5", "v1")
    else:
        monkeypatch.delenv("FPB_K5", raising=False)
    large, ids, ref = big["holder"]["large"], big["plan"].probe, big["ref"]
    n = len(ids)
    R, B = n + 3, 4
    n_rerank = np.array([R, 1, R - 1, R])
    for Q in MAXSIM_Q:
        rerank = gk._rerank_lists(n, B, R, seed=Q)
        q = _queries(big, B, Q)
        want = _maxsim(big["small"], q, rerank, n_rerank)
        got = _maxsim(large, q, ids[rerank], n_rerank)
        what = f"{big['name']} Q={Q} {variant}"
        assert np.array_equal(_b16(got), _b16(want)), f"{what}: MaxSim scores differ from the small index's"
        _check_scores(ref, q, rerank, n_rerank, want, what)


@gpu
def test_search(big):
    """Whole search, stage by stage, with each approximate mode pinned, at Q = 16, 32, 64 and 256."""
    _check_search(big, big["holder"]["large"], big["plan"].probe, big["name"])


@gpu
def test_search_subset_and_filter(big):
    """subset= and a filter= mask naming the probe documents plus fillers on both sides of each boundary (which are
    not candidates: their cells are not probed) give the small index's search over all its documents."""
    from fast_plaid_b200.engine import FPB_FLAG_APPROX_TWO_PASS, DeviceIndex, Filter

    large, ids, plan = big["holder"]["large"], big["plan"].probe, big["plan"]
    small, n, dev = big["small"], len(ids), big["dev"]
    fillers = np.setdiff1d(np.arange(len(plan.lengths)), ids)
    near = np.concatenate([fillers[np.abs(plan.off[fillers] - X) < 5 * FILL] for X in (B1, B2)] + [fillers[-3:]])
    named = np.union1d(ids, near)
    q16 = torch.from_numpy(_queries(big, 3, 32)).half().to(dev)
    params = DeviceIndex.make_params(10, 64, 32, flags=FPB_FLAG_APPROX_TWO_PASS)
    s = _run(small, q16, params, subset=[list(range(n))] * 3)
    g = _run(large, q16, params, subset=[named.tolist()] * 3)
    _compare_stages(s, g, ids, f"{big['name']} subset", True, False)
    mask = torch.zeros(len(plan.lengths), dtype=torch.bool)
    mask[torch.from_numpy(named)] = True
    s = _run(small, q16, params, filter=Filter.from_mask(torch.ones(n, dtype=torch.bool), dev, 3))
    g = _run(large, q16, params, filter=Filter.from_mask(mask, dev, 3))
    _compare_stages(s, g, ids, f"{big['name']} filter", True, False)


@gpu
def test_exhaustive(big):
    _check_exhaustive(big, big["holder"]["large"], big["plan"].probe, big["name"])


@gpu
@pytest.mark.parametrize("case", ["one", "block"])
def test_delete(big, case):
    """After the delete the probe documents sit at new offsets (checked against the plan); load, reconstruct and
    search give the small index's bytes under the new id map."""
    large, plan = big["holder"]["large"], big["plan"]
    drop = _deletes(plan)[case]
    new = large.delete(drop.tolist())
    big["holder"]["deleted"] = new
    try:
        ids = _remap(plan.probe, drop)
        keep = np.setdiff1d(np.arange(len(plan.lengths)), drop)
        assert np.array_equal(np.diff(new.doc_offsets.cpu().numpy()), plan.lengths[keep])
        what = f"{big['name']} delete {case}"
        _check_load(big, new, ids, what)
        _check_reconstruct(big, new, ids, what)
        _check_search(big, new, ids, what, Qs=(32, 64))
    finally:
        big["holder"].pop("deleted").close()
        new = None
        _settle()


def _settle() -> None:
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@gpu
def test_append(big):
    """Copies of the probe documents appended to the large index land past residual byte 2^32 (its buffers grow in
    place past 4 GiB); they and the originals give the small index's bytes.  Runs last for its layout: the large
    index is then no longer the newest of its chain."""
    large, plan, small_t = big["holder"]["large"], big["plan"], big["small_t"]
    N, E = large.num_documents, large.num_tokens
    new = large.append(small_t.doc_codes, small_t.doc_residuals, small_t.doc_lengths)
    big["holder"]["appended"] = new
    try:
        assert E * PD > 1 << 32 and new.growable.residuals.mapped_bytes >= (E + int(plan.probe_lens.sum())) * PD
        copies = N + np.arange(len(plan.probe))
        what = f"{big['name']} append"
        for ids in (plan.probe, copies):
            _check_load(big, new, ids, what)
            _check_reconstruct(big, new, ids, what)
        _check_exhaustive(big, new, copies, what)
        from fast_plaid_b200.engine import FPB_FLAG_APPROX_TWO_PASS, DeviceIndex

        n = len(copies)
        q16 = torch.from_numpy(_queries(big, 3, 32)).half().to(big["dev"])
        params = DeviceIndex.make_params(10, 64, 32, flags=FPB_FLAG_APPROX_TWO_PASS)
        s = _run(big["small"], q16, params, subset=[list(range(n))] * 3)
        g = _run(new, q16, params, subset=[copies.tolist()] * 3)
        _compare_stages(s, g, copies, f"{what} subset", True, False)
    finally:
        big["holder"].pop("appended").close()
        new = None
        _settle()


# ---- the large score table -------------------------------------------------------------------------------------------
K_BIG, S_B, S_Q = 1 << 20, 40, 64


@pytest.fixture(scope="module")
def table(cuda_device):
    """An index of gk.LENGTHS (2 722 tokens) over K = 2^20 centroids; B = 40 queries of 64 planted rows.  Needs about
    7 GiB (the 5.4 GB score table, the centroids, the rest of the workspace)."""
    from fast_plaid_b200.engine import DeviceIndex

    free0 = _start(8 * GiB, "the K = 2^20 score table")
    t0 = time.time()
    t = ek._with_ivf(gk._synthetic(DIM, NBITS, gk.LENGTHS, K=K_BIG, seed=5))
    didx = DeviceIndex(t, cuda_device)
    ref = _Ref(t, didx)
    q = gk._planted_queries(ref, S_B, S_Q)
    holder = {"didx": didx}
    _live.append(holder)
    peak = _Peak(free0)
    print(f"\n[table] built in {time.time() - t0:.1f} s")
    yield dict(t=t, didx=didx, ref=ref, q=q, q16=torch.from_numpy(q).half().to(cuda_device), peak=peak,
               holder=holder, dev=cuda_device)
    print(peak.report("[table]"))
    _release()


def _params(flag_name: str):
    from fast_plaid_b200 import engine
    from fast_plaid_b200.engine import DeviceIndex

    return DeviceIndex.make_params(10, 64, 8, flags=getattr(engine, "FPB_FLAG_" + flag_name))


LAST = (S_B - 3, S_B - 2, S_B - 1)


@gpu
@pytest.mark.parametrize("variant", ["default", "v1"])
def test_table_centroid_scores(table, variant, monkeypatch):
    """S rows of the last three queries, the first and the last 4 096 centroids, in the float64 bracket of
    test_gpu_kernels.test_centroid_scores (K1 v2, then FPB_K1=v1); padded columns are none at Q = 64."""
    if variant == "v1":
        monkeypatch.setenv("FPB_K1", "v1")
    else:
        monkeypatch.delenv("FPB_K1", raising=False)
    didx, q16 = table["didx"], table["q16"]
    st = didx.run_stages(q16, _params("APPROX_TWO_PASS"), upto="centroid_scores")
    torch.cuda.synchronize()
    table["peak"].sample()
    lay = st["layout"]
    assert lay.B * didx.num_centroids * lay.Qp > 1 << 31 and st["S"].numel() > 1 << 31 and lay.Qp == S_Q
    assert LAST[0] * didx.num_centroids * lay.Qp >= 1 << 31, "the checked rows start below element 2^31"
    C = table["t"].centroids.half().double().numpy()
    rows = np.r_[0:4096, K_BIG - 4096:K_BIG]
    differ = total = 0
    for b in LAST:
        qb = table["q"][b]
        S_ref = gk._f16(C[rows] @ qb.T)
        tol = gk._tol(S_ref, np.abs(C[rows]) @ np.abs(qb).T, DIM)
        got = st["S"][b, torch.from_numpy(rows).to(q16.device)].double().cpu().numpy()
        err = np.abs(got - S_ref)
        assert (err <= tol).all(), f"{variant} query {b}: S off by {err.max()}"
        differ += int((got != S_ref).sum())
        total += got.size
    assert differ / total < 0.01, f"{differ}/{total} S entries differ from S*"


@gpu
def test_table_position_in_batch_and_one_pass_fallback(table, monkeypatch):
    """Each of the last three queries gives the same bytes at every stage at B = 40 as alone at B = 1.  TWO_PASS falls
    back to one pass at this K: n_refine is 0 and the approximate scores equal EXACT_ALL's."""
    monkeypatch.delenv("FPB_K1", raising=False)
    didx, q16 = table["didx"], table["q16"]
    two = _params("APPROX_TWO_PASS")
    lay = didx.layout(S_B, S_Q, two)
    assert lay.hb_words * 4 > 96 * 1024, "the high-centroid bitmap fits: no fallback to test"
    st = didx.run_stages(q16, two)
    torch.cuda.synchronize()
    table["peak"].sample()
    keys = ("S", "cells", "n_cand", "cand", "approx", "n_refine", "n_rerank", "rerank", "rerank_approx", "exact",
            "ids", "scores", "counts")
    batch = {k: st[k][list(LAST)].clone() for k in keys}
    assert (st["n_refine"] == 0).all(), "TWO_PASS did not fall back to one pass"
    n_cand, approx = st["n_cand"].clone(), st["approx"].clone()  # the next run reuses the workspace
    ex = didx.run_stages(q16, _params("APPROX_EXACT_ALL"))
    torch.cuda.synchronize()
    assert torch.equal(ex["n_cand"], n_cand)
    for b in range(S_B):
        n = int(n_cand[b])
        assert n > 0
        assert torch.equal(ex["approx"][b, :n].view(torch.int32), approx[b, :n].view(torch.int32)), \
            f"query {b}: one-pass scores differ from EXACT_ALL"
    del st, ex
    for i, b in enumerate(LAST):
        one = didx.run_stages(q16[b: b + 1], two)
        torch.cuda.synchronize()
        n, r, c = int(batch["n_cand"][i]), int(batch["n_rerank"][i]), int(batch["counts"][i])
        assert r > 0 and c > 0
        for k in keys:
            x, y = one[k][0], batch[k][i]
            if k in ("cand", "approx"):
                x, y = x[:n], y[:n]
            elif k in ("rerank", "rerank_approx", "exact"):
                x, y = x[:r], y[:r]
            elif k in ("ids", "scores"):
                x, y = x[:c], y[:c]
            assert torch.equal(x.reshape(-1).view(torch.uint8), y.reshape(-1).view(torch.uint8)), \
                f"query {b}: {k} differs between B = {S_B} and B = 1"


# ---- without a GPU: the arithmetic of the fixtures -------------------------------------------------------------------
def _spans(plan: Plan) -> list[tuple[int, int]]:
    return [(int(plan.off[d]), int(plan.lengths[d])) for d in plan.probe]


@pytest.mark.parametrize("name", list(LAYOUTS))
def test_layout_plants_documents_at_the_boundaries(name):
    plan = _plan(name)
    spans = _spans(plan)
    want = {
        "edges": [(B1 - 300, 300), (B1, 0), (B1, 129), (B2 - 301, 300), (B2 - 1, 1), (B2, 0), (B2, 1), (B2 + 1, 129)],
        "straddle": [(B1 - 7, 300), (B2 - 7, 300)],
        "pass": [(B1 - 3, 129), (B2 - 3, 129)],
        "long": [(B1 - 1000, 2000), (B2 - 1000, 2000)],
    }[name]
    assert set(want) <= set(spans), sorted(set(want) - set(spans))
    for X in (B1, B2):
        nonempty = [(s, n) for s, n in spans if n > 0]
        hit = [(s, n) for s, n in nonempty if s < X <= s + n or s == X]
        assert hit, f"no probe document at {X}"
        empty = [s for s, n in spans if n == 0]
        assert any(abs(s - X) <= 1000 for s in empty), f"no empty document next to {X}"
    assert spans[: len(gk.LENGTHS)] == list(zip(np.concatenate([[0], np.cumsum(gk.LENGTHS)[:-1]]).tolist(),
                                                 gk.LENGTHS))
    assert plan.probe[-1] == len(plan.lengths) - 1 and plan.off[-1] == E_END and plan.lengths[-1] > 0
    assert E_END * PD > 1 << 32
    fillers = np.setdiff1d(np.arange(len(plan.lengths)), plan.probe)
    assert 60_000 < len(fillers) < 70_000 and plan.lengths[fillers].max() == FILL
    assert plan.lengths.max() == 2000 and (np.diff(plan.probe) > 0).all()


@pytest.mark.parametrize("name", list(LAYOUTS))
def test_deletes_move_documents_across_the_boundaries(name):
    """"one" moves a probe document from past each boundary to below it; "block" drops more than 2^25 tokens and
    moves a probe document with rows past 2^26 (above 4 GiB) to rows below 2^25 (below 2 GiB), and the index still
    ends past 2^25."""
    plan = _plan(name)
    for case, drop in _deletes(plan).items():
        assert not np.isin(drop, plan.probe).any()
        shift = np.array([plan.lengths[drop[drop < d]].sum() for d in plan.probe])
        old_end = plan.off[plan.probe] + plan.lengths[plan.probe]
        new_end = old_end - shift
        if case == "one":
            assert plan.lengths[drop].tolist() == [FILL]
            for X in (B1, B2):
                assert ((old_end > X) & (new_end <= X)).any(), f"{case}: nothing crosses {X}"
        else:
            assert plan.lengths[drop].sum() > B1
            assert ((old_end > B2) & (new_end <= B1) & (plan.lengths[plan.probe] > 0)).any()
            assert E_END - plan.lengths[drop].sum() > B1
        assert np.array_equal(_remap(plan.probe, drop), plan.probe - np.searchsorted(drop, plan.probe))


def test_score_table_crosses_two_to_the_31():
    """B K Qp > 2^31 elements, the last three queries' rows start past it, and at this K the bound pass's bitmap
    (K / 32 words) exceeds the 96 KiB it may take, so TWO_PASS runs one pass."""
    Qp = S_Q
    assert S_B * K_BIG * Qp > 1 << 31 and (S_B - 1) * K_BIG * Qp < 1 << 32
    assert LAST[0] * K_BIG * Qp >= 1 << 31
    assert K_BIG // 32 * 4 > 96 * 1024 and K_BIG > 786_432


def test_remap():
    assert _remap(np.array([0, 5, 9]), np.array([1, 2, 7])).tolist() == [0, 3, 6]
