"""1-bit residuals (nbits 1) at dim 128, through every layer: the decoder and every kernel built on it against the
float64 references of test_gpu_kernels.py and the oracle, the encode kernel against the oracle's bucketize + packbits,
the search stages against the oracle, and the FastPlaid surface.  dim 64 at nbits 1 stays refused.

The GPU tests reuse the float64 references and the checks of the existing suites (imported, not copied) at
(dim, nbits) = (128, 1).  The unmarked tests at the end run without a GPU: the refusals and the on-disk format."""

from __future__ import annotations

import ctypes
import json
import os

import numpy as np
import pytest
import torch

import test_gpu_build_kernels as bk
import test_gpu_exhaustive as ex
import test_gpu_kernels as gk
from util import (build_oracle_index, fp16_ulp_diff, make_docs, make_queries, oracle_exact_scores,
                  oracle_token_matrix, ranking_consistent, to_index_tensors)

from fast_plaid_b200 import engine
from oracle import index_oracle as io
from oracle import plaid_oracle as po

DIM, NBITS = 128, 1
gpu = pytest.mark.gpu


# ---- decoder: norm table and MaxSim (float64 reference of test_gpu_kernels.py) -----------------------------------------
@gpu
def test_token_norm_table(cuda_device):
    gk.test_token_norm_table(DIM, NBITS, cuda_device)


@gpu
@pytest.mark.parametrize("variant", ["default", "v1"])
@pytest.mark.parametrize("Q", gk.K5_Q)
def test_maxsim_stage(Q, variant, cuda_device, monkeypatch):
    """Every query length on the boundary-length index (empty documents, every length around a pass and tile
    boundary, a 2000-token document), with planted maxima, a query with zero rows and an all-negative one."""
    gk.test_maxsim_stage(DIM, NBITS, Q, variant, cuda_device, monkeypatch)


@gpu
@pytest.mark.parametrize("variant", ["default", "v1"])
@pytest.mark.parametrize("Q", [1, 17, 32, 33, 64, 128, 256])
def test_one_hot_maxima(Q, variant, cuda_device, monkeypatch):
    gk.test_one_hot_maxima(DIM, NBITS, Q, variant, cuda_device, monkeypatch)


@gpu
@pytest.mark.parametrize("Q", [16, 32, 64, 128, 256])
def test_maxsim_dispatch_never_reaches_v4_or_v5(Q, cuda_device, monkeypatch):
    """v4 and v5 decode dim 128 / nbits 4 only.  At nbits 1 every FPB_K5 setting gives the bytes of the generic
    kernel pinned by FPB_K5=v1, at every padded query length: v4 or v5 would read the 16-byte rows as 64-byte ones."""
    t, didx, ref = gk._index(DIM, NBITS)
    N = len(gk.LENGTHS)
    rerank = gk._rerank_lists(N, 2, N + 1, seed=Q)
    q = gk._planted_queries(ref, 2, Q)
    outs = {}
    for pin in ("v1", None, "v4", "v5"):
        if pin:
            monkeypatch.setenv("FPB_K5", pin)
        else:
            monkeypatch.delenv("FPB_K5", raising=False)
        outs[pin] = gk._maxsim(didx, q, rerank, np.array([N + 1, N + 1]))
    gk._check_scores(ref, q, rerank, np.array([N + 1, N + 1]), outs["v1"], f"nbits 1 Q={Q}")
    for pin, got in outs.items():
        assert np.array_equal(got.view(np.int32), outs["v1"].view(np.int32)), f"FPB_K5={pin} changes the scores"


# ---- K7: exhaustive scores --------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("Q", [1, 32, 100, 256])
def test_exhaustive_scores_against_float64(Q, cuda_device):
    """Every document of the boundary-length index: each score inside the bracket of the float64 reference's fp16
    maxima (plus the fp32 rounding of their sum), and the exact sum of the kernel's own maxima."""
    t, didx, ref = gk._index(DIM, NBITS)
    q = gk._planted_queries(ref, 3, Q)
    q16 = torch.from_numpy(q).half().to(cuda_device)
    got = didx.exhaustive_scores(q16).cpu().numpy().astype(np.float64)
    empty = ref.lens == 0
    for b in range(q.shape[0]):
        lo, hi, ms = ref.maxima(q[b])
        slack = Q * 2.0 ** -24 * np.abs(ms[~empty]).sum(1)
        s = got[b, ~empty]
        assert (got[b, empty] == np.float32(Q * gk.SENTINEL)).all()
        ok = (lo[~empty].sum(1) - slack <= s) & (s <= hi[~empty].sum(1) + slack)
        assert ok.all(), f"query {b}: {int((~ok).sum())} scores outside their bracket"
    B = q.shape[0]
    maxima = didx.exhaustive_scores(q16.reshape(B * Q, 1, DIM)).cpu().view(B, Q, -1).transpose(1, 2)
    assert np.array_equal(got.astype(np.float32), maxima.double().sum(-1).float().numpy())


@gpu
@pytest.mark.parametrize("Q", [1, 32, 100])
def test_exhaustive_scores_against_the_oracle(Q, cuda_device):
    docs = make_docs(150, 1, 40, dim=DIM, seed=61 + Q)
    oidx, _ = build_oracle_index(docs, nbits=NBITS)
    didx = ex._device_index(oidx, cuda_device)
    queries = make_queries(3, Q, dim=DIM, seed=62 + Q, docs=docs)
    got = didx.exhaustive_scores(queries.half().to(cuda_device)).cpu()
    ex._assert_scores_match(got, oidx, queries, f"nbits 1 Q={Q}", didx)


@gpu
def test_exhaustive_chunks_of_many_documents(cuda_device, monkeypatch):
    """FPB_K7_DOCS_PER_CHUNK 32, 13, 4, 2, 1 on ragged and empty documents: the oracle's scores, the same bytes."""
    ex.test_chunks_of_many_documents(DIM, NBITS, cuda_device, monkeypatch)


@gpu
def test_exhaustive_every_docs_per_chunk_gives_the_same_bytes(cuda_device, monkeypatch):
    t, didx, ref = gk._index(DIM, NBITS)
    q16 = torch.from_numpy(gk._planted_queries(ref, 2, 32)).half().to(cuda_device)
    first = None
    for dpc in range(1, 33):
        monkeypatch.setenv("FPB_K7_DOCS_PER_CHUNK", str(dpc))
        got = didx.exhaustive_scores(q16).cpu()
        first = got if first is None else first
        assert torch.equal(got.view(torch.int32), first.view(torch.int32)), f"{dpc} documents per chunk"


@gpu
def test_exhaustive_subset_scores_are_the_full_scan_scores(cuda_device):
    """The list walk (one filter for every query, then per-query lists with duplicates and ids outside the index)
    returns the full scan's scores bit for bit, ranked by (score desc, id asc)."""
    docs = make_docs(400, 1, 60, dim=DIM, seed=81)
    oidx, _ = build_oracle_index(docs, nbits=NBITS)
    didx = ex._device_index(oidx, cuda_device)
    q16 = make_queries(4, 32, dim=DIM, seed=82, docs=docs).half().to(cuda_device)
    every = didx.exhaustive_scores(q16).cpu()
    filt = list(range(399, 0, -7))
    per_query = [filt, [3, 3, 17, -1, 400], list(range(0, 400, 2)), [250]]
    for subset in ([filt] * 4, per_query):
        ids, scores, counts = (x.cpu() for x in didx.search_exhaustive(q16, 400, subset=subset))
        for b in range(4):
            members = sorted({d for d in subset[b] if 0 <= d < 400})
            want = sorted(members, key=lambda d: (-float(every[b, d]), d))
            n = int(counts[b])
            assert n == len(members) and ids[b, :n].tolist() == want, f"query {b}"
            assert torch.equal(scores[b, :n], every[b, want]), f"query {b}: subset scores differ from the full scan"


# ---- encode ----------------------------------------------------------------------------------------------------------
def _one_cutoff_cases() -> list[np.ndarray]:
    """The single cutoff on an fp16 value (a residual can equal it), strictly between two fp16 values, and at 0."""
    on = np.float32(np.float16(0.0137))
    nxt = bk._f16_step(np.float16(on), np.inf)
    between = np.float32(on + (np.float32(nxt) - on) * np.float32(0.375))
    assert on < between < np.float32(nxt)
    return [np.array([c], dtype=np.float32) for c in (on, between, np.float32(0.0))]


@gpu
@pytest.mark.parametrize("case", [0, 1, 2])
def test_pack_on_the_cutoff_is_byte_exact(case, cuda_device):
    """Residuals on, one step around and on either side of the cutoff, +-0, and every byte value: the kernel's bytes
    equal the spec packer's and the oracle's packbits."""
    cut = _one_cutoff_cases()[case]
    X = bk._edge_residuals(cut, NBITS)
    C = np.zeros((1, DIM), dtype=np.float16)  # one centroid at 0: the residual is the token itself
    codes, packed, _ = bk._encode(torch.from_numpy(X), torch.from_numpy(C), cuda_device, NBITS, torch.from_numpy(cut))
    assert int(codes.abs().sum()) == 0
    bucket = (cut[None, None, :] < X.astype(np.float32)[:, :, None]).sum(-1)
    if case == 0:
        assert (X == np.float16(cut[0])).any() and (bucket[X == np.float16(cut[0])] == 0).all()  # on the cutoff: 0
    want = bk._pack_ref(X, C, codes.numpy(), cut, NBITS)
    bits = torch.from_numpy(bucket[..., None].astype(np.int64))
    assert np.array_equal(want, io.packbits(bits.flatten()).reshape(X.shape[0], DIM // 8).numpy())
    bad = np.argwhere(packed.numpy() != want)
    assert bad.shape[0] == 0, f"{bad.shape[0]} bytes differ; first (row, byte): {bad[:8].tolist()}"


@gpu
@pytest.mark.parametrize("family", ["ternary", "dense"])
def test_encode_codes_and_bytes_are_bit_exact(family, cuda_device):
    """Exact inputs (every score exact in fp32): codes equal the float64 argmax with the smallest-id tie rule, and
    the packed bytes equal bucketize + packbits of the fp16 residuals."""
    K, n = 1000, 3000
    X16, C16, _, _ = bk._exact_inputs(K, n, family, kmeans=False, seed=K * 7 + n)
    cut = torch.tensor([0.0])
    codes, packed, _ = bk._encode(X16, C16, cuda_device, NBITS, cut)
    assert torch.equal(codes, bk._exact_reference(X16, C16, False, cuda_device).cpu().long())
    want = bk._pack_ref(X16.numpy(), C16.numpy(), codes.numpy(), cut.numpy(), NBITS)
    assert np.array_equal(packed.numpy(), want)


@gpu
def test_gpu_build_is_byte_identical_to_the_cpu_build(tmp_path, cuda_device):
    bk.test_gpu_build_is_byte_identical_to_the_cpu_build(NBITS, tmp_path, cuda_device)


# ---- search stages against the oracle ---------------------------------------------------------------------------------
_parity: dict = {}


def _parity_setup(Q: int, device: str):
    if Q not in _parity:
        from fast_plaid_b200.engine import FPB_FLAG_APPROX_EXACT_ALL, DeviceIndex

        docs = make_docs(500, 20, 80, dim=DIM, seed=1234)
        oidx, _ = build_oracle_index(docs, nbits=NBITS)
        didx = DeviceIndex(to_index_tensors(oidx), device)
        queries = make_queries(4 if Q < 256 else 2, Q, dim=DIM, seed=4321, docs=docs)
        params = DeviceIndex.make_params(10, 256, 8)
        st = didx.run_stages(queries.half().to(device), DeviceIndex.with_flags(params, FPB_FLAG_APPROX_EXACT_ALL))
        st = {k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in st.items() if k != "workspace"}
        torch.cuda.synchronize()
        _parity[Q] = (oidx, didx, queries, params, st)
    return _parity[Q]


@gpu
@pytest.mark.parametrize("Q", [32, 100, 256])
def test_stages_match_the_oracle(Q, cuda_device):
    """Given the GPU's own S: probe cells, candidates and the re-rank list exactly, approximate scores exactly (or
    within fp32 summation order); exact scores within 1e-3 relative, almost all bit-identical; final ids and ranks
    those of the oracle's canonical search."""
    oidx, didx, queries, params, st = _parity_setup(Q, cuda_device)
    flips = total = 0
    for b in range(queries.shape[0]):
        S_b = st["S"][b, :, :Q].cpu().contiguous()
        kw = dict(ties="canonical", return_stages=True, inject={"S": S_b})
        ref = po.search_one(queries[b], oidx, params.n_ivf_probe, 2000, params.n_full_scores, params.top_k, **kw)
        cells = torch.unique(st["cells"][b].cpu().flatten().long())
        assert torch.equal(cells[cells >= 0], ref["cells"]), f"query {b}: probed cells differ"
        n = int(st["n_cand"][b])
        assert torch.equal(st["cand"][b, :n].cpu().long(), ref["candidates"]), f"query {b}: candidates differ"
        approx = st["approx"][b, :n].cpu()
        if not torch.equal(approx, ref["approx"]):
            rel = ((approx - ref["approx"]).abs() / ref["approx"].abs().clamp_min(1.0)).max()
            assert float(rel) < 1e-6, f"query {b}: approx scores differ by {float(rel)}"
            kw["inject"] = {"S": S_b, "approx": approx}
            ref = po.search_one(queries[b], oidx, params.n_ivf_probe, 2000, params.n_full_scores, params.top_k, **kw)
        r = int(st["n_rerank"][b])
        rer = st["rerank"][b, :r].cpu().long()
        assert torch.equal(rer, ref["rerank"]), f"query {b}: re-rank list differs"
        oracle_exact = oracle_exact_scores(oidx, queries[b], rer.tolist())
        got = st["exact"][b, :r].cpu()
        rel = (got - oracle_exact).abs() / oracle_exact.abs().clamp_min(1.0)
        assert float(rel.max()) < 1e-3, f"query {b}: exact scores off by {float(rel.max())} relative"
        flips += int((got != oracle_exact).sum())
        total += r
        cnt = int(st["counts"][b])
        assert cnt == min(params.top_k, len(ref["ids"]))
        ok, why = ranking_consistent(st["ids"][b, :cnt].cpu().tolist(), st["scores"][b, :cnt].cpu().tolist(),
                                     dict(zip(ref["ids"], ref["scores"])), 1e-3,
                                     fallback=lambda d, b=b: float(oracle_exact_scores(oidx, queries[b], [d])[0]))
        assert ok, f"query {b}: {why}"
    # a score is not bit-identical as soon as one of its Q fp16 maxima rounds the other way (the CPU matmul and the
    # tensor cores accumulate a dot product in different orders), so the share grows with Q
    bound = 0.05 if Q <= 32 else 0.1 if Q <= 100 else 0.25
    assert flips / max(total, 1) < bound, f"{flips}/{total} exact scores not bit-identical"


@gpu
def test_reconstruct_and_token_scores_match_the_oracle(cuda_device):
    oidx, didx, queries, params, st = _parity_setup(32, cuda_device)
    docs = [0, 5, 17, 499]
    bad = tot = 0
    for d, g in zip(docs, didx.reconstruct(docs)):
        sel = torch.tensor([d])
        codes, _ = po.ragged_lookup(oidx.doc_codes, oidx.doc_offsets, oidx.doc_lengths, sel)
        res, _ = po.ragged_lookup(oidx.doc_residuals, oidx.doc_offsets, oidx.doc_lengths, sel)
        ref = po.decompress_residuals(res, oidx.bucket_weights, oidx.byte_reversed_bits_map,
                                      oidx.bucket_weight_indices_lookup, codes, oidx.centroids, oidx.dim, oidx.nbits)
        dlt = fp16_ulp_diff(g.cpu(), ref)
        assert int(dlt.max()) <= 1
        bad += int((dlt > 0).sum())
        tot += dlt.numel()
    assert bad / tot < 5e-3
    B, Q = queries.shape[0], queries.shape[1]
    pairs = [(b, int(d)) for b in range(B) for d in st["ids"][b, : int(st["counts"][b])].tolist()]
    mats = didx.token_scores(queries.half().to(cuda_device), torch.tensor([p[0] for p in pairs], dtype=torch.int32),
                             torch.tensor([p[1] for p in pairs], dtype=torch.int32)).cpu()
    bad = tot = 0
    for k, (b, d) in enumerate(pairs):
        ref = oracle_token_matrix(oidx, queries[b], d)
        got = mats[k, : ref.shape[1], :].transpose(0, 1)
        dlt = fp16_ulp_diff(got, ref)
        assert float((got.float() - ref.float()).abs()[dlt > 1].max() if bool((dlt > 1).any()) else 0.0) <= 1e-3
        bad += int((dlt > 0).sum())
        tot += dlt.numel()
    assert bad / max(tot, 1) < 5e-3, f"{bad}/{tot} token scores differ by one ulp"


# ---- the FastPlaid surface --------------------------------------------------------------------------------------------
@gpu
def test_fastplaid_round_trip(tmp_path, cuda_device):
    """create -> search (with and without subset) -> update past start_from_scratch (append) -> delete -> reload;
    get_embeddings and search_token_scores against the oracle, search_exhaustive, and a (0, 1) shard."""
    from fast_plaid_b200 import search
    from fast_plaid_b200.engine import DeviceIndex
    from fast_plaid_b200.index import store

    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device=cuda_device)
    docs = make_docs(300, 20, 80, seed=11)
    fp.create(docs, kmeans_niters=4, nbits=NBITS, start_from_scratch=100)
    assert json.load(open(os.path.join(path, "plan.json")))["nbits"] == 1
    queries = make_queries(6, 30, seed=12, docs=docs)

    def oracle_of(p):
        data = store.read_index(p)
        assert data.nbits == 1 and data.doc_residuals.shape[1] == 16
        return po.OracleIndex(data.nbits, data.centroids, data.bucket_weights, data.ivf, data.ivf_lengths.long(),
                              data.doc_codes, data.doc_residuals, data.doc_lengths)

    def check(res, oidx, subset=None):
        for b in range(len(res)):
            sub = None if subset is None else torch.tensor(subset, dtype=torch.int64)
            ref = po.search_one(queries[b], oidx, top_k=10**9, subset=sub, return_stages=True)
            ok, why = ranking_consistent([d for d, _ in res[b]], [s for _, s in res[b]],
                                         dict(zip(ref["ids"], ref["scores"])), 1e-3,
                                         fallback=lambda d, b=b: float(oracle_exact_scores(oidx, queries[b], [d])[0]))
            assert ok, f"query {b}: {why}"

    oidx = oracle_of(path)
    check(fp.search(queries, top_k=10), oidx)
    sub = list(range(0, 300, 3))
    r_sub = fp.search(queries, top_k=10, subset=sub)
    assert all(d in set(sub) for r in r_sub for d, _ in r)
    check(r_sub, oidx, sub)
    # append with the existing codec (more new documents than start_from_scratch), delete, reload from disk
    cent = store.read_index(path).centroids.clone()
    fp.update(make_docs(120, 20, 80, seed=13), start_from_scratch=100)
    assert torch.equal(store.read_index(path).centroids, cent) and store.read_index(path).num_documents == 420
    fp.delete(list(range(0, 100)))
    fp.close()
    fp = search.FastPlaid(path, device=cuda_device)
    oidx = oracle_of(path)
    assert int(oidx.doc_lengths.shape[0]) == 320
    res = fp.search(queries, top_k=10)
    assert all(0 <= d < 320 for r in res for d, _ in r)
    check(res, oidx)
    # decompressed embeddings
    ids = [0, 7, 250, 319]
    for d, e in zip(ids, fp.get_embeddings(ids)):
        sel = torch.tensor([d])
        codes, _ = po.ragged_lookup(oidx.doc_codes, oidx.doc_offsets, oidx.doc_lengths, sel)
        rr, _ = po.ragged_lookup(oidx.doc_residuals, oidx.doc_offsets, oidx.doc_lengths, sel)
        ref = po.decompress_residuals(rr, oidx.bucket_weights, oidx.byte_reversed_bits_map,
                                      oidx.bucket_weight_indices_lookup, codes, oidx.centroids, oidx.dim, oidx.nbits)
        assert e.shape == ref.shape and int(fp16_ulp_diff(e.cpu(), ref).max()) <= 1
    # token-score matrices
    for b, rq in enumerate(fp.search_token_scores(queries[:2], top_k=3)):
        for d, s, m in rq:
            ref = oracle_token_matrix(oidx, queries[b], d)
            assert m.shape == ref.shape
            dlt = fp16_ulp_diff(m.cpu(), ref)
            assert float((m.cpu().float() - ref.float()).abs()[dlt > 1].max() if bool((dlt > 1).any()) else 0.0) <= 1e-3
            assert abs(float(m.float().max(dim=1).values.sum()) - s) <= 1e-3 * max(1.0, abs(s))
    # exhaustive search: its top 10 under the oracle's exact score of every document
    every = [oracle_exact_scores(oidx, queries[b], list(range(320))).tolist() for b in range(queries.shape[0])]
    for b, r in enumerate(fp.search_exhaustive(queries, top_k=10)):
        ok, why = ranking_consistent([d for d, _ in r], [s for _, s in r], dict(enumerate(every[b])), 1e-3)
        assert ok, f"exhaustive query {b}: {why}"
        assert abs(r[0][1] - max(every[b])) <= 1e-3 * max(1.0, abs(max(every[b])))
    # one shard of one: the same results as the unsharded search
    whole = fp.search(queries, top_k=10)
    didx = DeviceIndex(to_index_tensors(oidx), cuda_device)
    sharded = search.FastPlaid.from_device_index(didx, shard=(0, 1))
    assert sharded.search(queries, top_k=10) == whole
    sharded.close()
    fp.close()


# ---- without a GPU: refusals and the index format ----------------------------------------------------------------------
def test_check_supported():
    engine.check_supported(128, 1)
    for dim, nbits in ((128, 2), (128, 4), (64, 2), (64, 4)):
        engine.check_supported(dim, nbits)
    for dim, nbits, words in ((64, 1, ("dim", "nbits")), (96, 4, ("dim",)), (128, 3, ("nbits",)), (128, 8, ("nbits",))):
        with pytest.raises(ValueError) as e:
            engine.check_supported(dim, nbits)
        assert all(w in str(e.value) for w in words), (dim, nbits, str(e.value))
    # the Python copy of the supported set is the library's: with NULL pointers fpb_index_create refuses an unsupported
    # pair and stops at the pointers for a supported one, both before any CUDA call
    lib = engine.load_library()
    handle = ctypes.c_void_p()
    for dim in (32, 64, 96, 128, 256):
        for nbits in (0, 1, 2, 3, 4, 8):
            try:
                engine.check_supported(dim, nbits)
                refused = False
            except ValueError:
                refused = True
            rc = lib.fpb_index_create(ctypes.byref(handle), 0, nbits, dim, 16, None, None, 0, None, None, None, None,
                                      None, None, 0, 0, 0)
            assert rc == (engine.FPB_ERR_UNSUPPORTED if refused else engine.FPB_ERR_INVALID), (dim, nbits, rc)


def test_cabi_refuses_dim_64_at_nbits_1_before_any_cuda_call():
    lib = engine.load_library()
    handle = ctypes.c_void_p()
    rc = lib.fpb_index_create(ctypes.byref(handle), 0, 1, 64, 16, None, None, 0, None, None, None, None, None, None, 0, 0, 0)
    assert rc == engine.FPB_ERR_UNSUPPORTED
    msg = lib.fpb_last_error()
    assert b"dim=64" in msg and b"nbits" in msg and b"nbits 1 at dim 128" in msg, msg
    # the old refusals keep their words
    rc = lib.fpb_index_create(ctypes.byref(handle), 0, 3, 128, 16, None, None, 0, None, None, None, None, None, None, 0, 0, 0)
    assert rc == engine.FPB_ERR_UNSUPPORTED and b"nbits" in lib.fpb_last_error()
    rc = lib.fpb_index_create(ctypes.byref(handle), 0, 4, 100, 16, None, None, 0, None, None, None, None, None, None, 0, 0, 0)
    assert rc == engine.FPB_ERR_UNSUPPORTED and b"dim" in lib.fpb_last_error()
    for nbits, dim in ((1, 64), (4, 64), (2, 96), (3, 128), (8, 128)):
        assert lib.fpb_encode(0, nbits, dim, 16, None, None, 10, None, None, None, None) == engine.FPB_ERR_UNSUPPORTED
        msg = lib.fpb_last_error()
        assert b"dim=128 with nbits 2 or 4" in msg and b"dim=128 with nbits 1" in msg, msg
    # accepted shapes get past the shape check (and stop at the NULL pointers, still before any CUDA call)
    assert lib.fpb_encode(0, 1, 128, 16, None, None, 10, None, None, None, None) == engine.FPB_ERR_INVALID
    rc = lib.fpb_index_create(ctypes.byref(handle), 0, 1, 128, 16, None, None, 0, None, None, None, None, None, None, 0, 0, 0)
    assert rc == engine.FPB_ERR_INVALID


def test_pack_reference_agrees_with_the_oracle_packbits():
    rng = np.random.default_rng(3)
    bucket = rng.integers(0, 2, (64, DIM))
    bits = torch.from_numpy(bucket[..., None].astype(np.int64))
    assert np.array_equal(bk._pack_buckets(bucket, NBITS), io.packbits(bits.flatten()).reshape(64, DIM // 8).numpy())


def test_cpu_build_matches_the_oracle_builder(tmp_path):
    """A CPU build at nbits 1 against the oracle's builder, byte for byte, and its on-disk shapes."""
    from fast_plaid_b200 import search
    from fast_plaid_b200.index import store

    path = str(tmp_path / "idx")
    docs = make_docs(260, 8, 50, seed=321)
    search.FastPlaid(path, device="cpu").create(docs, kmeans_niters=2, batch_size=100, seed=7, nbits=NBITS)
    data = store.read_index(path)
    oidx, extra = io.build_index(docs, data.centroids, nbits=NBITS, batch_size=100, seed=7)
    assert torch.equal(oidx.doc_codes, data.doc_codes)
    assert torch.equal(oidx.doc_residuals, data.doc_residuals)
    assert torch.equal(oidx.ivf, data.ivf) and torch.equal(oidx.ivf_lengths, data.ivf_lengths.long())
    assert torch.equal(oidx.bucket_weights, data.bucket_weights)
    assert torch.equal(extra["bucket_cutoffs"].half(), data.bucket_cutoffs)
    assert np.load(os.path.join(path, "bucket_cutoffs.npy")).shape == (1,)
    assert np.load(os.path.join(path, "bucket_weights.npy")).shape == (2,)
    for i in range(3):
        c = np.load(os.path.join(path, f"{i}.codes.npy"))
        r = np.load(os.path.join(path, f"{i}.residuals.npy"))
        assert r.dtype == np.uint8 and r.shape == (c.shape[0], 16)
    assert json.load(open(os.path.join(path, "plan.json"))) == {"nbits": 1, "num_chunks": 3}
    assert json.load(open(os.path.join(path, "metadata.json")))["nbits"] == 1
