"""Search filters in their device form (csrc/filter.cu): packed bitmaps over global document ids, built from id
tensors and bool masks on the GPU, expanded once per distinct filter.  The contract: for the same documents every
filter form returns the bytes of the per-query list path, in `search`, `search_exhaustive` and
`search_token_scores`, sharded or not."""

from __future__ import annotations

import ctypes
import random

import pytest
import torch
from util import build_oracle_index, make_docs, make_queries, to_index_tensors

from fast_plaid_b200 import engine
from fast_plaid_b200.engine import DeviceIndex, Filter, IndexTensors, shard_tensors

CODECS = [(128, 4), (128, 2), (64, 4), (64, 2), (128, 1)]
N_DOCS = 300  # 300 % 32 = 12: the last word of every document bitmap is partial
B, Q = 6, 32


def _bits(bitmap: torch.Tensor, n_bits: int) -> torch.Tensor:
    """bool [F, n_bits] of an int32 [F, words] bitmap."""
    w = bitmap.cpu().to(torch.int64) & 0xFFFFFFFF
    shifts = torch.arange(32, dtype=torch.int64)
    return (((w.unsqueeze(-1) >> shifts) & 1).bool().reshape(w.shape[0], -1))[:, :n_bits]


def _mask_of(sets: list[list[int]], n_bits: int) -> torch.Tensor:
    m = torch.zeros((len(sets), n_bits), dtype=torch.bool)
    for f, s in enumerate(sets):
        ok = [i for i in s if 0 <= i < n_bits]
        if ok:
            m[f, torch.tensor(ok)] = True
    return m


def _padded(sets: list[list[int]]) -> torch.Tensor:
    L = max(1, max(len(s) for s in sets))
    return torch.tensor([s + [-1] * (L - len(s)) for s in sets], dtype=torch.int64)


# ---- kernels 1 and 2: ids and masks into bitmaps ------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n_bits", [1, 31, 32, 33, 10**6 + 7])
def test_bitmaps_from_ids_and_masks_equal_torch(n_bits, cuda_device):
    g = torch.Generator().manual_seed(n_bits)
    rows = []
    for f in range(4):
        ids = torch.randint(-3, n_bits + 40, (f * 50 + 7,), generator=g)
        ids = torch.cat([ids, ids[: len(ids) // 2], torch.tensor([-1, n_bits, n_bits + 31, 2**40, -(2**40)])])
        rows.append(ids[torch.randperm(len(ids), generator=g)].tolist())
    rows.append([])  # an empty row
    expect = _mask_of(rows, n_bits)
    # one filter per row: a padded [F, L] tensor, and ragged rows through row offsets
    f2 = Filter.from_ids(_padded(rows).to(cuda_device), n_bits, cuda_device, len(rows))
    assert f2.bitmap.shape == (len(rows), (n_bits + 31) // 32)
    assert torch.equal(_bits(f2.bitmap, n_bits), expect)
    assert f2.query_filter == list(range(len(rows)))
    flat = torch.tensor([i for r in rows for i in r], dtype=torch.int64, device=cuda_device)
    offs = torch.tensor([0] + [sum(len(r) for r in rows[: f + 1]) for f in range(len(rows))], device=cuda_device)
    bm = torch.full((len(rows), (n_bits + 31) // 32), -1, dtype=torch.int32, device=cuda_device)
    lib = engine.load_library()
    assert lib.fpb_filter_from_ids(0, flat.data_ptr(), flat.numel(), len(rows), offs.data_ptr(), n_bits,
                                   bm.data_ptr(), None) == 0
    assert torch.equal(_bits(bm, n_bits), expect) and torch.equal(bm, f2.bitmap)
    # bits past n_bits stay clear in the last word
    assert torch.equal(_bits(bm, bm.shape[1] * 32)[:, n_bits:], torch.zeros_like(_bits(bm, bm.shape[1] * 32)[:, n_bits:]))
    # one shared row
    f1 = Filter.from_ids(torch.tensor(rows[2]), n_bits, cuda_device, 3)
    assert torch.equal(_bits(f1.bitmap, n_bits), expect[2:3]) and f1.query_filter == [0, 0, 0]
    # masks, bool and uint8, shared and per row
    fm = Filter.from_mask(expect.to(cuda_device), cuda_device, len(rows))
    assert torch.equal(fm.bitmap, f2.bitmap)
    bm8 = torch.full_like(bm, -1)
    m8 = (expect.to(torch.uint8) * 7).to(cuda_device)
    assert lib.fpb_filter_from_mask(0, m8.data_ptr(), len(rows), n_bits, bm8.data_ptr(), None) == 0
    assert torch.equal(bm8, f2.bitmap)
    fs = Filter.from_mask(expect[1], cuda_device, 2)
    assert torch.equal(fs.bitmap, f2.bitmap[1:2]) and fs.query_filter == [0, 0]


# ---- kernels 3 and 4: range expansion and the centroid bitmap ----------------------------------------------------
def _oracle(dim: int = 128, nbits: int = 4, n: int = N_DOCS, seed: int = 5):
    docs = make_docs(n, 1, 40, dim=dim, seed=seed)
    oidx, _ = build_oracle_index(docs, nbits=nbits, kmeans_niters=2)
    return oidx, docs


def _expected_centroids(t: IndexTensors, local_docs: torch.Tensor, K: int) -> torch.Tensor:
    offs = torch.zeros(t.doc_lengths.shape[0] + 1, dtype=torch.int64)
    offs[1:] = t.doc_lengths.cpu().to(torch.int64).cumsum(0)
    codes = t.doc_codes.cpu().to(torch.int64)
    sel = [codes[offs[d]:offs[d + 1]] for d in local_docs.tolist()]
    m = torch.zeros(K, dtype=torch.bool)
    if sel:
        m[torch.unique(torch.cat(sel))] = True
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("base", [0, 1, 17, 31, 32 * 5 + 17])
def test_expansion_of_an_unaligned_range(base, cuda_device):
    """An index holding global ids [base, base + 300): its document bitmap is the filter's bits of that range, bits
    past the range clear, and its centroid bitmap the unique codes of those documents; sbitmap, cbitmap and clist
    equal the list path's for the same ids."""
    oidx, docs = _oracle()
    t = to_index_tensors(oidx)
    didx = DeviceIndex(t, cuda_device, doc_id_base=base)
    n_bits = base + N_DOCS + 40
    rng = random.Random(base)
    sets = [sorted(rng.sample(range(n_bits), 120)), [base, base + N_DOCS - 1], list(range(n_bits)), [],
            [base + N_DOCS + 3, max(0, base - 1)], sorted(rng.sample(range(base, base + N_DOCS), 3))]
    q16 = make_queries(len(sets), Q, seed=7, docs=docs).half().to(cuda_device)
    params = DeviceIndex.make_params(10, 64, 8)
    for filt in (Filter.from_ids(_padded(sets).to(cuda_device), n_bits, cuda_device, len(sets)),
                 Filter.from_mask(_mask_of(sets, n_bits).to(cuda_device), cuda_device, len(sets))):
        got = didx.run_stages(q16, params, upto="filter", filter=filt)
        got = {k: v.clone() for k, v in got.items() if isinstance(v, torch.Tensor)}  # views of the workspace
        ref = didx.run_stages(q16, params, upto="subset", subset=[list(s) for s in sets])
        sb = _bits(got["sbitmap"], got["sbitmap"].shape[1] * 32)
        for b, s in enumerate(sets):
            local = torch.tensor(sorted({i - base for i in s if base <= i < base + N_DOCS}), dtype=torch.int64)
            exp = torch.zeros(sb.shape[1], dtype=torch.bool)
            exp[local] = True
            assert torch.equal(sb[b], exp), b
            K = didx.num_centroids
            cb = _bits(got["cbitmap"][b:b + 1], K)[0]
            assert torch.equal(cb, _expected_centroids(t, local, K)), b
            assert not _bits(got["cbitmap"][b:b + 1], got["cbitmap"].shape[1] * 32)[0, K:].any()
        for key in ("sbitmap", "cbitmap", "n_clist"):
            assert torch.equal(got[key], ref[key]), key
        for b in range(len(sets)):
            n = int(got["n_clist"][b])
            assert torch.equal(got["clist"][b, :n], ref["clist"][b, :n])


def _random_index(K: int, n_docs: int, device: str, seed: int = 0, empty: tuple = ()) -> IndexTensors:
    """A compress_only index of random codes over K centroids (dim 128, nbits 4), with empty documents at `empty`."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, 300, (n_docs,), generator=g)
    for d in empty:
        lens[d] = 0
    E = int(lens.sum())
    cent = torch.nn.functional.normalize(torch.randn(K, 128, generator=g), dim=-1).half()
    return IndexTensors(4, cent.to(device), torch.linspace(-0.1, 0.1, 16).to(device), lens,
                        torch.randint(0, K, (E,), generator=g, dtype=torch.int32).to(device),
                        torch.randint(0, 256, (E, 64), generator=g, dtype=torch.uint8).to(device), None, None)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1000, 262_144, 2_097_152 + 5])
def test_centroid_bitmap_equals_torch_unique(K, cuda_device):
    """K not a multiple of 32, cfg3's K, and a K whose bitmap does not fit in shared memory (the global-atomic
    path); empty documents, an empty filter, a filter of empty documents only, and shared filters."""
    empty = (0, 5, 63, 64)
    t = _random_index(K, 700, cuda_device, seed=K, empty=empty)
    didx = DeviceIndex(t, cuda_device)
    # the shared-memory bitmap of the kernel holds cbitmap_words = K / 32 + 1 words
    in_shared = ((K + 31) // 32 + 1) * 4 <= torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    assert in_shared == (K < 1_800_000)
    rng = random.Random(K)
    sets = [sorted(rng.sample(range(700), 350)), [], list(empty), sorted(rng.sample(range(700), 7))]
    filt = Filter.from_ids(_padded(sets).to(cuda_device), 700, cuda_device, len(sets))
    filt = Filter(filt.bitmap, [0, 1, 0, 2, 3, 2], 700)  # queries 0 and 2 share filter 0, 3 and 5 filter 2
    q16 = torch.nn.functional.normalize(torch.randn(6, 4, 128), dim=-1).half().to(cuda_device)
    got = didx.run_stages(q16, DeviceIndex.make_params(10, 64, 8), upto="filter", filter=filt)
    for b, f in enumerate(filt.query_filter):
        exp = _expected_centroids(t, torch.tensor(sets[f], dtype=torch.int64), K)
        assert torch.equal(_bits(got["cbitmap"][b:b + 1], K)[0], exp), (b, f)
        n = int(got["n_clist"][b])
        assert n == int(exp.sum()) and torch.equal(got["clist"][b, :n].cpu().to(torch.int64), exp.nonzero().flatten())


# ---- every form against the list path, at every codec ------------------------------------------------------------
@pytest.fixture(scope="module", params=CODECS, ids=[f"d{d}n{n}" for d, n in CODECS])
def codec_index(request):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    dim, nbits = request.param
    oidx, docs = _oracle(dim, nbits, seed=11 + dim + nbits)
    didx = DeviceIndex(to_index_tensors(oidx), "cuda:0")
    q16 = make_queries(B, Q, dim=dim, seed=13, docs=docs).half().to("cuda:0")
    return didx, q16


def _shared_sets(n: int, seed: int) -> dict[str, list[int]]:
    rng = random.Random(seed)
    return {"empty": [], "one": [n // 3], "all": list(range(n)), "range": list(range(40, 140)),
            "1pct": rng.sample(range(n), max(1, n // 100)), "50pct": rng.sample(range(n), n // 2)}


def _forms(sets: list[list[int]], n: int, device: str, shared: bool):
    """Every device form of the per-query sets `sets` (all equal when shared)."""
    if shared:
        ids = torch.tensor(sets[0], dtype=torch.int64)
        yield "ids", Filter.from_ids(ids, n, device, len(sets))
        yield "ids-cuda", Filter.from_ids(ids.to(device), n, device, len(sets))
        yield "mask", Filter.from_mask(_mask_of(sets[:1], n)[0].to(device), device, len(sets))
    yield "rows", Filter.from_ids(_padded(sets).to(device), n, device, len(sets))
    yield "masks", Filter.from_mask(_mask_of(sets, n), device, len(sets))


@pytest.mark.gpu
@pytest.mark.parametrize("n_probe", [8, 32, 33, 256])
def test_search_forms_equal_the_list_path(codec_index, n_probe):
    didx, q16 = codec_index
    n = didx.num_documents
    params = DeviceIndex.make_params(10, 64, n_probe)
    cases = [[s] * B for s in _shared_sets(n, n_probe).values()]
    rng = random.Random(n_probe)
    cases.append([rng.sample(range(n), rng.randrange(1, n)) for _ in range(B)])  # per-query sets that differ
    for sets in cases:
        ref = didx.search(q16, params, subset=[list(s) for s in sets])
        for name, filt in _forms(sets, n, "cuda:0", shared=all(s == sets[0] for s in sets)):
            got = didx.search(q16, params, filter=filt)
            for r, g_ in zip(ref, got):
                assert torch.equal(r, g_), (name, n_probe, len(sets[0]))


@pytest.mark.gpu
def test_exhaustive_forms_equal_the_list_path_and_the_filtered_full_scan(codec_index):
    didx, q16 = codec_index
    n = didx.num_documents
    every = didx.exhaustive_scores(q16).cpu()
    cases = [[s] * B for s in _shared_sets(n, 3).values()]
    rng = random.Random(4)
    cases.append([rng.sample(range(n), rng.randrange(1, n)) for _ in range(B)])
    for k in (1, 10, n + 3):
        for sets in cases:
            ref = didx.search_exhaustive(q16, k, subset=[list(s) for s in sets])
            forms = list(_forms(sets, n, "cuda:0", shared=all(s == sets[0] for s in sets)))
            forms.append(("id-rows", _padded(sets).to("cuda:0")))
            for name, filt in forms:
                got = (didx.search_exhaustive(q16, k, subset=filt) if name == "id-rows"
                       else didx.search_exhaustive(q16, k, filter=filt))
                for r, g_ in zip(ref, got):
                    assert torch.equal(r, g_), (name, k, len(sets[0]))
            ids, sc, counts = (t.cpu() for t in ref)
            for b, s in enumerate(sets):
                exp = sorted(set(s), key=lambda d: (-float(every[b, d]), d))[:k]
                assert int(counts[b]) == len(exp) and ids[b, : len(exp)].tolist() == exp
                assert torch.equal(sc[b, : len(exp)], every[b, torch.tensor(exp, dtype=torch.int64)]) if exp else True


@pytest.mark.gpu
def test_exhaustive_filter_batch_split_gives_the_same_bytes(codec_index):
    """A budget that splits the batch into calls of one query: per-query filters then pass one row each, and a
    non-contiguous set of shared rows goes through a gathered copy."""
    didx, q16 = codec_index
    n = didx.num_documents
    rng = random.Random(9)
    sets = [rng.sample(range(n), 50) for _ in range(3)]
    filt = Filter.from_ids(_padded(sets).to("cuda:0"), n, "cuda:0", 3)
    filt = Filter(filt.bitmap, [0, 2, 0, 1, 2, 0], n)
    per = [sets[f] for f in filt.query_filter]
    ref = didx.search_exhaustive(q16, 10, subset=per)
    for budget in (6 << 30, 1):
        got = didx.search_exhaustive(q16, 10, budget_bytes=budget, filter=filt)
        for r, g_ in zip(ref, got):
            assert torch.equal(r, g_), budget


# ---- FastPlaid surface --------------------------------------------------------------------------------------------
def _fastplaid(didx):
    from fast_plaid_b200 import search

    return search.FastPlaid.from_device_index(didx)


@pytest.mark.gpu
def test_fastplaid_forms_equal_the_list_forms(cuda_device):
    """Every `subset=` form of search, search_exhaustive and search_token_scores, on CPU and CUDA tensors, against
    per-query lists; the broadcast list and id forms against per-query copies, byte for byte."""
    oidx, docs = _oracle()
    didx = DeviceIndex(to_index_tensors(oidx), cuda_device)
    fp = _fastplaid(didx)
    queries = make_queries(B, Q, seed=21, docs=docs)
    n = didx.num_documents
    rng = random.Random(22)
    shared = rng.sample(range(n), 60)
    per = [rng.sample(range(n), 40) for _ in range(B)]
    mask = _mask_of([shared], n)[0]
    masks = _mask_of(per, n)
    for fn in (lambda s: fp.search(queries, top_k=10, n_ivf_probe=32, subset=s),
               lambda s: fp.search_exhaustive(queries, top_k=10, subset=s)):
        ref_shared = fn([list(shared) for _ in range(B)])
        for form in (shared, torch.tensor(shared), torch.tensor(shared, device=cuda_device), mask,
                     mask.to(cuda_device), torch.tensor(shared, dtype=torch.int32)):
            assert fn(form) == ref_shared
        ref_one = fn([[shared[0]] for _ in range(B)])
        assert fn(shared[0]) == ref_one and fn([shared[0]]) == ref_one
        ref_per = fn(per)
        for form in (_padded(per), _padded(per).to(cuda_device), masks, masks.to(cuda_device)):
            assert fn(form) == ref_per
        assert fn(torch.zeros(n, dtype=torch.bool)) == fn([[] for _ in range(B)])
    ts_ref = fp.search_token_scores(queries, top_k=5, subset=per)
    ts = fp.search_token_scores(queries, top_k=5, subset=masks.to(cuda_device))
    assert [[(d, s) for d, s, _ in r] for r in ts] == [[(d, s) for d, s, _ in r] for r in ts_ref]
    assert all(torch.equal(a[2], b[2]) for ra, rb in zip(ts, ts_ref) for a, b in zip(ra, rb))


@pytest.mark.gpu
def test_fastplaid_refusals(cuda_device):
    oidx, docs = _oracle()
    fp = _fastplaid(DeviceIndex(to_index_tensors(oidx), cuda_device))
    queries = make_queries(3, Q, seed=23, docs=docs)
    for call in (fp.search, fp.search_exhaustive):
        with pytest.raises(ValueError, match="float32"):
            call(queries, subset=torch.tensor([1.0, 2.0]))
        with pytest.raises(ValueError, match=r"\[299\].*300 documents"):
            call(queries, subset=torch.ones(N_DOCS - 1, dtype=torch.bool))
        with pytest.raises(ValueError, match=r"\[3, 301\].*300 documents"):
            call(queries, subset=torch.ones(3, N_DOCS + 1, dtype=torch.bool))
        with pytest.raises(ValueError, match="Subset length must match number of queries"):
            call(queries, subset=torch.ones(2, N_DOCS, dtype=torch.bool))
        with pytest.raises(ValueError, match="Subset length must match number of queries"):
            call(queries, subset=torch.zeros(4, 5, dtype=torch.int64))
        with pytest.raises(ValueError, match=r"\[1, 2, 3\]"):
            call(queries, subset=torch.zeros(1, 2, 3, dtype=torch.int64))


@pytest.mark.gpu
def test_two_devices_equal_one(cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from fast_plaid_b200 import search

    oidx, docs = _oracle()
    t = to_index_tensors(oidx)
    one = _fastplaid(DeviceIndex(t, cuda_device))
    two = search.FastPlaid.from_device_index(DeviceIndex(t, "cuda:0"))
    two.devices = ["cuda:0", "cuda:1"]
    two.indices = {"cuda:0": DeviceIndex(t, "cuda:0"), "cuda:1": DeviceIndex(t, "cuda:1")}
    queries = make_queries(7, Q, seed=25, docs=docs)
    per = [list(range(b, N_DOCS, 7)) for b in range(7)]
    for form in (_padded(per), _mask_of(per, N_DOCS), torch.arange(50, 90)):
        assert two.search(queries, top_k=10, subset=form) == one.search(queries, top_k=10, subset=form)
        assert two.search_exhaustive(queries, top_k=10, subset=form) == one.search_exhaustive(queries, top_k=10,
                                                                                               subset=form)


# ---- document-sharded search ---------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3, 5])
def test_sharded_steps_with_filters_equal_the_unsharded_search(world, cuda_device):
    """The step functions on `world` shards of 300 documents (unaligned bases: 150; 100, 200; 60, 120, ..): each
    shard expands its own range of the global bitmaps, and the result is the unsharded search's."""
    oidx, docs = _oracle(seed=31)
    t = to_index_tensors(oidx)
    didx = DeviceIndex(t, cuda_device)
    q16 = make_queries(B, Q, seed=32, docs=docs).half().to(cuda_device)
    params = DeviceIndex.with_flags(DeviceIndex.make_params(10, 64, 16), engine.FPB_FLAG_SUBSET)
    shards = []
    for r in range(world):
        sh, base = shard_tensors(t, r, world)
        shards.append(DeviceIndex(sh, cuda_device, doc_id_base=base))
    rng = random.Random(world)
    per = [rng.sample(range(N_DOCS), 90) for _ in range(B)]
    for sets in (per, [list(range(37, 251))] * B):
        ref = didx.search(q16, params, subset=sets)
        for filt in (Filter.from_ids(_padded(sets).to(cuda_device), N_DOCS, cuda_device, B),
                     Filter.from_mask(_mask_of(sets[:1], N_DOCS)[0], cuda_device, B) if sets[0] == sets[-1] else None):
            if filt is None:
                continue
            cbs = torch.stack([sh.shard_subset_begin(q16, params, filter=filt) for sh in shards])
            keys = torch.stack([sh.shard_subset_keys(cbs, Q, params) for sh in shards])
            recs = torch.stack([sh.shard_exact_records(keys, r, Q, params) for r, sh in enumerate(shards)])
            got = shards[0].merge_records(recs, 10)
            for r, g_ in zip(ref, got):
                assert torch.equal(r, g_), world


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_attached_shards_build_their_filters_from_global_ids(world, cuda_device, monkeypatch):
    """FastPlaid on attached shards (from_device_index(shard=(rank, world)), whose metadata holds the shard's own
    document count, bases 150 or 100 and 200): every `subset=` form, the broadcast list and the single id included,
    becomes filters that keep the shard's own global ids, and the step functions then return the unsharded bytes.
    A mask covers the whole index: one of the shard's own length is refused."""
    from fast_plaid_b200.search import fast_plaid as fpmod

    oidx, docs = _oracle(seed=36)
    t = to_index_tensors(oidx)
    didx = DeviceIndex(t, cuda_device)
    q16 = make_queries(B, Q, seed=37, docs=docs).half().to(cuda_device)
    params = DeviceIndex.with_flags(DeviceIndex.make_params(10, 64, 16), engine.FPB_FLAG_SUBSET)
    fps = []
    for r in range(world):
        sh, base = shard_tensors(t, r, world)
        assert r == 0 or base > 0
        fps.append(fpmod.FastPlaid.from_device_index(DeviceIndex(sh, cuda_device, doc_id_base=base),
                                                     shard=(r, world)))
    # the all-reduce of the ranks' range ends, which one process cannot run for several ranks
    monkeypatch.setattr(fpmod, "_sharded_num_documents", lambda end, device: N_DOCS)
    rng = random.Random(world + 10)
    per = [rng.sample(range(N_DOCS), 90) for _ in range(B)]
    shared = list(range(37, 251))
    one = N_DOCS - 7  # held by the last shard
    cases = [(shared, [shared] * B), (one, [[one]] * B), (torch.tensor(shared), [shared] * B),
             (_mask_of([shared], N_DOCS)[0], [shared] * B), (_padded(per), per), (_mask_of(per, N_DOCS), per)]
    for form, sets in cases:
        ref = didx.search(q16, params, subset=[list(x) for x in sets])
        filts = []
        for fp in fps:
            idx = fp.indices[fp.devices[0]]
            spec = fp._subset_tensor(form, B, lambda: fp._num_documents(idx))
            filts.append(spec.to_filter(idx, B))
        shards = [fp.indices[fp.devices[0]] for fp in fps]
        cbs = torch.stack([sh.shard_subset_begin(q16, params, filter=f) for sh, f in zip(shards, filts)])
        keys = torch.stack([sh.shard_subset_keys(cbs, Q, params) for sh in shards])
        recs = torch.stack([sh.shard_exact_records(keys, r, Q, params) for r, sh in enumerate(shards)])
        got = shards[0].merge_records(recs, 10)
        for r_, g_ in zip(ref, got):
            assert torch.equal(r_, g_), (world, type(form))
    last = fps[-1].indices[fps[-1].devices[0]]
    with pytest.raises(ValueError, match=f"{N_DOCS} documents"):
        fps[-1]._subset_tensor(torch.ones(last.num_documents, dtype=torch.bool), B,
                               lambda: fps[-1]._num_documents(last))


@pytest.mark.gpu
def test_device_list_split_on_one_gpu(cuda_device):
    """Several devices in one process split the batch: here two entries of the same device (one replica, its calls
    serialised), so the split of every form runs on one GPU.  7 queries over 2 entries: chunks of 4 and 3."""
    oidx, docs = _oracle(seed=38)
    didx = DeviceIndex(to_index_tensors(oidx), cuda_device)
    one = _fastplaid(didx)
    two = _fastplaid(didx)
    two.devices = [cuda_device, cuda_device]
    queries = make_queries(7, Q, seed=39, docs=docs)
    per = [list(range(b, N_DOCS, 7)) for b in range(7)]
    for form in (_padded(per), _mask_of(per, N_DOCS), _mask_of(per, N_DOCS).to(cuda_device), torch.arange(50, 90),
                 list(range(50, 90)), 61, per):
        assert two.search(queries, top_k=10, subset=form) == one.search(queries, top_k=10, subset=form)
        assert two.search_exhaustive(queries, top_k=10, subset=form) == one.search_exhaustive(queries, top_k=10,
                                                                                               subset=form)


@pytest.mark.gpu
def test_each_call_passes_only_its_own_filters(cuda_device, monkeypatch):
    """A batch split into calls of 2 queries: each call passes the rows of the filters its queries use (a view of a
    contiguous run, a gathered copy otherwise), so a call never sees more filters than queries."""
    oidx, docs = _oracle(seed=40)
    didx = DeviceIndex(to_index_tensors(oidx), cuda_device)
    q16 = make_queries(B, Q, seed=41, docs=docs).half().to(cuda_device)
    rng = random.Random(42)
    sets = [rng.sample(range(N_DOCS), 60) for _ in range(4)]
    base = Filter.from_ids(_padded(sets).to(cuda_device), N_DOCS, cuda_device, 4)
    filt = Filter(base.bitmap, [3, 0, 2, 2, 1, 3], N_DOCS)
    per = [sets[f] for f in filt.query_filter]
    params = DeviceIndex.make_params(10, 64, 16)
    ref = didx.search(q16, params, subset=per)
    seen = []
    lib = didx._lib
    real = lib.fpb_search_batch_filter

    def spy(*a):
        seen.append(a[6])  # n_filters of the call
        return real(*a)

    monkeypatch.setattr(didx, "max_queries_per_call", lambda *a, **k: 2)
    monkeypatch.setattr(lib, "fpb_search_batch_filter", spy)
    got = didx.search(q16, params, filter=filt)
    monkeypatch.setattr(lib, "fpb_search_batch_filter", real)
    assert seen == [2, 1, 2]
    for r_, g_ in zip(ref, got):
        assert torch.equal(r_, g_)
    rows, local = filt.call_rows(0, 2)
    assert rows.shape[0] == 2 and local == [1, 0]
    rows, local = filt.call_rows(4, 6)
    assert torch.equal(rows, base.bitmap[[1, 3]]) and local == [0, 1]


@pytest.mark.gpu
def test_understated_max_count_cuts_the_lists(cuda_device):
    """fpb_search_exhaustive_filter with max_count below a filter's documents: the list keeps its first max_count
    documents in id order (the compaction never writes past the workspace), so the result is that of the shorter
    list; with the exact count it is the whole filter's."""
    oidx, docs = _oracle(seed=43)
    didx = DeviceIndex(to_index_tensors(oidx), cuda_device)
    q16 = make_queries(3, Q, seed=44, docs=docs).half().to(cuda_device)
    rng = random.Random(45)
    members = sorted(rng.sample(range(N_DOCS), 50))
    filt = Filter.from_ids(torch.tensor(members), N_DOCS, cuda_device, 3)
    assert int(didx.filter_counts(filt).max()) == 50
    lib = didx._lib
    for max_count in (10, 1, 50):
        k = 20
        ids = torch.empty((3, k), dtype=torch.int64, device=cuda_device)
        sc = torch.empty((3, k), dtype=torch.float32, device=cuda_device)
        cnt = torch.empty((3,), dtype=torch.int32, device=cuda_device)
        nbytes = didx.exhaustive_filter_workspace_bytes(3, Q, k, 1, max_count)
        ws = torch.zeros(nbytes + 4096, dtype=torch.uint8, device=cuda_device)
        ws[nbytes:] = 0xA5  # past the workspace: must stay untouched
        h_map = (ctypes.c_int32 * 3)(0, 0, 0)
        rc = lib.fpb_search_exhaustive_filter(didx._handle, q16.data_ptr(), 3, Q, k, filt.bitmap.data_ptr(), 1,
                                              N_DOCS, max_count, h_map, ws.data_ptr(), nbytes, ids.data_ptr(),
                                              sc.data_ptr(), cnt.data_ptr(), None)
        assert rc == 0
        torch.cuda.synchronize()
        assert bool((ws[nbytes:] == 0xA5).all())
        ref = didx.search_exhaustive(q16, k, subset=[members[:max_count]] * 3)
        for r_, g_ in zip(ref, (ids, sc, cnt)):
            assert torch.equal(r_, g_), max_count


@pytest.mark.gpu
def test_malformed_filter_bitmaps_are_refused(cuda_device):
    oidx, docs = _oracle()
    didx = DeviceIndex(to_index_tensors(oidx), cuda_device)
    q16 = make_queries(2, Q, seed=46, docs=docs).half().to(cuda_device)
    params = DeviceIndex.make_params(10, 64, 8)
    good = Filter.from_ids(torch.arange(10), N_DOCS, cuda_device, 2)
    wide = torch.zeros((2, 20), dtype=torch.int32, device=cuda_device)
    for bad in (Filter(good.bitmap[:, :5].contiguous(), [0, 0], N_DOCS),  # narrower than ceil(n_bits / 32)
                Filter(wide[:, ::2], [0, 1], N_DOCS),                    # strided
                Filter(good.bitmap.to(torch.int64), [0, 0], N_DOCS),     # wrong dtype
                Filter(good.bitmap.cpu(), [0, 0], N_DOCS)):              # wrong device
        with pytest.raises(ValueError, match="contiguous filter bitmaps"):
            didx.search(q16, params, filter=bad)
        with pytest.raises(ValueError, match="contiguous filter bitmaps"):
            didx.search_exhaustive(q16, 10, filter=bad)


@pytest.mark.gpu
def test_fastplaid_shard_of_one(cuda_device):
    from fast_plaid_b200 import search

    oidx, docs = _oracle(seed=33)
    t = to_index_tensors(oidx)
    plain = _fastplaid(DeviceIndex(t, cuda_device))
    sharded = search.FastPlaid.from_device_index(DeviceIndex(t, cuda_device), shard=(0, 1))
    queries = make_queries(B, Q, seed=34, docs=docs)
    per = [list(range(b, N_DOCS, 5)) for b in range(B)]
    for form in (_padded(per), _mask_of(per, N_DOCS).to(cuda_device), list(range(10, 200)), 17):
        assert sharded.search(queries, top_k=10, subset=form) == plain.search(queries, top_k=10, subset=form)
    with pytest.raises(NotImplementedError, match="document-sharded"):
        sharded.search_exhaustive(queries, top_k=10, subset=torch.arange(5))


@pytest.mark.gpu
def test_c_abi_refusals_on_the_gpu(cuda_device):
    """The refusals of the filtered entry points with a real index: a map entry out of range, a missing
    FPB_FLAG_SUBSET, n_filters < 1 and n_bits < 0, each before any work."""
    oidx, docs = _oracle()
    didx = DeviceIndex(to_index_tensors(oidx), cuda_device)
    q16 = make_queries(2, Q, seed=35, docs=docs).half().to(cuda_device)
    filt = Filter.from_ids(torch.arange(10), N_DOCS, cuda_device, 2)
    with pytest.raises(ValueError, match=r"\[1\]=1 is not in \[0, n_filters=1\)"):
        didx.search(q16, DeviceIndex.make_params(10, 64, 8), filter=Filter(filt.bitmap, [0, 1], N_DOCS))
    with pytest.raises(ValueError, match=r"\[1\]=-1 is not in \[0, n_filters=1\)"):
        didx.search_exhaustive(q16, 10, filter=Filter(filt.bitmap, [0, -1], N_DOCS))
    lib = engine.load_library()
    params = DeviceIndex.make_params(10, 64, 8)
    buf, _ = didx.workspace(2, Q, params)
    out = torch.empty(64, dtype=torch.int64, device=cuda_device)
    h_map = (ctypes.c_int32 * 2)(0, 0)
    rc = lib.fpb_search_batch_filter(didx._handle, q16.data_ptr(), 2, Q, ctypes.byref(params), filt.bitmap.data_ptr(),
                                     1, N_DOCS, h_map, buf.data_ptr(), buf.numel(), out.data_ptr(), out.data_ptr(),
                                     out.data_ptr(), None)
    assert rc == engine.FPB_ERR_INVALID and b"FPB_FLAG_SUBSET" in lib.fpb_last_error()
