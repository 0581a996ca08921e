"""Appending documents to a loaded index in place (DeviceIndex.append, fpb_index_append, fpb_ivf_append) and the
update path built on it: the grown index equals a fresh load of the same directory, tensor for tensor, its results
equal a fresh load's, its files equal what a reload-path update writes, and the codes, residuals and norms never
move."""

from __future__ import annotations

import ctypes
import filecmp
import os
import shutil

import pytest
import torch

from util import make_docs, make_queries

pytestmark = pytest.mark.gpu

CODECS = [(128, 4), (128, 2), (64, 4), (64, 2), (128, 1)]


def _unit(n: int, dim: int, seed: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.nn.functional.normalize(torch.randn(n, dim, generator=g), dim=-1)


def _batches(dim: int) -> list[list[torch.Tensor]]:
    """One update, then three: a 1-token document and one of 1100 tokens, short documents, a batch of one document,
    and 160 documents of 10 windows each, which move walk_group from 4 (every document of the first index has at
    most 4 windows) to 5."""
    first = make_docs(40, 20, 80, dim=dim, seed=301) + [_unit(1, dim, 302), _unit(1100, dim, 303)]
    return [first, make_docs(25, 1, 120, dim=dim, seed=304), [_unit(3, dim, 305)],
            make_docs(160, 289, 320, dim=dim, seed=306)]


def _fresh(path: str, device: str):
    from fast_plaid_b200.engine import DeviceIndex
    from fast_plaid_b200.index import store

    data, base = store.read_index_to_device(path, device)
    return DeviceIndex(data, device, doc_id_base=base)


def _walk(idx):
    n = ctypes.c_int64()
    lib = idx._lib
    assert lib.fpb_index_walk_layout(idx._handle, ctypes.byref(n), None, None) == 0
    codes = torch.empty(max(32 * n.value, 1), dtype=torch.int32, device=idx.device)
    win = torch.empty(idx.num_documents + 1, dtype=torch.int64, device=idx.device)
    assert lib.fpb_index_walk_layout(idx._handle, ctypes.byref(n), codes.data_ptr(), win.data_ptr()) == 0
    return codes[: 32 * n.value], win


def assert_same_index(a, b) -> None:
    """Every device tensor and derived table of two DeviceIndexes is equal."""
    assert (a.num_documents, a.num_tokens, a.max_doc_len) == (b.num_documents, b.num_tokens, b.max_doc_len)
    for name in ("doc_offsets", "doc_codes", "doc_residuals", "token_norms", "centroids", "bucket_weights"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name
    assert a.has_ivf == b.has_ivf
    if b.has_ivf:
        assert torch.equal(a.ivf_offsets, b.ivf_offsets)
        assert torch.equal(a.ivf_pids, b.ivf_pids)
    wa, wb = _walk(a), _walk(b)
    assert torch.equal(wa[0], wb[0]) and torch.equal(wa[1], wb[1])
    assert a.walk_group == b.walk_group


class _CountLoads:
    def __init__(self, monkeypatch):
        from fast_plaid_b200 import search

        self.calls = 0
        orig = search.FastPlaid._load_all

        def counted(fp):
            self.calls += 1
            return orig(fp)

        monkeypatch.setattr(search.FastPlaid, "_load_all", counted)


def _results(fp, queries, subset):
    out = {}
    for n_probe in (8, 64):
        out[f"search{n_probe}"] = fp.search(queries, top_k=10, n_ivf_probe=n_probe, show_progress=False)
        out[f"subset{n_probe}"] = fp.search(queries, top_k=10, n_ivf_probe=n_probe, subset=subset,
                                            show_progress=False)
    out["exhaustive"] = fp.search_exhaustive(queries, top_k=10)
    ts = fp.search_token_scores(queries[:3], top_k=3, show_progress=False)
    out["token_scores"] = [[(d, s) for d, s, _ in r] for r in ts]
    out["token_mats"] = [m for r in ts for _, _, m in r]
    out["embeddings"] = fp.get_embeddings([0, 5, fp.indices[fp.devices[0]].num_documents - 1])
    return out


def _assert_same_results(a: dict, b: dict) -> None:
    for k in a:
        if k in ("token_mats", "embeddings"):
            assert len(a[k]) == len(b[k]) and all(torch.equal(x, y) for x, y in zip(a[k], b[k])), k
        else:
            assert a[k] == b[k], k


@pytest.mark.parametrize("dim,nbits", CODECS)
def test_update_appends_in_place(tmp_path, cuda_device, monkeypatch, dim, nbits):
    """1 and then 3 more updates: every device tensor equals a fresh load of the directory, the results equal a
    fresh FastPlaid's, the files equal what the reload path writes on a copy, no reload runs, and the codes,
    residuals and norms stay where they are."""
    from fast_plaid_b200 import search

    path, copy = str(tmp_path / "idx"), str(tmp_path / "copy")
    fp = search.FastPlaid(path, device=cuda_device)
    docs = make_docs(200, 20, 100, dim=dim, seed=300)
    fp.create(docs, nbits=nbits, kmeans_niters=2)
    queries = make_queries(6, 24, dim=dim, seed=307, docs=docs)
    idx0 = fp.indices[cuda_device]
    ptrs = [t.data_ptr() for t in (idx0.doc_codes, idx0.doc_residuals, idx0.token_norms)]
    assert idx0.growable is not None and idx0.doc_codes.data_ptr() == idx0.growable.codes.ptr
    shutil.copytree(path, copy)
    ref = search.FastPlaid(copy, device=cuda_device)
    ref._appendable = lambda: None  # the reload path: rebuild the IVF from the chunk files, load the directory again
    loads = _CountLoads(monkeypatch)
    groups = [idx0.walk_group]
    for i, batch in enumerate(_batches(dim)):
        mapped0 = idx0.growable.mapped_bytes if i == 0 else mapped
        fp.update(batch, start_from_scratch=0)
        ref.update(batch, start_from_scratch=0)
        idx = fp.indices[cuda_device]
        assert loads.calls == i + 1, "only the reference path may load the directory"
        assert [t.data_ptr() for t in (idx.doc_codes, idx.doc_residuals, idx.token_norms)] == ptrs
        mapped = idx.growable.mapped_bytes
        n_tok = sum(int(d.shape[0]) for d in batch)
        grain = 4 * (2 << 20)  # each of the four buffers rounds up to its 2 MB granule
        assert mapped - mapped0 <= n_tok * (4 + dim * nbits // 8 + 2) + 8 * len(batch) + grain
        fresh = _fresh(path, cuda_device)
        assert_same_index(idx, fresh)
        groups.append(idx.walk_group)
        if i in (0, 3):
            names = sorted(os.listdir(path))
            assert names == sorted(os.listdir(copy))
            match, mismatch, errors = filecmp.cmpfiles(path, copy, names, shallow=False)
            assert not mismatch and not errors, mismatch
    assert groups[0] == 4 and groups[-1] == 5, groups
    subset = list(range(0, idx.num_documents, 3))
    got = _results(fp, queries, subset)
    fresh_fp = search.FastPlaid(path, device=cuda_device)
    _assert_same_results(got, _results(fresh_fp, queries, subset))
    fp.close(), fresh_fp.close(), ref.close()


def test_old_snapshot_keeps_its_results(tmp_path, cuda_device):
    """A DeviceIndex taken before an append returns its pre-append results afterwards, and cannot be appended to."""
    from fast_plaid_b200 import search
    from fast_plaid_b200.engine import DeviceIndex

    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device=cuda_device)
    docs = make_docs(150, 20, 80, seed=310)
    fp.create(docs, kmeans_niters=2)
    snap = fp.indices[cuda_device]
    q = make_queries(5, 32, seed=311, docs=docs).half().to(cuda_device)
    params = DeviceIndex.make_params(10, 64, 8)
    before = (snap.search(q, params), snap.search_exhaustive(q, 10))
    fp.update(make_docs(60, 20, 300, seed=312), start_from_scratch=0)
    fp.update(make_docs(10, 20, 300, seed=313), start_from_scratch=0)
    assert fp.indices[cuda_device] is not snap and fp.indices[cuda_device].num_documents == 220
    after = (snap.search(q, params), snap.search_exhaustive(q, 10))
    for x, y in zip(before, after):
        assert all(torch.equal(a, b) for a, b in zip(x, y))
    with pytest.raises(ValueError, match="newest"):
        snap.append(torch.zeros(1, dtype=torch.int32), torch.zeros((1, 64), dtype=torch.uint8), torch.tensor([1]))
    fp.close()


def test_fallbacks_reload(tmp_path, cuda_device, monkeypatch):
    """A sharded FastPlaid and one whose directory another FastPlaid changed load the directory again; a
    compress_only index appends in place.  All three end equal to a fresh load."""
    from fast_plaid_b200 import search

    loads = _CountLoads(monkeypatch)
    path = str(tmp_path / "idx")
    a = search.FastPlaid(path, device=cuda_device)
    docs = make_docs(120, 20, 80, seed=320)
    a.create(docs, kmeans_niters=2)
    b = search.FastPlaid(path, device=cuda_device)
    queries = make_queries(4, 16, seed=321, docs=docs)

    def check(fp):
        fresh = search.FastPlaid(path, device=cuda_device)
        assert_same_index(fp.indices[cuda_device], fresh.indices[cuda_device])
        assert fp.search(queries, top_k=10, show_progress=False) == fresh.search(queries, top_k=10,
                                                                                 show_progress=False)
        fresh.close()

    n = loads.calls
    b.update(make_docs(20, 20, 80, seed=322), start_from_scratch=0)
    assert loads.calls == n  # b appended in place
    a.update(make_docs(20, 20, 80, seed=323), start_from_scratch=0)
    assert loads.calls == n + 1  # a saw b's change on disk and loaded the directory
    check(a)
    sharded = search.FastPlaid(path, device=cuda_device, shard=(0, 1))
    n = loads.calls
    sharded.update(make_docs(10, 20, 80, seed=324), start_from_scratch=0)
    assert loads.calls == n + 1
    check(sharded)
    for fp in (a, b, sharded):
        fp.close()

    cpath = str(tmp_path / "compress")
    c = search.FastPlaid(cpath, device=cuda_device)
    c.create(docs, kmeans_niters=2, compress_only=True)
    n = loads.calls
    c.update(make_docs(30, 1, 1100, seed=325), start_from_scratch=0)
    assert loads.calls == n and not c.indices[cuda_device].has_ivf
    fresh = search.FastPlaid(cpath, device=cuda_device)
    assert_same_index(c.indices[cuda_device], fresh.indices[cuda_device])
    assert c.search_exhaustive(queries, top_k=10) == fresh.search_exhaustive(queries, top_k=10)
    c.close(), fresh.close()


def test_append_to_tensor_built_index_copies_once(cuda_device):
    """An index built from device tensors copies into growable buffers on its first append; centroids whose old
    lists were empty gain postings; the result equals a DeviceIndex built from all the tensors."""
    from fast_plaid_b200.engine import DeviceIndex, IndexTensors
    from fast_plaid_b200.index.layout import build_ivf

    K, dim, nbits = 300, 128, 4
    g = torch.Generator().manual_seed(330)
    lens_old = torch.randint(1, 90, (120,), generator=g)
    lens_new = torch.cat([torch.randint(0, 90, (40,), generator=g), torch.tensor([1, 1300, 0])])
    codes_old = torch.randint(0, K // 2, (int(lens_old.sum()),), generator=g, dtype=torch.int32)  # cells >= K/2 empty
    codes_new = torch.randint(0, K, (int(lens_new.sum()),), generator=g, dtype=torch.int32)
    res_old = torch.randint(0, 256, (codes_old.shape[0], dim * nbits // 8), generator=g, dtype=torch.uint8)
    res_new = torch.randint(0, 256, (codes_new.shape[0], dim * nbits // 8), generator=g, dtype=torch.uint8)
    cent = torch.nn.functional.normalize(torch.randn(K, dim, generator=g), dim=-1).half()
    weights = torch.linspace(-0.1, 0.1, 1 << nbits).half()

    def tensors(codes, res, lens, device):
        ivf, ivf_len = build_ivf(codes.long(), lens, K)
        return IndexTensors(nbits=nbits, centroids=cent, bucket_weights=weights, doc_lengths=lens,
                            doc_codes=codes.to(device), doc_residuals=res.to(device), ivf=ivf.int(),
                            ivf_lengths=ivf_len)

    old = DeviceIndex(tensors(codes_old, res_old, lens_old, cuda_device), cuda_device)
    assert old.growable is None  # device tensors are used where they are
    grown = old.append(codes_new, res_new, lens_new)
    assert old.growable is not None and grown.doc_codes.data_ptr() == old.growable.codes.ptr
    full = DeviceIndex(tensors(torch.cat([codes_old, codes_new]), torch.cat([res_old, res_new]),
                               torch.cat([lens_old, lens_new]), "cpu"), cuda_device)
    assert_same_index(grown, full)
    # zero new documents, then one
    g2 = grown.append(torch.zeros(0, dtype=torch.int32), torch.zeros((0, 64), dtype=torch.uint8),
                      torch.zeros(0, dtype=torch.int64))
    assert_same_index(g2, full)
    g3 = g2.append(torch.tensor([K - 1, K - 1, 7], dtype=torch.int32), res_new[:3], torch.tensor([3]))
    full3 = DeviceIndex(tensors(torch.cat([codes_old, codes_new, torch.tensor([K - 1, K - 1, 7], dtype=torch.int32)]),
                                torch.cat([res_old, res_new, res_new[:3]]), torch.cat([lens_old, lens_new,
                                                                                         torch.tensor([3])]), "cpu"),
                        cuda_device)
    assert_same_index(g3, full3)
    q = make_queries(4, 32, seed=331).half().to(cuda_device)
    p = DeviceIndex.make_params(10, 64, 8)
    for x, y in zip(g3.search(q, p), full3.search(q, p)):
        assert torch.equal(x, y)
    for x, y in zip(old.search_exhaustive(q, 10), DeviceIndex(tensors(codes_old, res_old, lens_old, "cpu"),
                                                              cuda_device).search_exhaustive(q, 10)):
        assert torch.equal(x, y)


def _ivf_append(old_codes, old_lens, new_codes, new_lens, n_cells, device):
    from fast_plaid_b200 import engine
    from fast_plaid_b200.index.layout import build_ivf

    lib = engine.load_library()
    ivf, ivf_len = build_ivf(old_codes.to(device).long(), old_lens, n_cells)
    offs = torch.zeros(n_cells + 1, dtype=torch.int64)
    offs[1:] = ivf_len.long()[:n_cells].cumsum(0)
    offs, pids = offs.to(device), ivf.int().to(device)
    if pids.numel() == 0:
        pids = torch.zeros(1, dtype=torch.int32, device=device)
    new_offs = torch.zeros(new_lens.shape[0] + 1, dtype=torch.int64)
    new_offs[1:] = new_lens.cumsum(0)
    new_offs = new_offs.to(device)
    codes = new_codes.int().to(device) if new_codes.numel() else torch.zeros(1, dtype=torch.int32, device=device)
    out_offs = torch.empty(n_cells + 1, dtype=torch.int64, device=device)
    n = ctypes.c_int64()
    args = (torch.device(device).index, n_cells, offs.data_ptr(), pids.data_ptr(), int(old_lens.shape[0]),
            int(new_lens.shape[0]), new_offs.data_ptr(), codes.data_ptr(), out_offs.data_ptr())
    assert lib.fpb_ivf_append(*args, None, 0, ctypes.byref(n), None) == 0, lib.fpb_last_error()
    out = torch.full((max(n.value, 1),), -7, dtype=torch.int32, device=device)
    assert lib.fpb_ivf_append(*args, out.data_ptr(), out.numel(), ctypes.byref(n), None) == 0, lib.fpb_last_error()
    return out_offs.cpu(), out[: n.value].cpu(), lib, args


@pytest.mark.parametrize("case", ["one_cell", "every_cell", "repeat300", "odd_k", "no_new", "one_new", "slabs"])
def test_ivf_merge_matches_build_ivf(cuda_device, case):
    """fpb_ivf_append equals build_ivf over all the documents on adversarial inputs."""
    from fast_plaid_b200.index.layout import build_ivf

    g = torch.Generator().manual_seed(340)
    K = {"odd_k": 1000, "every_cell": 777, "slabs": (1 << 21) + 3}.get(case, 256)
    n_old, n_new = (50, 0) if case == "no_new" else (50, 1) if case == "one_new" else (60, 700)
    old_lens = torch.randint(0, 40, (n_old,), generator=g)
    new_lens = torch.randint(0, 40, (n_new,), generator=g)
    if case == "repeat300":
        new_lens[3] = 300
    old_codes = torch.randint(0, K, (int(old_lens.sum()),), generator=g)
    new_codes = torch.randint(0, K, (int(new_lens.sum()),), generator=g)
    if case == "one_cell":
        old_codes[:] = 17
        new_codes[:] = 17
    elif case == "every_cell":
        new_codes[:K] = torch.arange(K)
    elif case == "repeat300":
        a = int(new_lens[:3].sum())
        new_codes[a : a + 300] = 5
    out_offs, out_pids, lib, args = _ivf_append(old_codes, old_lens, new_codes, new_lens, K, cuda_device)
    ivf, ivf_len = build_ivf(torch.cat([old_codes, new_codes]), torch.cat([old_lens, new_lens]), K)
    exp = torch.zeros(K + 1, dtype=torch.int64)
    exp[1:] = ivf_len.long().cumsum(0)
    assert torch.equal(out_offs, exp)
    assert torch.equal(out_pids.long(), ivf)
    if case == "every_cell":
        assert bool((out_offs[1:] - out_offs[:-1] > 0).all())
    if case == "one_new":  # too small an output is refused
        n = ctypes.c_int64()
        small = torch.zeros(1, dtype=torch.int32, device=cuda_device)
        rc = lib.fpb_ivf_append(*args, small.data_ptr(), 0, ctypes.byref(n), None)
        assert rc == -1 and b"do not fit" in lib.fpb_last_error()


def test_ivf_merge_refuses_codes_outside_the_cells(cuda_device):
    from fast_plaid_b200 import engine

    with pytest.raises(AssertionError):
        _ivf_append(torch.tensor([1, 2]), torch.tensor([2]), torch.tensor([3, 256]), torch.tensor([2]), 256,
                    cuda_device)
    assert b"outside" in engine.load_library().fpb_last_error()


def test_index_append_refusals(cuda_device):
    """fpb_index_append refuses shrinking sizes, NULL arrays, an IVF of the wrong kind and an offsets array that does
    not continue the old one."""
    from fast_plaid_b200 import engine
    from fast_plaid_b200.engine import DeviceIndex, IndexTensors

    lib = engine.load_library()
    K, dim = 64, 128
    g = torch.Generator().manual_seed(350)
    lens = torch.tensor([3, 5])
    data = IndexTensors(nbits=4, centroids=torch.randn(K, dim, generator=g).half(),
                        bucket_weights=torch.zeros(16).half(), doc_lengths=lens,
                        doc_codes=torch.randint(0, K, (8,), generator=g), doc_residuals=torch.zeros((8, 64),
                                                                                               dtype=torch.uint8),
                        ivf=None, ivf_lengths=None)
    idx = DeviceIndex(data, cuda_device)
    h = ctypes.c_void_p()
    v = idx.growable.views(3, 9)
    ptrs = [v[k].data_ptr() for k in ("offsets", "codes", "residuals", "norms")]
    assert lib.fpb_index_append(ctypes.byref(h), idx._handle, 1, 9, *ptrs, None, None, 0, 5) == -1  # shrinks N
    assert lib.fpb_index_append(ctypes.byref(h), idx._handle, 3, 7, *ptrs, None, None, 0, 5) == -1  # shrinks E
    assert lib.fpb_index_append(ctypes.byref(h), idx._handle, 3, 9, *ptrs, None, None, 0, 4) == -1  # max_doc_len
    assert lib.fpb_index_append(ctypes.byref(h), idx._handle, 3, 9, ptrs[0], None, ptrs[2], ptrs[3], None, None, 0,
                                5) == -1
    ivf = torch.zeros(K + 1, dtype=torch.int64, device=cuda_device)
    assert lib.fpb_index_append(ctypes.byref(h), idx._handle, 3, 9, *ptrs, ivf.data_ptr(), ivf.data_ptr(), 0, 5) == -1
    assert b"inverted file" in lib.fpb_last_error()
    v["offsets"][2] = 7  # entry N is not E
    assert lib.fpb_index_append(ctypes.byref(h), idx._handle, 3, 9, *ptrs, None, None, 0, 5) == -1
    assert b"offsets" in lib.fpb_last_error() and not h.value
    v["offsets"][2] = 8
    v["offsets"][3] = 9
    v["codes"][8] = 1  # the new token: a valid code, so that its norm can be computed
    v["residuals"][8] = 0
    assert lib.fpb_index_append(ctypes.byref(h), idx._handle, 3, 9, *ptrs, None, None, 0, 5) == 0
    assert lib.fpb_index_append(ctypes.byref(h), idx._handle, 3, 9, *ptrs, None, None, 0, 5) == -1  # twice
    assert b"already been appended" in lib.fpb_last_error()
    lib.fpb_index_destroy(h)
