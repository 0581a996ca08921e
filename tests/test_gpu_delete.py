"""Deleting documents from a loaded index in place (DeviceIndex.delete, fpb_docs_compact, fpb_ivf_delete) and the
FastPlaid.delete path built on it: the compacted index equals a fresh load of the directory, tensor for tensor, its
results equal a fresh load's, its files equal what the host delete writes, and the directory is not loaded again."""

from __future__ import annotations

import ctypes
import filecmp
import gc
import os
import shutil
import time
import weakref

import pytest
import torch

from test_gpu_append import CODECS, _CountLoads, _assert_same_results, _fresh, _results, _unit, assert_same_index
from util import make_docs, make_queries

pytestmark = pytest.mark.gpu

# ---- the kernels against torch ------------------------------------------------------------------------------------

K_CELLS = 200
N_DOCS = 300


def _data(pd: int):
    """300 documents of 0 to 60 tokens, document 7 of 1 token and document 100 of 1100, codes in [0, 200)."""
    g = torch.Generator().manual_seed(400 + pd)
    lens = torch.randint(0, 61, (N_DOCS,), generator=g)
    lens[7], lens[100] = 1, 1100
    E = int(lens.sum())
    codes = torch.randint(0, K_CELLS, (E,), generator=g, dtype=torch.int32)
    res = torch.randint(0, 256, (E, pd), generator=g, dtype=torch.uint8)
    norms = torch.randn(E, generator=g).half()
    return lens, codes, res, norms


def _drop_set(case: str, lens: torch.Tensor, codes: torch.Tensor) -> list[int]:
    N = int(lens.shape[0])
    if case == "empty_cell":  # every document with a token in cell 5: the cell ends empty
        doc_of = torch.repeat_interleave(torch.arange(N), lens)
        return sorted(set(doc_of[codes == 5].tolist()))
    g = torch.Generator().manual_seed(410)
    return {
        "none": [], "all": list(range(N)), "all_but_one": [d for d in range(N) if d != 150], "first": [0],
        "last": [N - 1], "alternate": list(range(0, N, 2)), "run": list(range(40, 260)),
        "random50": sorted(torch.randperm(N, generator=g)[: N // 2].tolist()),
        "boundaries": [31, 32, 63, 64, 95, 96, 127, 128, 159, 160, 255, 256, 288],
        "long_docs": [7, 100],
    }[case]


def _offsets(lens: torch.Tensor) -> torch.Tensor:
    offs = torch.zeros(lens.shape[0] + 1, dtype=torch.int64)
    offs[1:] = lens.cumsum(0)
    return offs


def _compact(lens, codes, res, norms, drop, device, with_norms=True, capacity=None):
    from fast_plaid_b200 import engine

    lib = engine.load_library()
    N, pd = int(lens.shape[0]), int(res.shape[1])
    offs = _offsets(lens).to(device)
    codes, res, norms = codes.to(device), res.to(device), norms.to(device)
    d_drop = torch.tensor(drop, dtype=torch.int32, device=device) if drop else None
    out_offs = torch.full((N - len(drop) + 1,), -7, dtype=torch.int64, device=device)
    n = ctypes.c_int64(-1)
    args = (torch.device(device).index, N, offs.data_ptr(), codes.data_ptr(), res.data_ptr(),
            norms.data_ptr() if with_norms else None, pd, None if d_drop is None else d_drop.data_ptr(), len(drop),
            out_offs.data_ptr())
    assert lib.fpb_docs_compact(*args, None, None, None, 0, ctypes.byref(n), None) == 0, lib.fpb_last_error()
    E1 = n.value
    out_codes = torch.full((max(E1, 1),), -7, dtype=torch.int32, device=device)
    out_res = torch.full((max(E1, 1), pd), 7, dtype=torch.uint8, device=device)
    out_norms = torch.full((max(E1, 1),), -7.0, dtype=torch.float16, device=device)
    rc = lib.fpb_docs_compact(*args, out_codes.data_ptr(), out_res.data_ptr(),
                              out_norms.data_ptr() if with_norms else None, E1 if capacity is None else capacity,
                              ctypes.byref(n), None)
    if capacity is not None:
        return rc, lib.fpb_last_error()
    assert rc == 0, lib.fpb_last_error()
    assert n.value == E1
    return out_offs.cpu(), out_codes[:E1].cpu(), out_res[:E1].cpu(), out_norms[:E1].cpu()


def _ivf_delete(ivf, ivf_len, n_docs, drop, device, capacity=None):
    from fast_plaid_b200 import engine

    lib = engine.load_library()
    offs = torch.zeros(K_CELLS + 1, dtype=torch.int64)
    offs[1:] = ivf_len.long()[:K_CELLS].cumsum(0)
    offs, pids = offs.to(device), ivf.int().to(device)
    d_drop = torch.tensor(drop, dtype=torch.int32, device=device) if drop else None
    out_offs = torch.full((K_CELLS + 1,), -7, dtype=torch.int64, device=device)
    n = ctypes.c_int64(-1)
    args = (torch.device(device).index, K_CELLS, offs.data_ptr(), pids.data_ptr(), n_docs,
            None if d_drop is None else d_drop.data_ptr(), len(drop), out_offs.data_ptr())
    assert lib.fpb_ivf_delete(*args, None, 0, ctypes.byref(n), None) == 0, lib.fpb_last_error()
    total = n.value
    out = torch.full((max(total, 1),), -7, dtype=torch.int32, device=device)
    rc = lib.fpb_ivf_delete(*args, out.data_ptr(), total if capacity is None else capacity, ctypes.byref(n), None)
    if capacity is not None:
        return rc, lib.fpb_last_error()
    assert rc == 0, lib.fpb_last_error()
    return out_offs.cpu(), out[:total].cpu(), total


CASES = ["none", "all", "all_but_one", "first", "last", "alternate", "run", "random50", "boundaries", "long_docs",
         "empty_cell"]


@pytest.mark.parametrize("pd", [16, 32, 64])
@pytest.mark.parametrize("case", CASES)
def test_docs_compact_matches_mask_indexing(cuda_device, case, pd):
    """fpb_docs_compact equals boolean-mask indexing of the offsets, codes, residuals and norms; the sizing call gives
    the exact token count, and a capacity one token short is refused."""
    lens, codes, res, norms = _data(pd)
    drop = _drop_set(case, lens, codes)
    keep = torch.ones(N_DOCS, dtype=torch.bool)
    keep[torch.tensor(drop, dtype=torch.int64)] = False
    keep_tok = torch.repeat_interleave(keep, lens)
    out_offs, out_codes, out_res, out_norms = _compact(lens, codes, res, norms, drop, cuda_device)
    assert torch.equal(out_offs, _offsets(lens[keep]))
    assert torch.equal(out_codes, codes[keep_tok])
    assert torch.equal(out_res, res[keep_tok])
    assert torch.equal(out_norms.view(torch.int16), norms[keep_tok].view(torch.int16))
    no_norms = _compact(lens, codes, res, norms, drop, cuda_device, with_norms=False)
    assert all(torch.equal(a, b) for a, b in zip(no_norms[:3], (out_offs, out_codes, out_res)))
    E1 = int(keep_tok.sum())
    if E1 > 0:
        rc, msg = _compact(lens, codes, res, norms, drop, cuda_device, capacity=E1 - 1)
        assert rc == -1 and b"do not fit" in msg


@pytest.mark.parametrize("case", CASES)
def test_ivf_delete_matches_build_ivf(cuda_device, case):
    """fpb_ivf_delete equals build_ivf over the kept documents' codes; the sizing call gives the exact posting count,
    and a capacity one posting short is refused."""
    from fast_plaid_b200.index.layout import build_ivf

    lens, codes, _, _ = _data(16)
    drop = _drop_set(case, lens, codes)
    keep = torch.ones(N_DOCS, dtype=torch.bool)
    keep[torch.tensor(drop, dtype=torch.int64)] = False
    keep_tok = torch.repeat_interleave(keep, lens)
    ivf, ivf_len = build_ivf(codes.long(), lens, K_CELLS)
    out_offs, out_pids, total = _ivf_delete(ivf, ivf_len, N_DOCS, drop, cuda_device)
    exp, exp_len = build_ivf(codes[keep_tok].long(), lens[keep], K_CELLS)
    exp_offs = torch.zeros(K_CELLS + 1, dtype=torch.int64)
    exp_offs[1:] = exp_len.long()[:K_CELLS].cumsum(0)
    assert total == exp.numel()
    assert torch.equal(out_offs, exp_offs)
    assert torch.equal(out_pids.long(), exp)
    if case == "empty_cell":
        assert int(ivf_len[5]) > 0 and int(out_offs[6] - out_offs[5]) == 0
    if total > 0:
        rc, msg = _ivf_delete(ivf, ivf_len, N_DOCS, drop, cuda_device, capacity=total - 1)
        assert rc == -1 and b"do not fit" in msg


def test_delete_kernels_refuse_bad_drop_lists(cuda_device):
    from fast_plaid_b200 import engine

    lens, codes, res, norms = _data(64)
    for drop in ([3, 3], [5, 2], [N_DOCS], [-1, 4]):
        with pytest.raises(AssertionError):
            _compact(lens, codes, res, norms, drop, cuda_device)
        assert b"sorted, unique" in engine.load_library().fpb_last_error()


# ---- DeviceIndex.delete and FastPlaid.delete ----------------------------------------------------------------------


def _docs(dim: int) -> list[torch.Tensor]:
    """200 documents in four chunks of 50 (create with batch_size=50), one of 1 token and one of 1100."""
    docs = make_docs(200, 20, 100, dim=dim, seed=420)
    docs[70], docs[130] = _unit(1, dim, 421), _unit(1100, dim, 422)
    return docs


def _mtimes(path: str, names) -> dict[str, int]:
    return {n: os.stat(os.path.join(path, n)).st_mtime_ns for n in names}


def _same_dirs(a: str, b: str) -> None:
    names = sorted(os.listdir(a))
    assert names == sorted(os.listdir(b))
    match, mismatch, errors = filecmp.cmpfiles(a, b, names, shallow=False)
    assert not mismatch and not errors, (mismatch, errors)


@pytest.mark.parametrize("dim,nbits", CODECS)
def test_delete_in_place(tmp_path, cuda_device, monkeypatch, dim, nbits):
    """A delete touching chunks 1 and 2 of 4: the index equals a fresh load, the results equal a fresh FastPlaid's,
    every file equals what the host delete writes on a copy, chunk 0 and chunk 3's arrays are not rewritten, and
    the directory is not loaded again."""
    from fast_plaid_b200 import search

    path, copy = str(tmp_path / "idx"), str(tmp_path / "copy")
    fp = search.FastPlaid(path, device=cuda_device)
    docs = _docs(dim)
    fp.create(docs, nbits=nbits, kmeans_niters=2, batch_size=50)
    shutil.copytree(path, copy)
    ref = search.FastPlaid(copy, device=cuda_device)
    ref._appendable = lambda: None  # the host delete, then a load of the directory
    untouched = [f"{i}.{k}.npy" for i in (0, 3) for k in ("codes", "residuals")] + ["0.metadata.json",
                                                                                       "doclens.3.json"]
    before = _mtimes(path, untouched)
    time.sleep(0.05)
    loads = _CountLoads(monkeypatch)
    drop = [60, 61, 99, 70, 130, 60, -3, 5000, 149]
    fp.delete(drop)
    assert loads.calls == 0, "the in-place delete must not load the directory"
    ref.delete(drop)
    assert loads.calls == 1
    assert _mtimes(path, untouched) == before
    _same_dirs(path, copy)
    idx = fp.indices[cuda_device]
    assert idx.num_documents == 194 and idx.growable is not None
    assert_same_index(idx, _fresh(path, cuda_device))
    assert_same_index(idx, ref.indices[cuda_device])
    queries = make_queries(6, 24, dim=dim, seed=423, docs=docs)
    subset = list(range(0, idx.num_documents, 3))
    fresh_fp = search.FastPlaid(path, device=cuda_device)
    _assert_same_results(_results(fp, queries, subset), _results(fresh_fp, queries, subset))
    fp.close(), fresh_fp.close(), ref.close()


def test_old_snapshot_keeps_its_results_and_is_released(tmp_path, cuda_device):
    """A DeviceIndex taken before a delete returns its pre-delete results afterwards; its buffers are freed once the
    last reference to it goes."""
    from fast_plaid_b200 import search
    from fast_plaid_b200.engine import DeviceIndex

    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device=cuda_device)
    docs = make_docs(150, 20, 80, seed=430)
    fp.create(docs, kmeans_niters=2)
    snap = fp.indices[cuda_device]
    q = make_queries(5, 32, seed=431, docs=docs).half().to(cuda_device)
    params = DeviceIndex.make_params(10, 64, 8)
    before = (snap.search(q, params), snap.search_exhaustive(q, 10))
    fp.delete(list(range(0, 150, 7)))
    assert fp.indices[cuda_device] is not snap and fp.indices[cuda_device].num_documents == 150 - 22
    after = (snap.search(q, params), snap.search_exhaustive(q, 10))
    for x, y in zip(before, after):
        assert all(torch.equal(a, b) for a, b in zip(x, y))
    arrays, codes_buf = weakref.ref(snap.growable), weakref.ref(snap.growable.codes)
    del snap, before, after
    gc.collect()
    assert arrays() is None and codes_buf() is None
    fp.close()


def test_chain_of_updates_and_deletes(tmp_path, cuda_device, monkeypatch):
    """create -> update (append in place) -> delete -> update -> delete, each step equal to a fresh load, with no
    load of the directory; then a compress_only index."""
    from fast_plaid_b200 import search

    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device=cuda_device)
    docs = make_docs(120, 20, 80, seed=440)
    fp.create(docs, kmeans_niters=2)
    loads = _CountLoads(monkeypatch)
    steps = [lambda: fp.update(make_docs(40, 1, 300, seed=441), start_from_scratch=0),
             lambda: fp.delete([0, 5, 119, 120, 159]),
             lambda: fp.update(make_docs(30, 20, 80, seed=442), start_from_scratch=0),
             lambda: fp.delete(list(range(50, 90)) + [184])]
    sizes = []
    for step in steps:
        step()
        idx = fp.indices[cuda_device]
        sizes.append(idx.num_documents)
        assert_same_index(idx, _fresh(path, cuda_device))
    assert loads.calls == 0 and sizes == [160, 155, 185, 144], sizes
    queries = make_queries(4, 16, seed=443, docs=docs)
    fresh = search.FastPlaid(path, device=cuda_device)
    assert fp.search(queries, top_k=10, show_progress=False) == fresh.search(queries, top_k=10, show_progress=False)
    fp.close(), fresh.close()

    cpath = str(tmp_path / "compress")
    c = search.FastPlaid(cpath, device=cuda_device)
    c.create(docs, kmeans_niters=2, compress_only=True)
    n = loads.calls
    c.delete([3, 4, 100])
    assert loads.calls == n and not c.indices[cuda_device].has_ivf
    fresh = search.FastPlaid(cpath, device=cuda_device)
    assert_same_index(c.indices[cuda_device], fresh.indices[cuda_device])
    assert c.search_exhaustive(queries, top_k=10) == fresh.search_exhaustive(queries, top_k=10)
    c.close(), fresh.close()


def test_delete_from_tensor_built_index(cuda_device):
    """An index built from device tensors (no growable buffers) deletes into new growable buffers; the result equals
    a DeviceIndex built from the kept tensors, and a document shard is refused."""
    from fast_plaid_b200.engine import DeviceIndex, IndexTensors
    from fast_plaid_b200.index.layout import build_ivf

    K, dim, nbits = 300, 128, 4
    g = torch.Generator().manual_seed(450)
    lens = torch.cat([torch.randint(0, 90, (130,), generator=g), torch.tensor([1, 1300, 0])])
    codes = torch.randint(0, K, (int(lens.sum()),), generator=g, dtype=torch.int32)
    res = torch.randint(0, 256, (codes.shape[0], dim * nbits // 8), generator=g, dtype=torch.uint8)
    cent = torch.nn.functional.normalize(torch.randn(K, dim, generator=g), dim=-1).half()
    weights = torch.linspace(-0.1, 0.1, 1 << nbits).half()

    def tensors(codes, res, lens, device):
        ivf, ivf_len = build_ivf(codes.long(), lens, K)
        return IndexTensors(nbits=nbits, centroids=cent, bucket_weights=weights, doc_lengths=lens,
                            doc_codes=codes.to(device), doc_residuals=res.to(device), ivf=ivf.int(),
                            ivf_lengths=ivf_len)

    old = DeviceIndex(tensors(codes, res, lens, cuda_device), cuda_device)
    assert old.growable is None
    drop = [0, 31, 32, 131, 64, 64, 900, -1]
    shrunk = old.delete(drop)
    assert old.growable is None and shrunk.growable is not None
    keep = torch.ones(lens.shape[0], dtype=torch.bool)
    keep[[0, 31, 32, 64, 131]] = False
    keep_tok = torch.repeat_interleave(keep, lens)
    full = DeviceIndex(tensors(codes[keep_tok], res[keep_tok], lens[keep], "cpu"), cuda_device)
    assert_same_index(shrunk, full)
    grown = shrunk.append(codes[:5], res[:5], torch.tensor([5]))  # the result can be appended to
    assert grown.num_documents == full.num_documents + 1
    q = make_queries(4, 32, seed=451).half().to(cuda_device)
    p = DeviceIndex.make_params(10, 64, 8)
    for x, y in zip(shrunk.search(q, p), full.search(q, p)):
        assert torch.equal(x, y)
    shard = DeviceIndex(tensors(codes, res, lens, "cpu"), cuda_device, doc_id_base=10)
    with pytest.raises(ValueError, match="shard"):
        shard.delete([1])


@pytest.mark.parametrize("case", ["sharded", "mtime", "raises", "everything"])
def test_fallbacks_reload(tmp_path, cuda_device, monkeypatch, case):
    """A sharded FastPlaid, a metadata.json changed since the load, a failing DeviceIndex.delete and a delete of every
    document take the host path and load the directory again; the files equal the host delete's on a copy."""
    from fast_plaid_b200 import search
    from fast_plaid_b200.engine import DeviceIndex

    path, copy = str(tmp_path / "idx"), str(tmp_path / "copy")
    docs = make_docs(120, 20, 80, seed=460)
    search.FastPlaid(path, device=cuda_device).create(docs, kmeans_niters=2, batch_size=50)
    shutil.copytree(path, copy)
    fp = search.FastPlaid(path, device=cuda_device, shard=(0, 1) if case == "sharded" else None)
    ref = search.FastPlaid(copy, device=cuda_device)
    ref._appendable = lambda: None
    if case == "mtime":
        t = os.stat(os.path.join(path, "metadata.json")).st_mtime + 5
        os.utime(os.path.join(path, "metadata.json"), (t, t))
    if case == "raises":
        def fail(self, doc_ids):
            raise RuntimeError("no memory")

        monkeypatch.setattr(DeviceIndex, "delete", fail)
    drop = list(range(120)) if case == "everything" else [2, 60, 61, 119]
    loads = _CountLoads(monkeypatch)
    fp.delete(drop)
    assert loads.calls == 1
    ref.delete(drop)
    _same_dirs(path, copy)
    if case != "everything":
        fresh = search.FastPlaid(path, device=cuda_device)
        assert_same_index(fp.indices[cuda_device], fresh.indices[cuda_device])
        queries = make_queries(4, 16, seed=461, docs=docs)
        assert fp.search(queries, top_k=10, show_progress=False) == fresh.search(queries, top_k=10,
                                                                                 show_progress=False)
        fresh.close()
    fp.close(), ref.close()
