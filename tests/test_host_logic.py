"""Host-side behaviour of the FastPlaid surface that needs no GPU: index bookkeeping through
create / update / delete, argument handling, and the loud failure of search on a CPU device
(structural checks borrowed from the reference's tests/test.py)."""

from __future__ import annotations

import json
import os

import pytest
import torch

from util import make_docs

from fast_plaid_b200 import search
from fast_plaid_b200.engine import EngineUnavailableError
from fast_plaid_b200.index import store


def _meta(path):
    return json.load(open(os.path.join(path, "metadata.json")))


def test_create_update_delete_bookkeeping(tmp_path):
    """tests/test.py:977-1303 of the reference: metadata.json num_documents follows the index."""
    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device="cpu")
    docs = make_docs(60, 5, 30, seed=1)
    fp.create(docs, kmeans_niters=2)
    assert _meta(path)["num_documents"] == 60
    assert os.path.exists(os.path.join(path, "embeddings.npy"))  # <= start_from_scratch docs keep raw copies
    fp.update(make_docs(15, 5, 30, seed=2))
    assert _meta(path)["num_documents"] == 75
    data = store.read_index(path)
    assert data.num_documents == 75 and int(data.doc_lengths.sum()) == data.doc_codes.shape[0]
    fp.delete([0, 3, 74])
    data = store.read_index(path)
    assert _meta(path)["num_documents"] == 72 and data.num_documents == 72
    assert int(data.ivf.max()) < 72
    assert int(data.doc_lengths.sum()) == data.doc_codes.shape[0] == _meta(path)["num_embeddings"]


def test_update_appends_with_existing_codec_when_large(tmp_path):
    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device="cpu")
    docs = make_docs(40, 5, 30, seed=1)
    fp.create(docs, kmeans_niters=2, start_from_scratch=10)  # no embeddings.npy kept
    assert not os.path.exists(os.path.join(path, "embeddings.npy"))
    cent_before = store.read_index(path).centroids.clone()
    fp.update(make_docs(12, 5, 30, seed=3), start_from_scratch=10)
    data = store.read_index(path)
    assert data.num_documents == 52
    assert torch.equal(data.centroids, cent_before)  # appended with the existing centroids
    # every appended document is reachable through the IVF
    offs = torch.cat([torch.zeros(1, dtype=torch.int64), data.doc_lengths.cumsum(0)])
    for d in (40, 51):
        codes = set(data.doc_codes[offs[d]:offs[d + 1]].tolist())
        ivf_offs = torch.cat([torch.zeros(1, dtype=torch.int64), data.ivf_lengths.long().cumsum(0)])
        for c in codes:
            assert d in data.ivf[ivf_offs[c]:ivf_offs[c + 1]].tolist()


def test_update_on_missing_index_creates_it(tmp_path):
    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device="cpu")
    fp.update(make_docs(20, 5, 30, seed=4), kmeans_niters=2)
    assert _meta(path)["num_documents"] == 20


def test_compress_only_has_no_ivf_files(tmp_path):
    """tests/test.py:734-746 of the reference."""
    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device="cpu")
    fp.create(make_docs(30, 5, 30, seed=5), kmeans_niters=2, compress_only=True)
    assert not os.path.exists(os.path.join(path, "ivf.npy"))
    assert not os.path.exists(os.path.join(path, "ivf_lengths.npy"))
    assert _meta(path)["compress_only"] is True
    assert store.read_index(path).ivf is None


def test_search_on_cpu_device_fails_loudly(tmp_path):
    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device="cpu")
    fp.create(make_docs(30, 5, 30, seed=6), kmeans_niters=2)
    with pytest.raises(EngineUnavailableError, match="no CPU search path"):
        fp.search(torch.randn(2, 8, 128), top_k=5)


def test_search_without_index_raises_file_not_found(tmp_path):
    fp = search.FastPlaid(str(tmp_path / "empty"), device="cpu")
    with pytest.raises(FileNotFoundError):
        fp.search(torch.randn(1, 4, 128))


def test_bad_device_string(tmp_path):
    with pytest.raises(ValueError, match="Unsupported device"):
        search.FastPlaid(str(tmp_path / "x"), device="tpu:0")


def test_metadata_length_must_match(tmp_path):
    fp = search.FastPlaid(str(tmp_path / "idx"), device="cpu")
    with pytest.raises(ValueError, match="metadata"):
        fp.create(make_docs(5, 5, 10, seed=7), metadata=[{"a": 1}])


def test_metadata_table_and_where(tmp_path):
    from fast_plaid_b200 import filtering

    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device="cpu")
    fp.create(make_docs(12, 5, 10, seed=8), kmeans_niters=1, metadata=[{"lang": "en" if i % 2 else "fr", "n": i} for i in range(12)])
    assert filtering.where(path, "lang = ?", ("en",)) == [1, 3, 5, 7, 9, 11]
    fp.delete([1])
    assert filtering.where(path, "lang = ?", ("en",)) == [2, 4, 6, 8, 10]


def test_k_heuristic():
    from fast_plaid_b200.index.build import num_partitions_for

    # SURVEY.md 8: K per BASELINE config
    assert num_partitions_for(1_000 * 300) == 8192
    assert num_partitions_for(100_000 * 300) == 65536
    assert num_partitions_for(1_000_000 * 300) == 262144
    assert num_partitions_for(50_000 * 1024) == 65536


def test_result_lists_c_helper_equals_the_python_zip():
    """csrc/py/results.c builds the list[list[(int, float)]] results; it must equal the pure-Python re-zip
    (types included) for full, partial and empty rows, and leave the garbage collector enabled."""
    import gc

    from fast_plaid_b200.search import fast_plaid as fp

    assert fp._fpb_results is not None, "the CPython helper was not built (make -C fast_plaid_b200/csrc)"
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(-5, 10**9, (7, 13), generator=g)
    sc = torch.randn(7, 13, generator=g)
    cnt = torch.tensor([13, 0, 5, 13, 1, 12, 7], dtype=torch.int32)
    a = fp._results_to_lists(ids, sc, cnt)
    helper, fp._fpb_results = fp._fpb_results, None
    try:
        b = fp._results_to_lists(ids, sc, cnt)
    finally:
        fp._fpb_results = helper
    assert a == b and [len(r) for r in a] == cnt.tolist()
    assert all(type(i) is int and type(s) is float for r in a for i, s in r)
    assert gc.isenabled()
    assert fp._results_to_lists(torch.empty((0, 4), dtype=torch.int64), torch.empty((0, 4)), torch.empty(0, dtype=torch.int32)) == []


def test_sharded_merge_record_limit():
    """The shard merge takes up to 16384 records per query (n_shards * n_full_scores/4): every n_full_scores one GPU
    accepts on 4 shards, up to 8192 (R = 2048) on 8.  A sharded search above that raises ValueError before it makes a
    communicator or gathers anything, in the one-call path and in the step-wise subset path."""
    from fast_plaid_b200.engine import MERGE_MAX_RECORDS, DeviceIndex, check_merge_records
    from fast_plaid_b200.search.fast_plaid import FastPlaid

    assert MERGE_MAX_RECORDS == 16384
    for n_shards, n_full in ((1, 16384), (4, 16384), (4, 16387), (8, 8192), (8, 8195), (16, 4096), (3, 1)):
        check_merge_records(n_shards, n_full)
    for n_shards, n_full in ((8, 8196), (8, 16384), (5, 16384), (16, 4100), (16385, 1)):
        with pytest.raises(ValueError, match="exceed the 16384"):
            check_merge_records(n_shards, n_full)

    class Reached(Exception):
        pass

    def shard_comm(idx):
        raise Reached

    fp = FastPlaid.__new__(FastPlaid)
    fp.shard = (0, 8)  # 8 ranks
    fp._shard_comm = shard_comm
    q = torch.zeros(1, 4, 128)
    for groups, n_full, subset, error in ((1, 8196, None, ValueError), (1, 8196, [[0, 1]], ValueError),
                                          (1, 8192, None, Reached), (2, 16384, None, Reached)):
        fp.query_groups = groups  # 8 / groups document shards
        with pytest.raises(error):
            fp._search_sharded(None, q, DeviceIndex.make_params(10, n_full, 8), subset)


def test_device_list_resolution():
    """fast_plaid.py:350-362: one string, a list, bare "cuda" -> cuda:0, duplicates dropped in order;
    anything else is refused like parse_device (load.rs:16-37)."""
    from fast_plaid_b200.search.fast_plaid import FastPlaid

    r = FastPlaid._resolve_devices
    assert r("cpu") == ["cpu"]
    assert r("cuda") == ["cuda:0"]
    assert r(["cuda:1", "cuda", "cuda:1", "cuda:0"]) == ["cuda:1", "cuda:0"]
    assert r(None) in (["cpu"], [f"cuda:{i}" for i in range(torch.cuda.device_count())])
    for bad in ("gpu", "cuda:x", "cuda:", "xpu:0"):
        with pytest.raises(ValueError):
            r(bad)


def test_query_padding_and_subset_broadcasting():
    """fast_plaid.py:772-793: a list of [Q_i, D] / [1, Q_i, D] tensors is zero-padded to the longest; `subset`
    may be one id, one shared list, one list per query, or empty (= no filter); a wrong length is an error."""
    from fast_plaid_b200.search.fast_plaid import FastPlaid

    a, b = torch.ones(3, 4), torch.full((1, 5, 4), 2.0)
    q = FastPlaid._as_query_tensor([a, b])
    assert q.shape == (2, 5, 4) and bool((q[0, 3:] == 0).all()) and bool((q[1] == 2).all())
    t = torch.zeros(2, 3, 4)
    assert FastPlaid._as_query_tensor(t) is t
    s = FastPlaid._per_query_subsets
    assert s(None, 3) is None and s([], 3) is None
    assert s(7, 2) == [[7], [7]]
    assert s([1, 2], 3) == [[1, 2]] * 3
    assert s([[1], [2, 3]], 2) == [[1], [2, 3]]
    with pytest.raises(ValueError, match="Subset length must match number of queries"):
        s([[1], [2]], 3)


def test_metadata_rows_follow_document_ids_through_updates(tmp_path):
    """update.py:300-311 of the reference: once metadata.db exists every update inserts one row per document
    (an empty one without metadata), so `_subset_` stays the document id."""
    from fast_plaid_b200 import filtering

    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device="cpu")
    fp.create(make_docs(30, 5, 10, seed=9), kmeans_niters=1, metadata=[{"tag": "old"} for _ in range(30)])
    fp.update(make_docs(2, 5, 10, seed=10))  # no metadata: two empty rows, ids 30 and 31
    fp.update(make_docs(1, 5, 10, seed=11), metadata=[{"tag": "new"}])
    assert filtering.where(path, "tag = ?", ("new",)) == [32]
    assert len(filtering.get(path)) == 33 == _meta(path)["num_documents"]
    with pytest.raises(ValueError, match="metadata"):
        fp.update(make_docs(2, 5, 10, seed=12), metadata=[{"tag": "x"}])
    assert not os.path.exists(os.path.join(path, "metadata.db.keep"))


def test_unsafe_metadata_column_names_are_refused(tmp_path):
    """filtering.py:10-12, :159-165 of the reference."""
    fp = search.FastPlaid(str(tmp_path / "idx"), device="cpu")
    with pytest.raises(ValueError, match="Invalid column name"):
        fp.create(make_docs(3, 5, 10, seed=13), kmeans_niters=1,
                  metadata=[{'x" TEXT); DROP TABLE METADATA; --': 1} for _ in range(3)])


def test_create_refuses_what_the_engine_cannot_search(tmp_path):
    fp = search.FastPlaid(str(tmp_path / "idx"), device="cpu")
    with pytest.raises(ValueError, match="dim"):
        fp.create(make_docs(5, 5, 10, dim=96, seed=14), kmeans_niters=1)
    with pytest.raises(ValueError, match="nbits"):
        fp.create(make_docs(5, 5, 10, seed=14), kmeans_niters=1, nbits=8)
    assert not os.path.exists(os.path.join(str(tmp_path / "idx"), "metadata.json"))


def test_delete_trims_a_reference_written_buffer(tmp_path):
    """fast_plaid.py:1118-1145 of the reference: `buffer.npy` holds the raw embeddings of the most recent documents;
    deleting some of them must remove their entries."""
    import numpy as np

    path = str(tmp_path / "idx")
    fp = search.FastPlaid(path, device="cpu")
    docs = make_docs(40, 5, 12, seed=21)
    fp.create(docs, kmeans_niters=1)
    search.fast_plaid.save_list_tensors_on_disk(os.path.join(path, "buffer.npy"), docs[-5:])  # docs 35..39
    fp.delete([3, 36, 39])
    buf = np.load(os.path.join(path, "buffer.npy"), allow_pickle=True)
    assert len(buf) == 3 and np.array_equal(buf[0], docs[35].numpy()) and np.array_equal(buf[2], docs[38].numpy())
    fp.delete([34, 35, 36])  # the three remaining buffer documents are now the last three ids, 34..36
    assert not os.path.exists(os.path.join(path, "buffer.npy"))
