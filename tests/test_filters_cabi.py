"""The filter entry points of the C ABI refuse bad arguments before any CUDA call (no GPU needed): NULL pointers,
n_filters < 1, n_bits < 0, a query-filter map entry out of range and a missing FPB_FLAG_SUBSET.  Host buffers stand
in for device ones: a refused call never touches them."""

from __future__ import annotations

import ctypes

import torch

from fast_plaid_b200 import engine


def _err() -> bytes:
    return engine.load_library().fpb_last_error()


def test_bitmap_builders_refuse_bad_arguments():
    lib = engine.load_library()
    ids = torch.zeros(4, dtype=torch.int64)
    offs = torch.tensor([0, 4], dtype=torch.int64)
    bm = torch.zeros(4, dtype=torch.int32)
    mask = torch.zeros(8, dtype=torch.bool)
    assert lib.fpb_filter_from_ids(0, None, 4, 1, offs.data_ptr(), 32, bm.data_ptr(), None) == engine.FPB_ERR_INVALID
    assert lib.fpb_filter_from_ids(0, ids.data_ptr(), 4, 1, None, 32, bm.data_ptr(), None) == engine.FPB_ERR_INVALID
    assert lib.fpb_filter_from_ids(0, ids.data_ptr(), 4, 1, offs.data_ptr(), 32, None, None) == engine.FPB_ERR_INVALID
    assert b"NULL" in _err()
    for n_filters, n_bits in ((0, 32), (-1, 32), (1, -1)):
        assert lib.fpb_filter_from_ids(0, ids.data_ptr(), 4, n_filters, offs.data_ptr(), n_bits, bm.data_ptr(),
                                       None) == engine.FPB_ERR_INVALID
        assert b"n_filters" in _err()
        assert lib.fpb_filter_from_mask(0, mask.data_ptr(), n_filters, n_bits, bm.data_ptr(), None) \
            == engine.FPB_ERR_INVALID
        assert b"n_filters" in _err()
    assert lib.fpb_filter_from_mask(0, None, 1, 8, bm.data_ptr(), None) == engine.FPB_ERR_INVALID
    assert lib.fpb_filter_from_mask(0, mask.data_ptr(), 1, 8, None, None) == engine.FPB_ERR_INVALID


def test_filtered_searches_refuse_bad_arguments():
    lib = engine.load_library()
    buf = torch.zeros(256, dtype=torch.uint8)
    bm = torch.zeros(2, dtype=torch.int32)
    out = torch.zeros(16, dtype=torch.int64)
    ok = engine.FpbParams(8, 64, 10, 2000, engine.FPB_FLAG_SUBSET)
    no_flag = engine.FpbParams(8, 64, 10, 2000, 0)
    good, bad = (ctypes.c_int32 * 2)(0, 0), (ctypes.c_int32 * 2)(0, 1)
    p = ctypes.byref

    def batch(params=ok, bitmap=bm.data_ptr(), n_filters=1, n_bits=64, h_map=good, queries=buf.data_ptr()):
        return lib.fpb_search_batch_filter(None, queries, 2, 4, p(params), bitmap, n_filters, n_bits, h_map,
                                           buf.data_ptr(), buf.numel(), out.data_ptr(), out.data_ptr(),
                                           out.data_ptr(), None)

    def begin(params=ok, bitmap=bm.data_ptr(), n_filters=1, n_bits=64, h_map=good, queries=buf.data_ptr()):
        return lib.fpb_shard_filter_begin(None, queries, 2, 4, p(params), bitmap, n_filters, n_bits, h_map,
                                          buf.data_ptr(), buf.numel(), out.data_ptr(), None)

    def stage(params=ok, bitmap=bm.data_ptr(), n_filters=1, n_bits=64, h_map=good, queries=None):
        return lib.fpb_stage_filter(None, bitmap, n_filters, n_bits, h_map, 2, 4, p(params), buf.data_ptr(),
                                    buf.numel(), None)

    for fn in (batch, begin, stage):
        for kw, what in (({"bitmap": None}, b"NULL"), ({"h_map": None}, b"NULL"), ({"n_filters": 0}, b"n_filters"),
                         ({"n_bits": -1}, b"n_bits"), ({"h_map": bad}, b"h_query_filter[1]=1"),
                         ({"params": no_flag}, b"FPB_FLAG_SUBSET")):
            assert fn(**kw) == engine.FPB_ERR_INVALID, (fn.__name__, kw)
            assert what in _err(), (fn.__name__, kw, _err())
        assert fn() == engine.FPB_ERR_INVALID and b"NULL index" in _err()  # the index is checked last
    assert batch(queries=None) == engine.FPB_ERR_INVALID and b"NULL query" in _err()
    assert begin(queries=None) == engine.FPB_ERR_INVALID and b"NULL query" in _err()

    def exhaustive(bitmap=bm.data_ptr(), n_filters=1, n_bits=64, max_count=10, h_map=good, top_k=10):
        return lib.fpb_search_exhaustive_filter(None, buf.data_ptr(), 2, 4, top_k, bitmap, n_filters, n_bits,
                                                max_count, h_map, buf.data_ptr(), buf.numel(), out.data_ptr(),
                                                out.data_ptr(), out.data_ptr(), None)

    for kw, what in (({"bitmap": None}, b"NULL"), ({"h_map": None}, b"NULL"), ({"n_filters": 0}, b"n_filters"),
                     ({"n_bits": -1}, b"n_bits"), ({"h_map": bad}, b"h_query_filter[1]=1"),
                     ({"max_count": -1}, b"max_count"), ({"top_k": 0}, b"top_k")):
        assert exhaustive(**kw) == engine.FPB_ERR_INVALID, kw
        assert what in _err(), (kw, _err())
    assert exhaustive(n_filters=70000, h_map=good) == engine.FPB_ERR_UNSUPPORTED
    assert exhaustive() == engine.FPB_ERR_INVALID and b"NULL index" in _err()
    size = ctypes.c_size_t()
    assert lib.fpb_exhaustive_filter_workspace_bytes(None, 2, 4, 10, 0, 10, p(size)) == engine.FPB_ERR_INVALID
    assert lib.fpb_exhaustive_filter_workspace_bytes(None, 2, 4, 10, 1, -1, p(size)) == engine.FPB_ERR_INVALID
    assert lib.fpb_exhaustive_filter_workspace_bytes(None, 2, 4, 10, 1, 10, None) == engine.FPB_ERR_INVALID
