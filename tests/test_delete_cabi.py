"""The delete entry points of the C ABI refuse bad arguments before any CUDA call (no GPU needed)."""

from __future__ import annotations

import ctypes

from fast_plaid_b200 import engine

FAKE = 1 << 40  # never dereferenced: every call below is refused first


def test_docs_compact_refusals():
    lib = engine.load_library()
    n = ctypes.c_int64()
    names = ["device", "n_docs", "offs", "codes", "res", "norms", "pd", "drop", "n_drop", "out_offs", "out_codes",
             "out_res", "out_norms", "cap", "n", "stream"]
    args = dict(zip(names, (0, 10, FAKE, FAKE, FAKE, FAKE, 64, FAKE, 3, FAKE, FAKE, FAKE, FAKE, 100, ctypes.byref(n),
                            None)))

    def call(**kw):
        a = dict(args, **kw)
        return lib.fpb_docs_compact(*[a[k] for k in names])

    for kw in ({"n_docs": -1}, {"n_drop": -1}, {"n_drop": 11}, {"cap": -1}, {"offs": None}, {"out_offs": None},
               {"n": None}, {"drop": None}):
        assert call(**kw) == engine.FPB_ERR_INVALID, kw
        assert b"bad sizes or NULL" in lib.fpb_last_error()
    for kw in ({"codes": None}, {"res": None}, {"out_res": None}, {"norms": None}, {"out_norms": None}):
        assert call(**kw) == engine.FPB_ERR_INVALID, kw
        assert b"NULL row arrays" in lib.fpb_last_error()
    assert call(res=FAKE + 8) == engine.FPB_ERR_INVALID and b"16-byte" in lib.fpb_last_error()
    assert call(out_res=FAKE + 4) == engine.FPB_ERR_INVALID and b"16-byte" in lib.fpb_last_error()
    for pd in (0, 8, 48, 128):
        assert call(pd=pd) == engine.FPB_ERR_UNSUPPORTED, pd
        assert b"bytes per residual row" in lib.fpb_last_error()
    assert call(n_docs=1 << 31) == engine.FPB_ERR_UNSUPPORTED and b"int32" in lib.fpb_last_error()


def test_ivf_delete_refusals():
    lib = engine.load_library()
    n = ctypes.c_int64()
    names = ["device", "n_cells", "offs", "pids", "n_docs", "drop", "n_drop", "out_offs", "out_pids", "cap", "n",
             "stream"]
    args = dict(zip(names, (0, 16, FAKE, FAKE, 10, FAKE, 3, FAKE, FAKE, 100, ctypes.byref(n), None)))

    def call(**kw):
        a = dict(args, **kw)
        return lib.fpb_ivf_delete(*[a[k] for k in names])

    for kw in ({"n_cells": 0}, {"n_docs": -1}, {"n_drop": -1}, {"n_drop": 11}, {"cap": -1}, {"offs": None},
               {"out_offs": None}, {"n": None}, {"drop": None}):
        assert call(**kw) == engine.FPB_ERR_INVALID, kw
        assert b"bad sizes or NULL" in lib.fpb_last_error()
    assert call(n_docs=1 << 31, n_drop=0) == engine.FPB_ERR_UNSUPPORTED
    assert b"int32" in lib.fpb_last_error()
