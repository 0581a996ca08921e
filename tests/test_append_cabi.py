"""The growable-buffer and append entry points of the C ABI refuse bad arguments before any CUDA call (no GPU
needed)."""

from __future__ import annotations

import ctypes

from fast_plaid_b200 import engine


def test_buffer_refusals():
    lib = engine.load_library()
    b = ctypes.c_void_p()
    assert lib.fpb_buffer_reserve(None, 0, 0) == engine.FPB_ERR_INVALID
    assert lib.fpb_buffer_reserve(ctypes.byref(b), -1, 0) == engine.FPB_ERR_INVALID and not b.value
    assert b"device" in lib.fpb_last_error()
    assert lib.fpb_buffer_commit(None, 1) == engine.FPB_ERR_INVALID
    assert lib.fpb_buffer_ptr(None) is None
    assert lib.fpb_buffer_mapped_bytes(None) == 0
    lib.fpb_buffer_destroy(None)


def test_index_append_refusals():
    lib = engine.load_library()
    h = ctypes.c_void_p()
    assert lib.fpb_index_append(None, None, 1, 1, None, None, None, None, None, None, 0, 0) == engine.FPB_ERR_INVALID
    assert b"out is NULL" in lib.fpb_last_error()
    assert lib.fpb_index_append(ctypes.byref(h), None, 1, 1, None, None, None, None, None, None, 0, 0) == \
        engine.FPB_ERR_INVALID
    assert b"NULL" in lib.fpb_last_error() and not h.value
    assert lib.fpb_index_walk_group(None) == -1


def test_ivf_append_refusals():
    lib = engine.load_library()
    n = ctypes.c_int64()
    fake = 1 << 40  # never dereferenced: every call below is refused first
    args = (0, 16, fake, fake, 10, 5, fake, fake, fake, fake, 100, ctypes.byref(n), None)

    def call(**kw):
        names = ["device", "n_cells", "offs", "pids", "n_old", "n_new", "new_offs", "codes", "out_offs", "out_pids",
                 "cap", "n", "stream"]
        a = dict(zip(names, args))
        a.update(kw)
        return lib.fpb_ivf_append(*[a[k] for k in names])

    assert call(n_cells=0) == engine.FPB_ERR_INVALID
    assert call(n_old=-1) == engine.FPB_ERR_INVALID
    assert call(n_new=-1) == engine.FPB_ERR_INVALID
    assert call(cap=-1) == engine.FPB_ERR_INVALID
    assert call(offs=None) == engine.FPB_ERR_INVALID
    assert call(out_offs=None) == engine.FPB_ERR_INVALID
    assert call(n=None) == engine.FPB_ERR_INVALID
    assert call(codes=None) == engine.FPB_ERR_INVALID
    assert b"bad sizes or NULL" in lib.fpb_last_error()
    assert call(n_old=1 << 31) == engine.FPB_ERR_UNSUPPORTED
    assert b"int32" in lib.fpb_last_error()
