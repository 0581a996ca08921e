"""The C-ABI library loads and exports every symbol include/fastplaid_b200.h declares.
No compute call is made (there is no GPU in the CPU test tier)."""

from __future__ import annotations

import ctypes
import os
import re

import pytest
import torch

from fast_plaid_b200 import engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "fastplaid_b200.h")


def _declared_symbols() -> list[str]:
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(fpb_[a-z_0-9]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = engine.load_library()
    declared = _declared_symbols()
    assert len(declared) >= 15
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
    assert sorted(engine.EXPORTED_SYMBOLS) == declared, "engine.EXPORTED_SYMBOLS is out of sync with the header"
    assert lib.fpb_abi_version() == 6


def test_struct_layouts_match_the_header():
    assert ctypes.sizeof(engine.FpbParams) == 20
    # 1 int64 + 10 int32 + 25 int64 + 2 int32
    assert ctypes.sizeof(engine.FpbLayout) == 8 + 10 * 4 + 25 * 8 + 2 * 4


def test_errors_are_reported_not_thrown():
    lib = engine.load_library()
    handle = ctypes.c_void_p()
    # unsupported nbits is rejected before any CUDA call, with a message
    rc = lib.fpb_index_create(ctypes.byref(handle), 0, 3, 128, 16, None, None, 0, None, None, None, None, None, None, 0, 0, 0)
    assert rc == engine.FPB_ERR_UNSUPPORTED
    assert b"nbits" in lib.fpb_last_error()
    rc = lib.fpb_index_create(ctypes.byref(handle), 0, 4, 100, 16, None, None, 0, None, None, None, None, None, None, 0, 0, 0)
    assert rc == engine.FPB_ERR_UNSUPPORTED and b"dim" in lib.fpb_last_error()
    rc = lib.fpb_workspace_layout(None, 1, 1, None, None)
    assert rc == engine.FPB_ERR_INVALID
    rc = lib.fpb_merge_shards(None, 1, 1, 1, 1, None, None, None, None)
    assert rc == engine.FPB_ERR_INVALID


def test_build_kernels_refuse_what_they_do_not_encode():
    """fpb_encode handles dim 128 with nbits 2 or 4 and the k-means kernels dim 128; the refusal comes before any
    CUDA call.  Zero tokens or points is a no-op that succeeds and writes nothing (host buffers stand in for device
    ones: they are never touched)."""
    lib = engine.load_library()
    for nbits, dim in ((4, 64), (2, 96), (3, 128), (8, 128)):
        rc = lib.fpb_encode(0, nbits, dim, 16, None, None, 10, None, None, None, None)
        assert rc == engine.FPB_ERR_UNSUPPORTED, (nbits, dim)
        assert b"dim=128 with nbits 2 or 4" in lib.fpb_last_error()
    assert lib.fpb_kmeans_assign(0, 64, 16, None, None, None, 10, None, None) == engine.FPB_ERR_UNSUPPORTED
    assert b"dim=128" in lib.fpb_last_error()
    assert lib.fpb_kmeans_update(0, 256, 16, None, None, None, None, None, None) == engine.FPB_ERR_UNSUPPORTED
    assert b"dim=128" in lib.fpb_last_error()
    cent = torch.zeros(16, 128, dtype=torch.float16)
    cut = torch.zeros(15)
    codes = torch.full((4,), -7, dtype=torch.int32)
    res = torch.full((4, 64), 0xA5, dtype=torch.uint8)
    rc = lib.fpb_encode(0, 4, 128, 16, cent.data_ptr(), cent.data_ptr(), 0, cut.data_ptr(), codes.data_ptr(),
                        res.data_ptr(), None)
    assert rc == engine.FPB_OK
    bias = torch.zeros(16)
    rc = lib.fpb_kmeans_assign(0, 128, 16, cent.data_ptr(), bias.data_ptr(), cent.data_ptr(), 0, codes.data_ptr(), None)
    assert rc == engine.FPB_OK
    assert bool((codes == -7).all()) and bool((res == 0xA5).all())


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback_without_cuda():
    from fast_plaid_b200.engine import DeviceIndex, EngineUnavailableError, IndexTensors

    t = IndexTensors(4, torch.zeros(16, 128), torch.zeros(16), torch.tensor([1]), torch.zeros(1, dtype=torch.int64),
                     torch.zeros(1, 64, dtype=torch.uint8), None, None)
    with pytest.raises(EngineUnavailableError):
        DeviceIndex(t, "cuda:0")


def test_product_never_imports_the_oracle():
    """The oracle is test infrastructure: nothing under fast_plaid_b200/ may reference it."""
    pkg = os.path.join(ROOT, "fast_plaid_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f"{f} imports oracle"
                assert "plaid_oracle" not in src and "index_oracle" not in src, f"{f} mentions the oracle modules"


def test_host_cast_equals_the_aten_cast():
    """fpb_cast_f32_to_f16_host (F16C) and its portable twin reproduce torch's fp32 -> fp16 cast bit for bit:
    random values over the whole exponent range, every fp16 rounding midpoint and its two neighbours,
    subnormals, overflow to inf, signed zeros, inf, NaN."""
    lib = engine.load_library()
    g = torch.Generator().manual_seed(0)
    h = torch.arange(0, 0x7C00, dtype=torch.int16).view(torch.float16).float()
    mid = (h[:-1] + h[1:]) / 2
    inf = torch.tensor(float("inf"))
    x = torch.cat([
        torch.randn(50_000, generator=g), torch.randn(20_000, generator=g) * 1e-5, torch.randn(20_000, generator=g) * 1e4,
        torch.randn(20_000, generator=g) * 1e-7, mid, -mid, torch.nextafter(mid, inf), torch.nextafter(mid, -inf),
        torch.tensor([0.0, -0.0, float("inf"), -float("inf"), float("nan"), 65504.0, 65519.9, 65520.0, 65536.0, 1e-8,
                      2.9802322e-8, 2.98e-8, 5.96e-8, 6.0975552e-05, 6.1e-5]),
    ]).contiguous()
    ref = x.to(torch.float16)
    for fn in (lib.fpb_cast_f32_to_f16_host, lib.fpb_cast_f32_to_f16_host_portable):
        out = torch.empty(x.shape, dtype=torch.float16)
        assert fn(x.data_ptr(), out.data_ptr(), x.numel()) == 0
        same = (out.view(torch.int16) == ref.view(torch.int16)) | (torch.isnan(out) & torch.isnan(ref))
        assert bool(same.all()), int((~same).sum())
