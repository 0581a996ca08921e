"""ctypes binding of ``libfastplaid_b200.so`` (C ABI in ``include/fastplaid_b200.h``).

This is the only bridge between the Python host and the CUDA kernels.  There is no CPU
fallback: if the shared library is missing or CUDA is unavailable every entry point raises.
PyTorch is used for device memory, streams and (in the sharded mode) ``torch.distributed``.

Reference counterpart: the PyO3 module ``fast_plaid.fast_plaid_rust`` (rust/lib.rs:366-383):
``construct_index`` -> :class:`DeviceIndex`, ``pysearch`` -> :meth:`DeviceIndex.search`.
"""

from __future__ import annotations

import contextlib
import ctypes
import dataclasses
import os
import threading
from typing import Any

import torch

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libfastplaid_b200.so")
_lib = None
_lib_lock = threading.Lock()

FPB_OK = 0
FPB_ERR_INVALID = -1
FPB_ERR_CUDA = -2
FPB_ERR_UNSUPPORTED = -3
FPB_ERR_WORKSPACE = -4
FPB_ERR_NO_IVF = -5


class EngineUnavailableError(RuntimeError):
    """The CUDA extension is missing or unusable.  There is deliberately no fallback."""


class FpbParams(ctypes.Structure):
    _fields_ = [
        ("n_ivf_probe", ctypes.c_int32),
        ("n_full_scores", ctypes.c_int32),
        ("top_k", ctypes.c_int32),
        ("batch_size", ctypes.c_int32),
        ("flags", ctypes.c_int32),
    ]


FPB_FLAG_SUBSET = 1
FPB_FLAG_APPROX_EXACT_ALL = 2  # off_approx holds the exact score of every candidate (parity tests)
FPB_FLAG_APPROX_DIRECT = 4  # one-pass approximate scoring (A/B alternative of the two-pass default)
FPB_FLAG_APPROX_TWO_PASS = 8  # two passes even for a job the library would score in one (small batch x index)


class FpbLayout(ctypes.Structure):
    _fields_ = [
        ("total_bytes", ctypes.c_int64),
        ("B", ctypes.c_int32),
        ("Q", ctypes.c_int32),
        ("Qp", ctypes.c_int32),
        ("n_tiles", ctypes.c_int32),
        ("R", ctypes.c_int32),
        ("n_probe", ctypes.c_int32),
        ("cand_cap", ctypes.c_int32),
        ("bitmap_words", ctypes.c_int32),
        ("cbitmap_words", ctypes.c_int32),
        ("reserved0", ctypes.c_int32),
        ("off_queries", ctypes.c_int64),
        ("off_S", ctypes.c_int64),
        ("off_tmax", ctypes.c_int64),
        ("off_cells", ctypes.c_int64),
        ("off_bitmap", ctypes.c_int64),
        ("off_n_cand", ctypes.c_int64),
        ("off_cand", ctypes.c_int64),
        ("off_approx", ctypes.c_int64),
        ("off_work", ctypes.c_int64),
        ("off_n_rerank", ctypes.c_int64),
        ("off_rerank", ctypes.c_int64),
        ("off_rerank_approx", ctypes.c_int64),
        ("off_exact", ctypes.c_int64),
        ("off_cbitmap", ctypes.c_int64),
        ("off_clist", ctypes.c_int64),
        ("off_n_clist", ctypes.c_int64),
        ("off_sbitmap", ctypes.c_int64),
        ("off_tau", ctypes.c_int64),
        ("off_hibits", ctypes.c_int64),
        ("off_lb", ctypes.c_int64),
        ("off_refine", ctypes.c_int64),
        ("off_n_refine", ctypes.c_int64),
        ("off_thresh", ctypes.c_int64),
        ("off_work2", ctypes.c_int64),
        ("off_stats", ctypes.c_int64),
        ("hb_words", ctypes.c_int32),
        ("flags", ctypes.c_int32),
    ]


# every symbol include/fastplaid_b200.h declares (checked by tests/test_cabi.py)
EXPORTED_SYMBOLS = [
    "fpb_last_error",
    "fpb_abi_version",
    "fpb_index_create",
    "fpb_index_destroy",
    "fpb_index_walk_layout",
    "fpb_index_walk_group",
    "fpb_index_append",
    "fpb_index_with_groups",
    "fpb_index_with_groups_max",
    "fpb_index_with_shard_groups",
    "fpb_index_with_bias",
    "fpb_ivf_append",
    "fpb_docs_compact",
    "fpb_ivf_delete",
    "fpb_buffer_reserve",
    "fpb_buffer_commit",
    "fpb_buffer_ptr",
    "fpb_buffer_mapped_bytes",
    "fpb_buffer_destroy",
    "fpb_workspace_layout",
    "fpb_search_batch",
    "fpb_search_batch_subset",
    "fpb_search_batch_host",
    "fpb_filter_from_ids",
    "fpb_filter_from_mask",
    "fpb_search_batch_filter",
    "fpb_stage_filter",
    "fpb_shard_filter_begin",
    "fpb_exhaustive_filter_workspace_bytes",
    "fpb_search_exhaustive_filter",
    "fpb_stage_centroid_scores",
    "fpb_stage_subset",
    "fpb_stage_probe",
    "fpb_stage_candidates",
    "fpb_stage_approx",
    "fpb_stage_select",
    "fpb_stage_maxsim",
    "fpb_stage_rank",
    "fpb_stage_keys",
    "fpb_stage_records",
    "fpb_stage_group_rank",
    "fpb_search_shard",
    "fpb_merge_shards",
    "fpb_merge_shards_grouped",
    "fpb_shard_approx_keys",
    "fpb_shard_subset_begin",
    "fpb_shard_subset_keys",
    "fpb_shard_apply_threshold",
    "fpb_shard_exact_records",
    "fpb_comm_unique_id",
    "fpb_comm_create",
    "fpb_comm_destroy",
    "fpb_comm_nccl_version",
    "fpb_sharded_scratch_bytes",
    "fpb_search_batch_sharded",
    "fpb_search_batch_sharded_host",
    "fpb_exhaustive_workspace_bytes",
    "fpb_exhaustive_scores",
    "fpb_search_exhaustive",
    "fpb_exhaustive_subset_workspace_bytes",
    "fpb_search_exhaustive_subset",
    "fpb_shard_exhaustive_records",
    "fpb_search_exhaustive_sharded",
    "fpb_reconstruct",
    "fpb_token_scores",
    "fpb_encode",
    "fpb_kmeans_assign",
    "fpb_kmeans_update",
    "fpb_cast_f32_to_f16_host",
    "fpb_cast_f32_to_f16_host_portable",
]


def library_path() -> str:
    return _LIB_PATH


def load_library() -> ctypes.CDLL:
    """dlopen the C-ABI library (no CUDA call is made)."""
    global _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(_LIB_PATH):
            raise EngineUnavailableError(
                f"{_LIB_PATH} not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                f"or `make -C fast_plaid_b200/csrc`. The engine has no CPU fallback."
            )
        lib = ctypes.CDLL(_LIB_PATH)
        vp, i32, i64, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_size_t
        lib.fpb_last_error.restype = ctypes.c_char_p
        lib.fpb_last_error.argtypes = []
        lib.fpb_abi_version.restype = i32
        lib.fpb_index_create.restype = i32
        lib.fpb_index_create.argtypes = [
            ctypes.POINTER(vp), i32, i32, i32, i64, vp, vp, i64, vp, vp, vp, vp, vp, vp, i64, i64, i64,
        ]
        lib.fpb_index_destroy.restype = None
        lib.fpb_index_destroy.argtypes = [vp]
        lib.fpb_index_walk_layout.restype = i32
        lib.fpb_index_walk_layout.argtypes = [vp, ctypes.POINTER(i64), vp, vp]
        lib.fpb_index_walk_group.restype = i32
        lib.fpb_index_walk_group.argtypes = [vp]
        lib.fpb_index_append.restype = i32
        lib.fpb_index_append.argtypes = [ctypes.POINTER(vp), vp, i64, i64, vp, vp, vp, vp, vp, vp, i64, i64]
        lib.fpb_index_with_groups.restype = i32
        lib.fpb_index_with_groups.argtypes = [ctypes.POINTER(vp), vp, vp, i64]
        lib.fpb_index_with_groups_max.restype = i32
        lib.fpb_index_with_groups_max.argtypes = [ctypes.POINTER(vp), vp, vp, i64, i32]
        lib.fpb_index_with_shard_groups.restype = i32
        lib.fpb_index_with_shard_groups.argtypes = [ctypes.POINTER(vp), vp, vp, i64, i32, vp, i64]
        lib.fpb_index_with_bias.restype = i32
        lib.fpb_index_with_bias.argtypes = [ctypes.POINTER(vp), vp, vp, i64]
        lib.fpb_ivf_append.restype = i32
        lib.fpb_ivf_append.argtypes = [i32, i64, vp, vp, i64, i64, vp, vp, vp, vp, i64, ctypes.POINTER(i64), vp]
        lib.fpb_docs_compact.restype = i32
        lib.fpb_docs_compact.argtypes = [i32, i64, vp, vp, vp, vp, i32, vp, i64, vp, vp, vp, vp, i64,
                                         ctypes.POINTER(i64), vp]
        lib.fpb_ivf_delete.restype = i32
        lib.fpb_ivf_delete.argtypes = [i32, i64, vp, vp, i64, vp, i64, vp, vp, i64, ctypes.POINTER(i64), vp]
        lib.fpb_buffer_reserve.restype = i32
        lib.fpb_buffer_reserve.argtypes = [ctypes.POINTER(vp), i32, sz]
        lib.fpb_buffer_commit.restype = i32
        lib.fpb_buffer_commit.argtypes = [vp, sz]
        lib.fpb_buffer_ptr.restype = vp
        lib.fpb_buffer_ptr.argtypes = [vp]
        lib.fpb_buffer_mapped_bytes.restype = sz
        lib.fpb_buffer_mapped_bytes.argtypes = [vp]
        lib.fpb_buffer_destroy.restype = None
        lib.fpb_buffer_destroy.argtypes = [vp]
        lib.fpb_workspace_layout.restype = i32
        lib.fpb_workspace_layout.argtypes = [vp, i32, i32, ctypes.POINTER(FpbParams), ctypes.POINTER(FpbLayout)]
        lib.fpb_search_batch.restype = i32
        lib.fpb_search_batch.argtypes = [vp, vp, i32, i32, ctypes.POINTER(FpbParams), vp, sz, vp, vp, vp, vp]
        lib.fpb_search_batch_subset.restype = i32
        lib.fpb_search_batch_subset.argtypes = [vp, vp, i32, i32, ctypes.POINTER(FpbParams), vp, vp, i64, vp, sz,
                                                vp, vp, vp, vp]
        lib.fpb_stage_subset.restype = i32
        lib.fpb_stage_subset.argtypes = [vp, vp, vp, i64, i32, i32, ctypes.POINTER(FpbParams), vp, sz, vp]
        lib.fpb_filter_from_ids.restype = i32
        lib.fpb_filter_from_ids.argtypes = [i32, vp, i64, i32, vp, i64, vp, vp]
        lib.fpb_filter_from_mask.restype = i32
        lib.fpb_filter_from_mask.argtypes = [i32, vp, i32, i64, vp, vp]
        lib.fpb_search_batch_filter.restype = i32
        lib.fpb_search_batch_filter.argtypes = [vp, vp, i32, i32, ctypes.POINTER(FpbParams), vp, i32, i64, vp, vp, sz,
                                                vp, vp, vp, vp]
        lib.fpb_stage_filter.restype = i32
        lib.fpb_stage_filter.argtypes = [vp, vp, i32, i64, vp, i32, i32, ctypes.POINTER(FpbParams), vp, sz, vp]
        lib.fpb_shard_filter_begin.restype = i32
        lib.fpb_shard_filter_begin.argtypes = [vp, vp, i32, i32, ctypes.POINTER(FpbParams), vp, i32, i64, vp, vp, sz,
                                               vp, vp]
        lib.fpb_exhaustive_filter_workspace_bytes.restype = i32
        lib.fpb_exhaustive_filter_workspace_bytes.argtypes = [vp, i32, i32, i32, i32, i64, ctypes.POINTER(sz)]
        lib.fpb_search_exhaustive_filter.restype = i32
        lib.fpb_search_exhaustive_filter.argtypes = [vp, vp, i32, i32, i32, vp, i32, i64, i64, vp, vp, sz, vp, vp,
                                                     vp, vp]
        lib.fpb_search_batch_host.restype = i32
        lib.fpb_search_batch_host.argtypes = [
            vp, vp, i32, i32, ctypes.POINTER(FpbParams), vp, sz, vp, vp, vp, vp, vp, vp, vp, vp,
        ]
        lib.fpb_stage_centroid_scores.restype = i32
        lib.fpb_stage_centroid_scores.argtypes = [vp, vp, i32, i32, ctypes.POINTER(FpbParams), vp, sz, vp]
        for name in ("fpb_stage_probe", "fpb_stage_candidates", "fpb_stage_approx", "fpb_stage_select",
                     "fpb_stage_maxsim"):
            fn = getattr(lib, name)
            fn.restype = i32
            fn.argtypes = [vp, i32, i32, ctypes.POINTER(FpbParams), vp, sz, vp]
        lib.fpb_stage_rank.restype = i32
        lib.fpb_stage_rank.argtypes = [vp, i32, i32, ctypes.POINTER(FpbParams), vp, sz, vp, vp, vp, vp]
        lib.fpb_stage_keys.restype = i32
        lib.fpb_stage_keys.argtypes = [vp, i32, i32, ctypes.POINTER(FpbParams), vp, sz, vp, vp]
        lib.fpb_stage_records.restype = i32
        lib.fpb_stage_records.argtypes = [vp, i32, i32, ctypes.POINTER(FpbParams), vp, sz, vp, vp]
        lib.fpb_stage_group_rank.restype = i32
        lib.fpb_stage_group_rank.argtypes = [vp, vp, vp, vp, i64, i32, i32, vp, sz, vp, vp, vp, vp]
        lib.fpb_search_shard.restype = i32
        lib.fpb_search_shard.argtypes = [vp, vp, i32, i32, ctypes.POINTER(FpbParams), vp, sz, vp, vp]
        lib.fpb_shard_approx_keys.restype = i32
        lib.fpb_shard_approx_keys.argtypes = [vp, vp, i32, i32, ctypes.POINTER(FpbParams), vp, sz, vp, vp]
        lib.fpb_shard_subset_begin.restype = i32
        lib.fpb_shard_subset_begin.argtypes = [vp, vp, i32, i32, ctypes.POINTER(FpbParams), vp, vp, i64, vp, sz, vp, vp]
        lib.fpb_shard_subset_keys.restype = i32
        lib.fpb_shard_subset_keys.argtypes = [vp, i32, i32, ctypes.POINTER(FpbParams), vp, sz, vp, i32, vp, vp]
        lib.fpb_shard_apply_threshold.restype = i32
        lib.fpb_shard_apply_threshold.argtypes = [vp, vp, i32, i32, i32, i32, ctypes.POINTER(FpbParams), vp, sz, vp]
        lib.fpb_shard_exact_records.restype = i32
        lib.fpb_shard_exact_records.argtypes = [vp, i32, i32, ctypes.POINTER(FpbParams), vp, sz, vp, vp]
        lib.fpb_comm_unique_id.restype = i32
        lib.fpb_comm_unique_id.argtypes = [vp]
        lib.fpb_comm_create.restype = i32
        lib.fpb_comm_create.argtypes = [ctypes.POINTER(vp), i32, i32, vp, i32]
        lib.fpb_comm_destroy.restype = None
        lib.fpb_comm_destroy.argtypes = [vp]
        lib.fpb_comm_nccl_version.restype = i32
        lib.fpb_sharded_scratch_bytes.restype = i64
        lib.fpb_sharded_scratch_bytes.argtypes = [i32, i32, i32]
        lib.fpb_search_batch_sharded.restype = i32
        lib.fpb_search_batch_sharded.argtypes = [vp, vp, i32, vp, i32, i32, ctypes.POINTER(FpbParams), vp, sz, vp, sz,
                                                 vp, vp, vp, vp]
        lib.fpb_search_batch_sharded_host.restype = i32
        lib.fpb_search_batch_sharded_host.argtypes = [vp, vp, i32, vp, i32, i32, ctypes.POINTER(FpbParams), vp, sz, vp,
                                                      sz, vp, vp, vp, vp, vp, vp, vp, vp]
        lib.fpb_merge_shards.restype = i32
        lib.fpb_merge_shards.argtypes = [vp, i32, i32, i32, i32, vp, vp, vp, vp]
        lib.fpb_merge_shards_grouped.restype = i32
        lib.fpb_merge_shards_grouped.argtypes = [vp, i32, i32, i32, i32, i32, vp, i64, i32, vp, vp, vp, vp]
        lib.fpb_reconstruct.restype = i32
        lib.fpb_reconstruct.argtypes = [vp, vp, i32, vp, vp, vp]
        for name in ("fpb_cast_f32_to_f16_host", "fpb_cast_f32_to_f16_host_portable"):
            fn = getattr(lib, name)
            fn.restype = i32
            fn.argtypes = [vp, vp, sz]
        lib.fpb_encode.restype = i32
        lib.fpb_encode.argtypes = [i32, i32, i32, i64, vp, vp, i64, vp, vp, vp, vp]
        lib.fpb_kmeans_assign.restype = i32
        lib.fpb_kmeans_assign.argtypes = [i32, i32, i64, vp, vp, vp, i64, vp, vp]
        lib.fpb_kmeans_update.restype = i32
        lib.fpb_kmeans_update.argtypes = [i32, i32, i64, vp, vp, vp, vp, vp, vp]
        lib.fpb_token_scores.restype = i32
        lib.fpb_token_scores.argtypes = [vp, vp, i32, vp, vp, i32, i64, vp, vp]
        lib.fpb_exhaustive_workspace_bytes.restype = i32
        lib.fpb_exhaustive_workspace_bytes.argtypes = [vp, i32, i32, i32, ctypes.POINTER(sz)]
        lib.fpb_exhaustive_scores.restype = i32
        lib.fpb_exhaustive_scores.argtypes = [vp, vp, i32, i32, vp, sz, vp, vp]
        lib.fpb_search_exhaustive.restype = i32
        lib.fpb_search_exhaustive.argtypes = [vp, vp, i32, i32, i32, vp, sz, vp, vp, vp, vp]
        lib.fpb_exhaustive_subset_workspace_bytes.restype = i32
        lib.fpb_exhaustive_subset_workspace_bytes.argtypes = [vp, i32, i32, i32, i32, i64, ctypes.POINTER(sz)]
        lib.fpb_search_exhaustive_subset.restype = i32
        lib.fpb_search_exhaustive_subset.argtypes = [vp, vp, i32, i32, i32, vp, vp, i32, i64, vp, vp, sz, vp, vp, vp,
                                                     vp]
        lib.fpb_shard_exhaustive_records.restype = i32
        lib.fpb_shard_exhaustive_records.argtypes = [vp, vp, i32, i32, i32, vp, sz, vp, vp]
        lib.fpb_search_exhaustive_sharded.restype = i32
        lib.fpb_search_exhaustive_sharded.argtypes = [vp, vp, i32, vp, i32, i32, i32, vp, sz, vp, sz, vp, vp, vp, vp]
        _lib = lib
        return lib


def _check(rc: int) -> None:
    if rc == FPB_OK:
        return
    msg = load_library().fpb_last_error().decode("utf-8", "replace")
    if rc in (FPB_ERR_INVALID, FPB_ERR_NO_IVF, FPB_ERR_UNSUPPORTED):
        raise ValueError(msg)  # anyhow -> PyValueError in the reference (rust/utils/errors.rs:5-7)
    raise RuntimeError(msg)


def group_subsets(subset) -> tuple[list, list[int]]:
    """Per-query id lists -> (distinct lists, the list of every query).  Identical lists become one, so that the
    queries that share it share one decode of each of its documents: by object identity first (the broadcast
    ``subset=[ids]`` form in one step), then by equal contents.  An empty list stays a list of its own."""
    lists: list = []
    query_list: list[int] = []
    by_object: dict[int, int] = {}
    by_contents: dict[tuple, int] = {}
    for s in subset:
        l = by_object.get(id(s))  # `subset` keeps every object alive, so an id is not reused during the loop
        if l is None:
            key = tuple(int(i) for i in s)
            l = by_contents.get(key)
            if l is None:
                l = by_contents[key] = len(lists)
                lists.append(s)
            by_object[id(s)] = l
        query_list.append(l)
    return lists, query_list


@dataclasses.dataclass
class Filter:
    """Search filters in their device form: `bitmap` int32 [n_filters, ceil(n_bits / 32)] over GLOBAL document ids
    (document i is bit i & 31 of word i >> 5; ids >= n_bits are never set) on the index's device, and the filter of
    every query (`query_filter`, host ints).  Queries that share a filter share its expansion on the device."""
    bitmap: torch.Tensor
    query_filter: list[int]
    n_bits: int

    @property
    def n_filters(self) -> int:
        return int(self.bitmap.shape[0])

    def queries(self, s: int, e: int) -> "Filter":
        """The filters of queries s..e-1 (the same bitmaps)."""
        return Filter(self.bitmap, self.query_filter[s:e], self.n_bits)

    def call_rows(self, s: int, e: int) -> tuple[torch.Tensor, list[int]]:
        """What one call over queries s..e-1 passes: the rows of the filters they use (a view when those rows are
        contiguous, a gathered copy otherwise) and every query's index among them."""
        used = sorted(set(self.query_filter[s:e]))
        if used[-1] - used[0] + 1 == len(used):
            rows = self.bitmap[used[0]:used[-1] + 1]
        else:
            rows = self.bitmap.index_select(0, torch.tensor(used, device=self.bitmap.device))
        local = {f: i for i, f in enumerate(used)}
        return rows, [local[f] for f in self.query_filter[s:e]]

    @staticmethod
    def from_ids(ids: torch.Tensor, n_bits: int, device: torch.device | str, num_queries: int) -> "Filter":
        """ids: integer [L] (one filter for all num_queries queries) or [num_queries, L] (one per query), any device.
        Any order; duplicates count once; ids outside [0, n_bits) are ignored (-1 pads a row)."""
        device = torch.device(device)
        rows = ids.reshape(1, -1) if ids.dim() == 1 else ids
        F, L = int(rows.shape[0]), int(rows.shape[1])
        flat = rows.to(device=device, dtype=torch.int64).contiguous().view(-1)
        offs = torch.arange(F + 1, dtype=torch.int64, device=device) * L
        words = (int(n_bits) + 31) // 32
        bitmap = torch.empty((F, words), dtype=torch.int32, device=device)
        with torch.cuda.device(device):
            _check(load_library().fpb_filter_from_ids(
                device.index or 0, flat.data_ptr() if flat.numel() else None, flat.numel(), F, offs.data_ptr(),
                int(n_bits), bitmap.data_ptr(), torch.cuda.current_stream(device).cuda_stream))
        return Filter(bitmap, [0] * num_queries if ids.dim() == 1 else list(range(F)), int(n_bits))

    @staticmethod
    def from_mask(mask: torch.Tensor, device: torch.device | str, num_queries: int) -> "Filter":
        """mask: bool [n] (one filter for all num_queries queries) or [num_queries, n] (one per query), any device;
        n_bits = n."""
        device = torch.device(device)
        rows = mask.reshape(1, -1) if mask.dim() == 1 else mask
        F, n = int(rows.shape[0]), int(rows.shape[1])
        m = rows.to(device=device, dtype=torch.bool).contiguous()
        bitmap = torch.empty((F, (n + 31) // 32), dtype=torch.int32, device=device)
        if m.numel():
            with torch.cuda.device(device):
                _check(load_library().fpb_filter_from_mask(device.index or 0, m.data_ptr(), F, n, bitmap.data_ptr(),
                                                           torch.cuda.current_stream(device).cuda_stream))
        return Filter(bitmap, [0] * num_queries if mask.dim() == 1 else list(range(F)), n)


# The largest max_per_group (FPB_MAX_PER_GROUP): exact search takes one pass over the scores per kept document
MAX_PER_GROUP = 64


@dataclasses.dataclass
class Groups:
    """Grouped results in their device form: `ids` int32 [num_documents] on the index's device, the group of every
    document renumbered densely to 0 .. n_groups - 1 (fpb_index_with_groups_max).  Each query then gets at most
    `max_per_group` documents per group, the group's best ones.  On one shard of a document-sharded index
    (`for_shard`), `ids` covers the shard's documents and `global_ids` int32 [n_total] the whole index's, for the merge
    across ranks (fpb_index_with_shard_groups)."""
    ids: torch.Tensor
    n_groups: int
    max_per_group: int = 1
    global_ids: torch.Tensor | None = None

    @staticmethod
    def check_max_per_group(max_per_group, group_by) -> None:
        """Refuses a max_per_group that is not an int in [1, MAX_PER_GROUP], or that is not 1 without a group map."""
        if type(max_per_group) is not int:  # noqa: E721  (bool is an int subclass, and is refused)
            raise ValueError(f"max_per_group must be an int, got {type(max_per_group).__name__}")
        if not 1 <= max_per_group <= MAX_PER_GROUP:
            raise ValueError(f"max_per_group={max_per_group} must be in [1, {MAX_PER_GROUP}]")
        if max_per_group != 1 and group_by is None:
            raise ValueError("max_per_group applies to grouped results: pass group_by= as well")

    @staticmethod
    def check(group_by, num_documents: int) -> None:
        """Refuses a group map that is not a 1-D integer tensor of `num_documents` non-negative values."""
        if not isinstance(group_by, torch.Tensor):
            raise ValueError(f"group_by must be a 1-D integer tensor, got {type(group_by).__name__}")
        if group_by.dtype.is_floating_point or group_by.dtype.is_complex or group_by.dtype == torch.bool:
            raise ValueError(f"group_by must hold integer group ids, got {group_by.dtype}")
        if group_by.dim() != 1:
            raise ValueError(f"group_by must be 1-D (one group per document), got shape {list(group_by.shape)}")
        if group_by.shape[0] != num_documents:
            raise ValueError(f"group_by has {group_by.shape[0]} entries, the index has {num_documents} documents")
        if group_by.numel() and bool((group_by < 0).any()):
            raise ValueError("group_by values must be non-negative")

    @staticmethod
    def from_tensor(group_by: torch.Tensor, num_documents: int, device: torch.device | str,
                    max_per_group: int = 1) -> "Groups":
        """The device form of a user's group map: any non-negative integers, not necessarily dense or sorted."""
        Groups.check(group_by, num_documents)
        Groups.check_max_per_group(max_per_group, group_by)
        uniq, inverse = torch.unique(group_by.to(device), return_inverse=True)
        return Groups(inverse.to(torch.int32).contiguous(), max(int(uniq.numel()), 1), max_per_group)

    @staticmethod
    def for_shard(group_by: torch.Tensor, doc_id_base: int, num_documents: int, device: torch.device | str,
                  max_per_group: int = 1) -> "Groups":
        """The device form of a group map of the WHOLE document-sharded index for the shard holding global ids
        [doc_id_base, doc_id_base + num_documents): its slice renumbered densely (`ids`) and the whole map renumbered
        densely (`global_ids`, the same on every rank that passes the same map)."""
        if not isinstance(group_by, torch.Tensor) or group_by.dim() != 1 or group_by.shape[0] < doc_id_base + num_documents:
            raise ValueError(f"group_by must cover the whole index, at least the shard's documents "
                             f"[{doc_id_base}, {doc_id_base + num_documents})")
        Groups.check(group_by, group_by.shape[0])
        Groups.check_max_per_group(max_per_group, group_by)
        whole = group_by.to(device)
        local = Groups.from_tensor(whole[doc_id_base : doc_id_base + num_documents], num_documents, device,
                                   max_per_group)
        local.global_ids = torch.unique(whole, return_inverse=True)[1].to(torch.int32).contiguous()
        return local


@dataclasses.dataclass
class ScoreBias:
    """A per-document score bias in its device form: `values` fp32 [num_documents], contiguous, on the index's device
    (fpb_index_with_bias).  Every exact score of document d becomes fp32(score + values[d]), where the score is
    produced, before anything selects on it."""
    values: torch.Tensor

    @staticmethod
    def check(score_bias, num_documents: int | None) -> None:
        """Refuses a bias that is not a 1-D floating-point tensor of `num_documents` finite values (num_documents=None:
        any length)."""
        if not isinstance(score_bias, torch.Tensor):
            raise ValueError(f"score_bias must be a 1-D floating-point tensor, got {type(score_bias).__name__}")
        if not score_bias.dtype.is_floating_point:  # bool, integer and complex dtypes are not
            raise ValueError(f"score_bias must hold floating-point values, got {score_bias.dtype}")
        if score_bias.dim() != 1:
            raise ValueError(f"score_bias must be 1-D (one value per document), got shape {list(score_bias.shape)}")
        if num_documents is not None and score_bias.shape[0] != num_documents:
            raise ValueError(f"score_bias has {score_bias.shape[0]} entries, the index has {num_documents} documents")
        if score_bias.numel() and not bool(torch.isfinite(score_bias.to(torch.float32)).all()):
            raise ValueError("score_bias values must be finite (no NaN or infinity, also after the cast to fp32)")

    @staticmethod
    def from_tensor(score_bias: torch.Tensor, num_documents: int, device: torch.device | str) -> "ScoreBias":
        """The device form of a user's bias: any floating-point dtype on any device, converted to fp32."""
        ScoreBias.check(score_bias, num_documents)
        return ScoreBias(score_bias.to(device=device, dtype=torch.float32).contiguous())

    @staticmethod
    def for_shard(score_bias: torch.Tensor, doc_id_base: int, num_documents: int,
                  device: torch.device | str) -> "ScoreBias":
        """The device form of a bias of the WHOLE document-sharded index for the shard holding global ids
        [doc_id_base, doc_id_base + num_documents): its slice.  The whole tensor is checked first, so that every rank
        passing the same tensor refuses it alike."""
        if not isinstance(score_bias, torch.Tensor) or score_bias.dim() != 1 \
                or score_bias.shape[0] < doc_id_base + num_documents:
            raise ValueError(f"score_bias must cover the whole index, at least the shard's documents "
                             f"[{doc_id_base}, {doc_id_base + num_documents})")
        ScoreBias.check(score_bias, score_bias.shape[0])
        return ScoreBias.from_tensor(score_bias[doc_id_base : doc_id_base + num_documents], num_documents, device)


def _popcount(x: torch.Tensor) -> torch.Tensor:
    """Set bits of every element of a non-negative int64 tensor holding 32-bit words."""
    x = x - ((x >> 1) & 0x55555555)
    x = (x & 0x33333333) + ((x >> 2) & 0x33333333)
    x = (x + (x >> 4)) & 0x0F0F0F0F
    return (x * 0x01010101 & 0xFFFFFFFF) >> 24


def _require_cuda() -> None:
    if not torch.cuda.is_available():
        raise EngineUnavailableError(
            "fast_plaid_b200 needs a CUDA device (H100, sm_90a); there is no CPU search path."
        )


def check_supported(dim: int, nbits: int) -> None:
    """The engine's compiled limits (csrc/index.cu fpb_index_create): raise before an index is written."""
    if int(nbits) not in (1, 2, 4):
        raise ValueError(f"unsupported nbits={nbits}: the engine supports nbits 2 and 4 at dim 64 and 128, "
                         "and nbits 1 at dim 128")
    if int(dim) not in (64, 128):
        raise ValueError(f"unsupported embedding dim={dim}: the engine supports dim 64 and 128")
    if int(nbits) == 1 and int(dim) != 128:
        raise ValueError(f"unsupported embedding dim={dim} with nbits=1: the engine supports nbits 1 at dim 128 only")


def _ptr(t: torch.Tensor | None) -> int | None:
    return None if t is None else t.data_ptr()


@dataclasses.dataclass
class IndexTensors:
    """The immutable tensors of one index (or one document shard), any device.

    Mirrors what ``construct_index`` receives (rust/search/load.rs:122-186).  ``doc_codes``
    may be int64 (on-disk dtype) or int32; ``ivf`` likewise.
    """

    nbits: int
    centroids: torch.Tensor  # [K, D] float
    bucket_weights: torch.Tensor  # [2**nbits]
    doc_lengths: torch.Tensor  # [N] int
    doc_codes: torch.Tensor  # [E] int
    doc_residuals: torch.Tensor  # [E, D*nbits/8] uint8
    ivf: torch.Tensor | None  # [n_ivf] int (doc ids, ascending within a list)
    ivf_lengths: torch.Tensor | None  # [K] int
    avg_residual: torch.Tensor | None = None  # unused at search time (load.rs:146)
    bucket_cutoffs: torch.Tensor | None = None  # unused at search time (load.rs:148)
    # the GrowableArrays whose buffers hold doc_codes / doc_residuals from their start (the loader's fast path):
    # DeviceIndex then adopts them, so that an append grows them in place
    growable: Any = None

    @property
    def num_documents(self) -> int:
        return int(self.doc_lengths.shape[0])

    @property
    def dim(self) -> int:
        return int(self.centroids.shape[1])


def encode_tokens(tokens: torch.Tensor, centroids: torch.Tensor, cutoffs: torch.Tensor,
                  nbits: int) -> tuple[torch.Tensor, torch.Tensor]:
    """Index-build encode step on the GPU (fpb_encode; create.rs:404-428): fp16 CUDA tokens [n, 128],
    fp16 centroids [K, 128], f32 cutoffs -> (codes int32 [n], packed residuals u8 [n, 128*nbits/8])."""
    _require_cuda()
    lib = load_library()
    dev = tokens.device
    tokens = tokens.to(torch.float16).contiguous()
    centroids = centroids.to(dev, torch.float16).contiguous()
    cutoffs = cutoffs.to(dev, torch.float32).contiguous()
    n, dim = tokens.shape
    codes = torch.empty((n,), dtype=torch.int32, device=dev)
    res = torch.empty((n, dim * nbits // 8), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _check(lib.fpb_encode(dev.index, int(nbits), int(dim), int(centroids.shape[0]), centroids.data_ptr(),
                              tokens.data_ptr(), n, cutoffs.data_ptr(), codes.data_ptr(), res.data_ptr(),
                              torch.cuda.current_stream(dev).cuda_stream))
    return codes, res


def kmeans_assign(points: torch.Tensor, centroids: torch.Tensor) -> torch.Tensor:
    """Nearest centroid (squared distance) of every fp16 CUDA point [n, 128]: int32 [n] (fpb_kmeans_assign)."""
    _require_cuda()
    lib = load_library()
    dev = points.device
    points = points.to(torch.float16).contiguous()
    centroids = centroids.to(dev, torch.float16).contiguous()
    bias = (-0.5 * (centroids.float() ** 2).sum(1)).contiguous()
    out = torch.empty((points.shape[0],), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _check(lib.fpb_kmeans_assign(dev.index, int(points.shape[1]), int(centroids.shape[0]), centroids.data_ptr(),
                                     bias.data_ptr(), points.data_ptr(), int(points.shape[0]), out.data_ptr(),
                                     torch.cuda.current_stream(dev).cuda_stream))
    return out


def kmeans_update(points: torch.Tensor, assign: torch.Tensor, centroids: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """In-place mean update of `centroids` (fp16 CUDA [K, 128]) from the assignment; returns (counts int64 [K],
    shift f32 [K] = |new - old| of the non-empty clusters, 0 elsewhere).  Deterministic: the points of a cluster
    are summed in index order (fpb_kmeans_update)."""
    _require_cuda()
    lib = load_library()
    dev = points.device
    K = int(centroids.shape[0])
    order = torch.argsort(assign.to(torch.int64), stable=True)
    counts = torch.bincount(assign.to(torch.int64), minlength=K)
    seg = torch.zeros(K + 1, dtype=torch.int64, device=dev)
    seg[1:] = counts.cumsum(0)
    shift = torch.zeros(K, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _check(lib.fpb_kmeans_update(dev.index, int(points.shape[1]), K, points.data_ptr(), order.data_ptr(),
                                     seg.data_ptr(), centroids.data_ptr(), shift.data_ptr(),
                                     torch.cuda.current_stream(dev).cuda_stream))
    return counts, shift


def shard_tensors(data: IndexTensors, rank: int, world: int) -> tuple[IndexTensors, int]:
    """Contiguous document-range shard ``rank`` of ``world`` (SURVEY.md 8e).

    Centroids and bucket weights are replicated; codes/residual rows are a contiguous slice;
    the IVF is rebuilt for the local id range (lists stay ascending because the global lists
    are ascending, create.rs:118-124).  Returns (shard, doc_id_base).
    """
    n = data.num_documents
    lo = (n * rank) // world
    hi = (n * (rank + 1)) // world
    lens = data.doc_lengths.to(torch.int64).cpu()
    offs = torch.cat([torch.zeros(1, dtype=torch.int64), lens.cumsum(0)])
    t0, t1 = int(offs[lo]), int(offs[hi])
    ivf = ivf_lengths = None
    if data.ivf is not None:
        g_ivf = data.ivf.to(torch.int64).cpu()
        g_len = data.ivf_lengths.to(torch.int64).cpu()
        cell_of = torch.repeat_interleave(torch.arange(g_len.shape[0], dtype=torch.int64), g_len)
        keep = (g_ivf >= lo) & (g_ivf < hi)
        ivf = (g_ivf[keep] - lo).to(torch.int32)
        ivf_lengths = torch.bincount(cell_of[keep], minlength=g_len.shape[0]).to(torch.int64)
    shard = IndexTensors(
        nbits=data.nbits,
        centroids=data.centroids,
        bucket_weights=data.bucket_weights,
        doc_lengths=lens[lo:hi],
        doc_codes=data.doc_codes[t0:t1],
        doc_residuals=data.doc_residuals[t0:t1],
        ivf=ivf,
        ivf_lengths=ivf_lengths,
    )
    return shard, lo


# Host -> device upload of the big index arrays (SURVEY 8(f)-2, the loader fast path; the reference goes
# through pageable `.to(device)` copies after materialising int64 codes, load.py:35-322).  Arrays above
# UPLOAD_DIRECT_BYTES are streamed through two pinned staging buffers: the CPU pass that narrows the
# dtype (int64 codes -> int32) writes straight into pinned memory while the previous chunk's DMA runs.
UPLOAD_DIRECT_BYTES = 256 << 20
UPLOAD_CHUNK_BYTES = 64 << 20


def upload_narrow(src: torch.Tensor, device: torch.device, dtype: torch.dtype,
                  out: torch.Tensor | None = None) -> torch.Tensor:
    """src (host, any integer/float dtype, contiguous in dim 0) -> device tensor of `dtype` (`out`, a device tensor
    of the same shape, or a new one).  `src` may be a view of a memory-mapped .npy file: the staging pass is then
    also the disk read."""
    src = src if src.is_contiguous() else src.contiguous()
    out_bytes = src.numel() * torch.empty((), dtype=dtype).element_size()
    if src.device.type != "cpu" or out_bytes <= UPLOAD_DIRECT_BYTES or src.dim() == 0 or src.shape[0] == 0:
        if out is None:
            return src.to(device, dtype).contiguous()
        out.copy_(src.to(dtype) if src.device.type == "cpu" else src)
        return out
    if out is None:
        out = torch.empty(src.shape, dtype=dtype, device=device)
    row_bytes = max(1, out_bytes // src.shape[0])
    rows = max(1, UPLOAD_CHUNK_BYTES // row_bytes)
    stage = [torch.empty((rows,) + tuple(src.shape[1:]), dtype=dtype).pin_memory() for _ in range(2)]
    done = [torch.cuda.Event(), torch.cuda.Event()]
    copy_stream = torch.cuda.Stream(device=device)
    with torch.cuda.stream(copy_stream):
        for i, r0 in enumerate(range(0, src.shape[0], rows)):
            r1 = min(src.shape[0], r0 + rows)
            slot = i & 1
            if i >= 2:
                done[slot].synchronize()  # the DMA that last read this staging buffer has finished
            stage[slot][: r1 - r0].copy_(src[r0:r1])  # dtype narrowing + copy into pinned memory, one pass
            out[r0:r1].copy_(stage[slot][: r1 - r0], non_blocking=True)
            done[slot].record(copy_stream)
    copy_stream.synchronize()
    return out


FPB_COMM_ID_BYTES = 128


class ShardComm:
    """One NCCL communicator created below the C ABI (fpb_comm_*), used by the document-sharded search.

    `ShardComm.from_process_group(device)` bootstraps it from an initialised torch.distributed group: rank 0
    makes the id, the 128 bytes travel through the group's own broadcast (any backend), every rank joins.
    `n_query_groups` x (world / n_query_groups) document shards is the search grid (csrc/comm.cu)."""

    def __init__(self, nranks: int, rank: int, unique_id: bytes, device: torch.device | str) -> None:
        _require_cuda()
        self._lib = load_library()
        self.device = torch.device(device)
        self.nranks, self.rank = int(nranks), int(rank)
        if len(unique_id) != FPB_COMM_ID_BYTES:
            raise ValueError("unique_id must be FPB_COMM_ID_BYTES bytes")
        buf = ctypes.create_string_buffer(bytes(unique_id), FPB_COMM_ID_BYTES)
        handle = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _check(self._lib.fpb_comm_create(ctypes.byref(handle), self.nranks, self.rank, buf, self.device.index))
        self._handle = handle

    @staticmethod
    def new_unique_id() -> bytes:
        buf = ctypes.create_string_buffer(FPB_COMM_ID_BYTES)
        _check(load_library().fpb_comm_unique_id(buf))
        return buf.raw

    @classmethod
    def from_process_group(cls, device: torch.device | str) -> "ShardComm":
        import torch.distributed as dist

        rank, world = dist.get_rank(), dist.get_world_size()
        box = [cls.new_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        return cls(world, rank, box[0], device)

    def close(self) -> None:
        if getattr(self, "_handle", None) is not None and self._handle.value:
            self._lib.fpb_comm_destroy(self._handle)
            self._handle = ctypes.c_void_p()

    def __del__(self) -> None:  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass


def shard_grid(rank: int, world: int, n_query_groups: int) -> tuple[int, int, int]:
    """(query group, document shard, document shards per group) of `rank` on the n_query_groups x n_shards grid
    of csrc/comm.cu."""
    if n_query_groups < 1 or world % n_query_groups != 0:
        raise ValueError(f"{n_query_groups} query groups do not divide {world} ranks")
    n_shards = world // n_query_groups
    return rank // n_shards, rank % n_shards, n_shards


# The shard merge (and the shard threshold) sorts the n_shards * n_full_scores/4 records of a query in shared memory
# (csrc/k6_rank.cu): at most this many.
MERGE_MAX_RECORDS = 16384


def _check_merge(n_shards: int, R: int, what: str) -> None:
    if n_shards * R > MERGE_MAX_RECORDS:
        raise ValueError(f"{what} over {n_shards} document shards: {n_shards}*{R} records per query exceed the "
                         f"{MERGE_MAX_RECORDS} the shard merge supports")


def check_merge_records(n_shards: int, n_full_scores: int) -> None:
    """Raise ValueError when a document-sharded search over `n_shards` shards cannot merge its records, the rule
    fpb_merge_shards and fpb_search_batch_sharded apply, so that a search is refused before any collective."""
    _check_merge(n_shards, max(int(n_full_scores) // 4, 1), f"n_full_scores={n_full_scores}")


def check_exhaustive_merge_records(n_shards: int, top_k: int) -> None:
    """The same rule for the document-sharded exhaustive search, whose shards send top_k records per query
    (fpb_search_exhaustive_sharded): n_shards * top_k <= MERGE_MAX_RECORDS."""
    _check_merge(n_shards, int(top_k), f"top_k={top_k}")


class GrowableBuffer:
    """One growable device buffer (fpb_buffer_*): address space reserved up to the device's memory, physical memory
    mapped in 2 MB granules as `commit` asks for it.  Its address never changes, so tensors viewing its start stay
    valid while it grows.  The views (`view`) keep this object alive, and it frees the memory when the last of them
    and the last owner are gone."""

    _TYPESTR = {torch.int32: "<i4", torch.int64: "<i8", torch.uint8: "|u1", torch.float16: "<f2"}

    def __init__(self, device: torch.device) -> None:
        self._lib = load_library()
        self.device = torch.device(device)
        handle = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _check(self._lib.fpb_buffer_reserve(ctypes.byref(handle), self.device.index, 0))
        self._handle = handle
        self.ptr = int(self._lib.fpb_buffer_ptr(handle))

    def commit(self, nbytes: int) -> None:
        _check(self._lib.fpb_buffer_commit(self._handle, max(int(nbytes), 1)))

    @property
    def mapped_bytes(self) -> int:
        return int(self._lib.fpb_buffer_mapped_bytes(self._handle))

    def view(self, dtype: torch.dtype, shape: tuple[int, ...]) -> torch.Tensor:
        """A tensor over the buffer's first bytes (committed here first)."""
        n = 1
        for d in shape:
            n *= int(d)
        self.commit(n * torch.empty((), dtype=dtype).element_size())
        return torch.as_tensor(_BufferView(self, shape, self._TYPESTR[dtype]), device=self.device)

    def __del__(self) -> None:  # pragma: no cover
        h = getattr(self, "_handle", None)
        if h is not None and h.value:
            try:
                torch.cuda.synchronize(self.device)  # kernels still reading the buffer
            except Exception:
                pass
            self._lib.fpb_buffer_destroy(h)
            self._handle = ctypes.c_void_p()


class _BufferView:
    """__cuda_array_interface__ of a GrowableBuffer's start; the tensor made from it holds this object, and this
    object holds the buffer."""

    def __init__(self, buf: GrowableBuffer, shape: tuple[int, ...], typestr: str) -> None:
        self.buf = buf
        self.__cuda_array_interface__ = {"shape": tuple(int(d) for d in shape), "typestr": typestr,
                                         "data": (buf.ptr, False), "version": 2}


class GrowableArrays:
    """The per-token arrays of an index (codes, residuals, token norms) and its document offsets in growable
    buffers, shared by a DeviceIndex and every DeviceIndex appended to it.  `n_docs` / `n_tokens` count what has
    been written: only the DeviceIndex that covers all of it may append, so that appends never overwrite rows
    another index uses."""

    def __init__(self, device: torch.device, pd: int) -> None:
        self.device = torch.device(device)
        self.pd = int(pd)
        self.codes = GrowableBuffer(self.device)
        self.residuals = GrowableBuffer(self.device)
        self.norms = GrowableBuffer(self.device)
        self.offsets = GrowableBuffer(self.device)
        self.n_docs = 0
        self.n_tokens = 0
        self.lock = threading.Lock()

    def views(self, n_docs: int, n_tokens: int) -> dict[str, torch.Tensor]:
        """Tensors over the first n_docs + 1 offsets and n_tokens rows (at least one row, as DeviceIndex keeps)."""
        rows = max(int(n_tokens), 1)
        return {"offsets": self.offsets.view(torch.int64, (int(n_docs) + 1,)),
                "codes": self.codes.view(torch.int32, (rows,)),
                "residuals": self.residuals.view(torch.uint8, (rows, self.pd)),
                "norms": self.norms.view(torch.float16, (rows,))}

    @property
    def mapped_bytes(self) -> int:
        return sum(b.mapped_bytes for b in (self.codes, self.residuals, self.norms, self.offsets))


class DeviceIndex:
    """One index (or shard) resident in HBM + its ``fpb_index`` handle."""

    def __init__(self, data: IndexTensors, device: str | torch.device, doc_id_base: int = 0) -> None:
        _require_cuda()
        self._lib = load_library()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise ValueError(f"Unsupported device string: '{device}' (the engine runs on CUDA only)")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        dev = self.device
        self.nbits = int(data.nbits)
        self.dim = data.dim
        self.doc_id_base = int(doc_id_base)
        with torch.cuda.device(dev):
            # codec tensors are cast to fp16 exactly as construct_index does (load.rs:145-152)
            self.centroids = data.centroids.to(dev, torch.float16).contiguous()
            self.bucket_weights = data.bucket_weights.to(dev, torch.float16).contiguous()
            lens = data.doc_lengths.to(torch.int64)
            self.num_documents = int(lens.shape[0])
            self.max_doc_len = int(lens.max()) if self.num_documents > 0 else 0
            offs = torch.zeros(self.num_documents + 1, dtype=torch.int64)
            offs[1:] = lens.cpu().cumsum(0)
            self.num_tokens = int(offs[-1])
            E = self.num_tokens
            # Codes, residuals, norms and offsets go to growable buffers (appends then grow them in place): the
            # loader's, or new ones for host tensors.  Device tensors outside them are used where they are, and the
            # first append copies them (`append`).
            arrays = data.growable
            if arrays is None and data.doc_codes.device.type == "cpu":
                arrays = GrowableArrays(dev, self.dim * self.nbits // 8)
            if arrays is not None:
                v = arrays.views(self.num_documents, E)
                v["offsets"].copy_(offs)
                if data.growable is None and E > 0:
                    # rows past the last document (the reference's tail padding, load.py:298-300) are dropped
                    upload_narrow(data.doc_codes[:E], dev, torch.int32, out=v["codes"][:E])
                    upload_narrow(data.doc_residuals[:E], dev, torch.uint8, out=v["residuals"][:E])
                elif data.growable is not None and data.doc_codes.data_ptr() != arrays.codes.ptr:
                    raise ValueError("IndexTensors.growable must hold doc_codes and doc_residuals from its start")
                if E == 0:
                    v["codes"].zero_()
                    v["residuals"].zero_()
                arrays.n_docs, arrays.n_tokens = self.num_documents, E
                self.doc_offsets, self.doc_codes, self.doc_residuals = v["offsets"], v["codes"], v["residuals"]
            else:
                self.doc_offsets = offs.to(dev)
                self.doc_codes = upload_narrow(data.doc_codes[:E], dev, torch.int32)
                self.doc_residuals = upload_narrow(data.doc_residuals[:E], dev, torch.uint8)
                if self.doc_codes.numel() == 0:
                    self.doc_codes = torch.zeros(1, dtype=torch.int32, device=dev)
                    self.doc_residuals = torch.zeros((1, self.dim * self.nbits // 8), dtype=torch.uint8, device=dev)
            self._arrays = arrays
            self.num_centroids = int(self.centroids.shape[0])
            if data.ivf is not None and data.ivf_lengths is not None:
                il = data.ivf_lengths.to(torch.int64).cpu()
                if il.shape[0] < self.num_centroids:
                    il = torch.cat([il, torch.zeros(self.num_centroids - il.shape[0], dtype=torch.int64)])
                io = torch.zeros(il.shape[0] + 1, dtype=torch.int64)
                io[1:] = il.cumsum(0)
                self.ivf_offsets = io.to(dev)
                self.ivf_pids = upload_narrow(data.ivf, dev, torch.int32)
                if self.ivf_pids.numel() == 0:
                    self.ivf_pids = torch.zeros(1, dtype=torch.int32, device=dev)
                n_ivf = int(io[-1])
            else:
                self.ivf_offsets = None
                self.ivf_pids = None
                n_ivf = 0
            # derived at load: the fp16 norm of every decompressed token (2 B/token), filled by fpb_index_create
            if arrays is not None:
                self.token_norms = v["norms"]
            else:
                self.token_norms = torch.empty(max(self.num_tokens, 1), dtype=torch.float16, device=dev)
            handle = ctypes.c_void_p()
            _check(
                self._lib.fpb_index_create(
                    ctypes.byref(handle), dev.index, self.nbits, self.dim, self.num_centroids,
                    _ptr(self.centroids), _ptr(self.bucket_weights), self.num_documents,
                    _ptr(self.doc_offsets), _ptr(self.doc_codes), _ptr(self.doc_residuals), _ptr(self.token_norms),
                    _ptr(self.ivf_offsets), _ptr(self.ivf_pids), n_ivf, self.max_doc_len, self.doc_id_base,
                )
            )
        self._handle = handle
        self._init_state()

    def _init_state(self) -> None:
        self._ws: dict[tuple, FpbLayout] = {}
        self._buf: torch.Tensor | None = None
        self._io: dict[tuple, dict[str, torch.Tensor]] = {}
        self._lock = threading.Lock()
        # One search at a time per DeviceIndex: the workspace and the staging buffers are shared, and ctypes
        # releases the GIL inside the C-ABI call.  (The fpb_index itself is immutable and thread-safe; callers
        # that want concurrent searches on one GPU give each thread its own workspace through the C ABI.)
        self._search_lock = threading.RLock()
        self._last_stream: torch.cuda.Stream | None = None
        # approximate-stage mode of the host-buffer path (results are identical in both; see _adapt_approx_mode)
        self._approx_direct = False
        self._approx_calls = 0
        self._approx_hold = 0

    @contextlib.contextmanager
    def _exclusive(self):
        with self._search_lock:
            if getattr(self, "_handle", None) is None or not self._handle.value:
                raise RuntimeError("this DeviceIndex has been closed")
            st = torch.cuda.current_stream(self.device)
            if self._last_stream is not None and self._last_stream != st:
                st.wait_stream(self._last_stream)  # the previous call's kernels still own the workspace
            self._last_stream = st
            yield

    @contextlib.contextmanager
    def _grouped(self, groups: Groups):
        """Within the block every search of this index ranks by `groups`: the index's handle is swapped for one that
        carries them (fpb_index_with_groups_max; fpb_index_with_shard_groups when they carry `global_ids`), under the
        search lock, and swapped back after.  groups=None: the block runs on the index's own handle."""
        if groups is None:
            yield
            return
        gl = groups.global_ids
        for t, n in ((groups.ids, self.num_documents), (gl, None)):
            if t is not None and (t.device != self.device or t.dtype != torch.int32 or t.dim() != 1
                                  or (n is not None and t.shape[0] != n) or not t.is_contiguous()):
                raise ValueError(f"expected contiguous group ids int32 [{n if n is not None else 'n_total'}] on "
                                 f"{self.device}, got {t.dtype} {list(t.shape)} on {t.device}")
        with self._search_lock:
            if getattr(self, "_handle", None) is None or not self._handle.value:
                raise RuntimeError("this DeviceIndex has been closed")
            handle = ctypes.c_void_p()
            if gl is None:
                _check(self._lib.fpb_index_with_groups_max(ctypes.byref(handle), self._handle, groups.ids.data_ptr(),
                                                           groups.n_groups, groups.max_per_group))
            else:
                _check(self._lib.fpb_index_with_shard_groups(ctypes.byref(handle), self._handle, groups.ids.data_ptr(),
                                                             groups.n_groups, groups.max_per_group, gl.data_ptr(),
                                                             gl.shape[0]))
            own, self._handle = self._handle, handle
            try:
                yield
            finally:
                self._handle = own
                self._lib.fpb_index_destroy(handle)
                self._groups_keepalive = self._stream_keep(groups.ids, gl)  # until the stream has consumed them

    @contextlib.contextmanager
    def _biased(self, bias: ScoreBias | None):
        """Within the block every exact score of this index is biased by `bias`: the handle is swapped for one that
        carries it (fpb_index_with_bias), under the search lock, and swapped back after.  Inside `_grouped` the
        biased handle keeps the groups (and the other way round).  bias=None: the block runs on the current handle."""
        if bias is None:
            yield
            return
        v = bias.values
        if (v.device != self.device or v.dtype != torch.float32 or v.dim() != 1 or v.shape[0] != self.num_documents
                or not v.is_contiguous()):
            raise ValueError(f"expected a contiguous score bias float32 [{self.num_documents}] on {self.device}, got "
                             f"{v.dtype} {list(v.shape)} on {v.device}")
        with self._search_lock:
            if getattr(self, "_handle", None) is None or not self._handle.value:
                raise RuntimeError("this DeviceIndex has been closed")
            handle = ctypes.c_void_p()
            _check(self._lib.fpb_index_with_bias(ctypes.byref(handle), self._handle, v.data_ptr(), v.shape[0]))
            own, self._handle = self._handle, handle
            try:
                yield
            finally:
                self._handle = own
                self._lib.fpb_index_destroy(handle)
                self._bias_keepalive = self._stream_keep(v)  # until the stream has consumed it

    @contextlib.contextmanager
    def _ranked(self, groups: Groups | None, bias: ScoreBias | None):
        """`_grouped` and `_biased` together: the block runs on a handle carrying both."""
        with self._grouped(groups), self._biased(bias):
            yield

    # -- lifetime ------------------------------------------------------------------------
    def close(self) -> None:
        lock = getattr(self, "_search_lock", None)
        with (lock if lock is not None else contextlib.nullcontext()):  # wait for a search in flight
            if getattr(self, "_handle", None) is not None and self._handle.value:
                try:
                    torch.cuda.synchronize(self.device)  # kernels still reading the index tensors
                except Exception:
                    pass
                self._lib.fpb_index_destroy(self._handle)
                self._handle = ctypes.c_void_p()
            self._ws = {}
            self._buf = None
            self._io = {}

    def __del__(self) -> None:  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    @property
    def has_ivf(self) -> bool:
        return self.ivf_offsets is not None

    @property
    def walk_group(self) -> int:
        """Windows per group of the approximate stage's bound pass, chosen from the walk layout (fpb_index_walk_group)."""
        return int(self._lib.fpb_index_walk_group(self._handle))

    @property
    def growable(self) -> "GrowableArrays | None":
        """The growable buffers this index's arrays live in (None until the first append for an index built from
        device tensors)."""
        return self._arrays

    # -- growth --------------------------------------------------------------------------
    def _copy_to_growable(self) -> GrowableArrays:
        """The one copy of an index built from device tensors: its arrays in new growable buffers."""
        N, E = self.num_documents, self.num_tokens
        arrays = GrowableArrays(self.device, self.dim * self.nbits // 8)
        v = arrays.views(N, E)
        v["offsets"].copy_(self.doc_offsets)
        for name, t in (("codes", self.doc_codes), ("residuals", self.doc_residuals), ("norms", self.token_norms)):
            v[name][:E].copy_(t[:E])
        arrays.n_docs, arrays.n_tokens = N, E
        return arrays

    @torch.inference_mode()
    def append(self, codes: torch.Tensor, residuals: torch.Tensor, doc_lengths: torch.Tensor) -> "DeviceIndex":
        """A new DeviceIndex over this index's documents followed by new ones, given by their codes [n_tokens],
        packed residuals [n_tokens, dim*nbits/8] and lengths [n_docs] (any device).  It shares this index's memory:
        the new rows are written after the old ones in the growable buffers, the token norms and the approximate
        stage's walk layout are computed for the new tokens and documents only (fpb_index_append), and the inverted
        file is merged on the device into a new array (fpb_ivf_append), the one copy of existing data an append
        makes (4 bytes per posting).  The result equals a DeviceIndex built from scratch over all the documents.

        This index stays valid and searchable, and its results do not change.  Only the newest index of a chain of
        appends may be appended to.  An index whose arrays are not in growable buffers (built from device tensors,
        as ``FastPlaid.from_tensors`` and ``bench.py`` do) first copies its codes, residuals, norms and offsets into
        them, once: that first append briefly holds those arrays twice."""
        dev = self.device
        lens = doc_lengths.to(torch.int64).cpu().reshape(-1)
        n_new, e_new = int(lens.shape[0]), int(lens.sum())
        pd = self.dim * self.nbits // 8
        codes = codes.reshape(-1)
        if bool((lens < 0).any()) or codes.shape[0] != e_new or tuple(residuals.shape) != (e_new, pd):
            raise ValueError(f"append: {n_new} documents of {e_new} tokens need codes [{e_new}] and residuals "
                             f"[{e_new}, {pd}], got {tuple(codes.shape)} and {tuple(residuals.shape)}")
        N, E = self.num_documents, self.num_tokens
        N1, E1 = N + n_new, E + e_new
        with torch.cuda.device(dev):
            if getattr(self, "_handle", None) is None or not self._handle.value:
                raise RuntimeError("this DeviceIndex has been closed")
            with self._lock:
                arrays = self._arrays
                if arrays is None:
                    arrays = self._arrays = self._copy_to_growable()
            with arrays.lock:  # appends to one chain, one at a time
                if arrays.n_docs != N or arrays.n_tokens != E:
                    raise ValueError(f"append: this index of {N} documents is not the newest of its chain "
                                     f"({arrays.n_docs} documents are laid out); append to the newest one")
                v = arrays.views(N1, E1)
                if e_new > 0:
                    v["codes"][E:E1].copy_(codes.to(dev, torch.int32))
                    v["residuals"][E:E1].copy_(residuals.to(dev, torch.uint8))
                new_offs = torch.zeros(n_new + 1, dtype=torch.int64)
                new_offs[1:] = lens.cumsum(0)
                v["offsets"][N + 1 :].copy_(new_offs[1:] + E)
                ivf_offsets = ivf_pids = None
                n_ivf = ctypes.c_int64(0)
                st = self._stream()
                if self.has_ivf:
                    n_cells = int(self.ivf_offsets.shape[0]) - 1
                    ivf_offsets = torch.empty(n_cells + 1, dtype=torch.int64, device=dev)
                    local = new_offs.to(dev)
                    new_codes = v["codes"].data_ptr() + 4 * E
                    args = (dev.index, n_cells, self.ivf_offsets.data_ptr(), self.ivf_pids.data_ptr(), N, n_new,
                            local.data_ptr(), new_codes, ivf_offsets.data_ptr())
                    _check(self._lib.fpb_ivf_append(*args, None, 0, ctypes.byref(n_ivf), st))  # sizes the output
                    ivf_pids = torch.zeros(max(n_ivf.value, 1), dtype=torch.int32, device=dev)
                    _check(self._lib.fpb_ivf_append(*args, ivf_pids.data_ptr(), ivf_pids.numel(), ctypes.byref(n_ivf), st))
                torch.cuda.current_stream(dev).synchronize()  # fpb_index_append works on the legacy default stream
                max_len = max(self.max_doc_len, int(lens.max()) if n_new > 0 else 0)
                handle = ctypes.c_void_p()
                _check(self._lib.fpb_index_append(
                    ctypes.byref(handle), self._handle, N1, E1, v["offsets"].data_ptr(), v["codes"].data_ptr(),
                    v["residuals"].data_ptr(), v["norms"].data_ptr(), _ptr(ivf_offsets), _ptr(ivf_pids), n_ivf.value,
                    max_len))
                arrays.n_docs, arrays.n_tokens = N1, E1
        return self._successor(arrays, v, N1, E1, max_len, ivf_offsets, ivf_pids, handle)

    def _successor(self, arrays: GrowableArrays, v: dict, n_docs: int, n_tokens: int, max_len: int,
                   ivf_offsets: torch.Tensor | None, ivf_pids: torch.Tensor | None, handle) -> "DeviceIndex":
        """A DeviceIndex with this one's codec over the arrays `v` of `arrays` and the fpb_index `handle`."""
        new = DeviceIndex.__new__(DeviceIndex)
        for name in ("_lib", "device", "nbits", "dim", "doc_id_base", "centroids", "bucket_weights", "num_centroids"):
            setattr(new, name, getattr(self, name))
        new.num_documents, new.num_tokens, new.max_doc_len = n_docs, n_tokens, max_len
        new.doc_offsets, new.doc_codes, new.doc_residuals, new.token_norms = (
            v["offsets"], v["codes"], v["residuals"], v["norms"])
        new.ivf_offsets, new.ivf_pids = ivf_offsets, ivf_pids
        new._arrays = arrays
        new._handle = handle
        new._init_state()
        return new

    @torch.inference_mode()
    def delete(self, doc_ids) -> "DeviceIndex":
        """A new DeviceIndex over this index's documents without `doc_ids` (this index's ids; duplicates, negative
        ids and ids >= num_documents are ignored), the rest renumbered in order, as ``delete_from_index`` leaves a
        directory.  The kept documents' offsets and rows are compacted on the device into new growable buffers
        (fpb_docs_compact), so the result can be appended to, and the inverted file of the kept documents is built
        from this one's (fpb_ivf_delete); fpb_index_create then derives the token norms and the walk layout.  The
        result equals a DeviceIndex loaded from the directory after the delete.

        Nothing this index reads is written: it stays valid and searchable, and its results do not change.  Until it
        is released both copies of the kept data are in memory.  A document shard (doc_id_base != 0) is refused."""
        if self.doc_id_base != 0:
            raise ValueError("delete: a document shard cannot delete in place (its range moves when the index "
                             "shrinks); load the directory again instead")
        dev, N = self.device, self.num_documents
        ids = torch.as_tensor(list(doc_ids) if not isinstance(doc_ids, torch.Tensor) else doc_ids,
                              dtype=torch.int64).reshape(-1).cpu()
        drop = torch.unique(ids[(ids >= 0) & (ids < N)])  # sorted
        n_drop, n_keep = int(drop.shape[0]), N - int(drop.shape[0])
        pd = self.dim * self.nbits // 8
        with torch.cuda.device(dev):
            if getattr(self, "_handle", None) is None or not self._handle.value:
                raise RuntimeError("this DeviceIndex has been closed")
            d_drop = drop.to(dev, torch.int32) if n_drop else None
            st = self._stream()
            arrays = GrowableArrays(dev, pd)
            offsets = arrays.offsets.view(torch.int64, (n_keep + 1,))
            n_tok = ctypes.c_int64(0)
            args = (dev.index, N, self.doc_offsets.data_ptr(), self.doc_codes.data_ptr(),
                    self.doc_residuals.data_ptr(), None, pd, _ptr(d_drop), n_drop, offsets.data_ptr())
            _check(self._lib.fpb_docs_compact(*args, None, None, None, 0, ctypes.byref(n_tok), st))  # sizes the rows
            E1 = n_tok.value
            v = arrays.views(n_keep, E1)
            if E1 > 0:
                _check(self._lib.fpb_docs_compact(*args, v["codes"].data_ptr(), v["residuals"].data_ptr(), None, E1,
                                                  ctypes.byref(n_tok), st))
            else:
                v["codes"].zero_()
                v["residuals"].zero_()
            ivf_offsets = ivf_pids = None
            n_ivf = ctypes.c_int64(0)
            if self.has_ivf:
                n_cells = int(self.ivf_offsets.shape[0]) - 1
                ivf_offsets = torch.empty(n_cells + 1, dtype=torch.int64, device=dev)
                args = (dev.index, n_cells, self.ivf_offsets.data_ptr(), self.ivf_pids.data_ptr(), N, _ptr(d_drop),
                        n_drop, ivf_offsets.data_ptr())
                _check(self._lib.fpb_ivf_delete(*args, None, 0, ctypes.byref(n_ivf), st))  # sizes the output
                ivf_pids = torch.zeros(max(n_ivf.value, 1), dtype=torch.int32, device=dev)
                _check(self._lib.fpb_ivf_delete(*args, ivf_pids.data_ptr(), ivf_pids.numel(), ctypes.byref(n_ivf), st))
            max_len = int((v["offsets"][1:] - v["offsets"][:-1]).max()) if n_keep > 0 else 0
            torch.cuda.current_stream(dev).synchronize()  # fpb_index_create works on the legacy default stream
            handle = ctypes.c_void_p()
            _check(self._lib.fpb_index_create(
                ctypes.byref(handle), dev.index, self.nbits, self.dim, self.num_centroids, _ptr(self.centroids),
                _ptr(self.bucket_weights), n_keep, v["offsets"].data_ptr(), v["codes"].data_ptr(),
                v["residuals"].data_ptr(), v["norms"].data_ptr(), _ptr(ivf_offsets), _ptr(ivf_pids), n_ivf.value,
                max_len, 0))
            arrays.n_docs, arrays.n_tokens = n_keep, E1
        return self._successor(arrays, v, n_keep, E1, max_len, ivf_offsets, ivf_pids, handle)

    # -- helpers -------------------------------------------------------------------------
    @staticmethod
    def make_params(top_k: int, n_full_scores: int, n_ivf_probe: int, batch_size: int = 2000,
                    flags: int = 0) -> FpbParams:
        return FpbParams(int(n_ivf_probe), int(n_full_scores), int(top_k), int(batch_size), int(flags))

    @staticmethod
    def with_flags(params: FpbParams, flags: int) -> FpbParams:
        return FpbParams(params.n_ivf_probe, params.n_full_scores, params.top_k, params.batch_size,
                         params.flags | int(flags))

    def layout(self, B: int, Q: int, params: FpbParams) -> FpbLayout:
        lay = FpbLayout()
        _check(self._lib.fpb_workspace_layout(self._handle, B, Q, ctypes.byref(params), ctypes.byref(lay)))
        return lay

    def workspace(self, B: int, Q: int, params: FpbParams) -> tuple[torch.Tensor, FpbLayout]:
        """One grow-only device buffer per index, carved up by fpb_workspace_layout."""
        key = (B, Q, params.n_ivf_probe, params.n_full_scores, params.top_k, params.flags)
        with self._lock:
            lay = self._ws.get(key)
            if lay is None:
                lay = self.layout(B, Q, params)
                if len(self._ws) > 64:
                    self._ws.clear()
                self._ws[key] = lay
        return self._buffer(int(lay.total_bytes)), lay

    def _buffer(self, nbytes: int) -> torch.Tensor:
        """The grow-only device buffer that `workspace` and the exhaustive search carve up (callers hold _exclusive)."""
        with self._lock:
            if self._buf is None or self._buf.numel() < nbytes:
                self._drop(self._buf)
                self._buf = None  # free the old buffer before allocating the larger one
                self._buf = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            return self._buf

    def _drop(self, cached: torch.Tensor | None) -> None:
        """Before a cached buffer is dropped: the caching allocator gives a freed block back to the stream it was
        allocated on, at once, and that stream is not ordered after the calls that used it since.  Marking it used by
        the current and the previous call's stream (each call waits for the one before, _exclusive) holds the block
        back until they are done with it."""
        if cached is not None:
            for st in {torch.cuda.current_stream(self.device), self._last_stream} - {None}:
                cached.record_stream(st)

    def _stream_keep(self, *tensors: torch.Tensor | None) -> tuple:
        """Tensors the caller owns that the call just queued reads: marked used by the current stream, so that the
        allocator does not hand out their memory before the stream has read it when the caller frees them.  Returns
        them, for the `_keepalive` attributes that hold them until the next call."""
        st = torch.cuda.current_stream(self.device)
        for t in tensors:
            if t is not None:
                t.record_stream(st)
        return tensors

    def max_queries_per_call(self, Q: int, params: FpbParams, budget_bytes: int = 6 << 30) -> int:
        key = ("maxq", Q, params.n_ivf_probe, params.n_full_scores, params.top_k, params.flags, budget_bytes)
        hit = self._ws.get(key)
        if hit is not None:
            return hit
        val = self._max_queries_per_call(Q, params, budget_bytes)
        self._ws[key] = val
        return val

    def _max_queries_per_call(self, Q: int, params: FpbParams, budget_bytes: int) -> int:
        one = self.layout(1, Q, params).total_bytes
        two = self.layout(2, Q, params).total_bytes
        per_q = max(1, two - one)
        return max(1, int((budget_bytes - one) // per_q) + 1)

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    # -- search --------------------------------------------------------------------------
    def _subset_csr(self, subset: list[list[int]], s: int, e: int) -> tuple[torch.Tensor, torch.Tensor, int]:
        lens = [len(x) for x in subset[s:e]]
        offs = torch.zeros(len(lens) + 1, dtype=torch.int64)
        offs[1:] = torch.tensor(lens, dtype=torch.int64).cumsum(0)
        flat = [i for x in subset[s:e] for i in x]
        ids = torch.tensor(flat if flat else [0], dtype=torch.int64)
        ids = ids.clamp(-1, 2**31 - 1).to(torch.int32)
        return ids.to(self.device), offs.to(self.device), (max(lens) if lens else 0)

    def _check_filter(self, filter: Filter, B: int) -> None:
        if len(filter.query_filter) != B:
            raise ValueError("Subset length must match number of queries.")
        bad = [(b, f) for b, f in enumerate(filter.query_filter) if not 0 <= f < filter.n_filters]
        if bad:
            raise ValueError(f"query_filter[{bad[0][0]}]={bad[0][1]} is not in [0, n_filters={filter.n_filters})")
        bm = filter.bitmap
        if (bm.device != self.device or bm.dtype != torch.int32 or bm.dim() != 2 or not bm.is_contiguous()
                or filter.n_bits < 0 or bm.shape[1] < (filter.n_bits + 31) // 32):
            raise ValueError(f"expected contiguous filter bitmaps int32 [n_filters, >= ceil(n_bits / 32)] with "
                             f"n_bits={filter.n_bits} on {self.device}, got {bm.dtype} {list(bm.shape)} on "
                             f"{bm.device}{'' if bm.is_contiguous() else ' (not contiguous)'}")

    def filter_counts(self, filter: Filter) -> torch.Tensor:
        """int64 [n_filters] on this device: the documents of each filter inside this index's range of global ids."""
        lo, hi = self.doc_id_base, min(self.doc_id_base + self.num_documents, filter.n_bits)
        if hi <= lo:
            return torch.zeros(filter.n_filters, dtype=torch.int64, device=self.device)
        w0, w1 = lo >> 5, (hi + 31) >> 5
        words = filter.bitmap[:, w0:w1].to(torch.int64) & 0xFFFFFFFF
        keep = torch.full((w1 - w0,), 0xFFFFFFFF, dtype=torch.int64, device=self.device)
        keep[0] &= (0xFFFFFFFF << (lo & 31)) & 0xFFFFFFFF
        if hi & 31:
            keep[-1] &= (1 << (hi & 31)) - 1
        return _popcount(words & keep).sum(1)

    def search(
        self, queries: torch.Tensor, params: FpbParams, subset: list[list[int]] | None = None,
        filter: Filter | None = None, groups: Groups | None = None, bias: ScoreBias | None = None,
    ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """queries: fp16 [B, Q, D] on this device.  Returns device tensors
        (ids int64 [B, top_k], scores f32 [B, top_k], counts int32 [B]).  Asynchronous, except with `subset` lists,
        whose copy from host memory (`_subset_csr`) waits for the stream.
        `subset`: per query a list of GLOBAL doc ids to restrict the search to
        (search.rs:494-517, :544-547).  `filter`: the same restriction in device form (fpb_search_batch_filter);
        for the same documents the result is the same bytes.  `groups`: at most groups.max_per_group documents per
        group among the n_full_scores / 4 re-ranked ones, each group's best ones (fpb_index_with_groups_max).
        `bias`: the re-ranked documents' exact scores biased before the ranking (fpb_index_with_bias)."""
        if groups is not None or bias is not None:
            with self._ranked(groups, bias):
                return self.search(queries, params, subset, filter)
        queries = self._check_queries(queries)
        B, Q, _ = queries.shape
        k = params.top_k
        ids = torch.empty((B, k), dtype=torch.int64, device=self.device)
        scores = torch.empty((B, k), dtype=torch.float32, device=self.device)
        counts = torch.empty((B,), dtype=torch.int32, device=self.device)
        if B == 0:
            return ids, scores, counts
        if subset is not None:
            if len(subset) != B:
                raise ValueError("Subset length must match number of queries.")
            params = self.with_flags(params, FPB_FLAG_SUBSET)
        if filter is not None:
            self._check_filter(filter, B)
            params = self.with_flags(params, FPB_FLAG_SUBSET)
        step = self.max_queries_per_call(Q, params)
        if filter is not None:
            step = min(step, 65535)  # the library's limit on filters per call
        keep = []
        with self._exclusive(), torch.cuda.device(self.device):
            for s in range(0, B, step):
                e = min(B, s + step)
                buf, lay = self.workspace(e - s, Q, params)
                if filter is not None:
                    # each call passes the filters of its own queries: at most e - s of them
                    rows, local = filter.call_rows(s, e)
                    keep.append(rows)
                    h_map = (ctypes.c_int32 * (e - s))(*local)
                    _check(
                        self._lib.fpb_search_batch_filter(
                            self._handle, queries[s:e].data_ptr(), e - s, Q, ctypes.byref(params),
                            rows.data_ptr(), rows.shape[0], filter.n_bits, h_map, buf.data_ptr(),
                            buf.numel(), ids[s:e].data_ptr(), scores[s:e].data_ptr(), counts[s:e].data_ptr(),
                            self._stream(),
                        )
                    )
                    self._keepalive = self._stream_keep(*keep)  # until the stream has consumed them
                elif subset is None:
                    _check(
                        self._lib.fpb_search_batch(
                            self._handle, queries[s:e].data_ptr(), e - s, Q, ctypes.byref(params), buf.data_ptr(),
                            buf.numel(), ids[s:e].data_ptr(), scores[s:e].data_ptr(), counts[s:e].data_ptr(),
                            self._stream(),
                        )
                    )
                else:
                    sid, soff, smax = self._subset_csr(subset, s, e)
                    _check(
                        self._lib.fpb_search_batch_subset(
                            self._handle, queries[s:e].data_ptr(), e - s, Q, ctypes.byref(params), sid.data_ptr(),
                            soff.data_ptr(), smax, buf.data_ptr(), buf.numel(), ids[s:e].data_ptr(),
                            scores[s:e].data_ptr(), counts[s:e].data_ptr(), self._stream(),
                        )
                    )
                    self._keepalive = (sid, soff)  # until the stream has consumed them
        return ids, scores, counts

    # -- exhaustive exact search ---------------------------------------------------------------
    def exhaustive_workspace_bytes(self, B: int, Q: int, top_k: int) -> int:
        """Workspace of fpb_search_exhaustive (top_k >= 1) or of fpb_exhaustive_scores alone (top_k = 0)."""
        out = ctypes.c_size_t()
        _check(self._lib.fpb_exhaustive_workspace_bytes(self._handle, B, Q, top_k, ctypes.byref(out)))
        return int(out.value)

    def _check_queries(self, queries: torch.Tensor, host: bool = False) -> torch.Tensor:
        """Device queries as the kernels read them: fp16 [B, Q, dim] on this device, made contiguous.  host=True: the
        host-buffer path's queries, floating-point [B, Q, dim] in host memory (cast to fp16 while they are staged)."""
        if queries.dim() != 3:
            raise ValueError(f"Expected a 3D tensor for queries, but got shape {list(queries.shape)}")
        if host:
            if queries.device.type != "cpu" or not queries.dtype.is_floating_point:
                raise ValueError("DeviceIndex expects floating-point queries in host memory")
        elif queries.dtype != torch.float16 or queries.device != self.device:
            raise ValueError("DeviceIndex expects fp16 queries on the index device")
        if queries.shape[2] != self.dim:
            raise ValueError(f"query dim {queries.shape[2]} != index dim {self.dim}")
        return queries if host else queries.contiguous()

    def _check_gathered(self, t: torch.Tensor, dtype: torch.dtype, trailing: tuple) -> torch.Tensor:
        """An all-gathered input as the kernels read it: `dtype` [n_shards, B, *trailing] on this device (None in
        `trailing`: any size), contiguous."""
        if (t.dtype != dtype or t.device != self.device or t.dim() != 2 + len(trailing)
                or any(n is not None and n != m for n, m in zip(trailing, t.shape[2:]))):
            raise ValueError(f"expected gathered {dtype} [n_shards, B, *{trailing}] on {self.device}, "
                             f"got {t.dtype} {list(t.shape)} on {t.device}")
        return t.contiguous()

    def _exhaustive_step(self, B: int, Q: int, top_k: int, budget_bytes: int, workspace_bytes=None) -> int:
        """Most queries per call whose workspace fits the budget (at least one).  The size grows with B but not
        linearly (query rows are padded to blocks of 128), so the largest fitting call is found by bisection.
        `workspace_bytes(B)`: the workspace of a call of B queries (default: fpb_search_exhaustive's)."""
        if workspace_bytes is None:
            def workspace_bytes(b: int) -> int:
                return self.exhaustive_workspace_bytes(b, Q, top_k)
        if workspace_bytes(B) <= budget_bytes:
            return B
        lo, hi = 1, B  # ws(lo) may exceed the budget: one query per call is the floor
        while lo < hi:
            mid = (lo + hi + 1) // 2
            if workspace_bytes(mid) <= budget_bytes:
                lo = mid
            else:
                hi = mid - 1
        return lo

    def exhaustive_scores(self, queries: torch.Tensor) -> torch.Tensor:
        """Exact MaxSim score of every local document for every query: f32 [B, num_documents]
        (one fpb_exhaustive_scores call).  Asynchronous."""
        queries = self._check_queries(queries)
        B, Q, _ = queries.shape
        scores = torch.empty((B, self.num_documents), dtype=torch.float32, device=self.device)
        if B == 0:
            return scores
        with self._exclusive(), torch.cuda.device(self.device):
            buf = self._buffer(self.exhaustive_workspace_bytes(B, Q, 0))
            _check(
                self._lib.fpb_exhaustive_scores(
                    self._handle, queries.data_ptr(), B, Q, buf.data_ptr(), buf.numel(), scores.data_ptr(),
                    self._stream(),
                )
            )
        return scores

    def exhaustive_subset_workspace_bytes(self, B: int, Q: int, top_k: int, n_lists: int, max_list_len: int) -> int:
        """Workspace of fpb_search_exhaustive_subset."""
        out = ctypes.c_size_t()
        _check(self._lib.fpb_exhaustive_subset_workspace_bytes(self._handle, B, Q, top_k, n_lists, max_list_len,
                                                               ctypes.byref(out)))
        return int(out.value)

    def search_exhaustive(self, queries: torch.Tensor, top_k: int, budget_bytes: int = 6 << 30,
                          subset: list[list[int]] | torch.Tensor | None = None, filter: Filter | None = None,
                          groups: Groups | None = None,
                          bias: ScoreBias | None = None) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Exact top_k over every document: (ids int64 [B, top_k] global, scores f32 [B, top_k], counts int32 [B]),
        the result contract of `search`.  The batch is split into calls whose workspace fits `budget_bytes`;
        the result does not depend on the split.  Asynchronous, except with `subset` lists (their copy from host
        memory waits for the stream) and with `filter` (the workspace is sized by its largest filter, read back).

        `subset`: per query a list of GLOBAL doc ids (any order; duplicates and ids outside the index are ignored).
        Query b is then ranked among the documents of subset[b] only, with counts[b] = min(top_k, #documents), and
        every score is the one `exhaustive_scores` gives the same document.  `subset` may also be an integer tensor
        [B, L] on this device, a row of ids per query (padded with any id outside the index, such as -1): each row is
        then a list of its own, with no host list made.  `filter`: the restriction in device form
        (fpb_search_exhaustive_filter); for the same documents the result is the same bytes.

        `groups`: at most groups.max_per_group documents per group, the group's best ones: the exhaustive ranking
        (restricted to the subset or filter) with each group's first max_per_group documents kept, cut to top_k.
        `bias`: every score biased before anything is selected, exactly (fpb_index_with_bias)."""
        if groups is not None or bias is not None:
            with self._ranked(groups, bias):
                return self.search_exhaustive(queries, top_k, budget_bytes, subset, filter)
        queries = self._check_queries(queries)
        B, Q, _ = queries.shape
        k = int(top_k)
        ids = torch.empty((B, k), dtype=torch.int64, device=self.device)
        scores = torch.empty((B, k), dtype=torch.float32, device=self.device)
        counts = torch.empty((B,), dtype=torch.int32, device=self.device)
        if B == 0:
            return ids, scores, counts
        if filter is not None:
            self._check_filter(filter, B)
            self._search_exhaustive_filter(queries, k, budget_bytes, filter, ids, scores, counts)
            return ids, scores, counts
        if isinstance(subset, torch.Tensor):
            if subset.dim() != 2 or subset.shape[0] != B:
                raise ValueError("Subset length must match number of queries.")
            self._search_exhaustive_id_rows(queries, k, budget_bytes, subset, ids, scores, counts)
            return ids, scores, counts
        if subset is not None:
            if len(subset) != B:
                raise ValueError("Subset length must match number of queries.")
            self._search_exhaustive_subset(queries, k, budget_bytes, subset, ids, scores, counts)
            return ids, scores, counts
        step = self._exhaustive_step(B, Q, k, budget_bytes)
        with self._exclusive(), torch.cuda.device(self.device):
            for s in range(0, B, step):
                e = min(B, s + step)
                buf = self._buffer(self.exhaustive_workspace_bytes(e - s, Q, k))
                _check(
                    self._lib.fpb_search_exhaustive(
                        self._handle, queries[s:e].data_ptr(), e - s, Q, k, buf.data_ptr(), buf.numel(),
                        ids[s:e].data_ptr(), scores[s:e].data_ptr(), counts[s:e].data_ptr(), self._stream(),
                    )
                )
        return ids, scores, counts

    def _search_exhaustive_subset(self, queries: torch.Tensor, k: int, budget_bytes: int, subset: list,
                                  ids: torch.Tensor, scores: torch.Tensor, counts: torch.Tensor) -> None:
        """search_exhaustive with per-query subsets: identical subsets become one list (group_subsets), and each call
        passes the lists of its own queries."""
        B, Q, _ = queries.shape
        lists, query_list = group_subsets(subset)
        max_len = max(len(x) for x in lists)
        # a call of b queries has at most min(b, len(lists)) lists, none longer than max_len: its workspace bound
        step = self._exhaustive_step(B, Q, k, budget_bytes, lambda b: self.exhaustive_subset_workspace_bytes(
            b, Q, k, min(b, len(lists)), max_len))
        step = min(step, 65535)  # the library's limit on lists per call
        keep = []
        with self._exclusive(), torch.cuda.device(self.device):
            for s in range(0, B, step):
                e = min(B, s + step)
                local: dict[int, int] = {}  # list -> its index in this call, in order of first use
                call_list = [local.setdefault(l, len(local)) for l in query_list[s:e]]
                call_lists = [lists[l] for l in local]
                sid, soff, smax = self._subset_csr(call_lists, 0, len(call_lists))
                h_list = (ctypes.c_int32 * (e - s))(*call_list)
                buf = self._buffer(self.exhaustive_subset_workspace_bytes(e - s, Q, k, len(call_lists), smax))
                _check(
                    self._lib.fpb_search_exhaustive_subset(
                        self._handle, queries[s:e].data_ptr(), e - s, Q, k, sid.data_ptr(), soff.data_ptr(),
                        len(call_lists), smax, h_list, buf.data_ptr(), buf.numel(), ids[s:e].data_ptr(),
                        scores[s:e].data_ptr(), counts[s:e].data_ptr(), self._stream(),
                    )
                )
                keep.append((sid, soff))
        self._keepalive = keep  # until the stream has consumed them

    def _search_exhaustive_id_rows(self, queries: torch.Tensor, k: int, budget_bytes: int, rows: torch.Tensor,
                                   ids: torch.Tensor, scores: torch.Tensor, counts: torch.Tensor) -> None:
        """search_exhaustive with ids [B, L]: row b is query b's list, offsets built on the device."""
        B, Q, _ = queries.shape
        L = int(rows.shape[1])
        # int32 like _subset_csr: an id past int32 is past every index and stays ignored
        flat = rows.to(self.device).clamp(-1, 2**31 - 1).to(torch.int32).contiguous().view(-1)
        if flat.numel() == 0:
            flat = torch.full((1,), -1, dtype=torch.int32, device=self.device)
        step = self._exhaustive_step(B, Q, k, budget_bytes, lambda b: self.exhaustive_subset_workspace_bytes(
            b, Q, k, b, L))
        step = min(step, 65535)  # the library's limit on lists per call
        offs = torch.arange(step + 1, dtype=torch.int64, device=self.device) * L
        with self._exclusive(), torch.cuda.device(self.device):
            for s in range(0, B, step):
                e = min(B, s + step)
                h_list = (ctypes.c_int32 * (e - s))(*range(e - s))
                buf = self._buffer(self.exhaustive_subset_workspace_bytes(e - s, Q, k, e - s, L))
                _check(
                    self._lib.fpb_search_exhaustive_subset(
                        self._handle, queries[s:e].data_ptr(), e - s, Q, k, flat[s * L:].data_ptr(), offs.data_ptr(),
                        e - s, L, h_list, buf.data_ptr(), buf.numel(), ids[s:e].data_ptr(), scores[s:e].data_ptr(),
                        counts[s:e].data_ptr(), self._stream(),
                    )
                )
        self._keepalive = (flat, offs)  # until the stream has consumed them

    def exhaustive_filter_workspace_bytes(self, B: int, Q: int, top_k: int, n_filters: int, max_count: int) -> int:
        """Workspace of fpb_search_exhaustive_filter."""
        out = ctypes.c_size_t()
        _check(self._lib.fpb_exhaustive_filter_workspace_bytes(self._handle, B, Q, top_k, n_filters, max_count,
                                                               ctypes.byref(out)))
        return int(out.value)

    def _search_exhaustive_filter(self, queries: torch.Tensor, k: int, budget_bytes: int, filter: Filter,
                                  ids: torch.Tensor, scores: torch.Tensor, counts: torch.Tensor) -> None:
        """search_exhaustive with filters: each call passes the filters of its own queries, one list each."""
        B, Q, _ = queries.shape
        n_used = len(set(filter.query_filter))
        max_count = int(self.filter_counts(filter).max())  # sizes the workspace: one synchronisation
        step = self._exhaustive_step(B, Q, k, budget_bytes, lambda b: self.exhaustive_filter_workspace_bytes(
            b, Q, k, min(b, n_used), max_count))
        step = min(step, 65535)  # the library's limit on filters per call
        keep = []
        with self._exclusive(), torch.cuda.device(self.device):
            for s in range(0, B, step):
                e = min(B, s + step)
                rows, local = filter.call_rows(s, e)
                keep.append(rows)
                h_map = (ctypes.c_int32 * (e - s))(*local)
                buf = self._buffer(self.exhaustive_filter_workspace_bytes(e - s, Q, k, rows.shape[0], max_count))
                _check(
                    self._lib.fpb_search_exhaustive_filter(
                        self._handle, queries[s:e].data_ptr(), e - s, Q, k, rows.data_ptr(), rows.shape[0],
                        filter.n_bits, max_count, h_map, buf.data_ptr(), buf.numel(), ids[s:e].data_ptr(),
                        scores[s:e].data_ptr(), counts[s:e].data_ptr(), self._stream(),
                    )
                )
            self._keepalive = self._stream_keep(*keep)  # until the stream has consumed them

    # -- document-sharded exhaustive search ------------------------------------------------------
    def shard_exhaustive_records(self, queries: torch.Tensor, top_k: int,
                                 groups: Groups | None = None, bias: ScoreBias | None = None) -> torch.Tensor:
        """Step-wise sharded exhaustive search, local half: uint8 [B, top_k, 16] records (score f32 twice, global
        doc id i64) of this shard's top_k documents per query, padded with (-inf, -inf, -1).  The shards' records,
        all-gathered, go to `merge_records(all_records, top_k)`.  Asynchronous.  `groups` (Groups.for_shard): the
        shard's top_k under the group rule; the records then go to `merge_records(all_records, top_k, groups,
        n_keep=n_shards * top_k)`."""
        if groups is not None or bias is not None:
            with self._ranked(groups, bias):
                return self.shard_exhaustive_records(queries, top_k)
        queries = self._check_queries(queries)
        B, Q, _ = queries.shape
        k = int(top_k)
        rec = torch.empty((B, max(k, 0), 16), dtype=torch.uint8, device=self.device)
        if B == 0:
            return rec
        with self._exclusive(), torch.cuda.device(self.device):
            buf = self._buffer(self.exhaustive_workspace_bytes(B, Q, k))
            _check(self._lib.fpb_shard_exhaustive_records(self._handle, queries.data_ptr(), B, Q, k, buf.data_ptr(),
                                                          buf.numel(), rec.data_ptr(), self._stream()))
        return rec

    def exhaustive_sharded_step(self, n_query_groups: int, B: int, Q: int, top_k: int,
                                budget_bytes: int = 6 << 30, groups: Groups | None = None) -> int:
        """Most queries per `search_exhaustive_sharded` call whose workspace on this rank, that of
        ceil(step / n_query_groups) queries, fits `budget_bytes`.  It depends on this shard's document count, so the
        ranks must agree on one step (the smallest of theirs) before the first collective call.  `groups`: the
        workspace of the grouped call."""
        if groups is not None:
            with self._grouped(groups):
                return self.exhaustive_sharded_step(n_query_groups, B, Q, top_k, budget_bytes)
        G = max(int(n_query_groups), 1)
        return min(B, self._exhaustive_step(-(-B // G), Q, top_k, budget_bytes) * G)

    def search_exhaustive_sharded(self, comm: ShardComm, n_query_groups: int, queries: torch.Tensor, top_k: int,
                                  step: int | None = None,
                                  groups: Groups | None = None,
                                  bias: ScoreBias | None = None) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Exhaustive search of a document-sharded index (fpb_search_exhaustive_sharded): queries fp16 [B, Q, D] on
        this device, the SAME batch on every rank of `comm` (collective call).  Returns device tensors (ids, scores,
        counts) for all B queries, the bytes `search_exhaustive` gives on one GPU holding the whole index.
        `step`: queries per collective call, the same on every rank (default: the whole batch in one call;
        `exhaustive_sharded_step` gives this rank's largest within a memory budget).  Asynchronous.  `groups`
        (Groups.for_shard): the grouped result of the whole index, exactly."""
        if groups is not None or bias is not None:
            with self._ranked(groups, bias):
                return self.search_exhaustive_sharded(comm, n_query_groups, queries, top_k, step)
        queries = self._check_queries(queries)
        B, Q, _ = queries.shape
        k, G = int(top_k), int(n_query_groups)
        ids = torch.empty((B, max(k, 0)), dtype=torch.int64, device=self.device)
        scores = torch.empty((B, max(k, 0)), dtype=torch.float32, device=self.device)
        counts = torch.empty((B,), dtype=torch.int32, device=self.device)
        if B == 0:
            return ids, scores, counts
        step = B if step is None else max(1, int(step))
        with self._exclusive(), torch.cuda.device(self.device):
            for s in range(0, B, step):
                e = min(B, s + step)
                b_local = -(-(e - s) // max(G, 1))
                buf = self._buffer(self.exhaustive_workspace_bytes(b_local, Q, k))
                need = max(1, int(self._lib.fpb_sharded_scratch_bytes(b_local, k, comm.nranks)))
                self._grow_scratch(need)
                _check(self._lib.fpb_search_exhaustive_sharded(
                    self._handle, comm._handle, G, queries[s:e].data_ptr(), e - s, Q, k, buf.data_ptr(), buf.numel(),
                    self._scratch.data_ptr(), self._scratch.numel(), ids[s:e].data_ptr(), scores[s:e].data_ptr(),
                    counts[s:e].data_ptr(), self._stream()))
        return ids, scores, counts

    def _host_io(self, B: int, Q: int, k: int) -> dict[str, Any]:
        """Cached pinned + device staging buffers of the host-buffer path."""
        key = (B, Q, k)
        with self._lock:
            io = self._io.get(key)
            if io is None:
                while len(self._io) >= 4:  # a few shapes stay cached (pinning memory costs milliseconds)
                    self._io.pop(next(iter(self._io)))
                D = self.dim
                io = {
                    "d_q": torch.empty((B, Q, D), dtype=torch.float16, device=self.device),
                    "d_ids": torch.empty((B, k), dtype=torch.int64, device=self.device),
                    "d_scores": torch.empty((B, k), dtype=torch.float32, device=self.device),
                    "d_counts": torch.empty((B,), dtype=torch.int32, device=self.device),
                    "h_q": torch.empty((B, Q, D), dtype=torch.float16).pin_memory(),
                    "h_ids": torch.empty((B, k), dtype=torch.int64).pin_memory(),
                    "h_scores": torch.empty((B, k), dtype=torch.float32).pin_memory(),
                    "h_counts": torch.empty((B,), dtype=torch.int32).pin_memory(),
                    "staged": torch.cuda.Event(),  # the last stage_queries copy out of h_q
                }
                self._io[key] = io
        return io

    def _cast_into_pinned(self, queries_host: torch.Tensor, io: dict[str, Any]) -> None:
        """fp32 -> fp16 on the host like the reference (fast_plaid.py:241), straight into the pinned `h_q`, once the
        copy a previous stage_queries queued out of it has run."""
        io["staged"].synchronize()
        h_q = io["h_q"]
        if queries_host.dtype == torch.float32 and queries_host.is_contiguous():
            # single-threaded F16C cast in the library: no dependence on ATen's intra-op pool (csrc/host_cast.cu)
            _check(self._lib.fpb_cast_f32_to_f16_host(queries_host.data_ptr(), h_q.data_ptr(), queries_host.numel()))
        else:
            h_q.copy_(queries_host)

    def stage_queries(self, queries_host: torch.Tensor, top_k: int) -> torch.Tensor:
        """Host queries [B, Q, D] -> fp16 device tensor (cached buffer; asynchronous on the current stream)."""
        B, Q, _ = queries_host.shape
        io = self._host_io(B, Q, top_k)
        self._cast_into_pinned(queries_host, io)
        io["d_q"].copy_(io["h_q"], non_blocking=True)
        io["staged"].record()
        return io["d_q"]

    def search_host(
        self, queries_host: torch.Tensor, params: FpbParams, groups: Groups | None = None,
        bias: ScoreBias | None = None,
    ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """queries_host: float [B, Q, D] in HOST memory.  The H2D copy, the search and the D2H copies of the
        results all happen inside the C-ABI call, which synchronises the stream.  Returns HOST tensors
        (ids, scores, counts).  `groups`: as in `search`."""
        if groups is not None or bias is not None:
            with self._ranked(groups, bias):
                return self.search_host(queries_host, params)
        B, Q, _ = self._check_queries(queries_host, host=True).shape
        if B == 0:
            k = params.top_k
            return (torch.empty((0, k), dtype=torch.int64), torch.empty((0, k), dtype=torch.float32),
                    torch.empty((0,), dtype=torch.int32))
        with self._exclusive(), torch.cuda.device(self.device):
            params = self._approx_flags(params)
            step = self.max_queries_per_call(Q, params)
            io = self._host_io(B, Q, params.top_k)
            self._cast_into_pinned(queries_host, io)
            queries_host = io["h_q"]
            for s in range(0, B, step):
                e = min(B, s + step)
                buf, lay = self.workspace(e - s, Q, params)
                _check(
                    self._lib.fpb_search_batch_host(
                        self._handle, queries_host[s:e].data_ptr(), e - s, Q, ctypes.byref(params),
                        buf.data_ptr(), buf.numel(), io["d_q"][s:e].data_ptr(), io["d_ids"][s:e].data_ptr(),
                        io["d_scores"][s:e].data_ptr(), io["d_counts"][s:e].data_ptr(),
                        io["h_ids"][s:e].data_ptr(), io["h_scores"][s:e].data_ptr(),
                        io["h_counts"][s:e].data_ptr(), self._stream(),
                    )
                )
            self._adapt_approx_mode(buf, lay)
            # the pinned result buffers are reused by the next call of this shape: hand out copies (77 KB at
            # 64 x 100) while this call still owns them
            return io["h_ids"].clone(), io["h_scores"].clone(), io["h_counts"].clone()

    def search_records(self, queries: torch.Tensor, params: FpbParams) -> torch.Tensor:
        """Sharded mode, local half: returns uint8 [B, R, 16] records (approx f32, exact f32,
        global doc id i64) for this shard's n_full_scores/4 best candidates per query."""
        queries = self._check_queries(queries)
        B, Q, _ = queries.shape
        with self._exclusive(), torch.cuda.device(self.device):
            buf, lay = self.workspace(B, Q, params)
            rec = torch.empty((B, lay.R, 16), dtype=torch.uint8, device=self.device)
            _check(
                self._lib.fpb_search_shard(
                    self._handle, queries.data_ptr(), B, Q, ctypes.byref(params), buf.data_ptr(), buf.numel(),
                    rec.data_ptr(), self._stream(),
                )
            )
        return rec

    # -- approximate-stage mode --------------------------------------------------------------
    # The two-pass approximate stage (bound pass + exact pass, csrc/k3_approx.cu) wins when most candidates can be
    # discarded by their upper bound (uniform codes: < 1 % re-scored) and loses its fixed costs when the candidates
    # of a query all score alike (strongly clustered corpora: the exact pass then re-scores most of them).  Both
    # modes give bit-identical results, so the host-buffer path simply looks, every APPROX_PROBE_EVERY calls, at the
    # fraction the exact pass re-scored and holds the one-pass mode for a while when it is high.
    APPROX_PROBE_EVERY = 8
    APPROX_DIRECT_ABOVE = 0.30
    APPROX_HOLD_CALLS = 64

    def _approx_flags(self, params: FpbParams) -> FpbParams:
        if self._approx_direct and not (params.flags & (FPB_FLAG_APPROX_EXACT_ALL | FPB_FLAG_APPROX_DIRECT |
                                                        FPB_FLAG_APPROX_TWO_PASS)):
            return self.with_flags(params, FPB_FLAG_APPROX_DIRECT)
        return params

    def _adapt_approx_mode(self, buf: torch.Tensor, lay: FpbLayout) -> None:
        """Called after a synchronised host-buffer search (the workspace still holds its counters)."""
        if self._approx_direct:
            self._approx_hold -= 1
            if self._approx_hold <= 0:
                self._approx_direct = False  # probe the two-pass mode again
            return
        self._approx_calls += 1
        if self._approx_calls % self.APPROX_PROBE_EVERY or lay.flags & FPB_FLAG_APPROX_DIRECT:
            return
        v = self.views(buf, lay)
        both = torch.stack([v["n_refine"].sum(), v["n_cand"].sum()]).cpu()
        n_ref, n_cand = int(both[0]), int(both[1])
        if n_cand > 0 and n_ref / n_cand > self.APPROX_DIRECT_ABOVE:
            self._approx_direct = True
            self._approx_hold = self.APPROX_HOLD_CALLS

    # the whole sharded search in one C-ABI call (both NCCL all-gathers issued inside, csrc/comm.cu)
    def _sharded_io(self, comm: ShardComm, n_query_groups: int, B: int, Q: int, params: FpbParams):
        b_local = -(-B // n_query_groups)
        buf, lay = self.workspace(b_local, Q, params)
        self._grow_scratch(int(self._lib.fpb_sharded_scratch_bytes(b_local, lay.R, comm.nranks)))
        return buf, self._scratch

    def _grow_scratch(self, nbytes: int) -> None:
        """The grow-only scratch of the sharded searches (callers hold _exclusive)."""
        old = getattr(self, "_scratch", None)
        if old is None or old.numel() < nbytes:
            self._drop(old)
            self._scratch = None
            self._scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)

    def search_sharded(self, comm: ShardComm, n_query_groups: int, queries: torch.Tensor, params: FpbParams,
                       groups: Groups | None = None,
                       bias: ScoreBias | None = None) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """queries: fp16 [B, Q, D] on this device, the SAME batch on every rank of `comm` (collective call).
        Returns device tensors (ids, scores, counts) for all B queries.  `groups` (Groups.for_shard): the merge keeps
        at most groups.max_per_group documents per group of the n_full_scores / 4 it re-ranks, as `search` does."""
        if groups is not None or bias is not None:
            with self._ranked(groups, bias):
                return self.search_sharded(comm, n_query_groups, queries, params)
        queries = self._check_queries(queries)
        B, Q, _ = queries.shape
        k = params.top_k
        ids = torch.empty((B, k), dtype=torch.int64, device=self.device)
        scores = torch.empty((B, k), dtype=torch.float32, device=self.device)
        counts = torch.empty((B,), dtype=torch.int32, device=self.device)
        with self._exclusive(), torch.cuda.device(self.device):
            buf, scratch = self._sharded_io(comm, n_query_groups, B, Q, params)
            _check(self._lib.fpb_search_batch_sharded(
                self._handle, comm._handle, n_query_groups, queries.data_ptr(), B, Q, ctypes.byref(params),
                buf.data_ptr(), buf.numel(), scratch.data_ptr(), scratch.numel(), ids.data_ptr(), scores.data_ptr(),
                counts.data_ptr(), self._stream()))
        return ids, scores, counts

    def search_sharded_host(self, comm: ShardComm, n_query_groups: int, queries_host: torch.Tensor,
                            params: FpbParams,
                            groups: Groups | None = None,
                            bias: ScoreBias | None = None) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Host-buffer form of `search_sharded`: fp32/fp16 queries in HOST memory in, host tensors out."""
        if groups is not None or bias is not None:
            with self._ranked(groups, bias):
                return self.search_sharded_host(comm, n_query_groups, queries_host, params)
        B, Q, _ = self._check_queries(queries_host, host=True).shape
        with self._exclusive(), torch.cuda.device(self.device):
            io = self._host_io(B, Q, params.top_k)
            self._cast_into_pinned(queries_host, io)
            buf, scratch = self._sharded_io(comm, n_query_groups, B, Q, params)
            _check(self._lib.fpb_search_batch_sharded_host(
                self._handle, comm._handle, n_query_groups, io["h_q"].data_ptr(), B, Q, ctypes.byref(params),
                buf.data_ptr(), buf.numel(), scratch.data_ptr(), scratch.numel(), io["d_q"].data_ptr(),
                io["d_ids"].data_ptr(), io["d_scores"].data_ptr(), io["d_counts"].data_ptr(), io["h_ids"].data_ptr(),
                io["h_scores"].data_ptr(), io["h_counts"].data_ptr(), self._stream()))
            return io["h_ids"].clone(), io["h_scores"].clone(), io["h_counts"].clone()

    # two-step sharded search (exact-scores only the globally surviving documents)
    def shard_approx_keys(self, queries: torch.Tensor, params: FpbParams) -> torch.Tensor:
        queries = self._check_queries(queries)
        B, Q, _ = queries.shape
        with self._exclusive(), torch.cuda.device(self.device):
            buf, lay = self.workspace(B, Q, params)
            keys = torch.empty((B, lay.R), dtype=torch.int64, device=self.device)
            _check(self._lib.fpb_shard_approx_keys(self._handle, queries.data_ptr(), B, Q, ctypes.byref(params),
                                                   buf.data_ptr(), buf.numel(), keys.data_ptr(), self._stream()))
        return keys

    def shard_subset_begin(self, queries: torch.Tensor, params: FpbParams, subset: list[list[int]] | None = None,
                           filter: Filter | None = None) -> torch.Tensor:
        """Sharded search with a `subset`, step 1a: centroid scores and this shard's bitmaps.  Returns the
        shard's centroid bitmap, int32 [B, cbitmap_words], for the all-gather.  `params.flags` must carry
        FPB_FLAG_SUBSET; `subset` holds GLOBAL document ids.  `filter`: the restriction in device form over global
        ids, of which this shard reads its own range (fpb_shard_filter_begin)."""
        queries = self._check_queries(queries)
        B, Q, _ = queries.shape
        if filter is not None:
            self._check_filter(filter, B)
            h_map = (ctypes.c_int32 * B)(*filter.query_filter)
            with self._exclusive(), torch.cuda.device(self.device):
                buf, lay = self.workspace(B, Q, params)
                cb = torch.empty((B, lay.cbitmap_words), dtype=torch.int32, device=self.device)
                _check(self._lib.fpb_shard_filter_begin(self._handle, queries.data_ptr(), B, Q, ctypes.byref(params),
                                                        filter.bitmap.data_ptr(), filter.n_filters, filter.n_bits,
                                                        h_map, buf.data_ptr(), buf.numel(), cb.data_ptr(),
                                                        self._stream()))
                self._stream_keep(filter.bitmap)  # the caller may free the filter before the stream reads it
            return cb
        sid, soff, smax = self._subset_csr(subset, 0, B)
        with self._exclusive(), torch.cuda.device(self.device):
            buf, lay = self.workspace(B, Q, params)
            cb = torch.empty((B, lay.cbitmap_words), dtype=torch.int32, device=self.device)
            _check(self._lib.fpb_shard_subset_begin(self._handle, queries.data_ptr(), B, Q, ctypes.byref(params),
                                                    sid.data_ptr(), soff.data_ptr(), smax, buf.data_ptr(),
                                                    buf.numel(), cb.data_ptr(), self._stream()))
            torch.cuda.current_stream(self.device).synchronize()  # sid/soff are temporaries
        return cb

    def shard_subset_keys(self, all_cbitmaps: torch.Tensor, Q: int, params: FpbParams) -> torch.Tensor:
        """Step 1b: all_cbitmaps int32 [n_shards, B, cbitmap_words] (all-gathered) -> int64 keys [B, R]."""
        with self._exclusive(), torch.cuda.device(self.device):
            buf, lay = self.workspace(all_cbitmaps.shape[1], Q, params)
            all_cbitmaps = self._check_gathered(all_cbitmaps, torch.int32, (lay.cbitmap_words,))
            n_shards, B, _ = all_cbitmaps.shape
            keys = torch.empty((B, lay.R), dtype=torch.int64, device=self.device)
            _check(self._lib.fpb_shard_subset_keys(self._handle, B, Q, ctypes.byref(params), buf.data_ptr(),
                                                   buf.numel(), all_cbitmaps.data_ptr(), n_shards,
                                                   keys.data_ptr(), self._stream()))
        return keys

    def shard_exact_records(self, all_keys: torch.Tensor, rank: int, Q: int, params: FpbParams,
                            bias: ScoreBias | None = None) -> torch.Tensor:
        """all_keys: int64 [n_shards, B, R] (all-gathered).  Applies the global pruning threshold to
        this shard's list, exact-scores the survivors, returns uint8 [B, R, 16] records.  `bias`
        (ScoreBias.for_shard): the exact scores are biased."""
        if bias is not None:
            with self._biased(bias):
                return self.shard_exact_records(all_keys, rank, Q, params)
        with self._exclusive(), torch.cuda.device(self.device):
            buf, lay = self.workspace(all_keys.shape[1], Q, params)
            all_keys = self._check_gathered(all_keys, torch.int64, (lay.R,))
            n_shards, B, R = all_keys.shape
            rec = torch.empty((B, R, 16), dtype=torch.uint8, device=self.device)
            _check(self._lib.fpb_shard_apply_threshold(self._handle, all_keys.data_ptr(), n_shards, rank,
                                                       B, Q, ctypes.byref(params), buf.data_ptr(), buf.numel(),
                                                       self._stream()))
            _check(self._lib.fpb_shard_exact_records(self._handle, B, Q, ctypes.byref(params), buf.data_ptr(),
                                                     buf.numel(), rec.data_ptr(), self._stream()))
        return rec

    def merge_records(
        self, all_records: torch.Tensor, top_k: int, groups: Groups | None = None, n_keep: int | None = None,
    ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """all_records: uint8 [n_shards, B, R, 16] (all-gathered).  Global prune + rank.  `groups` (Groups.for_shard,
        its `global_ids` read): the n_keep best records by approximate score (default R: the approximate search's
        pruning; n_shards * R: every record, for exhaustive records) ranked by exact score, at most
        groups.max_per_group per group (fpb_merge_shards_grouped)."""
        all_records = self._check_gathered(all_records, torch.uint8, (None, 16))
        n_shards, B, R, _ = all_records.shape
        ids = torch.empty((B, top_k), dtype=torch.int64, device=self.device)
        scores = torch.empty((B, top_k), dtype=torch.float32, device=self.device)
        counts = torch.empty((B,), dtype=torch.int32, device=self.device)
        with self._exclusive(), torch.cuda.device(self.device):
            if groups is not None:
                gl = groups.global_ids
                if gl is None or gl.device != self.device or gl.dtype != torch.int32 or not gl.is_contiguous():
                    raise ValueError(f"merge_records needs the int32 map of the whole index on {self.device} "
                                     "(Groups.for_shard)")
                _check(self._lib.fpb_merge_shards_grouped(
                    all_records.data_ptr(), n_shards, B, R, R if n_keep is None else int(n_keep), top_k,
                    gl.data_ptr(), gl.shape[0], groups.max_per_group, ids.data_ptr(), scores.data_ptr(),
                    counts.data_ptr(), self._stream()))
                self._groups_keepalive = self._stream_keep(gl)  # until the stream has consumed it
                return ids, scores, counts
            _check(
                self._lib.fpb_merge_shards(
                    all_records.data_ptr(), n_shards, B, R, top_k, ids.data_ptr(),
                    scores.data_ptr(), counts.data_ptr(), self._stream(),
                )
            )
        return ids, scores, counts

    # -- stage-level access for the parity tests and the roofline bench -------------------
    def run_stages(self, queries: torch.Tensor, params: FpbParams, upto: str = "rank",
                   subset: list[list[int]] | None = None, filter: Filter | None = None) -> dict[str, Any]:
        """Run the pipeline stage by stage and return views of every intermediate.  With `subset` or `filter` the
        "subset" / "filter" stage runs after centroid_scores, and the views include sbitmap, cbitmap and clist."""
        order = ["centroid_scores", "probe", "candidates", "approx", "select", "maxsim", "rank"]
        if subset is not None or filter is not None:
            params = self.with_flags(params, FPB_FLAG_SUBSET)
            order.insert(1, "subset" if filter is None else "filter")
        queries = self._check_queries(queries)
        B, Q, _ = queries.shape
        p = ctypes.byref(params)
        with self._exclusive(), torch.cuda.device(self.device):
            buf, lay = self.workspace(B, Q, params)
            st = self._stream()
            out: dict[str, Any] = {"layout": lay, "workspace": buf}
            for name in order:
                if name == "centroid_scores":
                    _check(self._lib.fpb_stage_centroid_scores(self._handle, queries.data_ptr(), B, Q, p,
                                                               buf.data_ptr(), buf.numel(), st))
                elif name == "subset":
                    sid, soff, smax = self._subset_csr(subset, 0, B)
                    _check(self._lib.fpb_stage_subset(self._handle, sid.data_ptr(), soff.data_ptr(), smax, B, Q, p,
                                                      buf.data_ptr(), buf.numel(), st))
                    torch.cuda.synchronize(self.device)
                elif name == "filter":
                    self._check_filter(filter, B)
                    h_map = (ctypes.c_int32 * B)(*filter.query_filter)
                    _check(self._lib.fpb_stage_filter(self._handle, filter.bitmap.data_ptr(), filter.n_filters,
                                                      filter.n_bits, h_map, B, Q, p, buf.data_ptr(), buf.numel(), st))
                elif name == "rank":
                    k = params.top_k
                    ids = torch.empty((B, k), dtype=torch.int64, device=self.device)
                    scores = torch.empty((B, k), dtype=torch.float32, device=self.device)
                    counts = torch.empty((B,), dtype=torch.int32, device=self.device)
                    _check(self._lib.fpb_stage_rank(self._handle, B, Q, p, buf.data_ptr(), buf.numel(),
                                                    ids.data_ptr(), scores.data_ptr(), counts.data_ptr(), st))
                    out.update(ids=ids, scores=scores, counts=counts)
                else:
                    fn = getattr(self._lib, f"fpb_stage_{name}")
                    _check(fn(self._handle, B, Q, p, buf.data_ptr(), buf.numel(), st))
                if name == upto:
                    break
        out.update(self.views(buf, lay))
        return out

    def stage_fn(self, name: str, queries: torch.Tensor, params: FpbParams):
        """A zero-argument callable that launches one stage on the cached workspace (bench)."""
        queries = self._check_queries(queries)
        B, Q, _ = queries.shape
        buf, lay = self.workspace(B, Q, params)
        p = ctypes.byref(params)
        st = self._stream()
        if name == "centroid_scores":
            return lambda: _check(self._lib.fpb_stage_centroid_scores(
                self._handle, queries.data_ptr(), B, Q, p, buf.data_ptr(), buf.numel(), st))
        fn = getattr(self._lib, f"fpb_stage_{name}")
        return lambda: _check(fn(self._handle, B, Q, p, buf.data_ptr(), buf.numel(), st))

    def views(self, buf: torch.Tensor, lay: FpbLayout) -> dict[str, torch.Tensor]:
        B, Q, Qp, R = lay.B, lay.Q, lay.Qp, lay.R
        K = self.num_centroids

        def v(off: int, nbytes: int, dtype: torch.dtype, shape: tuple) -> torch.Tensor:
            return buf[off : off + nbytes].view(dtype).view(*shape)

        return {
            "S": v(lay.off_S, B * K * Qp * 2, torch.float16, (B, K, Qp)),
            "tmax": v(lay.off_tmax, B * Qp * lay.n_tiles * 2, torch.float16, (B, Qp, lay.n_tiles)),
            "cells": v(lay.off_cells, B * Q * lay.n_probe * 4, torch.int32, (B, Q, lay.n_probe)),
            "n_cand": v(lay.off_n_cand, B * 4, torch.int32, (B,)),
            "cand": v(lay.off_cand, B * lay.cand_cap * 4, torch.int32, (B, lay.cand_cap)),
            "approx": v(lay.off_approx, B * lay.cand_cap * 4, torch.float32, (B, lay.cand_cap)),
            "n_rerank": v(lay.off_n_rerank, B * 4, torch.int32, (B,)),
            "rerank": v(lay.off_rerank, B * R * 4, torch.int32, (B, R)),
            "rerank_approx": v(lay.off_rerank_approx, B * R * 4, torch.float32, (B, R)),
            "exact": v(lay.off_exact, B * R * 4, torch.float32, (B, R)),
            # two-pass approximate stage (absent with FPB_FLAG_APPROX_DIRECT)
            **({} if lay.flags & FPB_FLAG_APPROX_DIRECT else {
                "tau": v(lay.off_tau, B * Qp * 2, torch.float16, (B, Qp)),
                "hibits": v(lay.off_hibits, B * lay.hb_words * 4, torch.int32, (B, lay.hb_words)),
                "approx_lb": v(lay.off_lb, B * lay.cand_cap * 4, torch.float32, (B, lay.cand_cap)),
                "refine": v(lay.off_refine, B * lay.cand_cap * 4, torch.int32, (B, lay.cand_cap)),
            }),
            "n_refine": v(lay.off_n_refine, B * 4, torch.int32, (B,)),
            "thresh": v(lay.off_thresh, B * 4, torch.float32, (B,)),
            "stats": v(lay.off_stats, 64, torch.int64, (8,)),
            # subset / filter structures (FPB_FLAG_SUBSET)
            **({} if not lay.flags & FPB_FLAG_SUBSET else {
                "sbitmap": v(lay.off_sbitmap, B * lay.bitmap_words * 4, torch.int32, (B, lay.bitmap_words)),
                "cbitmap": v(lay.off_cbitmap, B * lay.cbitmap_words * 4, torch.int32, (B, lay.cbitmap_words)),
                "n_clist": v(lay.off_n_clist, B * 4, torch.int32, (B,)),
                "clist": v(lay.off_clist, B * K * 4, torch.int32, (B, K)),
            }),
        }

    def walk_layout(self) -> tuple[torch.Tensor, torch.Tensor]:
        """Copies of the approximate stage's walk layout (csrc/common.cuh): codes int32 [windows, 32] and each
        document's first window, int64 [N + 1]."""
        n = ctypes.c_int64()
        with self._exclusive(), torch.cuda.device(self.device):
            _check(self._lib.fpb_index_walk_layout(self._handle, ctypes.byref(n), None, None))
            codes = torch.empty((max(n.value, 1), 32), dtype=torch.int32, device=self.device)
            win = torch.empty(self.num_documents + 1, dtype=torch.int64, device=self.device)
            _check(self._lib.fpb_index_walk_layout(self._handle, ctypes.byref(n), codes.data_ptr(), win.data_ptr()))
        return codes[: n.value], win

    # -- by-products -----------------------------------------------------------------------
    def reconstruct(self, doc_ids: list[int]) -> list[torch.Tensor]:
        """reconstruct_embeddings (rust/utils/embeddings.rs:12-69): fp16 [len, D] per doc."""
        if not doc_ids:
            return []
        ids = torch.tensor(doc_ids, dtype=torch.int64)
        if int(ids.min()) < 0 or int(ids.max()) >= self.num_documents:
            raise ValueError("document id out of range")
        offs = self.doc_offsets.cpu()
        lens = offs[ids + 1] - offs[ids]
        out_off = torch.zeros(len(doc_ids) + 1, dtype=torch.int64)
        out_off[1:] = lens.cumsum(0)
        total = int(out_off[-1])
        out = torch.empty((max(total, 1), self.dim), dtype=torch.float16, device=self.device)
        d_ids = ids.to(self.device, torch.int32)
        d_off = out_off.to(self.device)
        with self._exclusive(), torch.cuda.device(self.device):
            _check(self._lib.fpb_reconstruct(self._handle, d_ids.data_ptr(), len(doc_ids), d_off.data_ptr(),
                                             out.data_ptr(), self._stream()))
        return [out[int(out_off[i]) : int(out_off[i + 1])] for i in range(len(doc_ids))]

    def token_scores(self, queries: torch.Tensor, query_of: torch.Tensor, doc_ids: torch.Tensor) -> torch.Tensor:
        """fp16 [n, max_len, Q] token matrices for explicit (query, local doc) pairs."""
        queries = self._check_queries(queries)
        n = int(doc_ids.shape[0])
        Q = int(queries.shape[1])
        out = torch.zeros((max(n, 1), max(self.max_doc_len, 1), Q), dtype=torch.float16, device=self.device)
        if n == 0:
            return out[:0]
        qo = query_of.to(self.device, torch.int32).contiguous()
        di = doc_ids.to(self.device, torch.int32).contiguous()
        with self._exclusive(), torch.cuda.device(self.device):
            _check(self._lib.fpb_token_scores(self._handle, queries.data_ptr(), Q, qo.data_ptr(), di.data_ptr(), n,
                                              max(self.max_doc_len, 1), out.data_ptr(), self._stream()))
        return out
