"""Index mutation: append documents / delete documents (host-side, off the hot path).

Kept from the reference (python/fast_plaid/search/update.py:206-452, rust/index/update.rs:30-473,
rust/index/delete.rs:26-145): create-if-missing, rebuild-from-scratch while the index is small
and the raw ``embeddings.npy`` is still around, otherwise encode with the EXISTING codec and
append; deletion rewrites the chunk files, renumbers the documents and rebuilds the IVF.
Not reproduced (mutation policy, SURVEY.md section 2 rows 8/15): the outlier buffer and the
centroid expansion of ``update_centroids``.
"""

from __future__ import annotations

import json
import os
from typing import Any

import numpy as np
import torch

from . import build, store


def _load_raw(path: str) -> list[torch.Tensor]:
    arr = np.load(path, allow_pickle=True)
    return [torch.from_numpy(a) for a in arr]


def process_update(fp: Any, docs: list[torch.Tensor], metadata: list[dict] | None, batch_size: int,
                   kmeans_niters: int, max_points_per_centroid: int, n_samples_kmeans: int | None, seed: int,
                   start_from_scratch: int, loaded: dict[str, Any] | None = None) -> dict[str, Any] | None:
    """Add `docs` to the index directory.  `loaded` (device -> DeviceIndex of the directory as it is on disk) asks
    for the appended documents to be added to those indexes in place as well; the grown indexes are returned when
    that happened, None when the caller has to load the directory again."""
    index_path = fp.index
    meta = store.read_metadata(index_path)
    if meta is None:  # update.py:271-290
        fp.create(docs, kmeans_niters=kmeans_niters, max_points_per_centroid=max_points_per_centroid,
                  n_samples_kmeans=n_samples_kmeans, batch_size=batch_size, seed=seed, metadata=metadata)
        return None
    n_old = int(meta.get("num_documents", 0))
    emb_path = os.path.join(index_path, "embeddings.npy")
    db = os.path.join(index_path, "metadata.db")
    if os.path.exists(db):
        # update.py:300-311: once a metadata table exists EVERY added document gets a row (an empty one when
        # no metadata is given), so that `_subset_` stays equal to the document id
        if metadata is None:
            metadata = [{} for _ in docs]
        if len(metadata) != len(docs):
            raise ValueError(
                f"The length of metadata ({len(metadata)}) must match the number of "
                f"documents_embeddings ({len(docs)})."
            )
        from ..filtering import update as _meta_update

        _meta_update(index=index_path, metadata=metadata)
    if n_old <= start_from_scratch and os.path.exists(emb_path):  # update.py:314-349
        old = _load_raw(emb_path)
        keep_db = os.path.exists(db)
        if keep_db:  # create() clears the directory's table: park it
            os.replace(db, db + ".keep")
        try:
            fp.create(old + docs, kmeans_niters=kmeans_niters, max_points_per_centroid=max_points_per_centroid,
                      nbits=int(meta["nbits"]), n_samples_kmeans=n_samples_kmeans, batch_size=batch_size, seed=seed,
                      start_from_scratch=start_from_scratch + 1,
                      compress_only=bool(meta.get("compress_only", False)))
        finally:
            if keep_db and os.path.exists(db + ".keep"):
                os.replace(db + ".keep", db)
        if len(old) + len(docs) > start_from_scratch and os.path.exists(emb_path):
            os.remove(emb_path)
        return None
    return append_documents(index_path, docs, batch_size=batch_size, device=fp.devices[0], loaded=loaded)


@torch.inference_mode()
def append_documents(index_path: str, docs: list[torch.Tensor], batch_size: int, device: str,
                     loaded: dict[str, Any] | None = None) -> dict[str, Any] | None:
    """Encode with the codec on disk and append as new chunk(s) (update.rs:30-473).

    With `loaded` (device -> the DeviceIndex of the directory before this call), the new documents are also
    appended to each of those indexes (DeviceIndex.append) and the grown indexes are returned; the inverted file
    written to disk is then the one merged on the device, the same bytes a rebuild from the chunk files gives.  If
    an append fails the inverted file is rebuilt from the chunk files and None is returned."""
    meta = store.read_metadata(index_path)
    nbits = int(meta["nbits"])
    dev = torch.device(device)
    cent = torch.from_numpy(np.load(os.path.join(index_path, "centroids.npy"))).to(dev, torch.float16)
    cutoffs = torch.from_numpy(np.load(os.path.join(index_path, "bucket_cutoffs.npy"))).to(dev)
    dim = int(cent.shape[1])
    cent_t = cent.t().contiguous()
    n_chunks = int(meta["num_chunks"])
    emb_offset = int(meta["num_embeddings"])
    n_docs = int(meta["num_documents"])
    per_chunk = max(1, int(batch_size))
    new_codes: list[torch.Tensor] = []
    new_res: list[torch.Tensor] = []
    new_lens: list[int] = []
    for s in range(0, len(docs), per_chunk):
        chunk_docs = docs[s : s + per_chunk]
        lens = [int(d.shape[0]) for d in chunk_docs]
        flat = torch.cat([d.reshape(-1, dim).to(torch.float16) for d in chunk_docs]).to(dev)
        codes_parts, res_parts = [], []
        for r in range(0, flat.shape[0], max(1, batch_size)):
            c, rr = build.encode(flat[r : r + batch_size], cent, cent_t, cutoffs, nbits)
            codes_parts.append(c)
            res_parts.append(rr)
        codes = torch.cat(codes_parts) if codes_parts else torch.empty(0, dtype=torch.int64, device=dev)
        res = torch.cat(res_parts) if res_parts else torch.empty((0, dim * nbits // 8), dtype=torch.uint8, device=dev)
        store.write_chunk(index_path, n_chunks, codes, res, lens, emb_offset)
        if loaded is not None:
            new_codes.append(codes.to(torch.int32))
            new_res.append(res)
            new_lens.extend(lens)
        n_chunks += 1
        emb_offset += int(codes.shape[0])
        n_docs += len(lens)
    compress_only = bool(meta.get("compress_only", False))
    n_cells = int(meta.get("num_partitions", cent.shape[0]))
    grown = None
    if loaded is not None:
        codes = torch.cat(new_codes) if new_codes else torch.empty(0, dtype=torch.int32, device=dev)
        res = torch.cat(new_res) if new_res else torch.empty((0, dim * nbits // 8), dtype=torch.uint8, device=dev)
        lens_t = torch.tensor(new_lens, dtype=torch.int64)
        try:
            grown = {d: idx.append(codes, res, lens_t) for d, idx in loaded.items()}
        except Exception as e:
            print(f"Warning: appending in place failed, the index will be loaded again: {e}")
            grown = None
        del codes, res
    if not compress_only:
        if grown is not None:
            _write_merged_ivf(index_path, grown[device], n_cells)
        else:
            _rebuild_ivf(index_path, n_chunks, n_cells, dev)
    store.write_metadata(index_path, num_chunks=n_chunks, nbits=nbits, num_partitions=n_cells,
                         num_embeddings=emb_offset, num_documents=n_docs, compress_only=compress_only)
    return grown


def _write_merged_ivf(index_path: str, idx: Any, n_cells: int) -> None:
    """ivf.npy / ivf_lengths.npy of a DeviceIndex's inverted file, as build_ivf writes them: one length per cell up
    to max(n_cells, the last non-empty cell + 1)."""
    offs = idx.ivf_offsets.cpu()
    lengths = offs[1:] - offs[:-1]
    nz = torch.nonzero(lengths).flatten()
    n = max(n_cells, int(nz[-1]) + 1 if nz.numel() else 0)
    if n > lengths.shape[0]:
        lengths = torch.cat([lengths, torch.zeros(n - lengths.shape[0], dtype=lengths.dtype)])
    store.write_ivf(index_path, idx.ivf_pids[: int(offs[-1])], lengths[:n])


def _rebuild_ivf(index_path: str, n_chunks: int, n_cells: int, dev: torch.device) -> None:
    codes, lens = [], []
    for i in range(n_chunks):
        cp = os.path.join(index_path, f"{i}.codes.npy")
        if os.path.exists(cp):
            codes.append(torch.from_numpy(np.load(cp)))
    lens = store.read_doclens(index_path, n_chunks)
    all_codes = torch.cat(codes) if codes else torch.empty(0, dtype=torch.int64)
    ivf, ivf_lengths = build.build_ivf(all_codes.to(dev), torch.tensor(lens, dtype=torch.int64), n_cells)
    store.write_ivf(index_path, ivf, ivf_lengths)


@torch.inference_mode()
def delete_in_place(index_path: str, subset: list[int], device: str,
                    loaded: dict[str, Any]) -> dict[str, Any] | None:
    """What delete_from_index does, from the indexes already in HBM: `loaded` (device -> the DeviceIndex of the
    directory as it is on disk) are compacted first (DeviceIndex.delete), on every device, and the compacted indexes
    are returned.  Only then are files written, from the compacted arrays of `device`: every file of a chunk that
    loses a document, the ``{i}.metadata.json`` of every later chunk (its embedding offset moves), the inverted file
    and ``metadata.json``, last.  The directory ends byte for byte as delete_from_index leaves it, and chunks before
    the first dropped document are not touched.

    Returns None, having written nothing, when the delete would leave no document or the compaction fails: the
    caller then runs delete_from_index."""
    meta = store.read_metadata(index_path)
    if meta is None:
        raise RuntimeError("Failed to delete from index: metadata.json not found")
    n_chunks = int(meta["num_chunks"])
    chunks: list[tuple[int, list[int]]] = []  # (chunk, its document lengths) of every chunk delete_from_index reads
    for i in range(n_chunks):
        dl_path = os.path.join(index_path, f"doclens.{i}.json")
        if os.path.exists(dl_path):
            with open(dl_path) as f:
                chunks.append((i, json.load(f)))
    n_docs = sum(len(lens) for _, lens in chunks)
    drop = sorted({int(d) for d in subset if 0 <= int(d) < n_docs})
    compact = bool(meta.get("compress_only", False))
    if len(drop) == n_docs or any(idx.num_documents != n_docs or idx.has_ivf == compact for idx in loaded.values()):
        return None
    try:
        shrunk = {d: idx.delete(drop) for d, idx in loaded.items()}
    except Exception as e:
        print(f"Warning: deleting in place failed, the chunk files will be rewritten and the index loaded again: {e}")
        return None
    idx = shrunk[device]
    offsets = idx.doc_offsets.cpu()
    drop_t = torch.tensor(drop, dtype=torch.int64)
    doc_base = new_base = 0
    moved = False  # a document before this chunk was dropped: its embedding offset changes
    for i, lens in chunks:
        lo, hi = doc_base, doc_base + len(lens)
        gone = drop_t[(drop_t >= lo) & (drop_t < hi)] - lo
        n_kept = len(lens) - int(gone.shape[0])
        t0, t1 = int(offsets[new_base]), int(offsets[new_base + n_kept])
        if gone.numel():
            keep = torch.ones(len(lens), dtype=torch.bool)
            keep[gone] = False
            new_lens = torch.tensor(lens, dtype=torch.int64)[keep].tolist()
            store.write_chunk(index_path, i, idx.doc_codes[t0:t1], idx.doc_residuals[t0:t1], new_lens, t0)
            moved = True
        elif moved:
            store.write_chunk_metadata(index_path, i, len(lens), t1 - t0, t0)
        doc_base, new_base = hi, new_base + n_kept
    n_cells = int(meta.get("num_partitions", 1))
    if not compact:
        _write_merged_ivf(index_path, idx, n_cells)
    store.write_metadata(index_path, num_chunks=n_chunks, nbits=int(meta["nbits"]), num_partitions=n_cells,
                         num_embeddings=int(offsets[-1]), num_documents=idx.num_documents, compress_only=compact)
    return shrunk


@torch.inference_mode()
def delete_from_index(index_path: str, subset: list[int], device: str) -> None:
    """delete.rs:26-145: drop the documents, keep the chunk structure, rebuild the IVF."""
    meta = store.read_metadata(index_path)
    if meta is None:
        raise RuntimeError("Failed to delete from index: metadata.json not found")
    n_chunks = int(meta["num_chunks"])
    drop = set(int(i) for i in subset)
    doc_base = 0
    emb_offset = 0
    n_docs = 0
    for i in range(n_chunks):
        dl_path = os.path.join(index_path, f"doclens.{i}.json")
        if not os.path.exists(dl_path):
            continue
        with open(dl_path) as f:
            lens = json.load(f)
        codes = torch.from_numpy(np.load(os.path.join(index_path, f"{i}.codes.npy")))
        res = torch.from_numpy(np.load(os.path.join(index_path, f"{i}.residuals.npy")))
        keep_doc = torch.tensor([(doc_base + j) not in drop for j in range(len(lens))], dtype=torch.bool)
        lens_t = torch.tensor(lens, dtype=torch.int64)
        keep_tok = torch.repeat_interleave(keep_doc, lens_t)
        new_lens = lens_t[keep_doc].tolist()
        store.write_chunk(index_path, i, codes[keep_tok], res[keep_tok], new_lens, emb_offset)
        emb_offset += int(keep_tok.sum())
        n_docs += len(new_lens)
        doc_base += len(lens)
    compress_only = bool(meta.get("compress_only", False))
    if not compress_only:
        _rebuild_ivf(index_path, n_chunks, int(meta.get("num_partitions", 1)), torch.device(device))
    store.write_metadata(index_path, num_chunks=n_chunks, nbits=int(meta["nbits"]),
                         num_partitions=int(meta.get("num_partitions", 1)), num_embeddings=emb_offset,
                         num_documents=n_docs, compress_only=compress_only)
