"""On-disk index directory: reader and writer of the reference's layout.

Byte-compatible with what ``create_index`` writes (rust/index/create.rs:296-299, :380-397,
:476-491, :548-582) and what ``_load_index_tensors_cpu`` reads
(python/fast_plaid/search/load.py:220-322); the table is Appendix B of SURVEY.md.

The reader streams the ``{i}.codes.npy`` / ``{i}.residuals.npy`` chunks directly (it does not
need, and does not write, the reference's ``merged_*.npy`` mmap cache -- load.py:35-217 --
which exists there only because the Rust side wants one flat CPU tensor).
"""

from __future__ import annotations

import json
import os
import warnings

import numpy as np
import torch

from ..engine import IndexTensors


def _npy(path: str) -> np.ndarray:
    if not os.path.exists(path):
        raise FileNotFoundError(f"Missing index file: {path}")
    return np.load(path)


def read_metadata(index_path: str) -> dict | None:
    meta_path = os.path.join(index_path, "metadata.json")
    if not os.path.exists(meta_path):
        return None
    with open(meta_path) as f:
        return json.load(f)


def read_doclens(index_path: str, num_chunks: int) -> list[int]:
    lens: list[int] = []
    for i in range(num_chunks):
        p = os.path.join(index_path, f"doclens.{i}.json")
        if os.path.exists(p):  # load.py:289-294
            with open(p) as f:
                lens.extend(json.load(f))
    return lens


def read_index(index_path: str) -> IndexTensors | None:
    """Load an index directory into CPU tensors (codes stay int64 as on disk)."""
    meta = read_metadata(index_path)
    if meta is None:
        return None
    num_chunks = int(meta["num_chunks"])
    centroids = torch.from_numpy(_npy(os.path.join(index_path, "centroids.npy"))).to(torch.float16)
    weights = torch.from_numpy(_npy(os.path.join(index_path, "bucket_weights.npy"))).to(torch.float16)
    cut_p = os.path.join(index_path, "bucket_cutoffs.npy")
    avg_p = os.path.join(index_path, "avg_residual.npy")
    cutoffs = torch.from_numpy(np.load(cut_p)).to(torch.float16) if os.path.exists(cut_p) else None
    avg = torch.from_numpy(np.load(avg_p)).to(torch.float16) if os.path.exists(avg_p) else None
    ivf = ivf_lengths = None
    ivf_p = os.path.join(index_path, "ivf.npy")
    ivfl_p = os.path.join(index_path, "ivf_lengths.npy")
    if os.path.exists(ivf_p) and os.path.exists(ivfl_p):  # load.py:269-286 (absent => compress_only)
        ivf = torch.from_numpy(np.load(ivf_p)).to(torch.int64)
        ivf_lengths = torch.from_numpy(np.load(ivfl_p)).to(torch.int32)
    doclens = read_doclens(index_path, num_chunks)
    codes_parts, res_parts = [], []
    for i in range(num_chunks):
        cp = os.path.join(index_path, f"{i}.codes.npy")
        rp = os.path.join(index_path, f"{i}.residuals.npy")
        if os.path.exists(cp) and os.path.exists(rp):
            c = np.load(cp)
            if c.shape[0] > 0:
                codes_parts.append(torch.from_numpy(c))
                res_parts.append(torch.from_numpy(np.load(rp)))
    dim = int(centroids.shape[1])
    pd = dim * int(meta["nbits"]) // 8
    codes = torch.cat(codes_parts) if codes_parts else torch.empty(0, dtype=torch.int64)
    residuals = torch.cat(res_parts) if res_parts else torch.empty((0, pd), dtype=torch.uint8)
    return IndexTensors(
        nbits=int(meta["nbits"]),
        centroids=centroids,
        bucket_weights=weights,
        doc_lengths=torch.tensor(doclens, dtype=torch.int64),
        doc_codes=codes,
        doc_residuals=residuals,
        ivf=ivf,
        ivf_lengths=ivf_lengths,
        avg_residual=avg,
        bucket_cutoffs=cutoffs,
    )


def read_index_to_device(index_path: str, device: str | torch.device,
                         doc_range: tuple[int, int] | None = None) -> tuple[IndexTensors, int] | None:
    """Loader fast path (SURVEY.md 8(f)-2; replaces load.py:35-322 for a CUDA device): the big arrays go
    chunk file -> pinned staging -> HBM without ever existing as one host tensor.  Every ``{i}.codes.npy`` /
    ``{i}.residuals.npy`` is memory-mapped and only the rows of the documents in ``doc_range`` (a shard's
    contiguous document range; default: all) are read; the int64 codes are narrowed to int32 by the staging pass.
    A shard's inverted file is rebuilt on the GPU from its own codes (ids local to the shard) instead of filtering
    the global ``ivf.npy`` on the host.  Returns (tensors with the big arrays on `device`, doc_id_base)."""
    from ..engine import GrowableArrays, upload_narrow
    from .layout import build_ivf

    meta = read_metadata(index_path)
    if meta is None:
        return None
    dev = torch.device(device)
    num_chunks = int(meta["num_chunks"])
    nbits = int(meta["nbits"])
    centroids = torch.from_numpy(_npy(os.path.join(index_path, "centroids.npy"))).to(torch.float16)
    weights = torch.from_numpy(_npy(os.path.join(index_path, "bucket_weights.npy"))).to(torch.float16)
    dim = int(centroids.shape[1])
    pd = dim * nbits // 8
    chunk_lens: list[list[int]] = []
    for i in range(num_chunks):
        p = os.path.join(index_path, f"doclens.{i}.json")
        if os.path.exists(p):
            with open(p) as f:
                chunk_lens.append(json.load(f))
        else:
            chunk_lens.append([])
    all_lens = torch.tensor([x for c in chunk_lens for x in c], dtype=torch.int64)
    n_docs = int(all_lens.shape[0])
    lo, hi = (0, n_docs) if doc_range is None else (max(0, int(doc_range[0])), min(n_docs, int(doc_range[1])))
    offs = torch.zeros(n_docs + 1, dtype=torch.int64)
    offs[1:] = all_lens.cumsum(0)
    t0, t1 = int(offs[lo]), int(offs[hi])
    c0 = 0  # first token of the chunk in the whole index
    with torch.cuda.device(dev), warnings.catch_warnings():
        # codes and residuals go straight into growable buffers, which DeviceIndex adopts and appends grow in place
        arrays = GrowableArrays(dev, pd)
        views = arrays.views(max(hi - lo, 0), t1 - t0)
        codes, residuals = views["codes"][: max(t1 - t0, 0)], views["residuals"][: max(t1 - t0, 0)]
        warnings.simplefilter("ignore", UserWarning)  # read-only memory maps are only ever read here
        for i in range(num_chunks):
            n_tok = int(sum(chunk_lens[i]))
            a, b = max(c0, t0), min(c0 + n_tok, t1)
            if a < b:
                cm = np.load(os.path.join(index_path, f"{i}.codes.npy"), mmap_mode="r")
                rm = np.load(os.path.join(index_path, f"{i}.residuals.npy"), mmap_mode="r")
                upload_narrow(torch.from_numpy(cm[a - c0 : b - c0]), dev, torch.int32, out=codes[a - t0 : b - t0])
                upload_narrow(torch.from_numpy(rm[a - c0 : b - c0]), dev, torch.uint8, out=residuals[a - t0 : b - t0])
                del cm, rm
            c0 += n_tok
        ivf = ivf_lengths = None
        ivf_p = os.path.join(index_path, "ivf.npy")
        ivfl_p = os.path.join(index_path, "ivf_lengths.npy")
        if os.path.exists(ivf_p) and os.path.exists(ivfl_p):  # absent => compress_only
            if lo == 0 and hi == n_docs:
                ivf = upload_narrow(torch.from_numpy(np.load(ivf_p, mmap_mode="r")), dev, torch.int32)
                ivf_lengths = torch.from_numpy(np.load(ivfl_p)).to(torch.int32)
            else:
                n_cells = max(int(centroids.shape[0]), int(meta.get("num_partitions", 0)))
                ivf64, ivf_lengths = build_ivf(codes, all_lens[lo:hi], n_cells)
                ivf = ivf64.to(torch.int32)
                del ivf64
        torch.cuda.synchronize(dev)
    data = IndexTensors(nbits=nbits, centroids=centroids, bucket_weights=weights, doc_lengths=all_lens[lo:hi],
                        doc_codes=codes, doc_residuals=residuals, ivf=ivf, ivf_lengths=ivf_lengths, growable=arrays)
    return data, lo


def write_codec(index_path: str, centroids: torch.Tensor, cutoffs: torch.Tensor, weights: torch.Tensor,
                avg_residual: torch.Tensor, cluster_threshold: torch.Tensor) -> None:
    """create.rs:333-339, :380-397 (dtypes: centroids f16, the rest f32)."""
    np.save(os.path.join(index_path, "centroids.npy"), centroids.detach().cpu().to(torch.float16).numpy())
    np.save(os.path.join(index_path, "bucket_cutoffs.npy"), cutoffs.detach().cpu().float().numpy())
    np.save(os.path.join(index_path, "bucket_weights.npy"), weights.detach().cpu().float().numpy())
    np.save(os.path.join(index_path, "avg_residual.npy"), avg_residual.detach().cpu().float().numpy())
    np.save(os.path.join(index_path, "cluster_threshold.npy"), cluster_threshold.detach().cpu().float().numpy())


def write_chunk(index_path: str, chunk_index: int, codes: torch.Tensor, residuals: torch.Tensor,
                doclens: list[int], embedding_offset: int) -> None:
    """create.rs:476-491 and :503-523 (chunk metadata carries the global embedding offset)."""
    np.save(os.path.join(index_path, f"{chunk_index}.codes.npy"), codes.cpu().to(torch.int64).numpy())
    np.save(os.path.join(index_path, f"{chunk_index}.residuals.npy"), residuals.cpu().to(torch.uint8).numpy())
    with open(os.path.join(index_path, f"doclens.{chunk_index}.json"), "w") as f:
        json.dump([int(x) for x in doclens], f)
    write_chunk_metadata(index_path, chunk_index, len(doclens), int(codes.shape[0]), embedding_offset)


def write_chunk_metadata(index_path: str, chunk_index: int, num_documents: int, num_embeddings: int,
                         embedding_offset: int) -> None:
    """{i}.metadata.json of a chunk (create.rs:503-523)."""
    with open(os.path.join(index_path, f"{chunk_index}.metadata.json"), "w") as f:
        json.dump(
            {"num_documents": int(num_documents), "num_embeddings": int(num_embeddings),
             "embedding_offset": int(embedding_offset)},
            f, indent=2,
        )


def write_ivf(index_path: str, ivf: torch.Tensor, ivf_lengths: torch.Tensor) -> None:
    """create.rs:548-558 (ivf int64, lengths int32)."""
    np.save(os.path.join(index_path, "ivf.npy"), ivf.cpu().to(torch.int64).numpy())
    np.save(os.path.join(index_path, "ivf_lengths.npy"), ivf_lengths.cpu().to(torch.int32).numpy())


def write_plan(index_path: str, nbits: int, num_chunks: int) -> None:
    with open(os.path.join(index_path, "plan.json"), "w") as f:  # create.rs:296-299
        json.dump({"nbits": nbits, "num_chunks": num_chunks}, f, indent=2)
        f.write("\n")


def write_metadata(index_path: str, *, num_chunks: int, nbits: int, num_partitions: int, num_embeddings: int,
                   num_documents: int, compress_only: bool) -> None:
    """create.rs:561-582."""
    avg = (num_embeddings / num_documents) if num_documents > 0 else 0.0
    with open(os.path.join(index_path, "metadata.json"), "w") as f:
        json.dump(
            {"num_chunks": num_chunks, "nbits": nbits, "num_partitions": num_partitions,
             "num_embeddings": num_embeddings, "avg_doclen": avg, "num_documents": num_documents,
             "compress_only": compress_only},
            f, indent=2,
        )
