"""Index construction (host orchestration in PyTorch; SURVEY.md 8(f-1) "next" row).

Same algorithm and on-disk result as the reference's ``compute_kmeans`` + ``create_index``
(python/fast_plaid/search/fast_plaid.py:71-185, rust/index/create.rs:206-585):

  1. k-means centroids on a document sample, K = 2^floor(log2(16*sqrt(#tokens)))
  2. codec: 5% held-out residuals -> 2^nbits-1 quantile cutoffs, 2^nbits quantile weights
  3. per chunk of `batch_size` docs: code = argmax_k <x, c_k>, residual buckets, bit packing
  4. inverted file: per centroid, sorted unique doc ids

This module is not on the search hot path; it runs on whichever torch device it is given
(CUDA on the GPU, CPU in the non-GPU tests) with dense torch ops.  The encode step
(argmax GEMM + bucketize + pack) runs in the sm_90a kernels behind `fpb_encode`
(csrc/encode.cu) when the tokens are on CUDA with dim=128; elsewhere it is dense torch ops.
"""

from __future__ import annotations

import math
import os

import torch

from . import store
from .layout import build_ivf, num_partitions_for  # noqa: F401  (re-exported)


def _quantile_kth(t: torch.Tensor, q: float) -> torch.Tensor:
    """kthvalue-based quantile with linear interpolation (rust/search/tensor.rs:18-34)."""
    n = t.shape[0]
    pos = q * (n - 1)
    lo, hi = math.floor(pos), math.ceil(pos)
    lv = t.kthvalue(lo + 1, 0, True).values
    if lo == hi:
        return lv
    hv = t.kthvalue(hi + 1, 0, True).values
    return torch.lerp(lv, hv, pos - lo)


@torch.inference_mode()
def lloyd_kmeans(data: torch.Tensor, k: int, niters: int, seed: int, device: torch.device,
                 max_points_per_centroid: int | None = 256, chunk: int = 51_200) -> torch.Tensor:
    """Chunked Lloyd iterations (python/fast_plaid/search/kmeans.py:60-223): random init from
    the data, nearest centroid by ||x||^2 + ||c||^2 - 2<x,c>, mean update, empty clusters
    re-seeded from random points.  fp16 on CUDA, fp32 on CPU (kmeans.py:113-114)."""
    torch.manual_seed(seed)  # kmeans.py:236-238
    n = data.shape[0]
    if max_points_per_centroid is not None and n > k * max_points_per_centroid:
        data = data[torch.randperm(n)[: k * max_points_per_centroid].to(data.device)]
        n = data.shape[0]
    if n < k:
        raise ValueError(f"Number of training points ({n}) is less than k ({k}).")
    dtype = torch.float16 if device.type == "cuda" else torch.float32
    centroids = data[torch.randperm(n)[:k].to(data.device)].to(device=device, dtype=dtype).clone()
    if device.type == "cuda" and data.shape[1] == 128:
        return _lloyd_kmeans_b200(data, centroids, niters, n, device)
    data_norms = (data.float() ** 2).sum(1)
    for _ in range(niters):
        cnorm = (centroids**2).sum(1)
        sums = torch.zeros((k, data.shape[1]), device=device, dtype=torch.float32)
        counts = torch.zeros((k,), device=device, dtype=torch.float32)
        for s in range(0, n, chunk):
            x = data[s : s + chunk].to(device=device, dtype=dtype)
            xn = data_norms[s : s + chunk].to(device=device, dtype=dtype)
            best_d = torch.full((x.shape[0],), float("inf"), device=device, dtype=dtype)
            best = torch.zeros((x.shape[0],), device=device, dtype=torch.int64)
            for c0 in range(0, k, 10_240):
                cc = centroids[c0 : c0 + 10_240]
                dist = xn[:, None] + cnorm[None, c0 : c0 + 10_240]
                dist = dist.addmm_(x, cc.t(), alpha=-2.0, beta=1.0)
                dmin, imin = dist.min(1)
                better = dmin < best_d
                best_d[better] = dmin[better]
                best[better] = c0 + imin[better]
            sums.index_add_(0, best, x.float())
            counts.index_add_(0, best, torch.ones_like(best, dtype=torch.float32))
        new = torch.zeros_like(centroids)
        ne = counts > 0
        new[ne] = (sums[ne] / counts[ne, None]).to(dtype)
        empty = (~ne).nonzero(as_tuple=True)[0]
        if len(empty) > 0:
            new[empty] = data[torch.randint(0, n, (len(empty),))].to(device=device, dtype=dtype)
        shift = torch.norm(new.float() - centroids.float(), dim=1).sum().item()
        centroids = new
        if shift < 1e-8:
            break
    return centroids.float().cpu()


def _lloyd_kmeans_b200(data: torch.Tensor, centroids: torch.Tensor, niters: int, n: int,
                       device: torch.device, chunk: int = 4_000_000) -> torch.Tensor:
    """The same Lloyd iterations on the sm_90a kernels (csrc/encode.cu): the assignment is the wgmma argmax
    GEMM with a -|c|^2/2 bias in the epilogue (fpb_kmeans_assign), the update a deterministic segmented mean
    (fpb_kmeans_update); empty clusters are re-seeded from random points and the loop stops on a zero shift, as
    kmeans.py:196-218 does.  The points are staged to the GPU in `chunk`-row pieces when they live on the host."""
    from ..engine import kmeans_assign, kmeans_update

    on_gpu = data.is_cuda
    pts = data.to(device=device, dtype=torch.float16) if (on_gpu or n <= chunk) else None
    for _ in range(niters):
        if pts is not None:
            assign = kmeans_assign(pts, centroids)
            counts, shift = kmeans_update(pts, assign, centroids)
        else:  # host-resident sample larger than one staging chunk: assign chunk by chunk, one update at the end
            parts = [kmeans_assign(data[s : s + chunk].to(device=device, dtype=torch.float16), centroids)
                     for s in range(0, n, chunk)]
            assign = torch.cat(parts)
            counts, shift = kmeans_update(data.to(device=device, dtype=torch.float16), assign, centroids)
        empty = (counts == 0).nonzero(as_tuple=True)[0]
        moved = float(shift.sum())
        if len(empty) > 0:
            old = centroids[empty].float()
            centroids[empty] = data[torch.randint(0, n, (len(empty),)).to(data.device)].to(device=device, dtype=torch.float16)
            moved += float(torch.norm(centroids[empty].float() - old, dim=1).sum())
        if moved < 1e-8:
            break
    return centroids.float().cpu()


@torch.inference_mode()
def compute_kmeans(documents_embeddings: list[torch.Tensor] | torch.Tensor, dim: int, device: str,
                   kmeans_niters: int, max_points_per_centroid: int, seed: int,
                   n_samples_kmeans: int | None = None, num_partitions: int | None = None) -> torch.Tensor:
    """Same contract as the reference's ``compute_kmeans`` (fast_plaid.py:71-185): returns
    L2-normalised fp16 centroids on ``device``."""
    n_docs = len(documents_embeddings)
    if n_samples_kmeans is None:
        n_samples_kmeans = min(1 + int(16 * math.sqrt(120 * n_docs)), n_docs)
    n_samples_kmeans = min(n_docs, n_samples_kmeans)
    idx = torch.randperm(n_docs)[:n_samples_kmeans]
    dev = torch.device(device)
    if isinstance(documents_embeddings, torch.Tensor):
        samples = documents_embeddings[idx].reshape(-1, dim)
    else:
        # the sampled documents stay where they live: on the host for host documents, in HBM for CUDA documents
        # (visited in ascending order so that a lazy, block-generated corpus produces each block once)
        order = sorted(idx.tolist())
        first = documents_embeddings[order[0]]
        keep = first.device if first.is_cuda else torch.device("cpu")
        samples = torch.cat([documents_embeddings[i].reshape(-1, dim).to(keep, torch.float16) for i in order])
    total = samples.shape[0]
    if num_partitions is None:
        num_partitions = num_partitions_for(total / n_samples_kmeans * n_docs)
    k = min(num_partitions, total)
    cent = lloyd_kmeans(samples, k, kmeans_niters, seed, dev, max_points_per_centroid)
    return torch.nn.functional.normalize(cent.to(dev), dim=-1).half()


def assign_codes(emb: torch.Tensor, centroids_t: torch.Tensor, rows: int = 2048) -> torch.Tensor:
    """argmax_k <x, c_k> in row chunks (create.rs:148-170)."""
    out = [emb[s : s + rows].matmul(centroids_t).argmax(1) for s in range(0, emb.shape[0], rows)]
    return torch.cat(out) if out else torch.empty(0, dtype=torch.int64, device=emb.device)


def pack_buckets(buckets: torch.Tensor, nbits: int) -> torch.Tensor:
    """[n, dim] bucket indices -> [n, dim*nbits/8] bytes.  Each index is written LSB-first
    into `nbits` consecutive bits and the bit stream is packed big-endian per byte
    (create.rs:413-427 + packbits :176-184)."""
    n, dim = buckets.shape
    shifts = torch.arange(nbits, device=buckets.device, dtype=torch.int32)
    bits = (buckets.to(torch.int32).unsqueeze(-1) >> shifts) & 1  # [n, dim, nbits]
    bits = bits.reshape(n, dim * nbits // 8, 8)
    w = torch.tensor([128, 64, 32, 16, 8, 4, 2, 1], device=buckets.device, dtype=torch.int32)
    return (bits * w).sum(-1).to(torch.uint8)


@torch.inference_mode()
def train_codec(docs: list[torch.Tensor], centroids: torch.Tensor, nbits: int, seed: int | None,
                device: torch.device) -> dict[str, torch.Tensor]:
    """Held-out residual statistics (create.rs:221-364)."""
    n_docs = len(docs)
    sample_count = int(min(1.0 + 16.0 * math.sqrt(120.0 * n_docs), n_docs))
    g = torch.Generator()
    if seed is not None:
        g.manual_seed(int(seed))
    sample_pids = torch.randperm(n_docs, generator=g)[:sample_count].tolist()
    known = getattr(docs, "doc_lengths", None)
    total = sum(int(known[p]) if known is not None else int(docs[p].shape[0]) for p in sample_pids)
    heldout_size = int(round(min(0.05 * total, 50_000.0)))
    parts: list[torch.Tensor] = []
    have = 0
    for p in reversed(sample_pids):
        need = heldout_size - have
        if need <= 0:
            break
        t = docs[p].to(torch.float16)
        take = t if t.shape[0] <= need else t[t.shape[0] - need :]
        parts.append(take)
        have += take.shape[0]
    parts.reverse()
    if not parts or have == 0:
        raise RuntimeError("Failed to create index: Cannot train codec: no heldout samples were generated.")
    held = torch.cat(parts).to(device)
    cent = centroids.to(device, torch.float16)
    codes = assign_codes(held, cent.t())
    res = (held - cent.index_select(0, codes)).float()
    threshold = _quantile_kth(res.norm(2, dim=1), 0.75)
    avg = res.abs().mean(0)
    flat = res.flatten()
    n_opt = 2**nbits
    cutoffs = torch.cat([_quantile_kth(flat, i / n_opt) for i in range(1, n_opt)])
    weights = torch.cat([_quantile_kth(flat, (i + 0.5) / n_opt) for i in range(n_opt)])
    return {"bucket_cutoffs": cutoffs, "bucket_weights": weights, "avg_residual": avg, "cluster_threshold": threshold}


@torch.inference_mode()
def encode(batch: torch.Tensor, centroids: torch.Tensor, centroids_t: torch.Tensor, cutoffs: torch.Tensor,
           nbits: int) -> tuple[torch.Tensor, torch.Tensor]:
    """One batch of fp16 token rows -> (codes int64, packed residual bytes) (create.rs:404-428).
    On a CUDA device with dim = 128 this is the sm_90a encode kernel pair (wgmma argmax GEMM +
    bucketize/pack, csrc/encode.cu); otherwise dense torch ops."""
    if batch.is_cuda and batch.shape[1] == 128 and nbits in (1, 2, 4):
        from ..engine import encode_tokens

        codes32, packed = encode_tokens(batch, centroids, cutoffs, nbits)
        return codes32.to(torch.int64), packed
    codes = assign_codes(batch, centroids_t)
    res = batch - centroids.index_select(0, codes)
    buckets = torch.bucketize(res, cutoffs, out_int32=True, right=False)
    return codes, pack_buckets(buckets, nbits)


@torch.inference_mode()
@torch.inference_mode()
def create_index(docs: list[torch.Tensor], index_path: str, centroids: torch.Tensor, nbits: int = 4,
                 batch_size: int = 25_000, seed: int | None = 42, compress_only: bool = False,
                 device: str = "cpu") -> None:
    """Write a complete index directory (create.rs:206-585)."""
    dev = torch.device(device)
    n_docs = len(docs)
    dim = int(centroids.shape[1])
    os.makedirs(index_path, exist_ok=True)
    docs_per_chunk = int(min(batch_size, 1 + n_docs))  # create.rs:400
    n_chunks = int(math.ceil(n_docs / min(float(batch_size), 1.0 + n_docs)))  # create.rs:218
    known = getattr(docs, "doc_lengths", None)  # a lazy document sequence knows its lengths without generating data
    total_tokens = int(known.sum()) if known is not None else sum(int(d.shape[0]) for d in docs)
    est_k = num_partitions_for(float(total_tokens))  # create.rs:292-294
    store.write_plan(index_path, nbits, n_chunks)
    codec = train_codec(docs, centroids, nbits, seed, dev)
    cent = centroids.to(dev, torch.float16)
    store.write_codec(index_path, cent, codec["bucket_cutoffs"], codec["bucket_weights"], codec["avg_residual"],
                      codec["cluster_threshold"])
    cent_t = cent.t().contiguous()
    cutoffs = codec["bucket_cutoffs"].to(dev)
    all_codes: list[torch.Tensor] = []
    all_lens: list[int] = []
    emb_offset = 0
    # streaming: one chunk of `docs_per_chunk` documents is resident at a time (the documents may be a lazy sequence)
    for ci in range(n_chunks):
        d_lo, d_hi = ci * docs_per_chunk, min(n_docs, (ci + 1) * docs_per_chunk)
        lens: list[int] = []
        codes_parts, res_parts = [], []
        acc: list[torch.Tensor] = []
        rows = 0
        for di in range(d_lo, d_hi):
            d = docs[di]
            lens.append(int(d.shape[0]))
            acc.append(d.reshape(-1, dim).to(torch.float16))
            rows += int(d.shape[0])
            if rows >= batch_size:
                c, r = encode(torch.cat(acc).to(dev), cent, cent_t, cutoffs, nbits)
                codes_parts.append(c.cpu())
                res_parts.append(r.cpu())
                acc, rows = [], 0
        if acc:
            c, r = encode(torch.cat(acc).to(dev), cent, cent_t, cutoffs, nbits)
            codes_parts.append(c.cpu())
            res_parts.append(r.cpu())
        codes = torch.cat(codes_parts) if codes_parts else torch.empty(0, dtype=torch.int64)
        res = torch.cat(res_parts) if res_parts else torch.empty((0, dim * nbits // 8), dtype=torch.uint8)
        store.write_chunk(index_path, ci, codes, res, lens, emb_offset)
        emb_offset += int(codes.shape[0])
        all_codes.append(codes)
        all_lens.extend(lens)
    if not compress_only:
        codes_all = torch.cat(all_codes) if all_codes else torch.empty(0, dtype=torch.int64)
        ivf, ivf_lengths = build_ivf(codes_all.to(dev), torch.tensor(all_lens, dtype=torch.int64), est_k)
        store.write_ivf(index_path, ivf, ivf_lengths)
    store.write_metadata(index_path, num_chunks=n_chunks, nbits=nbits, num_partitions=est_k,
                         num_embeddings=emb_offset, num_documents=n_docs, compress_only=compress_only)
