"""CPU oracle for index construction (defines the bytes the search path reads).
TEST INFRASTRUCTURE ONLY -- see the header of ``plaid_oracle.py`` for the import rules.

Restates, op for op in PyTorch-CPU, ``create_index`` (rust/index/create.rs:206-585) for a
given centroid table, plus the K heuristic and normalisation of ``compute_kmeans``
(python/fast_plaid/search/fast_plaid.py:71-185) with a plain Lloyd k-means standing in
for the third-party ``fastkmeans==0.5.0`` dependency (pyproject.toml:30; not part of the
fast-plaid source tree).  The in-tree chunked Lloyd loop that the reference
layers on it (python/fast_plaid/search/kmeans.py:60-223) is what ``kmeans`` follows.

Two things cannot be reproduced bit-for-bit and are documented instead:
  * the held-out sample is drawn with Rust's ``StdRng`` shuffle (create.rs:225-233); here
    a seeded ``torch.randperm`` draws it, so cutoffs/weights differ from a reference run
    with the same seed (the algorithm is the same);
  * k-means initialisation uses torch's global RNG after ``torch.manual_seed(seed)``
    (kmeans.py:236, :131) -- reproduced the same way.
"""

from __future__ import annotations

import math

import torch

from .plaid_oracle import OracleIndex


def scalar_quantile_kthvalue(t: torch.Tensor, q: float) -> torch.Tensor:
    """rust/search/tensor.rs:18-34"""
    n = t.shape[0]
    idx = q * (n - 1)
    lo, hi = math.floor(idx), math.ceil(idx)
    if lo == hi:
        return t.kthvalue(lo + 1, 0, True).values
    lv = t.kthvalue(lo + 1, 0, True).values
    hv = t.kthvalue(hi + 1, 0, True).values
    return torch.lerp(lv, hv, idx - lo)


def compress_into_codes(emb: torch.Tensor, centroids: torch.Tensor) -> torch.Tensor:
    """rust/index/create.rs:148-170 (2048-row chunks, argmax over K)."""
    ct = centroids.transpose(0, 1)
    out = []
    for s in range(0, emb.shape[0], 2048):
        out.append(emb[s : s + 2048].matmul(ct).argmax(1))
    return torch.cat(out, 0) if out else torch.empty(0, dtype=torch.int64)


def packbits(bits: torch.Tensor) -> torch.Tensor:
    """rust/index/create.rs:176-184 (big-endian within a byte, via an fp16 matmul)."""
    m = bits.reshape(-1, 8).to(torch.float16)
    w = torch.tensor([128, 64, 32, 16, 8, 4, 2, 1], dtype=torch.float16)
    return m.matmul(w).to(torch.uint8)


def num_partitions_for(n_embeddings: float) -> int:
    """fast_plaid.py:152-154 / create.rs:292-294:  2**floor(log2(16*sqrt(E)))."""
    return int(2 ** math.floor(math.log2(16 * math.sqrt(n_embeddings))))


def kmeans(data: torch.Tensor, k: int, niters: int, seed: int, max_points_per_centroid: int = 256) -> torch.Tensor:
    """Lloyd iterations as in kmeans.py:60-223 (CPU => fp32 compute, kmeans.py:113-114)."""
    torch.manual_seed(seed)  # kmeans.py:236
    dn = (data**2).sum(1)  # kmeans.py:241: squared norms in the data's own dtype (fp16 from compute_kmeans)
    n = data.shape[0]
    if max_points_per_centroid is not None and n > k * max_points_per_centroid:  # :119-126
        sel = torch.randperm(n)[: k * max_points_per_centroid]
        data, dn = data[sel], dn[sel]
        n = data.shape[0]
    if n < k:
        raise ValueError(f"Number of training points ({n}) is less than k ({k}).")
    data, dn = data.float(), dn.float()  # CPU => fp32 compute (:113-114, :148-153)
    centroids = data[torch.randperm(n)[:k]].clone()  # :133-134
    for _ in range(niters):
        cn = (centroids**2).sum(1)
        best = torch.empty(n, dtype=torch.int64)
        for s in range(0, n, 51_200):  # :144
            chunk = data[s : s + 51_200]
            dist = dn[s : s + 51_200, None] + cn[None, :]
            dist = dist.addmm_(chunk, centroids.t(), alpha=-2.0, beta=1.0)  # :175-180
            best[s : s + 51_200] = dist.argmin(1)
        sums = torch.zeros_like(centroids).index_add_(0, best, data)  # :189
        counts = torch.zeros(k).index_add_(0, best, torch.ones(n))
        new = torch.zeros_like(centroids)
        ne = counts > 0
        new[ne] = sums[ne] / counts[ne, None]  # :199-203
        empty = (~ne).nonzero(as_tuple=True)[0]
        if len(empty) > 0:  # :205-213
            new[empty] = data[torch.randint(0, n, (len(empty),))]
        shift = torch.norm(new - centroids, dim=1).sum().item()
        centroids = new
        if shift < 1e-8:
            break
    return centroids


def compute_centroids(docs: list[torch.Tensor], kmeans_niters: int = 4, seed: int = 42,
                      max_points_per_centroid: int = 256) -> torch.Tensor:
    """compute_kmeans (fast_plaid.py:71-185): sample docs, K heuristic, normalise, fp16."""
    n_docs = len(docs)
    n_samples = min(1 + int(16 * math.sqrt(120 * n_docs)), n_docs)  # :109-115
    g = torch.Generator().manual_seed(seed)
    idx = torch.randperm(n_docs, generator=g)[:n_samples].tolist()  # :118
    samples = torch.cat([docs[i].to(torch.float16) for i in idx], 0)  # :130-142
    total = samples.shape[0]
    k = num_partitions_for(total / n_samples * n_docs)  # :150-154
    k = min(k, total)  # :160
    c = kmeans(samples, k, kmeans_niters, seed, max_points_per_centroid)
    return torch.nn.functional.normalize(c, dim=-1).half()  # :182-185


def build_index(
    docs: list[torch.Tensor],
    centroids: torch.Tensor,
    nbits: int = 4,
    batch_size: int = 25_000,
    seed: int = 42,
) -> tuple[OracleIndex, dict]:
    """create_index (create.rs:206-585) without the file writes.  Returns the in-memory
    index plus the extra codec tensors that go to disk (cutoffs, avg_residual, threshold)."""
    n_docs = len(docs)
    dim = centroids.shape[1]
    centroids = centroids.to(torch.float16)  # lib.rs:148
    sample_count = int(min(1.0 + 16.0 * math.sqrt(120.0 * n_docs), n_docs))  # :222-223
    g = torch.Generator().manual_seed(seed)
    sample_pids = torch.randperm(n_docs, generator=g)[:sample_count].tolist()  # :231-233 (own RNG)
    total_samples = sum(docs[p].shape[0] for p in sample_pids)
    heldout_size = int(round(min(0.05 * total_samples, 50_000.0)))  # :255
    held: list[torch.Tensor] = []
    have = 0
    for p in reversed(sample_pids):  # :260-282
        need = heldout_size - have
        if need <= 0:
            break
        t = docs[p].to(torch.float16)
        if t.shape[0] <= need:
            held.append(t)
            have += t.shape[0]
        else:
            held.append(t[t.shape[0] - need :])
            have += need
    held.reverse()
    heldout = torch.cat(held, 0)
    if heldout.shape[0] == 0:
        raise RuntimeError("Cannot train codec: no heldout samples were generated.")  # :301-305
    avg_doc_len = sum(d.shape[0] for d in docs) / n_docs
    est_k = num_partitions_for(n_docs * avg_doc_len)  # :292-294

    codes = compress_into_codes(heldout, centroids)  # :317
    res = (heldout - centroids.index_select(0, codes)).float()  # :326-327
    threshold = scalar_quantile_kthvalue(res.norm(2, dim=1), 0.75)  # :333-334
    avg_res = res.abs().mean(0)  # :341-344
    n_opt = 2**nbits
    flat = res.flatten()
    cutoffs = torch.cat([scalar_quantile_kthvalue(flat, i / n_opt) for i in range(1, n_opt)])  # :352-357
    weights = torch.cat([scalar_quantile_kthvalue(flat, (i + 0.5) / n_opt) for i in range(n_opt)])  # :359-364

    bit_helper = torch.arange(0, nbits, dtype=torch.int8)  # residual_codec.rs:80
    all_codes, all_res, doclens = [], [], []
    acc, rows = [], 0

    def process(batch: torch.Tensor) -> None:  # :404-428
        c = compress_into_codes(batch, centroids)
        r = batch - centroids.index_select(0, c)
        b = torch.bucketize(r, cutoffs, out_int32=True, right=False)  # :414 (tch arg order: out_int32, right)
        b = b.unsqueeze(-1).expand(*b.shape, nbits)
        b = b.bitwise_right_shift(bit_helper)
        b = b.bitwise_and(torch.ones_like(b))
        packed = packbits(b.flatten())
        all_codes.append(c)
        all_res.append(packed.reshape(batch.shape[0], dim // 8 * nbits))

    for dtensor in docs:  # :441-471 (chunk boundaries do not change bytes)
        doclens.append(dtensor.shape[0])
        acc.append(dtensor.to(torch.float16))
        rows += dtensor.shape[0]
        if rows >= batch_size:
            process(torch.cat(acc, 0))
            acc, rows = [], 0
    if acc:
        process(torch.cat(acc, 0))
    codes_all = torch.cat(all_codes, 0)
    res_all = torch.cat(all_res, 0)
    doc_lengths = torch.tensor(doclens, dtype=torch.int64)

    # global IVF, create.rs:528-559 + optimize_ivf :55-132
    sorted_codes, sorted_idx = codes_all.sort(0, False)
    counts = torch.bincount(sorted_codes, minlength=est_k)
    emb2pid = torch.repeat_interleave(torch.arange(n_docs, dtype=torch.int64), doc_lengths)
    pids = emb2pid.index_select(0, sorted_idx)
    ivf_parts, ivf_lens = [], []
    off = 0
    for ln in counts.tolist():
        u = torch.unique(pids[off : off + ln], sorted=True)
        ivf_parts.append(u)
        ivf_lens.append(u.shape[0])
        off += ln
    ivf = torch.cat(ivf_parts, 0) if ivf_parts else torch.empty(0, dtype=torch.int64)
    ivf_lengths = torch.tensor(ivf_lens, dtype=torch.int32)

    idx = OracleIndex(
        nbits=nbits,
        centroids=centroids,
        bucket_weights=weights,
        ivf=ivf,
        ivf_lengths=ivf_lengths,
        doc_codes=codes_all,
        doc_residuals=res_all,
        doc_lengths=doc_lengths,
    )
    extra = {
        "bucket_cutoffs": cutoffs,  # f32, create.rs:385-388
        "bucket_weights": weights,  # f32, create.rs:389-392
        "avg_residual": avg_res,  # f32, create.rs:393-397
        "cluster_threshold": threshold,  # create.rs:333-339
        "num_partitions": est_k,
    }
    return idx, extra
