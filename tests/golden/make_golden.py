"""Mint the golden fixtures under tests/golden/ from the CPU oracle.

    python tests/golden/make_golden.py
    python tests/golden/make_golden.py --add-variant [OUT_DIR]

PARITY UNPINNED: the reference ships no golden vectors and is not built by this project
(Rust), so these vectors come from oracle/plaid_oracle.py -- the op-for-op PyTorch-CPU
restatement of rust/search/search.rs run on torch 2.11.0 (the version the reference's CI
pins).  They freeze the oracle's behaviour so that (a) a torch upgrade that changes an ATen
CPU kernel is noticed, and (b) the GPU tests compare against committed numbers, not only
against a live oracle.

ATen's fp16 CPU matmul (the centroid scores S) is not bit-identical across host CPUs: its fp32
accumulation order follows the GEMM kernel the host gets, and one fp16 ulp of S moves an
approximate score.  `expected_variants` therefore holds the oracle's complete outputs as minted
on each host family seen so far; `--add-variant` recomputes them from the stored index and
queries on this machine and appends them when they are new (to the fixtures in place, or to
copies under OUT_DIR).
"""

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from util import build_oracle_index, make_docs, make_queries  # noqa: E402

from oracle import plaid_oracle as po  # noqa: E402


def run_queries(oidx, queries, n_probe, n_full, top_k):
    per_query = []
    for b in range(queries.shape[0]):
        st = po.search_one(queries[b], oidx, n_probe, 2000, n_full, top_k, ties="canonical", return_stages=True)
        per_query.append({
            "cells": st["cells"], "candidates": st["candidates"], "approx": st["approx"],
            "rerank": st["rerank"], "exact": st["exact"], "ids": st["ids"], "scores": st["scores"],
            "S_checksum": float(st["S"].float().sum()),
        })
    return per_query


def load_index(blob) -> po.OracleIndex:
    ix = blob["index"]
    return po.OracleIndex(nbits=ix["nbits"], centroids=ix["centroids"], bucket_weights=ix["bucket_weights"],
                          ivf=ix["ivf"].long(), ivf_lengths=ix["ivf_lengths"].long(), doc_codes=ix["doc_codes"].long(),
                          doc_residuals=ix["doc_residuals"], doc_lengths=ix["doc_lengths"].long())


STAGES = ("cells", "candidates", "approx", "rerank", "exact")


def same_outputs(got: list, exp: list) -> bool:
    """Bit-identical stages, ids and scores for every query."""
    return len(got) == len(exp) and all(
        all(torch.equal(g[k], e[k]) for k in STAGES) and g["ids"] == e["ids"] and g["scores"] == e["scores"]
        for g, e in zip(got, exp))


def add_variant(out_dir: str) -> None:
    os.makedirs(out_dir, exist_ok=True)
    for name in ("small_d128_n4", "small_d64_n2"):
        blob = torch.load(os.path.join(HERE, f"{name}.pt"), weights_only=False)
        m = blob["meta"]
        got = run_queries(load_index(blob), blob["queries"], m["n_probe"], m["n_full"], m["top_k"])
        variants = blob.setdefault("expected_variants", [])
        if not any(same_outputs(got, v) for v in variants):
            variants.append(got)
        torch.save(blob, os.path.join(out_dir, f"{name}.pt"))
        print(name, len(variants), "variant(s)")


def make(name, n_docs, lo, hi, dim, nbits, B, Q, top_k, n_full, n_probe, noisy):
    docs = make_docs(n_docs, lo, hi, dim=dim, seed=2024)
    oidx, extra = build_oracle_index(docs, nbits=nbits, seed=42)
    queries = make_queries(B, Q, dim=dim, seed=99, docs=docs if noisy else None)
    per_query = run_queries(oidx, queries, n_probe, n_full, top_k)
    blob = {
        "meta": dict(name=name, torch=torch.__version__, n_docs=n_docs, dim=dim, nbits=nbits, B=B, Q=Q,
                     top_k=top_k, n_full=n_full, n_probe=n_probe),
        "index": dict(nbits=nbits, centroids=oidx.centroids, bucket_weights=oidx.bucket_weights, ivf=oidx.ivf.to(torch.int32),
                      ivf_lengths=oidx.ivf_lengths.to(torch.int32), doc_codes=oidx.doc_codes.to(torch.int32),
                      doc_residuals=oidx.doc_residuals, doc_lengths=oidx.doc_lengths.to(torch.int32)),
        "queries": queries.half(),
        "expected": per_query,
        "expected_variants": [per_query],
    }
    path = os.path.join(HERE, f"{name}.pt")
    torch.save(blob, path)
    print(name, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__" and sys.argv[1:2] == ["--add-variant"]:
    add_variant(sys.argv[2] if len(sys.argv) > 2 else HERE)
elif __name__ == "__main__":
    make("small_d128_n4", 150, 10, 60, 128, 4, 4, 32, 10, 64, 8, True)
    make("small_d64_n2", 120, 5, 40, 64, 2, 3, 20, 5, 32, 4, True)
