"""Exhaustive exact search over document subsets on the benchmark's synthetic indexes: one JSON line per run.

    python tools/bench_exhaustive_subset.py --config cfg3 [--seconds 1.0] [--warmup 2]

Two workloads, each timed as the raw fpb_search_exhaustive_subset call with CUDA events over at least --seconds of
work after warm-up:

* filtered: one random subset of 1 / 10 / 50 / 100 % of the documents shared by the whole batch (the result of a
  metadata filter), against the full scan (fpb_search_exhaustive) timed in the same run;
* rerank: a distinct random list of 100 / 1 000 / 4 096 documents per query (exact re-ranking of first-stage
  candidates), against search() (default parameters) on the same batch.

Every timed result is checked against the full scan's scores of the same batch: the number of returned scores that
differ from the full scan's score of the same document (and of wrong counts) is reported and must be 0.  Needs a
CUDA device; there is no fallback.
"""

from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from bench_exhaustive import PEAK_TFLOPS, card, timed  # noqa: E402  (tools/ is the script's directory)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg3", choices=["cfg2", "cfg3", "tiny"])
    ap.add_argument("--workload", default="both", choices=["filtered", "rerank", "both"])
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_exhaustive_subset.py needs a CUDA device (the engine has no CPU path)")
    from fast_plaid_b200.engine import DeviceIndex, IndexTensors, _check

    cfg = bench.CONFIGS[args.config]
    device = "cuda:0"
    n_docs, B, Q, k = cfg["n_docs"], cfg["B"], cfg["Q"], cfg["top_k"]
    synth = bench.load_synthetic_module()
    arrays, base = synth.synthetic_arrays(n_docs, cfg["doc_len"], bench.DIM, bench.NBITS, device, bench.SEED_INDEX,
                                          doc_range=(0, n_docs), topics=cfg.get("topics", 0), mix=cfg.get("mix", 0.05))
    data = IndexTensors(nbits=arrays.nbits, centroids=arrays.centroids, bucket_weights=arrays.bucket_weights,
                        doc_lengths=arrays.doc_lengths, doc_codes=arrays.doc_codes,
                        doc_residuals=arrays.doc_residuals, ivf=arrays.ivf, ivf_lengths=arrays.ivf_lengths)
    didx = DeviceIndex(data, device, doc_id_base=base)
    q = bench.make_query_batches(arrays, bench.query_source_docs(n_docs), cfg, 1)[0]
    del data, arrays
    q16 = q.to(device).half().contiguous()
    doc_lens = (didx.doc_offsets[1:] - didx.doc_offsets[:-1]).cpu()
    lib, h, st = didx._lib, didx._handle, didx._stream()
    ids = torch.empty((B, k), dtype=torch.int64, device=device)
    top = torch.empty((B, k), dtype=torch.float32, device=device)
    counts = torch.empty((B,), dtype=torch.int32, device=device)
    t0 = time.time()

    # the full scan: its time, and every score of the batch for the parity check
    ws_full_bytes = didx.exhaustive_workspace_bytes(B, Q, k)
    ws_full = torch.empty(ws_full_bytes, dtype=torch.uint8, device=device)

    def run_full():
        _check(lib.fpb_search_exhaustive(h, q16.data_ptr(), B, Q, k, ws_full.data_ptr(), ws_full_bytes,
                                         ids.data_ptr(), top.data_ptr(), counts.data_ptr(), st))

    ms_full, _ = timed(run_full, args.seconds, args.warmup)
    del ws_full
    every = didx.exhaustive_scores(q16).cpu()

    def run_lists(lists: list[torch.Tensor], query_list: list[int]) -> dict:
        """Time one fpb_search_exhaustive_subset call; check its result against the full scan."""
        lens = [int(x.numel()) for x in lists]
        offs = torch.zeros(len(lists) + 1, dtype=torch.int64)
        offs[1:] = torch.tensor(lens, dtype=torch.int64).cumsum(0)
        sid = torch.cat(lists).to(torch.int32).to(device)
        soff = offs.to(device)
        max_len = max(lens)
        h_list = (ctypes.c_int32 * B)(*query_list)
        ws_bytes = didx.exhaustive_subset_workspace_bytes(B, Q, k, len(lists), max_len)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)

        def run():
            _check(lib.fpb_search_exhaustive_subset(h, q16.data_ptr(), B, Q, k, sid.data_ptr(), soff.data_ptr(),
                                                    len(lists), max_len, h_list, ws.data_ptr(), ws_bytes,
                                                    ids.data_ptr(), top.data_ptr(), counts.data_ptr(), st))

        ms, calls = timed(run, args.seconds, args.warmup)
        run()
        torch.cuda.synchronize()
        got_ids, got_sc, got_cnt = ids.cpu(), top.cpu(), counts.cpu()
        mismatches, tokens = 0, 0
        for b in range(B):
            members = torch.unique(lists[query_list[b]] - base)
            tokens += int(doc_lens[members].sum())
            m = int(got_cnt[b])
            mismatches += int(m != min(k, int(members.numel())))
            local = got_ids[b, :m] - base
            mismatches += int((got_sc[b, :m] != every[b, local]).sum())
            mismatches += int(not bool(torch.isin(local, members).all()))
        tflop = 2.0 * bench.DIM * Q * tokens / 1e12  # every query against every token of its list
        return {"ms": round(ms, 3), "calls": calls, "ws_gb": round(ws_bytes / 1e9, 3),
                "tokens_scored": tokens, "tflops": round(tflop / (ms * 1e-3), 1),
                "share_of_989_tflops": round(tflop / (ms * 1e-3) / PEAK_TFLOPS, 3),
                "parity_mismatches": mismatches}

    g = torch.Generator().manual_seed(bench.SEED_QUERY + 1)
    out: dict = {"metric": "exhaustive_subset_search", "config": args.config, "desc": cfg["desc"], "card": card(),
                 "B": B, "Q": Q, "top_k": k, "n_docs": n_docs, "n_tokens": didx.num_tokens,
                 "full_scan_ms": round(ms_full, 3)}
    if args.workload in ("filtered", "both"):
        filtered = {}
        for frac in (0.01, 0.1, 0.5, 1.0):
            n_sub = max(1, round(frac * n_docs))
            sub = torch.randperm(n_docs, generator=g)[:n_sub] + base  # unsorted global ids
            r = run_lists([sub], [0] * B)
            r["vs_full_scan"] = round(r["ms"] / ms_full, 3)
            filtered[f"{frac:g}"] = r
        out["filtered_one_shared_subset"] = filtered
    if args.workload in ("rerank", "both"):
        params = DeviceIndex.make_params(k, bench.N_FULL, bench.N_IVF_PROBE)
        ms_search, _ = timed(lambda: didx.search(q16, params), args.seconds, args.warmup)
        rerank = {"search_ms": round(ms_search, 3)}
        for L in (100, 1000, 4096):
            lists = [torch.randperm(n_docs, generator=g)[:L] + base for _ in range(B)]
            r = run_lists(lists, list(range(B)))
            r["tokens_per_s"] = round(r["tokens_scored"] / (r["ms"] * 1e-3), 1)
            rerank[str(L)] = r
        out["rerank_distinct_lists"] = rerank
    out["wall_s"] = round(time.time() - t0, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
