"""Exhaustive exact search on the benchmark's synthetic indexes: one JSON line per run.

    python tools/bench_exhaustive.py --config cfg2 [--seconds 1.0] [--warmup 2]

Times fpb_exhaustive_scores (K7 + finalize) and the whole fpb_search_exhaustive (plus k3b_select and k6_rank) with CUDA events over at least --seconds of work after warm-up, and compares the approximate search()
(default parameters) against the exact result of the same batch: recall@top_k and the number of search() results
whose score disagrees with the exhaustive score of the same document.  Needs a CUDA device; there is no fallback.
"""

from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402

PEAK_TFLOPS = 989.0  # H100 SXM data sheet, dense fp16 tensor-core rate (not measured)


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:  # the number is reported as unknown rather than guessed
        pass
    return out


def timed(fn, seconds: float, warmup: int) -> tuple[float, int]:
    """Mean CUDA-event milliseconds per call over at least `seconds` of work."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n, total = 0, 0.0
    while total < seconds * 1e3:
        reps = max(1, n)  # doubling batches of calls between two events
        start.record()
        for _ in range(reps):
            fn()
        stop.record()
        stop.synchronize()
        total += start.elapsed_time(stop)
        n += reps
    return total / n, n


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2", choices=["cfg2", "cfg3", "cfg3c", "cfg5", "tiny"])
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_exhaustive.py needs a CUDA device (the engine has no CPU path)")
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
    E = didx.num_tokens

    lib, h, st = didx._lib, didx._handle, didx._stream()
    ws_bytes = didx.exhaustive_workspace_bytes(B, Q, k)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
    scores = torch.empty((B, n_docs), dtype=torch.float32, device=device)
    ids = torch.empty((B, k), dtype=torch.int64, device=device)
    top = torch.empty((B, k), dtype=torch.float32, device=device)
    counts = torch.empty((B,), dtype=torch.int32, device=device)

    def run_scores():
        _check(lib.fpb_exhaustive_scores(h, q16.data_ptr(), B, Q, ws.data_ptr(), ws_bytes, scores.data_ptr(), st))

    def run_search():
        _check(lib.fpb_search_exhaustive(h, q16.data_ptr(), B, Q, k, ws.data_ptr(), ws_bytes, ids.data_ptr(),
                                         top.data_ptr(), counts.data_ptr(), st))

    t0 = time.time()
    ms_scores, n_scores = timed(run_scores, args.seconds, args.warmup)
    ms_search, n_search = timed(run_search, args.seconds, args.warmup)
    # time split: the kernel decodes every tile once, then runs one MMA + epilogue pass per 128 query rows.  A batch
    # that fills exactly one row block separates the per-tile cost (decode, query packing, finalize) from the
    # per-row-block cost (MMA + epilogue), by a linear fit over the number of row blocks.
    qs = (Q + 15) // 16 * 16
    b1 = max(1, 128 // qs)
    n_rb = (B * qs + 127) // 128

    def run_one_block():
        _check(lib.fpb_exhaustive_scores(h, q16.data_ptr(), b1, Q, ws.data_ptr(), ws_bytes, scores.data_ptr(), st))

    ms_one, _ = timed(run_one_block, args.seconds, args.warmup)
    per_rb = (ms_scores - ms_one) / max(1, n_rb - 1)
    # timing variants of the kernel (dim 128 / nbits 4 only; their scores are meaningless): the MMAs without the
    # epilogue, and the decode of every tile without any MMA
    parts = {}
    if didx.dim == 128 and didx.nbits == 4:
        for part in ("mma", "decode"):
            os.environ["FPB_K7"] = part
            try:
                parts[part], _ = timed(run_scores, args.seconds, args.warmup)
            finally:
                del os.environ["FPB_K7"]
    wall = time.time() - t0

    # the approximate search (default parameters) against the exact answer of the same batch
    run_scores()
    run_search()
    a_ids, a_sc, a_cnt = didx.search(q16, DeviceIndex.make_params(k, bench.N_FULL, bench.N_IVF_PROBE))
    torch.cuda.synchronize()
    e_ids, a_ids, a_sc, a_cnt, every = ids.cpu(), a_ids.cpu(), a_sc.cpu(), a_cnt.cpu(), scores.cpu()
    hits, disagree, n_cmp = 0, 0, 0
    for b in range(B):
        exact = set(e_ids[b].tolist()) - {-1}
        got = a_ids[b, : int(a_cnt[b])].tolist()
        hits += len(exact & set(got))
        for i, d in enumerate(got):
            ex = float(every[b, d - base])
            n_cmp += 1
            disagree += int(abs(ex - float(a_sc[b, i])) > 1e-3 * max(1.0, abs(ex)))

    flop = 2.0 * bench.DIM * Q * B * E
    idx_bytes = E * (didx.dim * didx.nbits // 8 + 4 + 2)
    tflops = flop / (ms_scores * 1e-3) / 1e12
    print(json.dumps({
        "metric": "exhaustive_exact_search",
        "config": args.config,
        "desc": cfg["desc"],
        "card": card(),
        "B": B, "Q": Q, "top_k": k, "n_docs": n_docs, "n_tokens": E,
        "scores_ms": round(ms_scores, 3), "scores_calls": n_scores,
        "search_ms": round(ms_search, 3), "search_calls": n_search,
        "selection_ms": round(ms_search - ms_scores, 3),
        "split": {
            "row_blocks": n_rb,
            "one_row_block_ms": round(ms_one, 3),
            "per_row_block_ms": round(per_rb, 3),
            "fixed_ms": round(ms_one - per_rb, 3),
            "per_row_block_ideal_ms": round(2.0 * 128 * bench.DIM * E / (PEAK_TFLOPS * 1e12) * 1e3, 3),
            "mma_only_ms": round(parts["mma"], 3) if "mma" in parts else None,
            "decode_only_ms": round(parts["decode"], 3) if "decode" in parts else None,
            "epilogue_ms": round(ms_scores - parts["mma"], 3) if "mma" in parts else None,
            "note": "fixed = decode of every tile once + query packing + finalize; per row block = 128 query rows "
                    "of MMA + per-document maxima + fixed-point sums over the whole index; mma_only = the kernel "
                    "without its epilogue (decode included), decode_only = the kernel without its MMA loop "
                    "(query packing and finalize included in both); epilogue = full - mma_only",
        },
        "algorithmic_tflop": round(flop / 1e12, 3),
        "index_bytes_gb": round(idx_bytes / 1e9, 3),
        "tflops": round(tflops, 1),
        "share_of_989_tflops": round(tflops / PEAK_TFLOPS, 3),
        "bound": "compute (fp16 tensor cores): the index bytes take %.2f ms at 3.35 TB/s" % (idx_bytes / 3.35e9),
        "queries_per_s": round(B / (ms_search * 1e-3), 1),
        "recall_at_k_of_search": round(hits / max(1, sum(min(k, n_docs) for _ in range(B))), 4),
        "recall_note": "synthetic codes" + (" (clustered)" if cfg.get("topics") else " (uniform)"),
        "search_scores_disagreeing": disagree,
        "search_scores_compared": n_cmp,
        "wall_s": round(wall, 1),
    }))


if __name__ == "__main__":
    main()
