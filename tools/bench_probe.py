"""Search cost and recall against n_ivf_probe on the benchmark's synthetic indexes: one JSON line.

    python tools/bench_probe.py [--config cfg3] [--n 8,32,33,64,256,1024,4096] [--seconds 1.0] [--rounds 2]
                                [--subset-pct 1.0]

For every n, with the config's query batch (64 queries x 32 tokens, top_k 100, n_full_scores 4096 as in bench.py):
  * search() per batch;
  * the probe (K1b) and the candidate pass (K2) alone, on the S of that batch;
  * mean candidates per query;
  * recall@top_k of search() against search_exhaustive() on the same batch.
Then the same with one shared subset of --subset-pct % of the documents (0: skip), against
search_exhaustive(subset=...).  Times are CUDA-event means over windows of at least --seconds after warm-up; every
round times every n in turn, and the median over the rounds is reported.  The residual codes are random, so the recall
figures describe this synthetic index, not a retrieval task.  Needs a CUDA device.
"""

from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from tools.bench_exhaustive import card, timed  # noqa: E402
from tools.bench_nbits import build  # noqa: E402


def recall(ids, counts, ref_ids, ref_counts) -> float:
    """Mean over queries of |found ∩ reference| / |reference|."""
    ids, counts, ref_ids, ref_counts = ids.cpu(), counts.cpu(), ref_ids.cpu(), ref_counts.cpu()
    r = []
    for b in range(ids.shape[0]):
        ref = set(ref_ids[b, : int(ref_counts[b])].tolist())
        if ref:
            r.append(len(set(ids[b, : int(counts[b])].tolist()) & ref) / len(ref))
    return round(sum(r) / max(1, len(r)), 4)


def sweep(didx, q, cfg, ns, subset, args) -> dict:
    """{n: measurements} for one scenario (subset: one list of global ids shared by every query, or None)."""
    from fast_plaid_b200.engine import FPB_FLAG_SUBSET, DeviceIndex

    B = q.shape[0]
    subsets = None if subset is None else [subset] * B
    k = cfg["top_k"]
    params = {n: DeviceIndex.make_params(k, bench.N_FULL, n) for n in ns}
    stage_params = {n: p if subset is None else DeviceIndex.with_flags(p, FPB_FLAG_SUBSET) for n, p in params.items()}
    e_ids, _, e_counts = didx.search_exhaustive(q, k, subset=subsets)
    out = {}
    for n in ns:
        ids, _, counts = didx.search(q, params[n], subset=subsets)
        st = didx.run_stages(q, params[n], upto="candidates", subset=subsets)
        torch.cuda.synchronize()
        out[n] = {"mean_candidates": round(float(st["n_cand"].float().mean()), 1),
                  f"recall@{k}": recall(ids, counts, e_ids, e_counts)}
    # the workspace buffer only grows, and every layout timed below has been used above: a stage function keeps
    # the buffer it was made with, and that buffer stays the index's from here on
    ms ={n: {"search": [], "probe": [], "candidates": []} for n in ns}
    for _ in range(args.rounds):
        for n in ns:
            ms[n]["search"].append(timed(lambda: didx.search(q, params[n], subset=subsets), args.seconds, args.warmup)[0])
            didx.run_stages(q, params[n], upto="candidates", subset=subsets)  # this n's S, subset lists and cells
            for stage in ("probe", "candidates"):
                ms[n][stage].append(timed(didx.stage_fn(stage, q, stage_params[n]), args.seconds, args.warmup)[0])
    for n in ns:
        for key, v in ms[n].items():
            out[n][f"{key}_ms"] = round(statistics.median(v), 3)
    return {str(n): v for n, v in out.items()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg3", choices=["cfg3", "cfg2", "tiny"])
    ap.add_argument("--n", default="8,32,33,64,256,1024,4096", help="comma-separated n_ivf_probe values")
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--subset-pct", type=float, default=1.0, help="shared subset, percent of the documents (0: skip)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_probe.py needs a CUDA device (the engine has no CPU path)")
    cfg = bench.CONFIGS[args.config]
    ns = [int(x) for x in args.n.split(",")]
    didx, _, q = build(cfg, bench.NBITS)
    out = {"metric": "n_ivf_probe_sweep", "card": card(), "config": args.config, "B": q.shape[0], "Q": q.shape[1],
           "top_k": cfg["top_k"], "n_full_scores": bench.N_FULL, "n_centroids": didx.num_centroids,
           "n_docs": cfg["n_docs"]}
    out["all"] = sweep(didx, q, cfg, ns, None, args)
    if args.subset_pct > 0:
        N = cfg["n_docs"]
        g = torch.Generator().manual_seed(7)
        m = max(1, int(N * args.subset_pct / 100))
        subset = sorted((torch.randperm(N, generator=g)[:m] + didx.doc_id_base).tolist())
        out["subset_docs"] = m
        out["subset"] = sweep(didx, q, cfg, ns, subset, args)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
