"""Biased scores (`score_bias=`) on the benchmark's synthetic indexes: one JSON line per config.

    python tools/bench_score_bias.py [--configs cfg2,cfg3,cfg5] [--seconds 1.0] [--warmup 2] [--rounds 3]

On the config's batch (at most 64 queries, 32 on cfg5) it reports, with CUDA events over at least --seconds after
warm-up, the device time of `DeviceIndex.search` and `DeviceIndex.search_exhaustive`, unbiased and biased by a random
bias in [-2, 2), alternated in one process (unbiased, biased, --rounds times; the smallest mean of each is kept), and
the time of the exhaustive finalize kernel alone, both instances, from one torch.profiler run.  Every biased result
is checked against the host reference: exact search against the unbiased `exhaustive_scores` plus the bias (fp32),
ranked by (score desc, id asc); `search` against the unbiased search with top_k = n_full_scores // 4, biased,
re-sorted and cut to top_k.  The card's name and power limit are read in the same run.  Needs a CUDA device.
"""

from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from bench_exhaustive import card, timed  # noqa: E402  (tools/ is the script's directory)


def canonical(scores: torch.Tensor, ids: torch.Tensor, k: int) -> tuple[torch.Tensor, torch.Tensor]:
    """The first k of (ids, scores) by (score desc, id asc), on the device."""
    order = torch.sort(ids, stable=True).indices
    order = order[torch.sort(scores[order], descending=True, stable=True).indices][:k]
    return ids[order], scores[order]


def finalize_times(fn) -> dict[str, float]:
    """Device milliseconds per launch of the K7 finalize kernels in one call of fn."""
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out: dict[str, float] = {}
    for e in prof.key_averages():
        if "k7_finalize_kernel" in e.key:
            label = "finalize_biased_ms" if "true" in e.key else "finalize_ms"
            out[label] = round(e.device_time_total / 1e3 / max(e.count, 1), 4)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="cfg2,cfg3,cfg5")
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_score_bias.py needs a CUDA device (the engine has no CPU path)")
    from fast_plaid_b200.engine import DeviceIndex, IndexTensors, ScoreBias

    device = "cuda:0"
    hw = card()
    for name in args.configs.split(","):
        cfg = bench.CONFIGS[name]
        n_docs, Q, k = cfg["n_docs"], cfg["Q"], cfg["top_k"]
        B = min(cfg["B"], 32 if name == "cfg5" else 64)
        synth = bench.load_synthetic_module()
        arrays, base = synth.synthetic_arrays(n_docs, cfg["doc_len"], bench.DIM, bench.NBITS, device,
                                              bench.SEED_INDEX, doc_range=(0, n_docs), topics=cfg.get("topics", 0),
                                              mix=cfg.get("mix", 0.05))
        data = IndexTensors(nbits=arrays.nbits, centroids=arrays.centroids, bucket_weights=arrays.bucket_weights,
                            doc_lengths=arrays.doc_lengths, doc_codes=arrays.doc_codes,
                            doc_residuals=arrays.doc_residuals, ivf=arrays.ivf, ivf_lengths=arrays.ivf_lengths)
        didx = DeviceIndex(data, device, doc_id_base=base)
        q = bench.make_query_batches(arrays, bench.query_source_docs(n_docs), cfg, 1)[0]
        del data, arrays
        q16 = q[:B].to(device).half().contiguous()
        params = DeviceIndex.make_params(k, bench.N_FULL, bench.N_IVF_PROBE)
        R = max(bench.N_FULL // 4, 1)
        wide = DeviceIndex.make_params(R, bench.N_FULL, bench.N_IVF_PROBE)
        n = didx.num_documents
        gen = torch.Generator().manual_seed(11)
        bias = ScoreBias.from_tensor((torch.rand(n, generator=gen) - 0.5) * 4.0, n, device)
        every = didx.exhaustive_scores(q16)
        base_ids, base_sc, base_counts = didx.search(q16, wide)

        # the checks: every timed biased call gives these bytes
        ids, sc, counts = didx.search_exhaustive(q16, k, bias=bias)
        all_ids = torch.arange(n, device=device)
        ok = True
        for b in range(B):
            exp_ids, exp_sc = canonical(every[b] + bias.values, all_ids, k)  # fp32 + fp32: one rounded addition
            ok &= int(counts[b]) == k and torch.equal(ids[b], exp_ids + base) and torch.equal(sc[b], exp_sc)
        a_ids, a_sc, a_counts = didx.search(q16, params, bias=bias)
        for b in range(B):
            c = int(base_counts[b])
            loc = base_ids[b, :c] - base
            exp_ids, exp_sc = canonical(base_sc[b, :c] + bias.values[loc], loc, k)
            m = exp_ids.shape[0]
            ok &= int(a_counts[b]) == m and torch.equal(a_ids[b, :m], exp_ids + base) \
                and torch.equal(a_sc[b, :m], exp_sc)
        row = {"config": name, "B": B, "Q": Q, "top_k": k, "n_docs": n, "n_full_scores": bench.N_FULL,
               "checked": bool(ok), "card": hw}
        timings: dict[str, float] = {}
        for _ in range(args.rounds):  # alternated: unbiased, biased
            for label, fn in (
                ("search_ms", lambda: didx.search(q16, params)),
                ("search_biased_ms", lambda: didx.search(q16, params, bias=bias)),
                ("exhaustive_ms", lambda: didx.search_exhaustive(q16, k)),
                ("exhaustive_biased_ms", lambda: didx.search_exhaustive(q16, k, bias=bias)),
            ):
                ms, _ = timed(fn, args.seconds, args.warmup)
                timings[label] = min(timings.get(label, float("inf")), ms)
        row.update({key: round(v, 4) for key, v in timings.items()})
        row["search_overhead_pct"] = round(100 * (timings["search_biased_ms"] / timings["search_ms"] - 1), 3)
        row["exhaustive_overhead_pct"] = round(100 * (timings["exhaustive_biased_ms"] / timings["exhaustive_ms"]
                                                      - 1), 3)
        row.update(finalize_times(lambda: didx.search_exhaustive(q16, k)))
        row.update(finalize_times(lambda: didx.search_exhaustive(q16, k, bias=bias)))
        print(json.dumps(row), flush=True)
        del every
        didx.close()
        del didx
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
