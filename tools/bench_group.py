"""Grouped results (`group_by=`) on the benchmark's synthetic indexes: one JSON line per (config, group map).

    python tools/bench_group.py [--configs cfg2,cfg3,cfg5] [--seconds 1.0] [--warmup 2]
                                [--maps singletons,runs10,random10,one] [--max-per-group 1,2,4,16]

Group maps over the N documents: singletons (every document its own group), runs of 10 consecutive documents, random
groups of 10 on average, and one group.  On the config's batch (at most 64 queries, 32 on cfg5) it reports, with
CUDA events over at least --seconds after warm-up, the device time of `DeviceIndex.search` and
`DeviceIndex.search_exhaustive`, grouped and ungrouped, alternated in one process (ungrouped, grouped, twice; the
smaller of the two means is kept).  Also: the wall time of the host remap (`Groups.from_tensor`, synchronised), and
the time of the grouping kernels alone (group_max, group_select, k6_rank_grouped) from one torch.profiler run.
Every grouped result is checked against the host collapse of the ungrouped ranking (exact: of the full
`exhaustive_scores` ranking; approximate: of the search with top_k = n_full_scores // 4).  The card's name and power
limit are read in the same run.  Needs a CUDA device.

With --max-per-group, each (config, group map) gives one line per m instead: the same timings with the groups'
max_per_group = m (plain and grouped alternated), the time of the grouping kernels of one call (the m rounds of
group_round_max summed; group_max at m = 1), and the check of every grouped result against the rule applied on the
host (keep a document when fewer than m of its group come before it in the ungrouped ranking).
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from bench_exhaustive import card, timed  # noqa: E402  (tools/ is the script's directory)


def group_maps(n: int) -> dict[str, torch.Tensor]:
    gen = torch.Generator().manual_seed(7)
    return {
        "singletons": torch.arange(n, dtype=torch.int64),
        "runs10": torch.arange(n, dtype=torch.int64) // 10,
        "random10": torch.randint(0, max(n // 10, 1), (n,), generator=gen, dtype=torch.int64),
        "one": torch.zeros(n, dtype=torch.int64),
    }


def exact_collapse(scores: torch.Tensor, ids: torch.Tensor, k: int) -> tuple[torch.Tensor, torch.Tensor]:
    """The first k documents of distinct groups in the canonical order of one query's [N] scores (device)."""
    n = scores.shape[0]
    order = torch.sort(scores, descending=True, stable=True).indices  # ties: smaller id first
    g = ids[order].long()
    first = torch.full((int(ids.max()) + 1,), n, dtype=torch.int64, device=scores.device)
    first.scatter_reduce_(0, g, torch.arange(n, device=scores.device), reduce="amin")
    pos = torch.sort(first[first < n]).values[:k]
    return order[pos], scores[order[pos]]


def host_collapse(ids: torch.Tensor, counts: torch.Tensor, groups: torch.Tensor, k: int) -> list[list[int]]:
    out = []
    for b in range(ids.shape[0]):
        seen, kept = set(), []
        for d in ids[b, : int(counts[b])].tolist():
            if int(groups[d]) not in seen:
                seen.add(int(groups[d]))
                kept.append(d)
        out.append(kept[:k])
    return out


def exact_limit(scores: torch.Tensor, ids: torch.Tensor, m: int, k: int) -> tuple[torch.Tensor, torch.Tensor]:
    """The first k documents, at most m per group, in the canonical order of one query's [N] scores (device)."""
    n = scores.shape[0]
    order = torch.sort(scores, descending=True, stable=True).indices  # ties: smaller id first
    g = ids[order].long()
    by_group = torch.sort(g, stable=True).indices  # rank positions, grouped, in rank order within a group
    gs = g[by_group]
    rank = torch.empty_like(by_group)
    rank[by_group] = torch.arange(n, device=scores.device) - torch.searchsorted(gs, gs)
    pos = torch.nonzero(rank < m).flatten()[:k]
    return order[pos], scores[order[pos]]


def host_limit(ids: torch.Tensor, counts: torch.Tensor, groups: torch.Tensor, m: int, k: int) -> list[list[int]]:
    out = []
    for b in range(ids.shape[0]):
        seen: dict[int, int] = {}
        kept = []
        for d in ids[b, : int(counts[b])].tolist():
            g = int(groups[d])
            if seen.get(g, 0) < m:
                seen[g] = seen.get(g, 0) + 1
                kept.append(d)
        out.append(kept[:k])
    return out


def call_kernel_times(fn, names: tuple[str, ...]) -> dict[str, float]:
    """Device milliseconds of the kernels named `names` in one call of fn, summed over their launches."""
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out: dict[str, float] = {}
    for e in prof.key_averages():
        for name in names:
            if name in e.key and (name != "group_max" or "group_max_kernel" in e.key):
                out[name + "_ms"] = round(out.get(name + "_ms", 0.0) + e.device_time_total / 1e3, 4)
    return out


def limit_rows(didx, q16, params, k, every, base_ids, base_counts, g, n, device, row, limits, args):
    """One line per m of --max-per-group: timings, kernel times and checks at max_per_group = m."""
    from fast_plaid_b200.engine import Groups

    B = q16.shape[0]
    for m in limits:
        groups = Groups.from_tensor(g, n, device, m)
        out = dict(row, max_per_group=m)
        ids, sc, counts = didx.search_exhaustive(q16, k, groups=groups)
        ok = True
        for b in range(B):
            exp_ids, exp_sc = exact_limit(every[b], groups.ids, m, k)
            c = exp_ids.shape[0]
            ok &= int(counts[b]) == c and torch.equal(ids[b, :c], exp_ids) and torch.equal(sc[b, :c], exp_sc)
        a_ids, _, a_counts = (t.cpu() for t in didx.search(q16, params, groups=groups))
        exp = host_limit(base_ids, base_counts, groups.ids.cpu(), m, k)
        ok &= all(a_ids[b, : int(a_counts[b])].tolist() == exp[b] for b in range(B))
        out["checked"] = bool(ok)
        timings = {}
        for _ in range(2):  # alternated: ungrouped, grouped
            for label, fn in (
                ("search_ms", lambda: didx.search(q16, params)),
                ("search_grouped_ms", lambda: didx.search(q16, params, groups=groups)),
                ("exhaustive_ms", lambda: didx.search_exhaustive(q16, k)),
                ("exhaustive_grouped_ms", lambda: didx.search_exhaustive(q16, k, groups=groups)),
            ):
                ms, _ = timed(fn, args.seconds, args.warmup)
                timings[label] = min(timings.get(label, float("inf")), ms)
        out.update({key: round(v, 4) for key, v in timings.items()})
        out["exhaustive_overhead_pct"] = round(100 * (timings["exhaustive_grouped_ms"] / timings["exhaustive_ms"]
                                                      - 1), 3)
        out["search_overhead_pct"] = round(100 * (timings["search_grouped_ms"] / timings["search_ms"] - 1), 3)
        out.update(call_kernel_times(lambda: didx.search_exhaustive(q16, k, groups=groups),
                                     ("group_max", "group_round_max", "group_select")))
        out.update(call_kernel_times(lambda: didx.search(q16, params, groups=groups), ("k6_rank_grouped",)))
        print(json.dumps(out), flush=True)


def kernel_times(fn) -> dict[str, float]:
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out: dict[str, float] = {}
    for e in prof.key_averages():
        for name in ("group_max", "group_select", "k6_rank_grouped"):
            if name in e.key:
                out[name + "_ms"] = round(e.device_time_total / 1e3 / max(e.count, 1), 4)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="cfg2,cfg3,cfg5")
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--maps", default="singletons,runs10,random10,one")
    ap.add_argument("--max-per-group", default="", help="comma-separated m values: one line per (map, m)")
    args = ap.parse_args()
    limits = [int(m) for m in args.max_per_group.split(",") if m]
    maps = args.maps.split(",")
    if not torch.cuda.is_available():
        raise SystemExit("bench_group.py needs a CUDA device (the engine has no CPU path)")
    from fast_plaid_b200.engine import DeviceIndex, Groups, IndexTensors

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
        every = didx.exhaustive_scores(q16)
        base_ids, _, base_counts = (t.cpu() for t in didx.search(q16, wide))
        for gname, g in group_maps(n).items():
            if gname not in maps:
                continue
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            groups = Groups.from_tensor(g, n, device)
            torch.cuda.synchronize()
            remap_ms = (time.perf_counter() - t0) * 1e3
            row = {"config": name, "B": B, "Q": Q, "top_k": k, "n_docs": n, "groups": gname,
                   "n_groups": groups.n_groups, "remap_ms": round(remap_ms, 3), "card": hw}
            if limits:
                limit_rows(didx, q16, params, k, every, base_ids, base_counts, g, n, device, row, limits, args)
                continue
            # the checks: every timed grouped call gives these bytes
            ids, sc, counts = didx.search_exhaustive(q16, k, groups=groups)
            ok = True
            for b in range(B):
                exp_ids, exp_sc = exact_collapse(every[b], groups.ids, k)
                m = exp_ids.shape[0]
                ok &= int(counts[b]) == m and torch.equal(ids[b, :m], exp_ids) and torch.equal(sc[b, :m], exp_sc)
            a_ids, _, a_counts = (t.cpu() for t in didx.search(q16, params, groups=groups))
            exp = host_collapse(base_ids, base_counts, groups.ids.cpu(), k)
            ok &= all(a_ids[b, : int(a_counts[b])].tolist() == exp[b] for b in range(B))
            row["checked"] = bool(ok)
            timings = {}
            for _ in range(2):  # alternated: ungrouped, grouped
                for label, fn in (
                    ("search_ms", lambda: didx.search(q16, params)),
                    ("search_grouped_ms", lambda: didx.search(q16, params, groups=groups)),
                    ("exhaustive_ms", lambda: didx.search_exhaustive(q16, k)),
                    ("exhaustive_grouped_ms", lambda: didx.search_exhaustive(q16, k, groups=groups)),
                ):
                    ms, _ = timed(fn, args.seconds, args.warmup)
                    timings[label] = min(timings.get(label, float("inf")), ms)
            row.update({key: round(v, 4) for key, v in timings.items()})
            row["exhaustive_overhead_pct"] = round(100 * (timings["exhaustive_grouped_ms"] / timings["exhaustive_ms"]
                                                          - 1), 3)
            row["search_overhead_pct"] = round(100 * (timings["search_grouped_ms"] / timings["search_ms"] - 1), 3)
            row.update(kernel_times(lambda: didx.search_exhaustive(q16, k, groups=groups)))
            row.update(kernel_times(lambda: didx.search(q16, params, groups=groups)))
            print(json.dumps(row), flush=True)
        del every
        didx.close()
        del didx
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
