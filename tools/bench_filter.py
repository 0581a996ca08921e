"""Filtered search on the benchmark's synthetic indexes, by `subset=` form: one JSON line per run.

    python tools/bench_filter.py --config cfg3 [--seconds 1.0] [--warmup 2]

Workloads, on the config's batch (B queries of Q tokens): one random filter shared by the batch holding 1 / 10 / 50 %
of the documents (a metadata filter), and a distinct row of 1 000 random candidates per query (first-stage ids to
re-rank).  For each, and each form of the same documents:

* lists      one Python list per query (the per-query path: the filter is built once per query);
* broadcast  one Python list for the whole batch (shared workloads only);
* ids        an int64 tensor in host memory, [L] shared or [B, L] per query;
* cuda_mask  a bool mask on the GPU, [num_documents] shared or [B, num_documents] per query;

it reports the wall time of one `FastPlaid.search` and one `FastPlaid.search_exhaustive` call (results returned to
the host, so synchronised), mean over at least --seconds, and whether every form returned identical results.  The
device time of the subset stage alone (fpb_stage_subset on B per-query lists, against fpb_stage_filter on the
filters) is timed with CUDA events over at least --seconds after warm-up.  Needs a CUDA device.
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
from bench_exhaustive import card, timed  # noqa: E402  (tools/ is the script's directory)


def wall(fn, seconds: float) -> tuple[float, object]:
    """Mean wall milliseconds of fn() (synchronised by its host results) over at least `seconds`, one call at
    least; and the last result."""
    fn()  # warm-up
    n, t0 = 0, time.perf_counter()
    while True:
        out = fn()
        n += 1
        if time.perf_counter() - t0 >= seconds:
            return (time.perf_counter() - t0) * 1e3 / n, out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg3", choices=["cfg2", "cfg3", "tiny"])
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_filter.py needs a CUDA device (the engine has no CPU path)")
    from fast_plaid_b200.engine import FPB_FLAG_SUBSET, DeviceIndex, Filter, IndexTensors, _check
    from fast_plaid_b200.search import FastPlaid

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
    queries = q.float().cpu()
    q16 = q.to(device).half().contiguous()
    fp = FastPlaid.from_device_index(didx)
    params = DeviceIndex.with_flags(DeviceIndex.make_params(k, bench.N_FULL, bench.N_IVF_PROBE), FPB_FLAG_SUBSET)
    buf, lay = didx.workspace(B, Q, params)
    lib, h, st = didx._lib, didx._handle, didx._stream()
    p = ctypes.byref(params)
    t0 = time.time()

    def stage_times(sets: list[torch.Tensor], filt: Filter) -> dict:
        """Device ms of the subset stage on B per-query lists, and of the filter stage on `filt`."""
        _check(lib.fpb_stage_centroid_scores(h, q16.data_ptr(), B, Q, p, buf.data_ptr(), buf.numel(), st))
        lens = [int(s.numel()) for s in sets]
        offs = torch.zeros(B + 1, dtype=torch.int64)
        offs[1:] = torch.tensor(lens).cumsum(0)
        sid = torch.cat(sets).to(torch.int32).to(device)
        soff = offs.to(device)
        h_map = (ctypes.c_int32 * B)(*filt.query_filter)
        ms_lists, _ = timed(lambda: _check(lib.fpb_stage_subset(h, sid.data_ptr(), soff.data_ptr(), max(lens), B, Q, p,
                                                                buf.data_ptr(), buf.numel(), st)),
                            args.seconds, args.warmup)
        ms_filter, _ = timed(lambda: _check(lib.fpb_stage_filter(h, filt.bitmap.data_ptr(), filt.n_filters,
                                                                 filt.n_bits, h_map, B, Q, p, buf.data_ptr(),
                                                                 buf.numel(), st)),
                             args.seconds, args.warmup)
        return {"per_query_lists_ms": round(ms_lists, 3), "filter_ms": round(ms_filter, 3)}

    g = torch.Generator().manual_seed(bench.SEED_QUERY + 2)
    workloads = {}
    for frac in (0.01, 0.1, 0.5):
        ids = torch.randperm(n_docs, generator=g)[: max(1, round(frac * n_docs))] + base
        workloads[f"shared_{frac:g}"] = [ids] * B
    workloads["per_query_1000"] = [torch.randperm(n_docs, generator=g)[:1000] + base for _ in range(B)]
    out: dict = {"metric": "filtered_search", "config": args.config, "desc": cfg["desc"], "card": card(), "B": B,
                 "Q": Q, "top_k": k, "n_docs": n_docs, "n_ivf_probe": bench.N_IVF_PROBE}
    for name, sets in workloads.items():
        shared = name.startswith("shared")
        lists = [s.tolist() for s in sets]
        mask = torch.zeros((B, n_docs), dtype=torch.bool)
        for b, s in enumerate(sets):
            mask[b, s - base] = True
        forms = {"lists": [list(x) for x in lists]}
        if shared:
            forms["broadcast"] = lists[0]
            forms["ids"] = sets[0].clone()
            forms["cuda_mask"] = mask[0].to(device)
        else:
            forms["ids"] = torch.stack(sets)
            forms["cuda_mask"] = mask.to(device)
        r: dict = {"n_filter_docs": int(sets[0].numel())}
        for what, fn in (("search", lambda s: fp.search(queries, top_k=k, subset=s)),
                         ("search_exhaustive", lambda s: fp.search_exhaustive(queries, top_k=k, subset=s))):
            ref, times = None, {}
            identical = True
            for form, s in forms.items():
                ms, res = wall(lambda: fn(s), args.seconds)
                times[form] = round(ms, 2)
                ref = res if ref is None else ref
                identical &= res == ref
            r[what] = {"wall_ms": times, "identical": identical}
        filt = (Filter.from_ids(sets[0], n_docs + base, device, B) if shared
                else Filter.from_ids(torch.stack(sets), n_docs + base, device, B))
        r["device_subset_stage"] = stage_times(sets, filt)
        out[name] = r
    out["wall_s"] = round(time.time() - t0, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
