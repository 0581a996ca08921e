"""Grouped results on document-sharded indexes: one JSON line per measurement.

    python tools/bench_group_sharded.py [--merge-shapes 4x1024,4x4096,8x2048,16x1024] [--configs cfg2,cfg3]
                                        [--max-per-group 1,4] [--seconds 1.0] [--warmup 2]

1. The merge alone, on synthetic gathered records of B = 64 queries ([n_shards, B, R], random scores, distinct global
   ids, random groups of about 10 documents) at each n_shards x R of --merge-shapes, m = 1 and 16: the device time of
   the grouped merge (fpb_merge_shards_grouped, n_keep = R) against the ungrouped one (fpb_merge_shards).  Multi-shard
   records are merged on one GPU.  Each grouped result is checked against the rule applied on the host to the
   ungrouped merge's full ranking (top_k = R).
2. At shard=(0, 1) on each config's batch (at most 64 queries), random groups of about 10 documents and each m of
   --max-per-group: the device time of DeviceIndex.search_sharded and search_exhaustive_sharded, grouped and
   ungrouped, and of the unsharded grouped calls, alternated in one process (the smaller of two means is kept).  The
   sharded grouped results are checked byte for byte against the unsharded grouped ones, and those against the rule
   applied on the host (bench_group.py's checks).
CUDA events over at least --seconds after warm-up; the card's name and power limit are read in the same run.  Needs a
CUDA device.
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
from bench_group import exact_limit, host_limit  # noqa: E402

B_MERGE = 64
TOP_K = 100


def merge_rows(shapes, limits, args, hw) -> None:
    from fast_plaid_b200 import engine

    lib = engine.load_library()
    dev = "cuda:0"
    gen = torch.Generator(device=dev).manual_seed(11)
    for shape in shapes:
        S, R = (int(x) for x in shape.split("x"))
        n_total = 2 * S * R
        rec = torch.empty((S, B_MERGE, R, 4), dtype=torch.float32, device=dev)
        rec[..., 0] = torch.randn((S, B_MERGE, R), generator=gen, device=dev)          # approx
        rec[..., 1] = rec[..., 0] + 0.3 * torch.randn((S, B_MERGE, R), generator=gen, device=dev)  # exact
        ids = torch.stack([torch.randperm(n_total, generator=gen, device=dev)[: S * R] for _ in range(B_MERGE)])
        rec.view(torch.int64)[..., 1] = ids.view(B_MERGE, S, R).transpose(0, 1)
        rec = rec.contiguous()
        gmap = torch.randint(0, n_total // 10, (n_total,), generator=gen, device=dev, dtype=torch.int32)
        out_ids = torch.empty((B_MERGE, R), dtype=torch.int64, device=dev)
        out_sc = torch.empty((B_MERGE, R), dtype=torch.float32, device=dev)
        out_n = torch.empty((B_MERGE,), dtype=torch.int32, device=dev)

        def plain(k=TOP_K):
            engine._check(lib.fpb_merge_shards(rec.data_ptr(), S, B_MERGE, R, k, out_ids.data_ptr(),
                                               out_sc.data_ptr(), out_n.data_ptr(),
                                               torch.cuda.current_stream().cuda_stream))

        plain(R)  # the full kept ranking, for the checks
        f_ids, f_n = out_ids.cpu(), out_n.cpu()
        for m in limits:
            g_ids = torch.empty((B_MERGE, TOP_K), dtype=torch.int64, device=dev)
            g_sc = torch.empty((B_MERGE, TOP_K), dtype=torch.float32, device=dev)
            g_n = torch.empty((B_MERGE,), dtype=torch.int32, device=dev)

            def grouped():
                engine._check(lib.fpb_merge_shards_grouped(
                    rec.data_ptr(), S, B_MERGE, R, R, TOP_K, gmap.data_ptr(), n_total, m, g_ids.data_ptr(),
                    g_sc.data_ptr(), g_n.data_ptr(), torch.cuda.current_stream().cuda_stream))

            grouped()
            exp = host_limit(f_ids, f_n, gmap.cpu(), m, TOP_K)
            got_ids, got_n = g_ids.cpu(), g_n.cpu()
            ok = all(got_ids[b, : int(got_n[b])].tolist() == exp[b] for b in range(B_MERGE))
            t = {}
            for _ in range(2):  # alternated
                for label, fn in (("merge_ms", plain), ("merge_grouped_ms", grouped)):
                    ms, _ = timed(fn, args.seconds, args.warmup)
                    t[label] = min(t.get(label, float("inf")), ms)
            print(json.dumps({"bench": "merge", "B": B_MERGE, "n_shards": S, "R": R, "top_k": TOP_K,
                              "max_per_group": m, "checked": bool(ok), **{k: round(v, 4) for k, v in t.items()},
                              "card": hw}), flush=True)


def config_rows(configs, limits, args, hw) -> None:
    from fast_plaid_b200.engine import DeviceIndex, Groups, IndexTensors, ShardComm

    device = "cuda:0"
    for name in configs:
        cfg = bench.CONFIGS[name]
        n_docs, Q, k = cfg["n_docs"], cfg["Q"], cfg["top_k"]
        B = min(cfg["B"], 64)
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
        wide = DeviceIndex.make_params(max(bench.N_FULL // 4, 1), bench.N_FULL, bench.N_IVF_PROBE)
        n = didx.num_documents
        comm = ShardComm(1, 0, ShardComm.new_unique_id(), device)
        g = torch.randint(0, max(n // 10, 1), (n,), generator=torch.Generator().manual_seed(7), dtype=torch.int64)
        every = didx.exhaustive_scores(q16)
        base_ids, _, base_counts = (t.cpu() for t in didx.search(q16, wide))
        for m in limits:
            whole = Groups.from_tensor(g, n, device, m)
            shard = Groups.for_shard(g, 0, n, device, m)
            ok = True
            s_ref = didx.search(q16, params, groups=whole)
            e_ref = didx.search_exhaustive(q16, k, groups=whole)
            s_got = didx.search_sharded(comm, 1, q16, params, shard)
            e_got = didx.search_exhaustive_sharded(comm, 1, q16, k, groups=shard)
            ok &= all(torch.equal(a, b) for a, b in zip(s_ref + e_ref, s_got + e_got))
            exp = host_limit(base_ids, base_counts, whole.ids.cpu(), m, k)
            a_ids, _, a_n = (t.cpu() for t in s_ref)
            ok &= all(a_ids[b, : int(a_n[b])].tolist() == exp[b] for b in range(B))
            for b in range(B):
                x_ids, x_sc = exact_limit(every[b], whole.ids, m, k)
                c = x_ids.shape[0]
                ok &= int(e_ref[2][b]) == c and torch.equal(e_ref[0][b, :c], x_ids) and torch.equal(e_ref[1][b, :c],
                                                                                                     x_sc)
            t = {}
            for _ in range(2):  # alternated
                for label, fn in (
                    ("sharded_search_ms", lambda: didx.search_sharded(comm, 1, q16, params)),
                    ("sharded_search_grouped_ms", lambda: didx.search_sharded(comm, 1, q16, params, shard)),
                    ("search_grouped_ms", lambda: didx.search(q16, params, groups=whole)),
                    ("sharded_exhaustive_ms", lambda: didx.search_exhaustive_sharded(comm, 1, q16, k)),
                    ("sharded_exhaustive_grouped_ms",
                     lambda: didx.search_exhaustive_sharded(comm, 1, q16, k, groups=shard)),
                    ("exhaustive_grouped_ms", lambda: didx.search_exhaustive(q16, k, groups=whole)),
                ):
                    ms, _ = timed(fn, args.seconds, args.warmup)
                    t[label] = min(t.get(label, float("inf")), ms)
            print(json.dumps({"bench": "shard_of_one", "config": name, "B": B, "Q": Q, "top_k": k, "n_docs": n,
                              "groups": "random10", "max_per_group": m, "checked": bool(ok),
                              **{key: round(v, 4) for key, v in t.items()}, "card": hw}), flush=True)
        comm.close()
        del every
        didx.close()
        del didx
        torch.cuda.empty_cache()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--merge-shapes", default="4x1024,4x4096,8x2048,16x1024")
    ap.add_argument("--merge-max-per-group", default="1,16")
    ap.add_argument("--configs", default="cfg2,cfg3")
    ap.add_argument("--max-per-group", default="1,4")
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_group_sharded.py needs a CUDA device (the engine has no CPU path)")
    hw = card()
    shapes = [s for s in args.merge_shapes.split(",") if s]
    merge_rows(shapes, [int(m) for m in args.merge_max_per_group.split(",") if m], args, hw)
    configs = [c for c in args.configs.split(",") if c]
    config_rows(configs, [int(m) for m in args.max_per_group.split(",") if m], args, hw)


if __name__ == "__main__":
    main()
