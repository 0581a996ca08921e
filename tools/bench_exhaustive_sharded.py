"""Exhaustive exact search on a document-sharded index: one JSON line per run, printed by rank 0.

    torchrun --nproc_per_node N tools/bench_exhaustive_sharded.py --config cfg3 [--seconds 1.0] [--warmup 2]
    python tools/bench_exhaustive_sharded.py --config cfg2          # world 1, no process group

Every rank generates its document shard of the benchmark's synthetic index (query groups: 1) and searches the same
batch of B x Q queries with fpb_search_exhaustive_sharded.  Reported, with CUDA events over windows of at least
--seconds after warm-up, as the maximum over ranks:
  * the time per batch of the one-call path;
  * the local part alone (fpb_shard_exhaustive_records: K7 over the shard, then the selection), and K7 alone
    (fpb_exhaustive_scores); the exchange is the one-call time minus the local part (all-gather + merge).
At world 1 the one-call path and fpb_search_exhaustive are timed in alternating windows on the same batch.  The
result is checked against fpb_search_exhaustive on one GPU holding the whole index (rank 0 builds it when the
world is larger).  Needs CUDA devices; there is no fallback.
"""

from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import bench  # noqa: E402


def card(index: int) -> dict:
    """Name and power limit of GPU `index`, read in the same run as the measurement."""
    import subprocess

    out = {"name": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:  # the number is reported as unknown rather than guessed
        pass
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2", choices=["cfg2", "cfg3", "tiny"])
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3, help="alternating windows per arm at world 1")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_exhaustive_sharded.py needs CUDA devices (the engine has no CPU path)")
    import torch.distributed as dist

    from fast_plaid_b200.engine import DeviceIndex, IndexTensors, ShardComm, _check

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    device = f"cuda:{local}"
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device(device))
    cfg = bench.CONFIGS[args.config]
    n_docs, B, Q, k = cfg["n_docs"], cfg["B"], cfg["Q"], cfg["top_k"]
    synth = bench.load_synthetic_module()

    def load(lo: int, hi: int):
        arrays, base = synth.synthetic_arrays(n_docs, cfg["doc_len"], bench.DIM, bench.NBITS, device,
                                              bench.SEED_INDEX, doc_range=(lo, hi), topics=cfg.get("topics", 0),
                                              mix=cfg.get("mix", 0.05))
        data = IndexTensors(nbits=arrays.nbits, centroids=arrays.centroids, bucket_weights=arrays.bucket_weights,
                            doc_lengths=arrays.doc_lengths, doc_codes=arrays.doc_codes,
                            doc_residuals=arrays.doc_residuals, ivf=None, ivf_lengths=None)
        return arrays, DeviceIndex(data, device, doc_id_base=base)

    lo, hi = (n_docs * rank) // world, (n_docs * (rank + 1)) // world
    arrays, didx = load(lo, hi)
    # the queries come from documents of rank 0's shard (bench.query_source_docs); rank 0 makes them for everyone
    q16 = torch.empty((B, Q, bench.DIM), dtype=torch.float16, device=device)
    if rank == 0:
        q16.copy_(bench.make_query_batches(arrays, bench.query_source_docs(n_docs), cfg, 1)[0].half())
    del arrays
    if world > 1:
        dist.broadcast(q16, src=0)
    comm = ShardComm.from_process_group(device) if world > 1 else ShardComm(1, 0, ShardComm.new_unique_id(), device)

    lib, h, st = didx._lib, didx._handle, didx._stream()
    ws_bytes = didx.exhaustive_workspace_bytes(B, Q, k)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
    sc_bytes = int(lib.fpb_sharded_scratch_bytes(B, k, world))
    scratch = torch.empty(sc_bytes, dtype=torch.uint8, device=device)
    ids = torch.empty((B, k), dtype=torch.int64, device=device)
    top = torch.empty((B, k), dtype=torch.float32, device=device)
    counts = torch.empty((B,), dtype=torch.int32, device=device)
    rec = torch.empty((B, k, 16), dtype=torch.uint8, device=device)
    scores = torch.empty((B, didx.num_documents), dtype=torch.float32, device=device)

    def run_sharded():
        _check(lib.fpb_search_exhaustive_sharded(h, comm._handle, 1, q16.data_ptr(), B, Q, k, ws.data_ptr(), ws_bytes,
                                                 scratch.data_ptr(), sc_bytes, ids.data_ptr(), top.data_ptr(),
                                                 counts.data_ptr(), st))

    def run_records():
        _check(lib.fpb_shard_exhaustive_records(h, q16.data_ptr(), B, Q, k, ws.data_ptr(), ws_bytes, rec.data_ptr(),
                                                st))

    def run_scores():
        _check(lib.fpb_exhaustive_scores(h, q16.data_ptr(), B, Q, ws.data_ptr(), ws_bytes, scores.data_ptr(), st))

    def run_single():  # world 1 only: the shard is the whole index
        _check(lib.fpb_search_exhaustive(h, q16.data_ptr(), B, Q, k, ws.data_ptr(), ws_bytes, ids.data_ptr(),
                                         top.data_ptr(), counts.data_ptr(), st))

    def worst(ms: float) -> float:  # the slowest rank's time
        if world == 1:
            return ms
        t = torch.tensor([ms], dtype=torch.float64, device=device)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t)

    def timed(fn) -> float:
        """Mean CUDA-event milliseconds per call over a window of at least --seconds after warm-up.  The number of
        calls is agreed over the ranks (from the slowest rank's first call), so that every rank makes the same
        collective calls."""
        for _ in range(args.warmup):
            fn()
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        fn()
        stop.record()
        stop.synchronize()
        reps = max(1, int(args.seconds * 1e3 / max(worst(start.elapsed_time(stop)), 1e-3)) + 1)
        start.record()
        for _ in range(reps):
            fn()
        stop.record()
        stop.synchronize()
        return start.elapsed_time(stop) / reps

    out = {"metric": "exhaustive_sharded_search", "config": args.config, "desc": cfg["desc"], "world": world,
           "query_groups": 1, "B": B, "Q": Q, "top_k": k, "n_docs": n_docs,
           "docs_per_rank": [(n_docs * (r + 1)) // world - (n_docs * r) // world for r in range(world)]}
    cards = [None] * world
    if world > 1:
        dist.all_gather_object(cards, card(local))
    else:
        cards = [card(local)]
    out["cards"] = cards
    # the result against fpb_search_exhaustive on one GPU holding the whole index (rank 0)
    run_sharded()
    got = (ids.cpu(), top.cpu(), counts.cpu())
    if world == 1:
        run_single()
        ref = (ids.cpu(), top.cpu(), counts.cpu())
    elif rank == 0:
        whole = load(0, n_docs)[1]
        ref = tuple(x.cpu() for x in whole.search_exhaustive(q16, k))
        whole.close()
    if rank == 0:
        out["result_equals_unsharded"] = all(torch.equal(a, b) for a, b in zip(got, ref))
    if world > 1:
        dist.barrier()

    if world == 1:
        # alternating windows of the two arms on the same batch and workspace
        one_call, single = [], []
        for _ in range(args.rounds):
            one_call.append(timed(run_sharded))
            single.append(timed(run_single))
        out["one_call_ms"] = [round(x, 3) for x in one_call]
        out["fpb_search_exhaustive_ms"] = [round(x, 3) for x in single]
        out["one_call_minus_single_ms"] = round(min(one_call) - min(single), 3)
    ms_batch = worst(timed(run_sharded))
    ms_local = worst(timed(run_records))
    ms_k7 = worst(timed(run_scores))
    out.update({
        "batch_ms": round(ms_batch, 3),
        "local_records_ms": round(ms_local, 3),
        "k7_ms": round(ms_k7, 3),
        "k7_share": round(ms_k7 / ms_batch, 3),
        "exchange_ms": round(ms_batch - ms_local, 3),
        "note": "every time is the slowest rank's mean over windows of at least --seconds; local_records = K7 + "
                "selection + records on the rank's shard; exchange = batch - local_records (all-gather + merge)",
        "queries_per_s": round(B / (ms_batch * 1e-3), 1),
    })
    if rank == 0:
        print(json.dumps(out), flush=True)
    comm.close()
    didx.close()
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
