"""1-bit against 4-bit residuals on the benchmark's synthetic indexes: one JSON line.

    python tools/bench_nbits.py [--config cfg3] [--seconds 1.0] [--rounds 3] [--big-docs 4000000]

Builds the same synthetic index (same codes, same centroids) at nbits 4 and at nbits 1 and, in one process, alternates
between the two for every measurement:
  * HBM held by each DeviceIndex: the torch.cuda.memory_allocated delta of building it, next to the bytes per token
    computed from the layout (residual row + int32 code + fp16 norm + walk-layout code + IVF entry);
  * search() per batch (default parameters of bench.py) and the MaxSim stage alone on the same re-rank lists;
  * search_exhaustive on cfg2.
Times are CUDA-event means over windows of at least --seconds after warm-up; every round times both indexes, and the
median over the rounds is reported.  With --big-docs N, after the others are freed, an nbits-1 index of N documents
(300 tokens each) is built and searched if the card's free memory allows; otherwise the output says it did not fit.
The residual codes are random: nothing here measures retrieval quality.  Needs a CUDA device.
"""

from __future__ import annotations

import argparse
import gc
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

DEVICE = "cuda:0"


def build(cfg: dict, nbits: int, n_docs: int | None = None):
    """(DeviceIndex, HBM bytes it holds, query batch or None) of the config's synthetic index at `nbits`.  The query
    batch is bench.py's (noisy copies of decoded tokens), made at nbits 4 only: its decoder knows that width alone."""
    from fast_plaid_b200.engine import DeviceIndex, IndexTensors

    n_docs = n_docs or cfg["n_docs"]
    gc.collect()
    torch.cuda.empty_cache()
    m0 = torch.cuda.memory_allocated(DEVICE)
    synth = bench.load_synthetic_module()
    a, base = synth.synthetic_arrays(n_docs, cfg["doc_len"], bench.DIM, nbits, DEVICE, bench.SEED_INDEX,
                                     doc_range=(0, n_docs), topics=cfg.get("topics", 0), mix=cfg.get("mix", 0.05))
    q = bench.make_query_batches(a, bench.query_source_docs(n_docs), cfg, 1)[0] if nbits == bench.NBITS else None
    data = IndexTensors(nbits=a.nbits, centroids=a.centroids, bucket_weights=a.bucket_weights,
                        doc_lengths=a.doc_lengths, doc_codes=a.doc_codes, doc_residuals=a.doc_residuals,
                        ivf=a.ivf, ivf_lengths=a.ivf_lengths)
    didx = DeviceIndex(data, DEVICE, doc_id_base=base)
    del a, data
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    held = torch.cuda.memory_allocated(DEVICE) - m0
    return didx, held, None if q is None else q.to(DEVICE).half().contiguous()


def layout_bytes_per_token(nbits: int) -> int:
    """Upper bound from the layout: residual row, int32 code, fp16 norm, walk-layout code, one IVF entry."""
    return bench.DIM * nbits // 8 + 4 + 2 + 4 + 4


def median_rounds(fns: dict, seconds: float, warmup: int, rounds: int) -> dict:
    """Alternate the timed functions round by round; the median ms of each."""
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            ms[k].append(timed(fn, seconds, warmup)[0])
    return {k: {"median_ms": round(statistics.median(v), 3), "rounds_ms": [round(x, 3) for x in v]} for k, v in ms.items()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg3", choices=["cfg3", "cfg3c", "cfg2", "tiny"])
    ap.add_argument("--exhaustive-config", default="cfg2", choices=["cfg2", "tiny"])
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--big-docs", type=int, default=0, help="documents of the large nbits-1 index (0: skip)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nbits.py needs a CUDA device (the engine has no CPU path)")
    from fast_plaid_b200.engine import DeviceIndex

    out = {"metric": "nbits1_vs_nbits4", "card": card(), "config": args.config}
    cfg = bench.CONFIGS[args.config]
    params = DeviceIndex.make_params(cfg["top_k"], bench.N_FULL, bench.N_IVF_PROBE)

    # ---- search() and MaxSim on the main config ----
    idx, q = {}, None
    for nb in (4, 1):
        didx, held, qq = build(cfg, nb)
        q = qq if q is None else q  # the nbits-4 batch for both: the codes and centroids are the same
        idx[nb] = didx
        out[f"nbits{nb}_index"] = {"hbm_bytes": held, "tokens": didx.num_tokens,
                                   "hbm_bytes_per_token": round(held / didx.num_tokens, 2),
                                   "layout_bytes_per_token_max": layout_bytes_per_token(nb)}
    fns = {}
    for nb, didx in idx.items():
        fns[f"search_nbits{nb}"] = lambda d=didx: d.search(q, params)
        didx.run_stages(q, params)  # leaves this batch's re-rank lists in the workspace for the MaxSim stage
        fns[f"maxsim_nbits{nb}"] = didx.stage_fn("maxsim", q, params)
    # the MaxSim stage reads the re-rank lists of the workspace: time each index's stage right after its own
    # run_stages, alternating the indexes round by round
    res = {}
    for _ in range(args.rounds):
        for nb, didx in idx.items():
            res.setdefault(f"search_nbits{nb}", []).append(timed(fns[f"search_nbits{nb}"], args.seconds, args.warmup)[0])
            didx.run_stages(q, params)
            res.setdefault(f"maxsim_nbits{nb}", []).append(timed(fns[f"maxsim_nbits{nb}"], args.seconds, args.warmup)[0])
    for k, v in res.items():
        out[k] = {"median_ms": round(statistics.median(v), 3), "rounds_ms": [round(x, 3) for x in v]}
    # result agreement of the two widths (informational: 1-bit residuals change the scores)
    i4, _, c4 = idx[4].search(q, params)
    i1, _, c1 = idx[1].search(q, params)
    torch.cuda.synchronize()
    shared = sum(len(set(i4[b, : int(c4[b])].tolist()) & set(i1[b, : int(c1[b])].tolist())) for b in range(q.shape[0]))
    out["top_k_overlap_nbits1_vs_nbits4"] = round(shared / max(1, int(c4.sum())), 4)
    out["overlap_note"] = "synthetic random residuals: not a retrieval-quality figure"
    del idx, fns
    gc.collect()
    torch.cuda.empty_cache()

    # ---- exhaustive search on cfg2 ----
    ecfg = bench.CONFIGS[args.exhaustive_config]
    eidx, eq = {}, None
    for nb in (4, 1):
        didx, held, qq = build(ecfg, nb)
        eq = qq if eq is None else eq
        eidx[nb] = didx
    k = ecfg["top_k"]
    ex = median_rounds({f"search_exhaustive_nbits{nb}": (lambda d=d: d.search_exhaustive(eq, k)) for nb, d in eidx.items()},
                       args.seconds, args.warmup, args.rounds)
    out["exhaustive_config"] = args.exhaustive_config
    out.update(ex)
    del eidx
    gc.collect()
    torch.cuda.empty_cache()

    # ---- an nbits-1 index that nbits 4 could not hold ----
    if args.big_docs:
        n = args.big_docs
        need = n * cfg["doc_len"] * layout_bytes_per_token(1)
        free, total = torch.cuda.mem_get_info(0)
        big = {"n_docs": n, "nbits4_bytes_estimate": n * cfg["doc_len"] * layout_bytes_per_token(4),
               "nbits1_bytes_estimate": need, "free_bytes_before": free, "total_bytes": total}
        if need * 1.6 > free:  # the IVF build sorts every code, and needs temporaries of the same order
            big["result"] = "not run: the free memory of the card does not leave room to build it"
        else:
            try:
                didx, held, _ = build(cfg, 1, n_docs=n)
                big["hbm_bytes"] = held
                big["hbm_bytes_per_token"] = round(held / didx.num_tokens, 2)
                big["search"] = median_rounds({"search": lambda: didx.search(q, params)}, args.seconds, args.warmup, 1)
                big["query_note"] = "the main config's query batch"
                big["result"] = "ok"
                del didx
            except torch.cuda.OutOfMemoryError as e:  # reported, not retried
                big["result"] = f"out of memory: {str(e).splitlines()[0]}"
        out["big_nbits1"] = big
    print(json.dumps(out))


if __name__ == "__main__":
    main()
