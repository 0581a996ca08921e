"""Where the approximate stage (K3) spends its time, kernel by kernel, on a bench.py workload.

Builds the workload's index and query batches exactly as bench.py does, then runs the pipeline stage by stage on
one GPU and reports:
  * the approximate stage's time per batch from CUDA events (profiler off), for each FPB_K3_LAMBDA value asked for
    (--lambdas; the values are interleaved batch by batch so that they see the same conditions);
  * per-kernel CUDA times of one batch's K3 launches (k3_tau, k3_hibits, k3_bound, k3_refine_list, the exact
    pass) from torch.profiler, in a separate run at the default lambda.
Every lambda gives the same results; it only moves work between the bound pass and the exact pass.

    python tools/profile_approx.py --config cfg3 --reps 20 --lambdas default,1.5,2.0,2.5 --out result.json
"""

from __future__ import annotations

import argparse
import ctypes
import json
import os
import re
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402

KERNELS = [  # (label, kernel-name pattern) in launch order
    ("k3_tau", r"k3_tau_kernel"),
    ("k3_hibits", r"k3_hibits_kernel"),
    ("k3_prefix", r"k3_prefix_kernel"),
    ("k3_bound", r"k3_bound_kernel"),
    ("k3_refine_list", r"k3_refine_list_kernel"),
    ("exact_pass", r"k3_exact_kernel"),
]


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:  # the numbers still stand; say that the card could not be read
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e!r:.80})"}


def set_lambda(value: str) -> None:
    if value == "default":
        os.environ.pop("FPB_K3_LAMBDA", None)
    else:
        os.environ["FPB_K3_LAMBDA"] = value


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--config", choices=list(bench.CONFIGS), default="cfg3")
    ap.add_argument("--reps", type=int, default=20, help="timed batches per lambda value")
    ap.add_argument("--profile-reps", type=int, default=4, help="batches traced by torch.profiler")
    ap.add_argument("--lambdas", default="default", help="comma-separated FPB_K3_LAMBDA values ('default' = unset)")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profile_approx.py needs a CUDA device")
    from fast_plaid_b200.engine import DeviceIndex, IndexTensors, _check

    device = "cuda:0"
    torch.cuda.set_device(0)
    cfg = bench.CONFIGS[args.config]
    synth = bench.load_synthetic_module()
    arrays, _ = synth.synthetic_arrays(cfg["n_docs"], cfg["doc_len"], bench.DIM, bench.NBITS, device, bench.SEED_INDEX,
                                       topics=cfg.get("topics", 0), mix=cfg.get("mix", 0.05))
    data = IndexTensors(nbits=arrays.nbits, centroids=arrays.centroids, bucket_weights=arrays.bucket_weights,
                        doc_lengths=arrays.doc_lengths, doc_codes=arrays.doc_codes, doc_residuals=arrays.doc_residuals,
                        ivf=arrays.ivf, ivf_lengths=arrays.ivf_lengths)
    didx = DeviceIndex(data, device)
    params = DeviceIndex.make_params(cfg["top_k"], bench.N_FULL, bench.N_IVF_PROBE)
    B, Q = cfg["B"], cfg["Q"]
    q_host = bench.make_query_batches(arrays, min(bench.query_source_docs(cfg["n_docs"]), cfg["n_docs"]), cfg,
                                      bench.N_QUERY_BATCHES)
    del data, arrays
    q_dev = q_host.to(device).half()
    lib, h = didx._lib, didx._handle
    buf, lay = didx.workspace(B, Q, params)
    st = didx._stream()
    pp = ctypes.byref(params)

    def front(qb: torch.Tensor) -> None:  # the stages before K3: S, probed cells, candidates
        _check(lib.fpb_stage_centroid_scores(h, qb.data_ptr(), B, Q, pp, buf.data_ptr(), buf.numel(), st))
        _check(lib.fpb_stage_probe(h, B, Q, pp, buf.data_ptr(), buf.numel(), st))
        _check(lib.fpb_stage_candidates(h, B, Q, pp, buf.data_ptr(), buf.numel(), st))

    def approx() -> None:
        _check(lib.fpb_stage_approx(h, B, Q, pp, buf.data_ptr(), buf.numel(), st))

    lambdas = [s.strip() for s in args.lambdas.split(",") if s.strip()]
    # warm-up: every batch and every lambda once
    for lam in lambdas:
        set_lambda(lam)
        for i in range(bench.N_QUERY_BATCHES):
            front(q_dev[i])
            approx()
    torch.cuda.synchronize()

    # ---- approximate-stage time per batch (CUDA events, no profiler) ----
    times: dict[str, list[float]] = {lam: [] for lam in lambdas}
    for r in range(args.reps):
        for k in range(len(lambdas)):
            lam = lambdas[(r + k) % len(lambdas)]  # rotate the order from one batch to the next
            set_lambda(lam)
            front(q_dev[r % bench.N_QUERY_BATCHES])
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            approx()
            e1.record()
            e1.synchronize()
            times[lam].append(e0.elapsed_time(e1))
    set_lambda("default")
    stage = {lam: {"median_ms": round(statistics.median(v), 4), "mean_ms": round(statistics.fmean(v), 4),
                   "min_ms": round(min(v), 4), "max_ms": round(max(v), 4)} for lam, v in times.items()}

    # ---- per-kernel split (torch.profiler, a run of its own) ----
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for r in range(args.profile_reps):
            front(q_dev[r % bench.N_QUERY_BATCHES])
            approx()
        torch.cuda.synchronize()
    split = {label: 0.0 for label, _ in KERNELS}
    launches = {label: 0 for label, _ in KERNELS}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0.0)
        for label, pat in KERNELS:
            if re.search(pat, ev.key):
                split[label] += t / 1000.0 / args.profile_reps
                launches[label] += ev.count
                break
    split = {k: round(v, 4) for k, v in split.items()}
    split["sum_of_k3_kernels"] = round(sum(split.values()), 4)

    out = {
        "gpu": gpu_info(),
        "config": f"{args.config}: {cfg['desc']}",
        "approx_stage_ms_per_batch": stage,
        "k3_kernel_ms_per_batch": split,
        "k3_launches": launches,
        "candidates_per_query_mean": float(didx.views(buf, lay)["n_cand"].float().mean()),
        "reps": args.reps,
        "profile_reps": args.profile_reps,
    }
    didx.close()
    torch.cuda.synchronize()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
