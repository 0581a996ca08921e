"""Time FastPlaid.delete on a benchmark-sized index: the in-place delete against the host delete and a reload.

Writes the synthetic index of a bench.py config (cfg2 by default, or cfg3) to a directory, then for each case (the
last document, the first document, 1 000 random documents, 1 % of the documents at random) copies it, loads it with
FastPlaid and times one delete on a fresh copy twice: in place (DeviceIndex.delete, files from the compacted arrays)
and with the path that filters every chunk file on the host and loads the directory again (forced here).  Per run:
seconds; for the in-place path the part spent in DeviceIndex.delete (device work) and the rest (file writes); the
peak of the device's memory in use sampled every 2 ms; the growable buffers' mapped bytes after; and, in place, the
CUDA-event times of the fpb_docs_compact, fpb_ivf_delete and fpb_index_create calls, with fpb_docs_compact's
achieved bytes/s (rows read and written over the time of its copying call) against the H100's 3.35 TB/s.  A second,
untimed in-place delete of each case runs under torch.profiler first, for the device time of each kernel.  One JSON
line per run, the first with the card's name and power limit.

    python tools/bench_delete.py [--config cfg2] [--cases last first random1000 random1pct] [--dir /tmp/x]
"""

from __future__ import annotations

import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time
from collections import defaultdict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench import CONFIGS, DIM, NBITS  # noqa: E402
from bench_update import PeakSampler, write_index  # noqa: E402
from fast_plaid_b200 import search  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
TIMED = ("fpb_docs_compact", "fpb_ivf_delete", "fpb_index_create")


class TimedLib:
    """The C-ABI library with CUDA events around every call of the TIMED entry points (milliseconds, in call order;
    each of the first two is called once to size its output and once to write it)."""

    def __init__(self, lib) -> None:
        self._lib = lib
        self.ms: dict[str, list[float]] = defaultdict(list)

    def __getattr__(self, name: str):
        fn = getattr(self._lib, name)
        if name not in TIMED:
            return fn

        def timed(*args):
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            rc = fn(*args)
            end.record()
            end.synchronize()
            self.ms[name].append(round(start.elapsed_time(end), 3))
            return rc

        return timed


def cases(n_docs: int) -> dict[str, list[int]]:
    g = torch.Generator().manual_seed(17)
    return {"last": [n_docs - 1], "first": [0],
            "random1000": torch.randperm(n_docs, generator=g)[:1000].tolist(),
            "random1pct": torch.randperm(n_docs, generator=g)[: n_docs // 100].tolist()}


def kernel_ms(idx, drop: list[int]) -> dict[str, float]:
    """Device milliseconds per kernel of one in-place delete of `idx` (the result is discarded)."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        shrunk = idx.delete(drop)
        torch.cuda.synchronize(idx.device)
    del shrunk
    out: dict[str, float] = defaultdict(float)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            m = re.search(r"([A-Za-z_]\w*)(?:<[^()]*>)?\(", e.name)  # the function name of a kernel's signature
            out[m.group(1) if m else e.name[:40]] += e.device_time_total / 1e3
    return {k: round(v, 3) for k, v in sorted(out.items(), key=lambda kv: -kv[1])}


def run(base: str, work: str, case: str, drop: list[int], mode: str, device: str) -> dict:
    shutil.rmtree(work, ignore_errors=True)
    shutil.copytree(base, work)
    fp = search.FastPlaid(work, device=device)
    idx = fp.indices[device]
    out = dict(case=case, mode=mode, dropped=len(drop))
    if mode == "reload":
        fp._appendable = lambda: None
    else:
        out["kernel_ms"] = kernel_ms(idx, drop)
        torch.cuda.empty_cache()
        lib = idx._lib = TimedLib(idx._lib)
        inner = idx.delete
        device_s = []

        def delete(doc_ids):
            t = time.perf_counter()
            r = inner(doc_ids)
            torch.cuda.synchronize(device)
            device_s.append(time.perf_counter() - t)
            return r

        idx.delete = delete
    del idx
    torch.cuda.synchronize(device)
    with PeakSampler(device) as ps:
        t0 = time.perf_counter()
        fp.delete(drop)
        torch.cuda.synchronize(device)
        secs = time.perf_counter() - t0
    new = fp.indices[device]
    out.update(seconds=round(secs, 3), peak_device_in_use=ps.peak, mapped_after=new.growable.mapped_bytes,
               num_documents=new.num_documents)
    if mode == "inplace":
        assert len(device_s) == 1, "the in-place path did not run"
        out.update(device_seconds=round(device_s[0], 3), file_seconds=round(secs - device_s[0], 3))
        out["call_ms"] = dict(lib.ms)
        moved = 2 * new.num_tokens * (4 + DIM * NBITS // 8)  # codes and residual rows, read and written
        copy_ms = lib.ms["fpb_docs_compact"][-1]
        out.update(compact_bytes=moved, compact_bytes_per_s=round(moved / (copy_ms / 1e3)),
                   compact_share_of_hbm_peak=round(moved / (copy_ms / 1e3) / HBM_BYTES_PER_S, 3))
    fp.close()
    del fp, new
    torch.cuda.empty_cache()
    shutil.rmtree(work, ignore_errors=True)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2", choices=["cfg2", "cfg3"])
    ap.add_argument("--cases", nargs="+", default=list(cases(1)), choices=list(cases(1)))
    ap.add_argument("--dir", default=None, help="where to write the index (default: a temporary directory)")
    args = ap.parse_args()
    device = "cuda:0"
    if not torch.cuda.is_available():
        raise SystemExit("bench_delete.py needs a CUDA device")
    root = args.dir or tempfile.mkdtemp(prefix="fpb_delete_")
    cfg = CONFIGS[args.config]
    need = cfg["n_docs"] * cfg["doc_len"] * (8 + DIM * NBITS // 8) * 2.5  # the index, one copy, the IVF and slack
    if shutil.disk_usage(root).free < need:
        print(json.dumps({"config": args.config, "skipped": f"needs ~{need / 1e9:.0f} GB of disk"}))
        return
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    base = os.path.join(root, "base")
    t0 = time.perf_counter()
    size = write_index(base, cfg, device)
    print(json.dumps({"config": args.config, "gpu": gpu, "index_bytes_on_disk": size,
                      "write_seconds": round(time.perf_counter() - t0, 1)}), flush=True)
    for case, drop in cases(cfg["n_docs"]).items():
        if case not in args.cases:
            continue
        for mode in ("inplace", "reload"):
            r = run(base, os.path.join(root, "work"), case, drop, mode, device)
            print(json.dumps({"config": args.config, **r}), flush=True)
    shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
