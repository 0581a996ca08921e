"""Time FastPlaid.update on a benchmark-sized index: the in-place append against a reload of the directory.

Writes the synthetic index of a bench.py config (cfg2 by default; cfg3 too with --config cfg3 when the disk holds it)
to a directory, then for each batch size (1 000 and 10 000 documents of 300 tokens by default) copies it, loads it
with FastPlaid and times one update twice on fresh copies: with the in-place append (DeviceIndex.append) and with the
path that rebuilds the inverted file from the chunk files and loads the directory again (forced here).  Reports
seconds, the growable buffers' mapped bytes before and after, torch's peak allocated bytes during the update, and
the peak of the device's memory in use sampled every 2 ms during the update.  One JSON line per run.

    python tools/bench_update.py [--config cfg2] [--docs 1000 10000] [--dir /tmp/x]
"""

from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CONFIGS, DIM, NBITS, SEED_INDEX  # noqa: E402
from fast_plaid_b200 import search  # noqa: E402
from fast_plaid_b200.index import store, synthetic  # noqa: E402


def write_index(path: str, cfg: dict, device: str) -> int:
    """The synthetic index of `cfg` as an index directory; returns its bytes on disk."""
    arrays, _ = synthetic.synthetic_arrays(cfg["n_docs"], cfg["doc_len"], DIM, NBITS, device, SEED_INDEX)
    os.makedirs(path, exist_ok=True)
    w = arrays.bucket_weights.float().cpu()
    cutoffs = (w[1:] + w[:-1]) / 2  # bucket boundaries halfway between the weights
    K = int(arrays.centroids.shape[0])
    store.write_codec(path, arrays.centroids, cutoffs, w, w.abs().mean().reshape(1), torch.zeros(K))
    lens = arrays.doc_lengths.to(torch.int64).cpu()
    per_chunk = 25_000
    emb = 0
    n_chunks = 0
    for c0 in range(0, int(lens.shape[0]), per_chunk):
        cl = lens[c0 : c0 + per_chunk]
        n = int(cl.sum())
        store.write_chunk(path, n_chunks, arrays.doc_codes[emb : emb + n], arrays.doc_residuals[emb : emb + n],
                          cl.tolist(), emb)
        emb += n
        n_chunks += 1
    store.write_plan(path, NBITS, n_chunks)
    store.write_ivf(path, arrays.ivf, arrays.ivf_lengths)
    store.write_metadata(path, num_chunks=n_chunks, nbits=NBITS, num_partitions=K, num_embeddings=emb,
                         num_documents=int(lens.shape[0]), compress_only=False)
    del arrays
    torch.cuda.empty_cache()
    return sum(os.path.getsize(os.path.join(path, f)) for f in os.listdir(path))


class PeakSampler:
    """Device memory in use (total - free), sampled on a thread while the block runs."""

    def __init__(self, device: str) -> None:
        self.device = torch.device(device)
        self.peak = 0
        self._stop = threading.Event()

    def _run(self) -> None:
        while not self._stop.is_set():
            free, total = torch.cuda.mem_get_info(self.device)
            self.peak = max(self.peak, total - free)
            time.sleep(0.002)

    def __enter__(self):
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *a) -> None:
        self._stop.set()
        self._t.join()


def new_docs(n: int, doc_len: int, seed: int) -> list[torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    x = torch.nn.functional.normalize(torch.randn(n, doc_len, DIM, generator=g), dim=-1).half()
    return list(x)


def run(base: str, work: str, n_docs: int, doc_len: int, mode: str, device: str) -> dict:
    shutil.rmtree(work, ignore_errors=True)
    shutil.copytree(base, work)
    fp = search.FastPlaid(work, device=device)
    if mode == "reload":
        fp._appendable = lambda: None
    idx = fp.indices[device]
    mapped_before = idx.growable.mapped_bytes
    docs = new_docs(n_docs, doc_len, seed=n_docs)
    torch.cuda.synchronize(device)
    torch.cuda.reset_peak_memory_stats(device)
    with PeakSampler(device) as ps:
        t0 = time.perf_counter()
        fp.update(docs, start_from_scratch=0)
        torch.cuda.synchronize(device)
        secs = time.perf_counter() - t0
    idx = fp.indices[device]
    out = dict(mode=mode, new_docs=n_docs, doc_len=doc_len, seconds=round(secs, 3),
               mapped_before=mapped_before, mapped_after=idx.growable.mapped_bytes,
               peak_allocated=torch.cuda.max_memory_allocated(device), peak_device_in_use=ps.peak,
               num_documents=idx.num_documents)
    fp.close()
    del fp, idx
    torch.cuda.empty_cache()
    shutil.rmtree(work, ignore_errors=True)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2", choices=list(CONFIGS))
    ap.add_argument("--docs", type=int, nargs="+", default=[1000, 10000])
    ap.add_argument("--doc-len", type=int, default=300)
    ap.add_argument("--dir", default=None, help="where to write the index (default: a temporary directory)")
    args = ap.parse_args()
    device = "cuda:0"
    if not torch.cuda.is_available():
        raise SystemExit("bench_update.py needs a CUDA device")
    root = args.dir or tempfile.mkdtemp(prefix="fpb_update_")
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
    for n in args.docs:
        for mode in ("append", "reload"):
            r = run(base, os.path.join(root, "work"), n, args.doc_len, mode, device)
            print(json.dumps({"config": args.config, **r}), flush=True)
    shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
