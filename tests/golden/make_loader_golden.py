"""Mint tests/golden/ref_loader_index/ and tests/golden/ref_loader.pt for tests/test_index_io.py.

ref_loader_index/ is a small index directory written by this project's builder (FastPlaid.create on the
CPU).  The reference's OWN loader (python/fast_plaid/search/load.py:220-322 of a lightonai/fast-plaid
checkout) then reads it; its module imports the Rust extension at import time, which is stubbed -- the
loader code that runs is the reference's, unmodified.  What it returned is saved in ref_loader.pt, and
the merged mmap caches it wrote stay in the directory.  The raw `embeddings.npy` the builder keeps for
later updates is left out: no loader reads it.

    python tests/golden/make_loader_golden.py <path to a fast-plaid checkout>
"""

import importlib.util
import os
import shutil
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

INDEX = os.path.join(HERE, "ref_loader_index")
OUT = os.path.join(HERE, "ref_loader.pt")
KEYS = ("nbits", "centroids", "bucket_weights", "bucket_cutoffs", "ivf", "ivf_lengths", "doc_lengths", "doc_codes",
        "doc_residuals")


def build_index(path: str) -> None:
    """The directory both the generator and the test build: 60 documents of 4..20 tokens, 3 chunks."""
    from util import make_docs

    from fast_plaid_b200 import search

    search.FastPlaid(path, device="cpu").create(make_docs(60, 4, 20, seed=321), kmeans_niters=2, batch_size=25, seed=7)


def reference_load(checkout: str, path: str) -> dict:
    ref_py = os.path.join(checkout, "python")
    stub = types.ModuleType("fast_plaid.fast_plaid_rust")
    pkg = types.ModuleType("fast_plaid")
    pkg.__path__ = [os.path.join(ref_py, "fast_plaid")]
    pkg.fast_plaid_rust = stub
    srch = types.ModuleType("fast_plaid.search")
    srch.__path__ = [os.path.join(ref_py, "fast_plaid", "search")]
    sys.modules.update({"fast_plaid": pkg, "fast_plaid.fast_plaid_rust": stub, "fast_plaid.search": srch})
    spec = importlib.util.spec_from_file_location("fast_plaid.search.load",
                                                  os.path.join(ref_py, "fast_plaid", "search", "load.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod._load_index_tensors_cpu(index_path=path)


def main():
    torch.set_num_threads(1)
    shutil.rmtree(INDEX, ignore_errors=True)
    build_index(INDEX)
    os.remove(os.path.join(INDEX, "embeddings.npy"))  # raw embeddings kept for updates; no loader reads them
    ref = reference_load(sys.argv[1], INDEX)
    torch.save({"source": "reference python/fast_plaid/search/load.py::_load_index_tensors_cpu, torch " +
                          torch.__version__,
                **{k: ref[k] for k in KEYS}}, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes;", sorted(os.listdir(INDEX)))


if __name__ == "__main__":
    main()
