"""Mint tests/golden/kmeans_ref.pt by running the REFERENCE's own k-means code.

The Lloyd loop the reference layers on the (absent) third-party `fastkmeans` package lives in
python/fast_plaid/search/kmeans.py:60-223 of a lightonai/fast-plaid checkout and is plain PyTorch.  This script
imports that file unmodified -- only `fastkmeans` itself is stubbed with an empty base class --
seeds the RNG exactly as `FastKMeans.train` does (kmeans.py:236-238) and records inputs and
outputs.  tests/test_oracle.py then requires oracle/index_oracle.py::kmeans to reproduce the
recorded centroids, which pins that part of the oracle on reference outputs.  A second file,
kmeans_ref_seed99.pt, holds the reference's centroids for one more problem that the test
regenerates from its seed.

    python tests/golden/make_kmeans_golden.py <path to a fast-plaid checkout>
"""

import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "kmeans_ref.pt")
OUT_SEED99 = os.path.join(HERE, "kmeans_ref_seed99.pt")


def seed99_problem() -> torch.Tensor:
    """The extra problem of kmeans_ref_seed99.pt (k=32, niters=3, seed=5, max_points_per_centroid=256)."""
    g = torch.Generator().manual_seed(99)
    return torch.nn.functional.normalize(torch.randn(1500, 24, generator=g), dim=-1).half()


def load_reference_kmeans(checkout: str):
    stub = types.ModuleType("fastkmeans")

    class FastKMeans:  # the third-party base class; never instantiated here
        pass

    stub.FastKMeans = FastKMeans
    sys.modules.setdefault("fastkmeans", stub)
    ref = os.path.join(checkout, "python", "fast_plaid", "search", "kmeans.py")
    spec = importlib.util.spec_from_file_location("ref_kmeans", ref)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def run_case(mod, data_f16: torch.Tensor, k: int, niters: int, seed: int, mppc: int):
    # FastKMeans.train (kmeans.py:236-241): seeds, then norms in the data's own dtype
    torch.manual_seed(seed)
    np.random.seed(seed)
    norms = (data_f16**2).sum(dim=1)
    centroids, labels = mod._kmeans_torch_double_chunked(
        data_f16, norms, k=k, device=torch.device("cpu"), dtype=None, max_iters=niters, tol=1e-8,
        chunk_size_data=51_200, chunk_size_centroids=10_240, max_points_per_centroid=mppc, use_triton=False)
    return centroids, labels


def main():
    torch.set_num_threads(1)  # the fixture must not depend on the blocking of a threaded GEMM
    mod = load_reference_kmeans(sys.argv[1])
    g = torch.Generator().manual_seed(2024)
    cases = []
    # (n, dim, k, niters, seed, max_points_per_centroid)
    for n, dim, k, niters, seed, mppc in [(3000, 32, 64, 4, 42, 256),     # plain
                                          (2600, 64, 8, 4, 7, 256),       # subsampling: n > k*mppc
                                          (600, 16, 256, 3, 11, 256)]:    # many clusters -> empty-cluster reseed
        mix = torch.randn(k if k < 100 else 20, dim, generator=g)
        x = mix[torch.randint(0, mix.shape[0], (n,), generator=g)] + 0.3 * torch.randn(n, dim, generator=g)
        x = torch.nn.functional.normalize(x, dim=-1).half()
        c, labels = run_case(mod, x, k, niters, seed, mppc)
        cases.append(dict(data=x, k=k, niters=niters, seed=seed, max_points_per_centroid=mppc,
                          centroids=c, labels=labels))
        print(f"n={n} dim={dim} k={k}: centroids {tuple(c.shape)}, empty-safe, labels {tuple(labels.shape)}")
    torch.save({"source": "reference python/fast_plaid/search/kmeans.py::_kmeans_torch_double_chunked, "
                          "torch " + torch.__version__ + ", CPU, 1 thread",
                "cases": cases}, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")
    c, _ = run_case(mod, seed99_problem(), 32, 3, 5, 256)
    torch.save({"source": "reference python/fast_plaid/search/kmeans.py::_kmeans_torch_double_chunked, "
                          "torch " + torch.__version__ + ", CPU, 1 thread", "centroids": c}, OUT_SEED99)
    print("wrote", OUT_SEED99, os.path.getsize(OUT_SEED99), "bytes")


if __name__ == "__main__":
    main()
