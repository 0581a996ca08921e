"""GPU index-build encode kernels (fpb_encode) against the oracle's create.rs restatement."""

from __future__ import annotations

import pytest
import torch

from util import make_docs

from oracle import index_oracle as io

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("nbits", [4, 2])
def test_encode_matches_oracle(nbits, cuda_device):
    from fast_plaid_b200.engine import encode_tokens

    g = torch.Generator().manual_seed(17)
    K, n = 1000, 5000  # K not a multiple of 128: the last centroid tile is partial
    cent = torch.nn.functional.normalize(torch.randn(K, 128, generator=g), dim=-1).half()
    x = torch.nn.functional.normalize(torch.randn(n, 128, generator=g), dim=-1).half()
    ref_codes = io.compress_into_codes(x, cent)
    res = (x - cent.index_select(0, ref_codes)).float().flatten()
    n_opt = 2 ** nbits
    cutoffs = torch.cat([io.scalar_quantile_kthvalue(res, i / n_opt) for i in range(1, n_opt)])
    codes, packed = encode_tokens(x.to(cuda_device), cent, cutoffs, nbits)
    torch.cuda.synchronize()
    codes, packed = codes.cpu().long(), packed.cpu()
    same = codes == ref_codes
    assert float(same.float().mean()) > 0.999, f"only {float(same.float().mean()):.5f} of the codes agree"
    # where the argmax differs the two centroids score within one fp16 ulp of each other (accumulation order)
    bad = (~same).nonzero().flatten()
    if bad.numel():
        sc = x[bad].float() @ cent.float().t()
        a = sc.gather(1, codes[bad, None]).half().float()
        b = sc.gather(1, ref_codes[bad, None]).half().float()
        assert float((a - b).abs().max()) <= 2.0 ** -10
    # residual bytes: reference packing of the residuals w.r.t. OUR codes (create.rs:413-427)
    r = x - cent.index_select(0, codes)
    bk = torch.bucketize(r, cutoffs, out_int32=True, right=False)
    bits = bk.unsqueeze(-1).expand(n, 128, nbits).bitwise_right_shift(torch.arange(nbits, dtype=torch.int8)) & 1
    ref_packed = io.packbits(bits.flatten()).reshape(n, 128 * nbits // 8)
    assert torch.equal(packed, ref_packed)


def test_create_on_gpu_uses_the_kernels_and_matches_the_cpu_builder(tmp_path, cuda_device):
    from fast_plaid_b200 import search
    from fast_plaid_b200.index import store

    docs = make_docs(200, 10, 50, seed=41)
    a = search.FastPlaid(str(tmp_path / "gpu"), device=cuda_device)
    a.create(docs, kmeans_niters=2, seed=5)
    da = store.read_index(str(tmp_path / "gpu"))
    # same centroids and cutoffs through the oracle's CPU encoder
    oidx, extra = io.build_index(docs, da.centroids, nbits=4, seed=5)
    agree = (oidx.doc_codes == da.doc_codes).float().mean()
    assert float(agree) > 0.995
    assert da.doc_residuals.shape == oidx.doc_residuals.shape
    a.close()


def test_kmeans_kernels_match_torch(cuda_device):
    """fpb_kmeans_assign (wgmma argmax of <x,c> - |c|^2/2) against the fp32 nearest-centroid search, and
    fpb_kmeans_update (deterministic segmented mean) against index_add_; un-normalised centroids, K not a
    multiple of 128, a cluster left empty."""
    from fast_plaid_b200.engine import kmeans_assign, kmeans_update

    g = torch.Generator().manual_seed(3)
    K, n = 700, 20_000
    cent = (torch.randn(K, 128, generator=g) * torch.rand(K, 1, generator=g)).half()
    cent[5] = 100.0  # far away: never the nearest -> empty cluster
    x = torch.randn(n, 128, generator=g).half()
    xd, cd = x.to(cuda_device), cent.to(cuda_device)
    assign = kmeans_assign(xd, cd)
    torch.cuda.synchronize()
    d2 = (xd.float() ** 2).sum(1, keepdim=True) + (cd.float() ** 2).sum(1)[None] - 2.0 * xd.float() @ cd.float().t()
    ref = d2.argmin(1)
    same = assign.long() == ref
    assert float(same.float().mean()) > 0.999
    bad = (~same).nonzero().flatten()
    if bad.numel():  # a different pick only between two centroids at (almost) the same distance
        a = d2[bad, assign.long()[bad]]
        b = d2[bad, ref[bad]]
        assert float(((a - b).abs() / b.abs().clamp_min(1.0)).max()) < 2e-3
    new = cd.clone()
    counts, shift = kmeans_update(xd, assign, new)
    torch.cuda.synchronize()
    sums = torch.zeros(K, 128, device=cuda_device).index_add_(0, assign.long(), xd.float())
    cnt = torch.bincount(assign.long(), minlength=K)
    assert torch.equal(counts, cnt) and int(cnt[5]) == 0
    ne = cnt > 0
    want = (sums[ne] / cnt[ne, None]).half()
    assert torch.allclose(new[ne].float(), want.float(), atol=2e-3, rtol=2e-3)
    assert torch.equal(new[~ne], cd[~ne])  # empty clusters untouched
    assert torch.allclose(shift[ne], (new[ne].float() - cd[ne].float()).norm(dim=1), atol=1e-2, rtol=1e-2)
    # deterministic
    again = cd.clone()
    kmeans_update(xd, assign, again)
    assert torch.equal(again, new)


def test_gpu_lloyd_kmeans_reaches_the_quality_of_the_cpu_loop(cuda_device):
    """The sm_90a Lloyd loop and the oracle's CPU loop start from the same seeded initial centroids and must end
    at the same clustering quality (inertia within 2 %): the reference's own CUDA path differs from its CPU path
    in exactly this way (fp16 tensor-core distances, kmeans.py:113-114)."""
    from fast_plaid_b200.index import build

    g = torch.Generator().manual_seed(9)
    centers = torch.randn(64, 128, generator=g)
    data = torch.nn.functional.normalize(centers[torch.randint(0, 64, (30_000,), generator=g)]
                                         + 0.3 * torch.randn(30_000, 128, generator=g), dim=-1)
    k = 256

    def inertia(c):
        d = torch.cdist(data, c.float())
        return float(d.min(1).values.pow(2).sum())

    c_gpu = build.lloyd_kmeans(data, k, 4, seed=42, device=torch.device(cuda_device))
    c_cpu = io.kmeans(data, k, 4, seed=42) if hasattr(io, "kmeans") else build.lloyd_kmeans(data, k, 4, 42, torch.device("cpu"))
    assert c_gpu.shape == (k, 128)
    a, b = inertia(c_gpu), inertia(c_cpu)
    assert abs(a - b) / b < 0.02, (a, b)
