"""The approximate stage's walk layout (csrc/common.cuh, k3_walk_layout_kernel): every document's codes dealt over
ceil(len/32) windows of its own with the bitmap banks spread, padding that tests a zero word in a free bank, and
approximate scores that do not depend on the token order."""

from __future__ import annotations

import math

import pytest
import torch

pytestmark = pytest.mark.gpu

# lengths every index holds: empty, single token, around one and two windows, long
EDGE_LENGTHS = [0, 1, 31, 32, 33, 63, 64, 65, 0, 300, 1000, 2]
N_RANDOM_DOCS = 400
DIM = 128

_cache: dict = {}


def _index(K: int, device: str):
    """A ragged index over K centroids: random lengths plus EDGE_LENGTHS, uniform codes, and a few documents whose
    codes all sit in one bank (or are one code)."""
    if K in _cache:
        return _cache[K]
    from fast_plaid_b200.engine import DeviceIndex, IndexTensors
    from fast_plaid_b200.index.layout import build_ivf

    g = torch.Generator().manual_seed(K)
    lens = torch.cat([torch.randint(0, 121, (N_RANDOM_DOCS,), generator=g), torch.tensor(EDGE_LENGTHS)])
    codes = torch.randint(0, K, (int(lens.sum()),), generator=g, dtype=torch.int32)
    offs = torch.zeros(lens.shape[0] + 1, dtype=torch.int64)
    offs[1:] = lens.cumsum(0)
    for j, d in enumerate(range(N_RANDOM_DOCS - 6, N_RANDOM_DOCS)):  # skewed documents
        a, b = int(offs[d]), int(offs[d + 1])
        if j % 2:
            codes[a:b] = int(torch.randint(0, K, (1,), generator=g))  # one code
        else:
            words = torch.arange(j % 32, (K + 31) // 32, 32)  # every word of one bank
            codes[a:b] = (words[torch.randint(0, len(words), (b - a,), generator=g)] * 32 +
                          torch.randint(0, 32, (b - a,), generator=g)).clamp_max(K - 1).int()
    centroids = torch.nn.functional.normalize(torch.randn(K, DIM, generator=g), dim=-1)
    weights = torch.linspace(-0.1, 0.1, 16)
    residuals = torch.randint(0, 256, (max(int(lens.sum()), 1), DIM // 2), generator=g, dtype=torch.uint8)
    ivf, ivf_lengths = build_ivf(codes, lens, K)
    data = IndexTensors(nbits=4, centroids=centroids, bucket_weights=weights, doc_lengths=lens, doc_codes=codes,
                        doc_residuals=residuals[: int(lens.sum())], ivf=ivf.to(torch.int32), ivf_lengths=ivf_lengths)
    didx = DeviceIndex(data, device)
    _cache[K] = (didx, codes, offs)
    return _cache[K]


@pytest.mark.parametrize("K", [1100, 2048])  # bitmap words: 36 (not a multiple of 32 banks) and 64
def test_walk_layout_deals_every_document_over_its_own_windows(K, cuda_device):
    from fast_plaid_b200.engine import DeviceIndex

    didx, codes, offs = _index(K, cuda_device)
    hb = didx.layout(1, 32, DeviceIndex.make_params(10, 256, 8)).hb_words
    assert hb == ((K + 31) // 32 + 3) // 4 * 4
    wc, win = (t.cpu() for t in didx.walk_layout())
    N = offs.shape[0] - 1
    assert int(win[0]) == 0 and int(win[N]) == wc.shape[0]
    pad_codes = {(hb + l) * 32 for l in range(32)}
    assert {((c // 32) % 32) for c in pad_codes} == set(range(32))  # one zero word per bank
    for d in range(N):
        doc = codes[int(offs[d]) : int(offs[d + 1])].long()
        n = doc.numel()
        nw = int(win[d + 1] - win[d])
        assert nw == math.ceil(n / 32), (d, n, nw)
        slots = wc[int(win[d]) : int(win[d + 1])].long()
        real = slots[slots < K]
        assert torch.equal(real.sort().values, doc.sort().values), f"doc {d}: the windows do not hold its codes"
        pads = slots[slots >= K]
        assert pads.numel() == 32 * nw - n
        assert set(pads.tolist()) <= pad_codes, f"doc {d}: a padding code outside the zero words"
        if n == 0:
            continue
        per_bank = torch.bincount((doc // 32) % 32, minlength=32)
        cap = (per_bank + nw - 1) // nw
        for w in range(nw):
            row = slots[w]
            is_real = row < K
            banks_real = torch.bincount((row[is_real] // 32) % 32, minlength=32)
            assert bool((banks_real <= cap).all()), f"doc {d} window {w}: {banks_real.tolist()} > {cap.tolist()}"
            banks_pad = ((row[~is_real] // 32) % 32).tolist()
            assert len(set(banks_pad)) == len(banks_pad), f"doc {d} window {w}: two padding codes share a bank"
            assert not any(banks_real[b] for b in banks_pad), f"doc {d} window {w}: padding shares a real code's bank"


@pytest.mark.parametrize("group", ["4", "5", "6"])  # windows per group of the bound pass (FPB_K3_GROUP)
@pytest.mark.parametrize("Q", [32, 64])  # shuffle-free (Qp <= 32) and shuffle one-pass kernels
@pytest.mark.parametrize("K", [1100, 2048])
def test_approx_scores_do_not_depend_on_the_walk_order(K, Q, group, cuda_device, monkeypatch):
    """One-pass (DIRECT) scores and the two-pass stage's resolved / refined scores equal scoring every candidate
    exactly (EXACT_ALL) bit for bit, and those equal the max-then-sum over each document's codes in their original
    order (fp32 sums of the same fp16 maxima, up to the summation order), whatever the bound pass's group width."""
    monkeypatch.setenv("FPB_K3_GROUP", group)
    from fast_plaid_b200.engine import (FPB_FLAG_APPROX_DIRECT, FPB_FLAG_APPROX_EXACT_ALL, FPB_FLAG_APPROX_TWO_PASS,
                                        DeviceIndex)

    didx, codes, offs = _index(K, cuda_device)
    B = 4
    g = torch.Generator().manual_seed(100 * K + Q)
    q16 = torch.nn.functional.normalize(torch.randn(B, Q, DIM, generator=g), dim=-1).half().to(cuda_device)
    params = DeviceIndex.make_params(10, 64, 8)

    def run(flag):
        st = didx.run_stages(q16, DeviceIndex.with_flags(params, flag), upto="select")
        torch.cuda.synchronize()
        return {k: v.clone().cpu() for k, v in st.items() if isinstance(v, torch.Tensor) and k != "workspace"}

    every, direct, pruned = (run(f) for f in (FPB_FLAG_APPROX_EXACT_ALL, FPB_FLAG_APPROX_DIRECT,
                                              FPB_FLAG_APPROX_TWO_PASS))
    checked = 0
    for b in range(B):
        n = int(every["n_cand"][b])
        cand = every["cand"][b, :n].long()
        exact_all = every["approx"][b, :n]
        assert torch.equal(direct["approx"][b, :n], exact_all), f"query {b}: one-pass scores differ"
        ub, lb = pruned["approx"][b, :n], pruned["approx_lb"][b, :n]
        refined = torch.zeros(n, dtype=torch.bool)
        refined[pruned["refine"][b, : int(pruned["n_refine"][b])].long()] = True
        known = refined | (lb == ub)
        assert torch.equal(ub[known], exact_all[known]), f"query {b}: a two-pass score differs"
        assert bool((ub >= exact_all).all())
        for other in (direct, pruned):
            r = int(every["n_rerank"][b])
            assert torch.equal(other["rerank"][b, :r], every["rerank"][b, :r])
            assert torch.equal(other["rerank_approx"][b, :r], every["rerank_approx"][b, :r])
        S = every["S"][b, :, :Q].float()
        for i in range(n):
            d = int(cand[i])
            doc = codes[int(offs[d]) : int(offs[d + 1])].long()
            ref = S[doc].max(0).values.double().sum()
            assert abs(float(exact_all[i]) - float(ref)) <= 1e-6 * max(1.0, abs(float(ref))), (b, d)
            checked += 1
    assert checked > 0
