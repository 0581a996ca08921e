"""The index-build kernels (csrc/encode.cu) against a float64 reference, bit for bit on inputs whose arithmetic is exact.

What each kernel computes, and where the reference rounds:

  encode assign   code  = smallest k with fp16(<x, c_k>) == max_k fp16(<x, c_k>)     dot in float64, one rounding to
                                                                                     fp16 (overflow -> +-inf)
  k-means assign  code  = smallest k with the largest <x, c_k> - |c_k|^2 / 2         float64, no rounding
  pack            r     = fp16(x - c[code])                                          one fp16 subtraction (numpy's
                                                                                     float64 -> float16 cast is
                                                                                     correctly rounded)
                  bucket = #{cutoffs < r}; bits of each bucket LSB-first, the bit stream packed big-endian per byte
  k-means update  new   = fp16(mean64), count exact, shift = sqrt(sum (new - old)^2) in float64 of the fp16 values

The assign cells use two families of inputs built from small multiples of powers of two, so that every dot product,
every partial sum and every bias is exact in fp32 whatever the accumulation order (tensor core, cuBLAS or numpy):

  ternary  tokens in {0, +-1/4}, centroids in {0, +-1/4, +-1/2}, sparse: every score is a multiple of 1/16 below 16,
           exact even in fp16, and ties between centroids are everywhere;
  dense    entries m / 256 with |m| <= 16: scores are multiples of 2^-16 below 1/2, exact in fp32 but not in fp16,
           so fp16 rounding merges maxima.

The fixture builder asserts the exactness (the float32 product equals the float64 one, score by score, bias by bias);
without it a failure would say nothing.  Into both families it plants, on dimensions the random part leaves at zero:
a pair of centroids whose scores differ by 2^-16 (below one fp16 ulp; the larger score at the larger id), ties in
columns owned by different lanes of one quad, by one thread, in several centroid tiles, and in the first and the last
centroid, centroids whose scores overflow fp16 to +inf (encode only), and tokens whose every score is negative.
The k-means cells use the same inputs: there the sub-ulp pair must go to the larger id, the truly nearer centroid.

Shapes: the centroid count K covers a partial last tile and 1, 2 and 0 centroid tiles modulo the 3-stage ring; every
K meets a token count past 128 x (SM count), where a CTA of the persistent loop runs a second token tile and carries
its pipeline phase over.
"""

from __future__ import annotations

import filecmp
import itertools
import os

import numpy as np
import pytest
import torch

import util  # noqa: F401  (puts the repository root on sys.path)
from oracle import index_oracle as io

pytestmark = pytest.mark.gpu

D = 128
RANDOM_DIMS = 112  # the random part of every vector; dimensions 112 .. 127 hold the planted structure
FLOOR_DIM = 125  # every centroid is positive here, so a token -e_125 / 4 scores negative against all of them
# planted centroid groups: (name, dimension(s), ids); a member holds 1 on the group's first dimension (the overflow
# group: OVERFLOW_VALUE).  A pair is (smaller id, larger id); the larger id
# adds 2^-8 on the second dimension, which the pair's token also carries: its score is 2^-16 higher.
GROUPS = (
    ("pair_lanes", (112, 113), (9, 10)),  # columns 9 and 10: quads 0 and 1 of one tile
    ("pair_tiles", (114, 115), (20, 149)),  # column 20 of tile 0, column 21 of tile 1
    ("first_last", (116,), (0, -1)),  # -1: the last centroid
    ("quad", (117,), (33, 35, 36, 38)),  # one column per lane of a quad
    ("thread", (118,), (40, 41, 48)),  # three columns of one thread
    ("tiles", (119,), (50, 178, 306, 562)),  # the same column in four centroid tiles
    ("overflow", (120,), (60, 61, 200)),  # scores 65 536, 131 072, 65 536: all +inf in fp16 (encode only)
)
OVERFLOW_VALUE = {60: 256.0, 61: 512.0, 200: 256.0}
TOKEN_KINDS = tuple(g[0] for g in GROUPS) + ("negative", "zero")

KS = (1, 37, 127, 128, 129, 384, 512, 640, 1000, 65_536)
# (K, n): n symbolic in the SM count ("sm" = 128 x SM count tokens, one token tile per CTA); every K meets an n that
# makes some CTA run two or more token tiles
CELLS = (
    (1, "1"), (1, "sm+1"),
    (37, "127"), (37, "2sm+129"),
    (127, "128"), (127, "25300"),
    (128, "129"), (128, "sm+1"),
    (129, "sm"), (129, "2sm+129"),
    (384, "1"), (384, "25300"),
    (512, "127"), (512, "sm+1"),
    (640, "128"), (640, "2sm+129"),
    (1000, "129"), (1000, "25300"),
    (65_536, "sm"), (65_536, "sm+1"),
)
assert {k for k, _ in CELLS} == set(KS)


@pytest.fixture(scope="module")
def sm_count(cuda_device):
    return torch.cuda.get_device_properties(cuda_device).multi_processor_count


def _n(spec: str, sm: int) -> int:
    return {"sm": sm * 128, "sm+1": sm * 128 + 1, "2sm+129": 2 * sm * 128 + 129}.get(spec) or int(spec)


def _ulp16(x: torch.Tensor) -> torch.Tensor:
    """Spacing of fp16 at |x|: 2^(e-10) in the binade [2^e, 2^(e+1)), 2^-24 below the normal range."""
    _, e = torch.frexp(x.abs().clamp_min(2.0 ** -14))
    return torch.ldexp(torch.ones_like(x), e - 11)


# ---- exact-arithmetic fixtures --------------------------------------------------------------------------------------
def _random_part(g: torch.Generator, rows: int, family: str, centroids: bool) -> torch.Tensor:
    if family == "ternary":
        density = 0.25 if centroids else 0.125
        mag = torch.where(torch.rand(rows, RANDOM_DIMS, generator=g) < 0.5, 0.25, 0.5) if centroids else 0.25
        sign = torch.where(torch.rand(rows, RANDOM_DIMS, generator=g) < 0.5, -1.0, 1.0)
        keep = torch.rand(rows, RANDOM_DIMS, generator=g) < density
        return torch.where(keep, sign * mag, 0.0).double()
    return torch.randint(-16, 17, (rows, RANDOM_DIMS), generator=g).double() / 256


def _planted_groups(K: int, kmeans: bool) -> dict[str, tuple[int, ...]]:
    """The groups whose ids fit in K (ids are never shared between groups; a group needs two members)."""
    used: set[int] = set()
    out = {}
    for name, _, ids in GROUPS:
        if kmeans and name == "overflow":
            continue
        keep = []
        for i in ids:
            i = K - 1 if i < 0 else i
            if i < K and i not in used and i not in keep:
                keep.append(i)
        if len(keep) == len(ids) or (not name.startswith("pair") and len(keep) >= 2):
            out[name] = tuple(keep)
            used.update(keep)
    return out


def _exact_inputs(K: int, n: int, family: str, kmeans: bool, seed: int):
    """fp16 tokens [n, 128] and centroids [K, 128] (host) with the planted structure; the planted token rows
    {row: kind}; the planted groups {name: ids}."""
    g = torch.Generator().manual_seed(seed)
    C = torch.zeros(K, D, dtype=torch.float64)
    C[:, :RANDOM_DIMS] = _random_part(g, K, family, True)
    if family == "ternary":
        C[:, FLOOR_DIM] = torch.where(torch.rand(K, generator=g) < 0.5, 0.25, 0.5)
    else:
        C[:, FLOOR_DIM] = torch.randint(1, 17, (K,), generator=g).double() / 256
    groups = _planted_groups(K, kmeans)
    dims = {name: d for name, d, _ in GROUPS}
    for name, ids in groups.items():
        for i in ids:
            C[i] = 0.0
            C[i, FLOOR_DIM] = 0.25  # equal norms inside a group: its members are equidistant from its token
            C[i, dims[name][0]] = OVERFLOW_VALUE[i] if name == "overflow" else 1.0
        if name.startswith("pair"):
            C[ids[1], dims[name][1]] = 2.0 ** -8
    X = torch.zeros(n, D, dtype=torch.float64)
    X[:, :RANDOM_DIMS] = _random_part(g, n, family, False)
    kinds = [k for k in TOKEN_KINDS if not (kmeans and k == "overflow")]
    T = len(kinds)
    pos = torch.unique(torch.cat([torch.arange(min(n, T)), torch.arange(max(0, n - T), n),
                                  torch.linspace(0, n - 1, 4 * T).round().long()])).tolist()
    planted = {}
    for j, r in enumerate(pos):
        kind = kinds[j % T]
        planted[r] = kind
        X[r] = 0.0
        if kind == "negative":
            X[r, FLOOR_DIM] = -0.25
        elif kind == "overflow":
            X[r, dims[kind][0]] = 256.0
        elif kind != "zero":
            X[r, dims[kind][0]] = 1.0
            if kind.startswith("pair"):
                X[r, dims[kind][1]] = 2.0 ** -8
    X16, C16 = X.half(), C.half()
    assert torch.equal(X16.double(), X) and torch.equal(C16.double(), C)
    return X16, C16, planted, groups


def _first_argmax(s: torch.Tensor) -> torch.Tensor:
    """Smallest column holding the row maximum (a row of -inf gives 0, like ATen's argmax)."""
    m = s.max(1, keepdim=True).values
    ids = torch.arange(s.shape[1], device=s.device)
    return torch.where(s == m, ids, s.shape[1]).min(1).values


def _exact_reference(X16: torch.Tensor, C16: torch.Tensor, kmeans: bool, dev: str, chunk: int = 2048) -> torch.Tensor:
    """Expected codes, computed in float64 on the GPU, after checking that fp32 arithmetic is exact on these inputs."""
    C64, C32 = C16.to(dev).double(), C16.to(dev).float()
    bias64 = -0.5 * (C64 * C64).sum(1)
    bias32 = -0.5 * (C32 ** 2).sum(1)  # the bias the engine hands the kernel
    if kmeans:
        assert torch.equal(bias32.double(), bias64), "the fixture's biases are not exact in fp32"
    out = []
    for s in range(0, X16.shape[0], chunk):
        X64 = X16[s : s + chunk].to(dev).double()
        d64 = X64 @ C64.t()
        d32 = X64.float() @ C32.t()
        assert torch.equal(d32.double(), d64), "the fixture's scores are not exact in fp32"
        if kmeans:
            sc = d64 + bias64
            assert torch.equal((d32 + bias32).double(), sc), "the fixture's k-means scores are not exact in fp32"
        else:
            sc = d64.float().half()  # d64 is exact in fp32: this is the one rounding fp16(dot)
        out.append(_first_argmax(sc))
        del d64, d32, sc
    return torch.cat(out).cpu()


def _check_planted(ref: torch.Tensor, planted: dict, groups: dict, kmeans: bool) -> None:
    """The reference itself resolves every planted row as the fixture intends (so a kernel agreeing with it does too)."""
    for r, kind in planted.items():
        code = int(ref[r])
        if kind in groups:
            ids = groups[kind]
            if kind.startswith("pair"):
                assert code == (ids[1] if kmeans else ids[0]), (kind, code)
            else:
                assert code == min(ids), (kind, code)
        elif kind == "zero" and not kmeans:
            assert code == 0


# ---- pack reference (create.rs:413-427, written from the spec) --------------------------------------------------------
def _pack_ref(X16: np.ndarray, C16: np.ndarray, codes: np.ndarray, cutoffs: np.ndarray, nbits: int) -> np.ndarray:
    r = (X16.astype(np.float64) - C16[codes].astype(np.float64)).astype(np.float16).astype(np.float64)
    bucket = (cutoffs.astype(np.float64)[None, None, :] < r[:, :, None]).sum(-1)
    return _pack_buckets(bucket, nbits)


def _pack_buckets(bucket: np.ndarray, nbits: int) -> np.ndarray:
    n = bucket.shape[0]
    bits = (bucket[..., None] >> np.arange(nbits)) & 1  # LSB-first inside the element's field
    return np.packbits(bits.reshape(n, -1).astype(np.uint8), axis=1, bitorder="big")


def _encode(X16, C16, dev, nbits=4, cutoffs=None):
    from fast_plaid_b200.engine import encode_tokens

    if cutoffs is None:
        cutoffs = torch.linspace(-0.3, 0.3, 2 ** nbits - 1)
    codes, packed = encode_tokens(X16.to(dev), C16.to(dev), cutoffs, nbits)
    torch.cuda.synchronize()
    return codes.cpu().long(), packed.cpu(), cutoffs.float()


# ---- encode assign ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", ["ternary", "dense"])
@pytest.mark.parametrize("K,nspec", CELLS)
def test_encode_assign_is_bit_exact(K, nspec, family, cuda_device, sm_count):
    n = _n(nspec, sm_count)
    X16, C16, planted, groups = _exact_inputs(K, n, family, kmeans=False, seed=K * 7 + n)
    ref = _exact_reference(X16, C16, False, cuda_device)
    _check_planted(ref, planted, groups, kmeans=False)
    codes, packed, cutoffs = _encode(X16, C16, cuda_device)
    bad = (codes != ref).nonzero().flatten()
    assert bad.numel() == 0, (f"{bad.numel()} of {n} codes differ; first rows {bad[:8].tolist()}: "
                              f"kernel {codes[bad[:8]].tolist()} reference {ref[bad[:8]].tolist()}")
    # the residual bytes of the same call (its codes are the reference's)
    want = _pack_ref(X16.numpy(), C16.numpy(), ref.numpy(), cutoffs.numpy(), 4)
    assert np.array_equal(packed.numpy(), want)


@pytest.mark.parametrize("K", [129, 1000])
def test_encode_all_scores_negative_infinity_gives_code_zero(K, cuda_device, sm_count):
    """Every score overflows to -inf in fp16: ATen's argmax returns 0; +inf rows go to the smallest overflowing id."""
    n = sm_count * 128 + 1
    g = torch.Generator().manual_seed(K)
    C = torch.zeros(K, D, dtype=torch.float64)
    C[:, 0] = torch.where(torch.rand(K, generator=g) < 0.5, 256.0, 512.0)
    C[:, 1:RANDOM_DIMS] = _random_part(g, K, "dense", True)[:, 1:]
    X = torch.zeros(n, D, dtype=torch.float64)
    X[:, 0] = -256.0
    X[1::3, 0] = 256.0  # every third row: all +inf
    X16, C16 = X.half(), C.half()
    ref = _exact_reference(X16, C16, False, cuda_device)
    assert (ref[0::3] == 0).all() and (ref[1::3] == 0).all()
    codes, _, _ = _encode(X16, C16, cuda_device)
    assert torch.equal(codes, ref)


@pytest.mark.parametrize("K,nspec", [(1000, "sm+1"), (65_536, "2048")])
def test_encode_natural_data_within_the_float64_bound(K, nspec, cuda_device, sm_count):
    """Normalised random data: the pick scores within ulp16 + D 2^-23 sum|a_k b_k| of the float64 maximum, and agrees
    with ATen's fp16 matmul + argmax except between centroids whose fp16 scores are one step apart."""
    n = _n(nspec, sm_count)
    g = torch.Generator().manual_seed(K + n)
    C16 = torch.nn.functional.normalize(torch.randn(K, D, generator=g), dim=-1).half()
    X16 = torch.nn.functional.normalize(torch.randn(n, D, generator=g), dim=-1).half()
    codes, packed, cutoffs = _encode(X16, C16, cuda_device)
    Xd, Cd = X16.to(cuda_device), C16.to(cuda_device)
    d64 = Xd.double() @ Cd.double().t()
    a64 = Xd.double().abs() @ Cd.double().abs().t()
    cd = codes.to(cuda_device)
    best = d64.max(1)
    pick = d64.gather(1, cd[:, None]).squeeze(1)
    absdot = torch.maximum(a64.gather(1, cd[:, None]).squeeze(1), a64.gather(1, best.indices[:, None]).squeeze(1))
    tol = _ulp16(best.values) + D * 2.0 ** -23 * absdot
    assert bool((best.values - pick <= tol).all()), float((best.values - pick - tol).max())
    aten = (Xd @ Cd.t()).argmax(1)
    same = aten == cd
    assert float(same.float().mean()) > 0.999
    s16 = d64.float().half().float()
    if bool((~same).any()):
        gap = (s16.gather(1, aten[:, None]) - s16.gather(1, cd[:, None])).abs().squeeze(1)
        assert float(gap[~same].max()) <= 2.0 ** -10
    want = _pack_ref(X16.numpy(), C16.numpy(), codes.numpy(), cutoffs.numpy(), 4)
    assert np.array_equal(packed.numpy(), want)


# ---- k-means assign ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", ["ternary", "dense"])
@pytest.mark.parametrize("K,nspec", CELLS)
def test_kmeans_assign_is_bit_exact(K, nspec, family, cuda_device, sm_count):
    from fast_plaid_b200.engine import kmeans_assign

    n = _n(nspec, sm_count)
    X16, C16, planted, groups = _exact_inputs(K, n, family, kmeans=True, seed=K * 11 + n)
    ref = _exact_reference(X16, C16, True, cuda_device)
    _check_planted(ref, planted, groups, kmeans=True)
    got = kmeans_assign(X16.to(cuda_device), C16.to(cuda_device))
    torch.cuda.synchronize()
    got = got.cpu().long()
    bad = (got != ref).nonzero().flatten()
    assert bad.numel() == 0, (f"{bad.numel()} of {n} assignments differ; first rows {bad[:8].tolist()}: "
                              f"kernel {got[bad[:8]].tolist()} reference {ref[bad[:8]].tolist()}")
    if K > 1:  # the planted centroids are nobody's nearest but their own tokens': some cluster stays empty
        assert int(torch.bincount(ref, minlength=K).eq(0).sum()) > 0


def test_encode_and_kmeans_compare_differently_on_a_sub_ulp_pair(cuda_device):
    """Two centroids 2^-16 apart in score: encode compares fp16 scores and keeps the smaller id, k-means compares fp32
    distances and takes the truly nearer (larger) id."""
    from fast_plaid_b200.engine import kmeans_assign

    X16, C16, planted, groups = _exact_inputs(640, 300, "dense", kmeans=True, seed=5)
    rows = [r for r, k in planted.items() if k.startswith("pair")]
    assert rows and {"pair_lanes", "pair_tiles"} <= set(groups)
    codes, _, _ = _encode(X16, C16, cuda_device)
    km = kmeans_assign(X16.to(cuda_device), C16.to(cuda_device)).cpu().long()
    for r in rows:
        small, large = groups[planted[r]]
        assert int(codes[r]) == small and int(km[r]) == large, (r, int(codes[r]), int(km[r]))


# ---- pack -------------------------------------------------------------------------------------------------------------
def _f16_step(v: np.float16, direction: float) -> np.float16:
    return np.nextafter(np.float16(v), np.float16(direction))


def _edge_cutoffs(nbits: int) -> np.ndarray:
    """Sorted fp32 cutoffs: even ones are fp16 values (a residual can equal them), odd ones lie strictly between two
    neighbouring fp16 values, and 0.0 is one of them (for nbits 2, the middle one)."""
    m = 2 ** nbits - 1
    base = np.linspace(-0.07, 0.07, m) if nbits == 4 else np.array([-0.0312, 0.0, 0.0217])
    out = []
    for i, v in enumerate(base):
        h = np.float16(0.0 if abs(v) < 1e-12 else v)
        if (i % 2 == 0 and nbits == 4) or h == 0 or (nbits == 2 and i == 0):
            out.append(np.float32(h))
            continue
        nxt = _f16_step(h, np.inf)
        t = np.float32(np.float32(h) + (np.float32(nxt) - np.float32(h)) * np.float32(0.375))
        assert np.float32(h) < t < np.float32(nxt)
        out.append(t)
    cut = np.array(out, dtype=np.float32)
    assert (np.diff(cut) > 0).all()
    return cut


def _edge_residuals(cut: np.ndarray, nbits: int) -> np.ndarray:
    """fp16 residual values on, one step around, and on either side of every cutoff; one value inside each bucket
    in every element position of a byte, together with every other bucket in the other positions; +-0."""
    per = 8 // nbits
    vals = [np.float16(0.0), np.float16(-0.0)]
    for t in cut:
        h = np.float16(t)
        if np.float32(h) == t:
            vals += [h, _f16_step(h, -np.inf), _f16_step(h, np.inf)]
        else:
            lo = h if np.float32(h) < t else _f16_step(h, -np.inf)
            hi = _f16_step(lo, np.inf)
            vals += [lo, hi, _f16_step(lo, -np.inf), _f16_step(hi, np.inf)]
    edges = np.array(vals, dtype=np.float16)
    mid = np.concatenate([[cut[0] - 0.5], (cut[:-1] + cut[1:]) / 2, [cut[-1] + 0.5]]).astype(np.float16)
    combos = np.array(list(itertools.product(range(2 ** nbits), repeat=per))).reshape(-1)
    rng = np.random.default_rng(nbits)
    stream = np.concatenate([np.repeat(edges, per), mid[combos], rng.permutation(np.tile(edges, per))])
    pad = (-len(stream)) % D
    return np.concatenate([stream, np.zeros(pad, dtype=np.float16)]).reshape(-1, D)


@pytest.mark.parametrize("nbits", [2, 4])
def test_pack_on_cutoff_edges_is_byte_exact(nbits, cuda_device):
    cut = _edge_cutoffs(nbits)
    X = _edge_residuals(cut, nbits)
    C = np.zeros((1, D), dtype=np.float16)  # one centroid at 0: the residual is the token itself
    X16, C16 = torch.from_numpy(X), torch.from_numpy(C)
    codes, packed, _ = _encode(X16, C16, cuda_device, nbits, torch.from_numpy(cut))
    assert int(codes.abs().sum()) == 0
    want = _pack_ref(X, C, codes.numpy(), cut, nbits)
    bucket = (cut[None, None, :] < X.astype(np.float32)[:, :, None]).sum(-1)
    assert set(np.unique(bucket)) == set(range(2 ** nbits))
    assert (X[bucket == 0] <= cut[0]).any() and (X == np.float16(cut[0])).any()  # a residual on a cutoff
    bad = np.argwhere(packed.numpy() != want)
    assert bad.shape[0] == 0, f"{bad.shape[0]} bytes differ; first (row, byte): {bad[:8].tolist()}"


@pytest.mark.parametrize("nbits", [2, 4])
def test_pack_reference_agrees_with_the_oracle_packbits(nbits):
    """The spec-written packer above and the oracle's restatement of create.rs:176-184 cannot drift apart."""
    rng = np.random.default_rng(3)
    bucket = rng.integers(0, 2 ** nbits, (64, D))
    bits = torch.from_numpy(((bucket[..., None] >> np.arange(nbits)) & 1).astype(np.int64))
    oracle = io.packbits(bits.flatten()).reshape(64, D * nbits // 8)
    assert np.array_equal(_pack_buckets(bucket, nbits), oracle.numpy())


# ---- k-means update ---------------------------------------------------------------------------------------------------
POW2_SIZES = (1, 2, 64, 4096)
OTHER_SIZES = (3, 7, 1000)


def _update_inputs(seed: int):
    """Cluster sizes {1, 2, 64, 4096} (exact means), {3, 7, 1000} and 0 (empty), in shuffled cluster order, with the
    points of all clusters interleaved; entries m / 256 with |m| <= 128, so every cluster sum is exact in fp32."""
    rng = np.random.default_rng(seed)
    sizes = np.array([1] * 8 + [2] * 8 + [64] * 4 + [4096] * 2 + [3] * 60 + [7] * 40 + [1000] * 6 + [0] * 4)
    rng.shuffle(sizes)
    K = len(sizes)
    assign = np.repeat(np.arange(K), sizes)
    rng.shuffle(assign)
    X = (rng.integers(-128, 129, (len(assign), D)) / 256).astype(np.float16)
    old = (rng.standard_normal((K, D)) * 0.2).astype(np.float16)
    sums64 = np.zeros((K, D))
    np.add.at(sums64, assign, X.astype(np.float64))
    sums32 = torch.zeros(K, D).index_add_(0, torch.from_numpy(assign), torch.from_numpy(X).float())
    assert np.array_equal(sums32.double().numpy(), sums64), "the fixture's cluster sums are not exact in fp32"
    return X, assign, old, sizes, sums64


def _run_update(X, assign, old, dev):
    from fast_plaid_b200.engine import kmeans_update

    cent = torch.from_numpy(old).to(dev)
    counts, shift = kmeans_update(torch.from_numpy(X).to(dev), torch.from_numpy(assign).to(dev, torch.int32), cent)
    torch.cuda.synchronize()
    return cent.cpu().numpy(), counts.cpu().numpy(), shift.cpu().numpy()


def test_kmeans_update_is_the_rounded_float64_mean(cuda_device):
    X, assign, old, sizes, sums64 = _update_inputs(1)
    new, counts, shift = _run_update(X, assign, old, cuda_device)
    assert np.array_equal(counts, sizes)
    ne = sizes > 0
    want = np.zeros_like(old)
    want[ne] = (sums64[ne] / sizes[ne, None]).astype(np.float16)
    pow2 = np.isin(sizes, POW2_SIZES)
    other = np.isin(sizes, OTHER_SIZES)
    assert np.array_equal(new[pow2].view(np.uint16), want[pow2].view(np.uint16))
    w, g = want[other].astype(np.float64), new[other].astype(np.float64)
    ulp = _ulp16(torch.from_numpy(w)).numpy()
    assert (np.abs(g - w) <= ulp).all(), float((np.abs(g - w) / ulp).max())
    assert (new[other].view(np.uint16) == want[other].view(np.uint16)).mean() >= 0.99
    # empty clusters: row untouched, shift 0
    assert np.array_equal(new[~ne].view(np.uint16), old[~ne].view(np.uint16)) and (shift[~ne] == 0).all()
    ref_shift = np.sqrt(((new.astype(np.float64) - old.astype(np.float64)) ** 2).sum(1))
    assert np.allclose(shift[ne], ref_shift[ne], rtol=1e-6, atol=0), float(np.abs(shift[ne] / ref_shift[ne] - 1).max())


def test_kmeans_update_does_not_depend_on_the_point_order(cuda_device):
    """Exact sums: the same result for any numbering of the points; natural data: byte-identical run to run."""
    X, assign, old, _, _ = _update_inputs(2)
    a = _run_update(X, assign, old, cuda_device)
    perm = np.random.default_rng(0).permutation(len(assign))
    b = _run_update(X[perm], assign[perm], old, cuda_device)
    for u, v in zip(a, b):
        assert np.array_equal(np.ascontiguousarray(u).view(np.uint8), np.ascontiguousarray(v).view(np.uint8))
    rng = np.random.default_rng(4)
    Xn = rng.standard_normal((50_000, D)).astype(np.float16)
    an = rng.integers(0, 300, 50_000)
    oldn = rng.standard_normal((300, D)).astype(np.float16)
    c = _run_update(Xn, an, oldn, cuda_device)
    d = _run_update(Xn, an, oldn, cuda_device)
    for u, v in zip(c, d):
        assert np.array_equal(np.ascontiguousarray(u).view(np.uint8), np.ascontiguousarray(v).view(np.uint8))


# ---- end to end: a GPU build equals a CPU build -----------------------------------------------------------------------
@pytest.mark.parametrize("nbits", [2, 4])
def test_gpu_build_is_byte_identical_to_the_cpu_build(nbits, tmp_path, cuda_device):
    """Ternary corpus and centroids (every score exact): `create_index` on the GPU (several fpb_encode calls per
    chunk, three chunks) writes the same codes, residuals, IVF, document lengths and codec as on the CPU."""
    from fast_plaid_b200.index import build

    g = torch.Generator().manual_seed(nbits)
    n_docs = 300
    lens = torch.randint(1, 120, (n_docs,), generator=g)
    lens[[0, 17, 299]] = 1
    lens[[5, 150, 298]] = torch.tensor([129, 200, 300])
    docs = [torch.cat([_random_part(g, int(L), "ternary", False), torch.zeros(int(L), D - RANDOM_DIMS, dtype=torch.float64)],
                      1).half() for L in lens]
    cent = torch.cat([_random_part(g, 256, "ternary", True), torch.zeros(256, D - RANDOM_DIMS, dtype=torch.float64)],
                     1).half()
    kw = dict(nbits=nbits, batch_size=128, seed=7)  # 128 documents per chunk, an encode call per >= 128 tokens
    build.create_index(docs, str(tmp_path / "gpu"), cent, device=cuda_device, **kw)
    build.create_index(docs, str(tmp_path / "cpu"), cent, device="cpu", **kw)
    names = sorted(os.listdir(tmp_path / "cpu"))
    assert names == sorted(os.listdir(tmp_path / "gpu"))
    exact = [f for f in names if f.endswith((".codes.npy", ".residuals.npy")) or f.startswith("doclens.")]
    exact += ["ivf.npy", "ivf_lengths.npy", "bucket_cutoffs.npy", "bucket_weights.npy", "centroids.npy"]
    assert len([f for f in exact if f.endswith(".codes.npy")]) == 3
    for f in exact:
        assert filecmp.cmp(tmp_path / "cpu" / f, tmp_path / "gpu" / f, shallow=False), f
    # fp32 reductions (a mean over the held-out residuals, a norm under a quantile): ATen's CPU and CUDA reductions
    # may order or scale the sum differently, so these are held to one fp32 ulp
    for f in ("avg_residual.npy", "cluster_threshold.npy"):
        a, b = np.load(tmp_path / "cpu" / f), np.load(tmp_path / "gpu" / f)
        assert a.shape == b.shape
        assert (np.abs(a - b) <= np.spacing(np.maximum(np.abs(a), np.abs(b)))).all(), f
