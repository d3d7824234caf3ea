"""The projection GEMMs (gemm_sm90.cuh and its epilogues) against float64 references, per element.  Needs an H100.

- `vtm_linear_f16` and `vtm_linear_residual_f16` (StoreEpi), `vtm_linear_geglu_f16` (GegluEpi), and the q/k/v and
  cross-attention kv projections inside `vtm_attention_ex` / `vtm_cross_attention` (HeadSplitEpi).
- Exact inputs: A on a 1/8 grid with |a| <= 4, W on a 1/16 grid with |w| <= 2, the bias on the 2^-7 grid, and
  sum_k |a_k w_k| + |b| < 2^16.  Every product is then a multiple of 2^-7 and every partial sum, in whatever order the
  MMA adds them, has at most 23 significant bits: exact in fp32.  The kernel's only approximations left are its fp16
  roundings, so the outputs are checked bit for bit against float64 results rounded once to fp16 (`_round16`).
- Real-valued inputs: a per-element bound derived for wgmma's fp32 accumulation (`_linear_bound`).
- Every call goes through the C-ABI.  The output has guard rows after row M and guard columns in [N, ldd) filled with a
  sentinel, and its [M, N] block is filled with NaN: an element left unwritten shows as NaN, a store past an edge
  changes the sentinel.  The attention workspace is filled with 0xFF bytes (fp16 NaN)."""
import pytest
import torch

from vidtome_b200 import _lib, ops

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A5A          # fp16 203.25: the guard value around every output
GUARD_ROWS = 40


# ---------------------------------------------------------------------------------------------------------------------
# fp16 rounding and spacing in float64

def _ulp16(x):
    """Spacing of fp16 numbers in the binade of |x| (2^-24 in the subnormal range)."""
    _, e = torch.frexp(x.abs().clamp(min=2.0 ** -14))
    return torch.ldexp(torch.ones_like(x), e - 11)


def _round16(x):
    """float64 -> the nearest fp16 value (ties to even), rounded once; still float64.  torch's own double -> half
    conversion goes through float and can round twice."""
    assert x.abs().max().item() < 65520, "rounds beyond the fp16 range"
    u = _ulp16(x)
    return torch.round(x / u) * u


def _gelu64(g):
    return g * torch.special.ndtr(g)


def _ordered(h):
    """fp16 tensor -> int32 that is monotonic in the value, one step per fp16 number (+0 and -0 both 0)."""
    b = h.view(torch.int16).int()
    return torch.where(b < 0, -(b & 0x7FFF), b)


# ---------------------------------------------------------------------------------------------------------------------
# inputs

def _grid(shape, step, lim, g):
    n = int(round(lim / step))
    return (torch.randint(-n, n + 1, shape, generator=g, device="cuda").double() * step).half()


def _exact_inputs(M, N, K, g, bias=True):
    a = _grid((M, K), 1 / 8, 4, g)
    w = _grid((N, K), 1 / 16, 2, g)
    b = _grid((N,), 2.0 ** -7, 8, g) if bias else None
    return a, w, b


def _check_exact(a, w, b):
    """Asserts the limits under which A W^T + b is exact in fp32 whatever the summation order."""
    a64, w64 = a.double(), w.double()
    assert torch.equal(a64 * 8, torch.round(a64 * 8)) and a64.abs().max().item() <= 4, "A off its 1/8 grid"
    assert torch.equal(w64 * 16, torch.round(w64 * 16)) and w64.abs().max().item() <= 2, "W off its 1/16 grid"
    s = a64.abs() @ w64.abs().t()
    if b is not None:
        b64 = b.double()
        assert torch.equal(b64 * 128, torch.round(b64 * 128)), "bias off the 2^-7 grid"
        s = s + b64.abs()
    assert s.max().item() < 2.0 ** 16, "sum |a w| + |b| >= 2^16: partial sums may round in fp32"


def _exact_product(a, w, b):
    """A W^T + b in float64: exact under _check_exact."""
    _check_exact(a, w, b)
    r = a.double() @ w.double().t()
    return r if b is None else r + b.double()


# ---------------------------------------------------------------------------------------------------------------------
# guarded outputs and C-ABI calls

def _stream():
    return torch.cuda.current_stream().cuda_stream


def _guarded(M, N, ldd):
    """[M + GUARD_ROWS, ldd] fp16: the sentinel everywhere, NaN in the [M, N] block."""
    buf = torch.full((M + GUARD_ROWS, ldd), SENTINEL, dtype=torch.int16, device="cuda").view(torch.float16)
    buf[:M, :N] = float("nan")
    return buf


def _check_guards(buf, M, N, what):
    bits = buf.view(torch.int16)
    for name, region in (("columns [N, ldd)", bits[:M, N:]), ("rows past M", bits[M:])):
        bad = region != SENTINEL
        if bad.any():
            pytest.fail(f"{what}: store into the guard {name} at {torch.nonzero(bad)[:4].tolist()}")


def _ptr(t):
    return None if t is None else t.data_ptr()


def _linear(a, w, b, ldd=None, resid=None, ldr=None):
    """vtm_linear_f16, or vtm_linear_residual_f16 with resid [M, ldr]; returns the [M, N] block of a guarded output."""
    lib = _lib.load()
    M, K = a.shape
    N = w.shape[0]
    ldd = ldd or N
    d = _guarded(M, N, ldd)
    if resid is None:
        rc = lib.vtm_linear_f16(a.data_ptr(), w.data_ptr(), _ptr(b), M, N, K, d.data_ptr(), ldd, _stream())
    else:
        rc = lib.vtm_linear_residual_f16(a.data_ptr(), w.data_ptr(), _ptr(b), resid.data_ptr(), ldr, M, N, K,
                                         d.data_ptr(), ldd, _stream())
    _lib.check(rc, "vtm_linear")
    torch.cuda.synchronize()
    what = f"linear M={M} N={N} K={K} ldd={ldd} bias={b is not None} resid={resid is not None} ldr={ldr}"
    _check_guards(d, M, N, what)
    return d[:M, :N], what


def _geglu(a, w_il, b_il, ldd=None):
    lib = _lib.load()
    M, K = a.shape
    N = w_il.shape[0]
    No = N // 2
    ldd = ldd or No
    d = _guarded(M, No, ldd)
    _lib.check(lib.vtm_linear_geglu_f16(a.data_ptr(), w_il.data_ptr(), _ptr(b_il), M, N, K, d.data_ptr(), ldd,
                                        _stream()), "vtm_linear_geglu_f16")
    torch.cuda.synchronize()
    what = f"geglu M={M} inner={No} K={K} ldd={ldd} bias={b_il is not None}"
    _check_guards(d, M, No, what)
    return d[:M, :No], what


def _assert_equal(y, want, what):
    """y fp16 kernel output, want float64 holding fp16 values: equal element by element (+0 == -0)."""
    yd = y.double()
    bad = ~(yd == want)
    if bad.any():
        i = tuple(torch.nonzero(bad)[0].tolist())
        pytest.fail(f"{what}: {int(bad.sum())} elements differ; first at {i}: y = {yd[i].item()!r}, "
                    f"want {want[i].item()!r}")


# ---------------------------------------------------------------------------------------------------------------------
# StoreEpi with exact inputs, bit for bit

def _run_exact(M, N, K, bias=True, ldd=None, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a, w, b = _exact_inputs(M, N, K, g, bias)
    y, what = _linear(a, w, b, ldd=ldd)
    _assert_equal(y, _round16(_exact_product(a, w, b)), what)


def _run_exact_residual(M, N, K, ldd, ldr, seed=0):
    """D = fp16(fp16(A W^T + b) + resid): the second sum is exact in float64 and rounded once.  The columns [N, ldr)
    of resid hold NaN, so a read at the wrong row stride shows."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    a, w, b = _exact_inputs(M, N, K, g)
    resid = torch.full((M, ldr), float("nan"), dtype=torch.float16, device="cuda")
    resid[:, :N] = (torch.randn((M, N), generator=g, device="cuda") * 64).half()
    y, what = _linear(a, w, b, ldd=ldd, resid=resid, ldr=ldr)
    want = _round16(_round16(_exact_product(a, w, b)) + resid[:, :N].double())
    _assert_equal(y, want, what)


RAGGED_M, RAGGED_K = 161, 200      # two m tiles, the second 33 rows; three K chunks and an 8-column tail


@pytest.mark.parametrize("N", range(8, 265, 8))
def test_linear_exact_n(N):
    """Partial 64-column chunks, the `full` and per-store paths, the bias guard; with and without bias."""
    _run_exact(RAGGED_M, N, RAGGED_K, bias=True, ldd=N + 24, seed=N)
    if N % 64 in (0, 8, 56):
        _run_exact(RAGGED_M, N, RAGGED_K, bias=False, seed=N + 1)


@pytest.mark.parametrize("K", list(range(8, 201, 8)) + [768, 1280, 5120])
def test_linear_exact_k(K):
    """The zero-filled K tail of the TMA loads, K below one chunk, and many passes around the stage ring."""
    _run_exact(RAGGED_M, 136, K, bias=K % 16 == 0, ldd=144, seed=K)


@pytest.mark.parametrize("M", (1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 257, 4099))
def test_linear_exact_m(M):
    """Warps whose rows run past M, half-filled m tiles."""
    _run_exact(M, 200, 72, bias=True, ldd=208, seed=M)


@pytest.mark.parametrize("M,N,K", [(1, 5120, 320), (100, 5120, 320), (4099, 1280, 640), (3000, 2048, 128)])
def test_linear_exact_work_split(M, N, K):
    """Small M with the most n-splits, and more work items than SMs (the persistent loop takes several)."""
    _run_exact(M, N, K, ldd=N + 8, seed=M + N)


@pytest.mark.parametrize("M,N,K,ldd,ldr", [(161, 200, 200, 200, 200), (161, 200, 200, 216, 264),
                                           (33, 72, 136, 136, 80), (257, 320, 320, 328, 320),
                                           (4099, 1280, 640, 1280, 1296)])
def test_linear_residual_exact(M, N, K, ldd, ldr):
    _run_exact_residual(M, N, K, ldd, ldr, seed=M + N + K)


# SD1.5 shapes: (C, M) with M = B * L from the merged lengths bench.py runs (B = 2; L = 10241 at C = 320, 2561 at C = 640)
# and the unmerged 16 frames of 16 x 16 tokens at C = 1280
PRODUCTION = ((320, 20482), (640, 5122), (1280, 4096))


@pytest.mark.parametrize("C,M", PRODUCTION)
def test_production_shapes_exact(C, M):
    """Attention output projection (K = N = C), feed-forward output with residual (K = 4C), GEGLU (inner = 4C)."""
    _run_exact(M, C, C, seed=C)
    _run_exact_residual(M, C, 4 * C, C, C, seed=C + 1)
    _run_geglu_exact(M, 4 * C, C, bias=True, seed=C + 2)


# ---------------------------------------------------------------------------------------------------------------------
# GegluEpi with exact inputs

def _geglu_reference(a16, g16):
    """fp16(a16 * fp16(gelu(g16))) in float64, for the fp16 value a16 and gate g16 (float64 tensors).

    gelu is correctly rounded here.  The kernel's gelu has a relative error below 4.5e-6 (the fit's 4e-6, ex2.approx's
    2^-22 and a few fp32 roundings), under 0.01 of an fp16 ulp, so it rounds the same way wherever the float64 gelu lies at least 0.01 ulp from a rounding midpoint.  Returns
    (want, alt, near): alt is the product with the other neighbour of the midpoint, accepted only where `near`."""
    gel = _gelu64(g16)
    q = _round16(gel)
    up = gel > q
    away = (q == 0) | ((q > 0) == up)                   # the neighbour on gel's side is further from zero
    s = torch.where(away, _ulp16(q), _ulp16(q * (1 - 2.0 ** -20)))
    near = ((gel - q).abs() - s / 2).abs() < 0.01 * s
    q_alt = torch.where(up, q + s, q - s)
    return _round16(a16 * q), _round16(a16 * q_alt), near


def _run_geglu_exact(M, inner, K, bias, ldd=None, seed=0):
    """Gate weights on the 1/16 grid scaled so that the gates have a standard deviation near 3 whatever K: most fall
    where gelu is curved, and the product with the value stays inside the fp16 range."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    a, w, b = _exact_inputs(M, 2 * inner, K, g, bias)
    w[inner:] = _grid((inner, K), 1 / 16, max(1, round(48 / (1.78 * K) ** 0.5)) / 16, g)
    wi, bi = ops.interleave_geglu(w, b)
    y, what = _geglu(a, wi, bi, ldd=ldd)
    r = _round16(_exact_product(a, w, b))
    want, alt, near = _geglu_reference(r[:, :inner], r[:, inner:])
    yd = y.double()
    ok = (yd == want) | (near & (yd == alt))
    if not ok.all():
        i = tuple(torch.nonzero(~ok)[0].tolist())
        pytest.fail(f"{what}: {int((~ok).sum())} elements differ; first at {i}: y = {yd[i].item()!r}, "
                    f"want {want[i].item()!r} (value {r[i].item()!r}, gate {r[i[0], inner + i[1]].item()!r})")


@pytest.mark.parametrize("inner", (32, 96, 160, 1280, 1312))
@pytest.mark.parametrize("bias", (True, False))
def test_geglu_exact(inner, bias):
    """inner % 64 in {0, 32}: GEMM width N % 128 in {0, 64}, i.e. a full or half-filled last GEGLU tile."""
    _run_geglu_exact(RAGGED_M, inner, RAGGED_K, bias, seed=inner + bias)
    _run_geglu_exact(33, inner, 24, bias, ldd=inner + 40, seed=inner + 7)


# ---------------------------------------------------------------------------------------------------------------------
# GegluEpi's gelu over every finite fp16 gate

def _all_finite_fp16():
    h = torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).view(torch.float16)
    return h[torch.isfinite(h)]


# One-ulp cases for gates above -3 on an H100 with the degree-7 fit (and 3 at or below -3).  In a CPU emulation with an
# exact ex2 every one-ulp case lies within 0.005 ulp of a rounding midpoint.  A refit must not raise the count.
GELU_ONE_ULP_ABOVE_MINUS_3 = 47


def test_geglu_gelu_exhaustive():
    """Every finite fp16 gate g: row [1, g, 0, ...] of A, value rows picking column 0 and gate rows column 1, so that
    every output is the kernel's fp16(gelu(g)).  Each is within one ulp of the correctly rounded float64 gelu, and is
    zero wherever that is.  At g = -0 the kernel returns +0 (g - g h with g >= 0 true for -0); gelu(-0) is -0."""
    gates = _all_finite_fp16()
    M, K, inner = gates.numel(), 8, 32
    a = torch.zeros((M, K), dtype=torch.float16, device="cuda")
    a[:, 0] = 1
    a[:, 1] = gates
    w = torch.zeros((2 * inner, K), dtype=torch.float16, device="cuda")
    w[:inner, 0] = 1
    w[inner:, 1] = 1
    wi, _ = ops.interleave_geglu(w, None)
    y, what = _geglu(a, wi, None)
    ref = _round16(_gelu64(gates.double())).half()
    assert torch.isfinite(y).all(), what
    dist = (_ordered(y) - _ordered(ref).view(M, 1)).abs().max(1).values
    if dist.max().item() > 1:
        i = int(dist.argmax())
        pytest.fail(f"gelu({gates[i].item()!r}) = {y[i, 0].item()!r}, correctly rounded {ref[i].item()!r}: "
                    f"{int(dist[i])} ulp apart ({int((dist > 1).sum())} gates beyond one ulp)")
    zero = ref == 0
    assert (y[zero] == 0).all(), f"non-zero gelu at g = {gates[zero][(y[zero] != 0).any(1)][:4].tolist()}"
    assert y[gates.view(torch.int16) == -32768].view(torch.int16).eq(0).all(), "gelu(-0) is not +0"
    common = gates.double() > -3
    n_common = int((dist[common] == 1).sum())
    print(f"gelu one-ulp cases: {n_common} for g > -3, {int((dist[~common] == 1).sum())} for g <= -3")
    assert n_common <= GELU_ONE_ULP_ABOVE_MINUS_3 + 3, f"{n_common} one-ulp cases for g > -3"


# ---------------------------------------------------------------------------------------------------------------------
# StoreEpi with real-valued inputs, per-element bound

def _linear_bound(a, w, b, r):
    """Bound on |fp32(acc + b) - r| and the rounded result's spacing, for r = A W^T + b in float64.

    wgmma adds K in k-steps of 16: each step sums 16 exact products (fp16 x fp16 fits in fp32) into the fp32
    accumulator with one rounding, relative error below 2^-23 even if it truncates.  Every partial sum is bounded by
    S = sum_k |a_k w_k|, so after ceil(K / 16) steps |acc - A W^T| <= c(K) S with c(K) = ceil(K / 16) 2^-23.  Adding
    the bias in fp32 rounds once more: 2^-24 (|r| + c(K) S).  Returns that error e; the fp16 rounding of a value within
    e of r then adds at most half an ulp of |r| + e."""
    K = a.shape[1]
    S = a.double().abs() @ w.double().abs().t()
    e = -(-K // 16) * 2.0 ** -23 * S
    if b is not None:
        e = e + 2.0 ** -24 * (r.abs() + e)
    return e


def _assert_bound(y, r, e, what):
    yd = y.double()
    assert torch.isfinite(yd).all(), f"{what}: non-finite output"
    bound = e + _ulp16(r.abs() + e) / 2
    ratio = (yd - r).abs() / bound
    worst = ratio.max().item()
    if worst > 1:
        i = tuple(torch.nonzero(ratio == ratio.max())[0].tolist())
        pytest.fail(f"{what}: |y - r| = {abs(yd[i] - r[i]).item():.3e} exceeds the bound {bound[i].item():.3e} at {i}: "
                    f"y = {yd[i].item()!r}, r = {r[i].item()!r} ({worst:.2f} x bound)")


@pytest.mark.parametrize("M,N,K,ldd,ldr", [(161, 264, 200, 272, 264), (1, 5120, 320, 5120, 5128),
                                           (4099, 320, 1280, 320, 328), (2561, 640, 2560, 648, 640),
                                           (129, 72, 5120, 72, 136), (65, 200, 8, 208, 200)])
def test_linear_random(M, N, K, ldd, ldr):
    """Random fp16 A, W, bias and residual (std 1 / sqrt(K) weights, as in a trained layer)."""
    g = torch.Generator(device="cuda").manual_seed(M + K)
    a = torch.randn((M, K), generator=g, device="cuda").half()
    w = (torch.randn((N, K), generator=g, device="cuda") / K ** 0.5).half()
    b = torch.randn((N,), generator=g, device="cuda").half()
    r = a.double() @ w.double().t() + b.double()
    e = _linear_bound(a, w, b, r)
    y, what = _linear(a, w, b, ldd=ldd)
    _assert_bound(y, r, e, what)
    # residual: y = fp16(t + resid) with t the fp16 result above, |t - r| <= e1; then one more half ulp
    resid = torch.full((M, ldr), float("nan"), dtype=torch.float16, device="cuda")
    resid[:, :N] = torch.randn((M, N), generator=g, device="cuda").half()
    r2 = r + resid[:, :N].double()
    e1 = e + _ulp16(r.abs() + e) / 2
    y2, what2 = _linear(a, w, b, ldd=ldd, resid=resid, ldr=ldr)
    _assert_bound(y2, r2, e1, what2)


# ---------------------------------------------------------------------------------------------------------------------
# HeadSplitEpi: q, k, v as the flash kernel reads them

def _check_head_major(ws, which, proj, B, H, L, d, DP, what):
    """ws: the workspace's fp16 view at the first projection written; proj [n][B * L, C] float64 (exact).  Layout
    [which][B][H][L][DP]: columns [0, d) hold the projection, [d, 16 ceil(d / 16)) zeros, the rest is never written."""
    n = proj.shape[0]
    qkv = ws[:n * B * H * L * DP].view(n, B, H, L, DP)
    dread = 16 * (-(-d // 16))
    for j in range(n):
        got = qkv[j]
        want = _round16(proj[j]).reshape(B, L, H, d).transpose(1, 2)
        _assert_equal(got[..., :d], want, f"{what}: {'qkv'[which + j]} values")
        assert (got[..., d:dread].view(torch.int16) == 0).all(), f"{what}: {'qkv'[which + j]} padding not zero"
        assert (got[..., dread:].view(torch.int16) == -1).all(), f"{what}: {'qkv'[which + j]} store beyond column {dread}"


def _run_self_split(B, L, d, H, seed):
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = d * H
    DP = 64 if d <= 64 else 128
    x, w, _ = _exact_inputs(B * L, 3 * C, C, g, bias=False)
    proj = _exact_product(x, w, None).view(B * L, 3, C).permute(1, 0, 2)
    ws_bytes = lib.vtm_attention_workspace_bytes(B, L, C, H)
    ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device="cuda")
    y = torch.full((B, L, C), float("nan"), dtype=torch.float16, device="cuda")
    wo = torch.eye(C, dtype=torch.float16, device="cuda")
    _lib.check(lib.vtm_attention_ex(x.data_ptr(), w.data_ptr(), wo.data_ptr(), None, B, L, C, H, 0.0, 0, y.data_ptr(),
                                    ws.data_ptr(), ws_bytes, _stream()), "vtm_attention_ex")
    torch.cuda.synchronize()
    _check_head_major(ws.view(torch.float16), 0, proj, B, H, L, d, DP, f"self B={B} L={L} d={d} H={H}")


def _run_cross_split(B, Lq, Lk, d, H, Cctx, seed):
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = d * H
    DP = 64 if d <= 64 else 128
    x, w_q, _ = _exact_inputs(B * Lq, C, C, g, bias=False)
    ctx, w_kv, _ = _exact_inputs(B * Lk, 2 * C, Cctx, g, bias=False)
    ws_bytes = lib.vtm_cross_attention_workspace_bytes(B, Lq, Lk, C, H)
    ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device="cuda")
    y = torch.full((B, Lq, C), float("nan"), dtype=torch.float16, device="cuda")
    wo = torch.eye(C, dtype=torch.float16, device="cuda")
    _lib.check(lib.vtm_cross_attention(x.data_ptr(), ctx.data_ptr(), w_q.data_ptr(), w_kv.data_ptr(), wo.data_ptr(),
                                       None, None, B, Lq, Lk, C, Cctx, H, 0.0, y.data_ptr(), ws.data_ptr(), ws_bytes,
                                       _stream()), "vtm_cross_attention")
    torch.cuda.synchronize()
    wsh = ws.view(torch.float16)
    what = f"cross B={B} Lq={Lq} Lk={Lk} d={d} H={H} Cctx={Cctx}"
    _check_head_major(wsh, 0, _exact_product(x, w_q, None).unsqueeze(0), B, H, Lq, d, DP, what)
    kv = _exact_product(ctx, w_kv, None).view(B * Lk, 2, C).permute(1, 0, 2)
    _check_head_major(wsh[B * H * Lq * DP:], 1, kv, B, H, Lk, d, DP, what)


SPLIT_LENGTHS = (1, 2, 3, 31, 33, 64, 65)
SPLIT_DIMS = (8, 40, 64, 72, 80, 128)


def _split_bh(L, d):
    """(B, H) cycling through a covering set; B >= 2 wherever L < 32 so that rows cross samples inside a warp."""
    i = SPLIT_LENGTHS.index(L) + SPLIT_DIMS.index(d)
    return ((2, 3), (3, 1), (3, 5), (2, 2), (1, 4))[i % 5] if L >= 32 else ((2, 3), (3, 2), (3, 5), (2, 1))[i % 4]


@pytest.mark.parametrize("d", SPLIT_DIMS)
@pytest.mark.parametrize("L", SPLIT_LENGTHS)
def test_head_split_self(L, d):
    B, H = _split_bh(L, d)
    _run_self_split(B, L, d, H, seed=100 * L + d)


@pytest.mark.parametrize("d", SPLIT_DIMS)
@pytest.mark.parametrize("L", SPLIT_LENGTHS)
def test_head_split_cross(L, d):
    """q from x (K = C); k and v from the context by one GEMM (which0 = 1, n_proj = 2, K = Cctx)."""
    B, H = _split_bh(L, d)
    _run_cross_split(B, 33 if L < 32 else 3, L, d, H, 768 if d % 16 else 1024, seed=100 * L + d + 1)


@pytest.mark.parametrize("d,H", [(40, 11), (80, 11), (8, 41)])
def test_head_split_projection_boundaries(d, H):
    """C = 440, 880 and 328: the fp32 product n * (1 / C) falls just below an integer at n = C and 2C, so these widths
    check that the epilogue's division sends the first column of k and of v to the right projection."""
    _run_self_split(2, 33, d, H, seed=d + H)
    _run_cross_split(2, 3, 33, d, H, 768, seed=d + H + 1)
