"""The dense kernels at the edges of fp16's range: results that round past 65504, subnormal and signed-zero results, and
infinite or NaN operands, against float64 and torch.  Needs an H100 (sm_90a).

The rule, element by element:
1. Class.  NaN, +inf, -inf or finite must be the class of the float64 IEEE evaluation of the same op at the library's
   fp16 storage points (the projection outputs, T = a D^T of a LoRA, the gelu output, O of the flash kernel).  For a
   GEMM this class does not depend on the summation order: |a w| <= 65504^2 and K <= 5120 cannot overflow fp32, so only
   inf / NaN operands and the final rounding to fp16 decide it (inf + -inf and inf * 0 give NaN in any order).
2. Value.  The GEMM designs are exact in fp32 in any order (asserted), so their finite elements are checked bit for bit,
   65504 / 65520 rounding, subnormals and the sign of zero included.  The flash kernel's finite rows meet
   tests/test_gpu_attention_core.py's bound, with keys of weight 0 left out of it.
3. Torch.  For the ops whose semantics come from torch, the class of torch's CUDA result on the same fp16 inputs as
   well: F.gelu (erf form), F.layer_norm, F.group_norm, math-backend softmax attention; KT bit for bit.

Every call goes through the C-ABI with NaN-filled, sentinel-guarded outputs (GEMMs) or a 0xFF workspace (attention)."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from vidtome_b200 import _lib, ops
from test_gpu_attention_core import LOG2E
from test_gpu_attention_core import _ulp16 as _ulp16_attn
from test_gpu_projection_core import _check_guards, _guarded, _ptr, _stream
from test_gpu_rows_core import _check_ln, _round16

pytestmark = pytest.mark.gpu

INF, NAN = math.inf, math.nan


# ---------------------------------------------------------------------------------------------------------------------
# IEEE helpers in float64

def _rn16(x):
    """float64 -> the fp16 value IEEE round-to-nearest-even gives (|x| >= 65520 -> +-inf, NaN stays); still float64."""
    fin = torch.isfinite(x)
    r = torch.where(fin, x, torch.zeros_like(x))
    r = _round16(r.clamp(-65504, 65504))
    r = torch.where(fin & (x.abs() >= 65520), torch.copysign(torch.full_like(x, INF), x), r)
    # the sign of a result that rounds to zero is the sign of x
    r = torch.where(fin & (r == 0), torch.copysign(torch.zeros_like(x), x), r)
    return torch.where(fin, r, x)


def _mm(a, b):
    """a [M, K] @ b [K, N] in float64, elementwise IEEE (inf * 0 = NaN, inf + -inf = NaN), for small operands."""
    return (a.unsqueeze(-1) * b.unsqueeze(0)).sum(1)


def _cls(t):
    """0 finite, 1 +inf, 2 -inf, 3 NaN."""
    t = t.double()
    c = torch.zeros(t.shape, dtype=torch.int8, device=t.device)
    c[t == INF] = 1
    c[t == -INF] = 2
    c[torch.isnan(t)] = 3
    return c


def _assert_class(y, want, what):
    cy, cw = _cls(y), _cls(want)
    bad = cy != cw
    if bad.any():
        i = tuple(torch.nonzero(bad)[0].tolist())
        pytest.fail(f"{what}: {int(bad.sum())} of {bad.numel()} elements in the wrong class; first at {i}: "
                    f"got {y[i].item()!r}, want {want[i].item()!r}")


def _assert_bits(y, want, what):
    """y fp16; want float64 holding fp16 values (or inf / NaN): bit-equal, or both NaN."""
    w16 = want.half()
    ok = (y.view(torch.int16) == w16.view(torch.int16)) | (torch.isnan(y) & torch.isnan(w16))
    if not ok.all():
        i = tuple(torch.nonzero(~ok)[0].tolist())
        pytest.fail(f"{what}: {int((~ok).sum())} of {ok.numel()} elements differ; first at {i}: got {y[i].item()!r} "
                    f"(0x{int(y.view(torch.int16)[i]) & 0xFFFF:04x}), want {w16[i].item()!r} "
                    f"(0x{int(w16.view(torch.int16)[i]) & 0xFFFF:04x})")


def _assert_fp32_exact(x, what):
    f = x[torch.isfinite(x)]
    assert torch.equal(f.float().double(), f), f"{what}: the design is not exact in fp32"


def _h(vals):
    return torch.tensor(vals, dtype=torch.float64, device="cuda").half()


# ---------------------------------------------------------------------------------------------------------------------
# StoreEpi / NchwEpi / LoRA: y[m, n] = a[m, 0] + c_n a[m, 1] (+ T U^T) + bias[n] (+ resid)

# (a0, a1) pairs: sums landing on 65504, 65519, 65520 (a tie that rounds to inf) and beyond, both signs; subnormal
# results, ties between subnormals and +-0 (2^-25 and 1.5 2^-24 through c = 0.5); inf / NaN operands, one of them meeting
# a zero weight.  A row's products are all on one grid (2^-2 or 2^-26) and small enough to be exact in fp32 in any order.
ROWS = [(65504, 0), (65504, 15), (65504, 16), (65504, 32), (-65504, -16), (-65504, -15), (60000, 5519), (60000, 5520),
        (2 ** -24, 0), (0, 2 ** -24), (0, -2 ** -24), (0, 3 * 2 ** -24), (2 ** -24, -2 ** -24), (-2 ** -24, 2 ** -24),
        (2 ** -14, -2 ** -24), (5, -5), (0, 0), (1, 1), (INF, 0), (INF, 1), (-INF, 1), (INF, -INF), (NAN, 0), (1, INF),
        (1, NAN), (0, -0.0)]
COEFS = [1, -1, 0, 0.5, -0.5, 2, -2, 0.25]                                # c_n, column n % 8
BIASES = [0, -0.0, 16, -16, 32, 2 ** -24, INF, NAN]                       # bias_n, column (n // 8) % 8
RESIDS = [0, -0.0, 16, -16, 32, -32, 2 ** -24, -2 ** -24, INF, -INF, NAN, 1]
K_EDGE = 32


def _edge_operands(M, N):
    rows = torch.tensor([ROWS[i % len(ROWS)] for i in range(M)], dtype=torch.float64, device="cuda")
    a = torch.zeros((M, K_EDGE), dtype=torch.float64, device="cuda")
    a[:, :2] = rows
    w = torch.zeros((N, K_EDGE), dtype=torch.float64, device="cuda")
    w[:, 0] = 1
    w[:, 1] = torch.tensor([COEFS[n % 8] for n in range(N)], dtype=torch.float64, device="cuda")
    b = torch.tensor([BIASES[(n // 8) % 8] for n in range(N)], dtype=torch.float64, device="cuda")
    return a.half(), w.half(), b.half()


def _resid(M, N):
    i = torch.arange(M * N, device="cuda").view(M, N)
    vals = torch.tensor(RESIDS, dtype=torch.float64, device="cuda")
    return vals[(i * 7 + i // N) % len(RESIDS)].half()


def _store_reference(a, w, b, t=None, u=None, resid=None):
    """The library's storage points: acc exact in fp32 (asserted, as is the sum of |products|, which bounds every
    partial sum), fp32(acc + bias) rounded once (the epilogue's __fadd_rn), fp16 of that, fp16(that + resid)."""
    acc = _mm(a.double(), w.double().t())
    mag = _mm(a.double().abs(), w.double().abs().t())
    if t is not None:
        acc = acc + _mm(t, u.double().t())
        mag = mag + _mm(t.abs(), u.double().abs().t())
    _assert_fp32_exact(acc, "acc")
    _assert_fp32_exact(mag, "sum of |products|")
    r = acc if b is None else (acc.float() + b.float()).double()
    y = _rn16(r)
    return y if resid is None else _rn16(y + resid.double())


def _call_linear(a, w, b, resid=None, lora=None):
    lib = _lib.load()
    M, K = a.shape
    N = w.shape[0]
    ldd = N + 8
    d = _guarded(M, N, ldd)
    if lora is not None:
        dn, up = lora
        desc = _lib.VtmLora(dn.data_ptr(), up.data_ptr(), dn.shape[0])
        ws_bytes = lib.vtm_linear_lora_workspace_bytes(M, dn.shape[0])
        ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device="cuda")
        rc = lib.vtm_linear_lora_f16(a.data_ptr(), w.data_ptr(), _ptr(b), _ptr(resid), N if resid is not None else 0,
                                     ctypes.byref(desc), M, N, K, d.data_ptr(), ldd, ws.data_ptr(), ws_bytes, _stream())
    elif resid is None:
        rc = lib.vtm_linear_f16(a.data_ptr(), w.data_ptr(), _ptr(b), M, N, K, d.data_ptr(), ldd, _stream())
    else:
        rc = lib.vtm_linear_residual_f16(a.data_ptr(), w.data_ptr(), _ptr(b), resid.data_ptr(), N, M, N, K,
                                         d.data_ptr(), ldd, _stream())
    _lib.check(rc, "linear")
    torch.cuda.synchronize()
    what = f"linear M={M} N={N} bias={b is not None} resid={resid is not None} lora={lora is not None}"
    _check_guards(d, M, N, what)
    return d[:M, :N], what


@pytest.mark.parametrize("M,N", [(len(ROWS), 64), (161, 72), (4 * len(ROWS), 200)])
@pytest.mark.parametrize("bias", (True, False))
def test_store_epi_range_edges(M, N, bias):
    """vtm_linear_f16 and vtm_linear_residual_f16, bit for bit: the full-chunk and per-store paths (N = 72, 200 and
    M = 161 leave partial chunks and warps)."""
    a, w, b = _edge_operands(M, N)
    b = b if bias else None
    y, what = _call_linear(a, w, b)
    _assert_bits(y, _store_reference(a, w, b), what)
    resid = _resid(M, N)
    y, what = _call_linear(a, w, b, resid=resid)
    _assert_bits(y, _store_reference(a, w, b, resid=resid), what)


def test_store_epi_lora_range_edges():
    """vtm_linear_lora_f16, bit for bit against y = fp16(a W^T + T U^T + bias (+ resid)) with T = fp16(a D^T) rounded
    as the library stores it.  First: T's column 1 = 2 a0 overflows to +-inf wherever |a0| >= 32768, against a column
    of U with no zero (a zero would turn the whole row to NaN), T's column 0 = a0 sums with the main product past 65504,
    and U holds a NaN in one column.  Second: D holds inf (T = a0 inf: NaN where a0 = 0)."""
    M, N, R = 2 * len(ROWS), 64, 8
    a, w, b = _edge_operands(M, N)
    n = torch.arange(N, device="cuda")
    pick = lambda vals, idx: torch.tensor(vals, dtype=torch.float64, device="cuda")[idx]
    designs = []
    dn = torch.zeros((R, K_EDGE), dtype=torch.float64, device="cuda")
    dn[0, 0], dn[1, 0], dn[2, 1] = 1, 2, 1
    up = torch.zeros((N, R), dtype=torch.float64, device="cuda")
    up[:, 0] = pick([0, 1, -1, 0.5], n % 4)
    up[:, 1] = pick([1, -1, 0.5, 2, -2], n % 5)
    up[:, 2] = pick([0, 1, 0.5], n % 3)
    up[N - 1, 0] = NAN
    designs.append((dn, up))
    dn = torch.zeros((R, K_EDGE), dtype=torch.float64, device="cuda")
    dn[0, 0] = INF
    up = torch.zeros((N, R), dtype=torch.float64, device="cuda")
    up[:, 0] = pick([1, -1], n % 2)
    designs.append((dn, up))
    for dn, up in designs:
        dn, up = dn.half(), up.half()
        t = _rn16(_mm(a.double(), dn.double().t()))
        for resid in (None, _resid(M, N)):
            y, what = _call_linear(a, w, b, resid=resid, lora=(dn, up))
            _assert_bits(y, _store_reference(a, w, b, t=t, u=up, resid=resid), what)


@pytest.mark.parametrize("HW", (1, 63, 64))
def test_nchw_epi_range_edges(HW):
    """vtm_linear_nchw_residual_f16 with HW = 1 and 63 (per-token stores) and 64 (16-byte vectors), with and without
    bias and residual: the StoreEpi reference, transposed."""
    lib = _lib.load()
    n_s = max(2, -(-len(ROWS) // HW) + 1)
    M, N = n_s * HW, 72
    a, w, b = _edge_operands(M, N)
    for bias, with_resid in ((True, True), (False, True), (True, False)):
        bb = b if bias else None
        resid = _resid(M, N).view(n_s, HW, N).transpose(1, 2).contiguous() if with_resid else None
        d = torch.full((n_s, N, HW), NAN, dtype=torch.float16, device="cuda")
        _lib.check(lib.vtm_linear_nchw_residual_f16(a.data_ptr(), w.data_ptr(), _ptr(bb), _ptr(resid), n_s, HW, N,
                                                    K_EDGE, d.data_ptr(), _stream()), "vtm_linear_nchw_residual_f16")
        torch.cuda.synchronize()
        r_tok = None if resid is None else resid.transpose(1, 2).reshape(M, N)
        want = _store_reference(a, w, bb, resid=r_tok).view(n_s, HW, N).transpose(1, 2)
        _assert_bits(d, want, f"nchw HW={HW} bias={bias} resid={with_resid}")


# ---------------------------------------------------------------------------------------------------------------------
# GegluEpi

# value and gate before the bias; every gate after its bias is 0, |g| >= 8 (where fp16(gelu(g)) is g or -0 exactly),
# +-inf or NaN, so that fp16(gelu) is known exactly
GEGLU_ROWS = [(1, 65504), (1, -65504), (1, 8), (1, -8), (2, 16), (-2, -16), (65504, 16), (65504, 8), (-65504, 8),
              (1000, 1000), (0.5, 0), (0, 65504), (-1, 1000), (65504, -65504), (1, 40)]
GATE_BIAS = [0, 16, -16, 32, NAN, -32, 0, 0]             # gate bias of output column j: j % 8
VALUE_BIAS = [0, 0, 32, 0, 0, 0, INF, -32]               # value bias of output column j: (j // 8) % 8


def _gelu16_exact(g):
    """fp16(gelu(g)) for the gates above (float64 holding fp16 values): gelu(+inf) = +inf, gelu(-inf) = NaN
    (-inf * 0, as float64's g * Phi(g) and torch's g / 2 (1 + erf(g / sqrt 2)) give), g for g >= 8, -0 for g <= -8,
    +0 for g = 0."""
    fin = torch.isfinite(g)
    assert ((g[fin] == 0) | (g[fin].abs() >= 8)).all(), "a gate outside the exactly known set"
    q = torch.where(g >= 8, g, torch.full_like(g, -0.0))
    q = torch.where(g == 0, torch.zeros_like(g), q)
    q = torch.where(g == INF, g, q)
    return torch.where(torch.isnan(g) | (g == -INF), torch.full_like(g, NAN), q)


def test_geglu_range_edges():
    """vtm_linear_geglu_f16 and vtm_linear_geglu_lora_f16: gates at +-inf (acc + bias overflowing), NaN, +-65504; the
    value at inf against gelu = -0 (inf * 0 = NaN) and the product overflowing through HMUL2.  Bit for bit against
    fp16(value * fp16(gelu(gate))) and, for the gelu alone, the class of CUDA F.gelu on the same fp16 gates.  The
    non-finite gates come from the biases and from overflow: an inf in A would meet the value rows' zero weights."""
    lib = _lib.load()
    M, inner, K = 2 * len(GEGLU_ROWS), 64, 16
    rows = torch.tensor([GEGLU_ROWS[i % len(GEGLU_ROWS)] for i in range(M)], dtype=torch.float64, device="cuda")
    a = torch.zeros((M, K), dtype=torch.float64, device="cuda")
    a[:, :2] = rows
    w = torch.zeros((2 * inner, K), dtype=torch.float64, device="cuda")
    w[:inner, 0] = 1
    w[inner:, 1] = 1
    j = torch.arange(inner, device="cuda")
    b = torch.cat([torch.tensor(VALUE_BIAS, dtype=torch.float64, device="cuda")[(j // 8) % 8],
                   torch.tensor(GATE_BIAS, dtype=torch.float64, device="cuda")[j % 8]])
    a, w, b = a.half(), w.half(), b.half()
    r = _rn16(_mm(a.double(), w.double().t()) + b.double())
    v16, g16 = r[:, :inner], r[:, inner:]
    q = _gelu16_exact(g16)
    assert torch.equal(_cls(F.gelu(g16.half())), _cls(q)), "CUDA F.gelu disagrees with float64 on a gate's class"
    want = _rn16(v16 * q)
    wi, bi = ops.interleave_geglu(w, b)
    R = 8
    dn = torch.zeros((R, K), dtype=torch.float16, device="cuda")
    up = torch.zeros((2 * inner, R), dtype=torch.float16, device="cuda")
    for lora in (False, True):
        d = _guarded(M, inner, inner + 8)
        if lora:
            # a zero LoRA: the K tail adds +0 products, which changes no class and no bit
            up_il = ops.interleave_geglu(up, None)[0].contiguous()
            desc = _lib.VtmLora(dn.data_ptr(), up_il.data_ptr(), R)
            ws_bytes = lib.vtm_linear_lora_workspace_bytes(M, R)
            ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device="cuda")
            rc = lib.vtm_linear_geglu_lora_f16(a.data_ptr(), wi.data_ptr(), bi.data_ptr(), ctypes.byref(desc), M,
                                               2 * inner, K, d.data_ptr(), inner + 8, ws.data_ptr(), ws_bytes,
                                               _stream())
        else:
            rc = lib.vtm_linear_geglu_f16(a.data_ptr(), wi.data_ptr(), bi.data_ptr(), M, 2 * inner, K, d.data_ptr(),
                                          inner + 8, _stream())
        _lib.check(rc, "geglu")
        torch.cuda.synchronize()
        what = f"geglu lora={lora}"
        _check_guards(d, M, inner, what)
        _assert_bits(d[:M, :inner], want, what)


# ---------------------------------------------------------------------------------------------------------------------
# HeadSplitEpi + the flash kernel

def _attn_ieee(q, k, v, scale):
    """softmax(q k^T scale) v in float64 IEEE for q [B, H, Lq, d] finite, k, v [B, H, Lk, d] with inf entries.
    Returns (O, bound): the bound of test_gpu_attention_core's _reference, over the keys of non-zero weight, where O
    is finite."""
    assert torch.isfinite(q).all()
    tl = float(scale) * LOG2E

    def ieee_mm(x, y):                          # x [..., M, K] @ y [..., K, N]; y may hold inf
        nf = ~torch.isfinite(y)
        r = x @ torch.where(nf, torch.zeros_like(y), y)
        for j in torch.nonzero(nf.flatten(0, -3).any(0).any(-1)).flatten().tolist():
            r = r + x[..., :, j:j + 1] * torch.where(nf[..., j:j + 1, :], y[..., j:j + 1, :], torch.zeros_like(y[..., j:j + 1, :]))
        return r

    t = ieee_mm(q, k.transpose(-1, -2)) * tl
    w = torch.exp2(t - t.amax(-1, keepdim=True))
    # a row whose every key scores -inf is 0 / 0 in IEEE; torch's attention (the math backend's safe softmax, as
    # FlashAttention-2) returns 0 for it, and so does the kernel (DESIGN §1)
    w = torch.where((t == -INF).all(-1, keepdim=True), torch.zeros_like(w), w)
    l = w.sum(-1, keepdim=True)
    O = ieee_mm(w, v) / torch.where(l == 0, torch.ones_like(l), l)
    tmax = torch.where(torch.isfinite(t), t.abs(), torch.zeros_like(t)).amax(-1)
    rows = torch.isfinite(O).any(-1)
    assert not rows.any() or tmax[rows].max().item() <= 512, "scores beyond the bound's range"
    va = torch.where(torch.isfinite(v), v.abs(), torch.zeros_like(v))
    pv = (w @ va) / l
    sub = (w.clamp(max=2.0 ** -25) @ va) / l
    return O, 2 * 2.0 ** -11 * pv + sub + _ulp16_attn(O)


def _check_flash(o, O, bound, torch_o, what):
    """o [B, H, L, d] fp16 (the flash kernel's output, read from the workspace), O / bound from _attn_ieee, torch_o the
    math-backend attention on the same fp16 q, k, v."""
    _assert_class(o, O, f"{what}: flash O against float64")
    _assert_class(o, torch_o, f"{what}: flash O against torch math attention")
    fin = torch.isfinite(O)
    err = (o.double() - O).abs()
    ratio = torch.where(fin, err / bound, torch.zeros_like(err))
    if ratio.max().item() > 1:
        i = tuple(torch.nonzero(ratio == ratio.max())[0].tolist())
        pytest.fail(f"{what}: |o - O| = {err[i].item():.3e} exceeds the bound {bound[i].item():.3e} at {i}: "
                    f"o = {o[i].item()!r}, O = {O[i].item()!r}")


def _eye_proj(o):
    """The class of o I^T in IEEE arithmetic: o_c, or NaN where another element of the row is non-finite (times 0)."""
    nf = ~torch.isfinite(o)
    other = (nf.sum(-1, keepdim=True) - nf.int()) > 0
    return torch.where(other, torch.full_like(o, NAN), o)


def _torch_attention(q16, k16, v16, scale):
    from torch.nn.attention import SDPBackend, sdpa_kernel
    with sdpa_kernel(SDPBackend.MATH):
        return F.scaled_dot_product_attention(q16, k16, v16, scale=scale)


def _heads(t, H):
    B, L, C = t.shape
    return t.view(B, L, H, C // H).transpose(1, 2)


def _hot_keys(where, L):
    nt = -(-L // 64)
    if where == "tile0":
        return range(0, min(64, L))
    if where == "middle":
        m = nt // 2
        return range(64 * m, min(64 * m + 64, L))
    if where == "last":
        return range(64 * (nt - 1), L)
    if where == "all":
        return range(L)
    if where == "none":
        return range(0)
    raise ValueError(where)


def _q_component(Lq, dev="cuda"):
    """The component of the overflowing K channel for every query: -1, 0, +1, -0.5 in turn (scores -inf, NaN, +inf)."""
    return torch.tensor([-1.0, 0.0, 1.0, -0.5], dtype=torch.float64, device=dev)[torch.arange(Lq, device=dev) % 4]


def _cross_edges(B, Lq, Lk, d, H, k_hot, v_hot, seed, scale=None):
    """vtm_cross_attention with W_q = I, W_k = [diag(s_k) | 0], W_v = [0 | diag(s_v)], W_o = I: s_k = 2 at channel 0
    of every head and s_v = 2 at channel 1, so a context value of +-40000 there overflows to +-inf in HeadSplitEpi's
    fp16 store, for the keys in k_hot (K) and v_hot (V: +inf in the first tile, -inf past it)."""
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = d * H
    DP = 64 * -(-(16 * -(-d // 16)) // 64)
    grid = lambda shape, lim: (torch.randint(-lim * 8, lim * 8 + 1, shape, generator=g, device="cuda") / 8).double()
    Q = grid((B, Lq, H, d), 2)
    Q[..., 0] = _q_component(Lq).view(1, Lq, 1)
    Kx, Vx = grid((B, Lk, H, d), 2), grid((B, Lk, H, d), 4)
    for j in k_hot:
        Kx[:, j, :, 0] = 40000
    for j in v_hot:
        Vx[:, j, :, 1] = 40000 if j < 64 else -40000
    Q, Kx, Vx = (t.reshape(t.shape[0], t.shape[1], C).half() for t in (Q, Kx, Vx))
    sk = torch.ones(C, dtype=torch.float64, device="cuda")
    sv = sk.clone()
    sk[0::d], sv[1::d] = 2, 2
    w_kv = torch.zeros((2 * C, 2 * C), dtype=torch.float64, device="cuda")
    w_kv[:C, :C] = torch.diag(sk)
    w_kv[C:, C:] = torch.diag(sv)
    w_kv = w_kv.half()
    eye = torch.eye(C, dtype=torch.float16, device="cuda")
    ctx = torch.cat([Kx, Vx], -1).contiguous()
    scale = d ** -0.5 if scale is None else scale
    ws_bytes = lib.vtm_cross_attention_workspace_bytes(B, Lq, Lk, C, H)
    ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device="cuda")
    y = torch.full((B, Lq, C), NAN, dtype=torch.float16, device="cuda")
    _lib.check(lib.vtm_cross_attention(Q.data_ptr(), ctx.data_ptr(), eye.data_ptr(), w_kv.data_ptr(), eye.data_ptr(),
                                       None, None, B, Lq, Lk, C, 2 * C, H, float(scale), y.data_ptr(), ws.data_ptr(),
                                       ws_bytes, _stream()), "vtm_cross_attention")
    torch.cuda.synchronize()
    off = B * H * (Lq + 2 * Lk) * DP
    o = ws.view(torch.float16)[off:off + B * Lq * C].view(B, Lq, C)
    K16 = _rn16(Kx.double() * sk).half()
    V16 = _rn16(Vx.double() * sv).half()
    q, k, v = _heads(Q, H), _heads(K16, H), _heads(V16, H)
    O, bound = _attn_ieee(q.double(), k.double(), v.double(), scale)
    what = f"cross B={B} Lq={Lq} Lk={Lk} d={d} H={H}"
    _check_flash(_heads(o, H), O, bound, _torch_attention(q, k, v, scale), what)
    # the output projection with W_o = I: a non-finite element of o meets the zeros of I, so its whole row is NaN
    _assert_class(y.view(B * Lq, C), _eye_proj(_rn16(O.transpose(1, 2).reshape(B * Lq, C))), f"{what}: y")
    return o, O


EDGE_LENGTHS = (1, 63, 64, 65, 129, 1000)


@pytest.mark.parametrize("where", ("tile0", "middle", "last", "all"))
@pytest.mark.parametrize("d", (40, 64, 128, 160))
@pytest.mark.parametrize("Lk", EDGE_LENGTHS)
def test_flash_k_overflow(Lk, d, where):
    """K's channel 0 overflows to +inf for every key of one tile (the first, a middle one, the masked last one) or of
    all tiles; the queries' component there is -1, 0 or +1, so those keys score -inf, NaN or +inf.  A row whose first
    tile is all -inf and whose later tiles are finite must come out finite (FlashAttention-2's safe maximum); a row
    whose every key scores -inf comes out 0, as torch's attention returns it (IEEE's 0 / 0 would be NaN)."""
    _cross_edges(2, 67, Lk, d, 2, _hot_keys(where, Lk), (), seed=Lk * 7 + d)


@pytest.mark.parametrize("d", (40, 160))
@pytest.mark.parametrize("Lk", (1, 65, 1000))
def test_flash_v_overflow(Lk, d):
    """V's channel 1 overflows to +inf for the keys of the first tile (and to -inf for a second group) at scale 0,
    where every key has weight 1: O is +inf, or NaN where +inf and -inf meet; the other channels stay finite."""
    hot = list(range(min(Lk, 3))) + list(range(max(3, Lk - 2), Lk))
    _cross_edges(2, 33, Lk, d, 2, (), hot, seed=Lk + d, scale=0.0)


def test_flash_v_overflow_underflowed_weight():
    """Deviation (DESIGN §1): an infinite v of a key whose weight underflows to 0 in the kernel's fp16 P gives NaN,
    where float64 and torch's math attention (whose weight stays positive) give inf.  Two keys, the second 60 log2 units
    below the first.  v overflows in HeadSplitEpi's store (context 40000 against a weight of 2), as in _cross_edges: an
    inf in the context itself would meet the projection's zero weights and make the whole row of v NaN."""
    lib = _lib.load()
    B, Lq, Lk, H, d = 1, 2, 2, 1, 16
    C = H * d
    Q = torch.zeros((B, Lq, C), dtype=torch.float16, device="cuda")
    Q[..., 0] = 1
    K = torch.zeros((B, Lk, C), dtype=torch.float16, device="cuda")
    K[0, 0, 0] = 4
    V = torch.zeros((B, Lk, C), dtype=torch.float16, device="cuda")
    V[0, 1, 1] = 40000
    scale = 60 / (4 * LOG2E)
    ctx = torch.cat([K, V], -1).contiguous()
    eye, eye2 = torch.eye(C, dtype=torch.float16, device="cuda"), torch.eye(2 * C, dtype=torch.float16, device="cuda")
    eye2[C + 1, C + 1] = 2
    V = _rn16(V.double() * 2).half()
    ws_bytes = lib.vtm_cross_attention_workspace_bytes(B, Lq, Lk, C, H)
    ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device="cuda")
    y = torch.empty((B, Lq, C), dtype=torch.float16, device="cuda")
    _lib.check(lib.vtm_cross_attention(Q.data_ptr(), ctx.data_ptr(), eye.data_ptr(), eye2.data_ptr(), eye.data_ptr(),
                                       None, None, B, Lq, Lk, C, 2 * C, H, float(scale), y.data_ptr(), ws.data_ptr(),
                                       ws_bytes, _stream()), "vtm_cross_attention")
    torch.cuda.synchronize()
    off = B * H * (Lq + 2 * Lk) * 64
    o = ws.view(torch.float16)[off:off + B * Lq * C].view(B, Lq, C)
    O, _ = _attn_ieee(_heads(Q, H).double(), _heads(K, H).double(), _heads(V, H).double(), scale)
    assert (O[0, 0, :, 1] == INF).all(), "float64 weight underflowed: the design no longer shows the deviation"
    assert torch.isnan(o[..., 1]).all(), f"o[:, 1] = {o[..., 1].tolist()}"
    assert (_torch_attention(_heads(Q, H), _heads(K, H), _heads(V, H), scale)[..., 1] == INF).all()
    assert torch.isfinite(o[..., [0] + list(range(2, C))]).all()


def _self_edges(B, L, d, H, where, seed, flags=0, n_valid=None, resid=False):
    """Self-attention with W_qkv = [I; 2 I; I]: x = +-40000 in channel 0 of the hot keys' rows overflows k to +inf
    there (q and v stay 40000); the other rows' channel 0 cycles through -1, 0, +1, -0.5.  flags = 1 shares q / k of
    sample 0 (VTM_ATTN_SHARED_QK); n_valid < L runs vtm_attention_dev with the first n_valid rows valid; resid runs
    vtm_attention_residual_ex."""
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = d * H
    n = L if n_valid is None else n_valid
    DP = 64 * -(-(16 * -(-d // 16)) // 64)
    x = (torch.randint(-16, 17, (B, L, H, d), generator=g, device="cuda") / 8).double()
    x[:, :, :, 0] = _q_component(L).view(1, L, 1)
    for j in _hot_keys(where, n):
        x[:, j, :, 0] = 40000
    x = x.reshape(B, L, C).half()
    eye = torch.eye(C, dtype=torch.float16, device="cuda")
    w = torch.cat([eye, 2 * eye, eye]).contiguous()
    ws_bytes = lib.vtm_attention_workspace_bytes(B, L, C, H)
    ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device="cuda")
    y = torch.full((B, L, C), NAN, dtype=torch.float16, device="cuda")
    r = (torch.randint(-16, 17, (B, L, C), generator=g, device="cuda") / 8).half()
    if resid:
        rc = lib.vtm_attention_residual_ex(x.data_ptr(), w.data_ptr(), eye.data_ptr(), None, r.data_ptr(), None, None,
                                           B, L, C, H, float(d ** -0.5), flags, 1, y.data_ptr(), ws.data_ptr(),
                                           ws_bytes, _stream())
    elif n_valid is not None:
        len_dev = torch.tensor([n], dtype=torch.int32, device="cuda")
        rc = lib.vtm_attention_dev(x.data_ptr(), w.data_ptr(), eye.data_ptr(), None, B, L, C, H, float(d ** -0.5),
                                   flags, len_dev.data_ptr(), y.data_ptr(), ws.data_ptr(), ws_bytes, _stream())
    else:
        rc = lib.vtm_attention_ex(x.data_ptr(), w.data_ptr(), eye.data_ptr(), None, B, L, C, H, float(d ** -0.5),
                                  flags, y.data_ptr(), ws.data_ptr(), ws_bytes, _stream())
    _lib.check(rc, "self-attention")
    torch.cuda.synchronize()
    off = 3 * B * H * L * DP
    o = ws.view(torch.float16)[off:off + B * L * C].view(B, L, C)[:, :n]
    xs = x[:, :n]
    qk = xs[:1].expand(B, -1, -1) if flags & 1 else xs
    q, k, v = _heads(qk, H), _heads(_rn16(2 * qk.double()).half(), H), _heads(xs, H)
    O, bound = _attn_ieee(q.double(), k.double(), v.double(), d ** -0.5)
    what = f"self B={B} L={L} n={n} d={d} H={H} {where} flags={flags} resid={resid}"
    _check_flash(_heads(o, H), O, bound, _torch_attention(q, k, v, d ** -0.5), what)
    want = _eye_proj(_rn16(O.transpose(1, 2).reshape(B * n, C)))
    if resid:
        want = _rn16(_rn16(want) + r[:, :n].reshape(B * n, C).double())
    _assert_class(y[:, :n].reshape(B * n, C), want, f"{what}: y")


@pytest.mark.parametrize("where", ("tile0", "last", "all"))
@pytest.mark.parametrize("L,d", [(1, 40), (65, 40), (129, 64), (64, 128), (1000, 160)])
def test_self_attention_k_overflow(L, d, where):
    """vtm_attention_ex: the QKV projection's HeadSplitEpi stores +inf into k; the query rows of the hot keys score
    +inf against them (NaN rows), the others -inf, NaN or +inf."""
    _self_edges(2, L, d, 2, where, seed=L + d)


@pytest.mark.parametrize("L,d", [(65, 40), (1000, 80)])
def test_shared_qk_k_overflow(L, d):
    """VTM_ATTN_SHARED_QK: sample 0's overflowing k serves every sample."""
    _self_edges(3, L, d, 2, "tile0", seed=L + d + 1, flags=1)


@pytest.mark.parametrize("n", (1, 65, 129))
def test_device_length_k_overflow(n):
    """vtm_attention_dev at a capacity of 200 rows: the overflowing tile is the first or the device-length last one;
    the rows past n hold finite values (the header asks for that) and take no part."""
    for where in ("tile0", "last"):
        _self_edges(2, 200, 40, 2, where, seed=n, n_valid=n)


@pytest.mark.parametrize("flags", (0, 1))
def test_attention_residual_k_overflow(flags):
    """vtm_attention_residual_ex: the residual is added after the output projection's fp16 rounding."""
    _self_edges(3, 129, 80, 2, "tile0", seed=5 + flags, flags=flags, resid=True)


# ---------------------------------------------------------------------------------------------------------------------
# fused LayerNorm, GroupNorm, KT

def _ln64_class(x):
    """Class of LayerNorm in float64 IEEE: a row holding inf or NaN has a non-finite mean: every element NaN."""
    bad = ~torch.isfinite(x.double()).all(-1, keepdim=True)
    return torch.where(bad, torch.full(x.shape, NAN, dtype=torch.float64, device=x.device),
                       torch.zeros(x.shape, dtype=torch.float64, device=x.device))


@pytest.mark.parametrize("C", (40, 320, 1280))
def test_layer_norm_range_edges(C):
    """ops.layer_norm (KC + LN): rows holding +inf, -inf, both, NaN, and finite rows of +-65504 (alternating, constant,
    one entry), against F.layer_norm's class and float64; the finite rows within `_check_ln`'s bound."""
    g = torch.Generator(device="cuda").manual_seed(C)
    x = torch.randn((12, C), generator=g, device="cuda", dtype=torch.float64)
    x[0, 3], x[1, 5], x[2, 0], x[2, C - 1], x[3, 7] = INF, -INF, INF, -INF, NAN
    x[4] = torch.where(torch.arange(C, device="cuda") % 2 == 0, 65504.0, -65504.0)
    x[5] = 65504
    x[6] = -65504
    x[7, 1] = 65504
    x[8] = 0
    x[8, 0] = -65504
    x = x.half()
    w = (1 + 0.5 * torch.randn(C, generator=g, device="cuda")).half()
    b = (0.5 * torch.randn(C, generator=g, device="cuda")).half()
    y = ops.layer_norm(x, (w, b, 1e-5))
    torch.cuda.synchronize()
    _assert_class(y, _ln64_class(x), f"layer_norm C={C} against float64")
    _assert_class(y, F.layer_norm(x, (C,), w, b, 1e-5), f"layer_norm C={C} against F.layer_norm")
    fin = torch.isfinite(x).all(-1)
    _check_ln(y[fin], x[fin], (w, b, 1e-5), f"layer_norm C={C} finite rows")


@pytest.mark.parametrize("C,HW,groups", [(320, 64, 32), (640, 63, 32), (40, 16, 8)])
def test_group_norm_range_edges(C, HW, groups):
    """KG1 + KG2 (ops.group_norm_tokens): one inf, one -inf, +inf and -inf together, and one NaN, each in its own group
    of its own sample; every element of those groups is NaN (a non-finite mean), as in float64 and F.group_norm, and
    every other group is finite."""
    g = torch.Generator(device="cuda").manual_seed(C + HW)
    n = 4
    x = torch.randn((n, C, HW), generator=g, device="cuda", dtype=torch.float64)
    cg = C // groups
    x[0, 0, 0] = INF
    x[1, cg * 3 + 1, HW // 2] = -INF
    x[2, cg * 5, 0], x[2, cg * 5 + cg - 1, HW - 1] = INF, -INF
    x[3, C - 1, HW - 1] = NAN
    x = x.half().contiguous()
    w = (1 + 0.5 * torch.randn(C, generator=g, device="cuda")).half()
    b = (0.5 * torch.randn(C, generator=g, device="cuda")).half()
    y = ops.group_norm_tokens(x.view(n, C, HW, 1), (w, b, 1e-6, groups))
    torch.cuda.synchronize()
    bad = ~torch.isfinite(x.double().view(n, groups, cg * HW)).all(-1)           # [n, groups]
    want = torch.where(bad.repeat_interleave(cg, 1).view(n, 1, C).expand(n, HW, C),
                       torch.full((n, HW, C), NAN, dtype=torch.float64, device="cuda"),
                       torch.zeros((n, HW, C), dtype=torch.float64, device="cuda"))
    what = f"group_norm C={C} HW={HW} groups={groups}"
    _assert_class(y, want, f"{what} against float64")
    ref = F.group_norm(x.view(n, C, HW, 1), groups, w, b, 1e-6).view(n, C, HW).transpose(1, 2)
    _assert_class(y, ref, f"{what} against F.group_norm")


@pytest.mark.parametrize("num_inputs,inject", [(1, False), (3, False), (3, True), (2, True)])
def test_resnet_tail_non_finite(num_inputs, inject):
    """KT bit for bit against the torch tail it replaces, (shortcut + h') / output_scale_factor in fp16 on CUDA, with
    +-inf, NaN, +-65504 and subnormals in h and the shortcut (sums overflowing, inf - inf)."""
    g = torch.Generator(device="cuda").manual_seed(num_inputs + 10 * inject)
    n = 2
    B = num_inputs * n
    vals = _h([INF, -INF, NAN, 65504, -65504, 2 ** -24, -2 ** -24, 0, -0.0, 1, 32, -32, 65000])
    pick = lambda shape: vals[torch.randint(0, vals.numel(), shape, generator=g, device="cuda")]
    h = pick((n if inject else B, 3, 67))                 # 201 elements per sample: vector body and scalar tail
    sc = pick((B, 3, 67))
    for osf in (1.0, 2.0, 0.5):
        out = ops.resnet_tail(h, sc, num_inputs, osf, inject)
        torch.cuda.synchronize()
        hh = h.repeat(num_inputs, 1, 1) if inject else h
        want = (sc + hh) / osf
        _assert_bits(out, want.double(), f"resnet_tail num_inputs={num_inputs} inject={inject} osf={osf}")
