"""The row kernels (rows.cu, reduce.cu) against float64 references, per element.  Needs an H100.

- K0 (`vtm_normalize_split[_ln]`), KC (`vtm_gather_rows[_ln|_dev|_peers]`), KE (`vtm_unmerge_add`), `ops.layer_norm`
  (KC with an identity map) and KR (`vtm_merge_reduce`).  Every call but `ops.layer_norm` goes through the C-ABI, so
  that outputs can be guarded and strides chosen freely.
- Row widths: every C from 8 to 2048 in steps of 8.  rows.cu hands a row of C halfs to G lanes holding P 16-byte
  vectors each (`_band`: 8 x 5 up to C = 320, 16 x 5 up to 640, 32 x 5 up to 1280, 32 x 8 up to 2048), so this covers all
  four builds, the widths that fill a build exactly (320, 640, 1280, 2048: K0's FULL instantiations) and every ragged
  width.  The loops over C sit inside the test functions, and every failure names its C.
- Row counts: small ragged counts, and for every kernel two widths per build at `_multi_pass_rows` rows: three full
  grid-stride passes at the highest occupancy a 256-thread CTA can have, with a partly empty last row group.
- Every output lies between sentinel guard rows: before its first row, after its last, between samples where a batch
  stride leaves room, and in the capacity rows of device-count outputs.  The rows the kernel must write hold FILL (a NaN
  no kernel computes) before the call: an element left unwritten shows as FILL, a store outside them changes a sentinel.
"""
import ctypes
import math

import pytest
import torch

import vidtome_oracle as O
from vidtome_b200 import _lib, ops
from vidtome_b200._lib import VtmSplit

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A5A          # fp16 203.25: every guard row
FILL = 0x7D5A              # an fp16 NaN payload no kernel computes: every element an output must write, before the call
LEAD, TRAIL = 8, 24        # guard rows before and after every output
ALL_C = tuple(range(8, 2049, 8))
U = 2.0 ** -24             # unit roundoff of fp32


def _band(C):
    """(G, P) of the rows.cu build that a row of C halfs is dispatched to (VTM_DISPATCH_GP)."""
    v = C // 8
    return (8, 5) if v <= 40 else (16, 5) if v <= 80 else (32, 5) if v <= 160 else (32, 8)


def _multi_pass_rows(G):
    """Three grid-stride passes of 132 SMs x 8 resident 256-thread CTAs (the most 2048 threads per SM allow) x 8 warps
    x 32 / G rows per warp; the + 3 leaves the last row group of a warp partly empty."""
    return 3 * 132 * 8 * 8 * (32 // G) + 3


# two widths per build: a ragged one and the one that fills the build exactly
MULTI_PASS_C = (200, 320, 392, 640, 1000, 1280, 1640, 2048)


# ---------------------------------------------------------------------------------------------------------------------
# fp16 helpers in float64

def _ulp16(x):
    """Spacing of fp16 numbers in the binade of |x| (2^-24 in the subnormal range)."""
    _, e = torch.frexp(x.abs().clamp(min=2.0 ** -14))
    return torch.ldexp(torch.ones_like(x), e - 11)


def _round16(x):
    """float64 -> the nearest fp16 value (ties to even), rounded once; still float64."""
    assert x.abs().max().item() < 65520, "rounds beyond the fp16 range"
    u = _ulp16(x)
    return torch.round(x / u) * u


def _round16_inf(x):
    """_round16 with IEEE overflow: |x| >= 65520 rounds to +-inf."""
    r = _round16(x.clamp(-65504, 65504))
    return torch.where(x.abs() >= 65520, torch.copysign(torch.full_like(x, math.inf), x), r)


def _ordered(h):
    """fp16 tensor -> int32 that is monotonic in the value, one step per fp16 number (+0 and -0 both 0)."""
    b = h.view(torch.int16).int()
    return torch.where(b < 0, -(b & 0x7FFF), b)


def _from_bits(b):
    """int tensor of fp16 bit patterns in [0, 65535] -> fp16."""
    return torch.where(b >= 0x8000, b - 0x10000, b).to(torch.int16).view(torch.float16)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _mixed(shape, g):
    """Finite fp16 values over the whole range: random bit patterns (every binade equally likely, subnormals included),
    with 5 % set to +-0 and 10 % within a factor two of the largest fp16 number."""
    sign = torch.randint(0, 2, shape, generator=g, device="cuda") * 0x8000
    bits = torch.randint(0, 0x7C00, shape, generator=g, device="cuda")
    p = torch.rand(shape, generator=g, device="cuda")
    bits = torch.where(p < 0.05, 0, bits)
    bits = torch.where((p >= 0.05) & (p < 0.15), torch.randint(0x7800, 0x7C00, shape, generator=g, device="cuda"), bits)
    return _from_bits(bits | sign)


# ---------------------------------------------------------------------------------------------------------------------
# guarded outputs and C-ABI calls

def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


class _Out:
    """A guarded fp16 output of `rows` rows of C halfs.  Rows where `live` is set must be written (FILL before the call);
    the other rows, and LEAD rows before and TRAIL rows after, keep SENTINEL."""

    def __init__(self, rows, C, live=None):
        self.rows = rows
        self.live = torch.ones(rows, dtype=torch.bool, device="cuda") if live is None else live
        self.bits = torch.full((LEAD + rows + TRAIL, C), SENTINEL, dtype=torch.int16, device="cuda")
        self.bits[LEAD:LEAD + rows][self.live] = FILL

    @property
    def ptr(self):
        return self.bits[LEAD:].data_ptr()

    def out(self):
        return self.bits[LEAD:LEAD + self.rows].view(torch.float16)

    def check_guards(self, what):
        guard = torch.ones(LEAD + self.rows + TRAIL, dtype=torch.bool, device="cuda")
        guard[LEAD:LEAD + self.rows] = ~self.live
        bad = (self.bits != SENTINEL).any(1) & guard
        if bad.any():
            rows = (torch.nonzero(bad)[:4, 0] - LEAD).tolist()
            pytest.fail(f"{what}: store into guard row(s) {rows} (numbered from the output's first row)")


def _live(B, rows, stride):
    """Live mask of B samples of `rows` rows at a row stride of `stride` rows."""
    return (torch.arange(stride, device="cuda") < rows).repeat(B)


def _same(got, want):
    """Element-wise: bit-equal, or both NaN; never FILL."""
    g, w = got.view(torch.int16), want.view(torch.int16)
    return ((g == w) | (torch.isnan(got) & torch.isnan(want))) & (g != FILL)


def _assert_same(got, want, what):
    ok = _same(got, want)
    if not ok.all():
        i = tuple(torch.nonzero(~ok)[0].tolist())
        gb, wb = int(got.view(torch.int16)[i]) & 0xFFFF, int(want.view(torch.int16)[i]) & 0xFFFF
        pytest.fail(f"{what}: {int((~ok).sum())} of {ok.numel()} elements differ; first at {i}: got "
                    f"{got[i].item()!r} (0x{gb:04x}), want {want[i].item()!r} (0x{wb:04x})")


def _sync(rc, what):
    _lib.check(rc, what)
    torch.cuda.synchronize()


def _ln_args(ln):
    return (None, None, 0.0) if ln is None else (_ptr(ln[0]), _ptr(ln[1]), float(ln[2]))


def _k0(x, rowmap, map_bs, split, B, C, a, b, ln=None, what=""):
    lw, lb, eps = _ln_args(ln)
    _sync(_lib.load().vtm_normalize_split_ln(x.data_ptr(), x.stride(0), _ptr(rowmap), map_bs, ctypes.byref(split), B, C,
                                             lw, lb, eps, a.ptr, b.ptr, _stream()), f"K0 {what}")
    a.check_guards(f"K0 {what}: src rows")
    b.check_guards(f"K0 {what}: dst rows")


def _kc(x, map_ptr, map_bs, B, L, C, y, y_bs, ln=None, peers=(), what=""):
    lw, lb, eps = _ln_args(ln)
    arr = (ctypes.c_void_p * max(1, len(peers)))(*[p.ptr for p in peers])
    _sync(_lib.load().vtm_gather_rows_peers(x.data_ptr(), x.stride(0), map_ptr, map_bs, B, L, C, lw, lb, eps, y.ptr,
                                            y_bs, arr, len(peers), _stream()), f"KC {what}")
    y.check_guards(f"KC {what}")


def _gather(x, rows):
    """x [B, *, C], rows [B|1, L] (any integer type) -> x[b, rows[b, i]]."""
    B, _, C = x.shape
    idx = rows.long().expand(B, -1)
    return torch.gather(x, 1, idx[..., None].expand(-1, -1, C))


# ---------------------------------------------------------------------------------------------------------------------
# K0: torch's fp16 `x / x.norm()`, bit for bit

def _normalize_ref(x):
    """fp16(fp32(x) / fp32(n)), n = fp16(sqrtf(sum of fp32 x^2)): torch's fp16 `metric / metric.norm(dim=-1)`.  Every
    square of an fp16 value is exact in fp32; the sum is taken by torch in fp32, which is the kernel's sum whenever the
    sum is exact in any order (the rows of the tests below that use this).

    One deviation is pinned (DESIGN §1): where the norm is a normal fp16 number, K0's fast division turns a -0 entry
    into +0 (rem = (-0)(-n) + (-0) = +0); the reference keeps -0."""
    xf = x.float()
    n = (xf * xf).sum(-1, keepdim=True).sqrt().half()
    q = (xf / n.float()).half()
    fast = (n >= 2.0 ** -14) & (n <= 65504)
    return torch.where(fast & (x.view(torch.int16) == -0x8000), torch.zeros_like(q), q)


def test_k0_two_entry_rows():
    """Rows with two non-zero entries (x, y) at random columns, C = 8 ... 64: their fp32 sum of squares is RN(x^2 + y^2)
    in any order, so the output is fully determined.  x runs over every finite fp16 value, each with four y: zero (a
    single-entry row, +-1 exactly; the zero row gives NaN), a random finite value, a value of at most |x| (with a
    subnormal x: a subnormal norm, the plain-division path), and a value of at least 16384 (norms from the fast path's
    top up to sqrt >= 65520, where the fp16 norm is inf and every element must be x / inf = +-0)."""
    xs = _from_bits(torch.arange(0, 0x10000, device="cuda"))
    xs = xs[torch.isfinite(xs)]
    n = xs.numel()
    counts = {"overflowing": 0, "subnormal": 0, "zero": 0, "fast path": 0}
    for C in range(8, 65, 8):
        g = _gen(C)
        sign = torch.randint(0, 2, (n,), generator=g, device="cuda") * 0x8000
        ys = (torch.zeros_like(xs),
              _from_bits(torch.randint(0, 0x7C00, (n,), generator=g, device="cuda") | sign),
              (xs.double().abs() * torch.rand(n, generator=g, device="cuda", dtype=torch.float64)).half()
              * torch.where(sign > 0, -1.0, 1.0).half(),
              _from_bits(torch.randint(0x7400, 0x7C00, (n,), generator=g, device="cuda") | sign))
        x, y = xs.repeat(4), torch.cat(ys)
        R = x.numel()
        cols = torch.rand((R, C), generator=g, device="cuda").argsort(1)[:, :2]
        rows = torch.zeros((R, C), dtype=torch.float16, device="cuda")
        rows.scatter_(1, cols[:, :1], x[:, None])
        rows.scatter_(1, cols[:, 1:], y[:, None])
        Ns = R // 3
        a, b = _Out(Ns, C), _Out(R - Ns, C)
        _k0(rows.view(1, R, C), None, 0, VtmSplit.prefix(R, Ns), 1, C, a, b, what=f"two-entry rows C={C}")
        want = _normalize_ref(rows)
        _assert_same(a.out(), want[:Ns], f"two-entry rows C={C}, src rows")
        _assert_same(b.out(), want[Ns:], f"two-entry rows C={C}, dst rows")
        rf = rows.float()
        nrm = (rf * rf).sum(-1).sqrt().half().float()
        c = {"overflowing": torch.isinf(nrm), "subnormal": (nrm > 0) & (nrm < 2.0 ** -14), "zero": nrm == 0,
             "fast path": (nrm >= 2.0 ** -14) & (nrm <= 65504)}
        for k, m in c.items():
            assert m.any(), f"C={C}: no row with a {k} norm"
            counts[k] += int(m.sum())
    print("two-entry rows by norm: " + ", ".join(f"{k} {v}" for k, v in counts.items()))


def _exact_rows(shape, g):
    """k / 8 * 2^s with integers |k| <= 64 (a quarter of them 0) and one s in [-21, 9] per row.  Every square is a
    multiple of 2^(2s-6), and the sum of at most 2048 of them is below 2^23 such multiples: exact in fp32 in any order.
    s = -21 gives subnormal entries and norms, s = 9 norms past the fp16 range at the wider C."""
    k = torch.randint(-64, 65, shape, generator=g, device="cuda")
    k = torch.where(torch.rand(shape, generator=g, device="cuda") < 0.25, 0, k)
    s = torch.randint(-21, 10, shape[:-1] + (1,), generator=g, device="cuda")
    return (k.double() * torch.exp2(s.double() - 3)).half()


def _rowmap(kind, B, N, N0, g):
    """(map or None, batch stride, [B, N] rows of x it selects)."""
    if kind == "none":
        return None, 0, torch.arange(N, device="cuda").expand(B, N)
    if kind == "shared":
        m = torch.randperm(N0, generator=g, device="cuda")[:N].int().view(1, N)
        return m, 0, m.expand(B, N)
    m = torch.randint(0, N0, (B, N + 3), generator=g, device="cuda", dtype=torch.int32)
    return m, N + 3, m[:, :N]


def _check_k0(x, kind, split, a_idx, b_idx, g, what, N=None):
    """K0 with the split against `_normalize_ref` of the rows at positions a_idx / b_idx; returns the outputs."""
    B, N0, C = x.shape
    N = split.N if N is None else N
    a_idx = torch.as_tensor(a_idx, device="cuda").long()
    b_idx = torch.as_tensor(b_idx, device="cuda").long()
    Ns, Nd = a_idx.numel(), b_idx.numel()
    assert ops.split_counts(split) == (Ns, Nd), what
    rm, mbs, rows = _rowmap(kind, B, N, N0 - 2, g)
    a, b = _Out(B * Ns, C), _Out(B * Nd, C)
    _k0(x, rm, mbs, split, B, C, a, b, what=what)
    want = _normalize_ref(_gather(x, rows))
    _assert_same(a.out().view(B, Ns, C), want[:, a_idx], f"{what}: src rows")
    _assert_same(b.out().view(B, Nd, C), want[:, b_idx], f"{what}: dst rows")


def _check_k0_mode2(x, kind, L, gcap, lg, coin_high, g, what):
    """Mode 2 (local L rows | global lg <= gcap rows, the coin picks the src half): src / dst rows at the capacity's
    row stride, equal to the reference and to K0 with the prefix split it stands for; rows [Ns, cap) and [Nd, cap) of
    every sample keep their sentinel."""
    B, N0, C = x.shape
    N, cap = L + gcap, max(L, gcap)
    rm, mbs, rows = _rowmap(kind, B, N, N0 - 2, g)
    coin = torch.tensor([0.75 if coin_high else 0.25], dtype=torch.float32, device="cuda")
    glen = torch.tensor([lg], dtype=torch.int32, device="cuda")
    loc, glob = torch.arange(L, device="cuda"), torch.arange(L, L + lg, device="cuda")
    src, dst = (loc, glob) if coin_high else (glob, loc)
    Ns, Nd = src.numel(), dst.numel()
    a, b = _Out(B * cap, C, _live(B, Ns, cap)), _Out(B * cap, C, _live(B, Nd, cap))
    _k0(x, rm, mbs, VtmSplit.prefix_coin_dev(L, glen, gcap, coin, 0.5), B, C, a, b, what=what)
    ga, gb = a.out().view(B, cap, C)[:, :Ns], b.out().view(B, cap, C)[:, :Nd]
    want = _normalize_ref(_gather(x, rows))
    _assert_same(ga, want[:, src], f"{what}: src rows")
    _assert_same(gb, want[:, dst], f"{what}: dst rows")
    host_map = rows[:, torch.cat([src, dst])].contiguous().int()
    a2, b2 = _Out(B * Ns, C), _Out(B * Nd, C)
    _k0(x, host_map, Ns + Nd, VtmSplit.prefix(Ns + Nd, Ns), B, C, a2, b2, what=f"{what}, host split")
    _assert_same(ga, a2.out().view(B, Ns, C), f"{what}: src rows against the host split")
    _assert_same(gb, b2.out().view(B, Nd, C), f"{what}: dst rows against the host split")


# mode-0 splits: (F, target_stride, randf) over F = 1 ... 9 and 16, every stride up to 4 and every randf < stride
MODE0 = [(F, ts, rf) for F in (*range(1, 10), 16) for ts in range(1, 5) if ts <= F for rf in range(ts)]
ROWMAPS = ("none", "shared", "per_sample")


def test_k0_exact_rows_every_width_and_split():
    """Exact rows (`_exact_rows`) at every C, bit for bit, through each split form: mode 0 (cycling through MODE0 with
    and without carried tokens, tnum 1 ... 5, B = 1 ... 3), the prefix split, the coin split with both branches of the
    coin, and the device-count split (mode 2) with a global length below its capacity.  Each form runs without a row
    map, with one map shared by all samples and with per-sample maps at a batch stride wider than the map."""
    g = _gen(1)
    for i, C in enumerate(ALL_C):
        F, ts, rf = MODE0[i % len(MODE0)]
        unm_pre, tnum, B = (0, 3, 0, 11)[i % 4], 1 + i % 5, 1 + i % 3
        N = unm_pre + F * tnum
        x = _exact_rows((B, 2 * N + 20, C), g)
        a_idx, b_idx, _, _ = O.split_indices_randframe(N, F, unm_pre, ts, rf)
        _check_k0(x, ROWMAPS[i % 3], VtmSplit.local(N, unm_pre, F, ts, rf), a_idx, b_idx, g,
                  f"C={C} mode 0 N={N} unm_pre={unm_pre} F={F} stride={min(ts, F)} randf={rf} B={B} map={ROWMAPS[i % 3]}")
        src_len = (7 * i) % (N + 1)
        _check_k0(x, ROWMAPS[(i + 1) % 3], VtmSplit.prefix(N, src_len), range(src_len), range(src_len, N), g,
                  f"C={C} prefix N={N} src_len={src_len} B={B} map={ROWMAPS[(i + 1) % 3]}")
        L = 1 + i % 9
        coin_high = i % 2 == 0
        coin = torch.tensor([0.75 if coin_high else 0.25], dtype=torch.float32, device="cuda")
        halves = (range(L), range(L, 2 * L))
        src, dst = halves if coin_high else halves[::-1]
        _check_k0(x, ROWMAPS[(i + 2) % 3], VtmSplit.prefix_coin(L, coin, 0.5), src, dst, g,
                  f"C={C} prefix_coin L={L} coin {'>' if coin_high else '<='} threshold B={B} map={ROWMAPS[(i + 2) % 3]}")
        L2 = 2 + i % 6
        gcap = L2 + 1 + i % 4 if i % 2 else max(1, L2 - 1 - i % 3)
        lg = max(1, min(gcap, max(L2, gcap) - 1 - i % 2))
        _check_k0_mode2(x, ROWMAPS[i % 3], L2, gcap, lg, (i // 2) % 2 == 0, g,
                        f"C={C} mode 2 L={L2} glob_cap={gcap} glob_len={lg} coin {'>' if (i // 2) % 2 == 0 else '<='}"
                        f" threshold B={B} map={ROWMAPS[i % 3]}")


def _reduction_depth_squares(C):
    """Roundings on the way of one x^2 into K0's sum of squares: a chain of 2P fmas per lane accumulator, the sum of the
    two accumulators, the pair sum and log2(G) shuffle levels."""
    G, P = _band(C)
    return 2 * P + 2 + int(math.log2(G))


def _gamma(n):
    return n * U / (1 - n * U)


def test_k0_real_rows_take_one_norm_per_row():
    """Gaussian rows of every scale from subnormal to 2^7, at every C.  The kernel's fp32 sum of squares lies within
    gamma(D) ss of the exact ss (D roundings on any square's way, `_reduction_depth_squares`; all terms are positive), and
    sqrtf rounds once more, so its fp16 norm is one of the fp16 values between the roundings of the ends of that
    interval: one or two candidates.  Every element of a row must be the division by one and the same candidate."""
    second = rows_total = 0
    for C in ALL_C:
        g = _gen(10_000 + C)
        R = 37
        s = torch.randint(-22, 8, (R, 1), generator=g, device="cuda").double()
        x = (torch.randn((R, C), generator=g, device="cuda", dtype=torch.float64) * torch.exp2(s)).half()
        Ns = R // 2
        a, b = _Out(Ns, C), _Out(R - Ns, C)
        _k0(x.view(1, R, C), None, 0, VtmSplit.prefix(R, Ns), 1, C, a, b, what=f"real rows C={C}")
        got = torch.cat([a.out(), b.out()])
        ss = (x.double() ** 2).sum(-1)
        gam = _gamma(_reduction_depth_squares(C)) + 2.0 ** -48          # + the float64 sum's own error
        n_lo = _round16((ss * (1 - gam)).sqrt() * (1 - 2.0 ** -23))
        n_hi = _round16((ss * (1 + gam)).sqrt() * (1 + 2.0 ** -23))
        assert (_ordered(n_hi.half()) - _ordered(n_lo.half())).max().item() <= 1, f"C={C}: more than two candidates"
        xf = x.float()
        neg0 = x.view(torch.int16) == -0x8000                            # -0 -> +0 on the fast path (_normalize_ref)

        def divided(nc):
            q = (xf / nc.float()[:, None]).half()
            fast = ((nc >= 2.0 ** -14) & (nc <= 65504))[:, None]
            return torch.where(fast & neg0, torch.zeros_like(q), q)

        ok_lo = _same(got, divided(n_lo)).all(1)
        ok_hi = _same(got, divided(n_hi)).all(1)
        bad = ~(ok_lo | ok_hi)
        if bad.any():
            r = int(torch.nonzero(bad)[0])
            pytest.fail(f"real rows C={C}: row {r} is not the division by one candidate norm "
                        f"({n_lo[r].item()!r}, {n_hi[r].item()!r})")
        second += int((~ok_lo).sum())
        rows_total += R
    print(f"K0 real rows: {second} of {rows_total} rows took the larger candidate norm")


# ---------------------------------------------------------------------------------------------------------------------
# the fused LayerNorm against float64

def _ln_reference(x, w, b, eps):
    """Y = gamma (x - mu) / sqrt(var + eps) + beta in float64 for x [..., C] fp16, and a bound delta on |y32 - Y| for
    the kernel's fp32 result y32 (before its rounding to fp16), element by element.

    With u = 2^-24, gamma(n) = n u / (1 - n u), A = sum |x_i|, d_i = x_i - mu, and the kernel's steps (rows.cu,
    layer_norm_row; G lanes, P vectors per lane):
    - the sum S: every x_i passes at most D1 = P + 3 + log2 G roundings (pair sum, P accumulator adds, the accumulators'
      sum, the pair's sum, the shuffle levels), so |S~ - S| <= gamma(D1) A.  m~ = RN(S~ / C):
      e_m = gamma(D1) A / C + u (|mu| + gamma(D1) A / C).
    - d~_i = RN(x_i - m~): e_d = e_m + u (|d_i| + e_m).
    - Q~ = fp32 sum of d~_i^2, a chain of 2P fmas per accumulator then 2 + log2 G adds (D2 = 2P + 2 + log2 G):
      |Q~ - Q| <= sum (2 |d_i| e_d + e_d^2) + gamma(D2) sum (|d_i| + e_d)^2, Q = sum d_i^2.
    - v~ = RN(Q~ / C), w~ = RN(v~ + eps): e_v = e_Q / C + u (var + e_Q / C), e_w = e_v + u (W + e_v) with W = var + eps
      (eps as the fp32 value the kernel receives).
    - r~ = rsqrtf(w~), at most 2 ulp (2^-22 relative) from 1 / sqrt(w~), which is within R rho of R = 1 / sqrt(W) for
      rho = e_w / W <= 1/2: e_r = R rho + 2^-22 R (1 + rho).
    - t~ = RN(r~ d~): e_t = e_r (|d| + e_d) + R e_d + u (R + e_r)(|d| + e_d).
    - y32 = RN(gamma t~ + beta) (one fma): delta = |gamma| e_t + u (|Y| + |gamma| e_t).
    A 2^-40 |Y| + 2^-60 term covers the float64 reference's own error."""
    C = x.shape[-1]
    G, P = _band(C)
    lg = int(math.log2(G))
    g1, g2 = _gamma(P + 3 + lg), _gamma(2 * P + 2 + lg)
    eps32 = float(torch.tensor(eps, dtype=torch.float32))
    x64 = x.double()
    gm = w.double()
    bt = b.double() if b is not None else torch.zeros_like(gm)
    mu = x64.mean(-1, keepdim=True)
    d = x64 - mu
    var = (d * d).mean(-1, keepdim=True)
    W = var + eps32
    R = W.rsqrt()
    Y = gm * (d * R) + bt
    A = x64.abs().sum(-1, keepdim=True)
    e_m = g1 * A / C + U * (mu.abs() + g1 * A / C)
    e_d = e_m + U * (d.abs() + e_m)
    dmax = d.abs() + e_d
    e_q = (2 * d.abs() * e_d + e_d * e_d).sum(-1, keepdim=True) + g2 * (dmax * dmax).sum(-1, keepdim=True)
    e_v = e_q / C + U * (var + e_q / C)
    e_w = e_v + U * (W + e_v)
    rho = e_w / W
    assert rho.max().item() <= 0.5
    e_r = R * rho + 2.0 ** -22 * R * (1 + rho)
    e_t = e_r * dmax + R * e_d + U * (R + e_r) * dmax
    delta = gm.abs() * e_t + U * (Y.abs() + gm.abs() * e_t) + 2.0 ** -40 * Y.abs() + 2.0 ** -60
    return Y, delta


def _check_ln(y, x, ln, what):
    """y fp16 [..., C] = LayerNorm(x): within delta of Y (so equal to RN16(Y) wherever the delta interval holds no fp16
    rounding midpoint), within one ulp of RN16(Y) wherever delta <= ulp / 2, and beta exactly on constant rows (where
    d~ = 0 exactly, which the bound does not see).  Returns (elements != RN16(Y),
    elements whose interval holds a midpoint)."""
    w, b, eps = ln
    assert not (y.view(torch.int16) == FILL).any(), f"{what}: element left unwritten"
    const = (x == x[..., :1]).all(-1)
    if const.any():
        beta = (b.double() if b is not None else torch.zeros_like(w.double())).expand_as(y)
        assert torch.equal(y.double()[const], beta[const]), f"{what}: a constant row's output is not beta"
    # the bound does not see that d~ = 0 exactly on a constant row; those rows are checked exactly above
    x, y = x[~const], y[~const]
    Y, delta = _ln_reference(x, w, b, eps)
    want = _round16(Y)
    lo, hi = _round16(Y - delta), _round16(Y + delta)
    yd = y.double()
    bad = ~((yd >= lo) & (yd <= hi))
    if bad.any():
        i = tuple(torch.nonzero(bad)[0].tolist())
        pytest.fail(f"{what}: {int(bad.sum())} elements outside [RN16(Y - delta), RN16(Y + delta)]; first at {i}: "
                    f"y = {yd[i].item()!r}, Y = {Y[i].item()!r}, delta = {delta[i].item():.3e}")
    # one ulp follows from the bound where delta <= half an ulp; where it does not (a mean far larger than the spread,
    # whose fp32 rounding R amplifies), the bound above is the check
    tight = delta <= _ulp16(Y) / 2
    far = ((_ordered(y) - _ordered(want.half())).abs() > 1) & tight
    assert not far.any(), f"{what}: {int(far.sum())} elements more than one ulp from RN16(Y) with delta <= ulp / 2"
    return int((yd != want).sum()), int((lo != hi).sum())


def _ln_rows(C, n, g):
    """n rows of each kind: Gaussian at scales 2^-3 ... 2^4 with an offset, constant rows (0, +-1.5, +-60000, 2^-20),
    mean 1000 with spread 0.1, subnormal-valued rows (var << eps), rows near +-60000, and rows alternating +-60000."""
    def randn(k):
        return torch.randn((k, C), generator=g, device="cuda", dtype=torch.float64)

    s = torch.randint(-3, 5, (n, 1), generator=g, device="cuda").double()
    consts = torch.tensor([0.0, 1.5, -1.5, 60000.0, -60000.0, 2.0 ** -20], device="cuda", dtype=torch.float64)
    c = consts[torch.randint(0, consts.numel(), (n, 1), generator=g, device="cuda")].expand(n, C)
    alt = torch.where(torch.arange(C, device="cuda") % 2 == 0, 60000.0, -60000.0).double().expand(n, C)
    sign = torch.where(torch.rand((n, 1), generator=g, device="cuda") < 0.5, -1.0, 1.0).double()
    kinds = (randn(n) * torch.exp2(s) + randn(1)[:, :1], c, 1000 + 0.1 * randn(n), randn(n) * 2.0 ** -20,
             sign * 60000 + 30 * randn(n), alt)
    return torch.cat(kinds).half()


def _ln_params(C, g, bias):
    w = 1 + 0.5 * torch.randn(C, generator=g, device="cuda")
    w = torch.where(torch.rand(C, generator=g, device="cuda") < 0.1, 0.0, w).half()
    b = (0.5 * torch.randn(C, generator=g, device="cuda")).half() if bias else None
    return w, b, 1e-5


def _run_kc_ln(x, ln, B, L, g, what):
    """KC + LN with a per-sample map and a gap of 2 rows between samples; returns (y [B, L, C], the rows it read)."""
    _, N0, C = x.shape
    m = torch.randint(0, N0, (B, L), generator=g, device="cuda", dtype=torch.int32)
    gap = 2
    y = _Out(B * (L + gap), C, _live(B, L, L + gap))
    _kc(x, m.data_ptr(), L, B, L, C, y, (L + gap) * C, ln=ln, what=what)
    return y.out().view(B, L + gap, C)[:, :L], _gather(x, m)


# Elements of the 12 632 064 KC + LN outputs of test_layer_norm_against_float64 that are not RN16(Y) (all inside the
# delta interval; 4 081 732 intervals hold a rounding midpoint), measured on an H100.  Most come from the rows whose mean
# is far larger than their spread.  A change to the kernel's arithmetic must not raise it.
LN_NOT_RN16 = 2_093_621


def test_layer_norm_against_float64():
    """KC + LN at every C, with ln_bias and with ln_bias = NULL, against `_ln_reference`; ops.layer_norm (KC with an
    identity map) equal to it bit for bit."""
    not_rn = near = total = 0
    for i, C in enumerate(ALL_C):
        for bias in (True, False):
            g = _gen(20_000 + 2 * C + bias)
            ln = _ln_params(C, g, bias)
            rows = _ln_rows(C, 3, g)
            B = 2
            x = rows[torch.randperm(rows.shape[0], generator=g, device="cuda")].view(B, -1, C)
            L = x.shape[1] + 3
            what = f"KC + LN C={C} bias={bias}"
            y, seq = _run_kc_ln(x, ln, B, L, g, what)
            a, b = _check_ln(y, seq, ln, what)
            not_rn, near, total = not_rn + a, near + b, total + y.numel()
            _assert_same(ops.layer_norm(seq.reshape(-1, C), ln).view(B, L, C), y, f"ops.layer_norm C={C} bias={bias}")
    print(f"KC + LN: {not_rn} of {total} elements not RN16(Y); {near} with a rounding midpoint within delta")
    assert not_rn <= LN_NOT_RN16 + 100, f"{not_rn} elements not RN16(Y), pinned at {LN_NOT_RN16}"


def test_layer_norm_paths_agree():
    """All LayerNorm instantiations share layer_norm_row: K0 + LN (x) == K0 (KC + LN (x)) bit for bit at every C, and
    ops.layer_norm == KC + LN."""
    for i, C in enumerate(ALL_C):
        g = _gen(30_000 + C)
        ln = _ln_params(C, g, i % 2 == 0)
        B = 2
        x = _ln_rows(C, 2, g).view(B, -1, C)
        N = x.shape[1]
        Ns = (5 * i) % (N + 1)
        sp = VtmSplit.prefix(N, Ns)
        a1, b1 = _Out(B * Ns, C), _Out(B * (N - Ns), C)
        _k0(x, None, 0, sp, B, C, a1, b1, ln=ln, what=f"K0 + LN C={C}")
        y = _Out(B * N, C)
        _kc(x, None, 0, B, N, C, y, N * C, ln=ln, what=f"KC + LN identity map C={C}")
        yv = y.out().view(B, N, C)
        a2, b2 = _Out(B * Ns, C), _Out(B * (N - Ns), C)
        _k0(yv, None, 0, sp, B, C, a2, b2, what=f"K0 of KC + LN C={C}")
        _assert_same(a1.out(), a2.out(), f"K0 + LN against K0(KC + LN) C={C}: src rows")
        _assert_same(b1.out(), b2.out(), f"K0 + LN against K0(KC + LN) C={C}: dst rows")
        _assert_same(ops.layer_norm(x.reshape(-1, C), ln), yv.reshape(-1, C), f"ops.layer_norm against KC + LN C={C}")


# ---------------------------------------------------------------------------------------------------------------------
# KC, KE and their variants, bit for bit

def _map(kind, B, L, N0, g):
    """(pointer, batch stride, [B|1, L] rows) of a row map: one shared map, per-sample maps at a stride of L + 5, or a
    column slice of a wider map."""
    if kind == "shared":
        m = torch.randint(0, N0, (1, L), generator=g, device="cuda", dtype=torch.int32)
        return m, (m.data_ptr() if L else None), 0, m
    full = torch.randint(0, N0, (B, L + 5), generator=g, device="cuda", dtype=torch.int32)
    off = 2 if kind == "slice" else 0
    return full, full.data_ptr() + 4 * off, L + 5, full[:, off:off + L]


def _run_kc(C, B, L, N0, kind, gap, g, n_peers=0, ln=None, what=""):
    """KC (or KC + LN) into [B, L + gap, C] with peers; plain KC must equal the gathered rows, each peer the output."""
    x = _mixed((B, N0 + 1, C), g)
    keep, mp, mbs, rows = _map(kind, B, L, N0, g)
    y = _Out(B * (L + gap), C, _live(B, L, L + gap))
    peers = [_Out(B * (L + gap), C, _live(B, L, L + gap)) for _ in range(n_peers)]
    _kc(x, mp, mbs, B, L, C, y, (L + gap) * C, ln=ln, peers=peers, what=what)
    got = y.out().view(B, L + gap, C)[:, :L]
    if ln is None:
        _assert_same(got, _gather(x, rows), what)
    for k, p in enumerate(peers):
        if not torch.equal(p.bits, y.bits):
            pytest.fail(f"{what}: peer buffer {k} of {n_peers} differs from the local output or its guards")
    del keep
    return got


def _run_kc_dev(C, B, Lcap, length, kind, g, what):
    """vtm_gather_rows_dev: rows below *len gathered, rows [len, L_cap) +0."""
    N0 = Lcap + 7
    x = _mixed((B, N0 + 1, C), g)
    keep, mp, mbs, rows = _map(kind, B, Lcap, N0, g)
    gap = 3
    y = _Out(B * (Lcap + gap), C, _live(B, Lcap, Lcap + gap))
    ln_dev = torch.tensor([length], dtype=torch.int32, device="cuda")
    _sync(_lib.load().vtm_gather_rows_dev(x.data_ptr(), x.stride(0), mp, mbs, B, Lcap, C, ln_dev.data_ptr(), y.ptr,
                                          (Lcap + gap) * C, _stream()), f"KC dev {what}")
    y.check_guards(f"KC dev {what}")
    got = y.out().view(B, Lcap + gap, C)[:, :Lcap]
    _assert_same(got[:, :length], _gather(x, rows)[:, :length], f"KC dev {what}: gathered rows")
    assert (got[:, length:].view(torch.int16) == 0).all(), f"KC dev {what}: rows past the length are not +0"
    del keep


def _sum16(a, b):
    """RN16(a + b) for fp16 a, b, rounded once (the float64 sum is exact), IEEE zero signs and overflow to +-inf."""
    return _round16_inf(a.double() + b.double()).half()


def _run_ke(C, B, L, N, kind, resid, g, what):
    """vtm_unmerge_add with y at a batch stride of L + 3 rows: out = RN16(y[map] + resid), or the plain gather.  The
    residual cancels a tenth of the gathered elements exactly (+0, or -0 where both are -0) and overflows where both
    are large."""
    y = _mixed((B, L + 3, C), g)
    keep, mp, mbs, rows = _map(kind, B, N, L, g)
    gath = _gather(y, rows)
    r = None
    if resid:
        r = _mixed((B, N, C), g)
        neg = torch.rand((B, N, C), generator=g, device="cuda") < 0.1
        r = torch.where(neg, -gath, r).contiguous()
    out = _Out(B * N, C)
    _sync(_lib.load().vtm_unmerge_add(y.data_ptr(), y.stride(0), mp, mbs, _ptr(r), B, N, C, out.ptr, _stream()),
          f"KE {what}")
    out.check_guards(f"KE {what}")
    want = gath if r is None else _sum16(gath, r)
    _assert_same(out.out().view(B, N, C), want, f"KE {what}")
    del keep
    return want


def test_kc_every_width():
    """KC at every C: B = 1 ... 3, shared and per-sample maps, L = 0, and a gap of guard rows between samples (as
    patch.py writes into cat[:, :L]); the peer stores with 1 ... 8 local buffers standing in for peers, with and
    without the fused LayerNorm; vtm_gather_rows_dev with len in {0, 1, L_cap - 1, L_cap}."""
    for i, C in enumerate(ALL_C):
        g = _gen(40_000 + C)
        B = 1 + i % 3
        kind = ("shared", "per_sample")[i % 2]
        L = (0, 1, 2, 3, 31, 33, 70)[i % 7]
        _run_kc(C, B, L, L + 9, kind, 1 + i % 3, g, what=f"C={C} B={B} L={L} map={kind}")
        n_peers = 1 + i % 8
        ln = _ln_params(C, g, i % 4 == 1) if i % 2 else None
        got = _run_kc(C, 2, 33, 40, kind, 2, g, n_peers=n_peers, ln=ln,
                      what=f"C={C} peers={n_peers} LN={ln is not None}")
        assert not (got.view(torch.int16) == FILL).any()
        Lcap = (1, 2, 5, 33)[i % 4]
        for length in sorted({0, 1, Lcap - 1, Lcap}):
            _run_kc_dev(C, B, Lcap, length, kind, g, f"C={C} B={B} L_cap={Lcap} len={length} map={kind}")


def test_ke_every_width():
    """KE at every C, with and without the residual: per-sample maps, a column slice of a wider map (row stride > N),
    a shared map; y at a batch stride above L C; sums overflowing to +-inf and cancelling to +-0."""
    inf = zeros = 0
    for i, C in enumerate(ALL_C):
        g = _gen(50_000 + C)
        B = 1 + i % 3
        L, N = (1, 3, 31, 33)[i % 4], (1, 2, 33, 65)[(i // 4) % 4]
        for resid in (True, False):
            kind = ("per_sample", "slice", "shared")[(i + resid) % 3]
            want = _run_ke(C, B, L, N, kind, resid, g, f"C={C} B={B} L={L} N={N} map={kind} resid={resid}")
            if resid:
                inf += int(torch.isinf(want).sum())
                zeros += int((want == 0).sum())
    assert inf > 0 and zeros > 0
    print(f"KE: {inf} sums overflowed, {zeros} were zero")


# ---------------------------------------------------------------------------------------------------------------------
# three grid-stride passes per build

@pytest.mark.parametrize("C", MULTI_PASS_C)
def test_multi_pass(C):
    """Every row kernel at _multi_pass_rows rows of width C: K0 (exact rows, bit for bit; plain, fused LayerNorm against
    K0 of KC + LN, mode 2), KC, KC + LN (against float64), its peer stores, vtm_gather_rows_dev, KE with and without
    the residual, and ops.layer_norm."""
    G, _ = _band(C)
    R = _multi_pass_rows(G)
    g = _gen(60_000 + C)
    B = 3
    N = -(-R // B)
    x = _exact_rows((B, N + 2, C), g)
    _check_k0(x, "per_sample", VtmSplit.prefix(N, N // 3), range(N // 3), range(N // 3, N), g,
              f"multi-pass C={C} prefix")
    F = 4
    unm = N - F * (N // F)
    a_idx, b_idx, _, _ = O.split_indices_randframe(N, F, unm, 4, 2)
    _check_k0(x, "shared", VtmSplit.local(N, unm, F, 4, 2), a_idx, b_idx, g, f"multi-pass C={C} mode 0")
    L2 = N // 2
    _check_k0_mode2(x, "none", L2, N - L2, N - L2 - 1, True, g, f"multi-pass C={C} mode 2")

    ln = _ln_params(C, g, True)
    xl = _ln_rows(C, -(-R // 6), g)[:B * N].view(B, N, C)
    sp = VtmSplit.prefix(N, N // 2)
    a1, b1 = _Out(B * (N // 2), C), _Out(B * (N - N // 2), C)
    _k0(xl, None, 0, sp, B, C, a1, b1, ln=ln, what=f"multi-pass K0 + LN C={C}")
    y, seq = _run_kc_ln(xl, ln, B, N, g, f"multi-pass KC + LN C={C}")
    n_not, n_near = _check_ln(y, seq, ln, f"multi-pass KC + LN C={C}")
    print(f"multi-pass C={C}: KC + LN {n_not} elements not RN16(Y), {n_near} near a midpoint")
    _assert_same(ops.layer_norm(seq.reshape(-1, C), ln).view(B, N, C), y, f"multi-pass ops.layer_norm C={C}")
    yi = _Out(B * N, C)
    _kc(xl, None, 0, B, N, C, yi, N * C, ln=ln, what=f"multi-pass KC + LN identity C={C}")
    a2, b2 = _Out(B * (N // 2), C), _Out(B * (N - N // 2), C)
    _k0(yi.out().view(B, N, C), None, 0, sp, B, C, a2, b2, what=f"multi-pass K0 of KC + LN C={C}")
    _assert_same(a1.out(), a2.out(), f"multi-pass K0 + LN C={C}: src rows")
    _assert_same(b1.out(), b2.out(), f"multi-pass K0 + LN C={C}: dst rows")

    _run_kc(C, B, N, N + 5, "per_sample", 1, g, n_peers=2, what=f"multi-pass KC C={C}")
    _run_kc_dev(C, B, N, N - 1, "shared", g, f"multi-pass C={C}")
    _run_ke(C, B, N // 2, N, "slice", True, g, f"multi-pass C={C} resid")
    _run_ke(C, B, N // 2, N, "shared", False, g, f"multi-pass C={C} plain")


# ---------------------------------------------------------------------------------------------------------------------
# KR: the reduction merge modes against exact sums

MODES = {"mean": 1, "sum": 2, "amax": 3, "amin": 4}


def _run_kr(C, B, Bp, split, a_idx, b_idx, r, mode, g, what, one_dst=False):
    """vtm_merge_reduce with a synthetic match: a random edge order per bp and random dst rows (all dst 0 with
    one_dst), packed as KA and KB1 pack them.  Returns the dst part of the output.

    With fp16 values (multiples of 2^-24 below 2^16) any sum of fewer than 2^13 of them is exact in float64."""
    a_idx = torch.as_tensor(a_idx, device="cuda").long()
    b_idx = torch.as_tensor(b_idx, device="cuda").long()
    Ns, Nd = a_idx.numel(), b_idx.numel()
    x = _mixed((B, split.N, C), g)
    x = torch.where(torch.rand((B, split.N, C), generator=g, device="cuda") < 0.3, -x, x)   # more cancellation
    edge = torch.stack([torch.randperm(Ns, generator=g, device="cuda") for _ in range(Bp)]).int()
    j = torch.zeros((Bp, Ns), dtype=torch.int64, device="cuda") if one_dst else \
        torch.randint(0, Nd, (Bp, Ns), generator=g, device="cuda")
    arg = j + (Nd * torch.randint(0, B, (Bp, Ns), generator=g, device="cuda") if Bp == 1 else 0)
    keys = (0xFFFFFFFF - arg).contiguous()
    Lout = Ns - r + Nd
    lib = _lib.load()
    ws_bytes = lib.vtm_merge_reduce_workspace_bytes(B, Nd, C)
    ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device="cuda")
    y = _Out(B * Lout, C)
    _sync(lib.vtm_merge_reduce(x.data_ptr(), x.stride(0), ctypes.byref(split), r, Bp, keys.data_ptr(), edge.data_ptr(),
                               B, C, MODES[mode], y.ptr, ws.data_ptr(), ws_bytes, _stream()), f"KR {what}")
    y.check_guards(f"KR {what}")
    got = y.out().view(B, Lout, C)
    eb = edge.long().expand(B, Ns)
    src = _gather(x, a_idx[None])                             # [B, Ns, C] src rows
    _assert_same(got[:, :Ns - r], _gather(src, eb[:, r:]), f"KR {what}: unmerged rows")
    dst = _gather(x, b_idx[None]).double()
    merged = _gather(src, eb[:, :r]).double()
    to = j.expand(B, Ns).gather(1, eb[:, :r])[..., None].expand(-1, -1, C)
    if mode in ("sum", "mean"):
        acc = dst.scatter_add(1, to, merged)
        cnt = torch.ones((B, Nd), dtype=torch.float64, device="cuda").scatter_add(
            1, to[..., 0], torch.ones(to.shape[:2], dtype=torch.float64, device="cuda"))
        want = _round16_inf(acc).half() if mode == "sum" else (acc.float() / cnt.float()[..., None]).half()
        zero = acc == 0
    else:
        want = dst.scatter_reduce(1, to, merged, reduce=mode, include_self=True).half()
        zero = want == 0
    dst_got = got[:, Ns - r:]
    # an exactly zero result is +0 (DESIGN §1), whatever its inputs' signs; a tiny mean keeps the sign it rounds with
    want = torch.where(zero, torch.zeros_like(want), want)
    _assert_same(dst_got, want, f"KR {what}: dst rows")
    return dst_got


KR_C = (8, 56, 320, 392, 640, 1000, 1280, 1288, 2048)


@pytest.mark.parametrize("mode", tuple(MODES))
def test_merge_reduce(mode):
    """Every mode at widths across all row builds: mode-0 and prefix splits, r = 0, r = Ns and in between, Bp = 1 (arg
    = b Nd + j, reduced mod Nd) and Bp = B; one dst row receiving 3000 src rows; and a case whose final pass is a
    grid-stride loop of several passes.  sum = RN16(exact) (overflow to +-inf), mean = RN16(RN32(RN32(exact) / count)),
    amax / amin the exact extremes; every zero result +0."""
    inf = 0
    for i, C in enumerate(KR_C):
        g = _gen(70_000 + 10 * C + MODES[mode])
        B = 1 + i % 3
        Bp = 1 if i % 2 else B
        if i % 3:
            F, ts, rf = MODE0[(7 * i) % len(MODE0)]
            unm_pre, tnum = (0, 5)[i % 2], 3 + i % 4
            N = unm_pre + F * tnum
            a_idx, b_idx, _, _ = O.split_indices_randframe(N, F, unm_pre, ts, rf)
            sp = VtmSplit.local(N, unm_pre, F, ts, rf)
        else:
            N = 40 + i
            a_idx, b_idx = range(N // 2), range(N // 2, N)
            sp = VtmSplit.prefix(N, N // 2)
        Ns = len(a_idx)
        if len(b_idx) == 0:
            continue
        for r in sorted({0, Ns // 2, Ns}):
            out = _run_kr(C, B, Bp, sp, a_idx, b_idx, r, mode, g, f"{mode} C={C} B={B} Bp={Bp} N={N} Ns={Ns} r={r}")
            inf += int(torch.isinf(out).sum())
    g = _gen(71_000 + MODES[mode])
    out = _run_kr(72, 2, 1, VtmSplit.prefix(3100, 3000), range(3000), range(3000, 3100), 3000, mode, g,
                  f"{mode} 3000 src rows into dst row 0", one_dst=True)
    inf += int(torch.isinf(out).sum())
    _run_kr(640, 2, 2, VtmSplit.prefix(8000, 4000), range(4000), range(4000, 8000), 2500, mode, g,
            f"{mode} B=2 Nd=4000 C=640")
    if mode == "sum":
        assert inf > 0, "no sum overflowed"
