"""The matching stage against exact and float64 references: KA (`vtm_sim_argmax[_dev|_simt]`), KB1 (`vtm_topr_sort
[_dev]`), KB2 (`vtm_compose_maps[_dev]`), `vtm_decode_match` and `vtm_split_counts_dev`.  Needs an H100.

- Every call goes through the C-ABI with its outputs between sentinel guard words.
- KA on rounding-exact inputs (`test_match_core_cpu.exact_case`): every score is an integer times a power of two whose
  fp32 accumulation is exact in any order, while its rounding to fp16 decides the row: midpoints, one unit beside them,
  several exact scores rounding to the row maximum, zero, subnormal, 2^-14, 65504 / 65520.  Keys are compared bit for
  bit with RN16-then-first-index computed in float64, at every C from 8 to 1280 and beyond, with the ties placed in the
  same lane, across lanes of a quad, 64-column groups, tiles, work items, samples and the partial last tile.
- KA on real-valued unit rows against float64 scores with a derived bound on the tensor core's error.
- The planners and builders these tests rely on are checked without a GPU in `test_match_core_cpu.py`.
"""
import ctypes

import numpy as np
import pytest
import torch

import vidtome_oracle as O
from test_match_core_cpu import (BN, ORDER_SHAPE, Q_EXP, SMS, SORT_CASES, SPLIT_RATIOS, exact_case, exact_operands,
                                 ka_width_cases, pack_keys, rn16, row_keys, sort_fused)
from vidtome_b200 import _lib
from vidtome_b200._lib import VtmSplit

pytestmark = pytest.mark.gpu

SENT64 = 0x5A5A5A5A5A5A5A5A     # guard words of every uint64 output
SENT32 = 0x5A5A5A5A             # guard words (and unwritten entries) of every int32 output
LEAD, TRAIL = 8, 24


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _sync(rc, what):
    _lib.check(rc, what)
    torch.cuda.synchronize()


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


class _Guarded:
    """A flat int64 / int32 device buffer of n entries between LEAD and TRAIL sentinel entries."""

    def __init__(self, n, dtype=torch.int64, fill=None):
        s = SENT64 if dtype == torch.int64 else SENT32
        self.n, self.s = n, s
        self.t = torch.full((LEAD + n + TRAIL,), s, dtype=dtype, device="cuda")
        if fill is not None:
            self.t[LEAD:LEAD + n] = fill

    @property
    def ptr(self):
        return self.t[LEAD:].data_ptr()

    def out(self):
        return self.t[LEAD:LEAD + self.n]

    def check(self, what):
        g = torch.cat([self.t[:LEAD], self.t[LEAD + self.n:]])
        if (g != self.s).any():
            pytest.fail(f"{what}: store into a guard word")


def _u64(t):
    return t.cpu().numpy().view(np.uint64)


def _ka(a, b, B, Ns, Nd, C, align, fn="vtm_sim_argmax", counts=None, ld=None):
    """Keys [B', ld] of KA (or its twin), guarded; ld = Ns unless capacity is given."""
    ld = Ns if ld is None else ld
    Bp = 1 if align else B
    k = _Guarded(Bp * ld)
    lib = _lib.load()
    what = f"{fn} B={B} Ns={Ns} Nd={Nd} C={C} align={align}"
    if counts is None:
        rc = getattr(lib, fn)(a.data_ptr(), b.data_ptr(), B, Ns, Nd, C, int(align), k.ptr, _stream())
    else:
        rc = lib.vtm_sim_argmax_dev(a.data_ptr(), b.data_ptr(), B, Ns, Nd, C, int(align), counts.data_ptr(), k.ptr,
                                    _stream())
    _sync(rc, what)
    k.check(what)
    return _u64(k.out()).reshape(Bp, ld)


def _assert_keys(got, want, what):
    bad = got != want
    if bad.any():
        b, i = (int(v) for v in np.argwhere(bad)[0])
        lib = _lib.load()

        def show(k):
            k = int(k)
            return "none" if k == 0 else f"(0x{lib.vtm_key_score_half_bits(k):04x}, arg {lib.vtm_key_arg(k)})"
        pytest.fail(f"{what}: {int(bad.sum())} of {bad.size} keys differ; first at sample {b} row {i}: got "
                    f"{show(got[b, i])}, want {show(want[b, i])}")


# ---------------------------------------------------------------------------------------------------------------------
# 1 + 2. KA on rounding-exact inputs, at every width and shape

def test_ka_exact_every_width():
    """Every C from 8 to 1280 in steps of 8, and 1288 ... 2048, each with one shape of the cycle in
    `test_match_core_cpu.KA_SHAPES` (all eight resident (k_chunks, stages), streaming, every K tail, every dst split form,
    more items than CTAs, every Nd mod 8 in a partial last tile): KA's keys equal the exact reference bit for bit, and
    the SIMT twin's keys equal them too."""
    assert torch.cuda.get_device_properties(0).multi_processor_count == SMS
    for i, (C, B, Ns, Nd, align) in enumerate(ka_width_cases()):
        what = f"C={C} B={B} Ns={Ns} Nd={Nd} align={align}"
        a, b, want, _, _ = exact_case(C, B, Ns, Nd, align, 5000 + i)
        a, b = _dev(a), _dev(b)
        _assert_keys(_ka(a, b, B, Ns, Nd, C, align), want, f"KA {what}")
        if B * Ns * Nd * C <= 4e9:
            _assert_keys(_ka(a, b, B, Ns, Nd, C, align, fn="vtm_sim_argmax_simt"), want, f"SIMT twin {what}")


def _order_design(rng, G, Nd):
    """Per group: the row maximum sits both in sample 1's first dst range (column Nd + j1) and in sample 0's second
    (column j0 in [256, Nd)), so the later item on the same CTA must tie what the earlier one published.  Kinds: +0
    (with -0 roundings around it), -65504 (everything else -inf), and an ordinary value reached by a larger exact
    score at j0.  j0 sits on lane 0 of its quad for half of the groups."""
    X = np.empty((1, G, 2 * Nd))
    e = np.empty((1, G), dtype=np.int64)
    for g in range(G):
        kind = g % 3
        j1 = int(rng.integers(0, BN))
        j0 = BN + int(rng.integers(0, Nd - BN))
        if g % 2:
            j0 -= j0 % 8
        if kind == 0:                       # +0 at e = 32: |X| <= 128 rounds to zero
            e[0, g] = Q_EXP + 24
            X[0, g] = -rng.integers(300, 2 ** 20, size=2 * Nd)
            X[0, g, Nd + j1] = 0
            X[0, g, j0] = -int(rng.integers(0, 129))
        elif kind == 1:                     # -65504 at e = 5; -65520 and below round to -inf
            e[0, g] = 5
            X[0, g] = -rng.integers(2096640, 2098176, size=2 * Nd)
            X[0, g, Nd + j1] = -2047 * 1024
            X[0, g, j0] = -2047 * 1024 + int(rng.integers(-511, 512))
        else:
            e[0, g] = 20
            X[0, g] = rng.integers(-2 ** 20, 2 ** 19, size=2 * Nd)
            X[0, g, Nd + j1] = 1536 * 1024 - 500
            X[0, g, j0] = 1536 * 1024 + 500
    return X, e


def test_ka_threshold_decides_across_items():
    """`RowBest::begin` turns the published maximum into the entry threshold of a later work item: +0 must step to the
    fp16 value below -0, and -65504 must leave room for -65504.  In this shape (align_batch, 132 src blocks, two dst
    ranges per sample) every CTA runs sample 1's first range before sample 0's second, which holds the smaller arg."""
    s = ORDER_SHAPE
    B, Ns, Nd, C = s["B"], s["Ns"], s["Nd"], s["C"]
    rng = np.random.default_rng(77)
    X, e = _order_design(rng, C // 2, Nd)
    a, b = exact_operands(X, e, B, Ns, Nd, C, True, rng)
    h = rn16(X * np.exp2(-e.astype(np.float64))[..., None])
    want = row_keys(h)[:, np.arange(Ns) % (C // 2)]
    args = np.uint64(0xFFFFFFFF) - (want & np.uint64(0xFFFFFFFF))
    assert (want != 0).all() and (args < Nd).all(), "every row's first maximum lies in sample 0"
    _assert_keys(_ka(_dev(a), _dev(b), B, Ns, Nd, C, True), want, "threshold order")


# ---------------------------------------------------------------------------------------------------------------------
# 3. KA on real-valued rows against float64

def _unit_rows(shape, kind, g):
    x = torch.randn(shape, generator=g, device="cuda", dtype=torch.float64)
    if kind == "video":
        x = torch.randn((shape[0], 1, shape[2]), generator=g, device="cuda", dtype=torch.float64) + 0.1 * x
    return (x / x.norm(dim=-1, keepdim=True)).half()


def _round16(x):
    """float64 tensor -> nearest fp16 value (ties to even) as float64; +-inf beyond +-65520."""
    _, ex = torch.frexp(x.abs().clamp(min=2.0 ** -14))
    u = torch.ldexp(torch.ones_like(x), ex - 11)
    r = torch.round(x / u) * u
    return torch.where(x.abs() >= 65520, torch.copysign(torch.full_like(x, float("inf")), x), r)


def _bound(a, b, align):
    """Exact scores s and the bound E on the kernel's fp32 accumulation error, [B', Ns, Nd'] in float64.

    The products a_ik b_jk of fp16 values are exact.  wgmma adds one 16-wide k-step at a time into the fp32
    accumulator; model each step as an aligned sum truncated to fp32 precision relative to the largest magnitude
    involved, which is at most sum_k |a_ik b_jk| (the accumulator never exceeds the sum of the magnitudes so far).
    Truncation loses less than 2^-23 of that magnitude, and a step may align to an operand twice as large as its
    result, so each of the ceil(C / 16) steps errs by less than 2^-22 sum_k |a_ik b_jk|:
        E_ij = ceil(C / 16) 2^-22 sum_k |a_ik b_jk|,
    plus 2^-45 of the same sum for the float64 reference's own rounding."""
    C = a.shape[-1]
    a64, b64 = a.double(), b.double()
    s = a64 @ b64.transpose(1, 2)
    m = a64.abs() @ b64.abs().transpose(1, 2)
    if align:
        s, m = torch.cat(list(s), -1)[None], torch.cat(list(m), -1)[None]
    return s, (-(-C // 16) * 2.0 ** -22 + 2.0 ** -45) * m


def _check_real(keys, s, E, what):
    """(a)-(d) of every row for kernel keys (M, j*); returns the number of rows the bound leaves undecided."""
    k = torch.from_numpy(keys.view(np.int64)).cuda()
    assert (k != 0).all(), f"{what}: a row published nothing"
    M = torch.from_numpy((keys >> np.uint64(32)).astype(np.int64)).cuda()
    hb = torch.where(M >= 0x8000, M & 0x7FFF, M ^ 0xFFFF).to(torch.int16).view(torch.float16).double()
    jst = torch.from_numpy((0xFFFFFFFF - (keys & np.uint64(0xFFFFFFFF))).astype(np.int64)).cuda()
    lo, hi = _round16(s - E), _round16(s + E)
    cols = torch.arange(s.shape[-1], device="cuda")
    lo_j, hi_j = lo.gather(-1, jst[..., None])[..., 0], hi.gather(-1, jst[..., None])[..., 0]
    checks = {
        "(a) M outside [RN16(s_j* - E), RN16(s_j* + E)]": (lo_j <= hb) & (hb <= hi_j),
        "(b) some RN16(s_j - E_j) above M": (lo <= hb[..., None]).all(-1),
        "(c) an earlier column certainly reaches M": ((lo < hb[..., None]) | (cols >= jst[..., None])).all(-1),
    }
    Mlo = lo.max(-1).values
    cand = hi >= Mlo[..., None]
    decided = (~cand | ((lo == Mlo[..., None]) & (hi == Mlo[..., None]))).all(-1)
    first = torch.where(cand, cols, s.shape[-1]).min(-1).values
    checks["(d) decided row differs"] = ~decided | ((hb == Mlo) & (jst == first))
    for name, ok in checks.items():
        if not ok.all():
            b, i = (int(v) for v in torch.nonzero(~ok)[0])
            pytest.fail(f"{what}: {name} on {int((~ok).sum())} rows; first sample {b} row {i}: M = {hb[b, i].item()!r}, "
                        f"j* = {int(jst[b, i])}")
    return int((~decided).sum())


# (kind, B, Ns, Nd, align) at each of C = 320, 640, 1280, plus the video-like rows of the former tie-tolerant test
REAL_CASES = (("gauss", 2, 1536, 2048, False), ("video", 2, 1536, 2048, True), ("video", 1, 300, 5000, False),
              ("gauss", 3, 257, 700, True))

# Rows of test_ka_real_rows_against_float64 whose (max, first arg) the bound does not decide (of 20 103), measured on
# an H100 80GB HBM3.  They depend on the inputs and the bound only, not on the kernel: the video-like rows hold many
# near ties, and a tighter bound, with its argument, is what would lower this.
REAL_UNDECIDED = 6369


def test_ka_real_rows_against_float64():
    """Random unit-norm fp16 rows (Gaussian, and video-like: one base vector plus noise) at C = 320, 640, 1280, with
    and without align_batch, and the numpy-built video rows of the earlier tie-tolerant test.  Every row satisfies
    (a)-(d) of `_check_real` against float64 scores with the bound of `_bound`."""
    undecided = rows = 0
    for C in (320, 640, 1280):
        for i, (kind, B, Ns, Nd, align) in enumerate(REAL_CASES):
            g = torch.Generator(device="cuda").manual_seed(100 * C + i)
            a, b = _unit_rows((B, Ns, C), kind, g), _unit_rows((B, Nd, C), kind, g)
            s, E = _bound(a, b, align)
            what = f"real {kind} C={C} B={B} Ns={Ns} Nd={Nd} align={align}"
            undecided += _check_real(_ka(a, b, B, Ns, Nd, C, align), s, E, what)
            rows += s.shape[0] * Ns
    for align in (False, True):
        rng = np.random.default_rng(7)
        B, Ns, Nd, C = 2, 1536, 2048, 320
        base = rng.standard_normal((B, 1, C))
        a = _dev(O.normalize_rows((base + 0.1 * rng.standard_normal((B, Ns, C))).astype(np.float16)))
        b = _dev(O.normalize_rows((base + 0.1 * rng.standard_normal((B, Nd, C))).astype(np.float16)))
        s, E = _bound(a, b, align)
        undecided += _check_real(_ka(a, b, B, Ns, Nd, C, align), s, E, f"numpy video rows align={align}")
        rows += s.shape[0] * Ns
    print(f"KA real rows: {undecided} of {rows} rows undecided by the bound")
    assert undecided == REAL_UNDECIDED, f"{undecided} undecided rows, pinned at {REAL_UNDECIDED}"


# ---------------------------------------------------------------------------------------------------------------------
# 4. KA with device counts, and the extremes

def test_ka_device_counts_ignore_capacity_rows():
    """vtm_sim_argmax_dev with capacities above the counts.  Capacity rows hold src rows scaled up (x 2) or NaN rows,
    capacity dst rows the best dst rows scaled up or NaN: any of them would change a key if read.  The first Ns keys
    equal vtm_sim_argmax at the host counts and the exact reference; keys [Ns, cap) stay 0."""
    ns_cap, nd_cap = 300, 700
    for i, (Ns, Nd) in enumerate([(300, 512), (299, 600), (100, 200), (300, 700), (129, 257)]):
        for B, align in ((1, False), (2, True), (3, False), (3, True)):
            C = (64, 320, 392, 640)[(i + B) % 4]
            what = f"dev counts Ns={Ns}/{ns_cap} Nd={Nd}/{nd_cap} B={B} C={C} align={align}"
            a, b, want, _, _ = exact_case(C, B, Ns, Nd, align, 9000 + 10 * i + B)
            A = np.zeros((B, ns_cap, C), np.float16)
            Bm = np.zeros((B, nd_cap, C), np.float16)
            A[:, :Ns], Bm[:, :Nd] = a, b
            for r in range(Ns, ns_cap):
                A[:, r] = np.float16(np.nan) if r % 3 == 0 else np.clip(a[:, r % Ns].astype(np.float32) * 2, -6e4, 6e4)
            for j in range(Nd, nd_cap):
                Bm[:, j] = np.float16(np.nan) if j % 5 == 0 else np.clip(b[:, j % Nd].astype(np.float32) * 2, -6e4, 6e4)
            counts = torch.tensor([Ns, Nd, 0, 0], dtype=torch.int32, device="cuda")
            got = _ka(_dev(A), _dev(Bm), B, ns_cap, nd_cap, C, align, counts=counts)
            _assert_keys(got[:, :Ns], want, what)
            host = _ka(_dev(a), _dev(b), B, Ns, Nd, C, align)
            _assert_keys(got[:, :Ns], host, f"{what} against host counts")
            assert (got[:, Ns:] == 0).all(), f"{what}: a key past the count was written"


def test_ka_extremes():
    """NaN and infinity at the C-ABI, as the header documents: a src row with a NaN entry publishes nothing (key 0), a
    NaN dst column is never the arg, an overflowing (+inf) score wins, a row whose every score is -inf publishes
    nothing; each in the full-tile and the partial-tile path of the arg-max."""
    for Nd in (256, 300):
        C, B, Ns = 64, 1, 130
        a, b, _, X, e = exact_case(C, B, Ns, Nd, False, 4242 + Nd, kinds=("overflow", "normal", "neginf"))
        a, b = a.copy(), b.copy()
        a[0, 5, 3] = np.float16(np.nan)            # row 5: a NaN entry
        nan_col = int(np.argmax(rn16(X[0, 1] * 2.0 ** -e[0, 1])))
        b[0, nan_col, 7] = np.float16(np.nan)      # the winning column of group 1 becomes NaN
        sc = np.einsum("ik,jk->ij", a[0].astype(np.float64), b[0].astype(np.float64))
        want = row_keys(rn16(sc))[None]
        h = rn16(sc).astype(np.float64)
        assert want[0, 5] == 0 and (want == 0).sum() > 1, "no row without a key besides the NaN row"
        assert (np.where(np.isnan(h), -np.inf, h).max(-1) == np.inf).any(), "no +inf maximum"
        _assert_keys(_ka(_dev(a), _dev(b), B, Ns, Nd, C, False), want, f"extremes Nd={Nd}")
        _assert_keys(_ka(_dev(a), _dev(b), B, Ns, Nd, C, False, fn="vtm_sim_argmax_simt"), want, f"extremes twin Nd={Nd}")


# ---------------------------------------------------------------------------------------------------------------------
# 5. KB1

def _sort_keys(rng, Bp, Ns):
    """Keys over every 16-bit ordered value and key 0, with heavy ties in the low byte, the high byte or both."""
    out = np.empty((Bp, Ns), np.uint64)
    for b in range(Bp):
        kind = rng.integers(0, 4)
        if kind == 0:
            k16 = rng.integers(0, 1 << 16, Ns)
        elif kind == 1:
            k16 = (rng.integers(0, 256, Ns) << 8) | int(rng.integers(0, 256))
        elif kind == 2:
            k16 = (int(rng.integers(0, 256)) << 8) | rng.integers(0, 256, Ns)
        else:
            k16 = rng.choice(rng.integers(0, 1 << 16, 5), Ns)
        if Ns > (1 << 16):
            k16[rng.permutation(Ns)[:1 << 16]] = np.arange(1 << 16)
        arg = rng.integers(0, 1 << 20, Ns).astype(np.uint64)
        out[b] = (k16.astype(np.uint64) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - arg)
        out[b, rng.random(Ns) < 0.05] = 0
    return out


def _barrier_word(ws, Bp, Ns):
    """The grid-barrier counter of KB1's workspace (after two [Bp][256][tiles] histograms, 256-byte aligned): the
    fused sort zeroes it and its three grid barriers leave 3 x (its CTAs); the six-launch fallback never touches it."""
    tiles = -(-Ns // 1024)
    off = 2 * (-(-4 * Bp * 256 * tiles // 256) * 256)
    return int(ws[off:off + 4].cpu().numpy().view(np.uint32)[0]), 3 * tiles * Bp


def _run_sort(keys, Bp, cap, count=None):
    lib = _lib.load()
    ws_bytes = lib.vtm_topr_workspace_bytes(Bp, cap)
    ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device="cuda")
    edge, rank = _Guarded(Bp * cap, torch.int32), _Guarded(Bp * cap, torch.int32)
    kd = _dev(keys.view(np.int64))
    cnt = None if count is None else torch.tensor([count, 0, 0, 0], dtype=torch.int32, device="cuda")

    def call():
        if cnt is None:
            rc = lib.vtm_topr_sort(kd.data_ptr(), Bp, cap, edge.ptr, rank.ptr, ws.data_ptr(), ws_bytes, _stream())
        else:
            rc = lib.vtm_topr_sort_dev(kd.data_ptr(), Bp, cap, cnt.data_ptr(), edge.ptr, rank.ptr, ws.data_ptr(),
                                       ws_bytes, _stream())
        _sync(rc, "vtm_topr_sort")
    call()
    edge.check(f"KB1 Bp={Bp} Ns={cap} edge")
    rank.check(f"KB1 Bp={Bp} Ns={cap} rank")
    return edge.out().view(Bp, cap).cpu().numpy(), rank.out().view(Bp, cap).cpu().numpy(), _barrier_word(ws, Bp, cap)


def _check_sort(keys, edge, rank, n, what):
    k16 = ((keys[:, :n] >> np.uint64(32)) & np.uint64(0xFFFF)).astype(np.int64)
    want = np.argsort(-k16, axis=-1, kind="stable")
    if not np.array_equal(edge[:, :n], want):
        b, k = np.argwhere(edge[:, :n] != want)[0]
        pytest.fail(f"{what}: edge differs first at sample {b} position {k}: {edge[b, k]} != {want[b, k]}")
    inv = np.empty_like(want)
    np.put_along_axis(inv, want, np.arange(n)[None].repeat(len(want), 0), -1)
    assert np.array_equal(rank[:, :n], inv), f"{what}: rank is not the inverse of edge"


def test_kb1_sort_both_paths():
    """KB1 against a stable descending sort at Ns around 1024-element tiles and Bp 1 ... 4, at the largest fused grid
    (264 CTAs) and past it (the six-launch fallback), with the path that ran read from the workspace's grid-barrier
    counter, so that a device with other than two co-resident sort CTAs per SM shows.  Keys cover every
    16-bit value, key 0 and heavy ties."""
    rng = np.random.default_rng(31)
    paths = set()
    for Bp, Ns in SORT_CASES:
        keys = _sort_keys(rng, Bp, Ns)
        edge, rank, (word, arrivals) = _run_sort(keys, Bp, Ns)
        what = f"KB1 Bp={Bp} Ns={Ns}"
        _check_sort(keys, edge, rank, Ns, what)
        fused = word == arrivals
        assert fused or word == 0xFFFFFFFF, f"{what}: barrier word {word:#x}"
        assert fused == sort_fused(Bp, Ns), f"{what}: ran the {'fused' if fused else 'fallback'} sort"
        paths.add(fused)
    assert paths == {True, False}


def test_kb1_sort_device_count():
    """vtm_topr_sort_dev with counts below capacity: keys past the count are the largest possible (they would sort
    first if read); edge / rank entries past the count are not written."""
    rng = np.random.default_rng(32)
    for Bp, cap, n in ((1, 1025, 1), (2, 3000, 2047), (3, 5000, 1024), (4, 2048, 2047), (1, 300_000, 280_000)):
        keys = _sort_keys(rng, Bp, cap)
        keys[:, n:] = np.uint64(0xFFFF) << np.uint64(32)
        edge, rank, _ = _run_sort(keys, Bp, cap, count=n)
        _check_sort(keys, edge, rank, n, f"KB1 dev Bp={Bp} cap={cap} n={n}")
        assert (edge[:, n:] == SENT32).all() and (rank[:, n:] == SENT32).all(), \
            f"KB1 dev Bp={Bp} cap={cap} n={n}: an entry past the count was written"


# ---------------------------------------------------------------------------------------------------------------------
# 5. KB2 and decode

def _match_data(rng, B, Bp, Ns, Nd):
    """Keys with random args (below B Nd when Bp = 1 < B) and heavily tied maxima; edge / rank from numpy."""
    nmax = rng.choice(np.array([-0.5, 0.0, 0.25, 0.5, 0.75, 1.0], np.float16), size=(Bp, Ns))
    arg = rng.integers(0, (B if Bp == 1 and B > 1 else 1) * Nd, size=(Bp, Ns))
    keys = pack_keys(nmax, arg) if Ns else np.zeros((Bp, 0), np.uint64)
    edge = O.stable_argsort_desc(nmax).astype(np.int32)
    rank = np.empty_like(edge)
    np.put_along_axis(rank, edge.astype(np.int64), np.arange(Ns, dtype=np.int32)[None].repeat(Bp, 0), -1)
    return keys, edge, rank, nmax, arg


def _oracle_match(N, a_idx, b_idx, r, B, Bp, edge, arg, nmax):
    """The oracle's Match for keys packed from (nmax, arg) and sorted as edge, with Bp rows (one shared by all B
    samples when Bp = 1: dst_idx = arg % Nd, as merge.py:103 takes it under align_batch)."""
    Nd = len(b_idx)
    B = Bp
    src = edge[:, :r].astype(np.int64)
    dst = np.take_along_axis(arg, src, 1) % max(Nd, 1)
    m = O.Match(N=N, a_idx=np.asarray(a_idx, np.int64), b_idx=np.asarray(b_idx, np.int64), r=r, node_max=nmax,
                node_idx=arg, unm_idx=np.broadcast_to(edge[:, r:].astype(np.int64), (B, len(a_idx) - r)),
                src_idx=np.broadcast_to(src, (B, r)), dst_idx=np.broadcast_to(dst, (B, r)))
    return m


def _maps(m, B, N):
    ids = np.broadcast_to(np.arange(N, dtype=np.float64)[None, :, None], (B, N, 1)).copy()
    mu = m.merge(ids)[..., 0].astype(np.int64)
    L = mu.shape[1]
    pos = np.broadcast_to(np.arange(L, dtype=np.float64)[None, :, None], (B, L, 1)).copy()
    pi = m.unmerge(pos)[..., 0].astype(np.int64)
    return mu, pi


def _compose(split, r, Ns, Nd, Bp, keys, edge, rank, mu_in=None, pi_in=None, pi_offset=0, N0=None, what=""):
    L = Ns - r + Nd
    mu, pi = _Guarded(Bp * L, torch.int32), _Guarded(Bp * N0, torch.int32)
    kd, ed, rd = (_dev(keys.view(np.int64)), _dev(edge), _dev(rank)) if Ns else (None, None, None)
    p = (lambda t: None if t is None else t.data_ptr())
    _sync(_lib.load().vtm_compose_maps(ctypes.byref(split), r, Ns, Nd, Bp, p(kd), p(ed), p(rd), p(mu_in), p(pi_in),
                                       pi_offset, N0, mu.ptr, pi.ptr, _stream()), f"KB2 {what}")
    mu.check(f"KB2 {what}: mu")
    pi.check(f"KB2 {what}: pi")
    return mu.out().view(Bp, L).cpu().numpy(), pi.out().view(Bp, N0).cpu().numpy()


def _eq(got, want, what):
    if not np.array_equal(got, want):
        b, k = np.argwhere(got != want)[0]
        pytest.fail(f"{what}: first difference at [{b}, {k}]: {got[b, k]} != {want[b, k]}")


MODE0 = [(F, ts, rf) for F in (*range(1, 10), 16) for ts in range(1, 5) if ts <= F for rf in range(ts)]


def _level(rng, kind, N, B, Bp, i):
    """(split, a_idx, b_idx, keepalive) of one level of length N."""
    if kind == "mode0":
        F, ts, rf = MODE0[i % len(MODE0)]
        unm = (0, 3, 5)[i % 3] if N > F * 1 + 5 else 0
        tnum = (N - unm) // F
        unm = N - F * tnum
        a_idx, b_idx, _, _ = O.split_indices_randframe(N, F, unm, ts, rf)
        if i % 4 == 3 and F % min(ts, F) == 0:
            rft = torch.tensor([rf], dtype=torch.int32, device="cuda")
            return VtmSplit.local(N, unm, F, ts, rft), a_idx, b_idx, f"mode 0 F={F} stride={min(ts, F)} randf_dev={rf} unm_pre={unm}"
        return VtmSplit.local(N, unm, F, ts, rf), a_idx, b_idx, f"mode 0 F={F} stride={min(ts, F)} randf={rf} unm_pre={unm}"
    if kind == "prefix":
        sl = int(rng.integers(0, N))
        return VtmSplit.prefix(N, sl), np.arange(sl), np.arange(sl, N), f"prefix src_len={sl}"
    L = N // 2
    high = i % 2 == 0
    if kind == "coin_dev":
        coin = torch.tensor([0.75 if high else 0.25], dtype=torch.float32, device="cuda")
        sp = VtmSplit.prefix_coin(L, coin, 0.5)
    else:                                     # the host coin: the prefix split of the order it chose
        sp = VtmSplit.prefix(2 * L, L)
    src, dst = (np.arange(L), np.arange(L, 2 * L)) if (high or kind == "coin_host") else (np.arange(L, 2 * L), np.arange(L))
    return sp, src, dst, f"{kind} L={L} coin {'>' if high else '<='} threshold"


def test_kb2_compose_every_split_form():
    """One level: mode 0 over F 1 ... 9 and 16 with every stride and randf (host and device draws, carried tokens or
    not, F = 1 giving Ns = 0), the prefix split, the coin split with both branches (host and device coin), at r in {0,
    1, Ns - 1, Ns}, Bp = B and Bp = 1 with args below B Nd: mu and pi equal the oracle's merge / unmerge of index
    tensors.  Then two and three chained levels through mu_in / pi_in with N0 > N."""
    rng = np.random.default_rng(41)
    for i in range(len(MODE0) + 24):
        kind = "mode0" if i < len(MODE0) else ("prefix", "coin_dev", "coin_host")[i % 3]
        B = 1 + i % 3
        Bp = 1 if i % 2 else B
        N = int(rng.integers(2, 60)) if kind == "prefix" else 2 * int(rng.integers(1, 30))
        if kind == "mode0":
            F = MODE0[i][0]
            N = F * (1 + i % 5) + (0, 3, 5)[i % 3]
        sp, a_idx, b_idx, desc = _level(rng, kind, N, B, Bp, i)
        Ns, Nd = len(a_idx), len(b_idx)
        if Nd == 0:
            continue
        keys, edge, rank, nmax, arg = _match_data(rng, B, Bp, Ns, Nd)
        for r in sorted({0, min(1, Ns), max(Ns - 1, 0), Ns}):
            what = f"{desc} N={N} Ns={Ns} Nd={Nd} B={B} Bp={Bp} r={r}"
            m = _oracle_match(N, a_idx, b_idx, r, B, Bp, edge, arg, nmax)
            mu_w, pi_w = _maps(m, Bp, N)
            mu, pi = _compose(sp, r, Ns, Nd, Bp, keys, edge, rank, N0=N, what=what)
            _eq(mu, mu_w, f"{what}: mu")
            _eq(pi, pi_w, f"{what}: pi")

    for depth in (2, 3):
        for i in range(6):
            B = 1 + i % 3
            Bp = 1 if i % 2 else B
            N0 = 4 * (8 + i) + 3
            N, mu_in, pi_in, matches = N0, None, None, []
            for lvl in range(depth):
                F = 4 if lvl == 0 else 2
                unm = N - F * (N // F) if lvl == 0 else (N % F)
                sp = VtmSplit.local(N, unm, F, 4, (i + lvl) % min(4, F))
                a_idx, b_idx, _, _ = O.split_indices_randframe(N, F, unm, 4, (i + lvl) % min(4, F))
                Ns, Nd = len(a_idx), len(b_idx)
                keys, edge, rank, nmax, arg = _match_data(rng, B, Bp, Ns, Nd)
                r = int(rng.integers(0, Ns // 2 + 1))
                matches.append(_oracle_match(N, a_idx, b_idx, r, B, Bp, edge, arg, nmax))
                mu, pi = _compose(sp, r, Ns, Nd, Bp, keys, edge, rank, mu_in, pi_in, 0, N0,
                                  what=f"chain depth={depth} level={lvl} B={B} Bp={Bp}")
                mu_in, pi_in = _dev(mu), _dev(pi)
                N = Ns - r + Nd
            res = O.MergeResult(merged_tokens=None, unmerge=None, matches=matches)
            mu_w, pi_w = O.composed_maps(res, Bp, N0)
            _eq(mu, mu_w, f"chain depth={depth} B={B} Bp={Bp}: mu")
            _eq(pi, pi_w, f"chain depth={depth} B={B} Bp={Bp}: pi")


def test_kb2_global_stage_pi_offset():
    """The global stage composes the local unmerge (pi_in over N0 positions) with its own level, whose local tokens sit
    at [pi_offset, pi_offset + L) of [global | local] when the coin keeps the global tokens first: pi_out[p] =
    level_pi[pi_in[p] + pi_offset]."""
    rng = np.random.default_rng(43)
    for i, (L, Lg, high) in enumerate([(20, 20, True), (20, 20, False), (37, 37, True), (1, 1, False)]):
        B, Bp, N0 = 2, 2 if i % 2 else 1, 3 * L + 5
        N = L + Lg
        sp = VtmSplit.prefix(N, L if high else Lg)
        Ns, Nd = (L, Lg) if high else (Lg, L)
        keys, edge, rank, nmax, arg = _match_data(rng, B, Bp, Ns, Nd)
        r = int(rng.integers(0, Ns + 1))
        m = _oracle_match(N, np.arange(Ns), np.arange(Ns, N), r, B, Bp, edge, arg, nmax)
        _, lvl_pi = _maps(m, Bp, N)
        pi_in = rng.integers(0, L, size=(Bp, N0)).astype(np.int32)
        off = 0 if high else Lg
        _, pi = _compose(sp, r, Ns, Nd, Bp, keys, edge, rank, None, _dev(pi_in), off, N0,
                         what=f"global L={L} coin {'>' if high else '<='}")
        _eq(pi, np.take_along_axis(lvl_pi, pi_in.astype(np.int64) + off, 1), f"global pi_offset={off} L={L}")


def test_kb2_compose_dev_mode2():
    """vtm_compose_maps_dev on mode-2 splits with the global length below its capacity, both coin branches, counts from
    vtm_split_counts_dev: mu and pi equal the oracle's maps; mu past M and pi past L + Lg keep their fill."""
    rng = np.random.default_rng(44)
    lib = _lib.load()
    for i, (L, gcap, lg) in enumerate([(30, 40, 25), (40, 30, 30), (17, 64, 1), (64, 17, 16), (5, 5, 4)]):
        for high in (True, False):
            B, Bp = 2, 1 + i % 2
            coin = torch.tensor([0.75 if high else 0.25], dtype=torch.float32, device="cuda")
            glen = torch.tensor([lg], dtype=torch.int32, device="cuda")
            sp = VtmSplit.prefix_coin_dev(L, glen, gcap, coin, 0.5)
            cap = max(L, gcap)
            ratio = (0.5, 0.9, 1.0)[i % 3]
            counts = torch.zeros(4, dtype=torch.int32, device="cuda")
            _sync(lib.vtm_split_counts_dev(ctypes.byref(sp), ratio, counts.data_ptr(), _stream()), "split counts")
            Ns, Nd = (L, lg) if high else (lg, L)
            r = O.merge_count(Ns, ratio)
            assert counts.tolist() == [Ns, Nd, r, Ns - r + Nd]
            keys, edge, rank, nmax, arg = _match_data(rng, B, Bp, Ns, Nd)
            K = np.zeros((Bp, cap), np.uint64)
            E = np.zeros((Bp, cap), np.int32)
            R = np.zeros((Bp, cap), np.int32)
            K[:, :Ns], E[:, :Ns], R[:, :Ns] = keys, edge, rank
            N = L + gcap
            mu, pi = _Guarded(Bp * N, torch.int32, SENT32), _Guarded(Bp * N, torch.int32, SENT32)
            what = f"KB2 dev L={L} glob_cap={gcap} glob_len={lg} coin {'>' if high else '<='} Bp={Bp}"
            kd, ed, rd = _dev(K.view(np.int64)), _dev(E), _dev(R)
            _sync(lib.vtm_compose_maps_dev(ctypes.byref(sp), counts.data_ptr(), Bp, kd.data_ptr(), ed.data_ptr(),
                                           rd.data_ptr(), None, N, mu.ptr, pi.ptr, _stream()), what)
            mu.check(what)
            pi.check(what)
            mu, pi = mu.out().view(Bp, N).cpu().numpy(), pi.out().view(Bp, N).cpu().numpy()
            src = np.arange(L) if high else np.arange(L, L + lg)
            dst = np.arange(L, L + lg) if high else np.arange(L)
            m = _oracle_match(L + lg, src, dst, r, B, Bp, edge, arg, nmax)
            mu_w, pi_w = _maps(m, Bp, L + lg)
            M = Ns - r + Nd
            _eq(mu[:, :M], mu_w, f"{what}: mu")
            _eq(pi[:, :L + lg], pi_w, f"{what}: pi")
            assert (mu[:, M:] == SENT32).all(), f"{what}: mu written past M"
            assert (pi[:, L + lg:] == SENT32).all(), f"{what}: pi written past L + Lg"


def test_decode_match():
    """vtm_decode_match's five outputs equal the oracle's Match fields (unm_idx, src_idx, dst_idx with % Nd under
    align_batch, node_max, node_idx)."""
    rng = np.random.default_rng(45)
    lib = _lib.load()
    for B, Bp, Ns, Nd in ((1, 1, 1, 1), (2, 2, 300, 77), (3, 1, 1025, 300), (2, 1, 64, 64)):
        keys, edge, rank, nmax, arg = _match_data(rng, B, Bp, Ns, Nd)
        for r in sorted({0, 1, Ns // 2, Ns}):
            m = _oracle_match(Ns + Nd, np.arange(Ns), np.arange(Ns, Ns + Nd), r, B, Bp, edge, arg, nmax)
            outs = [_Guarded(Bp * n) for n in (Ns - r, r, r)]
            nm = _Guarded(Bp * Ns, torch.int32)
            ni = _Guarded(Bp * Ns)
            what = f"decode B={B} Bp={Bp} Ns={Ns} Nd={Nd} r={r}"
            kd, ed = _dev(keys.view(np.int64)), _dev(edge)
            _sync(lib.vtm_decode_match(kd.data_ptr(), ed.data_ptr(), Bp, Ns, Nd, r,
                                       outs[0].ptr, outs[1].ptr, outs[2].ptr, nm.t[LEAD:].data_ptr(), ni.ptr,
                                       _stream()), what)
            for o in outs + [ni]:
                o.check(what)
            got = [o.out().view(Bp, -1).cpu().numpy() for o in outs]
            _eq(got[0], m.unm_idx[:Bp], f"{what}: unm_idx")
            _eq(got[1], m.src_idx[:Bp], f"{what}: src_idx")
            _eq(got[2], m.dst_idx[:Bp], f"{what}: dst_idx")
            half = nm.t[LEAD:].view(torch.int16)[:Bp * Ns].view(Bp, Ns).cpu().numpy().view(np.float16)
            want_h = np.where(m.node_max == 0, np.float16(0), m.node_max)     # -0 is packed as +0
            _eq(half.view(np.uint16), want_h.view(np.uint16), f"{what}: node_max")
            _eq(ni.out().view(Bp, Ns).cpu().numpy(), m.node_idx, f"{what}: node_idx")


def test_split_counts_dev():
    """vtm_split_counts_dev: r = min(Ns, int(Ns * ratio)) for every Ns up to 1024 and a sample of larger ones."""
    lib = _lib.load()
    ns_list = list(range(1, 1025)) + [1031, 4096, 12288, 49152, 65535, 100_003]
    out = torch.zeros((len(ns_list), len(SPLIT_RATIOS), 4), dtype=torch.int32, device="cuda")
    coin = torch.tensor([0.75], dtype=torch.float32, device="cuda")
    keep = []
    for i, Ns in enumerate(ns_list):
        glen = torch.tensor([3], dtype=torch.int32, device="cuda")
        sp = VtmSplit.prefix_coin_dev(Ns, glen, 3, coin, 0.5)
        keep.append(sp)
        for k, ratio in enumerate(SPLIT_RATIOS):
            _lib.check(lib.vtm_split_counts_dev(ctypes.byref(sp), ratio, out[i, k].data_ptr(), _stream()), "counts")
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    for i, Ns in enumerate(ns_list):
        for k, ratio in enumerate(SPLIT_RATIOS):
            r = min(Ns, int(Ns * ratio))
            assert got[i, k].tolist() == [Ns, 3, r, Ns - r + 3], f"Ns={Ns} ratio={ratio}: {got[i, k].tolist()}"
