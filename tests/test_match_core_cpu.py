"""The matching stage's planners and reference builders, checked without a GPU.

`tests/test_gpu_match_core.py` tests KA (sim_argmax.cu), KB1 and KB2 (topr.cu) against references built here.  This file
restates what decides which code path a call takes (`Layout::plan`, `Items::plan` / `Items::decode` for KA, the fused /
six-launch choice of KB1, on a 132-SM H100) and asserts that the GPU tests' shapes reach every one of them.  It also checks
the reference builders themselves: the rounding-exact KA inputs give the intended float64 scores, their fp16 roundings
hit every case the tests name, and the oracle's fast row arg-max agrees with them.
"""
import math

import numpy as np

import vidtome_oracle as O

SMS = 132                      # streaming multiprocessors of an H100 SXM
TARGET_ITEMS_PER_SM = 8        # ka::TARGET_ITEMS_PER_SM
BM, BN, BK = 128, 256, 64      # KA tile: src rows, dst columns, channels per k-chunk
A_BYTES, B_BYTES = BM * BK * 2, BN * BK * 2
MAX_STAGES, MIN_RESIDENT_STAGES, MAX_A_CHUNKS = 6, 3, 8
SMEM_LIMIT = 227 * 1024
FIXED = 1024 + 8 * (2 * MAX_STAGES + 2 * MAX_A_CHUNKS)
SORT_TILE = 1024               # KB1: elements per CTA
SORT_CTAS_PER_SM = 2           # co-resident radix_sort_fused_kernel CTAs per SM (1024 threads, 32 registers, 45 KB)
Q_EXP = 8                      # the rounding-exact dst rows hold integers times 2^-Q_EXP


# ---------------------------------------------------------------------------------------------------------------------
# KA planners (sim_argmax.cu)

def layout_plan(k_chunks):
    """Layout::plan -> (resident, ring stages)."""
    a_res = k_chunks * A_BYTES
    resident = k_chunks <= MAX_A_CHUNKS and FIXED + a_res + MIN_RESIDENT_STAGES * B_BYTES <= SMEM_LIMIT
    a_bytes = a_res if resident else 0
    stage_bytes = B_BYTES if resident else A_BYTES + B_BYTES
    return resident, min(MAX_STAGES, (SMEM_LIMIT - FIXED - a_bytes) // stage_bytes)


def items_plan(Ns, Nd, C, B):
    """Items::plan (SMS SMs) plus the grid: a dict of its fields."""
    m_tiles, n_tiles, k_chunks = -(-Ns // BM), -(-Nd // BN), -(-C // BK)
    base = m_tiles * B
    s = 1
    while base * s < TARGET_ITEMS_PER_SM * SMS and s * 2 <= n_tiles:
        s *= 2
    tps = -(-n_tiles // s)
    n_splits = -(-n_tiles // tps)
    total = base * n_splits
    return dict(m_tiles=m_tiles, n_tiles=n_tiles, k_chunks=k_chunks, tps=tps, n_splits=n_splits, total=total,
                grid=min(total, SMS), B=B)


def decode(w, plan):
    """Items::decode: work item w -> (m_tile, b, nt0, nt1)."""
    m = w % plan["m_tiles"]
    rest = w // plan["m_tiles"]
    b, sp = rest % plan["B"], rest // plan["B"]
    nt0 = sp * plan["tps"]
    return m, b, nt0, min(nt0 + plan["tps"], plan["n_tiles"])


def cta_items(c, plan):
    """The work items CTA c runs, in order: c, c + grid, ..."""
    return [decode(w, plan) for w in range(c, plan["total"], plan["grid"])]


def split_case(plan):
    """Which form of the dst sweep split a plan takes."""
    if plan["n_splits"] == 1:
        return "one split"
    if plan["n_tiles"] % plan["tps"]:
        return "short last split"
    return "even splits"


# Shapes of the every-width sweep, (B, Ns, Nd, align), cycled through the widths.  Ns: one row, one 128-row block
# +-1, 255, 300, a last block of one row; Nd: 1, 7, 255, 256, 257, 300, and sweeps split into several dst ranges with
# a short last one; (3, 2000, 3000) has more work items than CTAs, so resident src blocks are reloaded.
KA_SHAPES = (
    (1, 1, 1, False), (2, 127, 7, True), (1, 128, 255, False), (3, 129, 256, False), (2, 255, 257, True),
    (1, 300, 300, False), (4, 257, 261, True), (1, 129, 2600, False), (2, 300, 1795, True), (3, 2000, 3000, False),
    (2, 385, 259, False), (1, 1, 262, True), (4, 130, 1283, False), (3, 64, 2822, True), (2, 300, 258, False),
    (1, 640, 263, True),
)
KA_WIDTHS = tuple(range(8, 1281, 8)) + (1288, 1480, 1720, 2040, 2048)


def ka_width_cases():
    """(C, B, Ns, Nd, align) of the every-width sweep."""
    return [(C,) + KA_SHAPES[i % len(KA_SHAPES)] for i, C in enumerate(KA_WIDTHS)]


# Threshold-order case: with align_batch and 132 src blocks of 128 rows, CTA m runs (m, b=0, range 0), (m, b=1,
# range 0), (m, b=0, range 1), (m, b=1, range 1), in that order; sample 0's second range holds smaller args than
# sample 1's first range, so a maximum published by the earlier item is the threshold the later one must tie.
ORDER_SHAPE = dict(B=2, Ns=SMS * BM, Nd=2 * BN, C=64)


# ---------------------------------------------------------------------------------------------------------------------
# fp16 keys

def rn16(x):
    """float64 -> fp16, correctly rounded (ties to even, overflow to +-inf)."""
    with np.errstate(over="ignore"):
        return np.asarray(x, dtype=np.float64).astype(np.float16)


def ordered16(h):
    """fp16 array -> the 16-bit order-preserving image KA packs (-0 as +0)."""
    u = h.view(np.uint16).astype(np.uint64)
    u = np.where(u == 0x8000, 0, u)
    return np.where(u & 0x8000, u ^ 0xFFFF, u | 0x8000)


def pack_keys(h, arg):
    return (ordered16(h) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - arg.astype(np.uint64))


def row_keys(h):
    """KA's key of each row of fp16 scores h [..., N]: the largest score and the first column holding it; NaN scores
    never win, and a row with no score above -inf publishes nothing (key 0)."""
    valid = ~np.isnan(h) & (h != -np.inf)
    hv = np.where(valid, h, np.float16(-np.inf))
    idx = hv.argmax(-1)
    mx = np.take_along_axis(hv, idx[..., None], -1)[..., 0]
    return np.where(valid.any(-1), pack_keys(mx, idx), np.uint64(0)).astype(np.uint64)


# ---------------------------------------------------------------------------------------------------------------------
# Rounding-exact KA inputs
#
# Src row i of sample b holds sigma 2^-p (2^10, 1) at columns (2g, 2g + 1), g = i mod C/2, and zeros elsewhere; dst row
# j holds (hi, lo) 2^-Q_EXP at every column pair g.  Every score is then sigma (hi 2^10 + lo) 2^-(p + Q_EXP) = X 2^-e:
# an integer X with |X| < 2^21 + 2^11 (the sum of |products| of the whole dot product, below 2^22 in units of 2^-e),
# so the fp32 accumulation is exact in any order and under any alignment, while its rounding to fp16 is not.  One
# group g of the rows of a sample (all samples with align_batch) has one exponent e and one design of X over the dst
# axis (the B Nd concatenated columns with align_batch).

KINDS = ("normal", "negative", "subnormal", "cross", "overflow", "zero", "neginf")
LIM = 2 ** 21 - 1


def _kind_params(kind, rng):
    """(e, T, U): row exponent, top value of the design and the fp16 spacing there, both in units of 2^-e."""
    if kind in ("normal", "negative"):
        t = int(rng.integers(12, 20))
        e = int(np.clip(t - rng.integers(-10, 12), Q_EXP - 5, Q_EXP + 24))
        U = 2 ** (t - 10)
        T = int(rng.integers(1024, 2048)) * U
        return e, (T if kind == "normal" else -T), U
    if kind == "subnormal":                  # scores m 2^-24, m < 1024: spacing 2^-24 = 256 units at e = 32
        return Q_EXP + 24, int(rng.integers(4, 1016)) * 256, 256
    if kind == "cross":                      # around 2^-14, where the subnormals end
        return Q_EXP + 24, int(rng.integers(1018, 1031)) * 256, 256
    if kind == "overflow":                   # around 65504 / 65520 at e = 5: spacing 32 = 1024 units
        return 5, int(rng.integers(2040, 2048)) * 1024, 1024
    if kind == "zero":
        return Q_EXP + 24, 0, 256
    return 5, -2096640, 1024                 # neginf: every score <= -65520


def _positions(rng, k, Ndv, Nd, tps):
    """k distinct dst positions (on the axis of Ndv = Nd or B Nd columns), spread over the places the arg-max code
    tells apart: the same lane, lanes of a quad, 64-column groups, tiles, work items, samples, the last tile."""
    j0 = int(rng.integers(0, Ndv))
    out = [j0]
    for _ in range(200):
        if len(out) == k:
            break
        cls = int(rng.integers(0, 7))
        r = int(rng.integers(1, 4)) * (1 if rng.random() < 0.7 else -1)
        j = {0: j0 + 8 * r, 1: j0 + int(rng.integers(1, 8)) * (1 if r > 0 else -1), 2: j0 + 64 * r + int(rng.integers(0, 8)),
             3: j0 + BN * r + int(rng.integers(0, 64)), 4: j0 + tps * BN * r + int(rng.integers(0, 16)),
             5: j0 + Nd * r, 6: (j0 // Nd) * Nd + (Nd - 1 - int(rng.integers(0, max(1, Nd % BN or BN))))}[cls]
        if 0 <= j < Ndv and j not in out:
            out.append(j)
    return out


def design_group(kind, rng, Ndv, Nd, tps):
    """(e, X [Ndv]) of one group."""
    e, T, U = _kind_params(kind, rng)
    if kind == "neginf":
        return e, -rng.integers(2096640, 2098176, size=Ndv).astype(np.float64)
    lo = max(-LIM, T - 2 ** 21)
    hi_fill = T - 2 * U
    X = rng.integers(lo, max(lo + 1, hi_fill), size=Ndv).astype(np.float64)
    k = int(rng.integers(2, 8))
    cols = sorted(_positions(rng, k, Ndv, Nd, tps))
    offs = np.array([-U // 2 - 1, -U // 2, -U // 2 + 1, -1, 0, 0, 1, U // 2 - 1, U // 2, U // 2 + 1, U])
    vals = np.clip(T + rng.choice(offs, size=len(cols)), -LIM, 2047 * 1024 + 2047)
    if rng.random() < 0.7:
        vals = np.sort(vals)                 # the larger exact value at the later column
    X[cols] = vals
    return e, X


def design(rng, B, Nd, C, align, tps, kinds=KINDS):
    """(X [Bq, G, Ndv], e [Bq, G]) for every group, the kinds cycled (randomly offset) over the groups."""
    G = C // 2
    Bq, Ndv = (1, B * Nd) if align else (B, Nd)
    X = np.empty((Bq, G, Ndv))
    e = np.empty((Bq, G), dtype=np.int64)
    off = int(rng.integers(0, len(kinds)))
    for q in range(Bq):
        for g in range(G):
            e[q, g], X[q, g] = design_group(kinds[(off + q * G + g) % len(kinds)], rng, Ndv, Nd, tps)
    return X, e


def exact_operands(X, e, B, Ns, Nd, C, align, rng):
    """fp16 a [B, Ns, C], b [B, Nd, C] whose scores are X 2^-e (see above); sigma = -1 for a random half of the groups."""
    Bq, G, _ = X.shape
    sigma = np.where(rng.random((Bq, G)) < 0.5, -1.0, 1.0)
    D = sigma[..., None] * X
    hi = np.sign(D) * np.minimum(2047, np.round(np.abs(D) / 1024))
    lo = D - 1024 * hi
    assert np.abs(hi).max() <= 2047 and np.abs(lo).max() <= 2047
    assert (1024 * np.abs(hi) + np.abs(lo)).max() < 2 ** 22, "exactness premise: partial sums within 23 bits"
    if align:
        hi, lo = hi.reshape(G, B, Nd).transpose(1, 0, 2), lo.reshape(G, B, Nd).transpose(1, 0, 2)
        sigma, p = np.broadcast_to(sigma, (B, G)), np.broadcast_to(e - Q_EXP, (B, G))
    else:
        p = e - Q_EXP
    assert p.min() >= -5 and p.max() <= 24
    b = np.empty((B, Nd, G, 2))
    b[..., 0], b[..., 1] = hi.transpose(0, 2, 1), lo.transpose(0, 2, 1)
    b = (b.reshape(B, Nd, C) * 2.0 ** -Q_EXP).astype(np.float16)
    g = np.arange(Ns) % G
    s = sigma[:, g] * np.exp2(-p[:, g].astype(np.float64))                     # [B, Ns]
    a = np.zeros((B, Ns, C))
    rows = np.arange(Ns)
    a[:, rows, 2 * g] = s * 1024.0
    a[:, rows, 2 * g + 1] = s
    a16 = a.astype(np.float16)
    assert np.array_equal(a16.astype(np.float64), a) and np.array_equal(b.astype(np.float64) * 2.0 ** Q_EXP,
                                                                        b.astype(np.float64) * 2.0 ** Q_EXP)
    return a16, b


def exact_scores16(X, e):
    """RN16 of every designed score, [Bq, G, Ndv]."""
    return rn16(X * np.exp2(-e.astype(np.float64))[..., None])


def expected_keys(X, e, Ns):
    """KA's keys [B', Ns] for the design."""
    kg = row_keys(exact_scores16(X, e))                                        # [Bq, G]
    return kg[:, np.arange(Ns) % X.shape[1]]


def exact_case(C, B, Ns, Nd, align, seed, kinds=KINDS):
    """a, b, expected keys and the design of one rounding-exact KA case."""
    rng = np.random.default_rng(seed)
    tps = items_plan(Ns, Nd, C, B)["tps"]
    X, e = design(rng, B, Nd, C, align, tps, kinds)
    a, b = exact_operands(X, e, B, Ns, Nd, C, align, rng)
    return a, b, expected_keys(X, e, Ns), X, e


# ---------------------------------------------------------------------------------------------------------------------
# KB1 path, split counts

def sort_fused(Bp, Ns):
    """KB1 runs its one-launch sort when every CTA can be resident at once, else the six-launch fallback."""
    return -(-Ns // SORT_TILE) * Bp <= SMS * SORT_CTAS_PER_SM


SORT_CASES = [(Bp, Ns) for Ns in (1, 1023, 1024, 1025, 2047, 3073, 49152) for Bp in (1, 2, 3, 4)] + [
    (1, 265 * 1024 + 1), (3, 89 * 1024), (1, 264 * 1024), (2, 132 * 1024)]

SPLIT_RATIOS = tuple(k / 10 for k in range(1, 11)) + (0.8, 0.9, 1 / 3)


# ---------------------------------------------------------------------------------------------------------------------
# tests

def test_layout_plan_bands():
    """The resident src block holds for C <= 512 (k_chunks <= 8) with the stages below; wider rows stream with 4."""
    want = {1: 6, 2: 6, 3: 5, 4: 5, 5: 4, 6: 4, 7: 3, 8: 3}
    for k in range(1, 33):
        res, st = layout_plan(k)
        assert res == (k <= 8), k
        assert st == (want[k] if res else 4), (k, st)


def test_width_sweep_reaches_every_configuration():
    """The every-width sweep covers every resident (k_chunks, stages), the streaming form, every K tail, every split
    form, more items than CTAs, a last src block of one row, and every residue of Nd mod 8 in a partial last tile."""
    cases = ka_width_cases()
    configs, splits, tails, residues = set(), set(), set(), set()
    reload = one_row = False
    for C, B, Ns, Nd, align in cases:
        p = items_plan(Ns, Nd, C, B)
        configs.add(layout_plan(p["k_chunks"]))
        tails.add(C % BK)
        splits.add(split_case(p))
        reload |= p["total"] > p["grid"] and layout_plan(p["k_chunks"])[0]
        one_row |= Ns % BM == 1 and Ns > 1
        if Nd % BN:
            residues.add(Nd % 8)
    assert configs == {(True, 6), (True, 5), (True, 4), (True, 3), (False, 4)}
    ks = {items_plan(1, 1, C, 1)["k_chunks"] for C, *_ in cases}
    assert set(range(1, 9)) <= ks and max(ks) > 8
    assert tails == set(range(0, BK, 8))
    assert splits == {"one split", "short last split", "even splits"}, splits
    assert reload and one_row
    assert residues == set(range(8)), residues


def test_threshold_order_case():
    """In the threshold-order shape every CTA runs sample 1's first dst range before sample 0's second, whose args
    are smaller: the later item must tie the maximum the earlier one published."""
    s = ORDER_SHAPE
    p = items_plan(s["Ns"], s["Nd"], s["C"], s["B"])
    assert p["grid"] == SMS and p["n_splits"] == 2 and p["m_tiles"] == SMS
    for c in range(p["grid"]):
        seq = cta_items(c, p)
        assert all(m == c for m, *_ in seq)
        assert seq.index((c, 1, 0, 1)) < seq.index((c, 0, 1, 2))


def test_sort_cases_reach_both_paths():
    fused = {sort_fused(Bp, Ns) for Bp, Ns in SORT_CASES}
    assert fused == {True, False}
    assert -(-264 * 1024 // SORT_TILE) == SMS * SORT_CTAS_PER_SM and sort_fused(1, 264 * 1024)
    assert not sort_fused(1, 265 * 1024 + 1) and not sort_fused(3, 89 * 1024)


def _exact_check(C, B, Ns, Nd, align, seed):
    a, b, keys, X, e = exact_case(C, B, Ns, Nd, align, seed)
    s = np.einsum("bik,bjk->bij", a.astype(np.float64), b.astype(np.float64))
    if align:
        s = np.concatenate(list(s), -1)[None]
    g = np.arange(Ns) % (C // 2)
    want = X[:, g] * np.exp2(-e[:, g].astype(np.float64))[..., None]
    assert np.array_equal(s, want), f"C={C}: scores are not the designed exact values"
    assert np.array_equal(row_keys(rn16(s)), keys)
    return X, e, keys


def test_exact_builder_scores_and_keys():
    """The operands' float64 products are the designed scores exactly, and the expected keys are those of their
    RN16 matrix, at a spread of widths and shapes."""
    for i, (C, B, Ns, Nd, align) in enumerate(ka_width_cases()[::9]):
        if Ns * Nd * B * C <= 2e8:
            _exact_check(C, B, Ns, Nd, align, 1000 + i)


def _lanes(j):
    return (j % 8) // 2


def test_exact_builder_rounding_and_tie_coverage():
    """Across the sweep's designs: midpoints rounding to even up and down, one unit above and below a midpoint,
    several distinct exact scores rounding to the row maximum with a larger one at a later column, negative, zero,
    subnormal, 2^-14-crossing and overflowing maxima, rows that publish nothing; and ties of the row maximum between
    the same lane, every pair of lanes of a quad, 64-column groups, tiles, work items, samples and the last partial
    tile.  The oracle's fast arg-max agrees wherever the maximum is finite."""
    seen = dict.fromkeys(("mid up", "mid down", "mid+1", "mid-1", "distinct later larger", "negative max", "zero max",
                          "subnormal max", "cross 2^-14", "inf max", "65504 max", "no key", "same lane", "group",
                          "tile", "item", "sample", "last tile"), 0)
    pairs = set()
    for i, (C, B, Ns, Nd, align) in enumerate(ka_width_cases()):
        rng = np.random.default_rng(2000 + i)
        tps = items_plan(Ns, Nd, C, B)["tps"]
        X, e = design(rng, B, Nd, C, align, tps)
        sc = X * np.exp2(-e.astype(np.float64))[..., None]
        h = rn16(sc)
        keys = row_keys(h)
        seen["no key"] += int((keys == 0).sum())
        fin = np.isfinite(h.astype(np.float64)).all(-1)
        hi, idx = O._rowmax_first_index_f16(sc.astype(np.float32)[fin])
        hv = np.where(np.isnan(h), -np.inf, h.astype(np.float64))
        mx = hv.max(-1)
        ok = fin & (mx > -np.inf)
        assert np.array_equal(hi.astype(np.float64), mx[fin]) and np.array_equal(idx, hv[fin].argmax(-1)), C
        seen["inf max"] += int((mx == np.inf).sum())
        seen["65504 max"] += int((mx == 65504).sum())
        seen["negative max"] += int(((mx < 0) & (mx > -np.inf)).sum())
        seen["zero max"] += int((mx == 0).sum())
        seen["subnormal max"] += int(((mx > 0) & (mx < 2.0 ** -14)).sum())
        # midpoints: an exact score halfway between two fp16 values rounds to the even one, down or up (65520 -> inf)
        with np.errstate(invalid="ignore", over="ignore"):
            h64 = h.astype(np.float64)
            m_up = (h64 + np.nextafter(h, np.float16(np.inf)).astype(np.float64)) / 2
            m_dn = (h64 + np.nextafter(h, np.float16(-np.inf)).astype(np.float64)) / 2
            q = np.exp2(-e.astype(np.float64))[..., None]
            seen["mid down"] += int((np.isfinite(m_up) & (sc == m_up)).sum())
            seen["mid up"] += int((np.isfinite(m_dn) & (sc == m_dn)).sum() + (np.abs(sc) == 65520).sum())
            near = np.isfinite(m_up) & np.isfinite(m_dn)
            seen["mid+1"] += int((near & ((sc - q == m_up) | (sc - q == m_dn))).sum())
            seen["mid-1"] += int((near & ((sc + q == m_up) | (sc + q == m_dn))).sum())
        seen["cross 2^-14"] += int(((np.abs(sc) < 2.0 ** -14) & (np.abs(h64) == 2.0 ** -14)).sum())
        for qq, g in zip(*np.nonzero(ok)):
            cols = np.nonzero(hv[qq, g] == mx[qq, g])[0]
            if len(cols) < 2:
                continue
            j, rest = cols[0], cols[1:]
            if (sc[qq, g, rest] > sc[qq, g, j]).any():
                seen["distinct later larger"] += 1
            for k in rest:
                jl, kl = j % Nd, k % Nd
                if j // Nd != k // Nd:
                    seen["sample"] += 1
                elif jl // (tps * BN) != kl // (tps * BN):
                    seen["item"] += 1
                elif jl // BN != kl // BN:
                    seen["tile"] += 1
                elif jl // 64 != kl // 64:
                    seen["group"] += 1
                elif jl % 8 == kl % 8:
                    seen["same lane"] += 1
                else:
                    pairs.add(tuple(sorted((_lanes(jl), _lanes(kl)))))
                if Nd % BN and kl // BN == Nd // BN:
                    seen["last tile"] += 1
    missing = [k for k, v in seen.items() if v == 0]
    assert not missing, f"no design exercises: {missing}"
    assert {(a, b) for a in range(4) for b in range(a + 1, 4)} <= pairs, pairs
    print("rounding-exact designs: " + ", ".join(f"{k} {v}" for k, v in seen.items()))


def test_row_keys_rules():
    """NaN scores never win, +inf wins, a row of -inf (or NaN) publishes nothing, -0 packs as +0, first index."""
    h = np.array([[np.nan, 1, 2, 2], [-np.inf, -np.inf, -np.inf, -np.inf], [np.nan] * 4, [1, np.inf, np.nan, np.inf],
                  [-0.0, 0.0, -1, 0.0]], dtype=np.float16)
    k = row_keys(h)
    assert k[1] == 0 and k[2] == 0
    assert k[0] == pack_keys(np.float16(2), np.array(2))
    assert k[3] == pack_keys(np.float16(np.inf), np.array(1))
    assert k[4] == pack_keys(np.float16(0), np.array(0))


def test_split_count_reference():
    """vtm_merge_count's rule, which vtm_split_counts_dev must reproduce: min(Ns, int(Ns * ratio)) in double."""
    for Ns in (0, 1, 3, 10, 1000, 1024, 65536):
        for ratio in SPLIT_RATIOS:
            assert O.merge_count(Ns, ratio) == min(Ns, math.floor(Ns * ratio))
