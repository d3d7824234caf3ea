"""CPU oracle for the VidToMe cross-frame token-merge hot path.  TEST INFRASTRUCTURE ONLY.

A plain-numpy restatement of the reference algorithm (lixirui142/VidToMe @ 064c7b1).  Only `tests/`,
`__graft_entry__.smoke()` and the CPU-baseline legs of `bench.py` may import this module; the product
package `vidtome_b200` never does and has no CPU fallback.

Every function cites the reference lines it follows (paths relative to the reference tree).  The
oracle is pinned against the reference itself: `tests/make_golden.py` imports the reference in the
build container, runs it on seeded inputs and stores its outputs under `tests/golden/`;
`tests/test_oracle_golden.py` replays those fixtures through this file.

Arithmetic model (matches torch CPU, verified bit-for-bit by tests/make_golden.py):
  * fp16 tensors: every op computes in fp32 and rounds its result to fp16 (norm, division, matmul);
  * `scores.max(-1)`: first index among equal maxima (numpy argmax has the same rule);
  * `argsort(descending=True)`: the reference's call is not stable on CPU; the oracle (and the CUDA
    path) define it as STABLE descending — ties keep ascending source-row order — which is what the
    reference's CUDA radix sort produces.  The golden fixtures are generated with the reference's
    argsort forced to stable=True, and separately record how far the unpatched CPU argsort deviates.
Random draws (`torch.randint` merge.py:56-57, `torch.rand` patch.py:62) are NOT restated: callers pass
the drawn values in, so the oracle is independent of the RNG engine.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np


# ----------------------------------------------------------------------------- helpers
def _compute_dtype(x: np.ndarray):
    return np.float32 if x.dtype in (np.float16, np.float32) else np.float64


def normalize_rows(metric: np.ndarray) -> np.ndarray:
    """merge.py:84  `metric = metric / metric.norm(dim=-1, keepdim=True)` (no epsilon)."""
    ct = _compute_dtype(metric)
    m = metric.astype(ct)
    nrm = np.sqrt((m * m).sum(-1, keepdims=True, dtype=ct)).astype(metric.dtype)
    with np.errstate(divide="ignore", invalid="ignore"):
        return (m / nrm.astype(ct)).astype(metric.dtype)


def scores_matmul(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """merge.py:87  `scores = a @ b.transpose(-1, -2)` in the tensors' dtype (fp32 accumulate)."""
    ct = _compute_dtype(a)
    return np.matmul(a.astype(ct), np.swapaxes(b.astype(ct), -1, -2)).astype(a.dtype)


def merge_count(num_src: int, ratio: float) -> int:
    """merge.py:90 / :395  `r = min(a.shape[1], int(a.shape[1] * ratio))`."""
    return min(num_src, int(num_src * ratio))


def stable_argsort_desc(v: np.ndarray) -> np.ndarray:
    """merge.py:98,113  argsort(descending=True), defined stable (see module docstring)."""
    # negating is exact for floats; -0.0 and 0.0 compare equal under both orders
    return np.argsort(-v.astype(np.float32), axis=-1, kind="stable")


def split_indices_randframe(N: int, F: int, unm_pre: int, target_stride: int, randf: int):
    """merge.py:41-71.  Returns (a_idx, b_idx, tnum, stride) as int64 vectors of positions."""
    tnum = (N - unm_pre) // F
    idx_buffer = np.arange(N - unm_pre, dtype=np.int64)                      # :51-52
    stride = min(target_stride, F)                                           # :55
    dst_select = ((idx_buffer // tnum) % stride) == randf                    # :58-60
    a_idx = idx_buffer[~dst_select] + unm_pre                                # :63
    b_idx = idx_buffer[dst_select] + unm_pre                                 # :64
    b_idx = np.concatenate([b_idx, np.arange(unm_pre, dtype=np.int64)])      # :67-69
    return a_idx, b_idx, tnum, stride


@dataclass
class Match:
    """Everything one bipartite matching produces (merge.py:93-117)."""
    N: int
    a_idx: np.ndarray          # [Ns] positions of src tokens
    b_idx: np.ndarray          # [Nd] positions of dst tokens
    r: int
    node_max: np.ndarray       # [B'|Ns] row maxima (B' = 1 when align_batch)
    node_idx: np.ndarray       # [B', Ns] arg maxima (index into the concatenated dst axis if aligned)
    unm_idx: np.ndarray        # [B, Ns - r]
    src_idx: np.ndarray        # [B, r]
    dst_idx: np.ndarray        # [B, r]
    unmerge_chunk: Optional[int] = None
    src_len: Optional[int] = None

    @property
    def num_dst(self) -> int:
        return int(self.b_idx.shape[0])

    @property
    def unm_num(self) -> int:
        return int(self.unm_idx.shape[1])

    # merge.py:119-133 (mode "replace" and "mean")
    def merge(self, x: np.ndarray, mode: str = "replace") -> np.ndarray:
        src, dst = x[:, self.a_idx], x[:, self.b_idx]                         # split(), :76-81
        B, _, c = src.shape
        unm = np.take_along_axis(src, self.unm_idx[:, :, None], axis=1)       # :124
        if mode != "replace":
            # merge.py:126-131: dst.scatter_reduce(-2, dst_idx, src[src_idx], reduce=mode, include_self=True).
            # Sums are formed exactly (fp64 here; fp16 inputs span < 2^41, far inside the 53-bit mantissa for any
            # realistic row count) and rounded ONCE; the reference accumulates in the tensor's dtype in index order,
            # which gives the same result whenever the partial sums are exactly representable (the "exact" fixtures).
            if mode not in ("mean", "sum", "amax", "amin"):
                raise NotImplementedError(mode)
            s = np.take_along_axis(src, self.src_idx[:, :, None], axis=1)        # :127
            if mode in ("mean", "sum"):
                acc = dst.astype(np.float64).copy()                           # include_self=True
                cnt = np.ones((B, dst.shape[1], 1), dtype=np.float64)
                for b in range(B):
                    np.add.at(acc[b], self.dst_idx[b], s[b].astype(np.float64))
                    np.add.at(cnt[b], self.dst_idx[b], 1)
                if mode == "mean":
                    # torch: fp16 sum, then div by the count in fp32 -> fp16; with an exact sum that is RN(sum / count)
                    acc = acc.astype(_compute_dtype(x)) / cnt.astype(_compute_dtype(x))
                dst = acc.astype(x.dtype)
            else:
                acc = dst.copy()
                fn = np.maximum if mode == "amax" else np.minimum
                for b in range(B):
                    fn.at(acc[b], self.dst_idx[b], s[b])
                dst = acc
        return np.concatenate([unm, dst], axis=1)                             # :133

    # merge.py:135-155 (+ :459 for the global matcher)
    def unmerge(self, x: np.ndarray) -> np.ndarray:
        unm_len = self.unm_idx.shape[1]
        unm, dst = x[:, :unm_len], x[:, unm_len:]                             # :138
        B, _, c = unm.shape
        src = np.take_along_axis(dst, self.dst_idx[:, :, None], axis=1)       # :142
        out = np.zeros((B, self.N, c), dtype=x.dtype)                         # :145
        out[:, self.b_idx] = dst                                              # :147
        for b in range(B):
            out[b, self.a_idx[self.unm_idx[b]]] = unm[b]                      # :149-150
            out[b, self.a_idx[self.src_idx[b]]] = src[b]                      # :152-153
        if self.unmerge_chunk is not None:                                    # :459
            out = out[:, : self.src_len] if self.unmerge_chunk == 0 else out[:, self.src_len:]
        return out


def _rowmax_first_index_f16(s32: np.ndarray):
    """max / first arg-max of fp16(s32) along the last axis WITHOUT converting the whole matrix to fp16
    (numpy's half conversion is slow).  Rounding is monotone, so the fp16 maximum is fp16(max s32) =: h, and
    an element rounds to h iff it lies above the midpoint between h and its fp16 predecessor (or exactly on
    it when h's mantissa is even: round-to-nearest-even).  Equivalent to `s32.astype(f16).argmax(-1)`;
    tests/test_oracle_golden.py checks the equivalence."""
    m32 = s32.max(-1)
    h = m32.astype(np.float16)
    prev = np.nextafter(h, np.float16(-np.inf))
    mid = (h.astype(np.float32) + prev.astype(np.float32)) * np.float32(0.5)     # exact in fp32
    even = (h.view(np.uint16) & 1) == 0
    cand = s32 > mid[..., None]
    tie = even[..., None] & (s32 == mid[..., None])
    idx = (cand | tie).argmax(-1)
    return h, idx


def _match(metric: np.ndarray, a_idx: np.ndarray, b_idx: np.ndarray, ratio: float, align_batch: bool,
           row_block: int = 4096, fast: bool = True) -> Match:
    """merge.py:84-117 (shared verbatim by :389-421).  The score matrix is produced in row blocks so
    that the full-size configurations fit in host memory; results are identical to the one-shot form."""
    B, N, _ = metric.shape
    mn = normalize_rows(metric)                                               # :84
    a, b = mn[:, a_idx], mn[:, b_idx]                                         # :85
    Ns, Nd = a.shape[1], b.shape[1]
    r = merge_count(Ns, ratio)                                                # :90
    Bp = 1 if align_batch else B
    node_max = np.empty((Bp, Ns), dtype=metric.dtype)
    node_idx = np.empty((Bp, Ns), dtype=np.int64)
    ct = _compute_dtype(metric)
    half = metric.dtype == np.float16
    a32, bT32 = a.astype(ct), np.ascontiguousarray(np.swapaxes(b.astype(ct), -1, -2))
    for lo in range(0, Ns, row_block):
        hi = min(Ns, lo + row_block)
        s = np.matmul(a32[:, lo:hi], bT32)                                    # :87  [B, rows, Nd] (fp32 accumulate)
        if align_batch:
            s = np.concatenate([s[i] for i in range(B)], axis=-1)[None]       # :96  [1, rows, B*Nd]
        if half and fast:
            node_max[:, lo:hi], node_idx[:, lo:hi] = _rowmax_first_index_f16(s)
        else:
            s = s.astype(metric.dtype)                                        # the reference's `scores` dtype
            node_idx[:, lo:hi] = s.argmax(-1)                                 # :97 / :112 (first max)
            node_max[:, lo:hi] = np.take_along_axis(s, node_idx[:, lo:hi, None], -1)[..., 0]
    edge_idx = stable_argsort_desc(node_max)                                  # :98 / :113
    unm_idx = edge_idx[:, r:]                                                 # :100 / :115
    src_idx = edge_idx[:, :r]                                                 # :101 / :116
    dst_idx = np.take_along_axis(node_idx, src_idx, axis=1)                   # :102 / :117
    if align_batch:
        dst_idx = dst_idx % Nd                                                # :103
        unm_idx = np.broadcast_to(unm_idx, (B,) + unm_idx.shape[1:])          # :106-108
        src_idx = np.broadcast_to(src_idx, (B,) + src_idx.shape[1:])
        dst_idx = np.broadcast_to(dst_idx, (B,) + dst_idx.shape[1:])
    return Match(N=N, a_idx=a_idx, b_idx=b_idx, r=r, node_max=node_max, node_idx=node_idx,
                 unm_idx=unm_idx, src_idx=src_idx, dst_idx=dst_idx)


# ----------------------------------------------------------------------------- matchers (L0)
def bipartite_soft_matching_randframe(metric: np.ndarray, F: int, ratio: float, unm_pre: int, randf: int,
                                      target_stride: int = 4, align_batch: bool = False) -> Optional[Match]:
    """merge.py:20-159.  `randf` is the value torch.randint drew at merge.py:56-57.
    Returns None for ratio <= 0 (merge.py:45-46: identity ops, unm_num = tnum)."""
    B, N, _ = metric.shape
    if ratio <= 0:
        return None
    a_idx, b_idx, _, _ = split_indices_randframe(N, F, unm_pre, target_stride, randf)
    return _match(metric, a_idx, b_idx, ratio, align_batch)


def bipartite_soft_matching_2s(metric: np.ndarray, src_len: int, ratio: float, align_batch: bool,
                               unmerge_chunk: int = 0) -> Match:
    """merge.py:343-463."""
    B, N, _ = metric.shape
    if ratio <= 0:
        # merge.py:364-365 returns a 2-tuple that the only caller unpacks into 3 (patch.py:73): a crash
        raise ValueError("not enough values to unpack (expected 3, got 2)")
    idx = np.arange(N, dtype=np.int64)
    m = _match(metric, idx[:src_len], idx[src_len:], ratio, align_batch)      # :375-376
    m.unmerge_chunk, m.src_len = unmerge_chunk, src_len
    return m


# ----------------------------------------------------------------------------- orchestration (L1)
def join_frame(x: np.ndarray, fsize: int) -> np.ndarray:
    """vidtome/utils.py:32-35  "(B F) N C -> B (F N) C"."""
    bf, n, c = x.shape
    return x.reshape(bf // fsize, fsize * n, c)


def split_frame(x: np.ndarray, fsize: int) -> np.ndarray:
    """vidtome/utils.py:37-40  "B (F N) C -> (B F) N C"."""
    b, fn, c = x.shape
    return x.reshape(b * fsize, fn // fsize, c)


@dataclass
class MergeResult:
    merged_tokens: np.ndarray
    unmerge: Callable[[np.ndarray], np.ndarray]
    matches: List[Match] = field(default_factory=list)
    global_tokens: Optional[np.ndarray] = None   # new value of module.global_tokens
    randf: List[int] = field(default_factory=list)
    coin: Optional[float] = None
    merged: bool = True


def compute_merge(x: np.ndarray, size: Tuple[int, int], *, batch_size: int, local_merge_ratio: float,
                  max_downsample: int = 2, target_stride: int = 4, align_batch: bool = False,
                  merge_global: bool = False, global_merge_ratio: float = 0.8, global_rand: float = 0.5,
                  global_tokens: Optional[np.ndarray] = None,
                  draw_randf: Callable[[int], int] = None,
                  draw_coin: Callable[[], float] = None) -> MergeResult:
    """vidtome/patch.py:14-91.  `draw_randf(stride)` returns the torch.randint(0, stride) value of
    merge.py:56-57 (one draw per level); `draw_coin()` returns the torch.rand(1) value of patch.py:62."""
    original_tokens = size[0] * size[1]
    downsample = int(math.ceil(math.sqrt(original_tokens // x.shape[1])))     # :15-17
    fsize = x.shape[0] // batch_size                                          # :23
    tsize = x.shape[1]                                                        # :24
    if downsample > max_downsample:                                           # :27, :86-88
        return MergeResult(merged_tokens=x, unmerge=lambda y: y, merged=False, global_tokens=global_tokens)

    local_tokens = join_frame(x, fsize)                                       # :37
    u_ls: List[Callable] = [lambda y: split_frame(y, fsize)]                  # :39
    matches: List[Match] = []
    randfs: List[int] = []
    unm, curF = 0, fsize
    while curF > 1:                                                           # :44
        N = local_tokens.shape[1]
        if local_merge_ratio <= 0:
            # merge.py:45-46: identity ops and unm_num = tnum; no RNG draw happens
            unm += (N - unm) // curF
        else:
            if min(target_stride, curF) < 2:
                # every frame is dst: nothing merges and curF never falls, so the reference loops forever
                raise ValueError(f"target_stride {target_stride}: the local levels never reduce the frame count")
            rf = int(draw_randf(min(target_stride, curF)))
            randfs.append(rf)
            m = bipartite_soft_matching_randframe(local_tokens, curF, local_merge_ratio, unm, rf,
                                                  target_stride, align_batch)  # :45-46
            unm += m.unm_num                                                  # :47
            matches.append(m)
            u_ls.append(m.unmerge)                                            # :49
            local_tokens = m.merge(local_tokens)                              # :50
        curF = (local_tokens.shape[1] - unm) // tsize                         # :54
    merged_tokens = local_tokens                                              # :56
    coin = None
    new_global = global_tokens
    if merge_global:                                                          # :59
        if global_tokens is not None:                                         # :60
            coin = float(draw_coin())
            g = global_tokens.astype(local_tokens.dtype)                      # .to(local_tokens) :65,:70
            # :62 torch compares its fp32 draw with the Python float in fp32: global_rand rounds to nearest first
            if np.float32(coin) > np.float32(global_rand):
                src_len = local_tokens.shape[1]
                tokens = np.concatenate([local_tokens, g], axis=1)            # :64-65
                local_chunk = 0
            else:
                src_len = g.shape[1]
                tokens = np.concatenate([g, local_tokens], axis=1)            # :69-70
                local_chunk = 1
            m = bipartite_soft_matching_2s(tokens, src_len, global_merge_ratio, align_batch,
                                           unmerge_chunk=local_chunk)         # :73-74
            merged_tokens = m.merge(tokens)                                   # :75
            matches.append(m)
            u_ls.append(m.unmerge)                                            # :77
            new_global = m.unmerge(merged_tokens).copy()                      # :80
        else:
            new_global = local_tokens.copy()                                  # :82

    def unmerge(y: np.ndarray) -> np.ndarray:                                 # :85  func_warper(u_ls[::-1])
        for f in u_ls[::-1]:
            y = f(y)
        return y

    return MergeResult(merged_tokens=merged_tokens, unmerge=unmerge, matches=matches,
                       global_tokens=new_global, randf=randfs, coin=coin)


# ----------------------------------------------------------------------------- attention + block
def _linear(x: np.ndarray, w: np.ndarray, b: Optional[np.ndarray] = None) -> np.ndarray:
    ct = _compute_dtype(x)
    y = x.astype(ct) @ w.astype(ct).T
    if b is not None:
        y = y + b.astype(ct)
    return y.astype(x.dtype)


def attention(x: np.ndarray, wq: np.ndarray, wk: np.ndarray, wv: np.ndarray, wo: np.ndarray,
              bo: Optional[np.ndarray], heads: int, scale: Optional[float] = None) -> np.ndarray:
    """Self-attention of diffusers' `Attention` as the reference restates it, utils/pnp_utils.py:47-95:
    to_q/to_k/to_v (no bias) -> head_to_batch_dim -> softmax(q k^T * scale) v -> batch_to_head_dim ->
    to_out[0] (bias).  Intermediate tensors are rounded to the input dtype like the eager fp16 path;
    the softmax itself is evaluated in fp32."""
    B, L, C = x.shape
    d = C // heads
    scale = d ** -0.5 if scale is None else scale
    ct = _compute_dtype(x)
    q = _linear(x, wq).reshape(B, L, heads, d).transpose(0, 2, 1, 3).astype(ct)
    k = _linear(x, wk).reshape(B, L, heads, d).transpose(0, 2, 1, 3).astype(ct)
    v = _linear(x, wv).reshape(B, L, heads, d).transpose(0, 2, 1, 3).astype(ct)
    out = np.empty((B, heads, L, d), dtype=ct)
    blk = 2048
    for lo in range(0, L, blk):
        s = np.matmul(q[:, :, lo:lo + blk], k.transpose(0, 1, 3, 2)) * scale
        s = s - s.max(-1, keepdims=True)
        p = np.exp(s)
        p = p / p.sum(-1, keepdims=True)
        out[:, :, lo:lo + blk] = np.matmul(p, v)
    o = out.transpose(0, 2, 1, 3).reshape(B, L, C).astype(x.dtype)
    return _linear(o, wo, bo)


def layer_norm(x: np.ndarray, w: np.ndarray, b: np.ndarray, eps: float = 1e-5) -> np.ndarray:
    ct = _compute_dtype(x)
    xf = x.astype(ct)
    mu = xf.mean(-1, keepdims=True)
    var = ((xf - mu) ** 2).mean(-1, keepdims=True)
    return ((xf - mu) / np.sqrt(var + eps) * w.astype(ct) + b.astype(ct)).astype(x.dtype)


def tome_block_self_attention(hidden: np.ndarray, size: Tuple[int, int], norm_w: np.ndarray, norm_b: np.ndarray,
                              wq, wk, wv, wo, bo, heads: int, **merge_kwargs):
    """vidtome/patch.py:139-169: norm1 -> compute_merge -> attn1 on merged tokens -> unmerge -> + residual.
    Returns (hidden_out, MergeResult)."""
    nh = layer_norm(hidden, norm_w, norm_b)                                   # :146
    res = compute_merge(nh, size, **merge_kwargs)                             # :149-150
    attn = attention(res.merged_tokens, wq, wk, wv, wo, bo, heads)            # :157-162
    out = res.unmerge(attn)                                                   # :168
    ct = _compute_dtype(hidden)
    return (out.astype(ct) + hidden.astype(ct)).astype(hidden.dtype), res     # :169


# ----------------------------------------------------------------------------- composed maps
def composed_maps(res: MergeResult, B: int, N0: int) -> Tuple[np.ndarray, np.ndarray]:
    """The whole merge as ONE gather and the whole unmerge as ONE gather (replace mode):
    merged[b, i] = table[b, mu[b, i]],  out[b, p] = y[b, pi[b, p]], where `table` is the level-0 token
    sequence join_frame(x) (followed by the global tokens when a global stage ran: rows N0.. ).
    Derived by pushing index tensors through the same merge/unmerge closures, so it inherits their
    exact semantics."""
    Ltot = N0
    glob = [m for m in res.matches if m.unmerge_chunk is not None]
    ids = np.broadcast_to(np.arange(N0, dtype=np.float64)[None, :, None], (B, N0, 1)).copy()
    cur = ids
    for m in res.matches:
        if m.unmerge_chunk is None:
            cur = m.merge(cur)
        else:
            Lg = m.N - cur.shape[1]
            gids = np.broadcast_to((N0 + np.arange(Lg, dtype=np.float64))[None, :, None], (B, Lg, 1))
            cur = np.concatenate([cur, gids] if m.unmerge_chunk == 0 else [gids, cur], axis=1)
            cur = m.merge(cur)
            Ltot = N0 + Lg
    mu = cur[..., 0].astype(np.int64)
    L = mu.shape[1]
    pos = np.broadcast_to(np.arange(L, dtype=np.float64)[None, :, None], (B, L, 1)).copy()
    y = pos
    for m in res.matches[::-1]:
        y = m.unmerge(y)
    pi = y[..., 0].astype(np.int64)
    return mu, pi
