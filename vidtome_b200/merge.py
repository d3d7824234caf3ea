"""Bipartite soft matching on the H100 — same operator interface as the reference's vidtome/merge.py.

`bipartite_soft_matching_randframe` (vidtome/merge.py:20-159) and `bipartite_soft_matching_2s`
(vidtome/merge.py:343-463) keep their names, argument meaning, return triple `(merge, unmerge, ret_dict)`
and error behaviour.  What changes is the machinery: the matching runs as four CUDA launches through the
C-ABI (K0 normalise+split, KA wgmma similarity+arg-max, KB1 stable radix order, KB2 map composition) and
the returned closures are single row-gather kernels over int32 maps instead of chains of
torch.gather/scatter_ calls on int64 indices expanded to `[b, n, c]`.

`merge_mode="replace"` — the only mode any caller in the reference uses (patch.py:45-50,73-75) — is the composed
single-gather path; the scatter_reduce modes "mean", "sum", "amax", "amin" (merge.py:126-131) run as an exact,
order-independent reduction (csrc/reduce.cu); "prod" raises NotImplementedError rather than silently doing something
else.  There is no CPU path: tensors must be CUDA fp16.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Optional, Tuple

import torch

from . import ops
from ._lib import VtmSplit
from .utils import draw_randf


def do_nothing(x: torch.Tensor, mode: str = None, **kwarg):
    """vidtome/merge.py:5-6."""
    return x


@dataclass
class LevelMatch:
    """Device-resident result of one matching (the state the reference keeps in closure variables
    `a_idx, b_idx, unm_idx, src_idx, dst_idx`, vidtome/merge.py:63-69,100-117)."""
    split: VtmSplit
    B: int
    Bp: int            # 1 when align_batch (one match shared by all samples), else B
    Ns: int
    Nd: int
    r: int
    keys: torch.Tensor   # [Bp, Ns] packed (ordered fp16 max, ~arg) — KA output
    edge: torch.Tensor   # [Bp, Ns] int32 stable descending order of the row maxima
    rank: torch.Tensor   # [Bp, Ns] int32 inverse of edge
    # device counts [Ns, Nd, r, M] of a mode-2 split (match_level_dev); Ns / Nd above are then capacities and r is None
    counts: Optional[torch.Tensor] = None

    @property
    def unm_num(self) -> int:
        return self.Ns - self.r

    def index_tensors(self, want_node: bool = False):
        """(unm_idx, src_idx, dst_idx) as int64 [B, *, 1] exactly like merge.py:100-108 / :115-117
        (expanded over the batch when align_batch)."""
        out = ops.decode_match(self.keys, self.edge, self.Nd, self.r, want_node=want_node)
        unm, src, dst = out[:3]
        if self.Bp != self.B:
            unm, src, dst = (t.expand(self.B, -1, -1) for t in (unm, src, dst))
        return (unm, src, dst) + tuple(out[3:])


def _check_metric(metric: torch.Tensor) -> None:
    if not isinstance(metric, torch.Tensor) or not metric.is_cuda:
        raise RuntimeError("vidtome_b200: tokens must live on a CUDA device — this path has no CPU fallback")
    if metric.dtype != torch.float16:
        raise RuntimeError(f"vidtome_b200: tokens must be float16 (the path computes in fp16), got {metric.dtype}")
    if metric.dim() != 3:
        raise RuntimeError("vidtome_b200: tokens must be [B, N, C]")


def match_level(table: torch.Tensor, rowmap: Optional[torch.Tensor], split: VtmSplit, ratio: float,
                align_batch: bool, ln=None) -> LevelMatch:
    """K0 + KA + KB1 for one level.  `table` [B, N0, C] fp16 holds the level-0 tokens, `rowmap`
    ([B'|1, N] int32 or None) maps this level's positions to rows of `table`; `ln` = (weight, bias, eps)
    applies the block's LayerNorm to the rows as they are read."""
    B = table.shape[0]
    Ns, Nd = ops.split_counts(split)
    if Ns == 0:
        # a single frame (stride 1): every token is dst (merge.py:58-69 with an empty a_idx), nothing to match
        empty64 = torch.empty((1 if align_batch else B, 0), dtype=torch.int64, device=table.device)
        empty32 = torch.empty((empty64.shape[0], 0), dtype=torch.int32, device=table.device)
        return LevelMatch(split=split, B=B, Bp=empty64.shape[0], Ns=0, Nd=Nd, r=0, keys=empty64, edge=empty32,
                          rank=empty32)
    a, b = ops.normalize_split(table, rowmap, split, ln)        # merge.py:84-85
    r = ops.merge_count(Ns, ratio)                              # merge.py:90
    keys = ops.sim_argmax(a, b, align_batch)                    # merge.py:87,93-97,112
    edge, rank = ops.topr_sort(keys)                            # merge.py:98,113
    return LevelMatch(split=split, B=B, Bp=keys.shape[0], Ns=Ns, Nd=Nd, r=r, keys=keys, edge=edge, rank=rank)


def match_level_dev(tokens: torch.Tensor, split: VtmSplit, ratio: float, align_batch: bool) -> LevelMatch:
    """K0 + KA + KB1 for a mode-2 split (VtmSplit.prefix_coin_dev): the counts are derived on the device first and every
    kernel reads them from there, so nothing depends on a value read back to the host."""
    B = tokens.shape[0]
    Ns, Nd = ops.split_counts(split)                            # capacities
    counts = ops.split_counts_dev(split, ratio)
    a, b = ops.normalize_split(tokens, None, split)
    keys = ops.sim_argmax(a, b, align_batch, counts=counts)
    edge, rank = ops.topr_sort(keys, counts=counts)
    return LevelMatch(split=split, B=B, Bp=keys.shape[0], Ns=Ns, Nd=Nd, r=None, keys=keys, edge=edge, rank=rank,
                      counts=counts)


def _closures(m: LevelMatch, N: int, unmerge_slice: Optional[Tuple[int, int]], merge_mode: str):
    mu, pi = ops.compose_maps(m.split, m.r, m.keys, m.edge, m.rank, None, None, 0, N)
    if unmerge_slice is not None:
        lo, hi = unmerge_slice
        pi = pi[:, lo:hi].contiguous()

    def merge(x: torch.Tensor, mode=None) -> torch.Tensor:
        mode = mode if mode is not None else merge_mode
        _check_metric(x)
        if mode != "replace":
            # merge.py:126-131: scatter_reduce of the matched src rows into their dst rows (include_self=True)
            return ops.merge_reduce(x.contiguous(), m.split, m.r, m.keys, m.edge, mode)
        return ops.gather_rows(x.contiguous(), mu)               # merge.py:119-133, one pass

    def unmerge(x: torch.Tensor, **kwarg) -> torch.Tensor:
        _check_metric(x)
        return ops.unmerge_add(x.contiguous(), pi, None)         # merge.py:135-155 (+ :459), one pass

    merge.match = m
    unmerge.match = m
    return merge, unmerge


def bipartite_soft_matching_randframe(metric: torch.Tensor, F: int, ratio: float, unm_pre: int,
                                      generator: torch.Generator, target_stride: int = 4,
                                      align_batch: bool = False, merge_mode: str = "replace"
                                      ) -> Tuple[Callable, Callable, dict]:
    """Local matcher, vidtome/merge.py:20-159: dst = tokens of one random frame per `target_stride`
    frames (plus the `unm_pre` tokens left unmerged by the previous level), src = the rest; merges
    `ratio` of the src tokens into their most similar dst token."""
    B, N, _ = metric.shape
    tnum = (N - unm_pre) // F                                    # merge.py:43
    if ratio <= 0:
        return do_nothing, do_nothing, {"unm_num": tnum}         # merge.py:45-46
    _check_metric(metric)
    stride = min(target_stride, F)                               # merge.py:55
    randf = draw_randf(generator, stride, F)                     # merge.py:56-57 (same draw)
    split = VtmSplit.local(N, unm_pre, F, target_stride, randf)
    m = match_level(metric.contiguous(), None, split, ratio, align_batch)
    merge, unmerge = _closures(m, N, None, merge_mode)
    return merge, unmerge, {"unm_num": m.unm_num}                # merge.py:158


def bipartite_soft_matching_2s(metric: torch.Tensor, src_len: int, ratio: float, align_batch: bool,
                               merge_mode: str = "replace", unmerge_chunk: int = 0):
    """Global matcher, vidtome/merge.py:343-463: src = first `src_len` tokens, dst = the rest;
    `unmerge` returns only partition `unmerge_chunk` (0 = src part, 1 = dst part)."""
    B, N, _ = metric.shape
    if ratio <= 0:
        return do_nothing, do_nothing                             # merge.py:364-365 (2-tuple, as the reference)
    _check_metric(metric)
    split = VtmSplit.prefix(N, src_len)
    m = match_level(metric.contiguous(), None, split, ratio, align_batch)
    sl = (0, src_len) if unmerge_chunk == 0 else (src_len, N)    # merge.py:459
    merge, unmerge = _closures(m, N, sl, merge_mode)
    return merge, unmerge, {"unm_num": m.unm_num}                # merge.py:462
