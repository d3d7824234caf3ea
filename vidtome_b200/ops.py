"""Thin torch-tensor wrappers over the C-ABI (one function per entry point of include/vidtome_b200.h).

torch is used here only for device memory and streams.  Every function requires CUDA fp16 / int32
tensors and raises on anything else — there is no CPU or eager-PyTorch implementation behind these.
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence, Optional, Tuple

import torch

from . import _lib
from ._lib import VtmSplit, check


class _Stats:
    """Launch accounting for bench.py: `launches` counts the CUDA kernels this library enqueued; with
    `reset(timed={"KA", "KD", ...})` every call of the named ops is bracketed by CUDA events on the launching stream
    and recorded in `events[name]` as (start, end, algorithmic FLOPs, algorithmic bytes)."""
    launches = 0
    timed = frozenset()
    events = {}

    @classmethod
    def reset(cls, timed=()):
        cls.launches, cls.timed, cls.events = 0, frozenset(timed), {}


STATS = _Stats


class _Timed:
    """Context manager: CUDA-event bracket around one op when STATS asks for it (no-op otherwise)."""
    __slots__ = ("name", "flops", "bytes", "ev")

    def __init__(self, name: str, flops: float, nbytes: float):
        self.name, self.flops, self.bytes, self.ev = name, flops, nbytes, None

    def __enter__(self):
        if self.name in STATS.timed:
            self.ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            self.ev[0].record()
        return self

    def __exit__(self, *exc):
        if self.ev is not None:
            self.ev[1].record()
            STATS.events.setdefault(self.name, []).append((self.ev[0], self.ev[1], self.flops, self.bytes))
        return False


def _stream() -> int:
    # raw cudaStream_t of torch's current stream (the cheap accessor: torch.cuda.current_stream() builds a Stream
    # object on every call, ~13 us, and every op below needs it)
    return torch._C._cuda_getCurrentRawStream(torch.cuda.current_device())


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _require(t: torch.Tensor, dtype, name: str) -> None:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"vidtome_b200: `{name}` must be a CUDA tensor (this path has no CPU fallback)")
    if t.dtype != dtype:
        raise RuntimeError(f"vidtome_b200: `{name}` must be {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise RuntimeError(f"vidtome_b200: `{name}` must be contiguous")


def split_counts(split: VtmSplit) -> Tuple[int, int]:
    ns, nd = C.c_int32(), C.c_int32()
    check(_lib.load().vtm_split_counts(C.byref(split), C.byref(ns), C.byref(nd)), "vtm_split_counts")
    return ns.value, nd.value


def merge_count(num_src: int, ratio: float) -> int:
    return int(_lib.load().vtm_merge_count(num_src, float(ratio)))


def split_counts_dev(split: VtmSplit, ratio: float) -> torch.Tensor:
    """Device counts of a mode-2 split (VtmSplit.prefix_coin_dev): an int32 CUDA tensor [Ns, Nd, r, M] written by one
    kernel; nothing is read back to the host."""
    dev = split._keepalive[0].device
    counts = torch.empty(4, dtype=torch.int32, device=dev)
    check(_lib.load().vtm_split_counts_dev(C.byref(split), float(ratio), counts.data_ptr(), _stream()),
          "vtm_split_counts_dev")
    STATS.launches += 1
    return counts


def _ln_args(ln):
    """ln = None or (weight [C] fp16, bias [C] fp16 | None, eps)."""
    if ln is None:
        return None, None, 0.0
    w, b, eps = ln
    _require(w, torch.float16, "ln weight")
    if b is not None:
        _require(b, torch.float16, "ln bias")
    return w.data_ptr(), _ptr(b), float(eps)


def normalize_split(x: torch.Tensor, rowmap: Optional[torch.Tensor], split: VtmSplit, ln=None):
    """K0.  x [B, N0, C] fp16; rowmap [B'|1, N] int32 or None; ln = (weight, bias, eps) fuses the block's
    LayerNorm in front.  Returns (a [B,Ns,C], b [B,Nd,C])."""
    _require(x, torch.float16, "x")
    B, _, Cc = x.shape
    ns, nd = split_counts(split)
    a = torch.empty((B, ns, Cc), dtype=torch.float16, device=x.device)
    b = torch.empty((B, nd, Cc), dtype=torch.float16, device=x.device)
    map_bs = 0
    if rowmap is not None:
        _require(rowmap, torch.int32, "rowmap")
        map_bs = 0 if rowmap.shape[0] == 1 else rowmap.shape[1]
    lw, lb, eps = _ln_args(ln)
    with _Timed("K0", 0.0, 4.0 * B * (ns + nd) * Cc):            # read N rows, write N rows
        check(_lib.load().vtm_normalize_split_ln(x.data_ptr(), x.stride(0), _ptr(rowmap), map_bs, C.byref(split),
                                                 B, Cc, lw, lb, eps, a.data_ptr(), b.data_ptr(), _stream()),
              "vtm_normalize_split_ln")
    STATS.launches += 1
    return a, b


def sim_argmax(a: torch.Tensor, b: torch.Tensor, align_batch: bool, simt: bool = False,
               counts: Optional[torch.Tensor] = None) -> torch.Tensor:
    """KA.  Returns the packed keys [B'|Ns] as an int64 tensor (bit pattern of the uint64 keys).  With `counts` (the
    device counts of a mode-2 split) a and b are sized for capacity and Ns / Nd are read on the device."""
    _require(a, torch.float16, "a")
    _require(b, torch.float16, "b")
    B, Ns, Cc = a.shape
    Nd = b.shape[1]
    keys = torch.empty((1 if align_batch else B, Ns), dtype=torch.int64, device=a.device)
    lib = _lib.load()
    if counts is not None:
        _require(counts, torch.int32, "counts")
        if simt:
            check(-3, "KA with device counts (the SIMT twin does not read them)")
        with _Timed("KA", 2.0 * B * Ns * Nd * Cc, 2.0 * B * (Ns + Nd) * Cc + 8.0 * keys.shape[0] * Ns):
            check(lib.vtm_sim_argmax_dev(a.data_ptr(), b.data_ptr(), B, Ns, Nd, Cc, int(bool(align_batch)),
                                         counts.data_ptr(), keys.data_ptr(), _stream()), "vtm_sim_argmax_dev")
        STATS.launches += 1
        return keys
    fn = lib.vtm_sim_argmax_simt if simt else lib.vtm_sim_argmax
    with _Timed("KA", 2.0 * B * Ns * Nd * Cc, 2.0 * B * (Ns + Nd) * Cc + 8.0 * keys.shape[0] * Ns):
        check(fn(a.data_ptr(), b.data_ptr(), B, Ns, Nd, Cc, int(bool(align_batch)), keys.data_ptr(), _stream()),
              "vtm_sim_argmax")
    STATS.launches += 1
    return keys


def topr_sort(keys: torch.Tensor, counts: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """KB1.  keys [Bp, Ns] -> (edge [Bp, Ns] int32, rank [Bp, Ns] int32).  With `counts` (device counts), Ns is the
    capacity and only the first counts[0] entries of each row are sorted."""
    _require(keys, torch.int64, "keys")
    Bp, Ns = keys.shape
    lib = _lib.load()
    ws_bytes = lib.vtm_topr_workspace_bytes(Bp, Ns)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=keys.device)
    edge = torch.empty((Bp, Ns), dtype=torch.int32, device=keys.device)
    rank = torch.empty((Bp, Ns), dtype=torch.int32, device=keys.device)
    with _Timed("KB1", 0.0, 24.0 * Bp * Ns):
        if counts is not None:
            _require(counts, torch.int32, "counts")
            check(lib.vtm_topr_sort_dev(keys.data_ptr(), Bp, Ns, counts.data_ptr(), edge.data_ptr(), rank.data_ptr(),
                                        ws.data_ptr(), ws_bytes, _stream()), "vtm_topr_sort_dev")
        else:
            check(lib.vtm_topr_sort(keys.data_ptr(), Bp, Ns, edge.data_ptr(), rank.data_ptr(), ws.data_ptr(),
                                    ws_bytes, _stream()), "vtm_topr_sort")
    # one cooperative launch when all (tiles x Bp) CTAs are co-resident (2 per SM), else 6 small launches
    STATS.launches += 1 if ((Ns + 1023) // 1024) * Bp <= 2 * torch.cuda.get_device_properties(keys.device).multi_processor_count else 6
    return edge, rank


def compose_maps(split: VtmSplit, r: int, keys: torch.Tensor, edge: torch.Tensor, rank: torch.Tensor,
                 mu_in: Optional[torch.Tensor], pi_in: Optional[torch.Tensor], pi_offset: int, N0: int):
    """KB2.  Returns (mu_out [Bp, Ns-r+Nd], pi_out [Bp, N0])."""
    Bp, Ns = keys.shape
    ns, nd = split_counts(split)
    assert ns == Ns
    mu_out = torch.empty((Bp, Ns - r + nd), dtype=torch.int32, device=keys.device)
    pi_out = torch.empty((Bp, N0), dtype=torch.int32, device=keys.device)
    if mu_in is not None:
        _require(mu_in, torch.int32, "mu_in")
    if pi_in is not None:
        _require(pi_in, torch.int32, "pi_in")
    kp, ep, rp = (None, None, None) if Ns == 0 else (keys.data_ptr(), edge.data_ptr(), rank.data_ptr())
    check(_lib.load().vtm_compose_maps(C.byref(split), r, Ns, nd, Bp, kp, ep, rp, _ptr(mu_in), _ptr(pi_in), pi_offset, N0,
                                       mu_out.data_ptr(), pi_out.data_ptr(), _stream()), "vtm_compose_maps")
    STATS.launches += 1
    return mu_out, pi_out


def compose_maps_dev(split: VtmSplit, counts: torch.Tensor, keys: torch.Tensor, edge: torch.Tensor,
                     rank: torch.Tensor, pi_in: Optional[torch.Tensor], N0: int):
    """KB2 with device counts (mode-2 split).  Returns (mu_out [Bp, split.N]: first M entries meaningful, pi_out
    [Bp, N0]: without pi_in only the first L + Lg entries are)."""
    _require(counts, torch.int32, "counts")
    Bp = keys.shape[0]
    mu_out = torch.empty((Bp, split.N), dtype=torch.int32, device=keys.device)
    pi_out = torch.empty((Bp, N0), dtype=torch.int32, device=keys.device)
    if pi_in is not None:
        _require(pi_in, torch.int32, "pi_in")
    check(_lib.load().vtm_compose_maps_dev(C.byref(split), counts.data_ptr(), Bp, keys.data_ptr(), edge.data_ptr(),
                                           rank.data_ptr(), _ptr(pi_in), N0, mu_out.data_ptr(), pi_out.data_ptr(),
                                           _stream()), "vtm_compose_maps_dev")
    STATS.launches += 1
    return mu_out, pi_out


def decode_match(keys: torch.Tensor, edge: torch.Tensor, Nd: int, r: int, want_node: bool = False):
    """Expand KA/KB1 results to the reference's int64 index tensors: (unm_idx, src_idx, dst_idx[, node_max, node_idx])."""
    Bp, Ns = keys.shape
    dev = keys.device
    if Ns == 0:
        e = torch.empty((Bp, 0, 1), dtype=torch.int64, device=dev)
        extra = (torch.empty((Bp, 0), dtype=torch.float16, device=dev), torch.empty((Bp, 0), dtype=torch.int64, device=dev))
        return (e, e.clone(), e.clone()) + (extra if want_node else ())
    unm = torch.empty((Bp, Ns - r, 1), dtype=torch.int64, device=dev)
    src = torch.empty((Bp, r, 1), dtype=torch.int64, device=dev)
    dst = torch.empty((Bp, r, 1), dtype=torch.int64, device=dev)
    nmax = torch.empty((Bp, Ns), dtype=torch.float16, device=dev) if want_node else None
    nidx = torch.empty((Bp, Ns), dtype=torch.int64, device=dev) if want_node else None
    check(_lib.load().vtm_decode_match(keys.data_ptr(), edge.data_ptr(), Bp, Ns, Nd, r, unm.data_ptr(),
                                       src.data_ptr(), dst.data_ptr(), _ptr(nmax), _ptr(nidx), _stream()),
          "vtm_decode_match")
    STATS.launches += 1
    return (unm, src, dst, nmax, nidx) if want_node else (unm, src, dst)


def gather_rows(x: torch.Tensor, row_map: Optional[torch.Tensor], L: Optional[int] = None,
                out: Optional[torch.Tensor] = None, ln=None) -> torch.Tensor:
    """KC.  y[b, i] = [LayerNorm](x[b, map[b, i]]).  x [B, N, C]; map [B'|1, L] int32."""
    _require(x, torch.float16, "x")
    B, _, Cc = x.shape
    map_bs = 0
    if row_map is not None:
        _require(row_map, torch.int32, "map")
        L = row_map.shape[1]
        map_bs = 0 if row_map.shape[0] == 1 else L
    if out is None:
        out = torch.empty((B, L, Cc), dtype=torch.float16, device=x.device)
    lw, lb, eps = _ln_args(ln)
    with _Timed("KC", 0.0, 4.0 * B * L * Cc + 4.0 * B * L):       # read L rows, write L rows, + map
        check(_lib.load().vtm_gather_rows_ln(x.data_ptr(), x.stride(0), _ptr(row_map), map_bs, B, L, Cc, lw, lb, eps,
                                             out.data_ptr(), out.stride(0), _stream()), "vtm_gather_rows_ln")
    STATS.launches += 1
    return out


def gather_rows_dev(x: torch.Tensor, row_map: torch.Tensor, length: torch.Tensor) -> torch.Tensor:
    """KC with a device row count: y[b, i] = x[b, map[b, i]] for i < *length, zeros up to the map's width (the
    capacity).  x [B, N, C]; map [B'|1, L_cap] int32; length a 1-element int32 CUDA tensor."""
    _require(x, torch.float16, "x")
    _require(row_map, torch.int32, "map")
    _require(length, torch.int32, "length")
    B, _, Cc = x.shape
    L = row_map.shape[1]
    map_bs = 0 if row_map.shape[0] == 1 else L
    out = torch.empty((B, L, Cc), dtype=torch.float16, device=x.device)
    with _Timed("KC", 0.0, 4.0 * B * L * Cc + 4.0 * B * L):
        check(_lib.load().vtm_gather_rows_dev(x.data_ptr(), x.stride(0), row_map.data_ptr(), map_bs, B, L, Cc,
                                              length.data_ptr(), out.data_ptr(), out.stride(0), _stream()),
              "vtm_gather_rows_dev")
    STATS.launches += 1
    return out


def gather_rows_peers(x: torch.Tensor, row_map: Optional[torch.Tensor], out: torch.Tensor, peer_ptrs: Sequence[int],
                      ln=None) -> torch.Tensor:
    """KC + exchange: like gather_rows into `out` [B, L, C], and the same rows are stored to the buffers at
    `peer_ptrs` (device addresses of identically laid out [B, L, C] regions in other GPUs' memory)."""
    _require(x, torch.float16, "x")
    _require(out, torch.float16, "out")
    B, _, Cc = x.shape
    L = out.shape[1]
    map_bs = 0
    if row_map is not None:
        _require(row_map, torch.int32, "map")
        if row_map.shape[1] != L:
            raise RuntimeError("gather_rows_peers: map length != out length")
        map_bs = 0 if row_map.shape[0] == 1 else L
    arr = (C.c_void_p * max(1, len(peer_ptrs)))(*[C.c_void_p(int(q)) for q in peer_ptrs])
    lw, lb, eps = _ln_args(ln)
    check(_lib.load().vtm_gather_rows_peers(x.data_ptr(), x.stride(0), _ptr(row_map), map_bs, B, L, Cc, lw, lb, eps,
                                            out.data_ptr(), out.stride(0), arr, len(peer_ptrs), _stream()),
          "vtm_gather_rows_peers")
    STATS.launches += 1
    return out


MERGE_MODES = {"mean": 1, "sum": 2, "amax": 3, "amin": 4}


def merge_reduce(x: torch.Tensor, split: VtmSplit, r: int, keys: torch.Tensor, edge: torch.Tensor, mode: str) -> torch.Tensor:
    """merge(x, mode) for the scatter_reduce modes (merge.py:126-131): [unmerged src | reduce(dst, matched src)]."""
    _require(x, torch.float16, "x")
    if mode not in MERGE_MODES:
        raise NotImplementedError(f"vidtome_b200: merge mode {mode!r} is not implemented (replace, mean, sum, amax, amin are)")
    B, _, Cc = x.shape
    ns, nd = split_counts(split)
    Bp = keys.shape[0]
    lib = _lib.load()
    ws_bytes = lib.vtm_merge_reduce_workspace_bytes(B, nd, Cc)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
    y = torch.empty((B, ns - r + nd, Cc), dtype=torch.float16, device=x.device)
    kp, ep = (None, None) if ns == 0 else (keys.data_ptr(), edge.data_ptr())
    check(lib.vtm_merge_reduce(x.data_ptr(), x.stride(0), C.byref(split), r, Bp, kp, ep, B, Cc, MERGE_MODES[mode],
                               y.data_ptr(), ws.data_ptr(), ws_bytes, _stream()), "vtm_merge_reduce")
    STATS.launches += 3
    return y


def unmerge_add(y: torch.Tensor, row_map: torch.Tensor, resid: Optional[torch.Tensor]) -> torch.Tensor:
    """KE.  out[b, p] = y[b, map[b, p]] (+ resid[b, p]).  y [B, L, C]; map [B'|1, N] int32 with contiguous rows (a
    column slice of a wider map is read in place); resid [B, N, C]."""
    _require(y, torch.float16, "y")
    N = row_map.shape[1] if isinstance(row_map, torch.Tensor) else 0
    if N and row_map.dim() == 2 and row_map.shape[0] > 1 and row_map.stride(1) == 1 and row_map.stride(0) > N:
        _require(row_map[0], torch.int32, "map")                  # column slice: read in place through its row stride
        map_bs = row_map.stride(0)
    else:
        _require(row_map, torch.int32, "map")
        map_bs = 0 if row_map.shape[0] == 1 else N
    B, _, Cc = y.shape
    if resid is not None:
        _require(resid, torch.float16, "resid")
    out = torch.empty((B, N, Cc), dtype=torch.float16, device=y.device)
    L = y.shape[1]
    nbytes = 2.0 * B * (L + (2 if resid is not None else 1) * N) * Cc + 4.0 * B * N    # SURVEY §8d: B(L + 2N)C*2 + map
    with _Timed("KE", 0.0, nbytes):
        check(_lib.load().vtm_unmerge_add(y.data_ptr(), y.stride(0), row_map.data_ptr(), map_bs, _ptr(resid),
                                          B, N, Cc, out.data_ptr(), _stream()), "vtm_unmerge_add")
    STATS.launches += 1
    return out


def _lora_arg(lora, K: int, N: int, name: str):
    """lora = None or (down [R, K], up [N, R]) fp16 CUDA tensors (lora.pack) -> (VtmLora or None, R)."""
    if lora is None:
        return None, 0
    down, up = lora
    _require(down, torch.float16, f"{name} lora down")
    _require(up, torch.float16, f"{name} lora up")
    R = down.shape[0]
    if tuple(down.shape) != (R, K) or tuple(up.shape) != (N, R) or R % 8 != 0:
        raise RuntimeError(f"vidtome_b200: {name} LoRA must be down [R, {K}] and up [{N}, R] with R % 8 == 0, got "
                           f"{tuple(down.shape)} and {tuple(up.shape)}")
    return _lib.VtmLora(down.data_ptr(), up.data_ptr(), R), R


def _lora_ref(desc):
    return None if desc is None else C.byref(desc)


def linear(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """D = A W^T (+ bias) on the wgmma GEMM.  a [M, K], w [N, K] fp16."""
    _require(a, torch.float16, "a")
    _require(w, torch.float16, "w")
    M, K = a.shape
    N = w.shape[0]
    d = torch.empty((M, N), dtype=torch.float16, device=a.device)
    if bias is not None:
        _require(bias, torch.float16, "bias")
    check(_lib.load().vtm_linear_f16(a.data_ptr(), w.data_ptr(), _ptr(bias), M, N, K, d.data_ptr(), N, _stream()),
          "vtm_linear_f16")
    STATS.launches += 1
    return d


def linear_residual(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], resid: torch.Tensor,
                    lora=None) -> torch.Tensor:
    """D = (A W^T + bias) + resid, with torch's fp16 roundings (`lin(x) + h`).  a [M, K], w [N, K], resid [M, N].
    lora = (down [R, K], up [N, R]) adds the LoRA term T up^T, T = fp16(A down^T), inside the projection's sum."""
    _require(a, torch.float16, "a")
    _require(w, torch.float16, "w")
    _require(resid, torch.float16, "resid")
    M, K = a.shape
    N = w.shape[0]
    if tuple(resid.shape) != (M, N):
        raise RuntimeError("linear_residual: resid must be [M, N]")
    d = torch.empty((M, N), dtype=torch.float16, device=a.device)
    if bias is not None:
        _require(bias, torch.float16, "bias")
    desc, R = _lora_arg(lora, K, N, "linear_residual")
    if desc is not None:
        lib = _lib.load()
        ws_bytes = lib.vtm_linear_lora_workspace_bytes(M, R)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=a.device)
        with _Timed("FF2", 2.0 * M * (N + R) * K + 2.0 * M * N * R, 2.0 * (M * K + N * K + 2 * M * N)):
            check(lib.vtm_linear_lora_f16(a.data_ptr(), w.data_ptr(), _ptr(bias), resid.data_ptr(), N, C.byref(desc), M,
                                          N, K, d.data_ptr(), N, ws.data_ptr(), ws_bytes, _stream()),
                  "vtm_linear_lora_f16")
        STATS.launches += 2
        return d
    with _Timed("FF2", 2.0 * M * N * K, 2.0 * (M * K + N * K + 2 * M * N)):
        check(_lib.load().vtm_linear_residual_f16(a.data_ptr(), w.data_ptr(), _ptr(bias), resid.data_ptr(), N, M, N, K,
                                                  d.data_ptr(), N, _stream()), "vtm_linear_residual_f16")
    STATS.launches += 1
    return d


def interleave_geglu(w: torch.Tensor, bias: Optional[torch.Tensor]):
    """Row order vtm_linear_geglu_f16 expects: groups of 32 value rows followed by their 32 gate rows."""
    N, K = w.shape
    No = N // 2
    if No % 32 != 0:
        raise RuntimeError("geglu: inner width must be a multiple of 32")
    wi = torch.stack([w[:No].reshape(No // 32, 32, K), w[No:].reshape(No // 32, 32, K)], dim=1).reshape(N, K).contiguous()
    bi = None
    if bias is not None:
        bi = torch.stack([bias[:No].reshape(No // 32, 32), bias[No:].reshape(No // 32, 32)], dim=1).reshape(N).contiguous()
    return wi, bi


def linear_geglu(a: torch.Tensor, w_il: torch.Tensor, bias_il: Optional[torch.Tensor], lora=None) -> torch.Tensor:
    """GEGLU projection: [h | gate] = A W^T + b, D = h * gelu(gate).  w_il / bias_il interleaved (interleave_geglu).
    lora = (down [R, K], up [N, R]) with up's rows interleaved like w_il: the LoRA term joins the projection's sum."""
    _require(a, torch.float16, "a")
    _require(w_il, torch.float16, "w_il")
    M, K = a.shape
    N = w_il.shape[0]
    d = torch.empty((M, N // 2), dtype=torch.float16, device=a.device)
    if bias_il is not None:
        _require(bias_il, torch.float16, "bias_il")
    desc, R = _lora_arg(lora, K, N, "linear_geglu")
    if desc is not None:
        lib = _lib.load()
        ws_bytes = lib.vtm_linear_lora_workspace_bytes(M, R)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=a.device)
        with _Timed("FF1", 2.0 * M * (N + R) * K + 2.0 * M * N * R, 2.0 * (M * K + N * K + M * N // 2)):
            check(lib.vtm_linear_geglu_lora_f16(a.data_ptr(), w_il.data_ptr(), _ptr(bias_il), C.byref(desc), M, N, K,
                                                d.data_ptr(), N // 2, ws.data_ptr(), ws_bytes, _stream()),
                  "vtm_linear_geglu_lora_f16")
        STATS.launches += 2
        return d
    with _Timed("FF1", 2.0 * M * N * K, 2.0 * (M * K + N * K + M * N // 2)):
        check(_lib.load().vtm_linear_geglu_f16(a.data_ptr(), w_il.data_ptr(), _ptr(bias_il), M, N, K, d.data_ptr(), N // 2,
                                               _stream()), "vtm_linear_geglu_f16")
    STATS.launches += 1
    return d


def layer_norm(x: torch.Tensor, ln) -> torch.Tensor:
    """Plain LayerNorm over the last dim of x [M, C] through the KC kernel with an identity map (torch half semantics)."""
    M, Cc = x.shape
    return gather_rows(x.view(1, M, Cc), None, L=M, ln=ln).view(M, Cc)


def attention(x: torch.Tensor, w_qkv: torch.Tensor, w_o: torch.Tensor, b_o: Optional[torch.Tensor], heads: int,
              scale: float, shared_qk: bool = False, seq_len: Optional[torch.Tensor] = None, lora_qkv=None,
              lora_o=None) -> torch.Tensor:
    """KD.  x [B, L, C] fp16 -> [B, L, C].  shared_qk: PnP injection — the attention map of sample 0 for every sample.
    seq_len: a 1-element int32 CUDA tensor; the sequence is then the first seq_len rows of x (rows past it must be
    finite) and only those rows of the result are defined.  lora_qkv = (down [R, C], up [3C, R]) and lora_o =
    (down [R, C], up [C, R]): LoRA terms of the QKV GEMM and of to_out[0] (vtm_attention_lora)."""
    _require(x, torch.float16, "x")
    _require(w_qkv, torch.float16, "w_qkv")
    _require(w_o, torch.float16, "w_o")
    B, L, Cc = x.shape
    lib = _lib.load()
    if lora_qkv is not None or lora_o is not None:
        dq, rq = _lora_arg(lora_qkv, Cc, 3 * Cc, "attention qkv")
        do, ro = _lora_arg(lora_o, Cc, Cc, "attention out")
        ws_bytes = lib.vtm_attention_lora_workspace_bytes(B, L, Cc, heads, rq, ro)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        y = torch.empty_like(x)
        if seq_len is not None:
            _require(seq_len, torch.int32, "seq_len")
        flops = 4.0 * B * L * L * Cc + 8.0 * B * L * Cc * Cc + 8.0 * B * L * Cc * (rq + ro)
        with _Timed("KD", flops, 4.0 * B * L * Cc + 8.0 * Cc * Cc):
            check(lib.vtm_attention_lora(x.data_ptr(), w_qkv.data_ptr(), w_o.data_ptr(), _ptr(b_o), _lora_ref(dq),
                                         _lora_ref(do), B, L, Cc, heads, float(scale), 1 if shared_qk else 0,
                                         _ptr(seq_len), y.data_ptr(), ws.data_ptr(), ws_bytes, _stream()),
                  "vtm_attention_lora")
        STATS.launches += 3 + (rq > 0) + (ro > 0)
        return y
    ws_bytes = lib.vtm_attention_workspace_bytes(B, L, Cc, heads)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
    y = torch.empty_like(x)
    if seq_len is not None:
        _require(seq_len, torch.int32, "seq_len")
        with _Timed("KD", 4.0 * B * L * L * Cc + 8.0 * B * L * Cc * Cc, 4.0 * B * L * Cc + 8.0 * Cc * Cc):
            check(lib.vtm_attention_dev(x.data_ptr(), w_qkv.data_ptr(), w_o.data_ptr(), _ptr(b_o), B, L, Cc, heads,
                                        float(scale), 1 if shared_qk else 0, seq_len.data_ptr(), y.data_ptr(),
                                        ws.data_ptr(), ws_bytes, _stream()), "vtm_attention_dev")
        STATS.launches += 3
        return y
    with _Timed("KD", 4.0 * B * L * L * Cc + 8.0 * B * L * Cc * Cc, 4.0 * B * L * Cc + 8.0 * Cc * Cc):
        check(lib.vtm_attention_ex(x.data_ptr(), w_qkv.data_ptr(), w_o.data_ptr(), _ptr(b_o), B, L, Cc, heads,
                                   float(scale), 1 if shared_qk else 0, y.data_ptr(), ws.data_ptr(), ws_bytes, _stream()),
              "vtm_attention_ex")
    STATS.launches += 3
    return y


def ddim_table(coefficients) -> torch.Tensor:
    """[n_steps, 4] fp32 rows (a, r, c, d) for ddim_update from python-float (a, b, c, d) per step: r = 1 / b in double,
    rounded once to fp32, which is the reciprocal torch multiplies by for `half_tensor / b` (div_true_kernel_cuda)."""
    return torch.tensor([(a, 1.0 / b, c, d) for a, b, c, d in coefficients], dtype=torch.float32)


def attention_residual(x: torch.Tensor, w_qkv: torch.Tensor, w_o: torch.Tensor, b_o: Optional[torch.Tensor],
                       heads: int, scale: float, resid: torch.Tensor, lora_qkv=None, lora_o=None) -> torch.Tensor:
    """KD with the residual in the out projection: attention(x, ...) + resid, bit for bit as torch's half add, for an
    unmerged block (`attn1(norm1(h)) + h`).  x, resid [B, L, C] fp16; lora_qkv / lora_o as in `attention`."""
    _require(x, torch.float16, "x")
    _require(w_qkv, torch.float16, "w_qkv")
    _require(w_o, torch.float16, "w_o")
    _require(resid, torch.float16, "resid")
    B, L, Cc = x.shape
    if resid.shape != x.shape:
        raise RuntimeError(f"attention_residual: resid {tuple(resid.shape)} must be shaped like x {tuple(x.shape)}")
    lib = _lib.load()
    dq, rq = _lora_arg(lora_qkv, Cc, 3 * Cc, "attention qkv")
    do, ro = _lora_arg(lora_o, Cc, Cc, "attention out")
    ws_bytes = lib.vtm_attention_lora_workspace_bytes(B, L, Cc, heads, rq, ro)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
    y = torch.empty_like(x)
    flops = 4.0 * B * L * L * Cc + 8.0 * B * L * Cc * Cc + 8.0 * B * L * Cc * (rq + ro)
    with _Timed("KD", flops, 6.0 * B * L * Cc + 8.0 * Cc * Cc):
        check(lib.vtm_attention_residual(x.data_ptr(), w_qkv.data_ptr(), w_o.data_ptr(), _ptr(b_o), resid.data_ptr(),
                                         _lora_ref(dq), _lora_ref(do), B, L, Cc, heads, float(scale), y.data_ptr(),
                                         ws.data_ptr(), ws_bytes, _stream()), "vtm_attention_residual")
    STATS.launches += 3 + (rq > 0) + (ro > 0)
    return y


def ddim_update(x: torch.Tensor, eps: torch.Tensor, coef: torch.Tensor, step: torch.Tensor,
                slots: Optional[torch.Tensor] = None, traj: Optional[torch.Tensor] = None) -> torch.Tensor:
    """KI, in place on x: with s = step[0] and (a, r, c, d) = coef[s], x <- c * ((x - a * eps) * r) + d * eps in torch's
    CUDA half roundings, and traj[slots[s]] <- x when slots[s] >= 0.  r = float(1.0 / b) (ddim_table) reproduces torch's
    `/ b`.  x, eps fp16 of one shape; coef [n_steps, 4] fp32;
    step a 1-element int32 tensor (read on the device, not advanced); slots [n_steps] int32 with traj [n_slots, *x.shape]
    fp16, or both None."""
    _require(x, torch.float16, "x")
    _require(eps, torch.float16, "eps")
    _require(coef, torch.float32, "coef")
    _require(step, torch.int32, "step")
    if eps.shape != x.shape:
        raise RuntimeError(f"ddim_update: eps {tuple(eps.shape)} must be shaped like x {tuple(x.shape)}")
    if coef.dim() != 2 or coef.shape[1] != 4 or step.numel() != 1:
        raise RuntimeError("ddim_update: coef must be [n_steps, 4] and step a 1-element tensor")
    if (slots is None) != (traj is None):
        raise RuntimeError("ddim_update: slots and traj go together")
    n_slots = 0
    if slots is not None:
        _require(slots, torch.int32, "slots")
        _require(traj, torch.float16, "traj")
        if tuple(slots.shape) != (coef.shape[0],) or traj.shape[1:] != x.shape:
            raise RuntimeError(f"ddim_update: slots must be [{coef.shape[0]}] and traj [n_slots, {tuple(x.shape)}]")
        n_slots = traj.shape[0]
    n = x.numel()
    with _Timed("KI", 6.0 * n, 2.0 * n * (3 + (slots is not None))):
        check(_lib.load().vtm_ddim_update_f16(x.data_ptr(), eps.data_ptr(), n, coef.data_ptr(), _ptr(slots),
                                              step.data_ptr(), coef.shape[0], _ptr(traj), n_slots, _stream()),
              "vtm_ddim_update_f16")
    STATS.launches += 1
    return x


def cross_attention(x: torch.Tensor, ctx: torch.Tensor, w_q: torch.Tensor, w_kv: torch.Tensor, w_o: torch.Tensor,
                    b_o: Optional[torch.Tensor], heads: int, scale: float, resid: Optional[torch.Tensor] = None,
                    lora_q=None, lora_kv=None, lora_o=None) -> torch.Tensor:
    """attn2 of the block: x [B, Lq, C] queries, ctx [B, Lk, Cctx] keys/values; returns o Wo^T + bo (+ resid).
    lora_q = (down [R, C], up [C, R]), lora_kv = (down [R, Cctx], up [2C, R]), lora_o = (down [R, C], up [C, R]): LoRA
    terms of to_q, to_k / to_v and to_out[0] (vtm_cross_attention_lora)."""
    _require(x, torch.float16, "x")
    _require(ctx, torch.float16, "ctx")
    _require(w_q, torch.float16, "w_q")
    _require(w_kv, torch.float16, "w_kv")
    _require(w_o, torch.float16, "w_o")
    B, Lq, Cc = x.shape
    Lk, Cctx = ctx.shape[1], ctx.shape[2]
    if ctx.shape[0] != B:
        raise RuntimeError("cross_attention: x and ctx must have the same number of items")
    if resid is not None:
        _require(resid, torch.float16, "resid")
    lib = _lib.load()
    flops = 4.0 * B * Lq * Lk * Cc + 4.0 * B * Lq * Cc * Cc + 4.0 * B * Lk * Cctx * Cc
    if lora_q is not None or lora_kv is not None or lora_o is not None:
        dq, rq = _lora_arg(lora_q, Cc, Cc, "cross_attention q")
        dkv, rkv = _lora_arg(lora_kv, Cctx, 2 * Cc, "cross_attention kv")
        do, ro = _lora_arg(lora_o, Cc, Cc, "cross_attention out")
        ws_bytes = lib.vtm_cross_attention_lora_workspace_bytes(B, Lq, Lk, Cc, heads, rq, rkv, ro)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        y = torch.empty_like(x)
        flops += 4.0 * B * Lq * Cc * (rq + ro) + 2.0 * B * Lk * (Cctx + 2 * Cc) * rkv
        with _Timed("XA", flops, 2.0 * B * Lq * Cc * (3 if resid is not None else 2)):
            check(lib.vtm_cross_attention_lora(x.data_ptr(), ctx.data_ptr(), w_q.data_ptr(), w_kv.data_ptr(),
                                               w_o.data_ptr(), _ptr(b_o), _ptr(resid), _lora_ref(dq), _lora_ref(dkv),
                                               _lora_ref(do), B, Lq, Lk, Cc, Cctx, heads, float(scale), y.data_ptr(),
                                               ws.data_ptr(), ws_bytes, _stream()), "vtm_cross_attention_lora")
        STATS.launches += 4 + (rq > 0) + (rkv > 0) + (ro > 0)
        return y
    ws_bytes = lib.vtm_cross_attention_workspace_bytes(B, Lq, Lk, Cc, heads)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
    y = torch.empty_like(x)
    with _Timed("XA", flops, 2.0 * B * Lq * Cc * (3 if resid is not None else 2)):
        check(lib.vtm_cross_attention(x.data_ptr(), ctx.data_ptr(), w_q.data_ptr(), w_kv.data_ptr(), w_o.data_ptr(), _ptr(b_o),
                                      _ptr(resid), B, Lq, Lk, Cc, Cctx, heads, float(scale), y.data_ptr(), ws.data_ptr(),
                                      ws_bytes, _stream()), "vtm_cross_attention")
    STATS.launches += 4
    return y


def resnet_tail(h: torch.Tensor, shortcut: torch.Tensor, num_inputs: int, output_scale_factor: float, inject: bool,
                out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """KT.  out = (shortcut + h') / output_scale_factor, h' = h with the first third (num_inputs = 3) or half (2) of the
    batch copied over the next two (one) when `inject` (utils/pnp_utils.py:146-162).  shortcut [num_inputs * n, ...]
    fp16; h like shortcut, or only its n source samples when injecting."""
    _require(h, torch.float16, "h")
    _require(shortcut, torch.float16, "shortcut")
    B = shortcut.shape[0]
    if num_inputs not in (1, 2, 3) or B % num_inputs:
        raise RuntimeError(f"vidtome_b200: resnet_tail needs a batch of num_inputs * n samples, num_inputs in 1..3 "
                           f"(got batch {B}, num_inputs {num_inputs})")
    n = B // num_inputs
    if h.shape[1:] != shortcut.shape[1:] or h.shape[0] not in ((n, B) if inject else (B,)):
        raise RuntimeError(f"vidtome_b200: resnet_tail: h {tuple(h.shape)} does not fit shortcut {tuple(shortcut.shape)}"
                           f" (inject={bool(inject)})")
    if out is None:
        out = torch.empty_like(shortcut)
    else:
        _require(out, torch.float16, "out")
        if out.shape != shortcut.shape:
            raise RuntimeError(f"vidtome_b200: resnet_tail: out {tuple(out.shape)} != shortcut {tuple(shortcut.shape)}")
    E = shortcut[0].numel()
    nbytes = 2.0 * E * (2 * B + (n if inject else B))
    with _Timed("KT", 0.0, nbytes):
        check(_lib.load().vtm_resnet_tail_f16(h.data_ptr(), shortcut.data_ptr(), out.data_ptr(), n, num_inputs, E,
                                              float(output_scale_factor), int(bool(inject)), _stream()),
              "vtm_resnet_tail_f16")
    STATS.launches += 1
    return out


def keys_to_score_arg(keys: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Unpack KA keys on the device with torch integer ops (test / debugging helper)."""
    o = (keys >> 32) & 0xFFFF
    hb = torch.where((o & 0x8000) != 0, o & 0x7FFF, o ^ 0xFFFF)
    score = torch.where(hb >= 0x8000, hb - 0x10000, hb).to(torch.int16).view(torch.float16)
    arg = 0xFFFFFFFF - (keys & 0xFFFFFFFF)
    return score, arg
