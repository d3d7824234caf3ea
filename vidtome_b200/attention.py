"""Host side of KD: run a diffusers-style `Attention` module's self-attention on merged tokens through
the CUDA kernel (`vtm_attention`) instead of the module's own forward.

`ToMeBlock.forward` uses this only for a stock attention module (see patch._plain_attention_module);
anything customised (PnP's replaced forward, attention masks, cross_attention_kwargs, added KV
projections) goes through the module itself, exactly as the reference does at patch.py:157-162.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import _lib, lora, ops

# Switched on once the attention kernel is built into the library.
ENABLED = True

# Largest head_dim that runs in the library (self-attention of merged blocks and cross-attention); wider modules run
# their own forward.  The flash kernel is built up to 160 (KERNEL_MAX_HEAD_DIM): setting 160 here also routes SD1.5's
# 1280-channel blocks (8 heads of 160) through it.  Read on every dispatch, so it may be changed at any time.
MAX_HEAD_DIM = 128
KERNEL_MAX_HEAD_DIM = 160


def max_head_dim() -> int:
    """MAX_HEAD_DIM, checked: a positive multiple of 8 no larger than KERNEL_MAX_HEAD_DIM."""
    v = MAX_HEAD_DIM
    if isinstance(v, bool) or not isinstance(v, int) or v <= 0 or v % 8 != 0 or v > KERNEL_MAX_HEAD_DIM:
        raise ValueError(f"vidtome_b200.attention.MAX_HEAD_DIM = {v!r}: must be a positive multiple of 8 and at most "
                         f"{KERNEL_MAX_HEAD_DIM}, the widest head the flash-attention kernel is built for")
    return v


def _packed(attn: torch.nn.Module, like: torch.Tensor):
    """(w_qkv, w_o, b_o, lora_qkv, lora_o): the tensors of _packed_weights and the LoRA packs (lora.pack) of the QKV GEMM
    and of to_out[0] (None without adapters) — cached on the module, refreshed when a weight or adapter tensor is replaced
    or modified in place, a scale changes or another set of adapters becomes active (lora.tag).  Under CUDA-graph replay
    nothing is re-read: LoRA changes after capture are as static as weight changes."""
    parts = [lora.linear_parts(m) for m in (attn.to_q, attn.to_k, attn.to_v, attn.to_out[0])]
    tag = lora.tag(parts) + (like.device,)
    cache = getattr(attn, "_vtm_packed", None)
    if cache is None or cache[0] != tag:
        dev = like.device
        w_qkv = torch.cat([p[0] for p in parts[:3]], dim=0).detach().to(device=dev, dtype=torch.float16).contiguous()
        w_o = parts[3][0].detach().to(device=dev, dtype=torch.float16).contiguous()
        b_o = None if parts[3][1] is None else parts[3][1].detach().to(device=dev, dtype=torch.float16).contiguous()
        cache = (tag, w_qkv, w_o, b_o, lora.pack(parts[:3], dev), lora.pack(parts[3:], dev))
        attn._vtm_packed = cache
    return cache[1:]


def _packed_weights(attn: torch.nn.Module, like: torch.Tensor):
    """[3C, C] fp16 (Wq | Wk | Wv), Wo [C, C], bo [C] — cached on the module, refreshed when a weight tensor is replaced
    or modified in place."""
    return _packed(attn, like)[:3]


def _packed_lora(attn: torch.nn.Module, like: torch.Tensor):
    """(lora_qkv, lora_o): the LoRA packs of the QKV GEMM and of to_out[0], None where there is no adapter."""
    return _packed(attn, like)[3:]


def self_attention(attn: torch.nn.Module, x: torch.Tensor, shared_qk: bool = False,
                   seq_len: Optional[torch.Tensor] = None) -> torch.Tensor:
    """softmax(q k^T * scale) v with q,k,v = to_q/to_k/to_v(x), then to_out[0] (utils/pnp_utils.py:47-95).
    shared_qk: PnP injection — q and k of sample 0 for every sample (utils/pnp_utils.py:57-68,87-91).
    seq_len: the sequence is the first seq_len (a 1-element int32 CUDA tensor) rows of x (GlobalTokenStore stage)."""
    w_qkv, w_o, b_o, lora_qkv, lora_o = _packed(attn, x)
    heads = int(attn.heads)
    scale = float(getattr(attn, "scale", (x.shape[-1] // heads) ** -0.5))
    return ops.attention(x, w_qkv, w_o, b_o, heads, scale, shared_qk=shared_qk, seq_len=seq_len, lora_qkv=lora_qkv,
                         lora_o=lora_o)


def self_attention_residual(attn: torch.nn.Module, x: torch.Tensor, resid: torch.Tensor) -> torch.Tensor:
    """attn(x) + resid for an unmerged block (vidtome/patch.py:157-169 with do_nothing merges) through
    vtm_attention_residual: the same kernels as self_attention, the add in the out projection's epilogue."""
    w_qkv, w_o, b_o, lora_qkv, lora_o = _packed(attn, x)
    heads = int(attn.heads)
    scale = float(getattr(attn, "scale", (x.shape[-1] // heads) ** -0.5))
    return ops.attention_residual(x, w_qkv, w_o, b_o, heads, scale, resid, lora_qkv=lora_qkv, lora_o=lora_o)


def cross_attention_eligible(attn: torch.nn.Module, ctx: torch.Tensor) -> bool:
    """True if `attn` is a stock diffusers-style cross-attention (to_q [C, C], to_k / to_v [C, Cctx] without bias,
    to_out = [Linear, Dropout], default processor, no hooks / overrides / options that alter the math).  The projections
    may be LoRA-adapted in any form lora.linear_parts reads."""
    from .patch import _PLAIN_PROCESSORS
    if attn is None or "forward" in vars(attn) or not isinstance(ctx, torch.Tensor) or ctx.dim() != 3:
        return False
    need = ("to_q", "to_k", "to_v", "to_out", "heads")
    if not all(hasattr(attn, n) for n in need):
        return False
    to_out = attn.to_out
    if not isinstance(to_out, (torch.nn.ModuleList, torch.nn.Sequential)) or len(to_out) < 1:
        return False
    linears = (attn.to_q, attn.to_k, attn.to_v, to_out[0])
    parts = [lora.linear_parts(m) for m in linears]
    if any(p is None for p in parts) or any(p[1] is not None for p in parts[:3]):
        return False
    for m in (attn,) + linears + tuple(to_out[1:]):
        if m._forward_hooks or m._forward_pre_hooks:
            return False
    for extra in to_out[1:]:
        if not isinstance(extra, torch.nn.Dropout) or (extra.p > 0 and extra.training):
            return False
    proc = getattr(attn, "processor", None)
    if proc is not None and type(proc).__name__ not in _PLAIN_PROCESSORS:
        return False
    for name, bad in (("group_norm", None), ("spatial_norm", None), ("norm_cross", None), ("added_kv_proj_dim", None)):
        if getattr(attn, name, None) not in (None, False):
            return False
    if getattr(attn, "residual_connection", False) or getattr(attn, "rescale_output_factor", 1.0) != 1.0:
        return False
    wq, wk, wv, wo = (p[0] for p in parts)
    C = wq.shape[1]
    Cctx = wk.shape[1]
    if wq.shape != (C, C) or wk.shape != (C, Cctx) or wv.shape != (C, Cctx):
        return False
    if wo.shape != (C, C) or ctx.shape[-1] != Cctx or Cctx % 8 != 0:
        return False
    if wq.dtype != torch.float16 or not wq.is_cuda or ctx.dtype != torch.float16:
        return False
    d = C // int(attn.heads)
    return d * int(attn.heads) == C and d % 8 == 0 and d <= max_head_dim()


def cross_attention_residual(attn: torch.nn.Module, x: torch.Tensor, ctx: torch.Tensor, resid: torch.Tensor) -> torch.Tensor:
    """attn2(x, encoder_hidden_states=ctx) + resid (vidtome/patch.py:171-185) through vtm_cross_attention."""
    parts = [lora.linear_parts(m) for m in (attn.to_q, attn.to_k, attn.to_v, attn.to_out[0])]
    tag = lora.tag(parts)
    cache = getattr(attn, "_vtm_packed_x", None)
    if cache is None or cache[0] != tag:
        (wq, _, _), (wk, _, _), (wv, _, _), (wo, bo, _) = parts
        w_kv = torch.cat([wk, wv], dim=0).detach().contiguous()
        dev = wq.device
        cache = (tag, wq.detach().contiguous(), w_kv, wo.detach().contiguous(),
                 None if bo is None else bo.detach().contiguous(),
                 lora.pack(parts[:1], dev), lora.pack(parts[1:3], dev), lora.pack(parts[3:], dev))
        attn._vtm_packed_x = cache
    _, w_q, w_kv, w_o, b_o, lora_q, lora_kv, lora_o = cache
    heads = int(attn.heads)
    scale = float(getattr(attn, "scale", (x.shape[-1] // heads) ** -0.5))
    return ops.cross_attention(x.contiguous(), ctx.contiguous(), w_q, w_kv, w_o, b_o, heads, scale, resid=resid.contiguous(),
                               lora_q=lora_q, lora_kv=lora_kv, lora_o=lora_o)
