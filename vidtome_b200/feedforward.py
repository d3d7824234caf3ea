"""Host side of the block's feed-forward on the tensor cores (SURVEY §8 row f3; vidtome/patch.py:187-199).

`ToMeBlock.forward` uses this for a stock GEGLU feed-forward — diffusers' `FeedForward` with
`net = [GEGLU(dim, 4 dim), Dropout, Linear(4 dim, dim)]`, or the skeleton's stand-in with the same two Linear layers —
preceded by a plain LayerNorm.  Its two Linear layers may be LoRA-adapted in any form lora.linear_parts reads: the
low-rank terms join the projections as extra K steps.  Anything else customised (other activations, hooks, AdaNorm)
goes through the modules themselves exactly as the reference does.  Three launches: LayerNorm (row kernel), GEGLU projection
(wgmma GEMM with the gate fused into its epilogue: the [M, 8 dim] projection is never written), output projection with
bias and residual fused into its epilogue.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import lora, ops


def geglu_parts(ff: torch.nn.Module) -> Optional[Tuple[torch.nn.Linear, torch.nn.Linear]]:
    """(projection Linear dim -> 2 inner, output Linear inner -> dim) of a stock GEGLU feed-forward, else None."""
    if ff is None or "forward" in vars(ff) or ff._forward_hooks or ff._forward_pre_hooks:
        return None
    proj = out = None
    net = getattr(ff, "net", None)
    if isinstance(net, (torch.nn.ModuleList, torch.nn.Sequential)) and len(net) >= 2:
        act = net[0]
        if type(act).__name__ != "GEGLU" or not hasattr(act, "proj") or act._forward_hooks or act._forward_pre_hooks:
            return None
        if getattr(act, "approximate", "none") not in ("none", None):
            return None
        proj = act.proj
        rest = list(net[1:])
        linears = [m for m in rest if lora.linear_parts(m) is not None]
        drops = [m for m in rest if isinstance(m, torch.nn.Dropout)]
        if len(linears) != 1 or len(linears) + len(drops) != len(rest):
            return None
        if any(m.p > 0 and m.training for m in drops):
            return None
        out = linears[0]
    elif type(ff).__name__ == "GEGLUFeedForward" and hasattr(ff, "proj") and hasattr(ff, "out"):
        proj, out = ff.proj, ff.out
    else:
        return None
    proj_parts, out_parts = lora.linear_parts(proj), lora.linear_parts(out)
    if proj_parts is None or out_parts is None:
        return None
    inner, dim = out_parts[0].shape[1], out_parts[0].shape[0]
    if proj_parts[0].shape != (2 * inner, dim) or inner % 32 != 0 or dim % 8 != 0:
        return None
    if proj_parts[0].dtype != torch.float16 or not proj_parts[0].is_cuda:
        return None
    return proj, out


def _packed_all(ff: torch.nn.Module, proj: torch.nn.Module, out: torch.nn.Module):
    """Interleaved GEGLU weight and bias, output weight and bias, and the LoRA packs of both projections (the GEGLU one
    with its up matrix interleaved like the weight rows) — cached on the module as attention._packed does."""
    parts = [lora.linear_parts(proj), lora.linear_parts(out)]
    tag = lora.tag(parts)
    cache = getattr(ff, "_vtm_packed", None)
    if cache is None or cache[0] != tag:
        (pw, pb, _), (ow, ob, _) = parts
        w_il, b_il = ops.interleave_geglu(pw.detach(), None if pb is None else pb.detach())
        lora_1 = lora.pack(parts[:1], pw.device)
        if lora_1 is not None:
            lora_1 = (lora_1[0], ops.interleave_geglu(lora_1[1], None)[0])
        cache = (tag, w_il, b_il, ow.detach().contiguous(), None if ob is None else ob.detach().contiguous(),
                 lora_1, lora.pack(parts[1:], pw.device))
        ff._vtm_packed = cache
    return cache[1:]


def _packed(ff: torch.nn.Module, proj: torch.nn.Module, out: torch.nn.Module):
    """(interleaved GEGLU weight, its bias, output weight, output bias), cached on the module."""
    return _packed_all(ff, proj, out)[:4]


def _packed_lora(ff: torch.nn.Module, proj: torch.nn.Module, out: torch.nn.Module):
    """(lora of the GEGLU projection with its up matrix interleaved, lora of the output projection), None where there is
    no adapter."""
    return _packed_all(ff, proj, out)[4:]


def feed_forward_residual(ff: torch.nn.Module, parts, ln, hidden_states: torch.Tensor) -> torch.Tensor:
    """hidden_states + ff(LayerNorm(hidden_states)) for a stock GEGLU feed-forward (patch.py:187-199).
    `ln` = (weight, bias, eps) of norm3; hidden_states [(B F), T, C] fp16 CUDA."""
    proj, out = parts
    w_il, b_il, w_o, b_o, lora_1, lora_2 = _packed_all(ff, proj, out)
    shape = hidden_states.shape
    h2 = hidden_states.contiguous().view(-1, shape[-1])
    n3 = ops.layer_norm(h2, ln)
    u = ops.linear_geglu(n3, w_il, b_il, lora=lora_1)
    return ops.linear_residual(u, w_o, b_o, h2, lora=lora_2).view(shape)
