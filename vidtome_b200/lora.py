"""LoRA-adapted projections on the library's GEMMs.

The reference loads a LoRA with `pipe.load_lora_weights` (generate.py:93-94).  diffusers then wraps each attention and
feed-forward projection in one of two ways, and a wrapped layer computes

    y = x W^T + b + sum_a s_a (x A_a^T) B_a^T

- the peft backend: a `lora.Linear` holding `base_layer`, ModuleDicts `lora_A` / `lora_B`, `scaling`, ...;
- without peft: a `LoRACompatibleLinear` (an nn.Linear subclass) whose `lora_layer` is a `LoRALinearLayer` (or None).

`linear_parts` reads any of these (and an exact nn.Linear) as (W, b, [(A, B, s), ...]); `pack` stacks the adapters of
the projections of one GEMM into the down matrix D [R, K] and the up matrix U [N, R] of vtm_lora_t, so that the library
computes fp16([x | fp16(x D^T)] [W | U]^T + b): the projection GEMM with R more K steps (include/vidtome_b200.h).

Anything else — hooks or an instance-level forward on a wrapper or one of its layers, DoRA, `lora_bias`, active dropout,
fan-in/fan-out weights — gives None, and the block then calls the module itself, exactly as before.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from .utils import isinstance_str

Adapter = Tuple[torch.Tensor, torch.Tensor, float]          # (A [r, K], B [N, r], scale)
Parts = Tuple[torch.Tensor, Optional[torch.Tensor], List[Adapter]]

_ADAPTER_DTYPES = (torch.float16, torch.float32)


def _plain(*mods) -> bool:
    """No forward hooks and no instance-level forward on any of `mods` (None entries are skipped)."""
    for m in mods:
        if m is None:
            continue
        if "forward" in vars(m) or m._forward_hooks or m._forward_pre_hooks or getattr(m, "_forward_hooks_with_kwargs", None):
            return False
    return True


def _adapter(a_mod, b_mod, scale, weight: torch.Tensor) -> Optional[Adapter]:
    """(A, B, s) of a pair of bias-free nn.Linear feeding `weight`'s outputs from its inputs, else None."""
    if type(a_mod) is not nn.Linear or type(b_mod) is not nn.Linear or a_mod.bias is not None or b_mod.bias is not None:
        return None
    if not _plain(a_mod, b_mod):
        return None
    A, B = a_mod.weight, b_mod.weight
    N, K = weight.shape
    r = A.shape[0]
    if tuple(A.shape) != (r, K) or tuple(B.shape) != (N, r) or r == 0:
        return None
    if A.dtype not in _ADAPTER_DTYPES or B.dtype not in _ADAPTER_DTYPES:
        return None
    if A.device != weight.device or B.device != weight.device:
        return None
    return A, B, float(scale)


def _diffusers_parts(m) -> Optional[Parts]:
    """LoRACompatibleLinear: super().forward(x) + scale * lora_layer(x), scale = 1 on the block's call path."""
    if not _plain(m):
        return None
    layer = m.lora_layer
    if layer is None:
        return m.weight, m.bias, []
    if not isinstance_str(layer, "LoRALinearLayer") or not _plain(layer):
        return None
    down, up = getattr(layer, "down", None), getattr(layer, "up", None)
    if down is None or up is None:
        return None
    alpha = getattr(layer, "network_alpha", None)
    rank = getattr(layer, "rank", down.weight.shape[0])
    ad = _adapter(down, up, 1.0 if alpha is None else alpha / rank, m.weight)
    return None if ad is None else (m.weight, m.bias, [ad])


def _active_adapters(m) -> Optional[List[str]]:
    names = getattr(m, "active_adapters", None)
    if names is None:
        names = getattr(m, "active_adapter", None)
    if isinstance(names, str):
        return [names]
    if isinstance(names, (list, tuple)) and all(isinstance(n, str) for n in names):
        return list(names)
    return None


def _peft_parts(m) -> Optional[Parts]:
    """peft lora.Linear: base_layer(x) + sum over active adapters of lora_B(lora_A(dropout(x))) * scaling."""
    base = m.base_layer
    if type(base) is not nn.Linear or not _plain(m, base) or getattr(m, "fan_in_fan_out", False):
        return None
    disabled, merged = bool(getattr(m, "disable_adapters", False)), bool(getattr(m, "merged", False))
    if disabled and merged:
        return None                 # peft unmerges the adapters out of the base weight before it runs the base layer
    if disabled or merged:
        return base.weight, base.bias, []
    lora_A, lora_B, scaling = m.lora_A, m.lora_B, m.scaling
    if not isinstance(lora_A, nn.ModuleDict) or not isinstance(lora_B, nn.ModuleDict):
        return None
    names = _active_adapters(m)
    if names is None:
        return None
    dropout = getattr(m, "lora_dropout", None) or {}
    use_dora = getattr(m, "use_dora", None) or {}
    lora_bias = getattr(m, "lora_bias", None) or {}
    adapters = []
    for name in names:
        if name not in lora_A:
            continue                                    # as peft: an active name without weights here is skipped
        if name not in lora_B or name not in scaling or use_dora.get(name, False) or lora_bias.get(name, False):
            return None
        drop = dropout[name] if name in dropout else None
        if drop is not None:
            if not _plain(drop):
                return None
            if type(drop) is not nn.Identity and not (type(drop) is nn.Dropout and (drop.p == 0 or not drop.training)):
                return None
        ad = _adapter(lora_A[name], lora_B[name], scaling[name], base.weight)
        if ad is None:
            return None
        adapters.append(ad)
    return base.weight, base.bias, adapters


def linear_parts(m) -> Optional[Parts]:
    """(weight [N, K], bias [N] or None, [(A [r, K], B [N, r], s), ...]) of a layer whose forward is
    x W^T + b + sum s (x A^T) B^T, or None:
      - an exact nn.Linear: no adapters;
      - diffusers' LoRACompatibleLinear (an nn.Linear subclass with `lora_layer`): none if lora_layer is None, else its
        LoRALinearLayer with s = network_alpha / rank (1 without network_alpha);
      - peft's lora.Linear (`base_layer`, `lora_A`, `lora_B`, `scaling`): the active adapters with s = scaling[name];
        base only when the adapters are disabled or merged.
    Hooks or an instance-level forward on the layer or any layer inside it give None."""
    if type(m) is nn.Linear:
        return (m.weight, m.bias, []) if _plain(m) else None
    if isinstance(m, nn.Linear) and isinstance_str(m, "LoRACompatibleLinear") and hasattr(m, "lora_layer"):
        return _diffusers_parts(m)
    if isinstance(m, nn.Module) and all(hasattr(m, n) for n in ("base_layer", "lora_A", "lora_B", "scaling")):
        return _peft_parts(m)
    return None


def tag(parts: Sequence[Parts]) -> tuple:
    """Identity of what `pack` and the weight packs read: (data_ptr, _version) of every base and adapter tensor and the
    scales.  The adapter list is the resolved one, so a change of the active adapters, of the disable / merged flags or
    of a scale changes the tag."""
    out = []
    for w, b, ads in parts:
        out.append((w.data_ptr(), w._version, None if b is None else (b.data_ptr(), b._version),
                    tuple((A.data_ptr(), A._version, B.data_ptr(), B._version, s) for A, B, s in ads)))
    return tuple(out)


def pack(parts: Sequence[Parts], device) -> Optional[Tuple[torch.Tensor, torch.Tensor]]:
    """(D [R, K], U [N, R]) fp16 for one GEMM whose output columns are the layers' outputs in order (e.g. q | k | v),
    or None when no layer has an adapter.  D stacks every adapter's A rows; U holds s B in the adapter's columns and
    the layer's rows, zeros elsewhere (s B formed in fp32 and rounded to fp16 once).  R is padded to a multiple of 8 with
    zero rows / columns."""
    R = sum(A.shape[0] for _, _, ads in parts for A, _, _ in ads)
    if R == 0:
        return None
    K = parts[0][0].shape[1]
    N = sum(w.shape[0] for w, _, _ in parts)
    Rp = (R + 7) // 8 * 8
    with torch.no_grad():
        down = torch.zeros((Rp, K), dtype=torch.float16, device=device)
        up = torch.zeros((N, Rp), dtype=torch.float32, device=device)
        r0 = n0 = 0
        for w, _, ads in parts:
            n = w.shape[0]
            for A, B, s in ads:
                r = A.shape[0]
                down[r0:r0 + r] = A.detach().to(device=device, dtype=torch.float16)
                up[n0:n0 + n, r0:r0 + r] = B.detach().to(device=device, dtype=torch.float32) * s
                r0 += r
            n0 += n
        return down, up.to(torch.float16)
