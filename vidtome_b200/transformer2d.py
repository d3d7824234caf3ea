"""The entry and exit of diffusers' `Transformer2DModel.forward` in the CUDA library.

`Transformer2DModel` owns every BasicTransformerBlock of a diffusers UNet / ControlNet and is where diffusers' NCHW
activations meet the token-major rows the blocks (and this library) work on:

    residual = x                                        # [(B F), C, h, w]
    x = norm(x)                                         # GroupNorm(32, C, eps=1e-6)
    x = proj_in(x)  ->  [(B F), h w, inner] tokens      # 1x1 Conv2d then permute (SD1.x), or permute then Linear (SD2.x)
    for block in transformer_blocks: x = block(x, ...)
    x -> proj_out -> [(B F), C, h, w]                   # permute then 1x1 Conv2d, or Linear then permute
    return x + residual

It is third-party code that the reference never touches (its patch swaps the blocks inside, vidtome/patch.py:319), so
its arithmetic is torch's and is not pinned by the reference (SURVEY §8c, like attn1's).  Both projection forms compute
the same function and differ only in where the transposing copy sits; the library path has none: GroupNorm writes
token-major rows (ops.group_norm_tokens), proj_in is the projection GEMM on them, and proj_out is the same GEMM storing
NCHW with the residual added in its epilogue (ops.linear_nchw_residual).  `patch.apply_patch` routes eligible modules
here while `patch.FUSE_TRANSFORMER_IO` is on.
"""
from __future__ import annotations

import sys
from dataclasses import dataclass
from typing import Optional

import torch

from . import ops


@dataclass
class Transformer2DModelOutput:
    """Stand-in for diffusers' output class of the same name, used when the module's own cannot be found."""
    sample: torch.Tensor


def _has_hooks(m: torch.nn.Module) -> bool:
    return bool(m._forward_hooks or m._forward_pre_hooks or getattr(m, "_forward_hooks_with_kwargs", None))


def _projection(m: torch.nn.Module) -> Optional[str]:
    """"conv" for exactly an nn.Conv2d 1x1 (stride 1, no padding, dilation 1, groups 1), "linear" for exactly an
    nn.Linear, else None (subclasses such as LoRACompatibleConv / LoRACompatibleLinear and peft wrappers carry terms the
    GEMM would miss)."""
    if type(m) is torch.nn.Conv2d:
        if (m.kernel_size == (1, 1) and m.stride == (1, 1) and m.padding == (0, 0) and m.dilation == (1, 1)
                and m.groups == 1 and m.padding_mode == "zeros"):
            return "conv"
        return None
    if type(m) is torch.nn.Linear:
        return "linear"
    return None


def ineligibility(module: torch.nn.Module, hidden_states: torch.Tensor) -> Optional[str]:
    """Why a call of `module` (a Transformer2DModel) runs its own torch forward instead of the library path, or None if it
    takes the library path.  That needs the continuous-input variant (not `is_input_vectorized` / `is_input_patches`),
    a contiguous NCHW input, `norm` a plain affine nn.GroupNorm whose groups divide C, `proj_in` and `proj_out` both
    exactly nn.Conv2d 1x1 or both exactly nn.Linear, with channel counts the GEMMs take (multiples of 8), no hooks on
    the three layers, no autograd (training with grad enabled), and CUDA fp16 tensors (checked last)."""
    x = hidden_states
    if getattr(module, "is_input_vectorized", False) or getattr(module, "is_input_patches", False):
        return "input_variant"
    if getattr(module, "is_input_continuous", True) is False:
        return "input_variant"
    if not isinstance(x, torch.Tensor) or x.dim() != 4 or x.numel() == 0:
        return "shape"
    if not x.is_contiguous():
        return "layout"
    norm = getattr(module, "norm", None)
    if type(norm) is not torch.nn.GroupNorm or not norm.affine:
        return "norm"
    if norm.num_channels != x.shape[1] or x.shape[1] % norm.num_groups:
        return "norm"
    kinds = (_projection(getattr(module, "proj_in", None)), _projection(getattr(module, "proj_out", None)))
    if kinds[0] is None or kinds[0] != kinds[1]:
        return "projection"
    form = getattr(module, "use_linear_projection", None)
    if form is not None and bool(form) != (kinds[0] == "linear"):
        return "projection"               # the layers do not match the form the module says it runs
    w_in, w_out = module.proj_in.weight, module.proj_out.weight
    C, inner = x.shape[1], w_in.shape[0]
    if w_in.shape[1] != C or tuple(w_out.shape[:2]) != (C, inner) or C % 8 or inner % 8:
        return "projection"
    if not (w_in.is_contiguous() and w_out.is_contiguous()):
        return "projection"
    if any(_has_hooks(m) for m in (norm, module.proj_in, module.proj_out)):
        return "hooks"
    if module.training and torch.is_grad_enabled():
        return "training"
    params = [norm.weight, norm.bias, w_in, w_out, module.proj_in.bias, module.proj_out.bias]
    if not x.is_cuda or x.dtype != torch.float16 or any(
            p is not None and (p.dtype != torch.float16 or p.device != x.device) for p in params):
        return "device"
    return None


def _output_class(module: torch.nn.Module):
    """The `Transformer2DModelOutput` defined next to the module's (unpatched) class, else ours."""
    for cls in type(module).__mro__:
        if cls.__name__ == "Transformer2DModel":
            found = getattr(sys.modules.get(cls.__module__), "Transformer2DModelOutput", None)
            if found is not None:
                return found
    return Transformer2DModelOutput


def library_forward(module: torch.nn.Module, hidden_states: torch.Tensor, encoder_hidden_states=None, timestep=None,
                    cross_attention_kwargs=None, attention_mask=None, encoder_attention_mask=None, class_labels=None,
                    return_dict: bool = True):
    """`Transformer2DModel.forward` of an eligible module (ineligibility(...) is None) with its entry and exit in the
    library; the module's own `transformer_blocks` run in between, patched or not."""
    x = hidden_states
    n, C, h, w = x.shape
    norm = module.norm
    tokens = ops.group_norm_tokens(x, (norm.weight, norm.bias, norm.eps, norm.num_groups))
    w_in, w_out = module.proj_in.weight, module.proj_out.weight
    inner = w_in.shape[0]
    # a 1x1 conv's weight [out, in, 1, 1] is the Linear's [out, in]
    t = ops.linear(tokens.view(n * h * w, C), w_in.view(inner, C), module.proj_in.bias).view(n, h * w, inner)
    for block in module.transformer_blocks:
        t = block(t, attention_mask=attention_mask, encoder_hidden_states=encoder_hidden_states,
                  encoder_attention_mask=encoder_attention_mask, timestep=timestep,
                  cross_attention_kwargs=cross_attention_kwargs, class_labels=class_labels)
    t = t.contiguous().view(n * h * w, inner)
    out = ops.linear_nchw_residual(t, w_out.view(C, inner), module.proj_out.bias, x, (h, w))
    if not return_dict:
        return (out,)
    return _output_class(module)(sample=out)


# the keyword arguments of Transformer2DModel.forward that library_forward restates
LIBRARY_KWARGS = frozenset(("encoder_hidden_states", "timestep", "cross_attention_kwargs", "attention_mask",
                            "encoder_attention_mask", "class_labels", "return_dict"))
