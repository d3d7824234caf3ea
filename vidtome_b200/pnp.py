"""PnP self-attention on merged tokens (SURVEY §8 row f2), and PnP's conv-feature injection (register_conv_control,
below).

The reference's PnP control (utils/pnp_utils.py:39-106, `register_attention_control`) replaces `attn1.forward` of the
decoder blocks by a closure that — while the current timestep `attn.t` is in the injection schedule — computes the
attention map from the SOURCE sample only (`q[:B/num_inputs]`, `k[:B/num_inputs]`) and applies it to the values of
all `num_inputs` samples (`attn.repeat(num_inputs, 1, 1)`).  With `align_batch=True` (generate.py:97-98: `use_pnp or
cfg`) the merged token sets of the samples are aligned, so this is well defined on merged tokens.

`register_attention_control(model, injection_schedule, num_inputs)` here has the reference's name and arguments.  It
installs (i) an equivalent torch forward for every call that does not come through a merged ToMeBlock, and (ii) a marker
(`attn._vtm_pnp`) that lets ToMeBlock run the same computation through KD (`vtm_attention_ex`, flag
VTM_ATTN_SHARED_QK: every sample reads the queries and keys of sample 0 and its own values).  `register_time(model, t)`
sets `attn.t` on every marked module.

The decoder-block addressing of the reference (`model.unet.up_blocks[res].attentions[block].transformer_blocks[0].attn1`
for res/block in {1: [1, 2], 2: [0, 1, 2], 3: [0, 1, 2]}) is used when the model has that hierarchy; any other
model (the skeleton) must pass the attention modules explicitly through `modules=`.
"""
from __future__ import annotations

from typing import Iterable, Optional, Sequence

import torch

from . import patch

RES_DICT = {1: [1, 2], 2: [0, 1, 2], 3: [0, 1, 2]}       # utils/pnp_utils.py:97 (blocks 4 - 11 of the decoder)


def _targets(model, modules: Optional[Iterable[torch.nn.Module]]):
    if modules is not None:
        return list(modules)
    unet = model.unet if hasattr(model, "unet") else model
    out = []
    for res, blocks in RES_DICT.items():
        for block in blocks:
            out.append(unet.up_blocks[res].attentions[block].transformer_blocks[0].attn1)
    return out


def injection_active(attn: torch.nn.Module) -> bool:
    """utils/pnp_utils.py:57-58: `self.injection_schedule is not None and (self.t in self.injection_schedule or self.t == 1000)`.
    Always False inside patch._unmerged_blocks(): DDIM inversion runs before PnP is registered (invert.py:117-140)."""
    if patch.unmerged_active():
        return False
    sched = getattr(attn, "injection_schedule", None)
    t = getattr(attn, "t", None)
    return sched is not None and t is not None and (t in sched or t == 1000)


def _torch_forward(attn: torch.nn.Module, num_inputs: int):
    """The reference's replaced forward (utils/pnp_utils.py:47-95) in torch ops; used outside merged blocks."""
    to_out = attn.to_out[0] if isinstance(attn.to_out, (torch.nn.ModuleList, torch.nn.Sequential)) else attn.to_out

    # [b, n, h d] <-> [b h, n, d] as the reference's head_to_batch_dim / batch_to_head_dim: the same op sequence on the same
    # layouts, so that the fp16 CPU kernels round exactly as the reference's forward does on any instruction set
    def heads_to_batch(t, h):
        b, n, c = t.shape
        return t.reshape(b, n, h, c // h).permute(0, 2, 1, 3).reshape(b * h, n, c // h)

    def forward(x, encoder_hidden_states=None, attention_mask=None, **kwargs):
        h = attn.heads
        is_cross = encoder_hidden_states is not None
        ctx = encoder_hidden_states if is_cross else x
        q, k, v = attn.to_q(x), attn.to_k(ctx), attn.to_v(ctx)
        inject = not is_cross and injection_active(attn)
        if inject:
            src = q.shape[0] // num_inputs
            q, k = q[:src], k[:src]
        sim = torch.einsum("b i d, b j d -> b i j", heads_to_batch(q, h), heads_to_batch(k, h)) * attn.scale
        if attention_mask is not None:
            mask = attention_mask.reshape(x.shape[0], -1)[:, None, :].repeat_interleave(h, 0)
            sim = sim.masked_fill(~mask, -torch.finfo(sim.dtype).max)
        p = sim.softmax(dim=-1)
        if inject:
            p = p.repeat(num_inputs, 1, 1)
        out = torch.einsum("b i j, b j d -> b i d", p, heads_to_batch(v, h))
        out = out.reshape(x.shape[0], h, x.shape[1], -1).permute(0, 2, 1, 3).reshape(x.shape[0], x.shape[1], -1)
        return to_out(out)

    forward._vtm_pnp_forward = True
    return forward


def register_attention_control(model, injection_schedule: Optional[Sequence[int]], num_inputs: int,
                               modules: Optional[Iterable[torch.nn.Module]] = None):
    """Same call as the reference's (utils/pnp_utils.py:39): mark the decoder self-attention modules for source-sample
    Q/K injection during the timesteps in `injection_schedule`."""
    for attn in _targets(model, modules):
        attn.forward = _torch_forward(attn, num_inputs)
        attn.injection_schedule = injection_schedule
        attn._vtm_pnp = int(num_inputs)
    return model


def register_time(model, t: int, modules: Optional[Iterable[torch.nn.Module]] = None):
    """utils/pnp_utils.py:12-37 for the modules PnP controls (the marked self-attention modules and ResNets): the current
    timestep, read by the injection test."""
    if modules is None:
        root = model.unet if hasattr(model, "unet") else model
        modules = [m for m in root.modules() if hasattr(m, "_vtm_pnp") or hasattr(m, "_vtm_pnp_conv")]
    for m in modules:
        m.t = t
    return model


# ------------------------------------------------------------------------------------------ conv-feature injection
# The reference's second PnP injection (utils/pnp_utils.py:108-172, `register_conv_control`) replaces the forward of
# `unet.up_blocks[1].resnets[1]`: while the timestep is in its schedule, the source samples' conv2 output is copied over
# the uncond and cond samples before the residual add.  `register_conv_control` here has the reference's name and
# arguments and installs (i) the reference's forward in torch ops, and (ii) a marker (`resnet._vtm_pnp_conv`) under which
# eligible calls (conv_eligible) take the library path: norm1 ... conv2 in torch ops, on the source samples only while
# injecting (the other samples' branch would be thrown away), and the residual tail in one kernel (KT, ops.resnet_tail).

def _conv_targets(model, modules: Optional[Iterable[torch.nn.Module]]):
    if modules is not None:
        return list(modules)
    unet = model.unet if hasattr(model, "unet") else model
    return [unet.up_blocks[1].resnets[1]]                              # utils/pnp_utils.py:168-169


def _has_hooks(m: torch.nn.Module) -> bool:
    return bool(m._forward_hooks or m._forward_pre_hooks or getattr(m, "_forward_hooks_with_kwargs", None))


def conv_ineligibility(resnet: torch.nn.Module, input_tensor: torch.Tensor,
                       temb: Optional[torch.Tensor]) -> Optional[str]:
    """Why a call of a marked ResNet takes the torch forward instead of the library path, or None if it takes the
    library path: that needs a batch of num_inputs * n samples (num_inputs 2 or 3) as a contiguous NCHW tensor, no up-
    or downsampling, the "default" time-embedding add, inactive dropout, no hooks on the submodules it runs (they would
    see the source samples only while injecting), and CUDA fp16 tensors (checked last)."""
    num_inputs = getattr(resnet, "_vtm_pnp_conv", None)
    x = input_tensor
    if num_inputs not in (2, 3):
        return "num_inputs"
    if not isinstance(x, torch.Tensor) or x.dim() != 4 or x.shape[0] == 0 or x.shape[0] % num_inputs:
        return "batch"
    if not x.is_contiguous():
        return "layout"
    if resnet.upsample is not None or resnet.downsample is not None:
        return "resample"
    if resnet.time_embedding_norm != "default":
        return "time_embedding_norm"
    drop = resnet.dropout
    if drop is not None and drop.training and getattr(drop, "p", 0.0) > 0:
        return "dropout"
    if temb is not None and (temb.dim() != 2 or temb.shape[0] not in (1, x.shape[0])):
        return "temb"
    if any(_has_hooks(m) for m in resnet.modules() if m is not resnet):
        return "hooks"
    if not x.is_cuda or x.dtype != torch.float16 or (temb is not None and temb.dtype != torch.float16):
        return "device"
    return None


def conv_eligible(resnet: torch.nn.Module, input_tensor: torch.Tensor, temb: Optional[torch.Tensor]) -> bool:
    """True if a call of a marked ResNet takes the library path (conv_ineligibility)."""
    return conv_ineligibility(resnet, input_tensor, temb) is None


def _conv_torch_forward(resnet: torch.nn.Module, num_inputs: int, input_tensor, temb):
    """The reference's conv_forward (utils/pnp_utils.py:110-164), op for op."""
    self = resnet
    hidden_states = input_tensor
    hidden_states = self.norm1(hidden_states)
    hidden_states = self.nonlinearity(hidden_states)
    if self.upsample is not None:
        if hidden_states.shape[0] >= 64:
            input_tensor = input_tensor.contiguous()
            hidden_states = hidden_states.contiguous()
        input_tensor = self.upsample(input_tensor)
        hidden_states = self.upsample(hidden_states)
    elif self.downsample is not None:
        input_tensor = self.downsample(input_tensor)
        hidden_states = self.downsample(hidden_states)
    hidden_states = self.conv1(hidden_states)
    if temb is not None:
        temb = self.time_emb_proj(self.nonlinearity(temb))[:, :, None, None]
    if temb is not None and self.time_embedding_norm == "default":
        hidden_states = hidden_states + temb
    hidden_states = self.norm2(hidden_states)
    if temb is not None and self.time_embedding_norm == "scale_shift":
        scale, shift = torch.chunk(temb, 2, dim=1)
        hidden_states = hidden_states * (1 + scale) + shift
    hidden_states = self.nonlinearity(hidden_states)
    hidden_states = self.dropout(hidden_states)
    hidden_states = self.conv2(hidden_states)
    if injection_active(self):
        n = int(hidden_states.shape[0] // num_inputs)
        hidden_states[n:2 * n] = hidden_states[:n]
        if num_inputs > 2:
            hidden_states[2 * n:3 * n] = hidden_states[:n]
    if self.conv_shortcut is not None:
        input_tensor = self.conv_shortcut(input_tensor)
    return (input_tensor + hidden_states) / self.output_scale_factor


def conv_library_forward(resnet: torch.nn.Module, input_tensor: torch.Tensor, temb: Optional[torch.Tensor]):
    """The library path of a marked ResNet (conv_eligible calls): while injecting, norm1 ... conv2 run on the n source
    samples only; the time embedding is projected for the whole batch (as the reference does) and its source rows
    taken.  The tail — the copy, the residual add and the scale — is one KT launch."""
    from . import ops
    num_inputs = resnet._vtm_pnp_conv
    inject = injection_active(resnet)
    n = input_tensor.shape[0] // num_inputs
    h = input_tensor[:n] if inject else input_tensor
    h = resnet.nonlinearity(resnet.norm1(h))
    h = resnet.conv1(h)
    if temb is not None:
        temb = resnet.time_emb_proj(resnet.nonlinearity(temb))[:, :, None, None]
        h = h + (temb[:n] if inject and temb.shape[0] > 1 else temb)
    h = resnet.nonlinearity(resnet.norm2(h))
    h = resnet.conv2(resnet.dropout(h))
    shortcut = input_tensor if resnet.conv_shortcut is None else resnet.conv_shortcut(input_tensor)
    return ops.resnet_tail(h, shortcut, num_inputs, resnet.output_scale_factor, inject)


def _conv_forward(resnet: torch.nn.Module, num_inputs: int):
    def forward(input_tensor, temb=None, **kwargs):
        if conv_eligible(resnet, input_tensor, temb):
            return conv_library_forward(resnet, input_tensor, temb)
        return _conv_torch_forward(resnet, num_inputs, input_tensor, temb)

    forward._vtm_pnp_conv_forward = True
    return forward


def register_conv_control(model, injection_schedule: Optional[Sequence[int]], num_inputs: int,
                          modules: Optional[Iterable[torch.nn.Module]] = None):
    """Same call as the reference's (utils/pnp_utils.py:108): mark `unet.up_blocks[1].resnets[1]` (or `modules`) for
    source-sample conv-feature injection during the timesteps in `injection_schedule`."""
    for resnet in _conv_targets(model, modules):
        resnet.forward = _conv_forward(resnet, int(num_inputs))
        resnet.injection_schedule = injection_schedule
        resnet._vtm_pnp_conv = int(num_inputs)
    return model
