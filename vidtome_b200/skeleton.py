"""SD-shaped skeleton UNet: the stand-in for diffusers used by the tests, the golden fixtures and bench.py.

diffusers and the Stable-Diffusion weights are not available offline, and both the reference's patch and
ours find their targets by class NAME (`ModelMixin`, `BasicTransformerBlock`, vidtome/patch.py:279-280,319),
so an `nn.Module` hierarchy with those names is patched exactly like a real diffusers UNet.  The skeleton
carries the transformer-block census of the SD UNets — (tokens per frame T, channels C, heads) per block,
in execution order — with random weights; the convolutional ResNet path between the blocks is replaced by
a cheap per-resolution linear lift of the latent, because it is outside the merge hot path
(SURVEY.md §8: rows a1-a15 are the self-attention section of each block).

`hot_path_only=True` (default) builds blocks with `attn2 = ff = None`: a block is then exactly the
self-attention section norm1 -> [merge] -> attn1 -> [unmerge] -> + residual (patch.py:139-169).
`hot_path_only=False` adds the cross-attention and GEGLU feed-forward of a real BasicTransformerBlock.

`ControlNetModel` / `make_controlnet` stand in for diffusers' ControlNet in the same way: the encoder half of the
census, whose per-block residuals the skeleton UNet adds to its encoder blocks' outputs.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from types import SimpleNamespace
from typing import List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F


class Attention(nn.Module):
    """diffusers.models.attention_processor.Attention, reduced to what SD uses: to_q/to_k/to_v without
    bias, `to_out = [Linear(bias), Dropout]`, multi-head softmax(q k^T * scale) v (math restated in the
    reference at utils/pnp_utils.py:47-95)."""

    def __init__(self, query_dim: int, heads: int, dim_head: int, cross_attention_dim: Optional[int] = None):
        super().__init__()
        inner = heads * dim_head
        kv_dim = cross_attention_dim if cross_attention_dim is not None else query_dim
        self.heads = heads
        self.scale = dim_head ** -0.5
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(kv_dim, inner, bias=False)
        self.to_v = nn.Linear(kv_dim, inner, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(inner, query_dim), nn.Dropout(0.0)])

    def forward(self, hidden_states, encoder_hidden_states=None, attention_mask=None, **kwargs):
        ctx = hidden_states if encoder_hidden_states is None else encoder_hidden_states
        B, L, _ = hidden_states.shape
        h = self.heads
        q = self.to_q(hidden_states).view(B, L, h, -1).transpose(1, 2)
        k = self.to_k(ctx).view(B, ctx.shape[1], h, -1).transpose(1, 2)
        v = self.to_v(ctx).view(B, ctx.shape[1], h, -1).transpose(1, 2)
        o = F.scaled_dot_product_attention(q, k, v, attn_mask=attention_mask, scale=self.scale)
        o = o.transpose(1, 2).reshape(B, L, -1)
        return self.to_out[1](self.to_out[0](o))


class GEGLUFeedForward(nn.Module):
    def __init__(self, dim: int, mult: int = 4):
        super().__init__()
        self.proj = nn.Linear(dim, dim * mult * 2)
        self.out = nn.Linear(dim * mult, dim)

    def forward(self, x):
        a, g = self.proj(x).chunk(2, dim=-1)
        return self.out(a * F.gelu(g))


class BasicTransformerBlock(nn.Module):
    """Same attribute names and (unpatched) forward as diffusers' BasicTransformerBlock of the 0.17-0.21
    era that the reference targets (attributes read by patch.py:139-199)."""

    def __init__(self, dim: int, heads: int, cross_attention_dim: int = 768, hot_path_only: bool = True):
        super().__init__()
        self.only_cross_attention = False
        self.use_ada_layer_norm = False
        self.use_ada_layer_norm_zero = False
        self.norm1 = nn.LayerNorm(dim)
        self.attn1 = Attention(dim, heads, dim // heads)
        if hot_path_only:
            self.attn2 = None
            self.norm2 = None
            self.norm3 = None
            self.ff = None
        else:
            self.norm2 = nn.LayerNorm(dim)
            self.attn2 = Attention(dim, heads, dim // heads, cross_attention_dim=cross_attention_dim)
            self.norm3 = nn.LayerNorm(dim)
            self.ff = GEGLUFeedForward(dim)

    def forward(self, hidden_states, attention_mask=None, encoder_hidden_states=None,
                encoder_attention_mask=None, timestep=None, cross_attention_kwargs=None, class_labels=None):
        hidden_states = self.attn1(self.norm1(hidden_states), attention_mask=attention_mask) + hidden_states
        if self.attn2 is not None:
            hidden_states = self.attn2(self.norm2(hidden_states),
                                       encoder_hidden_states=encoder_hidden_states) + hidden_states
        if self.ff is not None:
            hidden_states = self.ff(self.norm3(hidden_states)) + hidden_states
        return hidden_states


class LoRALinearLayer(nn.Module):
    """diffusers' LoRALinearLayer (the adapter of LoRACompatibleLinear): up(down(x)), times network_alpha / rank when
    network_alpha is set, computed in the adapter's dtype and cast back to the input's."""

    def __init__(self, in_features: int, out_features: int, rank: int, network_alpha: Optional[float] = None):
        super().__init__()
        self.down = nn.Linear(in_features, rank, bias=False)
        self.up = nn.Linear(rank, out_features, bias=False)
        self.network_alpha = network_alpha
        self.rank = rank

    def forward(self, hidden_states):
        orig_dtype = hidden_states.dtype
        up = self.up(self.down(hidden_states.to(self.down.weight.dtype)))
        if self.network_alpha is not None:
            up = up * (self.network_alpha / self.rank)
        return up.to(orig_dtype)


class LoRACompatibleLinear(nn.Linear):
    """diffusers' LoRACompatibleLinear: an nn.Linear whose forward adds `scale * lora_layer(x)` when it has one."""

    def __init__(self, *args, lora_layer: Optional[LoRALinearLayer] = None, **kwargs):
        super().__init__(*args, **kwargs)
        self.lora_layer = lora_layer

    def forward(self, hidden_states, scale: float = 1.0):
        if self.lora_layer is None:
            return super().forward(hidden_states)
        return super().forward(hidden_states) + scale * self.lora_layer(hidden_states)


class PeftLoraLinear(nn.Module):
    """peft's lora.Linear: `base_layer` plus, per active adapter, lora_B(lora_A(dropout(x))) * scaling, each adapter
    computed in its own dtype, and the sum cast back to the base layer's output dtype."""

    def __init__(self, base_layer: nn.Linear):
        super().__init__()
        self.base_layer = base_layer
        self.lora_A = nn.ModuleDict()
        self.lora_B = nn.ModuleDict()
        self.lora_dropout = nn.ModuleDict()
        self.scaling = {}
        self.use_dora = {}
        self.lora_bias = {}
        self.fan_in_fan_out = False
        self._active_adapter = []
        self._disable_adapters = False
        self.merged_adapters = []

    def update_layer(self, name: str, r: int, lora_alpha: float, dropout: float = 0.0):
        self.lora_A[name] = nn.Linear(self.base_layer.in_features, r, bias=False)
        self.lora_B[name] = nn.Linear(r, self.base_layer.out_features, bias=False)
        self.lora_dropout[name] = nn.Dropout(dropout) if dropout > 0 else nn.Identity()
        self.scaling[name] = lora_alpha / r
        self.use_dora[name] = False
        self.lora_bias[name] = False
        if name not in self._active_adapter:
            self._active_adapter.append(name)

    @property
    def weight(self):
        return self.base_layer.weight

    @property
    def bias(self):
        return self.base_layer.bias

    @property
    def active_adapters(self):
        return list(self._active_adapter)

    def set_adapter(self, names):
        self._active_adapter = [names] if isinstance(names, str) else list(names)

    @property
    def disable_adapters(self) -> bool:
        return self._disable_adapters

    @property
    def merged(self) -> bool:
        return bool(self.merged_adapters)

    def forward(self, x):
        result = self.base_layer(x)
        if self.disable_adapters or self.merged:
            return result
        torch_result_dtype = result.dtype
        for name in self.active_adapters:
            if name not in self.lora_A:
                continue
            lora_A = self.lora_A[name]
            xa = x.to(lora_A.weight.dtype)
            result = result + self.lora_B[name](lora_A(self.lora_dropout[name](xa))) * self.scaling[name]
        return result.to(torch_result_dtype)


LORA_TARGETS = ("to_q", "to_k", "to_v", "to_out", "ff")


def add_lora(net: nn.Module, rank: int, form: str = "peft", targets=LORA_TARGETS, dtype=None, seed: int = 7,
             attns=("attn1", "attn2")) -> nn.Module:
    """Wrap the chosen projections of every BasicTransformerBlock in `net` (a skeleton UNet or ControlNet) with one
    seeded LoRA adapter of `rank`, as `load_lora_weights` does: form "diffusers" (LoRACompatibleLinear with a
    LoRALinearLayer, network_alpha = rank / 2) or "peft" (PeftLoraLinear, adapter "default", lora_alpha = rank / 2).
    targets: any of "to_q", "to_k", "to_v", "to_out" (to_out[0]) of the `attns` modules, and "ff" (both Linear layers of
    the feed-forward).  Adapter weights are drawn so that the LoRA term is a sizeable fraction of the projection's
    output (lora_B is not zero-initialised), in `dtype` (default: the base weight's)."""
    if form not in ("diffusers", "peft"):
        raise ValueError(f"add_lora: form must be 'diffusers' or 'peft', got {form!r}")
    gen = torch.Generator().manual_seed(seed)

    def wrap(lin: nn.Linear) -> nn.Module:
        w = lin.weight
        dt = dtype or w.dtype
        K, N = lin.in_features, lin.out_features
        a = torch.randn((rank, K), generator=gen) * K ** -0.5
        b = torch.randn((N, rank), generator=gen) * (0.5 * rank ** -0.5)
        if form == "diffusers":
            layer = LoRALinearLayer(K, N, rank, network_alpha=rank / 2)
            new = LoRACompatibleLinear(K, N, bias=lin.bias is not None, lora_layer=layer)
            with torch.no_grad():
                new.weight.copy_(lin.weight.cpu())
                if lin.bias is not None:
                    new.bias.copy_(lin.bias.cpu())
                layer.down.weight.copy_(a)
                layer.up.weight.copy_(b)
            new = new.to(device=w.device, dtype=w.dtype)
            layer.to(dtype=dt)
            return new
        new = PeftLoraLinear(lin)
        new.update_layer("default", rank, rank / 2)
        with torch.no_grad():
            new.lora_A["default"].weight.copy_(a)
            new.lora_B["default"].weight.copy_(b)
        new.lora_A.to(device=w.device, dtype=dt)
        new.lora_B.to(device=w.device, dtype=dt)
        return new

    for block in [m for m in net.modules() if type(m).__name__ in ("BasicTransformerBlock", "ToMeBlock")]:
        for an in attns:
            attn = getattr(block, an, None)
            if attn is None:
                continue
            for t in ("to_q", "to_k", "to_v"):
                if t in targets:
                    setattr(attn, t, wrap(getattr(attn, t)))
            if "to_out" in targets:
                attn.to_out[0] = wrap(attn.to_out[0])
        ff = getattr(block, "ff", None)
        if ff is not None and "ff" in targets:
            ff.proj = wrap(ff.proj)
            ff.out = wrap(ff.out)
    return net


class ResnetBlock2D(nn.Module):
    """diffusers' ResnetBlock2D as SD's UNet builds it: GroupNorm -> SiLU -> conv1 (3x3) -> + time embedding ->
    GroupNorm -> SiLU -> dropout -> conv2 (3x3), plus a 1x1 conv_shortcut when the channel count changes, and
    (shortcut + h) / output_scale_factor.  It carries every attribute the reference's PnP conv_forward reads
    (utils/pnp_utils.py:110-164); no up- or downsampling, time_embedding_norm "default".  The GroupNorm affines are drawn
    around (1, 0) rather than left at it, so that they take part in a comparison."""

    def __init__(self, in_channels: int, out_channels: Optional[int] = None, temb_channels: Optional[int] = 1280,
                 groups: int = 32, eps: float = 1e-5, output_scale_factor: float = 1.0, dropout: float = 0.0):
        super().__init__()
        out_channels = in_channels if out_channels is None else out_channels
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=eps, affine=True)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, padding=1)
        self.time_emb_proj = nn.Linear(temb_channels, out_channels) if temb_channels else None
        self.norm2 = nn.GroupNorm(groups, out_channels, eps=eps, affine=True)
        self.dropout = nn.Dropout(dropout)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, padding=1)
        self.nonlinearity = nn.SiLU()
        self.upsample = None
        self.downsample = None
        self.time_embedding_norm = "default"
        self.output_scale_factor = output_scale_factor
        self.conv_shortcut = nn.Conv2d(in_channels, out_channels, 1) if in_channels != out_channels else None
        with torch.no_grad():
            for norm in (self.norm1, self.norm2):
                norm.weight.normal_(1.0, 0.1)
                norm.bias.normal_(0.0, 0.1)

    def forward(self, input_tensor, temb, scale: float = 1.0):
        h = self.conv1(self.nonlinearity(self.norm1(input_tensor)))
        if temb is not None:
            h = h + self.time_emb_proj(self.nonlinearity(temb))[:, :, None, None]
        h = self.conv2(self.dropout(self.nonlinearity(self.norm2(h))))
        shortcut = input_tensor if self.conv_shortcut is None else self.conv_shortcut(input_tensor)
        return (shortcut + h) / self.output_scale_factor


def timestep_embedding(timestep, batch: int, dim: int, device, dtype) -> torch.Tensor:
    """diffusers' get_timestep_embedding(flip_sin_to_cos=True, downscale_freq_shift=0) of a scalar timestep (an int or a
    0-dim / 1-element tensor, which may live on the device), broadcast to [batch, dim]."""
    t = torch.as_tensor(timestep, device=device).reshape(-1)[:1].float()
    half = dim // 2
    freqs = torch.exp(torch.arange(half, dtype=torch.float32, device=device) * (-math.log(10000.0) / half))
    args = t[:, None] * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1).to(dtype).expand(batch, dim)


@dataclass
class Transformer2DModelOutput:
    sample: torch.Tensor


class Transformer2DModel(nn.Module):
    """diffusers' Transformer2DModel with continuous input, as SD's UNet builds it around every BasicTransformerBlock:
    GroupNorm(32, C, eps=1e-6) -> proj_in -> tokens -> transformer_blocks -> NCHW -> proj_out -> + residual, with
    proj_in / proj_out 1x1 convolutions on the NCHW side (SD1.x) or, with `use_linear_projection`, Linear layers on the
    token side (SD2.x).  The block is handed in, so that the skeleton's census blocks are the ones that run inside.
    `torch_calls` counts runs of this torch forward, as tests count `Attention.forward`."""

    torch_calls = 0

    def __init__(self, in_channels: int, block: nn.Module, use_linear_projection: bool = False, norm_num_groups: int = 32):
        super().__init__()
        self.is_input_continuous = True
        self.is_input_vectorized = False
        self.is_input_patches = False
        self.use_linear_projection = use_linear_projection
        self.in_channels = in_channels
        inner = in_channels
        self.norm = nn.GroupNorm(norm_num_groups, in_channels, eps=1e-6, affine=True)
        if use_linear_projection:
            self.proj_in = nn.Linear(in_channels, inner)
            self.proj_out = nn.Linear(inner, in_channels)
        else:
            self.proj_in = nn.Conv2d(in_channels, inner, kernel_size=1, stride=1, padding=0)
            self.proj_out = nn.Conv2d(inner, in_channels, kernel_size=1, stride=1, padding=0)
        self.transformer_blocks = nn.ModuleList([block])
        with torch.no_grad():             # drawn around (1, 0), so that the affine takes part in a comparison
            self.norm.weight.normal_(1.0, 0.1)
            self.norm.bias.normal_(0.0, 0.1)

    def forward(self, hidden_states, encoder_hidden_states=None, timestep=None, cross_attention_kwargs=None,
                attention_mask=None, encoder_attention_mask=None, class_labels=None, return_dict: bool = True):
        Transformer2DModel.torch_calls += 1
        batch, _, height, width = hidden_states.shape
        residual = hidden_states
        hidden_states = self.norm(hidden_states)
        if not self.use_linear_projection:
            hidden_states = self.proj_in(hidden_states)
            inner = hidden_states.shape[1]
            hidden_states = hidden_states.permute(0, 2, 3, 1).reshape(batch, height * width, inner)
        else:
            inner = hidden_states.shape[1]
            hidden_states = hidden_states.permute(0, 2, 3, 1).reshape(batch, height * width, inner)
            hidden_states = self.proj_in(hidden_states)
        for block in self.transformer_blocks:
            hidden_states = block(hidden_states, attention_mask=attention_mask,
                                  encoder_hidden_states=encoder_hidden_states,
                                  encoder_attention_mask=encoder_attention_mask, timestep=timestep,
                                  cross_attention_kwargs=cross_attention_kwargs, class_labels=class_labels)
        if not self.use_linear_projection:
            hidden_states = hidden_states.reshape(batch, height, width, inner).permute(0, 3, 1, 2).contiguous()
            hidden_states = self.proj_out(hidden_states)
        else:
            hidden_states = self.proj_out(hidden_states)
            hidden_states = hidden_states.reshape(batch, height, width, inner).permute(0, 3, 1, 2).contiguous()
        output = hidden_states + residual
        if not return_dict:
            return (output,)
        return Transformer2DModelOutput(sample=output)


def _make_wrappers(blocks, census, transformer_io: Optional[str]) -> Optional[nn.ModuleList]:
    """One Transformer2DModel per census block (transformer_io "conv" or "linear"), or None."""
    if transformer_io is None:
        return None
    if transformer_io not in ("conv", "linear"):
        raise ValueError(f"transformer_io must be None, 'conv' or 'linear', got {transformer_io!r}")
    return nn.ModuleList([Transformer2DModel(s.dim, b, use_linear_projection=transformer_io == "linear")
                          for s, b in zip(census, blocks)])


def _to_nchw(tokens: torch.Tensor, hw: Tuple[int, int]) -> torch.Tensor:
    return tokens.transpose(1, 2).reshape(tokens.shape[0], -1, *hw).contiguous()


def _to_tokens(nchw: torch.Tensor) -> torch.Tensor:
    return nchw.flatten(2).transpose(1, 2)


class ModelMixin(nn.Module):
    """Name-only stand-in for diffusers.ModelMixin (patch.py:279-280 matches the class name)."""


@dataclass(frozen=True)
class BlockSpec:
    downsample: int     # 1, 2, 4, 8
    dim: int
    heads: int


def sd15_census() -> List[BlockSpec]:
    """The 16 BasicTransformerBlocks of the SD1.5 UNet in execution order: down 2+2+2, mid 1, up 3+3+3
    (SURVEY.md App. B).  heads = 8 everywhere, head_dim = 40 / 80 / 160."""
    d = [BlockSpec(1, 320, 8)] * 2 + [BlockSpec(2, 640, 8)] * 2 + [BlockSpec(4, 1280, 8)] * 2
    m = [BlockSpec(8, 1280, 8)]
    u = [BlockSpec(4, 1280, 8)] * 3 + [BlockSpec(2, 640, 8)] * 3 + [BlockSpec(1, 320, 8)] * 3
    return d + m + u


def sd21_census() -> List[BlockSpec]:
    """SD2.1: same layout, head_dim = 64 (heads 5 / 10 / 20), cross-attention dim 1024."""
    d = [BlockSpec(1, 320, 5)] * 2 + [BlockSpec(2, 640, 10)] * 2 + [BlockSpec(4, 1280, 20)] * 2
    m = [BlockSpec(8, 1280, 20)]
    u = [BlockSpec(4, 1280, 20)] * 3 + [BlockSpec(2, 640, 10)] * 3 + [BlockSpec(1, 320, 5)] * 3
    return d + m + u


def tiny_census() -> List[BlockSpec]:
    """A 4-block miniature (for CPU plumbing tests and golden fixtures)."""
    return [BlockSpec(1, 64, 2), BlockSpec(2, 128, 2), BlockSpec(4, 128, 2), BlockSpec(1, 64, 2)]


CENSUSES = {"sd15": sd15_census, "sd21": sd21_census, "tiny": tiny_census}


def mid_position(census: List[BlockSpec]) -> int:
    """Census position of the mid block: the first block at the deepest resolution.  The blocks before it are the down
    blocks; together they are the encoder half that a ControlNet copies (6 down + 1 mid in the SD census)."""
    deepest = max(s.downsample for s in census)
    return next(i for i, s in enumerate(census) if s.downsample == deepest)


class SkeletonUNet(ModelMixin):
    """forward(latent [(B F), in_channels, h, w], t, encoder_hidden_states) -> object with `.sample`
    [(B F), out_channels, h, w].  For every block: the latent is average-pooled to the block's resolution, lifted to `dim`
    channels by a fixed linear map, added to the running state of that resolution, run through the block,
    and projected back into the noise prediction.

    `down_block_additional_residuals` / `mid_block_additional_residual` (a ControlNet's outputs) are added to the output
    state of the matching encoder block, the skeleton's stand-in for diffusers' skip-sample add: one residual per down
    block in block order, one for the mid block, each shaped like that block's output [(B F), T, C].

    `pnp_conv=True` adds `resnet`, a ResnetBlock2D at the census position of diffusers' `up_blocks[1].resnets[1]` (the
    target of PnP's conv-feature injection, utils/pnp_utils.py:168-169), run ahead of census block 8: it takes the
    state of that resolution concatenated with a skip (the last encoder block's output there, 2C channels, as the
    decoder's skip concatenation), gives C channels back to the state, and gets the sinusoidal embedding of the
    timestep.  Its weights are drawn after all others, so the rest of the skeleton is the same with and without it.

    `transformer_io="conv"` / `"linear"` adds `wrappers`, one Transformer2DModel around every census block, as diffusers'
    UNet has: the state of each resolution is then kept NCHW [(B F), C, h, w] and every block is called through its
    wrapper (additional residuals are NCHW as well, shaped like the wrapper's output).  The wrappers' weights are drawn
    last of all, so every other parameter is the same with and without them.

    `out_channels` (default: `in_channels`) is the channel count of the prediction.  SD2-depth's UNet takes the 4 latent
    channels and a depth channel and predicts the 4 latent channels: in_channels 5, out_channels 4
    (make_skeleton(..., depth=True))."""

    def __init__(self, census: List[BlockSpec], in_channels: int = 4, cross_attention_dim: int = 768,
                 hot_path_only: bool = True, max_downsample: Optional[int] = None, pnp_conv: bool = False,
                 transformer_io: Optional[str] = None, out_channels: Optional[int] = None):
        super().__init__()
        keep = [i for i, s in enumerate(census) if max_downsample is None or s.downsample <= max_downsample]
        self.census_index = keep                  # position of every block in the full census
        self.census = [census[i] for i in keep]
        self.mid_position = mid_position(census)
        self.in_channels = in_channels
        self.out_channels = in_channels if out_channels is None else out_channels
        self.blocks = nn.ModuleList(
            [BasicTransformerBlock(s.dim, s.heads, cross_attention_dim, hot_path_only) for s in self.census])
        dims = sorted({(s.downsample, s.dim) for s in self.census})
        self.lift = nn.ModuleDict({f"ds{ds}": nn.Linear(in_channels, dim) for ds, dim in dims})
        self.drop = nn.ModuleDict({f"ds{ds}": nn.Linear(dim, self.out_channels) for ds, dim in dims})
        self.resnet = None
        if pnp_conv:
            if PNP_CONV_POSITION not in keep:
                raise ValueError(f"pnp_conv=True needs census block {PNP_CONV_POSITION} (up_blocks[1]), which this "
                                 f"census / max_downsample leaves out")
            C = census[PNP_CONV_POSITION].dim
            self.resnet = ResnetBlock2D(2 * C, C, temb_channels=TEMB_CHANNELS)
        self.wrappers = _make_wrappers(self.blocks, self.census, transformer_io)

    def _run_resnet(self, state: torch.Tensor, skip: torch.Tensor, timestep, hw: Tuple[int, int]) -> torch.Tensor:
        """[(B F), T, C] state and skip -> the ResNet's [(B F), T, C] output (NCHW in and out with wrappers)."""
        BF = state.shape[0]
        temb = timestep_embedding(timestep, BF, TEMB_CHANNELS, state.device, state.dtype)
        if self.wrappers is not None:
            return self.resnet(torch.cat([state, skip], dim=1), temb)
        nchw = lambda t: t.transpose(1, 2).reshape(BF, -1, *hw).contiguous()   # noqa: E731  (NCHW, as diffusers)
        out = self.resnet(torch.cat([nchw(state), nchw(skip)], dim=1), temb)
        return out.flatten(2).transpose(1, 2).contiguous()

    def _residuals(self, down, mid) -> dict:
        """{census position: residual} of the encoder blocks; raises unless the residuals match them one-to-one."""
        down_pos = [p for p in self.census_index if p < self.mid_position]
        mid_pos = [p for p in self.census_index if p == self.mid_position]
        res = {}
        if down is not None:
            down = list(down)
            if len(down) != len(down_pos):
                raise ValueError(f"down_block_additional_residuals: {len(down)} residuals for the UNet's "
                                 f"{len(down_pos)} down blocks")
            res.update(zip(down_pos, down))
        if mid is not None:
            if not mid_pos:
                raise ValueError("mid_block_additional_residual: the UNet has no mid block")
            res[mid_pos[0]] = mid
        return res

    def forward(self, sample: torch.Tensor, timestep=None, encoder_hidden_states=None,
                down_block_additional_residuals=None, mid_block_additional_residual=None, **kwargs):
        BF, _, H, W = sample.shape
        state = {}
        eps = sample.new_zeros((BF, self.out_channels, H, W))
        res = self._residuals(down_block_additional_residuals, mid_block_additional_residual)
        skips = {}
        for i, (pos, spec, block) in enumerate(zip(self.census_index, self.census, self.blocks)):
            key = f"ds{spec.downsample}"
            ds = spec.downsample
            if key not in state:
                pooled = F.avg_pool2d(sample, spec.downsample) if spec.downsample > 1 else sample
                tok = pooled.flatten(2).transpose(1, 2)                       # [(B F), T, 4]
                state[key] = self.lift[key](tok)
                if self.wrappers is not None:
                    state[key] = _to_nchw(state[key], (H // ds, W // ds))
            if self.resnet is not None and pos == PNP_CONV_POSITION:
                state[key] = self._run_resnet(state[key], skips.get(key, state[key]), timestep, (H // ds, W // ds))
            if self.wrappers is not None:
                h = self.wrappers[i](state[key], encoder_hidden_states=encoder_hidden_states, timestep=timestep,
                                     return_dict=False)[0]
            else:
                h = block(state[key], encoder_hidden_states=encoder_hidden_states, timestep=timestep)
            if pos < self.mid_position:
                skips[key] = h
            if pos in res:
                if res[pos].shape != h.shape:
                    raise ValueError(f"additional residual for census block {pos}: shape {tuple(res[pos].shape)}, "
                                     f"the block's output is {tuple(h.shape)}")
                h = h + res[pos]
            state[key] = h
        for key, h in state.items():
            ds = int(key[2:])
            if self.wrappers is not None:
                h = _to_tokens(h)
            out = self.drop[key](h).transpose(1, 2).reshape(BF, self.out_channels, H // ds, W // ds)
            if ds > 1:
                out = F.interpolate(out, scale_factor=ds, mode="nearest")
            eps = eps + out
        return SimpleNamespace(sample=eps)


class ControlNetModel(ModelMixin):
    """Stand-in for diffusers' ControlNetModel, built the way SkeletonUNet stands in for the UNet: its blocks are the
    encoder half of the census (down blocks and mid block).  forward(latent [n, 4, h, w], t, encoder_hidden_states,
    controlnet_cond [n, 3, H, W]) -> (down_block_res_samples, mid_block_res_sample), one residual per block shaped like
    the block's output [n, T, C], which is what SkeletonUNet's additional-residual keywords take.

    The state of each resolution starts as the lifted latent (as in SkeletonUNet) plus the control image average-pooled
    to that resolution and lifted by a fixed linear map (the stand-in for the conditioning embedding); every block's
    output then goes through its own linear "zero conv".  The zero convs keep nn.Linear's random initialisation instead
    of zeros, so that the residuals are not all zero and their path shows in the UNet's prediction."""

    def __init__(self, census: List[BlockSpec], in_channels: int = 4, cond_channels: int = 3,
                 cross_attention_dim: int = 768, hot_path_only: bool = True, transformer_io: Optional[str] = None):
        super().__init__()
        mid = mid_position(census)
        self.census_index = list(range(mid + 1))
        self.census = census[:mid + 1]
        self.in_channels = in_channels
        self.blocks = nn.ModuleList(
            [BasicTransformerBlock(s.dim, s.heads, cross_attention_dim, hot_path_only) for s in self.census])
        dims = sorted({(s.downsample, s.dim) for s in self.census})
        self.lift = nn.ModuleDict({f"ds{ds}": nn.Linear(in_channels, dim) for ds, dim in dims})
        self.cond_lift = nn.ModuleDict({f"ds{ds}": nn.Linear(cond_channels, dim) for ds, dim in dims})
        self.zero_convs = nn.ModuleList([nn.Linear(s.dim, s.dim) for s in self.census])
        # as in SkeletonUNet: NCHW state, blocks called through their Transformer2DModel, NCHW residuals out
        self.wrappers = _make_wrappers(self.blocks, self.census, transformer_io)

    def forward(self, sample: torch.Tensor, timestep=None, encoder_hidden_states=None, controlnet_cond=None,
                return_dict: bool = False):
        n, _, h, w = sample.shape
        if controlnet_cond is None or controlnet_cond.dim() != 4 or controlnet_cond.shape[0] != n:
            raise ValueError(f"controlnet_cond must be [{n}, C, H, W] for a [{n}, ...] sample")
        ch, cw = controlnet_cond.shape[2:]
        f = ch // h
        if f < 1 or ch != f * h or cw != f * w:
            raise ValueError(f"controlnet_cond {tuple(controlnet_cond.shape[2:])} is not a whole multiple of the "
                             f"latent {h}x{w}")
        state, outs = {}, []
        for i, (spec, block, zero_conv) in enumerate(zip(self.census, self.blocks, self.zero_convs)):
            key, ds = f"ds{spec.downsample}", spec.downsample
            if key not in state:
                pooled = F.avg_pool2d(sample, ds) if ds > 1 else sample
                cpooled = F.avg_pool2d(controlnet_cond, f * ds) if f * ds > 1 else controlnet_cond
                state[key] = (self.lift[key](pooled.flatten(2).transpose(1, 2))
                              + self.cond_lift[key](cpooled.flatten(2).transpose(1, 2)))
                if self.wrappers is not None:
                    state[key] = _to_nchw(state[key], (h // ds, w // ds))
            if self.wrappers is not None:
                state[key] = self.wrappers[i](state[key], encoder_hidden_states=encoder_hidden_states,
                                              timestep=timestep, return_dict=False)[0]
                outs.append(_to_nchw(zero_conv(_to_tokens(state[key])), (h // ds, w // ds)))
                continue
            state[key] = block(state[key], encoder_hidden_states=encoder_hidden_states, timestep=timestep)
            outs.append(zero_conv(state[key]))
        down, mid = outs[:-1], outs[-1]
        if return_dict:
            return SimpleNamespace(down_block_res_samples=down, mid_block_res_sample=mid)
        return down, mid


# Census positions of the reference's PnP targets (utils/pnp_utils.py:97, RES_DICT = {1: [1, 2], 2: [0, 1, 2], 3: [0, 1, 2]}):
# up_blocks[1].attentions[1, 2], up_blocks[2].attentions[0..2] and up_blocks[3].attentions[0..2] are blocks 8 - 15 of
# the 16-block SD census (down 6, mid 1, up 9).
PNP_CENSUS_BLOCKS = range(8, 16)


def pnp_attention_modules(net: SkeletonUNet) -> List[nn.Module]:
    """The attn1 modules PnP controls (pnp.register_attention_control(modules=...)) for a skeleton built from the SD
    census; blocks that max_downsample left out are skipped."""
    return [b.attn1 for i, b in zip(net.census_index, net.blocks) if i in PNP_CENSUS_BLOCKS]


# diffusers' up_blocks[1].resnets[1], PnP's conv-injection target (utils/pnp_utils.py:168-169), runs right before
# up_blocks[1].attentions[1], census block 8.  SD's time embedding has 4 x 320 channels.
PNP_CONV_POSITION = 8
TEMB_CHANNELS = 1280


def pnp_conv_module(net: SkeletonUNet) -> nn.Module:
    """The ResNet PnP's conv injection controls (pnp.register_conv_control(modules=[...])) in a skeleton built with
    pnp_conv=True."""
    if getattr(net, "resnet", None) is None:
        raise ValueError("pnp_conv_module: the skeleton has no stand-in ResNet (make_skeleton(..., pnp_conv=True))")
    return net.resnet


def make_skeleton(name: str = "sd15", hot_path_only: bool = True, max_downsample: Optional[int] = None,
                  device="cuda", dtype=torch.float16, seed: int = 123, pnp_conv: bool = False,
                  transformer_io: Optional[str] = None, depth: bool = False) -> SkeletonUNet:
    """`depth=True`: the stand-in for SD2-depth's UNet (stabilityai/stable-diffusion-2-depth), which takes the latent
    with each frame's depth map appended as a fifth channel and predicts the 4 latent channels."""
    census = CENSUSES[name]()
    cad = 1024 if name == "sd21" else 768
    gen_state = torch.get_rng_state()
    torch.manual_seed(seed)
    try:
        net = SkeletonUNet(census, in_channels=5 if depth else 4, cross_attention_dim=cad, hot_path_only=hot_path_only,
                           max_downsample=max_downsample, pnp_conv=pnp_conv, transformer_io=transformer_io,
                           out_channels=4)
    finally:
        torch.set_rng_state(gen_state)
    return net.to(device=device, dtype=dtype).eval()


def make_controlnet(name: str = "sd15", hot_path_only: bool = True, device="cuda", dtype=torch.float16,
                    seed: int = 321, transformer_io: Optional[str] = None) -> ControlNetModel:
    """The ControlNet stand-in for make_skeleton(name): the encoder half of the same census, seeded the same way."""
    census = CENSUSES[name]()
    cad = 1024 if name == "sd21" else 768
    gen_state = torch.get_rng_state()
    torch.manual_seed(seed)
    try:
        net = ControlNetModel(census, cross_attention_dim=cad, hot_path_only=hot_path_only,
                              transformer_io=transformer_io)
    finally:
        torch.set_rng_state(gen_state)
    return net.to(device=device, dtype=dtype).eval()
