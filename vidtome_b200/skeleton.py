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
    """forward(latent [(B F), 4, h, w], t, encoder_hidden_states) -> object with `.sample` of the latent's
    shape.  For every block: the latent is average-pooled to the block's resolution, lifted to `dim`
    channels by a fixed linear map, added to the running state of that resolution, run through the block,
    and projected back into the noise prediction.

    `down_block_additional_residuals` / `mid_block_additional_residual` (a ControlNet's outputs) are added to the output
    state of the matching encoder block, the skeleton's stand-in for diffusers' skip-sample add: one residual per down
    block in block order, one for the mid block, each shaped like that block's output [(B F), T, C]."""

    def __init__(self, census: List[BlockSpec], in_channels: int = 4, cross_attention_dim: int = 768,
                 hot_path_only: bool = True, max_downsample: Optional[int] = None):
        super().__init__()
        keep = [i for i, s in enumerate(census) if max_downsample is None or s.downsample <= max_downsample]
        self.census_index = keep                  # position of every block in the full census
        self.census = [census[i] for i in keep]
        self.mid_position = mid_position(census)
        self.in_channels = in_channels
        self.blocks = nn.ModuleList(
            [BasicTransformerBlock(s.dim, s.heads, cross_attention_dim, hot_path_only) for s in self.census])
        dims = sorted({(s.downsample, s.dim) for s in self.census})
        self.lift = nn.ModuleDict({f"ds{ds}": nn.Linear(in_channels, dim) for ds, dim in dims})
        self.drop = nn.ModuleDict({f"ds{ds}": nn.Linear(dim, in_channels) for ds, dim in dims})

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
        BF, Cin, H, W = sample.shape
        state = {}
        eps = torch.zeros_like(sample)
        res = self._residuals(down_block_additional_residuals, mid_block_additional_residual)
        for pos, spec, block in zip(self.census_index, self.census, self.blocks):
            key = f"ds{spec.downsample}"
            if key not in state:
                pooled = F.avg_pool2d(sample, spec.downsample) if spec.downsample > 1 else sample
                tok = pooled.flatten(2).transpose(1, 2)                       # [(B F), T, 4]
                state[key] = self.lift[key](tok)
            h = block(state[key], encoder_hidden_states=encoder_hidden_states, timestep=timestep)
            if pos in res:
                if res[pos].shape != h.shape:
                    raise ValueError(f"additional residual for census block {pos}: shape {tuple(res[pos].shape)}, "
                                     f"the block's output is {tuple(h.shape)}")
                h = h + res[pos]
            state[key] = h
        for key, h in state.items():
            ds = int(key[2:])
            out = self.drop[key](h).transpose(1, 2).reshape(BF, Cin, H // ds, W // ds)
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
                 cross_attention_dim: int = 768, hot_path_only: bool = True):
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
        for spec, block, zero_conv in zip(self.census, self.blocks, self.zero_convs):
            key, ds = f"ds{spec.downsample}", spec.downsample
            if key not in state:
                pooled = F.avg_pool2d(sample, ds) if ds > 1 else sample
                cpooled = F.avg_pool2d(controlnet_cond, f * ds) if f * ds > 1 else controlnet_cond
                state[key] = (self.lift[key](pooled.flatten(2).transpose(1, 2))
                              + self.cond_lift[key](cpooled.flatten(2).transpose(1, 2)))
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


def make_skeleton(name: str = "sd15", hot_path_only: bool = True, max_downsample: Optional[int] = None,
                  device="cuda", dtype=torch.float16, seed: int = 123) -> SkeletonUNet:
    census = CENSUSES[name]()
    cad = 1024 if name == "sd21" else 768
    gen_state = torch.get_rng_state()
    torch.manual_seed(seed)
    try:
        net = SkeletonUNet(census, cross_attention_dim=cad, hot_path_only=hot_path_only,
                           max_downsample=max_downsample)
    finally:
        torch.set_rng_state(gen_state)
    return net.to(device=device, dtype=dtype).eval()


def make_controlnet(name: str = "sd15", hot_path_only: bool = True, device="cuda", dtype=torch.float16,
                    seed: int = 321) -> ControlNetModel:
    """The ControlNet stand-in for make_skeleton(name): the encoder half of the same census, seeded the same way."""
    census = CENSUSES[name]()
    cad = 1024 if name == "sd21" else 768
    gen_state = torch.get_rng_state()
    torch.manual_seed(seed)
    try:
        net = ControlNetModel(census, cross_attention_dim=cad, hot_path_only=hot_path_only)
    finally:
        torch.set_rng_state(gen_state)
    return net.to(device=device, dtype=dtype).eval()
