"""Patch layer — the drop-in boundary.  Same API as the reference's vidtome/patch.py:
`apply_patch / remove_patch / update_patch / collect_from_patch`, the `_tome_info` dict, the
`module.generator` / `module.global_tokens` attributes and the `ToMeBlock` class swap (patch.py:206-387).

What differs from the reference is inside `compute_merge` and the self-attention section of
`ToMeBlock.forward` (patch.py:14-91, :139-169):
  * every matching level runs as CUDA kernels through the C-ABI (merge.match_level);
  * the per-level merge/unmerge closures are never chained: their int32 index maps are composed on the
    device (KB2), so the merged tokens are produced by ONE row gather of the block input (KC) and the
    unmerge + split_frame + residual add is ONE gather-add pass (KE);
  * `module.global_tokens` stays in HBM (the reference parks it on the CPU, patch.py:80,82).
The RNG protocol is unchanged: one `torch.randint` per local level and one `torch.rand` per block when
global tokens exist, drawn from `module.generator` on the generator's device (merge.py:56-57, patch.py:62).
"""
from __future__ import annotations

import contextlib
import math
from dataclasses import dataclass, field
from typing import Any, Callable, Dict, List, Optional, Tuple, Type

import torch

from . import attention, feedforward, merge, ops
from ._lib import VtmSplit
from .utils import (draw_coin, draw_randf, func_warper, init_generator, isinstance_str, join_frame, join_warper,
                    split_frame, split_warper)


@dataclass
class MergePlan:
    """Composed result of compute_merge for one block call."""
    fsize: int
    N0: int                               # F * T tokens per sample before merging
    merged_tokens: torch.Tensor           # [B, L, C] fp16, input of attn1
    pi: torch.Tensor                      # [B'|1, N0] int32: out[b, p] = y[b, pi[b, p]]
    levels: List[merge.LevelMatch] = field(default_factory=list)
    randf: List[Any] = field(default_factory=list)      # ints (eager) or 1-element int32 CUDA tensors (graph capture)
    coin: Any = None                      # float (host coin) or 1-element fp32 CUDA tensor (device coin, DEVICE_COIN / capture)
    mu: Optional[torch.Tensor] = None     # [B'|1, L_local] int32: local merged token i = table row mu[i] (before a global stage)
    # GlobalTokenStore stage: merged_tokens is sized for capacity and its first seq_len rows (a 1-element int32 CUDA
    # tensor) are the merged sequence; KD reads the length on the device
    seq_len: Optional[torch.Tensor] = None

    def unmerge(self, y: torch.Tensor, **kwarg) -> torch.Tensor:
        """u_a of the reference (patch.py:85,168): all unmerges + split_frame, one gather pass."""
        out = ops.unmerge_add(y.contiguous(), self.pi, None)
        return split_frame(out, self.fsize)

    def unmerge_add(self, y: torch.Tensor, hidden_states: torch.Tensor) -> torch.Tensor:
        """patch.py:168-169 fused: u_a(attn_output) + hidden_states in one pass (KE)."""
        resid = join_frame(hidden_states.contiguous(), self.fsize)
        out = ops.unmerge_add(y.contiguous(), self.pi, resid)
        return split_frame(out, self.fsize)


# Fuse a plain nn.LayerNorm norm1 into the K0 / KC kernels (its output is then never materialised).
FUSE_LAYERNORM = True

# Run a stock GEGLU feed-forward (norm3 + ff + residual, patch.py:187-199) through the CUDA kernels (feedforward.py).
FUSE_FEED_FORWARD = True
# Run a stock cross-attention (norm2 + attn2 + residual, patch.py:171-185) through the CUDA library (attention.py).
FUSE_CROSS_ATTENTION = True

# Run the entry and exit of every diffusers Transformer2DModel of a patched model (GroupNorm -> proj_in -> token-major
# rows, and proj_out -> NCHW + residual) through the CUDA library (transformer2d.py); modules it cannot serve keep their
# own forward (transformer2d.ineligibility).
FUSE_TRANSFORMER_IO = True

# How `merge_global=True` obtains the global token set when several ranks each hold one chunk:
#   "recurrence" — the reference's semantics (patch.py:59-82): whatever the previous chunk processed by THIS
#                  process left in module.global_tokens;
#   "allgather"  — chunk-per-GPU variant (SURVEY §8e, option A): one NCCL all-gather of the local merged tokens
#                  per merged block; rank k matches against the tokens of rank (k-1) mod G (dist.py);
#   "p2p"        — the same exchange fused into the kernel that produces the tokens: KC stores each merged row into
#                  the peer-mapped buffer of its consumer, rank k+1, over NVLink (one barrier, no collective pass);
#   "p2p_all"    — as "p2p" but into every rank's buffer (all-gather semantics; 7x the bytes on 8 GPUs).
GLOBAL_EXCHANGE = "recurrence"

# Keep the global stage's coin (patch.py:62) on the device, as CUDA-graph capture always does: the local and global
# token sets sit in one buffer in a fixed order and the kernels read the coin to pick which half is src
# (VtmSplit.prefix_coin), so nothing is read back to the host.  Results are bit-identical to the host coin.  It needs
# both sets to be equally long (equal chunks); eagerly, a block whose sets differ keeps the host coin.
DEVICE_COIN = False

# Run the self-attention of every block that does not merge at this call (block_merges) through the CUDA library during
# generation too: norm1 -> KD with the residual in its out projection, as inside _unmerged_blocks(), for a stock attn1
# (_plain_attention_module) up to attention.MAX_HEAD_DIM.  PnP-marked modules included: while their injection is active
# item b of the [source | uncond | cond] frame batch uses the attention map of item b mod (B / num_inputs)
# (vtm_attention_residual_ex).  Off by default: the library's flash kernel takes its softmax in fp32 where the module's
# own forward rounds it in fp16 (torch's `softmax` / SDPA), so these blocks' results change within fp16 tolerance.
# Read on every call, so it may be changed at any time.
FUSE_UNMERGED_ATTENTION = False

# Run the transformer blocks and Transformer2DModel wrappers of a model that apply_patch did not patch, and that
# serve_unmerged served (the step driver and the inverter serve an unpatched ControlNet while this is on), through the
# library, always unmerged: every block takes the path of a patched block inside _unmerged_blocks() (fused norm1 -> KD
# with the residual in its out projection, norm2 -> cross-attention, norm3 -> GEGLU -> residual projection) and every
# wrapper the library's entry and exit.  Off by default for the reason FUSE_UNMERGED_ATTENTION is: the flash kernel
# takes its softmax in fp32, so results change within fp16 tolerance against the modules' own forwards.  Read on every
# call; while it is off a served module runs its own forward.
FUSE_CONTROLNET_BLOCKS = False

# Depth of _unmerged_blocks() contexts: while > 0 every ToMeBlock runs as the reference's UNPATCHED block.
_UNMERGED = 0


@contextlib.contextmanager
def _unmerged_blocks():
    """Run patched models as the reference runs them before apply_patch, for DDIM inversion (invert.py:117-140 runs
    first, on the unpatched UNet; SURVEY App. C.13).  Inside, a ToMeBlock builds no merge plan (nothing is drawn,
    `global_tokens` is left alone), its pre-hook forks no generator, and no PnP injection runs whatever `t` the marked
    modules hold (pnp.injection_active).  attn1 of a stock module (_plain_attention_module) runs as norm1 -> KD with the
    residual in its out projection (vtm_attention_residual_ex), PnP-marked modules included; any other attn1 runs its own
    forward.  attn2 and ff go through the library as they do outside."""
    global _UNMERGED
    _UNMERGED += 1
    try:
        yield
    finally:
        _UNMERGED -= 1


def unmerged_active() -> bool:
    """True inside _unmerged_blocks()."""
    return _UNMERGED > 0


class GlobalTokenStore:
    """A block's global tokens at a fixed address: `tokens` [B, cap, C] fp16 and their count `length` (a 1-element int32
    CUDA tensor), allocated once, eagerly, outside any CUDA-graph pool.  Set it as `module.global_tokens` and
    build_merge_plan runs the global stage of patch.py:59-82 with the counts that depend on the coin kept on the device
    (VtmSplit.prefix_coin_dev), eagerly or under capture, so that chunks of different lengths can follow each other in
    one captured sequence.  `cap` is the local merged length of a chunk of `max_frames` frames.  `filled` is the host's
    knowledge of whether the store holds tokens (the reference's `global_tokens is not None`); `reset()` empties it,
    as `update_patch(global_tokens=None)` does for a plain tensor."""

    def __init__(self, max_frames: int):
        if not isinstance(max_frames, int) or max_frames <= 0:
            raise ValueError(f"GlobalTokenStore: max_frames must be a positive int, got {max_frames!r}")
        self.max_frames = max_frames
        self.tokens: Optional[torch.Tensor] = None
        self.length: Optional[torch.Tensor] = None
        self.filled = False

    @property
    def cap(self) -> int:
        return 0 if self.tokens is None else self.tokens.shape[1]

    def reset(self) -> None:
        """Empty the store (host state only: `length` is meaningful while `filled`, and the next write sets it)."""
        self.filled = False

    def ensure(self, B: int, C: int, tsize: int, args: Dict[str, Any], device) -> None:
        if self.tokens is not None and tuple(self.tokens.shape[::2]) == (B, C) and self.tokens.device == device:
            return
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("GlobalTokenStore: the store is allocated by an eager call, before any capture")
        cap = local_merged_len(self.max_frames, tsize, args)
        self.tokens = torch.zeros((B, cap, C), dtype=torch.float16, device=device)
        self.length = torch.zeros(1, dtype=torch.int32, device=device)
        self.filled = False

    def write(self, rows: torch.Tensor) -> None:
        """global_tokens <- rows [B, L, C] (L <= cap): the first L rows and the length."""
        self.tokens[:, :rows.shape[1]].copy_(rows)
        self.length.fill_(rows.shape[1])
        self.filled = True


def local_merged_len(frames: int, tsize: int, args: Dict[str, Any]) -> int:
    """Length of the local merged token set of a chunk of `frames` frames of `tsize` tokens (the counts of
    build_merge_plan's local levels, computed on the host; with F % stride != 0 they assume the draw randf = 0)."""
    L, unm, curF = frames * tsize, 0, frames
    ratio = args["local_merge_ratio"]
    while curF > 1:
        if ratio <= 0:
            unm += (L - unm) // curF
        else:
            ns, nd = ops.split_counts(VtmSplit.local(L, unm, curF, args["target_stride"], 0))
            r = ops.merge_count(ns, ratio)
            unm += ns - r
            L = ns - r + nd
        curF = (L - unm) // tsize
    return L


def _global_stage_store(module, store: GlobalTokenStore, table, mu, pi, ln, args, levels, tsize):
    """patch.py:59-82 on a GlobalTokenStore.  As in _global_stage_device_coin the sets are stored as cat = [local (L
    rows) | global (store.cap rows, the first *store.length valid)] and the coin picks the src half, but the lengths may
    differ, so Ns, Nd, r and the merged length M are derived and read on the device (VtmSplit.prefix_coin_dev).  The
    merged tokens are [B, L + cap, C], zero past M.  Returns (merged tokens, composed unmerge map, coin, M tensor)."""
    B, _, C = table.shape
    L = mu.shape[1]
    store.ensure(B, C, tsize, args, table.device)
    if L > store.cap:
        raise RuntimeError(f"GlobalTokenStore: {L} local tokens exceed the store's capacity of {store.cap} "
                           f"(max_frames={store.max_frames})")
    if not store.filled:                                                    # patch.py:81-82: no global tokens yet
        local = ops.gather_rows(table, mu, ln=ln)
        store.write(local)
        return local, pi, None, None
    coin = draw_coin(module.generator, on_device=True)                      # patch.py:62
    gratio = args["global_merge_ratio"]
    if gratio <= 0:
        raise ValueError("not enough values to unpack (expected 3, got 2)")  # as the host-coin path
    cap = store.cap
    cat = torch.empty((B, L + cap, C), dtype=torch.float16, device=table.device)
    ops.gather_rows(table, mu, ln=ln, out=cat[:, :L])                       # merged local tokens, straight into cat
    cat[:, L:].copy_(store.tokens)
    split = VtmSplit.prefix_coin_dev(L, store.length, cap, coin, args["global_rand"])
    m = merge.match_level_dev(cat, split, gratio, bool(args["align_batch"]))   # patch.py:73-74
    levels.append(m)
    merged_len = m.counts[3:4]
    mu_g, tau = ops.compose_maps_dev(split, m.counts, m.keys, m.edge, m.rank, None, L + cap)
    merged_tokens = ops.gather_rows_dev(cat, mu_g, merged_len)             # patch.py:75
    if pi.shape[0] != tau.shape[0]:
        pi = pi.expand(tau.shape[0], -1).contiguous()
    _, pi = ops.compose_maps_dev(split, m.counts, m.keys, m.edge, m.rank, pi, pi.shape[1])
    # patch.py:80, the local half.  Last: the split reads the global length from the store, which this rewrites.
    store.write(ops.unmerge_add(merged_tokens, tau[:, :L], None))
    return merged_tokens, pi, coin, merged_len


def _fusable_layer_norm(norm: torch.nn.Module, x: torch.Tensor):
    """(weight, bias, eps) if `norm` is a stock affine nn.LayerNorm over the channel dim in fp16, else None."""
    if not FUSE_LAYERNORM or type(norm) is not torch.nn.LayerNorm or not norm.elementwise_affine:
        return None
    if tuple(norm.normalized_shape) != (x.shape[-1],) or norm.weight.dtype != torch.float16 or not norm.weight.is_cuda:
        return None
    return (norm.weight.contiguous(), None if norm.bias is None else norm.bias.contiguous(), float(norm.eps))


def _global_stage_device_coin(module, table, mu, pi, g, ln, args, levels):
    """patch.py:60-80 with the coin left on the device.  The reference concatenates [local | global] or
    [global | local] depending on the coin; here both sets are stored once as cat = [local (L rows) | global (L rows)]
    and the coin picks which half is src (VtmSplit.prefix_coin).  Src row i and dst row j name the same tokens as in
    the reference's concatenation, so the match, the merged tokens and the unmerge are the same; only positions are
    numbered in storage order, which is what makes the local tokens' unmerge map tau[:, :L] independent of the coin.
    Returns (merged tokens, composed unmerge map, coin tensor)."""
    B, _, C = table.shape
    L = mu.shape[1]
    coin = draw_coin(module.generator, on_device=True)                      # patch.py:62
    gratio = args["global_merge_ratio"]
    if gratio <= 0:
        raise ValueError("not enough values to unpack (expected 3, got 2)")  # as the host-coin path
    cat = torch.empty((B, 2 * L, C), dtype=torch.float16, device=table.device)
    ops.gather_rows(table, mu, ln=ln, out=cat[:, :L])                       # merged local tokens, straight into cat
    cat[:, L:].copy_(g)                                                     # the stored global tokens
    split = VtmSplit.prefix_coin(L, coin, args["global_rand"])
    m = merge.match_level(cat, None, split, gratio, bool(args["align_batch"]))   # patch.py:73-74
    levels.append(m)
    # tau: position in cat -> position in the merged sequence
    mu_g, tau = ops.compose_maps(split, m.r, m.keys, m.edge, m.rank, None, None, 0, 2 * L)
    merged_tokens = ops.gather_rows(cat, mu_g)                               # patch.py:75
    # patch.py:80: global_tokens <- u(merged_tokens), the local half after unmerging (kept on the device)
    module.global_tokens = ops.unmerge_add(merged_tokens, tau[:, :L], None)
    # compose with the local unmerge: pi_total[p] = tau[pi[p]]
    if pi.shape[0] != tau.shape[0]:
        pi = pi.expand(tau.shape[0], -1).contiguous()
    _, pi = ops.compose_maps(split, m.r, m.keys, m.edge, m.rank, None, pi, 0, pi.shape[1])
    return merged_tokens, pi, coin


def block_merges(x: torch.Tensor, tome_info: Dict[str, Any]) -> bool:
    """Whether a block whose input `x` has x.shape[1] tokens per item merges at this call: its downsampling of the
    latent recorded in tome_info["size"] is at most max_downsample (patch.py:15-17,27,86-88).  Decided before anything
    is drawn from the block's generator."""
    original_h, original_w = tome_info["size"]
    original_tokens = original_h * original_w
    downsample = int(math.ceil(math.sqrt(original_tokens // x.shape[1])))    # patch.py:15-17
    return downsample <= tome_info["args"]["max_downsample"]


def build_merge_plan(module: torch.nn.Module, x: torch.Tensor, tome_info: Dict[str, Any],
                     ln=None) -> Optional[MergePlan]:
    """The body of compute_merge (vidtome/patch.py:14-91).  Returns None when the block is not merged
    (block_merges).  With `ln = (weight, bias, eps)`, `x` is the RAW hidden state and norm1 is applied inside the
    kernels that read it (K0, KC)."""
    if not block_merges(x, tome_info):
        return None
    args = tome_info["args"]
    merge._check_metric(x)
    generator = module.generator
    fsize = x.shape[0] // args["batch_size"]                                 # patch.py:23
    tsize = x.shape[1]                                                       # patch.py:24
    align = bool(args["align_batch"])

    table = join_frame(x.contiguous(), fsize)                                # patch.py:37 (view)
    B, N0, C = table.shape
    mu: Optional[torch.Tensor] = None      # position -> row of `table` (None = identity)
    pi: Optional[torch.Tensor] = None      # level-0 position -> current position (None = identity)
    L, unm, curF = N0, 0, fsize
    levels: List[merge.LevelMatch] = []
    randfs: List[int] = []
    ratio = args["local_merge_ratio"]
    while curF > 1:                                                          # patch.py:44
        if ratio <= 0:
            unm += (L - unm) // curF                                         # merge.py:45-46 (no draw)
        else:
            stride = min(args["target_stride"], curF)                        # merge.py:55
            randf = draw_randf(generator, stride, curF)                      # merge.py:56-57
            randfs.append(randf)
            split = VtmSplit.local(L, unm, curF, args["target_stride"], randf)
            m = merge.match_level(table, mu, split, ratio, align, ln)        # patch.py:45-46
            mu, pi = ops.compose_maps(split, m.r, m.keys, m.edge, m.rank, mu, pi, 0, N0)
            levels.append(m)
            unm += m.unm_num                                                 # patch.py:47
            L = mu.shape[1]                                                  # patch.py:50
        curF = (L - unm) // tsize                                            # patch.py:54

    if mu is None:   # nothing merged (single frame or ratio <= 0): identity maps
        mu = torch.arange(N0, dtype=torch.int32, device=x.device)[None]
        pi = mu
    coin = None
    if args["merge_global"]:                                                 # patch.py:59
        g = getattr(module, "global_tokens", None)
        if isinstance(g, GlobalTokenStore):
            if GLOBAL_EXCHANGE != "recurrence":
                raise RuntimeError(f"GlobalTokenStore needs GLOBAL_EXCHANGE='recurrence' (got {GLOBAL_EXCHANGE!r}): "
                                   f"the cross-rank exchange modes keep their own global tokens")
            merged_tokens, pi, coin, seq_len = _global_stage_store(module, g, table, mu, pi, ln, args, levels, tsize)
            return MergePlan(fsize=fsize, N0=N0, merged_tokens=merged_tokens, pi=pi, levels=levels, randf=randfs,
                             coin=coin, mu=mu, seq_len=seq_len)
        if x.is_cuda and torch.cuda.is_current_stream_capturing():
            if GLOBAL_EXCHANGE != "recurrence":
                raise RuntimeError(f"CUDA-graph capture of global merging needs GLOBAL_EXCHANGE='recurrence' (got "
                                   f"{GLOBAL_EXCHANGE!r}): the cross-rank exchange is not captured")
            if g is not None and g.shape[1] != L:
                raise RuntimeError(f"CUDA-graph capture of global merging needs chunks of equal length, i.e. a frame "
                                   f"count divisible by the chunk size (got {L} local and {g.shape[1]} global tokens): "
                                   f"token counts would depend on the draw")
            device_coin = True
        else:
            device_coin = DEVICE_COIN and GLOBAL_EXCHANGE == "recurrence" and g is not None and g.shape[1] == L
        if device_coin and g is not None:
            merged_tokens, pi, coin = _global_stage_device_coin(module, table, mu, pi, g, ln, args, levels)
            return MergePlan(fsize=fsize, N0=N0, merged_tokens=merged_tokens, pi=pi, levels=levels, randf=randfs,
                             coin=coin, mu=mu)
        exchanged = False
        local_tokens = None
        if GLOBAL_EXCHANGE in ("allgather", "p2p", "p2p_all"):
            from . import dist as _dist
            if _dist.world() > 1:
                # "KF" = the merge gather together with the exchange (bench.py brackets it with CUDA events): bytes that
                # cross NVLink per rank = (G - 1) * B * L * C * 2 in either mode (SURVEY §8d)
                fan = 1 if GLOBAL_EXCHANGE == "p2p" else _dist.world() - 1
                nvl = 2.0 * fan * B * mu.shape[1] * C
                with ops._Timed("KF", 0.0, nvl):
                    if GLOBAL_EXCHANGE in ("p2p", "p2p_all"):
                        # KC stores the merged tokens straight into the consumer's ("p2p": rank k+1) or every rank's
                        # ("p2p_all") symmetric buffer: no separate collective pass
                        local_tokens, g = _dist.exchange_fused(table, mu, ln=ln, everyone=GLOBAL_EXCHANGE == "p2p_all")
                    else:
                        local_tokens = ops.gather_rows(table, mu, ln=ln)
                        g = _dist.exchange_global_tokens(local_tokens)      # the one collective of this path
                exchanged = True
        if local_tokens is None:
            local_tokens = ops.gather_rows(table, mu, ln=ln)                 # merged local tokens [B, L, C]
        if g is not None:                                                    # patch.py:60
            coin = draw_coin(generator, on_device=False)                     # patch.py:62
            g = g.to(local_tokens).contiguous()                              # patch.py:65,70
            Lg = g.shape[1]
            if coin > args["global_rand"]:
                src_len, tokens, off = L, torch.cat([local_tokens, g], dim=1), 0          # patch.py:63-66
            else:
                src_len, tokens, off = Lg, torch.cat([g, local_tokens], dim=1), Lg        # patch.py:68-71
            gratio = args["global_merge_ratio"]
            if gratio <= 0:
                # merge.py:364-365 returns two values and patch.py:73 unpacks three
                raise ValueError("not enough values to unpack (expected 3, got 2)")
            split = VtmSplit.prefix(L + Lg, src_len)
            m = merge.match_level(tokens, None, split, gratio, align)        # patch.py:73-74
            levels.append(m)
            # tau: position in `tokens` -> position in the merged sequence (the 2s unmerge as a map)
            mu_g, tau = ops.compose_maps(split, m.r, m.keys, m.edge, m.rank, None, None, 0, L + Lg)
            merged_tokens = ops.gather_rows(tokens, mu_g)                    # patch.py:75
            # patch.py:80: global_tokens <- u(merged_tokens), the local partition after unmerging;
            # kept on the device instead of .cpu()
            tau_local = tau[:, off:off + L].contiguous()
            if not exchanged:
                module.global_tokens = ops.unmerge_add(merged_tokens, tau_local, None)
            # compose with the local unmerge: pi_total[p] = tau[off + pi[p]]
            if pi.shape[0] != tau.shape[0]:
                pi = pi.expand(tau.shape[0], -1)
            pi = torch.gather(tau, 1, (pi.long() + off)).to(torch.int32).contiguous()
        else:
            merged_tokens = local_tokens
            module.global_tokens = local_tokens.detach().clone()            # patch.py:82
    else:
        merged_tokens = ops.gather_rows(table, mu, ln=ln)                    # patch.py:50,56 composed
    return MergePlan(fsize=fsize, N0=N0, merged_tokens=merged_tokens, pi=pi, levels=levels, randf=randfs,
                     coin=coin, mu=mu)


def compute_merge(module: torch.nn.Module, x: torch.Tensor, tome_info: Dict[str, Any]) -> Tuple[Callable, ...]:
    """Reference signature and return triple (patch.py:14,91): (merge op, unmerge op, merged tokens).
    The merge op is returned for interface parity only — like the reference's diffusers block
    (patch.py:149-152) nothing here calls it: the merged tokens are already the third element."""
    plan = build_merge_plan(module, x, tome_info)
    if plan is None:
        return merge.do_nothing, merge.do_nothing, x                         # patch.py:86-88
    merged = plan.merged_tokens

    def m(_x: torch.Tensor, **kwarg) -> torch.Tensor:
        return merged
    def u(y: torch.Tensor, **kwarg) -> torch.Tensor:
        return plan.unmerge(y)
    m.plan = u.plan = plan
    return m, u, merged


def _plain_attention_module(attn: torch.nn.Module) -> bool:
    """True only if replacing `attn.forward` by KD cannot change the result: `attn` is a stock Attention
    (attention.stock_attention_parts; LoRA-adapted projections run as extra K steps of KD's projection GEMMs) with no
    instance-level forward override other than PnP's (utils/pnp_utils.py:99-101), to_q / to_k / to_v / to_out[0] all
    [C, C], and heads KD runs (attention.head_dim_fits).  Anything else goes through `self.attn1(...)` exactly as the
    reference does (patch.py:157-162), e.g. after `pipe.load_lora_weights` (generate.py:93-94)."""
    override = vars(attn).get("forward")
    if override is not None and not getattr(override, "_vtm_pnp_forward", False):
        return False                       # someone else's replaced forward (e.g. the reference's own PnP closure)
    parts = attention.stock_attention_parts(attn)
    if parts is None:
        return False
    wq, wk, wv, wo = (p[0] for p in parts)
    C = wq.shape[1]
    if wq.shape[0] != C or wk.shape != wq.shape:
        return False                       # inner dim != query dim or cross-attention shaped K/V
    if wv.shape != wq.shape or wo.shape != (C, C):
        return False
    return attention.head_dim_fits(attn, C)


def _pnp_shared_items(attn: torch.nn.Module, batch: int) -> Optional[int]:
    """While PnP injects into `attn` (pnp.injection_active; the batch is num_inputs runs of [source | uncond | cond]
    items): how many items lead, item b taking the attention map of item b mod that count (batch / num_inputs), or 0 if
    the batch is not a whole number of runs.  None when nothing is injected."""
    num_inputs = getattr(attn, "_vtm_pnp", 0)
    if not num_inputs:
        return None
    from . import pnp
    if not pnp.injection_active(attn):                                    # never inside _unmerged_blocks()
        return None
    return 0 if batch % num_inputs else batch // num_inputs


def _self_attention_stage(block, hidden_states, attention_mask, encoder_hidden_states, timestep, class_labels,
                          cross_attention_kwargs):
    """norm1 -> [merge] -> attn1 -> [unmerge] + residual (patch.py:139-169).  Returns the hidden states and, for an
    AdaNorm-zero norm1, its (shift_mlp, scale_mlp, gate_mlp) for the feed-forward, else None."""
    unmerged = _UNMERGED > 0 or block._vtm_unmerged
    only_cross = getattr(block, "only_cross_attention", False)

    def library_attn1(route) -> bool:
        # attn1 runs in the library (KD): no mask, no kwargs, a stock module; `route()` is the route's own condition
        return (attention.ENABLED and not only_cross and attention_mask is None and not cross_attention_kwargs
                and route() and _plain_attention_module(block.attn1))

    if (hidden_states.is_cuda and hidden_states.dtype == torch.float16 and not block.use_ada_layer_norm
            and not block.use_ada_layer_norm_zero
            and library_attn1(lambda: unmerged or (FUSE_UNMERGED_ATTENTION
                                                   and not block_merges(hidden_states, block._tome_info)))):
        ln1 = _fusable_layer_norm(block.norm1, hidden_states)
        shared_items = None if ln1 is None else _pnp_shared_items(block.attn1, hidden_states.shape[0])
        if ln1 is not None and shared_items != 0:   # else the module's forward, which fails as the reference's
            # a block that does not merge (_unmerged_blocks, or FUSE_UNMERGED_ATTENTION): attn1(norm1(h)) + h, the add
            # in the out projection of KD; with PnP injecting, item b takes the map of item b mod shared_items
            shape = hidden_states.shape
            hidden_states = hidden_states.contiguous()
            n1 = ops.layer_norm(hidden_states.view(-1, shape[-1]), ln1).view(shape)
            return attention.self_attention_residual(block.attn1, n1, hidden_states, shared_items=shared_items), None

    plan = None
    mlp_terms = None
    if block.use_ada_layer_norm:                                                  # patch.py:139-146
        norm_hidden_states = block.norm1(hidden_states, timestep)
    elif block.use_ada_layer_norm_zero:
        norm_hidden_states, gate_msa, *mlp_terms = block.norm1(hidden_states, timestep, class_labels,
                                                               hidden_dtype=hidden_states.dtype)
    else:
        ln = _fusable_layer_norm(block.norm1, hidden_states) if hidden_states.is_cuda and not unmerged else None
        if ln is not None:
            # norm1 fused into the merge kernels: only the kept rows are ever normalised
            plan = build_merge_plan(block, hidden_states, block._tome_info, ln=ln)
        norm_hidden_states = None if plan is not None else block.norm1(hidden_states)

    if plan is None and not unmerged:
        plan = build_merge_plan(block, norm_hidden_states, block._tome_info)   # patch.py:149-150
    if plan is not None:
        norm_hidden_states = plan.merged_tokens

    # 1. Self-Attention (patch.py:154-162)
    if library_attn1(lambda: plan is not None):
        # KD; with PnP control registered (pnp.py) and the timestep inside the injection schedule, the attention map of
        # the source sample is applied to every sample's values (utils/pnp_utils.py:57-68, 87-91)
        shared_items = _pnp_shared_items(block.attn1, norm_hidden_states.shape[0])
        if shared_items not in (None, 1):
            raise RuntimeError("PnP injection needs one merged token set per input (batch_size == num_inputs)")
        attn_output = attention.self_attention(block.attn1, norm_hidden_states, shared_qk=shared_items == 1,
                                               seq_len=plan.seq_len)                                      # KD
    elif plan is not None and plan.seq_len is not None:
        raise RuntimeError("GlobalTokenStore: the merged tokens are sized for capacity with their length on the device, "
                           "which only the library's self-attention (KD) reads; this block's attn1 runs its own forward")
    else:
        attn_output = block.attn1(norm_hidden_states, encoder_hidden_states=encoder_hidden_states if only_cross else None,
                                  attention_mask=attention_mask, **cross_attention_kwargs)
    if block.use_ada_layer_norm_zero:
        attn_output = gate_msa.unsqueeze(1) * attn_output                        # patch.py:164-165

    # Unmerge + residual (patch.py:168-169), fused into one pass
    if plan is not None:
        return plan.unmerge_add(attn_output, hidden_states), mlp_terms
    return attn_output + hidden_states, mlp_terms


def _cross_attention_stage(block, hidden_states, encoder_hidden_states, encoder_attention_mask, timestep,
                           cross_attention_kwargs):
    """norm2 -> attn2 + residual (patch.py:171-185)."""
    attn2 = getattr(block, "attn2", None)
    if attn2 is None:
        return hidden_states
    if (FUSE_CROSS_ATTENTION and hidden_states.is_cuda and not block.use_ada_layer_norm
            and encoder_attention_mask is None and not cross_attention_kwargs
            and attention.cross_attention_eligible(attn2, encoder_hidden_states)
            and encoder_hidden_states.shape[0] == hidden_states.shape[0]):
        ln2 = _fusable_layer_norm(block.norm2, hidden_states)
        if ln2 is not None:
            # norm2 -> q / kv projections (head-major) -> flash attention over the context -> out projection with bias
            # and residual fused, all in the CUDA library
            shape = hidden_states.shape
            n2 = ops.layer_norm(hidden_states.contiguous().view(-1, shape[-1]), ln2).view(shape)
            return attention.cross_attention_residual(attn2, n2, encoder_hidden_states, hidden_states)
    norm_hidden_states = block.norm2(hidden_states, timestep) if block.use_ada_layer_norm else block.norm2(hidden_states)
    attn_output = attn2(norm_hidden_states, encoder_hidden_states=encoder_hidden_states,
                        attention_mask=encoder_attention_mask, **cross_attention_kwargs)
    return attn_output + hidden_states


def _feed_forward_stage(block, hidden_states, mlp_terms):
    """norm3 -> ff + residual (patch.py:187-199), with AdaNorm-zero's (shift_mlp, scale_mlp, gate_mlp) or None.  A block
    without `ff` (the hot-path skeleton used by bench.py) stops after the earlier stages."""
    ff = getattr(block, "ff", None)
    if ff is None:
        return hidden_states
    if FUSE_FEED_FORWARD and hidden_states.is_cuda and not block.use_ada_layer_norm_zero:
        parts = feedforward.geglu_parts(ff)
        ln3 = _fusable_layer_norm(block.norm3, hidden_states) if parts is not None else None
        if ln3 is not None:
            # norm3 -> GEGLU projection (gate fused) -> output projection (+ bias + residual), wgmma
            return feedforward.feed_forward_residual(ff, parts, ln3, hidden_states)
    norm_hidden_states = block.norm3(hidden_states)
    if mlp_terms is not None:
        shift_mlp, scale_mlp, gate_mlp = mlp_terms
        norm_hidden_states = norm_hidden_states * (1 + scale_mlp[:, None]) + shift_mlp[:, None]
    ff_output = ff(norm_hidden_states)
    if mlp_terms is not None:
        ff_output = gate_mlp.unsqueeze(1) * ff_output
    return ff_output + hidden_states


def make_tome_block(block_class: Type[torch.nn.Module]) -> Type[torch.nn.Module]:
    """CompVis-LDM variant (patch.py:94-116).  The reference's version unpacks six values from
    compute_merge's three (patch.py:105 vs :91) and cannot run; we refuse at patch time instead."""
    raise NotImplementedError(
        "vidtome_b200: the LDM (non-diffusers) ToMeBlock of the reference is not runnable upstream "
        "(patch.py:105 unpacks 6 values from a 3-tuple); only diffusers models are supported")


def make_diffusers_tome_block(block_class: Type[torch.nn.Module]) -> Type[torch.nn.Module]:
    """Patched class for a diffusers BasicTransformerBlock (patch.py:119-203)."""

    class ToMeBlock(block_class):
        # the original class, restored by remove_patch
        _parent = block_class
        # True in the served class of serve_unmerged: the block never merges, as inside _unmerged_blocks()
        _vtm_unmerged = False

        def forward(self, hidden_states, attention_mask=None, encoder_hidden_states=None,
                    encoder_attention_mask=None, timestep=None, cross_attention_kwargs=None,
                    class_labels=None) -> torch.Tensor:
            cross_attention_kwargs = cross_attention_kwargs if cross_attention_kwargs is not None else {}
            hidden_states, mlp_terms = _self_attention_stage(self, hidden_states, attention_mask, encoder_hidden_states,
                                                             timestep, class_labels, cross_attention_kwargs)
            hidden_states = _cross_attention_stage(self, hidden_states, encoder_hidden_states, encoder_attention_mask,
                                                   timestep, cross_attention_kwargs)
            return _feed_forward_stage(self, hidden_states, mlp_terms)

    return ToMeBlock


def make_library_transformer2d(wrapper_class: Type[torch.nn.Module]) -> Type[torch.nn.Module]:
    """Patched class for a diffusers Transformer2DModel: the library path of transformer2d.py while FUSE_TRANSFORMER_IO
    is on and the call is eligible, else the class's own forward.  It does not depend on merging, so it stays on the
    library path inside _unmerged_blocks() too.  The module gets no `_tome_info`: update_patch and collect_from_patch
    see what they saw before."""

    class ToMeTransformer2D(wrapper_class):
        # the original class, restored by remove_patch
        _parent = wrapper_class

        def forward(self, hidden_states, *args, **kwargs):
            from . import transformer2d as _t2d
            # keyword arguments library_forward does not restate (a later diffusers release's) go to the class's forward
            if (FUSE_TRANSFORMER_IO and not args and _t2d.LIBRARY_KWARGS.issuperset(kwargs)
                    and _t2d.ineligibility(self, hidden_states) is None):
                return _t2d.library_forward(self, hidden_states, **kwargs)
            return super().forward(hidden_states, *args, **kwargs)

    return ToMeTransformer2D


# the keyword arguments of BasicTransformerBlock.forward that ToMeBlock.forward restates
SERVED_BLOCK_KWARGS = frozenset(("attention_mask", "encoder_hidden_states", "encoder_attention_mask", "timestep",
                                 "cross_attention_kwargs", "class_labels"))
# class names of the modules serve_unmerged swaps in
_SERVED_CLASSES = ("UnmergedBlock", "UnmergedTransformer2D")


def served_block_ineligibility(block: torch.nn.Module, hidden_states, args: tuple, kwargs: dict) -> Optional[str]:
    """Why a call of a served block (serve_unmerged) runs the block class's own forward instead of the unmerged library
    path, or None if it takes that path.  It takes it with FUSE_CONTROLNET_BLOCKS on, keyword arguments only and those
    ToMeBlock.forward restates, no attention masks and no cross_attention_kwargs, the plain-LayerNorm block of the
    diffusers releases the reference targets (use_ada_layer_norm / use_ada_layer_norm_zero present and false, not
    only_cross_attention), no autograd, and a CUDA fp16 input.  Past this gate each stage keeps the rule it has inside
    _unmerged_blocks(): attn1 through KD when _plain_attention_module and norm1 is _fusable_layer_norm, attn2 when
    attention.cross_attention_eligible, the feed-forward when feedforward.geglu_parts; otherwise that stage's modules."""
    if not FUSE_CONTROLNET_BLOCKS:
        return "switch"
    if args or not SERVED_BLOCK_KWARGS.issuperset(kwargs):
        return "arguments"
    if (kwargs.get("attention_mask") is not None or kwargs.get("encoder_attention_mask") is not None
            or kwargs.get("cross_attention_kwargs")):
        return "arguments"
    if not (hasattr(block, "use_ada_layer_norm") and hasattr(block, "use_ada_layer_norm_zero")):
        return "norm"
    if block.use_ada_layer_norm or block.use_ada_layer_norm_zero or getattr(block, "only_cross_attention", False):
        return "norm"
    if block.training and torch.is_grad_enabled():
        return "training"
    if not isinstance(hidden_states, torch.Tensor) or not hidden_states.is_cuda or hidden_states.dtype != torch.float16:
        return "device"
    return None


def make_unmerged_block(block_class: Type[torch.nn.Module]) -> Type[torch.nn.Module]:
    """Served class for a BasicTransformerBlock of a model apply_patch did not patch (serve_unmerged): ToMeBlock's
    forward in its unmerged state, which builds no merge plan and reads no `_tome_info`, `generator` or
    `global_tokens`, while served_block_ineligibility passes; else the block class's own forward."""
    tome = make_diffusers_tome_block(block_class)

    class UnmergedBlock(tome):
        # the original class, restored by unserve_unmerged
        _parent = block_class
        _vtm_unmerged = True

        def forward(self, hidden_states, *args, **kwargs):
            if served_block_ineligibility(self, hidden_states, args, kwargs) is None:
                return tome.forward(self, hidden_states, **kwargs)
            return block_class.forward(self, hidden_states, *args, **kwargs)

    return UnmergedBlock


def make_unmerged_transformer2d(wrapper_class: Type[torch.nn.Module]) -> Type[torch.nn.Module]:
    """Served class for a Transformer2DModel of a model apply_patch did not patch (serve_unmerged): the patched class's
    forward (the library's entry and exit under FUSE_TRANSFORMER_IO and transformer2d.ineligibility) while
    FUSE_CONTROLNET_BLOCKS is on, else the wrapper class's own forward."""
    library = make_library_transformer2d(wrapper_class)

    class UnmergedTransformer2D(library):
        # the original class, restored by unserve_unmerged
        _parent = wrapper_class

        def forward(self, hidden_states, *args, **kwargs):
            if FUSE_CONTROLNET_BLOCKS:
                return library.forward(self, hidden_states, *args, **kwargs)
            return wrapper_class.forward(self, hidden_states, *args, **kwargs)

    return UnmergedTransformer2D


def is_patched(model: torch.nn.Module) -> bool:
    """True if apply_patch patched `model` (or a module inside it) and remove_patch has not undone it: some module has
    a patched class or the hooks of a `_tome_info`."""
    return any(type(m).__name__ in ("ToMeBlock", "ToMeTransformer2D") or getattr(m, "_tome_info", {}).get("hooks")
               for m in model.modules())


def is_served(model: torch.nn.Module) -> bool:
    """True if serve_unmerged served some module of `model`."""
    return any(type(m).__name__ in _SERVED_CLASSES for m in model.modules())


def serve_unmerged(model: torch.nn.Module) -> torch.nn.Module:
    """Serve a model that apply_patch did not patch (the reference's unpatched ControlNet, generate.py:96-98) from the
    library, always unmerged, while FUSE_CONTROLNET_BLOCKS is on: every BasicTransformerBlock gets the class of
    make_unmerged_block and every Transformer2DModel that of make_unmerged_transformer2d.  Nothing else changes: no
    `_tome_info`, no hooks (so no generator is forked and nothing is drawn), no `global_tokens`, no PnP, and the
    parameters and buffers are the model's own.  A model patched by apply_patch is refused; serving a served model
    again changes nothing.  unserve_unmerged undoes it.  Returns `model`."""
    if is_patched(model):
        raise ValueError("serve_unmerged: the model is patched by apply_patch, whose blocks already run in the library; "
                         "serve only an unpatched model")
    from . import _lib
    _lib.load()   # fail here, loudly, if the CUDA library is missing
    for module in model.modules():
        if type(module).__name__ in _SERVED_CLASSES:
            continue
        if isinstance_str(module, "BasicTransformerBlock"):
            module.__class__ = make_unmerged_block(module.__class__)
        elif isinstance_str(module, "Transformer2DModel"):
            module.__class__ = make_unmerged_transformer2d(module.__class__)
    return model


def unserve_unmerged(model: torch.nn.Module) -> torch.nn.Module:
    """Undo serve_unmerged: every served module gets its original class back.  A model patched by apply_patch is
    refused (remove_patch undoes apply_patch).  Returns `model`."""
    if is_patched(model):
        raise ValueError("unserve_unmerged: the model is patched by apply_patch; undo that with remove_patch")
    for module in model.modules():
        if type(module).__name__ in _SERVED_CLASSES:
            module.__class__ = module._parent
    return model


def hook_tome_model(model: torch.nn.Module):
    """Forward pre-hook recording the latent size (patch.py:206-212).  The UNet must be called with the
    latent as positional argument 0, as generate.py:275 does."""
    def hook(module, args):
        if _UNMERGED:                        # an unpatched model records nothing (_unmerged_blocks)
            return None
        module._tome_info["size"] = (args[0].shape[2], args[0].shape[3])
        return None

    model._tome_info["hooks"].append(model.register_forward_pre_hook(hook))


def hook_tome_module(module: torch.nn.Module):
    """Forward pre-hook that gives the block its own `module.generator`, forked from the default RNG of the
    input's device the first time the block runs (and again if the block moves to another device), so that all
    blocks draw the same random target frames within one pass (patch.py:215-231)."""
    def hook(module, args):
        if _UNMERGED:                        # an unpatched block has no generator (_unmerged_blocks)
            return None
        device = args[0].device
        current = getattr(module, "generator", None)
        if current is None:
            module.generator = init_generator(device)
        elif current.device != device:
            module.generator = init_generator(device, fallback=current)
        return None

    module._tome_info["hooks"].append(module.register_forward_pre_hook(hook))


def apply_patch(
        model: torch.nn.Module,
        local_merge_ratio: float = 0.9,
        merge_global: bool = False,
        global_merge_ratio=0.8,
        max_downsample: int = 2,
        seed: int = 123,
        batch_size: int = 2,
        include_control: bool = False,
        align_batch: bool = False,
        target_stride: int = 4,
        global_rand=0.5):
    """Patch a Stable-Diffusion model with VidToMe (signature, defaults and semantics of
    vidtome/patch.py:234-334).

     - model: a diffusers pipeline (uses `.unet`, and `.controlnet` when it is a
       StableDiffusionControlNetPipeline and include_control) or a bare diffusers UNet; detected by class
       NAME (DiffusionPipeline / ModelMixin), blocks by the name BasicTransformerBlock.
     - local_merge_ratio: fraction of src tokens merged inside a frame chunk (0.9 -> 1.3/4.0 kept for 4 frames).
     - merge_global / global_merge_ratio / global_rand: inter-chunk (global) token merging.
     - max_downsample: merge only in layers with at most this downsampling (1, 2, 4 or 8).
     - seed: stored, unused (as in the reference).   - batch_size: number of video chunks per pass (2 = CFG, 3 = PnP).
     - align_batch: share one matching across the batch (PnP).   - target_stride: one target frame per this many frames.
    """
    # start from an unpatched model: a second apply_patch must not stack hooks or subclasses
    remove_patch(model)

    is_diffusers = isinstance_str(model, "DiffusionPipeline") or isinstance_str(model, "ModelMixin")

    if not is_diffusers:
        if not hasattr(model, "model") or not hasattr(model.model, "diffusion_model"):
            raise RuntimeError("Provided model was not a Stable Diffusion / Latent Diffusion model, as expected.")
        diffusion_model = model.model.diffusion_model
    else:
        # a pipeline carries its UNet as `.unet`; a bare UNet is used as is
        diffusion_model = model.unet if hasattr(model, "unet") else model

    if isinstance_str(model, "StableDiffusionControlNetPipeline") and include_control:
        diffusion_models = [diffusion_model, model.controlnet]
    else:
        diffusion_models = [diffusion_model]

    from . import _lib
    _lib.load()   # fail at patch time, loudly, if the CUDA library is missing

    for diffusion_model in diffusion_models:
        diffusion_model._tome_info = {
            "size": None,
            "hooks": [],
            "args": {
                "max_downsample": max_downsample,
                "generator": None,
                "seed": seed,
                "batch_size": batch_size,
                "align_batch": align_batch,
                "merge_global": merge_global,
                "global_merge_ratio": global_merge_ratio,
                "local_merge_ratio": local_merge_ratio,
                "global_rand": global_rand,
                "target_stride": target_stride
            }
        }
        hook_tome_model(diffusion_model)

        for name, module in diffusion_model.named_modules():
            if isinstance_str(module, "BasicTransformerBlock"):
                make_tome_block_fn = make_diffusers_tome_block if is_diffusers else make_tome_block
                module.__class__ = make_tome_block_fn(module.__class__)
                module._tome_info = diffusion_model._tome_info
                hook_tome_module(module)

                # blocks of diffusers releases that predate the ada-norm flags: read as "plain LayerNorm"
                if not hasattr(module, "use_ada_layer_norm_zero") and is_diffusers:
                    module.use_ada_layer_norm = False
                    module.use_ada_layer_norm_zero = False
            elif is_diffusers and isinstance_str(module, "Transformer2DModel"):
                module.__class__ = make_library_transformer2d(module.__class__)

    return model


def _roots_of(model: torch.nn.Module, controlnet_owner: torch.nn.Module) -> List[torch.nn.Module]:
    """[UNet (or the model itself)] + [controlnet_owner.controlnet] when that attribute exists.

    The three lifecycle calls of the reference differ in WHERE they look for `.controlnet`:
      * remove_patch rebinds `model` to the UNet first (patch.py:341-344), so it looks on the UNet — a ControlNet
        patched through `include_control=True` is therefore not reached by remove_patch;
      * update_patch / collect_from_patch keep the object they were given (patch.py:361-364, :376-378), so on a
        pipeline they DO reach `pipe.controlnet`.
    Both behaviours are reproduced; the caller passes the object the reference would test."""
    root = model.unet if hasattr(model, "unet") else model
    roots = [root]
    if hasattr(controlnet_owner, "controlnet"):
        roots.append(controlnet_owner.controlnet)
    return roots


def remove_patch(model: torch.nn.Module):
    """Undo apply_patch if the model is patched: drop the hooks and restore the block classes
    (patch.py:337-355).  Returns what the reference returns: the last module it walked."""
    unet = model.unet if hasattr(model, "unet") else model
    roots = _roots_of(model, unet)                       # `.controlnet` is looked up on the UNet here
    for root in roots:
        for _, module in root.named_modules():
            info = getattr(module, "_tome_info", None)
            if info is not None:
                for handle in info["hooks"]:
                    handle.remove()
                info["hooks"].clear()
            if module.__class__.__name__ in ("ToMeBlock", "ToMeTransformer2D"):
                module.__class__ = module._parent
    return roots[-1]


def update_patch(model: torch.nn.Module, **kwargs):
    """Set attributes on every module that carries `_tome_info` (the UNet, each patched block and — on a
    pipeline that has one — the ControlNet and its blocks), e.g. `update_patch(pipe, global_tokens=None)`
    after each denoising step (patch.py:358-370, generate.py:233-236).  Like the reference, the return
    value is the last root walked (its loop variable shadows `model`), not the object passed in."""
    roots = _roots_of(model, model)                      # `.controlnet` is looked up on the object passed in
    for root in roots:
        for _, module in root.named_modules():
            if hasattr(module, "_tome_info"):
                for key, value in kwargs.items():
                    setattr(module, key, value)
    return roots[-1]


def collect_from_patch(model: torch.nn.Module, attr="tome"):
    """{qualified module name: getattr(module, attr)} for every module that has `attr` (patch.py:373-387);
    a pipeline's ControlNet is included, later roots overwrite equal names exactly as the reference's dict does."""
    found = dict()
    for root in _roots_of(model, model):
        for name, module in root.named_modules():
            if hasattr(module, attr):
                found[name] = getattr(module, attr)
    return found
