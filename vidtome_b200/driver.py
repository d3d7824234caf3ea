"""Minimal denoising driver around a patched UNet — the loop the metric "denoising steps/sec" counts.

Restates, on synthetic latents, the parts of the reference's Generator that sit around the hot path:
  get_chunks      generate.py:172-203   (frame chunking; order seq / rand / mix for global merging)
  ddim_sample     generate.py:205-224   (per step: every chunk's pred_noise, then the DDIM update)
  pred_noise      generate.py:238-279   (CFG batch cat([x, x]), UNet forward, guidance combine)
  pred_next_x     generate.py:281-311   (closed-form DDIM step)
  post_iter       generate.py:233-236   (reset global tokens after each step)
  init_pnp        generate.py:313-319   (PnP self-attention and conv-feature injection schedules; with `source_latents`)
  pre_iter        generate.py:226-231   (PnP: set the timestep, fetch the source latents of the step)
  ControlNet      generate.py:56-63,264-275, utils/utils.py:280-295 (residuals of `controlnet`, with `control_images`)
  SD2-depth       generate.py:131-132,255-262 (each frame's depth map appended to the UNet input, with `depth`)
and, in ChunkedInverter, the reference's Inverter around its hot path:
  ddim_inversion  invert.py:117-140     (reversed timesteps, frame batches, the kept latents)
  ddim_sample     invert.py:142-157     (`recon`: the inverted latents sampled back, reconstruct())
  pred_noise      invert.py:159-179     (UNet forward, optional depth channel, optional ControlNet residuals)
  pred_next_x     invert.py:182-211     (inversion=True and, for reconstruct(), inversion=False)
Text conditioning, VAE, ControlNet and depth preprocessing and file IO are outside the hot path and not restated.
"""
from __future__ import annotations

import contextlib
from typing import Callable, Iterable, List, NamedTuple, Optional

import numpy as np
import torch

from . import patch, pnp

# On CUDA fp16 latents (shard=False), every chunk of a ChunkedDenoiser step ends with KS (ops.cfg_ddim_update): the
# guidance combine and the DDIM update of the chunk's rows in one kernel, its coefficients read from a device table at a
# device step index, so that a captured step includes the update.  Bit-identical to pred_noise's combine followed by
# pred_next_x.  Off: the step takes those torch ops.  Read at every eager step and at capture; a graph replays the path
# it was captured with.
FUSE_STEP_UPDATE = True

# A step captured into one CUDA graph (cuda_graph=True with local merging, or capture_global=True) issues chunk k on
# side stream ("lane") k % LANES, forked from the capture stream and joined back into it, so the graph runs the chunks
# concurrently.  With local merging nothing links two chunks; with global merging the one edge is the global-token
# recurrence, per merged block (patch.LaneEdges).  Each captured draw has a fixed Philox offset, so the latents are those
# of one stream, bit for bit.  A step of one chunk, or shard=True, captures on the capture stream alone.  DESIGN §5 and
# §7 give the reasons for the count.
LANES = 3


def run_on_lanes(n: int, lanes: list, body: Callable[[int], None], edges=None) -> None:
    """body(k) for k in range(n), inside a capture: on the current stream when fewer than two lanes are given, else
    chunk k on lanes[k % len(lanes)], every lane forked from the current stream first and joined into it at the end,
    with `edges` (patch.LaneEdges, or None) installed for the global stages."""
    if len(lanes) < 2:
        for k in range(n):
            body(k)
        return
    main = torch.cuda.current_stream()
    for lane in lanes:
        lane.wait_stream(main)
    try:
        with patch.lane_edges(edges):
            for k in range(n):
                with torch.cuda.stream(lanes[k % len(lanes)]):
                    body(k)
    finally:
        for lane in lanes:
            main.wait_stream(lane)


def ddim_alphas_cumprod(num_train_timesteps: int = 1000, beta_start: float = 0.00085,
                        beta_end: float = 0.012) -> torch.Tensor:
    """Stable Diffusion's "scaled_linear" schedule (what DDIMScheduler.from_pretrained gives for SD1.5/2.1)."""
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float64) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


def ddim_timesteps(n_timesteps: int, num_train_timesteps: int = 1000) -> List[int]:
    """DDIMScheduler.set_timesteps with 'leading' spacing and steps_offset=1 (SD's scheduler config)."""
    ratio = num_train_timesteps // n_timesteps
    return [int(t) + 1 for t in (np.arange(0, n_timesteps) * ratio).round()[::-1]]


def ddim_coefficients(alpha_from: torch.Tensor, alpha_to: torch.Tensor):
    """(a, b, c, d) = (sigma_from, mu_from, mu_to, sigma_to) of the DDIM step from cumulative alpha `alpha_from` to
    `alpha_to` (mu = alpha ** 0.5, sigma = (1 - alpha) ** 0.5), the floats ddim_step and ops.ddim_table take."""
    return (float((1 - alpha_from) ** 0.5), float(alpha_from ** 0.5), float(alpha_to ** 0.5),
            float((1 - alpha_to) ** 0.5))


def ddim_step(x: torch.Tensor, eps: torch.Tensor, coefficients) -> torch.Tensor:
    """x <- c * ((x - a * eps) / b) + d * eps: the predicted x0 moved to the other timestep (generate.py:281-311,
    invert.py:182-211)."""
    a, b, c, d = coefficients
    return c * ((x - a * eps) / b) + d * eps


def _rows(frames: dict, lo: int, hi: int) -> dict:
    """Frames lo..hi-1 of every per-frame input ({"src" | "ctrl" | "depth": [flen, ...]}) of a step."""
    return {k: v[lo:hi] for k, v in frames.items()}


def _spans(chunks: List[torch.Tensor]) -> List[tuple]:
    """(lo, hi) of every chunk: chunks are contiguous frame ranges (possibly visited in another order), so a step slices
    instead of indexing with a host tensor, which would cost a synchronous host->device copy per chunk per step."""
    return [(int(c[0]), int(c[-1]) + 1) for c in chunks]


class _Graph(NamedTuple):
    """A captured step or chunk: `graph` reads the static inputs `x`, `t` and `frames` ({"src" | "ctrl" | "depth"})
    and writes `out`, x_{t-1} when `fused` (KS ends every chunk), else the noise prediction.  The first five fields
    keep the positions the driver's graph tuples always had (graph, x, t, out, key), for code that indexes them."""
    graph: torch.cuda.CUDAGraph
    x: torch.Tensor
    t: torch.Tensor
    out: torch.Tensor
    key: tuple                      # _graph_key for a step graph, the chunk key for a chunk graph
    frames: dict
    fused: bool
    phase: tuple                    # the PnP injections it was captured with (_phase)
    slots: Optional[tuple] = None   # capture_global: (slot index on the device, its pinned host copy, upload event)


class _ControlNetServing:
    """The lazy serving of an unpatched ControlNet shared by both drivers: at the first step that runs with
    patch.FUSE_CONTROLNET_BLOCKS on, a ControlNet that apply_patch did not patch (the reference's default,
    include_control=False) and that is not served yet is served (patch.serve_unmerged); close() unserves it again.  A
    patched ControlNet, or one the caller served, is left as it is and close() leaves it alone."""

    def __init__(self, controlnet: Optional[torch.nn.Module]):
        self.controlnet = controlnet
        self.decided = controlnet is None
        self.served = False

    def before_step(self):
        if self.decided or not patch.FUSE_CONTROLNET_BLOCKS:
            return
        self.decided = True
        if not patch.is_patched(self.controlnet) and not patch.is_served(self.controlnet):
            patch.serve_unmerged(self.controlnet)
            self.served = True

    def close(self):
        if self.served:
            patch.unserve_unmerged(self.controlnet)
        self.served = False
        self.decided = self.controlnet is None


class _Driver:
    """What both drivers share: the UNet, the optional ControlNet with its control images or the optional depth maps,
    and the DDIM schedule."""

    def __init__(self, unet: torch.nn.Module, controlnet: Optional[torch.nn.Module],
                 control_images: Optional[torch.Tensor], control_scale: float, depth: Optional[torch.Tensor],
                 source_latents: Optional[Callable[[int], torch.Tensor]] = None):
        if depth is not None and (depth.dim() != 4 or depth.shape[1] != 1):
            raise ValueError(f"depth must be [flen, 1, h, w] (got {tuple(depth.shape)})")
        if depth is not None and controlnet is not None:
            raise ValueError("depth and controlnet are exclusive: the reference's ControlNets are SD1.5 models with a "
                             "4-channel input, and its configs use no control with the depth model")
        if controlnet is not None and source_latents is not None:
            raise ValueError("controlnet and source_latents (PnP) are exclusive: the reference runs one control mode "
                             "(generate.py:61-68)")
        if (controlnet is None) != (control_images is None):
            raise ValueError("controlnet and control_images go together")
        if control_images is not None and (control_images.dim() != 4 or control_images.shape[1] != 3):
            raise ValueError(f"control_images must be [flen, 3, H, W] (got {tuple(control_images.shape)})")
        self.unet = unet
        self.controlnet = controlnet
        self.control_images = control_images
        self.control_scale = control_scale
        self.depth = depth
        self._serving = _ControlNetServing(controlnet)
        self.alphas_cumprod = ddim_alphas_cumprod()
        self.final_alpha_cumprod = self.alphas_cumprod[0]     # set_alpha_to_one=False in SD's config

    def _models(self) -> List[torch.nn.Module]:
        """The UNet and, with ControlNet control, the ControlNet: the models whose blocks the driver serves."""
        return [self.unet] + ([self.controlnet] if self.controlnet is not None else [])

    def _alpha(self, timesteps: List[int], k: int) -> torch.Tensor:
        """The cumulative alpha at timesteps[k]; final_alpha_cumprod before the first and after the last one."""
        return self.alphas_cumprod[timesteps[k]] if 0 <= k < len(timesteps) else self.final_alpha_cumprod

    def _frames(self, x: torch.Tensor, frames: dict) -> dict:
        """`frames` with the control images ("ctrl") or the depth maps ("depth") of the latents x added, checked against
        x and cast to its dtype (prepare_data's .to(self.init_noise)).  An unpatched ControlNet is served here."""
        if self.controlnet is not None:
            if len(self.control_images) != len(x):
                raise ValueError(f"control_images has {len(self.control_images)} frames, the latents {len(x)}")
            frames["ctrl"] = self.control_images.to(x)
            self._serving.before_step()
        if self.depth is not None:
            # one depth map per frame at the latents' resolution, for a model that takes the latent channels + 1
            if len(self.depth) != len(x) or self.depth.shape[2:] != x.shape[2:]:
                raise ValueError(f"depth is {tuple(self.depth.shape)}, the latents {tuple(x.shape)}: it needs one map "
                                 f"per frame at the latents' resolution")
            n = getattr(getattr(self.unet, "config", None), "in_channels", getattr(self.unet, "in_channels", None))
            if isinstance(n, int) and n != x.shape[1] + 1:
                raise ValueError(f"depth: the model takes {n} input channels, not the latents' {x.shape[1]} and one "
                                 f"depth channel")
            frames["depth"] = self.depth.to(x)
        return frames


class ChunkedDenoiser(_Driver):
    """Chunked classifier-free-guidance DDIM sampling on a (patched) UNet, generate.py:205-311."""

    def __init__(self, unet: torch.nn.Module, n_timesteps: int = 50, chunk_size: int = 16,
                 guidance_scale: float = 7.5, merge_global: bool = False, chunk_ord: str = "seq",
                 perm_div: float = 3.0, randomize_chunks: bool = False, cond: Optional[torch.Tensor] = None,
                 cuda_graph: bool = False, graph_warmup: int = 2, shard: bool = False, capture_global: bool = False,
                 chunk_graphs: bool = False, source_latents: Optional[Callable[[int], torch.Tensor]] = None,
                 pnp_attn_t: float = 0.5, pnp_modules: Optional[Iterable[torch.nn.Module]] = None,
                 controlnet: Optional[torch.nn.Module] = None, control_images: Optional[torch.Tensor] = None,
                 control_scale: float = 1.0, pnp_f_t: Optional[float] = None,
                 pnp_conv_modules: Optional[Iterable[torch.nn.Module]] = None, depth: Optional[torch.Tensor] = None):
        """`cuda_graph=True`: after `graph_warmup` eager steps, the noise prediction of a whole step (every chunk:
        CFG batch, UNet forward with the merge path, guidance combine) is captured once into a CUDA graph and
        replayed; per step the host then issues one graph launch instead of ~250 kernel launches.  On CUDA fp16
        latents the DDIM update is inside the graph too (FUSE_STEP_UPDATE: KS ends every chunk); otherwise it follows
        the replay in torch ops.  The frame draws of the local matcher stay on the device (utils.draw_randf) and come
        from the blocks' generators, which are registered with the graph, so replays produce the same sequence of
        draws — and bit-identical latents — as eager stepping.  Needs static shapes: `randomize_chunks=False`, frame counts
        divisible by the target stride, and local merging only (`merge_global=False`) unless `capture_global=True`.

        `capture_global=True` (with `merge_global=True, cuda_graph=True`) captures global merging too.  The graph runs
        chunk *slots*: slot k takes a static [chunk_size, ...] input, and the global-token recurrence runs slot 0 -> K-1
        inside the graph, with the coin of every block drawn on the device (patch.DEVICE_COIN).  Each step still draws
        the chunk order on the host with get_chunks, exactly as eager stepping does, and applies it as data: one
        index_select of the latents into the slots, one of the noise back.  Needs every chunk to be equally long
        (frame count divisible by chunk_size), patch.GLOBAL_EXCHANGE == "recurrence", and no sharding.

        `chunk_graphs=True` (with `cuda_graph=True`) captures one graph per chunk instead of one per step, keyed by
        (chunk length, first chunk of the step?), lazily on first use: at most 2 * chunk_size graphs.  Each step calls
        get_chunks once on the host, as eager stepping does, and replays the graph of every chunk in visiting order on
        its contiguous frame range.  So the reference's own chunking runs from graphs: `randomize_chunks=True`, any frame
        count, `merge_global` true or false.  With `merge_global=True` every block keeps its global tokens in a
        patch.GlobalTokenStore (installed before the warm-up steps, emptied where eager stepping calls
        `update_patch(global_tokens=None)`), whose global stage keeps the counts that depend on the coin on the device.
        Needs chunk lengths whose local counts do not depend on the frame draw (every length up to chunk_size when
        chunk_size <= target_stride; see draw_dependent_lengths), patch.GLOBAL_EXCHANGE == "recurrence", the library's
        self-attention (KD) in every merged block, and no sharding.

        `source_latents` (a callable t -> [flen, 4, h, w], the inverted source latents at timestep t; the reference's
        load_latent) switches on PnP control, the reference's default generation (generate.py:60-68, `control: "pnp"`):
        every UNet call gets the batch [source | x | x] with `cond` = [3, 77, D] (the pnp guidance "", uncond, cond text
        embeddings, generate.py:101-109), and the first int(n_timesteps * pnp_attn_t) steps take the attention map of
        the decoder self-attention modules from the source sample (pnp.register_attention_control; `pnp_modules` names
        those modules for a model without the diffusers up_blocks hierarchy).  The model must be patched with
        batch_size=3 and align_batch=True.  In every graph mode the injection is decided on the host when a graph is
        captured, so graphs are keyed by it as well; the injected ones are released once the schedule has passed.

        `pnp_f_t` (with `source_latents`) adds PnP's conv-feature injection, the other half of the reference's default
        PnP config (generate.py:64,315-319, `pnp_f_t: 0.8`): for the first int(n_timesteps * pnp_f_t) steps the ResNet
        `unet.up_blocks[1].resnets[1]` (or `pnp_conv_modules` for a model without that hierarchy) adds the source
        sample's conv2 output to the uncond and cond samples in place of their own (pnp.register_conv_control; on CUDA
        fp16 its branch runs on the source samples only and the tail is one kernel).  The graph modes key their graphs
        by both injections then: three phases (both, conv only, neither) when pnp_f_t >= pnp_attn_t.  With
        `pnp_f_t=None` (the default) nothing of this is installed and the graph keys are those of attention-only PnP.

        `controlnet` with `control_images` ([flen, 3, H, W], the reference's prepare_control output) switches on
        ControlNet control (generate.py:56-63, `control: "depth"`, `"softedge"`, ...): every UNet call first runs the
        ControlNet on the same batch and text with the chunk's control images repeated over the CFG batch, scales its
        residuals by `control_scale` and passes them to the UNet (utils/utils.py:280-295).  The ControlNet may be
        patched too (apply_patch(include_control=True) on a StableDiffusionControlNetPipeline); its blocks then draw
        from their own generators and keep their own global tokens, which every graph mode registers and resets like
        the UNet's.  The control images are a static input of every graph.  One control mode at a time: ControlNet
        and PnP (`source_latents`) are refused together, as the reference takes one (generate.py:61-68).
        An unpatched ControlNet (the reference's default) runs its modules' own forwards; with
        patch.FUSE_CONTROLNET_BLOCKS on, the first step serves it (patch.serve_unmerged), so that its blocks and
        Transformer2DModel wrappers run in the library, never merged.  Its shapes are static, so graph keys do not
        change; a graph replays the path it was captured with.  close() gives the ControlNet its own classes back.

        `depth` ([flen, 1, h, w], the reference's prepare_depth output: one depth map per frame at latent resolution,
        normalised to [-1, 1]) runs SD2-depth (stabilityai/stable-diffusion-2-depth, `sd_version: "depth"`), whose UNet
        takes 5 input channels: every UNet call gets the chunk's depth maps, cast to the latents' dtype (generate.py:
        131-132), repeated over the batch ([x | x], or [source | x | x] with PnP) and appended as a fifth channel
        (generate.py:255-262).  Depth combines with PnP (the reference's default `control: "pnp"`) and with every graph
        mode, in each of which the depth maps are a static input like the control images; graph keys do not change.
        Depth with `controlnet` is refused: the reference's ControlNets are SD1.5 models with a 4-channel input.

        `cond` of shape [K, S, 77, D] (S = 2, or 3 with PnP) runs K edits of one video in one pass: step() takes and
        returns latents [K, flen, 4, h, w] and every UNet call carries the chunk of all K edits, edit-major: edit k's
        slice is exactly the batch a single-prompt run builds with cond[k] ([source |] uncond | cond, each chunk-long),
        and the per-frame inputs (source latents, control images, depth) are shared by all edits.  Edit k is the
        single-prompt run of cond[k] from the same RNG state: every draw (get_chunks, the blocks' randints and coins)
        is issued once per step, as by one run.  The model must be patched for K edits (apply_patch, then
        update_patch(model, edits=K)).  Every graph mode runs it; graph keys and static buffers include K.

        `shard=True` with K > 1 edits splits the edits over the ranks of an initialised torch.distributed job: rank r
        runs the K_r edits k with k % world == r (dist.shard_edits) as a plain K_r-edit pass, with no chunk sharding, so
        KS, lanes and every graph mode apply.  `cond` is the whole [K, S, 77, D] on every rank; the model is patched with
        update_patch(model, edits=K_r).  step() takes and returns the rank's [K_r, flen, 4, h, w]; sample() takes
        [K, flen, ...] (and keeps its rows), [K_r, flen, ...] or one [flen, ...] for all edits, and returns the gathered
        [K, flen, 4, h, w] on every rank (dist.gather_edits).  Every rank makes the draws of the whole job, so each edit
        is what the unsharded K-edit run computes for it: nothing crosses ranks during the steps.  sample() first checks
        that the ranks agree on K, the latents' shape, the steps, the mode and the RNG states (dist.check_ranks_agree).
        Needs world <= K and patch.GLOBAL_EXCHANGE == "recurrence"."""
        super().__init__(unet, controlnet, control_images, control_scale, depth, source_latents)
        # K for a [K, S, 77, D] cond (K edits, latents [K, flen, ...]), None for the single-prompt [S, 77, D]
        self.edits = None
        if cond is not None and cond.dim() == 4:
            if cond.shape[0] < 1 or cond.shape[1] not in (2, 3):
                raise ValueError(f"cond of several edits must be [K, S, 77, D] with S = 2 or 3 (got "
                                 f"{tuple(cond.shape)})")
            self.edits = int(cond.shape[0])
        K = self.job_edits = self.edits or 1
        # shard=True with K > 1 edits: this rank runs the edits dist.shard_edits(K) (their rows of cond) as a plain
        # K_r-edit pass, with no chunk sharding; sample() gathers all K.  None otherwise.
        self.edit_rows: Optional[List[int]] = None
        if shard and K > 1:
            from . import dist as _dist
            if not _dist.initialized():
                raise ValueError("shard=True needs an initialised torch.distributed process group (one rank per process)")
            if _dist.world() > K:
                raise ValueError(f"shard=True with {K} edits needs at most {K} ranks (world size {_dist.world()}): "
                                 f"the edits are split over the ranks")
            self._check_edit_exchange()
            self.edit_rows = _dist.shard_edits(K)
            cond = cond[self.edit_rows]
            self.edits = len(self.edit_rows)
            shard = False
        for model in self._models():
            if hasattr(model, "_tome_info") and patch.edits_of(model) != (self.edits or 1):
                runs = (f"this rank runs {self.edits} of the {K} edits" if self.edit_rows is not None
                        else f"the cond has {K} edit(s)")
                raise ValueError(f"the model is patched with edits={patch.edits_of(model)}, {runs}: set it with "
                                 f"update_patch(model, edits={self.edits or 1})")
        # shard=True (one edit): this process is one rank of a torch.distributed job and takes chunks i % world == rank
        # of every step (dist.shard_chunks); with merge_global and a collective exchange mode the ranks are checked for
        # lock-step once per step (dist.check_step_lockstep)
        self.shard = bool(shard)
        self.cuda_graph = bool(cuda_graph)
        self.graph_warmup = int(graph_warmup)
        self._graph: Optional[_Graph] = None     # the step graph of cuda_graph=True or capture_global=True
        self._eager_steps = 0
        self.capture_global = bool(capture_global)
        self.chunk_graphs = bool(chunk_graphs)
        if self.capture_global and not (self.cuda_graph and merge_global):
            raise ValueError("capture_global=True needs cuda_graph=True and merge_global=True")
        if self.chunk_graphs and (not self.cuda_graph or self.capture_global):
            raise ValueError("chunk_graphs=True needs cuda_graph=True and capture_global=False")
        if self.chunk_graphs and merge_global and self.graph_warmup < 1:
            raise ValueError("chunk_graphs=True with merge_global=True needs graph_warmup >= 1: the blocks' global token "
                             "stores are allocated by an eager step, outside the graphs' memory pools")
        if self.chunk_graphs and self.shard:
            raise ValueError("chunk_graphs=True does not capture the cross-rank chunk sharding of shard=True")
        if self.cuda_graph and not self.chunk_graphs and ((merge_global and not self.capture_global) or randomize_chunks):
            raise ValueError("cuda_graph=True needs merge_global=False and randomize_chunks=False (static work)")
        if self.capture_global and self.shard:
            raise ValueError("capture_global=True does not capture the cross-rank exchange of shard=True")
        # (chunk length, first in step, frame shape) + _phase + (fused update,) -> _Graph
        self._chunk_graphs = {}
        self._chunk_t = None        # the UNet's timestep input shared by the chunk graphs
        self._stores = []           # patch.GlobalTokenStore of every block (chunk_graphs with merge_global)
        self._tables = {}           # device -> (KS's coefficient table, its step index), made on first use
        self._lane_count = LANES    # streams of a captured step (LANES; fewer when the KB1 sorts would not fit)
        self._lanes = {}            # device -> its lane streams, made before the first capture
        # with K edits, whether a lane capture runs edits 1..K-1 of each merged block on side streams of the lane
        # (patch.LaneEdges.edit_streams; off again when their KB1 sorts would not fit beside each other)
        self._branch_edits = True
        self._branches = {}         # device -> {lane stream handle: its K - 1 side streams}, made before any capture
        self.chunk_size = chunk_size
        self.guidance_scale = guidance_scale
        self.merge_global = merge_global
        # generate.py:86-89: "mix-#" means a partial permutation of len/# chunks ("mix" alone: # = 3)
        if "mix" in chunk_ord:
            perm_div = float(chunk_ord.split("-")[-1]) if "-" in chunk_ord else (perm_div if perm_div else 3.0)
            chunk_ord = "mix"
        self.chunk_ord, self.perm_div = chunk_ord, perm_div
        self.randomize_chunks = randomize_chunks
        self.cond = cond                      # [2, 77, D] (uncond, cond) text embeddings, may be None
        self.timesteps = ddim_timesteps(n_timesteps)
        self.source_latents = source_latents
        self.pnp_schedule: List[int] = []
        self._pnp_targets: List[torch.nn.Module] = []
        if pnp_f_t is not None and source_latents is None:
            raise ValueError("pnp_f_t (PnP conv injection) needs source_latents")
        self.pnp_f_t = None if pnp_f_t is None else float(pnp_f_t)
        self.pnp_conv_schedule: List[int] = []
        if source_latents is not None:
            self._init_pnp(n_timesteps, pnp_attn_t, pnp_modules)
            if self.pnp_f_t is not None:
                self._init_pnp_conv(n_timesteps, self.pnp_f_t, pnp_conv_modules)

    # generate.py:64,315,318-319 (the conv half of init_pnp)
    def _init_pnp_conv(self, n_timesteps: int, pnp_f_t: float, modules):
        f_t = int(n_timesteps * pnp_f_t)
        self.pnp_conv_schedule = self.timesteps[:f_t] if f_t >= 0 else []
        if modules is None and not hasattr(getattr(self.unet, "unet", self.unet), "up_blocks"):
            raise ValueError("pnp_f_t: the model has no up_blocks[1].resnets[1]; name the ResNet with pnp_conv_modules")
        pnp.register_conv_control(self.unet, self.pnp_conv_schedule, num_inputs=3, modules=modules)
        self._pnp_targets = self._pnp_targets + pnp._conv_targets(self.unet, modules)

    # generate.py:60-68,313-319 (the attention half of init_pnp)
    def _init_pnp(self, n_timesteps: int, pnp_attn_t: float, modules):
        args = self.unet._tome_info["args"] if hasattr(self.unet, "_tome_info") else None
        if args is None or args["batch_size"] != 3 or not args["align_batch"]:
            raise ValueError("PnP (source_latents) needs a model patched with batch_size=3 and align_batch=True "
                             "(generate.py:96-98): the source, uncond and cond samples of every UNet call")
        if self.cond is None or self.cond.dim() not in (3, 4) or self.cond.shape[-3] != 3 or self.cond.shape[-2] != 77:
            raise ValueError("PnP (source_latents) needs cond = [3, 77, D] (or [K, 3, 77, D] for K edits): the pnp "
                             "guidance, uncond and cond text embeddings (generate.py:101-109)")
        qk_t = int(n_timesteps * pnp_attn_t)
        self.pnp_schedule = self.timesteps[:qk_t] if qk_t >= 0 else []
        pnp.register_attention_control(self.unet, self.pnp_schedule, num_inputs=3, modules=modules)
        self._pnp_targets = pnp._targets(self.unet, modules)
        if self.job_edits > 1:                  # on every rank of a sharded job, whatever its share of the edits
            for m in self.unet.modules():
                f = vars(m).get("forward")
                if (f is not None and hasattr(m, "injection_schedule") and not getattr(f, "_vtm_pnp_forward", False)
                        and not getattr(f, "_vtm_pnp_conv_forward", False)):
                    raise ValueError(f"{type(m).__name__} carries the reference's PnP forward, which takes the source "
                                     f"sample by position over the whole batch; it cannot serve several edits")

    def injecting(self, t: int) -> bool:
        """True if the self-attention of step t takes its map from the source sample (pnp.injection_active)."""
        return self.source_latents is not None and (int(t) in self.pnp_schedule or int(t) == 1000)

    def conv_injecting(self, t: int) -> bool:
        """True if the controlled ResNet of step t takes the source sample's features (pnp_f_t set; the test of
        utils/pnp_utils.py:146)."""
        return (self.source_latents is not None and self.pnp_f_t is not None
                and (int(t) in self.pnp_conv_schedule or int(t) == 1000))

    # generate.py:172-203
    def get_chunks(self, flen: int) -> List[torch.Tensor]:
        x_index = torch.arange(flen)
        # The first chunk has a random length in the reference; benchmarks pin it to chunk_size
        rand_first = (np.random.randint(0, self.chunk_size) + 1) if self.randomize_chunks else self.chunk_size
        rest = x_index[rand_first:].split(self.chunk_size, dim=0)
        chunks = [x_index[:rand_first]] + (list(rest) if len(rest) and len(rest[0]) > 0 else [])
        if self.randomize_chunks and np.random.rand() > 0.5:
            chunks = chunks[::-1]
        if not self.merge_global:
            return chunks
        if self.chunk_ord == "rand":
            order = torch.randperm(len(chunks)).tolist()
        elif self.chunk_ord == "mix":
            randord = torch.randperm(len(chunks)).tolist()
            rand_len = int(len(randord) / self.perm_div)
            seqord = sorted(randord[rand_len:])
            if rand_len > 0:
                randord = randord[:rand_len]
                if abs(seqord[-1] - randord[-1]) < abs(seqord[0] - randord[-1]):
                    seqord = seqord[::-1]
                order = randord + seqord
            else:
                order = seqord
        else:
            order = list(range(len(chunks)))
        return [chunks[i] for i in order]

    # generate.py:238-279
    @torch.no_grad()
    def pred_noise(self, x: torch.Tensor, t: int, src: Optional[torch.Tensor] = None,
                   ctrl: Optional[torch.Tensor] = None, depth: Optional[torch.Tensor] = None) -> torch.Tensor:
        """`src`: the source latents of the chunk (PnP), prepended to the batch.  `ctrl`: the control images of the
        chunk (ControlNet).  `depth`: the depth maps of the chunk (SD2-depth), appended to every sample as a channel."""
        return self.guide(*self.unet_output(x, t, src, ctrl, depth))

    # generate.py:274-279
    def guide(self, eps: torch.Tensor, batch_size: int) -> torch.Tensor:
        """Classifier-free guidance on the raw UNet output of `batch_size` samples (of each edit: [K, ...] with K
        edits)."""
        if self.edits is None:
            return self._guide_edit(eps, batch_size)
        return torch.stack([self._guide_edit(e, batch_size) for e in eps.chunk(self.edits)])

    def _guide_edit(self, eps: torch.Tensor, batch_size: int) -> torch.Tensor:
        noise_pred_uncond, noise_pred_cond = eps.chunk(batch_size)[-2:]
        return noise_pred_uncond + self.guidance_scale * (noise_pred_cond - noise_pred_uncond)

    # generate.py:238-273
    def unet_output(self, x: torch.Tensor, t: int, src: Optional[torch.Tensor] = None,
                    ctrl: Optional[torch.Tensor] = None, depth: Optional[torch.Tensor] = None):
        """The raw UNet output of the chunk's batch ([source |] uncond | cond, each len(x) frames) and its number of
        samples, before the guidance combine of pred_noise.  With K edits (x [K, c, ...]) the batch is edit-major: K
        such batches of one edit each, in edit order."""
        if self.edits is not None:
            return self._edits_output(x, t, src, ctrl, depth)
        flen = len(x)
        text = None if self.cond is None else self.cond.repeat_interleave(flen, dim=0)
        latent_model_input = torch.cat([x, x])                                # classifier-free guidance
        batch_size = 2
        if src is not None:
            latent_model_input = torch.cat([src.to(x), latent_model_input])
            batch_size += 1
        return self._call_models(latent_model_input, t, text, batch_size, ctrl, depth), batch_size

    def _edits_output(self, x: torch.Tensor, t, src, ctrl, depth):
        """unet_output of K edits x [K, c, ...]: edit k's slice of the batch is [source |] x[k] | x[k] with cond[k]'s
        rows repeated over its c frames, as a single-prompt run builds it."""
        text = None if self.cond is None else self.cond.repeat_interleave(x.shape[1], dim=1).flatten(0, 1)
        lead = [] if src is None else [src.to(x)]
        latent_model_input = torch.cat([r for xk in x for r in lead + [xk, xk]])
        batch_size = 2 + len(lead)
        return self._call_models(latent_model_input, t, text, batch_size, ctrl, depth, repeats=len(x)), batch_size

    def _call_models(self, latent_model_input: torch.Tensor, t, text, batch_size: int, ctrl, depth, repeats: int = 1):
        """The ControlNet (with `ctrl`) and the UNet on `repeats` batches of `batch_size` samples each; the per-frame
        inputs are repeated over every sample, as generate.py:255-273 repeats them."""
        batch_size = batch_size * repeats
        if depth is not None:                                                 # generate.py:256-262
            latent_model_input = torch.cat([latent_model_input, depth.repeat(batch_size, 1, 1, 1).to(latent_model_input)],
                                           dim=1)
        kwargs = {}
        if ctrl is not None:                                                  # generate.py:264-273
            controlnet_cond = ctrl.repeat(batch_size, 1, 1, 1)
            down, mid = self.controlnet(latent_model_input, t, encoder_hidden_states=text,
                                        controlnet_cond=controlnet_cond, return_dict=False)
            down = [d * self.control_scale for d in down]                    # utils/utils.py:288-292
            mid *= self.control_scale
            kwargs = {"down_block_additional_residuals": down, "mid_block_additional_residual": mid}
        return self.unet(latent_model_input, t, encoder_hidden_states=text, **kwargs).sample

    # generate.py:281-311 (inversion=False branch)
    def pred_next_x(self, x: torch.Tensor, eps: torch.Tensor, i: int) -> torch.Tensor:
        return ddim_step(x, eps, self.coefficients(i))

    def coefficients(self, i: int):
        """(a, b, c, d) of step i for x <- c * ((x - a * eps) / b) + d * eps: (sigma, mu, mu_prev, sigma_prev), the
        floats pred_next_x takes (generate.py:281-311, inversion=False)."""
        return ddim_coefficients(self._alpha(self.timesteps, i), self._alpha(self.timesteps, i + 1))

    def step_tables(self, device: torch.device):
        """KS's coefficient table ([n_steps, 4] fp32, ops.ddim_table of `coefficients`) and its step index (one int32,
        which every step sets) on `device`, made once: captured graphs hold their addresses."""
        device = torch.device(device)
        if device not in self._tables:
            from . import ops
            coef = ops.ddim_table(self.coefficients(i) for i in range(len(self.timesteps))).to(device)
            self._tables[device] = (coef, torch.zeros(1, dtype=torch.int32, device=device))
        return self._tables[device]

    def _fuses_update(self, x: torch.Tensor) -> bool:
        """Whether a step on `x` that starts (or is captured) now ends each chunk with KS."""
        return (FUSE_STEP_UPDATE and not self.shard and x.is_cuda and x.dtype == torch.float16
                and x.is_contiguous())

    def _chunk_into(self, x: torch.Tensor, t, frames: dict, out: torch.Tensor, lo: int, hi: int, fused: bool):
        """The chunk of frames lo..hi-1 of `x` (with those rows of the per-frame inputs `frames`) into the same rows of
        `out`: with `fused` its x_{t-1} by KS at the step index that step() set, else its noise prediction
        (pred_noise).  Fused, a UNet output of another dtype gets pred_noise's guidance combine in torch, rounded to
        the latents' dtype as the torch path stores it, and KI's update of the same step.  With K edits, KS (or KI)
        runs once per edit on its rows and its slice of the UNet output."""
        x, frames, out = self._frame_rows(x, lo, hi), _rows(frames, lo, hi), self._frame_rows(out, lo, hi)
        if not fused:
            out.copy_(self.pred_noise(x, t, **frames))
            return
        from . import ops
        coef, step = self.step_tables(x.device)
        eps, samples = self.unet_output(x, t, **frames)
        edits = [(x, eps, out)] if self.edits is None else list(zip(x, eps.chunk(self.edits), out))
        for x, eps, out in edits:
            if eps.dtype == torch.float16:
                ops.cfg_ddim_update(x, eps.contiguous(), samples, self.guidance_scale, coef, step, out)
                continue
            noise = self._guide_edit(eps, samples).to(x.dtype)
            out.copy_(x)
            ops.ddim_update(out, noise.contiguous(), coef, step)

    def _frame_rows(self, x: torch.Tensor, lo: int, hi: int) -> torch.Tensor:
        """Frames lo..hi-1 of latents x: [flen, ...], or [K, flen, ...] with K edits."""
        return x[lo:hi] if self.edits is None else x[:, lo:hi]

    def _flen(self, x: torch.Tensor) -> int:
        return x.shape[0 if self.edits is None else 1]

    def _step_chunks(self, flen: int) -> List[torch.Tensor]:
        chunks = self.get_chunks(flen)
        if not self.shard:
            return chunks
        from . import dist as _dist
        chunks = _dist.shard_chunks(chunks)
        if self.merge_global and patch.GLOBAL_EXCHANGE in ("allgather", "p2p", "p2p_all") and _dist.world() > 1:
            uniform = _dist.check_step_lockstep([len(c) for c in chunks])
            if not uniform and patch.GLOBAL_EXCHANGE in ("p2p", "p2p_all"):
                raise RuntimeError("GLOBAL_EXCHANGE='p2p' needs equally long chunks on every rank (fixed chunking); "
                                   "use 'allgather' for ragged chunks")
        return chunks

    def _block_generators(self) -> List[torch.Generator]:
        seen, gens = set(), []
        for model in self._models():
            for m in model.modules():
                g = getattr(m, "generator", None)
                if isinstance(g, torch.Generator) and g.device.type == "cuda" and id(g) not in seen:
                    seen.add(id(g))
                    gens.append(g)
        return gens

    def _phase(self, t: int) -> tuple:
        """The PnP injections of step t, decided on the host when a graph is captured: attention, and conv when
        pnp_f_t is set."""
        return (self.injecting(t),) if self.pnp_f_t is None else (self.injecting(t), self.conv_injecting(t))

    def _graph_key(self, x: torch.Tensor, t: int):
        return (tuple(x.shape),) + self._phase(t)

    def _lane_streams(self, device: torch.device, n_chunks: int) -> list:
        """The lanes of a capture of `n_chunks` chunks: min(_lane_count, n_chunks) streams of `device`, made once per
        driver (before any capture).  None with shard=True, or before any eager step: then the state that the first
        call of a module creates (packed weights, generators) would be made on one lane and read on another."""
        n = 0 if self.shard or self._eager_steps < 1 else min(self._lane_count, n_chunks)
        lanes = self._lanes.setdefault(device, [])
        while n > 1 and len(lanes) < n:
            lanes.append(torch.cuda.Stream(device))
        return lanes[:n] if n > 1 else []

    def _lane_edges(self, lanes: list, branches: Optional[dict] = None):
        """patch.LaneEdges over every merged block of the models, for a capture on `lanes` (None on one stream), with
        the side streams `branches` of _edit_branches."""
        if not lanes:
            return None
        return patch.LaneEdges((m for model in self._models() for m in model.modules()
                                if type(m).__name__ == "ToMeBlock"), branches=branches)

    def _edit_branches(self, device, lanes: list) -> dict:
        """With K > 1 edits and `lanes`: {lane stream handle: K - 1 side streams}, on which a lane capture runs edits
        1..K-1 of each merged block (their merge paths do not depend on each other), made once per driver and device
        before any capture.  Empty without lanes, with one edit, or once _branch_edits is off."""
        K = getattr(self, "edits", None) or 1
        if K < 2 or not lanes or not self._branch_edits:
            return {}
        made = self._branches.setdefault(device, {})
        for lane in lanes:
            side = made.setdefault(lane.cuda_stream, [])
            while len(side) < K - 1:
                side.append(torch.cuda.Stream(device))
        return {lane.cuda_stream: made[lane.cuda_stream][:K - 1] for lane in lanes}

    def _lanes_fit(self, lanes: list, grids: List[int], device, per_lane: int = 1) -> bool:
        """Whether the KB1 sorts of a capture on `lanes` (their CTA counts `grids`) can all be resident together:
        a sort of at most ops.sort_co_resident CTAs is one launch whose CTAs wait for each other at spin barriers, so
        the sorts that several lanes, each with `per_lane` concurrent branches, may run at once must fit on the device
        side by side."""
        from . import ops
        cap = ops.sort_co_resident(device)
        return len(lanes) * per_lane * max([c for c in grids if c <= cap], default=0) <= cap

    def _record(self, x: torch.Tensor, t: torch.Tensor, frames: dict, spans: List[tuple], *, fused: bool,
                first: bool, key: tuple, phase: tuple) -> _Graph:
        """Capture the chunks `spans` ((lo, hi) rows) of inputs shaped like `x`, with its per-frame inputs `frames` and
        the UNet's timestep input `t`, into one graph: chunk k by _chunk_into on lane k % LANES (run_on_lanes).  The
        global tokens start as at the first chunk of a step (`first`: none) or at a later one (the stores' tokens).
        With K edits, the K merge paths of each merged block run on branches of the lane (_edit_branches).  When the
        KB1 sorts of the lanes and branches would not fit on the device together, it captures again without the
        branches, then on one stream.  Called
        after the eager warm-up steps, so that every lazily created piece of state — generators forked by the hook,
        cached packed weights, the library handle, allocator pools — already exists."""
        from . import ops
        gx = x.clone()
        gframes = {k: v.clone() for k, v in frames.items()}                # the per-frame inputs, set per replay
        lanes = self._lane_streams(x.device, len(spans))
        branches = self._edit_branches(x.device, lanes)
        graph = torch.cuda.CUDAGraph()
        for g in self._block_generators():
            graph.register_generator_state(g)
        if self.merge_global:                                               # host state only
            self._reset_global()
            for st in self._stores:
                st.filled = not first
        torch.cuda.synchronize(x.device)
        with ops.recording_sort_grids() as grids, torch.cuda.graph(graph):
            out = torch.empty_like(gx) if fused else torch.zeros_like(gx)
            run_on_lanes(len(spans), lanes, lambda k: self._chunk_into(gx, t, gframes, out, *spans[k], fused),
                         self._lane_edges(lanes, branches))
        if not self._lanes_fit(lanes, grids, x.device, 1 + max(map(len, branches.values()), default=0)):
            if branches:
                self._branch_edits = False
            else:
                self._lane_count = 1
            return self._record(x, t, frames, spans, fused=fused, first=first, key=key, phase=phase)
        return _Graph(graph=graph, x=gx, t=t, out=out, key=key, frames=gframes, fused=fused, phase=phase)

    def _capture(self, x: torch.Tensor, t: int, frames: dict):
        """Capture the step graph for inputs shaped like `x`: the chunks of _step_chunks or, with capture_global, chunk
        slots (slot k runs rows [k * chunk_size, (k + 1) * chunk_size) of the step's visiting order, which _replay
        applies as data).  Neither draws from the host RNG: fixed chunking with local merging draws nothing, and the
        slots need no chunk list."""
        if self.capture_global and patch.GLOBAL_EXCHANGE != "recurrence":
            raise RuntimeError(f"capture_global=True needs patch.GLOBAL_EXCHANGE='recurrence' (got "
                               f"{patch.GLOBAL_EXCHANGE!r}): the cross-rank exchange is not captured")
        self._graph = None                                                   # release the previous graph first
        cs = self.chunk_size
        flen = self._flen(x)
        spans = ([(lo, lo + cs) for lo in range(0, flen, cs)] if self.capture_global
                 else _spans(self._step_chunks(flen)))
        gt = torch.tensor(int(t), device=x.device, dtype=torch.long)      # the UNet's timestep input, set per replay
        graph = self._record(x, gt, frames, spans, fused=self._fuses_update(x), first=True,
                             key=self._graph_key(x, t), phase=self._phase(t))
        if self.capture_global:
            # the pinned buffer is rewritten only after its last upload has run (the event)
            graph = graph._replace(slots=(torch.empty((2, flen), dtype=torch.int64, device=x.device),
                                          torch.empty((2, flen), dtype=torch.int64).pin_memory(),
                                          torch.cuda.Event()))
        self._graph = graph

    @staticmethod
    def slot_index(chunks: List[torch.Tensor], flen: int) -> torch.Tensor:
        """[2, flen] int64 for a chunk list of equally long chunks: row 0 maps slot position s (slot k covers
        [k * chunk_size, (k + 1) * chunk_size)) to the frame it processes, in the order the chunks are visited; row 1
        is its inverse, frame -> slot position."""
        fwd = torch.cat([c.to(torch.int64) for c in chunks])
        if len(fwd) != flen or len({len(c) for c in chunks}) != 1:
            raise RuntimeError("slot_index: the chunks must be equally long and cover every frame once")
        inv = torch.empty_like(fwd)
        inv[fwd] = torch.arange(flen)
        if not torch.equal(fwd[inv], torch.arange(flen)):
            raise RuntimeError("slot_index: the chunks must cover every frame exactly once")
        return torch.stack([fwd, inv])

    def _replay(self, x: torch.Tensor, t: int, frames: dict):
        """Replay the step graph, capturing it first when the step's key is new; returns its output in frame order and
        whether that is x_{t-1} rather than the noise prediction (a graph replays the path it was captured with).
        With capture_global the step still draws its chunk order on the host with get_chunks, as eager stepping does,
        and applies it as data: one index_select of the inputs into the slots, one of the output back."""
        flen = self._flen(x)
        fd = 0 if self.edits is None else 1                           # the latents' frame dim
        if self.capture_global:
            if flen % self.chunk_size != 0:
                raise RuntimeError(f"capture_global=True needs a frame count divisible by chunk_size (got {flen} "
                                   f"frames, chunk_size {self.chunk_size}): chunks of unequal length cannot share one "
                                   f"graph")
            order = self.slot_index(self.get_chunks(flen), flen)    # the same host draws as eager stepping
        if self._graph is None or self._graph.key != self._graph_key(x, t):
            self._capture(x, t, frames)
        g = self._graph
        if g.slots is None:
            g.x.copy_(x, non_blocking=True)
            for k, v in g.frames.items():
                v.copy_(frames[k], non_blocking=True)
        else:
            index, index_host, copied = g.slots
            copied.synchronize()
            index_host.copy_(order)
            index.copy_(index_host, non_blocking=True)
            copied.record()
            torch.index_select(x, fd, index[0], out=g.x)               # latents -> slots
            for k, v in g.frames.items():
                torch.index_select(frames[k], 0, index[0], out=v)
        g.t.fill_(int(t))
        g.graph.replay()
        if g.slots is not None:
            return torch.index_select(g.out, fd, index[1]), g.fused    # slots -> frames
        return (g.out.clone() if g.fused else g.out), g.fused           # the next replay rewrites out

    @staticmethod
    def draw_dependent_lengths(chunk_size: int, target_stride: int) -> List[int]:
        """Chunk lengths in 1..chunk_size whose local token counts depend on the frame draw: some local level has a
        frame count F with F % min(target_stride, F) != 0 (merge.py:55-57), so its number of dst frames, and every
        count after it, follows the draw.  A level with F % stride == 0 leaves F / stride frames for the next."""
        out = []
        for n in range(1, chunk_size + 1):
            f = n
            while f > 1:
                stride = min(target_stride, f)
                if f % stride:
                    out.append(n)
                    break
                f //= stride
        return out

    def possible_lengths(self, flen: int) -> List[int]:
        """Every chunk length get_chunks can produce for `flen` frames, over all draws."""
        firsts = range(1, self.chunk_size + 1) if self.randomize_chunks else (self.chunk_size,)
        lens = set()
        for f in firsts:
            first = min(f, flen)
            lens.add(first)
            rest = flen - first
            if rest >= self.chunk_size:
                lens.add(self.chunk_size)
            if rest % self.chunk_size:
                lens.add(rest % self.chunk_size)
        return sorted(lens)

    def _check_chunk_lengths(self, flen: int):
        args = self.unet._tome_info["args"] if hasattr(self.unet, "_tome_info") else None
        if patch.GLOBAL_EXCHANGE != "recurrence":
            raise RuntimeError(f"chunk_graphs=True needs patch.GLOBAL_EXCHANGE='recurrence' (got "
                               f"{patch.GLOBAL_EXCHANGE!r}): the cross-rank exchange is not captured")
        if args is None or args["local_merge_ratio"] <= 0:
            return
        bad = sorted(set(self.possible_lengths(flen)) & set(self.draw_dependent_lengths(self.chunk_size,
                                                                                      args["target_stride"])))
        if bad:
            raise RuntimeError(f"chunk_graphs=True: chunks of {bad} frames (possible with {flen} frames and chunk_size "
                               f"{self.chunk_size}) have local token counts that depend on the frame draw (target_stride "
                               f"{args['target_stride']}); they cannot be captured")

    def _install_stores(self):
        self._stores = []
        for model in self._models():
            for m in model.modules():
                if type(m).__name__ == "ToMeBlock":
                    stores = [patch.GlobalTokenStore(self.chunk_size) for _ in range(patch.edits_of(m))]
                    m.global_tokens = stores[0] if len(stores) == 1 else stores       # one per edit
                    self._stores.extend(stores)

    def _reset_global(self):
        if self._stores:
            for st in self._stores:                                         # generate.py:233-236 on the stores
                st.reset()
        else:
            # generate.py:233-236: update_patch(pipe, ...) reaches the UNet and pipe.controlnet
            for model in self._models():
                patch.update_patch(model, global_tokens=None)

    def _chunk_graph_step(self, x: torch.Tensor, t: int, frames: dict, fused: bool) -> torch.Tensor:
        """Replay the graph of every chunk of the step on its rows, capturing it first when its key is new; returns the
        step's x_{t-1} with `fused` (the graphs are keyed by it), else its noise prediction."""
        flen = self._flen(x)
        chunks = self.get_chunks(flen)                                      # the same host draws as eager stepping
        if not self._chunk_graphs:
            self._check_chunk_lengths(flen)                                 # before anything is captured
        phase = self._phase(t)
        # the PnP schedules are prefixes of the steps: a graph captured with an injection that has ended never runs
        # again
        self._chunk_graphs = {k: g for k, g in self._chunk_graphs.items()
                              if all(now or not then for then, now in zip(g.phase, phase))}
        if self._chunk_t is None:
            self._chunk_t = torch.tensor(int(t), device=x.device, dtype=torch.long)
        self._chunk_t.fill_(int(t))
        out = torch.empty_like(x)
        # the shape of a frame, and with K edits K
        shape = tuple(x.shape[1:]) if self.edits is None else (self.edits,) + tuple(x.shape[2:])
        for k, (lo, hi) in enumerate(_spans(chunks)):
            first = self.merge_global and k == 0        # whether the blocks' stores are empty when the chunk runs
            key = (hi - lo, first, shape) + phase + (fused,)
            rows = self._frame_rows(x, lo, hi)
            g = self._chunk_graphs.get(key)
            if g is None:
                g = self._chunk_graphs[key] = self._record(rows, self._chunk_t, _rows(frames, lo, hi),
                                                           [(0, hi - lo)], fused=fused, first=first, key=key,
                                                           phase=phase)
            g.x.copy_(rows)
            for name, v in g.frames.items():
                v.copy_(frames[name][lo:hi])
            g.graph.replay()
            self._frame_rows(out, lo, hi).copy_(g.out)
        return out

    # one iteration of generate.py:211-224
    @torch.no_grad()
    def step(self, x: torch.Tensor, i: int) -> torch.Tensor:
        """One denoising step of latents x [flen, 4, h, w], or [K, flen, 4, h, w] with K edits."""
        if self.edits is not None and (x.dim() != 5 or x.shape[0] != self.edits):
            raise ValueError(f"latents of {self.edits} edits must be [{self.edits}, flen, C, h, w] "
                             f"(got {tuple(x.shape)})")
        if self.edit_rows is not None:
            self._check_edit_exchange()
        t = self.timesteps[i]
        frames = {}                                                          # the per-frame inputs, cast to x's dtype
        if self.source_latents is not None:                                 # generate.py:226-231 (pre_iter)
            pnp.register_time(self.unet, t, modules=self._pnp_targets)
            frames["src"] = self.source_latents(t).to(x)
        frames = self._frames(x if self.edits is None else x[0], frames)    # shared by every edit
        if self.chunk_graphs and self.merge_global and x.is_cuda and not self._stores:
            self._install_stores()
        fused = self._fuses_update(x)
        if fused or x.device in self._tables:                               # KS's step index, read on the device
            self.step_tables(x.device)[1].fill_(i)
        if not (self.cuda_graph and x.is_cuda and self._eager_steps >= self.graph_warmup):
            self._eager_steps += 1
            out = torch.empty_like(x) if fused else torch.zeros_like(x)
            for lo, hi in _spans(self._step_chunks(self._flen(x))):
                self._chunk_into(x, t, frames, out, lo, hi, fused)
        elif self.chunk_graphs:
            out = self._chunk_graph_step(x, t, frames, fused)
        else:
            out, fused = self._replay(x, t, frames)
        x = out if fused else self.pred_next_x(x, out, i)
        if self.merge_global:
            self._reset_global()
        return x

    @torch.no_grad()
    def sample(self, x: torch.Tensor) -> torch.Tensor:
        """Every step from x.  With K edits, x [flen, 4, h, w] starts every edit (the reference's one init_noise for
        all prompts); [K, flen, 4, h, w] gives each its own.  With the edits sharded (shard=True, K > 1) x may also be
        the rank's [K_r, flen, 4, h, w], and every rank returns all K edits."""
        if self.edit_rows is not None:
            self._check_edit_lockstep(x)
            if x.dim() == 5 and x.shape[0] == self.job_edits:
                x = x[self.edit_rows]
        if self.edits is not None and x.dim() == 4:
            x = x.expand(self.edits, *x.shape).contiguous()
        for i in range(len(self.timesteps)):
            x = self.step(x, i)
        if self.edit_rows is not None:
            from . import dist as _dist
            x = _dist.gather_edits(x, self.job_edits)
        return x

    @staticmethod
    def _check_edit_exchange():
        if patch.GLOBAL_EXCHANGE != "recurrence":
            raise ValueError(f"shard=True over several edits needs patch.GLOBAL_EXCHANGE='recurrence' (got "
                             f"{patch.GLOBAL_EXCHANGE!r}): every rank runs the whole recurrence of its own edits, and "
                             f"the exchange modes, made for chunk sharding, would mix edits between ranks")

    def _check_edit_lockstep(self, x: torch.Tensor):
        """Before a sharded sample(): ValueError on every rank unless all ranks agree on what decides their draws and
        their shapes (dist.check_ranks_agree).  The draws are those of get_chunks (torch's CPU generator, and numpy's
        with randomize_chunks), of the blocks' generators once forked, else of the default generator of x's device from
        which they are forked."""
        import hashlib
        from . import dist as _dist
        digest = hashlib.sha256(torch.get_rng_state().numpy().tobytes())
        if x.is_cuda:
            digest.update(torch.cuda.get_rng_state(x.device).numpy().tobytes())
        for model in self._models():
            for m in model.modules():
                g = getattr(m, "generator", None)
                if isinstance(g, torch.Generator):
                    digest.update(g.get_state().numpy().tobytes())
        if self.randomize_chunks:
            name, keys, pos, gauss, cached = np.random.get_state()
            digest.update(keys.tobytes() + repr((name, pos, gauss, cached)).encode())
        _dist.check_ranks_agree({
            "edits": self.job_edits,
            "latents": (x.dim() == 4 or (x.dim() == 5 and x.shape[0] in (self.job_edits, self.edits)),
                        tuple(x.shape[-4:])),
            "n_timesteps": len(self.timesteps),
            "mode": (self.cuda_graph, self.capture_global, self.chunk_graphs, self.graph_warmup, self.merge_global,
                     self.chunk_size, self.chunk_ord, self.perm_div, self.randomize_chunks),
            "exchange": patch.GLOBAL_EXCHANGE,
            "rng": digest.hexdigest()[:16],
        })

    def close(self):
        """Release the captured graphs and give a ControlNet this driver served its own classes back.  The driver may
        step again afterwards: it then serves the ControlNet and captures anew."""
        self._graph = None
        self._chunk_graphs = {}
        self._eager_steps = 0
        self._serving.close()


class ChunkedInverter(_Driver):
    """DDIM inversion of source latents in frame batches, invert.py:117-211 (`Inverter.ddim_inversion`, `pred_noise`,
    `pred_next_x(..., inversion=True)`): the trajectory PnP generation reads (`ChunkedDenoiser(source_latents=...)`).

    Per step, over the reversed DDIM timesteps, every batch of `batch_size` frames (the last one may be ragged) gets
    the noise prediction of the UNet under torch.autocast("cuda", fp16) (invert.py:121) with its rows of `cond`
    ([F | 1, 77, D]: one text embedding per frame as prepare_cond builds it, or one for all), optionally with the
    residuals of `controlnet` on `control_images` ([F, 3, H, W]) scaled by `control_scale` (invert.py:170-176, no CFG
    repeat); then the latents take the inversion step
        x <- mu * (x - sigma_prev * eps) / mu_prev + sigma * eps.
    The latents after every step whose timestep is in the save schedule (`save_steps` DDIM steps, the reference's
    `timesteps_to_save`; only with `save_intermediate`) and after the last step are kept, as invert.py:132-138 saves
    them, in one device tensor `trajectory` [n_saved, F, 4, h, w] ordered as `saved_timesteps`.

    A patched model (apply_patch) runs inside patch._unmerged_blocks(), i.e. as the reference's unpatched UNet: no merge,
    no draw, no PnP injection, and attn1 of stock modules through KD with the residual in its out projection.  An
    unpatched model runs its own forward.  On CUDA fp16 latents the update is KI (vtm_ddim_update_f16), which also stores
    the kept latents; elsewhere it is pred_next_x in torch ops (float64 schedule constants as ChunkedDenoiser).

    `cuda_graph=True` (CUDA fp16 latents): after `graph_warmup` eager steps one CUDA graph covers a whole step, i.e.
    every batch's ControlNet and UNet call and KI with the trajectory store.  The UNet's timestep input, KI's
    coefficients and its trajectory slot are read on the device from a step counter the graph advances, so each further
    step is one replay, bit-identical to eager stepping.

    `depth` ([F, 1, h, w], the reference's prepare_depth output) inverts with SD2-depth's 5-channel UNet: every UNet call
    gets the batch's latents with its depth maps appended as a fifth channel, cast to the latents' dtype
    (invert.py:161-166), eagerly and in the captured step.  The update and the trajectory keep the 4 latent channels.
    Depth with `controlnet` is refused, as in ChunkedDenoiser.

    An unpatched `controlnet` runs its modules' own forwards; with patch.FUSE_CONTROLNET_BLOCKS on, the first invert()
    serves it (patch.serve_unmerged), so that its blocks and Transformer2DModel wrappers run in the library, unmerged,
    as a patched model's do here.  close() gives it its own classes back.

    reconstruct() samples the inverted latents back to clean latents (the reference's `recon`, invert.py:142-157): the
    same batches and per-frame inputs over the forward timesteps, with the sampling update, eagerly or from one CUDA
    graph per step as above.

    `shard=True`: this process is one rank of an initialised torch.distributed job.  No op of the unmerged UNet mixes
    frames, so every batch is independent of the others for all steps: rank r runs the batches k with k % world == r
    (dist.shard_batches) on compact local latents, per-frame inputs and cond rows, and captures only those batches.
    invert() and reconstruct() end with one all-gather (dist.gather_batches, outside any graph) that gives every rank
    the whole result in frame order.  Batch shapes are those of the unsharded run, so every frame is computed as there:
    bit-identical to it whenever the UNet computes a batch the same way in every process, as the library does (torch's
    SDPA, which runs attention above attention.MAX_HEAD_DIM, may differ between processes in the last bits).  A rank
    without a batch still joins the gather.  Nothing crosses ranks during the steps."""

    def __init__(self, unet: torch.nn.Module, n_timesteps: int = 50, batch_size: int = 8,
                 save_steps: Optional[int] = None, save_intermediate: bool = True, cond: Optional[torch.Tensor] = None,
                 controlnet: Optional[torch.nn.Module] = None, control_images: Optional[torch.Tensor] = None,
                 control_scale: float = 1.0, cuda_graph: bool = False, graph_warmup: int = 2,
                 depth: Optional[torch.Tensor] = None, shard: bool = False):
        if not isinstance(n_timesteps, int) or n_timesteps <= 0:
            raise ValueError(f"n_timesteps must be a positive int (got {n_timesteps!r})")
        if not isinstance(batch_size, int) or batch_size <= 0:
            raise ValueError(f"batch_size must be a positive int (got {batch_size!r})")
        save_steps = n_timesteps if save_steps is None else save_steps
        if not isinstance(save_steps, int) or save_steps <= 0:
            raise ValueError(f"save_steps must be a positive int (got {save_steps!r})")
        super().__init__(unet, controlnet, control_images, control_scale, depth)
        if cond is not None and (cond.dim() != 3 or cond.shape[1] != 77):
            raise ValueError(f"cond must be [F | 1, 77, D] (got {tuple(cond.shape)})")
        if cuda_graph and int(graph_warmup) < 1:
            raise ValueError(f"cuda_graph=True needs graph_warmup >= 1 (got {graph_warmup!r}): the modules' packed "
                             f"weights are created by an eager step, outside the graph's memory pool")
        from . import dist as _dist
        if shard and not _dist.initialized():
            raise ValueError("shard=True needs an initialised torch.distributed process group (one rank per process)")
        self.shard = bool(shard)
        self.batch_size = batch_size
        self.cond = cond
        self.cuda_graph = bool(cuda_graph)
        self.graph_warmup = int(graph_warmup)
        self.timesteps = ddim_timesteps(n_timesteps)[::-1]    # invert.py:120: reversed(scheduler.timesteps)
        self.sample_timesteps = ddim_timesteps(n_timesteps)   # invert.py:145: reconstruct() runs forward
        to_save = set(ddim_timesteps(save_steps)) if save_intermediate else set()
        saved = [t for t in self.timesteps if t in to_save]   # invert.py:132
        if self.timesteps[-1] not in saved:                   # invert.py:137-138: the final latents
            saved.append(self.timesteps[-1])
        self.saved_timesteps: List[int] = saved
        self._slot_of = {t: k for k, t in enumerate(saved)}
        self.slots = [self._slot_of.get(t, -1) for t in self.timesteps]
        self.trajectory: Optional[torch.Tensor] = None

    def _patched(self) -> bool:
        return any(hasattr(m, "_tome_info") for m in self._models())

    def coefficients(self, i: int):
        """(a, b, c, d) of step i for x <- c * ((x - a * eps) / b) + d * eps: (sigma_prev, mu_prev, mu, sigma),
        invert.py:182-211 with inversion=True."""
        return ddim_coefficients(self._alpha(self.timesteps, i - 1), self._alpha(self.timesteps, i))

    # invert.py:182-211 (inversion=True branch)
    def pred_next_x(self, x: torch.Tensor, eps: torch.Tensor, i: int) -> torch.Tensor:
        return ddim_step(x, eps, self.coefficients(i))

    # invert.py:159-179
    @torch.no_grad()
    def pred_noise(self, x: torch.Tensor, cond: Optional[torch.Tensor], t, ctrl: Optional[torch.Tensor] = None,
                   depth: Optional[torch.Tensor] = None):
        if depth is not None:                                               # invert.py:161-166
            x = torch.cat([x, depth.to(x)], dim=1)
        kwargs = {}
        if ctrl is not None:                                                # utils/utils.py:280-295
            down, mid = self.controlnet(x, t, encoder_hidden_states=cond, controlnet_cond=ctrl, return_dict=False)
            down = [d * self.control_scale for d in down]
            mid *= self.control_scale
            kwargs = {"down_block_additional_residuals": down, "mid_block_additional_residual": mid}
        return self.unet(x, t, encoder_hidden_states=cond, **kwargs).sample

    # invert.py:142-157 (ddim_sample) and 182-211 (inversion=False branch)
    def sample_coefficients(self, i: int):
        """(a, b, c, d) of reconstruction step i for x <- c * ((x - a * eps) / b) + d * eps: (sigma, mu, mu_prev,
        sigma_prev) over the forward timesteps `sample_timesteps`, final_alpha_cumprod at the last step; the floats
        ChunkedDenoiser.coefficients gives for the same schedule."""
        return ddim_coefficients(self._alpha(self.sample_timesteps, i), self._alpha(self.sample_timesteps, i + 1))

    def sample_next_x(self, x: torch.Tensor, eps: torch.Tensor, i: int) -> torch.Tensor:
        """Reconstruction step i in torch ops (invert.py:182-211 with inversion=False)."""
        return ddim_step(x, eps, self.sample_coefficients(i))

    def _check_cond(self, flen: int):
        if self.cond is not None and self.cond.shape[0] not in (1, flen):
            raise ValueError(f"cond has {self.cond.shape[0]} rows for {flen} frames (one per frame, or one for all)")

    @staticmethod
    def _batch_cond(cond: Optional[torch.Tensor], lo: int, hi: int) -> Optional[torch.Tensor]:
        """Frames lo..hi-1 of `cond`: its rows, or its one row for every frame."""
        if cond is None:
            return None
        return cond.expand(hi - lo, -1, -1) if cond.shape[0] == 1 else cond[lo:hi]

    def _all_noises(self, x: torch.Tensor, t, frames: dict, cond: Optional[torch.Tensor],
                    out: Optional[torch.Tensor] = None):
        """`frames`: the per-frame inputs besides the latents, {"ctrl" | "depth": [F, ...]} (those in use), and `cond`
        the text embeddings ([F | 1, 77, D] or None), both for the frames of `x`."""
        flen = len(x)
        noises = torch.empty_like(x) if out is None else out
        for lo in range(0, flen, self.batch_size):                         # invert.py:124-129
            hi = min(lo + self.batch_size, flen)
            noises[lo:hi] = self.pred_noise(x[lo:hi], self._batch_cond(cond, lo, hi), t, **_rows(frames, lo, hi))
        return noises

    def _inputs(self, x: torch.Tensor):
        """Check the latents x [F, 4, h, w] against the per-frame inputs; returns this process's frames of x (a copy)
        and of {"ctrl" | "depth"} and cond (all frames unless shard=True), and whether KI updates them."""
        if x.dim() != 4:
            raise ValueError(f"latents must be [F, 4, h, w] (got {tuple(x.shape)})")
        frames = self._frames(x, {})
        self._check_cond(len(x))                                             # the row count, up front
        kernel = x.is_cuda and x.dtype == torch.float16
        if self.cuda_graph and not kernel:
            raise ValueError("cuda_graph=True needs CUDA fp16 latents: the captured step updates them with KI")
        if not self.shard:
            return x.clone(), frames, self.cond, kernel
        # the rank's whole batches, back to back: the local batches keep the unsharded run's boundaries and shapes
        from . import dist as _dist
        idx = [f for lo, hi in _dist.shard_batches(len(x), self.batch_size) for f in range(lo, hi)]
        idx = torch.tensor(idx, dtype=torch.int64, device=x.device)
        frames = {k: v.index_select(0, idx) for k, v in frames.items()}
        cond = self.cond
        if cond is not None and cond.shape[0] != 1:
            cond = cond.index_select(0, idx.to(cond.device))
        return x.index_select(0, idx), frames, cond, kernel

    def _gather(self, local: torch.Tensor, flen: int, frame_dim: int) -> torch.Tensor:
        if not self.shard:
            return local
        from . import dist as _dist
        return _dist.gather_batches(local, flen, self.batch_size, frame_dim)

    @torch.no_grad()
    def invert(self, x: torch.Tensor) -> torch.Tensor:
        """Invert the clean latents x [F, 4, h, w] (invert.py:117-140).  Returns the final latents (the last entry of
        `trajectory`); `x` itself is not modified.  With shard=True every rank runs its batches
        (dist.shard_batches) and one all-gather at the end gives every rank the whole trajectory, bit-identical to
        the unsharded run's (see the class's note on sharding)."""
        flen = len(x) if x.dim() == 4 else 0
        x, frames, cond, kernel = self._inputs(x)
        traj = torch.empty((len(self.saved_timesteps),) + tuple(x.shape), dtype=x.dtype, device=x.device)
        scope = patch._unmerged_blocks() if self._patched() else contextlib.nullcontext()
        with scope:
            if len(x) == 0:                                                 # a rank without a batch
                pass
            elif kernel:
                coefficients = [self.coefficients(i) for i in range(len(self.timesteps))]
                self._run_device(x, frames, cond, coefficients, self.timesteps, self.slots, traj)
            else:
                with torch.autocast(x.device.type, dtype=torch.float16, enabled=x.is_cuda):
                    for i, t in enumerate(self.timesteps):
                        x = self.pred_next_x(x, self._all_noises(x, t, frames, cond), i)
                        if self.slots[i] >= 0:
                            traj[self.slots[i]] = x
        self.trajectory = self._gather(traj, flen, 1)
        return self.trajectory[-1]

    @torch.no_grad()
    def reconstruct(self, x: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Sample the inverted latents back to clean latents (the reference's `recon`, Inverter.ddim_sample,
        invert.py:142-157 and 272-273): over the forward DDIM timesteps, every batch's noise prediction with its rows
        of cond and of the ControlNet or depth inputs, as in invert() (no CFG), then x <- mu_prev * (x - sigma * eps) /
        mu + sigma_prev * eps.  `x` [F, 4, h, w] defaults to the last entry of `trajectory`; it is not modified.
        Returns [F, 4, h, w].  On CUDA fp16 the update is KI with the sampling coefficients and no trajectory, and
        with cuda_graph=True each step after the `graph_warmup` eager ones is one replay; elsewhere it is
        sample_next_x.  With shard=True the ranks split the batches as in invert() and gather the result once."""
        if x is None:
            if self.trajectory is None:
                raise RuntimeError("reconstruct: call invert() first or pass the latents")
            x = self.trajectory[-1]
        flen = len(x) if x.dim() == 4 else 0
        x, frames, cond, kernel = self._inputs(x)
        scope = patch._unmerged_blocks() if self._patched() else contextlib.nullcontext()
        with scope:
            if len(x) == 0:
                pass
            elif kernel:
                coefficients = [self.sample_coefficients(i) for i in range(len(self.sample_timesteps))]
                self._run_device(x, frames, cond, coefficients, self.sample_timesteps)
            else:
                with torch.autocast(x.device.type, dtype=torch.float16, enabled=x.is_cuda):
                    for i, t in enumerate(self.sample_timesteps):
                        x = self.sample_next_x(x, self._all_noises(x, t, frames, cond), i)
        return self._gather(x, flen, 0)

    def _run_device(self, x: torch.Tensor, frames: dict, cond: Optional[torch.Tensor], coefficients,
                    timesteps: List[int], slots: Optional[List[int]] = None, traj: Optional[torch.Tensor] = None):
        """Every step of `timesteps` on x in place, each ending with KI on the step's `coefficients` (a, b, c, d), and
        with `slots` its store of x into `traj`: `graph_warmup` eager steps, then, with cuda_graph=True, one replay
        per step of a graph that reads the UNet's timestep, KI's coefficients and its slot at a device step counter and
        advances it."""
        from . import ops
        coef = ops.ddim_table(coefficients).to(x.device)
        ts = torch.tensor(timesteps, dtype=torch.int64, device=x.device)
        step = torch.zeros(1, dtype=torch.int32, device=x.device)
        if slots is not None:
            slots = torch.tensor(slots, dtype=torch.int32, device=x.device)
        n = len(timesteps)
        eager = n if not self.cuda_graph else min(self.graph_warmup, n)
        with torch.autocast("cuda", dtype=torch.float16):
            for i in range(eager):
                eps = self._all_noises(x, timesteps[i], frames, cond)
                ops.ddim_update(x, eps, coef, step, slots, traj)
                step.add_(1)
        if eager == n:
            return
        graph = torch.cuda.CUDAGraph()
        torch.cuda.synchronize(x.device)
        with torch.cuda.graph(graph), torch.autocast("cuda", dtype=torch.float16, cache_enabled=False):
            gt = torch.index_select(ts, 0, step)                          # the UNet's timestep input, [1]
            eps = self._all_noises(x, gt, frames, cond)
            ops.ddim_update(x, eps, coef, step, slots, traj)
            step.add_(1)
        for _ in range(eager, n):
            graph.replay()
        torch.cuda.synchronize(x.device)
        del graph

    def close(self):
        """Give a ControlNet this inverter served its own classes back (invert() serves it again if called)."""
        self._serving.close()

    def source_latents(self, frame_ids=None) -> Callable[[int], torch.Tensor]:
        """The callable ChunkedDenoiser(source_latents=...) takes: t -> the inverted latents at timestep t [flen, 4,
        h, w] (the reference's load_latent, generate.py:321-341), for the frames `frame_ids` (all when None).  A
        timestep that was not kept raises."""
        if self.trajectory is None:
            raise RuntimeError("source_latents: call invert() first")
        traj = self.trajectory if frame_ids is None else self.trajectory[:, torch.as_tensor(frame_ids).tolist()]

        def load(t: int) -> torch.Tensor:
            k = self._slot_of.get(int(t))
            if k is None:
                raise KeyError(f"no inverted latents were kept at timestep {int(t)} (kept: {self.saved_timesteps}); "
                               f"PnP needs one at every generation timestep: invert with save_intermediate=True and "
                               f"save_steps equal to the generation's n_timesteps")
            return traj[k]

        return load
