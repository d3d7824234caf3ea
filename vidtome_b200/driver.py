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
from typing import Callable, Iterable, List, Optional

import numpy as np
import torch

from . import patch, pnp

# On CUDA fp16 latents (shard=False), every chunk of a ChunkedDenoiser step ends with KS (ops.cfg_ddim_update): the
# guidance combine and the DDIM update of the chunk's rows in one kernel, its coefficients read from a device table at a
# device step index, so that a captured step includes the update.  Bit-identical to pred_noise's combine followed by
# pred_next_x.  Off: the step takes those torch ops.  Read at every eager step and at capture; a graph replays the path
# it was captured with.
FUSE_STEP_UPDATE = True


def ddim_alphas_cumprod(num_train_timesteps: int = 1000, beta_start: float = 0.00085,
                        beta_end: float = 0.012) -> torch.Tensor:
    """Stable Diffusion's "scaled_linear" schedule (what DDIMScheduler.from_pretrained gives for SD1.5/2.1)."""
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float64) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


def ddim_timesteps(n_timesteps: int, num_train_timesteps: int = 1000) -> List[int]:
    """DDIMScheduler.set_timesteps with 'leading' spacing and steps_offset=1 (SD's scheduler config)."""
    ratio = num_train_timesteps // n_timesteps
    return [int(t) + 1 for t in (np.arange(0, n_timesteps) * ratio).round()[::-1]]


def _rows(frames: dict, lo: int, hi: int) -> dict:
    """Frames lo..hi-1 of every per-frame input ({"src" | "ctrl" | "depth": [flen, ...]}) of a step."""
    return {k: v[lo:hi] for k, v in frames.items()}


def _check_depth_arg(depth: Optional[torch.Tensor], controlnet: Optional[torch.nn.Module]):
    if depth is None:
        return
    if depth.dim() != 4 or depth.shape[1] != 1:
        raise ValueError(f"depth must be [flen, 1, h, w] (got {tuple(depth.shape)})")
    if controlnet is not None:
        raise ValueError("depth and controlnet are exclusive: the reference's ControlNets are SD1.5 models with a "
                         "4-channel input, and its configs use no control with the depth model")


def _check_depth(depth: torch.Tensor, x: torch.Tensor, model: torch.nn.Module):
    """One depth map per frame at the latents' resolution, for a model that takes the latent channels + 1."""
    if len(depth) != len(x) or depth.shape[2:] != x.shape[2:]:
        raise ValueError(f"depth is {tuple(depth.shape)}, the latents {tuple(x.shape)}: it needs one map per frame at "
                         f"the latents' resolution")
    n = getattr(getattr(model, "config", None), "in_channels", getattr(model, "in_channels", None))
    if isinstance(n, int) and n != x.shape[1] + 1:
        raise ValueError(f"depth: the model takes {n} input channels, not the latents' {x.shape[1]} and one depth "
                         f"channel")


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


class ChunkedDenoiser:
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
        Depth with `controlnet` is refused: the reference's ControlNets are SD1.5 models with a 4-channel input."""
        _check_depth_arg(depth, controlnet)
        self.depth = depth
        if controlnet is not None and source_latents is not None:
            raise ValueError("controlnet and source_latents (PnP) are exclusive: the reference runs one control mode "
                             "(generate.py:61-68)")
        if (controlnet is None) != (control_images is None):
            raise ValueError("controlnet and control_images go together")
        if control_images is not None and (control_images.dim() != 4 or control_images.shape[1] != 3):
            raise ValueError(f"control_images must be [flen, 3, H, W] (got {tuple(control_images.shape)})")
        self.controlnet = controlnet
        self.control_images = control_images
        self.control_scale = control_scale
        self._serving = _ControlNetServing(controlnet)
        self.unet = unet
        # shard=True: this process is one rank of a torch.distributed job and takes chunks i % world == rank of every
        # step (dist.shard_chunks); with merge_global and a collective exchange mode the ranks are checked for
        # lock-step once per step (dist.check_step_lockstep)
        self.shard = bool(shard)
        self.cuda_graph = bool(cuda_graph)
        self.graph_warmup = int(graph_warmup)
        self._graph = None          # (CUDAGraph, static x, static timestep, static noise or x_{t-1}, key[, slot
                                    #  index state], static per-frame inputs, fused update)
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
        # (chunk length, first in step, frame shape, PnP injection[, PnP conv injection when pnp_f_t is set], fused
        #   update) -> (CUDAGraph, static x, static noise or x_{t-1}, static per-frame inputs {"src" | "ctrl" | "depth"})
        self._chunk_graphs = {}
        self._chunk_t = None        # the UNet's timestep input shared by the chunk graphs
        self._stores = []           # patch.GlobalTokenStore of every block (chunk_graphs with merge_global)
        self._tables = {}           # device -> (KS's coefficient table, its step index), made on first use
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
        self.alphas_cumprod = ddim_alphas_cumprod()
        self.final_alpha_cumprod = self.alphas_cumprod[0]     # set_alpha_to_one=False in SD's config
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
        if self.cond is None or self.cond.dim() != 3 or self.cond.shape[0] != 3 or self.cond.shape[1] != 77:
            raise ValueError("PnP (source_latents) needs cond = [3, 77, D]: the pnp guidance, uncond and cond text "
                             "embeddings (generate.py:101-109)")
        qk_t = int(n_timesteps * pnp_attn_t)
        self.pnp_schedule = self.timesteps[:qk_t] if qk_t >= 0 else []
        pnp.register_attention_control(self.unet, self.pnp_schedule, num_inputs=3, modules=modules)
        self._pnp_targets = pnp._targets(self.unet, modules)

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
        """Classifier-free guidance on the raw UNet output of `batch_size` samples."""
        noise_pred_uncond, noise_pred_cond = eps.chunk(batch_size)[-2:]
        return noise_pred_uncond + self.guidance_scale * (noise_pred_cond - noise_pred_uncond)

    # generate.py:238-273
    def unet_output(self, x: torch.Tensor, t: int, src: Optional[torch.Tensor] = None,
                    ctrl: Optional[torch.Tensor] = None, depth: Optional[torch.Tensor] = None):
        """The raw UNet output of the chunk's batch ([source |] uncond | cond, each len(x) frames) and its number of
        samples, before the guidance combine of pred_noise."""
        flen = len(x)
        text = None if self.cond is None else self.cond.repeat_interleave(flen, dim=0)
        latent_model_input = torch.cat([x, x])                                # classifier-free guidance
        batch_size = 2
        if src is not None:
            latent_model_input = torch.cat([src.to(x), latent_model_input])
            batch_size += 1
        if depth is not None:                                                 # generate.py:256-262
            latent_model_input = torch.cat([latent_model_input, depth.repeat(batch_size, 1, 1, 1).to(x)], dim=1)
        kwargs = {}
        if ctrl is not None:                                                  # generate.py:264-273
            controlnet_cond = ctrl.repeat(batch_size, 1, 1, 1)
            down, mid = self.controlnet(latent_model_input, t, encoder_hidden_states=text,
                                        controlnet_cond=controlnet_cond, return_dict=False)
            down = [d * self.control_scale for d in down]                    # utils/utils.py:288-292
            mid *= self.control_scale
            kwargs = {"down_block_additional_residuals": down, "mid_block_additional_residual": mid}
        eps = self.unet(latent_model_input, t, encoder_hidden_states=text, **kwargs).sample
        return eps, batch_size

    # generate.py:281-311 (inversion=False branch)
    def pred_next_x(self, x: torch.Tensor, eps: torch.Tensor, i: int) -> torch.Tensor:
        t = self.timesteps[i]
        alpha_prod_t = self.alphas_cumprod[t]
        alpha_prod_t_prev = (self.alphas_cumprod[self.timesteps[i + 1]] if i < len(self.timesteps) - 1
                             else self.final_alpha_cumprod)
        mu, sigma = float(alpha_prod_t ** 0.5), float((1 - alpha_prod_t) ** 0.5)
        mu_prev, sigma_prev = float(alpha_prod_t_prev ** 0.5), float((1 - alpha_prod_t_prev) ** 0.5)
        pred_x0 = (x - sigma * eps) / mu
        return mu_prev * pred_x0 + sigma_prev * eps

    def coefficients(self, i: int):
        """(a, b, c, d) of step i for x <- c * ((x - a * eps) / b) + d * eps: (sigma, mu, mu_prev, sigma_prev), the
        floats pred_next_x takes (generate.py:281-311, inversion=False)."""
        t = self.timesteps[i]
        alpha_prod_t = self.alphas_cumprod[t]
        alpha_prod_t_prev = (self.alphas_cumprod[self.timesteps[i + 1]] if i < len(self.timesteps) - 1
                             else self.final_alpha_cumprod)
        mu, sigma = float(alpha_prod_t ** 0.5), float((1 - alpha_prod_t) ** 0.5)
        mu_prev, sigma_prev = float(alpha_prod_t_prev ** 0.5), float((1 - alpha_prod_t_prev) ** 0.5)
        return sigma, mu, mu_prev, sigma_prev

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

    def _next_x_rows(self, x: torch.Tensor, t, frames: dict, out: torch.Tensor):
        """x_{t-1} of one chunk (`x`, with its rows of the per-frame inputs) into `out`, by KS at the step index that
        step() set.  UNet output of another dtype gets pred_noise's guidance combine in torch, rounded to the
        latents' dtype as the torch path stores it, and KI's update of the same step."""
        from . import ops
        coef, step = self.step_tables(x.device)
        eps, samples = self.unet_output(x, t, **frames)
        if eps.dtype == torch.float16:
            ops.cfg_ddim_update(x, eps.contiguous(), samples, self.guidance_scale, coef, step, out)
            return
        noise = self.guide(eps, samples).to(x.dtype)
        out.copy_(x)
        ops.ddim_update(out, noise.contiguous(), coef, step)

    def _all_next_x(self, x: torch.Tensor, t, frames: dict, out: torch.Tensor) -> torch.Tensor:
        """The step's x_{t-1} of every frame into `out`, chunk by chunk (the fused form of _all_noises + pred_next_x;
        shard=False, so the chunks cover every frame)."""
        for chunk in self.get_chunks(len(x)):
            lo, hi = int(chunk[0]), int(chunk[-1]) + 1
            self._next_x_rows(x[lo:hi], t, _rows(frames, lo, hi), out[lo:hi])
        return out

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

    def _all_noises(self, x: torch.Tensor, t, frames: dict) -> torch.Tensor:
        """`frames`: the step's per-frame inputs besides the latents, {"src" | "ctrl" | "depth": [flen, ...]} (those in
        use), passed to pred_noise under these names."""
        noises = torch.zeros_like(x)
        for chunk in self._step_chunks(len(x)):
            # chunks are contiguous frame ranges (possibly visited in another order): slice instead of indexing with
            # a host tensor, which would cost a synchronous host->device copy per chunk per step
            lo, hi = int(chunk[0]), int(chunk[-1]) + 1
            noises[lo:hi] = self.pred_noise(x[lo:hi], t, **_rows(frames, lo, hi))
        return noises

    def _models(self) -> List[torch.nn.Module]:
        """The UNet and, with ControlNet control, the ControlNet: the models whose blocks the driver serves."""
        return [self.unet] + ([self.controlnet] if self.controlnet is not None else [])

    def _block_generators(self) -> List[torch.Generator]:
        seen, gens = set(), []
        for model in self._models():
            for m in model.modules():
                g = getattr(m, "generator", None)
                if isinstance(g, torch.Generator) and g.device.type == "cuda" and id(g) not in seen:
                    seen.add(id(g))
                    gens.append(g)
        return gens

    def _graph_key(self, x: torch.Tensor, t: int):
        if self.pnp_f_t is None:
            return tuple(x.shape), self.injecting(t)
        return tuple(x.shape), self.injecting(t), self.conv_injecting(t)

    def _capture(self, x: torch.Tensor, t: int, frames: dict):
        """Capture the step for inputs shaped like `x`: `_all_next_x` (every chunk's x_{t-1}) when the update is fused
        (_fuses_update), else `_all_noises` (called after the eager warm-up steps, so that every
        lazily created piece of state — generators forked by the hook, cached packed weights, the library handle,
        allocator pools — already exists)."""
        self._graph = None                                                   # release the previous graph first
        gx = x.clone()
        gframes = {k: v.clone() for k, v in frames.items()}                # the per-frame inputs, set per replay
        gt = torch.tensor(int(t), device=x.device, dtype=torch.long)      # the UNet's timestep input, set per replay
        fused = self._fuses_update(x)
        graph = torch.cuda.CUDAGraph()
        for g in self._block_generators():
            graph.register_generator_state(g)
        torch.cuda.synchronize(x.device)
        with torch.cuda.graph(graph):
            # gn: the step's x_{t-1} with the fused update, else its noise prediction
            gn = self._all_next_x(gx, gt, gframes, torch.empty_like(gx)) if fused else self._all_noises(gx, gt, gframes)
        self._graph = (graph, gx, gt, gn, self._graph_key(x, t), gframes, fused)

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

    def _capture_slots(self, x: torch.Tensor, t: int, frames: dict):
        """Capture the noise prediction of one step over chunk slots (capture_global=True): slot k runs chunk k of the
        step's visiting order on gx[k * chunk_size:(k + 1) * chunk_size].  get_chunks is not called here, so capturing
        consumes no draw of the host RNG that eager stepping would not."""
        flen, cs = len(x), self.chunk_size
        if patch.GLOBAL_EXCHANGE != "recurrence":
            raise RuntimeError(f"capture_global=True needs patch.GLOBAL_EXCHANGE='recurrence' (got "
                               f"{patch.GLOBAL_EXCHANGE!r}): the cross-rank exchange is not captured")
        self._graph = None                                                   # release the previous graph first
        gx = x.clone()
        gframes = {k: v.clone() for k, v in frames.items()}                # the per-frame inputs in slot order
        gt = torch.tensor(int(t), device=x.device, dtype=torch.long)
        graph = torch.cuda.CUDAGraph()
        for g in self._block_generators():
            graph.register_generator_state(g)
        for model in self._models():                                        # slot 0 starts the recurrence afresh
            patch.update_patch(model, global_tokens=None)
        fused = self._fuses_update(x)
        torch.cuda.synchronize(x.device)
        with torch.cuda.graph(graph):
            # gn, in slot order: the step's x_{t-1} with the fused update, else its noise prediction
            gn = torch.empty_like(gx) if fused else torch.zeros_like(gx)
            for k in range(flen // cs):
                lo, hi = k * cs, (k + 1) * cs
                if fused:
                    self._next_x_rows(gx[lo:hi], gt, _rows(gframes, lo, hi), gn[lo:hi])
                else:
                    gn[lo:hi] = self.pred_noise(gx[lo:hi], gt, **_rows(gframes, lo, hi))
        idx_dev = torch.empty((2, flen), dtype=torch.int64, device=x.device)
        idx_host = torch.empty((2, flen), dtype=torch.int64).pin_memory()
        copied = torch.cuda.Event()          # the pinned buffer is rewritten only after its last upload has run
        self._graph = (graph, gx, gt, gn, self._graph_key(x, t), idx_dev, idx_host, copied, gframes, fused)

    def _slot_noises(self, x: torch.Tensor, t: int, frames: dict):
        """Replay the slot graph of the step; returns (its output in frame order, whether it is x_{t-1} rather than
        the noise prediction)."""
        flen = len(x)
        if flen % self.chunk_size != 0:
            raise RuntimeError(f"capture_global=True needs a frame count divisible by chunk_size (got {flen} frames, "
                               f"chunk_size {self.chunk_size}): chunks of unequal length cannot share one graph")
        order = self.slot_index(self.get_chunks(flen), flen)        # the same host draws as eager stepping
        if self._graph is None or self._graph[4] != self._graph_key(x, t):
            self._capture_slots(x, t, frames)
        graph, gx, gt, gn, _, idx_dev, idx_host, copied, gframes, fused = self._graph
        copied.synchronize()
        idx_host.copy_(order)
        idx_dev.copy_(idx_host, non_blocking=True)
        copied.record()
        torch.index_select(x, 0, idx_dev[0], out=gx)                # latents -> slots
        for k, g in gframes.items():
            torch.index_select(frames[k], 0, idx_dev[0], out=g)
        gt.fill_(int(t))
        graph.replay()
        return torch.index_select(gn, 0, idx_dev[1]), fused         # slots -> frames

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
                    m.global_tokens = patch.GlobalTokenStore(self.chunk_size)
                    self._stores.append(m.global_tokens)

    def _reset_global(self):
        if self._stores:
            for st in self._stores:                                         # generate.py:233-236 on the stores
                st.reset()
        else:
            # generate.py:233-236: update_patch(pipe, ...) reaches the UNet and pipe.controlnet
            for model in self._models():
                patch.update_patch(model, global_tokens=None)

    def _capture_chunk(self, key, x: torch.Tensor, frames: dict):
        """Capture the noise prediction of one chunk shaped like `x` (with the chunk's rows of the per-frame inputs), or
        with `key[-1]` (the fused update) its x_{t-1}; `key[1]` says whether it is the first chunk of a step, i.e.
        whether the blocks' stores are empty when it runs."""
        gx = x.clone()
        gframes = {k: v.clone() for k, v in frames.items()}
        graph = torch.cuda.CUDAGraph()
        for g in self._block_generators():
            graph.register_generator_state(g)
        for st in self._stores:
            st.filled = not key[1]
        fused = key[-1]
        torch.cuda.synchronize(x.device)
        with torch.cuda.graph(graph):
            # gn: the chunk's x_{t-1} with the fused update, else its noise prediction
            if fused:
                gn = torch.empty_like(gx)
                self._next_x_rows(gx, self._chunk_t, gframes, gn)
            else:
                gn = self.pred_noise(gx, self._chunk_t, **gframes)
        self._chunk_graphs[key] = (graph, gx, gn, gframes)
        return self._chunk_graphs[key]

    def _chunk_graph_step(self, x: torch.Tensor, t: int, i: int, frames: dict) -> torch.Tensor:
        """Replay every chunk's graph; returns the step's x_{t-1}.  The graphs are keyed by whether the step fuses the
        update (_fuses_update): those captured without it give the noise prediction, which pred_next_x then takes."""
        flen = len(x)
        chunks = self.get_chunks(flen)                                      # the same host draws as eager stepping
        if not self._chunk_graphs:
            self._check_chunk_lengths(flen)                                 # before anything is captured
        inject = self.injecting(t)
        if not inject and any(k[3] for k in self._chunk_graphs):
            # the schedule is a prefix of the steps: the injected graphs never run again
            self._chunk_graphs = {k: v for k, v in self._chunk_graphs.items() if not k[3]}
        conv = self.conv_injecting(t)
        if self.pnp_f_t is not None and not conv and any(k[4] for k in self._chunk_graphs):
            # so is the conv schedule
            self._chunk_graphs = {k: v for k, v in self._chunk_graphs.items() if not k[4]}
        if self._chunk_t is None:
            self._chunk_t = torch.tensor(int(t), device=x.device, dtype=torch.long)
        self._chunk_t.fill_(int(t))
        fused = self._fuses_update(x)
        out = torch.empty_like(x)                       # x_{t-1} with the fused update, else the noise prediction
        for k, chunk in enumerate(chunks):
            lo, hi = int(chunk[0]), int(chunk[-1]) + 1
            key = (hi - lo, self.merge_global and k == 0, tuple(x.shape[1:]), inject)
            if self.pnp_f_t is not None:
                key = key + (conv,)
            key = key + (fused,)
            entry = self._chunk_graphs.get(key)
            if entry is None:
                entry = self._capture_chunk(key, x[lo:hi], _rows(frames, lo, hi))
            graph, gx, gn, gframes = entry
            gx.copy_(x[lo:hi])
            for name, g in gframes.items():
                g.copy_(frames[name][lo:hi])
            graph.replay()
            out[lo:hi].copy_(gn)
        return out if fused else self.pred_next_x(x, out, i)

    # one iteration of generate.py:211-224
    @torch.no_grad()
    def step(self, x: torch.Tensor, i: int) -> torch.Tensor:
        t = self.timesteps[i]
        frames = {}                                                          # the per-frame inputs, cast to x's dtype
        if self.depth is not None:
            _check_depth(self.depth, x, self.unet)
        if self.source_latents is not None:                                 # generate.py:226-231 (pre_iter)
            pnp.register_time(self.unet, t, modules=self._pnp_targets)
            frames["src"] = self.source_latents(t).to(x)
        if self.controlnet is not None:
            if len(self.control_images) != len(x):
                raise ValueError(f"control_images has {len(self.control_images)} frames, the latents {len(x)}")
            frames["ctrl"] = self.control_images.to(x)                      # prepare_data's .to(self.init_noise)
            self._serving.before_step()
        if self.depth is not None:
            frames["depth"] = self.depth.to(x)                              # prepare_data's .to(self.init_noise)
        if self.chunk_graphs and self.merge_global and x.is_cuda and not self._stores:
            self._install_stores()
        if self._fuses_update(x) or x.device in self._tables:             # KS's step index, read on the device
            self.step_tables(x.device)[1].fill_(i)
        if self.cuda_graph and x.is_cuda and self._eager_steps >= self.graph_warmup and self.chunk_graphs:
            x = self._chunk_graph_step(x, t, i, frames)
        elif self.cuda_graph and x.is_cuda and self._eager_steps >= self.graph_warmup and self.capture_global:
            out, fused = self._slot_noises(x, t, frames)
            x = out if fused else self.pred_next_x(x, out, i)
        elif self.cuda_graph and x.is_cuda and self._eager_steps >= self.graph_warmup:
            if self._graph is None or self._graph[4] != self._graph_key(x, t):
                self._capture(x, t, frames)
            graph, gx, gt, gn, _, gframes, fused = self._graph
            gx.copy_(x, non_blocking=True)
            for k, g in gframes.items():
                g.copy_(frames[k], non_blocking=True)
            gt.fill_(int(t))
            graph.replay()
            x = gn.clone() if fused else self.pred_next_x(x, gn, i)     # the next replay rewrites gn
        else:
            self._eager_steps += 1
            if self._fuses_update(x):
                x = self._all_next_x(x, t, frames, torch.empty_like(x))
            else:
                x = self.pred_next_x(x, self._all_noises(x, t, frames), i)
        if self.merge_global:
            self._reset_global()
        return x

    @torch.no_grad()
    def sample(self, x: torch.Tensor) -> torch.Tensor:
        for i in range(len(self.timesteps)):
            x = self.step(x, i)
        return x

    def close(self):
        """Release the captured graphs and give a ControlNet this driver served its own classes back.  The driver may
        step again afterwards: it then serves the ControlNet and captures anew."""
        self._graph = None
        self._chunk_graphs = {}
        self._eager_steps = 0
        self._serving.close()


class ChunkedInverter:
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
        if (controlnet is None) != (control_images is None):
            raise ValueError("controlnet and control_images go together")
        if control_images is not None and (control_images.dim() != 4 or control_images.shape[1] != 3):
            raise ValueError(f"control_images must be [F, 3, H, W] (got {tuple(control_images.shape)})")
        if cond is not None and (cond.dim() != 3 or cond.shape[1] != 77):
            raise ValueError(f"cond must be [F | 1, 77, D] (got {tuple(cond.shape)})")
        if cuda_graph and int(graph_warmup) < 1:
            raise ValueError(f"cuda_graph=True needs graph_warmup >= 1 (got {graph_warmup!r}): the modules' packed "
                             f"weights are created by an eager step, outside the graph's memory pool")
        _check_depth_arg(depth, controlnet)
        from . import dist as _dist
        if shard and not _dist.initialized():
            raise ValueError("shard=True needs an initialised torch.distributed process group (one rank per process)")
        self.shard = bool(shard)
        self.depth = depth
        self.unet = unet
        self.batch_size = batch_size
        self.cond = cond
        self.controlnet = controlnet
        self.control_images = control_images
        self.control_scale = control_scale
        self._serving = _ControlNetServing(controlnet)
        self.cuda_graph = bool(cuda_graph)
        self.graph_warmup = int(graph_warmup)
        self.alphas_cumprod = ddim_alphas_cumprod()
        self.final_alpha_cumprod = self.alphas_cumprod[0]     # set_alpha_to_one=False in SD's config
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

    def _models(self) -> List[torch.nn.Module]:
        return [self.unet] + ([self.controlnet] if self.controlnet is not None else [])

    def coefficients(self, i: int):
        """(a, b, c, d) of step i for x <- c * ((x - a * eps) / b) + d * eps: (sigma_prev, mu_prev, mu, sigma),
        invert.py:182-211 with inversion=True."""
        t = self.timesteps[i]
        alpha_prod_t = self.alphas_cumprod[t]
        alpha_prod_t_prev = self.alphas_cumprod[self.timesteps[i - 1]] if i > 0 else self.final_alpha_cumprod
        mu, sigma = float(alpha_prod_t ** 0.5), float((1 - alpha_prod_t) ** 0.5)
        mu_prev, sigma_prev = float(alpha_prod_t_prev ** 0.5), float((1 - alpha_prod_t_prev) ** 0.5)
        return sigma_prev, mu_prev, mu, sigma

    # invert.py:182-211 (inversion=True branch)
    def pred_next_x(self, x: torch.Tensor, eps: torch.Tensor, i: int) -> torch.Tensor:
        sigma_prev, mu_prev, mu, sigma = self.coefficients(i)
        pred_x0 = (x - sigma_prev * eps) / mu_prev
        return mu * pred_x0 + sigma * eps

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
        ts = self.sample_timesteps
        alpha_prod_t = self.alphas_cumprod[ts[i]]
        alpha_prod_t_prev = self.alphas_cumprod[ts[i + 1]] if i < len(ts) - 1 else self.final_alpha_cumprod
        mu, sigma = float(alpha_prod_t ** 0.5), float((1 - alpha_prod_t) ** 0.5)
        mu_prev, sigma_prev = float(alpha_prod_t_prev ** 0.5), float((1 - alpha_prod_t_prev) ** 0.5)
        return sigma, mu, mu_prev, sigma_prev

    def sample_next_x(self, x: torch.Tensor, eps: torch.Tensor, i: int) -> torch.Tensor:
        """Reconstruction step i in torch ops (invert.py:182-211 with inversion=False)."""
        sigma, mu, mu_prev, sigma_prev = self.sample_coefficients(i)
        pred_x0 = (x - sigma * eps) / mu
        return mu_prev * pred_x0 + sigma_prev * eps

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
        frames = {}
        if self.controlnet is not None:
            if len(self.control_images) != len(x):
                raise ValueError(f"control_images has {len(self.control_images)} frames, the latents {len(x)}")
            frames["ctrl"] = self.control_images.to(x)
            self._serving.before_step()
        if self.depth is not None:
            _check_depth(self.depth, x, self.unet)
            frames["depth"] = self.depth.to(x)
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
