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
and, in ChunkedInverter, the reference's Inverter around its hot path:
  ddim_inversion  invert.py:117-140     (reversed timesteps, frame batches, the kept latents)
  pred_noise      invert.py:159-179     (UNet forward, optional ControlNet residuals)
  pred_next_x     invert.py:182-211     (inversion=True branch)
Text conditioning, VAE, ControlNet preprocessing and file IO are outside the hot path and not restated.
"""
from __future__ import annotations

import contextlib
from typing import Callable, Iterable, List, Optional

import numpy as np
import torch

from . import patch, pnp


def ddim_alphas_cumprod(num_train_timesteps: int = 1000, beta_start: float = 0.00085,
                        beta_end: float = 0.012) -> torch.Tensor:
    """Stable Diffusion's "scaled_linear" schedule (what DDIMScheduler.from_pretrained gives for SD1.5/2.1)."""
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float64) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


def ddim_timesteps(n_timesteps: int, num_train_timesteps: int = 1000) -> List[int]:
    """DDIMScheduler.set_timesteps with 'leading' spacing and steps_offset=1 (SD's scheduler config)."""
    ratio = num_train_timesteps // n_timesteps
    return [int(t) + 1 for t in (np.arange(0, n_timesteps) * ratio).round()[::-1]]


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
                 pnp_conv_modules: Optional[Iterable[torch.nn.Module]] = None):
        """`cuda_graph=True`: after `graph_warmup` eager steps, the noise prediction of a whole step (every chunk:
        CFG batch, UNet forward with the merge path, guidance combine) is captured once into a CUDA graph and
        replayed; per step the host then issues one graph launch plus the DDIM update instead of ~250 kernel
        launches.  The frame draws of the local matcher stay on the device (utils.draw_randf) and come from the
        blocks' generators, which are registered with the graph, so replays produce the same sequence of draws —
        and bit-identical latents — as eager stepping.  Needs static shapes: `randomize_chunks=False`, frame counts
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
        and PnP (`source_latents`) are refused together, as the reference takes one (generate.py:61-68)."""
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
        self.unet = unet
        # shard=True: this process is one rank of a torch.distributed job and takes chunks i % world == rank of every
        # step (dist.shard_chunks); with merge_global and a collective exchange mode the ranks are checked for
        # lock-step once per step (dist.check_step_lockstep)
        self.shard = bool(shard)
        self.cuda_graph = bool(cuda_graph)
        self.graph_warmup = int(graph_warmup)
        self._graph = None          # (CUDAGraph, static x, static timestep, static noise, shape[, slot index state])
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
        # (chunk length, first in step, frame shape, PnP injection[, PnP conv injection when pnp_f_t is set])
        #   -> (CUDAGraph, static x, static noise, static source, static control images)
        self._chunk_graphs = {}
        self._chunk_t = None        # the UNet's timestep input shared by the chunk graphs
        self._stores = []           # patch.GlobalTokenStore of every block (chunk_graphs with merge_global)
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
                   ctrl: Optional[torch.Tensor] = None) -> torch.Tensor:
        """`src`: the source latents of the chunk (PnP), prepended to the batch.  `ctrl`: the control images of the
        chunk (ControlNet)."""
        flen = len(x)
        text = None if self.cond is None else self.cond.repeat_interleave(flen, dim=0)
        latent_model_input = torch.cat([x, x])                                # classifier-free guidance
        batch_size = 2
        if src is not None:
            latent_model_input = torch.cat([src.to(x), latent_model_input])
            batch_size += 1
        kwargs = {}
        if ctrl is not None:                                                  # generate.py:264-273
            controlnet_cond = ctrl.repeat(batch_size, 1, 1, 1)
            down, mid = self.controlnet(latent_model_input, t, encoder_hidden_states=text,
                                        controlnet_cond=controlnet_cond, return_dict=False)
            down = [d * self.control_scale for d in down]                    # utils/utils.py:288-292
            mid *= self.control_scale
            kwargs = {"down_block_additional_residuals": down, "mid_block_additional_residual": mid}
        eps = self.unet(latent_model_input, t, encoder_hidden_states=text, **kwargs).sample
        noise_pred_uncond, noise_pred_cond = eps.chunk(batch_size)[-2:]
        return noise_pred_uncond + self.guidance_scale * (noise_pred_cond - noise_pred_uncond)

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

    def _all_noises(self, x: torch.Tensor, t, src: Optional[torch.Tensor] = None,
                    ctrl: Optional[torch.Tensor] = None) -> torch.Tensor:
        noises = torch.zeros_like(x)
        for chunk in self._step_chunks(len(x)):
            # chunks are contiguous frame ranges (possibly visited in another order): slice instead of indexing with
            # a host tensor, which would cost a synchronous host->device copy per chunk per step
            lo, hi = int(chunk[0]), int(chunk[-1]) + 1
            noises[lo:hi] = self.pred_noise(x[lo:hi], t, None if src is None else src[lo:hi],
                                            None if ctrl is None else ctrl[lo:hi])
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

    def _capture(self, x: torch.Tensor, t: int, src: Optional[torch.Tensor], ctrl: Optional[torch.Tensor]):
        """Capture `_all_noises` for inputs shaped like `x` (called after the eager warm-up steps, so that every
        lazily created piece of state — generators forked by the hook, cached packed weights, the library handle,
        allocator pools — already exists)."""
        self._graph = None                                                   # release the previous graph first
        gx = x.clone()
        gsrc = None if src is None else src.to(x).clone()                    # the source latents, set per replay
        gctrl = None if ctrl is None else ctrl.clone()                       # the control images, set per replay
        gt = torch.tensor(int(t), device=x.device, dtype=torch.long)      # the UNet's timestep input, set per replay
        graph = torch.cuda.CUDAGraph()
        for g in self._block_generators():
            graph.register_generator_state(g)
        torch.cuda.synchronize(x.device)
        with torch.cuda.graph(graph):
            gn = self._all_noises(gx, gt, gsrc, gctrl)
        self._graph = (graph, gx, gt, gn, self._graph_key(x, t), gsrc, gctrl)

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

    def _capture_slots(self, x: torch.Tensor, t: int, src: Optional[torch.Tensor], ctrl: Optional[torch.Tensor]):
        """Capture the noise prediction of one step over chunk slots (capture_global=True): slot k runs chunk k of the
        step's visiting order on gx[k * chunk_size:(k + 1) * chunk_size].  get_chunks is not called here, so capturing
        consumes no draw of the host RNG that eager stepping would not."""
        flen, cs = len(x), self.chunk_size
        if patch.GLOBAL_EXCHANGE != "recurrence":
            raise RuntimeError(f"capture_global=True needs patch.GLOBAL_EXCHANGE='recurrence' (got "
                               f"{patch.GLOBAL_EXCHANGE!r}): the cross-rank exchange is not captured")
        self._graph = None                                                   # release the previous graph first
        gx = x.clone()
        gsrc = None if src is None else src.to(x).clone()                   # source latents in slot order
        gctrl = None if ctrl is None else ctrl.clone()                      # control images in slot order
        gt = torch.tensor(int(t), device=x.device, dtype=torch.long)
        graph = torch.cuda.CUDAGraph()
        for g in self._block_generators():
            graph.register_generator_state(g)
        for model in self._models():                                        # slot 0 starts the recurrence afresh
            patch.update_patch(model, global_tokens=None)
        torch.cuda.synchronize(x.device)
        with torch.cuda.graph(graph):
            gn = torch.zeros_like(gx)
            for k in range(flen // cs):
                s = slice(k * cs, (k + 1) * cs)
                gn[s] = self.pred_noise(gx[s], gt, None if gsrc is None else gsrc[s],
                                        None if gctrl is None else gctrl[s])
        idx_dev = torch.empty((2, flen), dtype=torch.int64, device=x.device)
        idx_host = torch.empty((2, flen), dtype=torch.int64).pin_memory()
        copied = torch.cuda.Event()          # the pinned buffer is rewritten only after its last upload has run
        self._graph = (graph, gx, gt, gn, self._graph_key(x, t), idx_dev, idx_host, copied, gsrc, gctrl)

    def _slot_noises(self, x: torch.Tensor, t: int, src: Optional[torch.Tensor] = None,
                     ctrl: Optional[torch.Tensor] = None) -> torch.Tensor:
        flen = len(x)
        if flen % self.chunk_size != 0:
            raise RuntimeError(f"capture_global=True needs a frame count divisible by chunk_size (got {flen} frames, "
                               f"chunk_size {self.chunk_size}): chunks of unequal length cannot share one graph")
        order = self.slot_index(self.get_chunks(flen), flen)        # the same host draws as eager stepping
        if self._graph is None or self._graph[4] != self._graph_key(x, t):
            self._capture_slots(x, t, src, ctrl)
        graph, gx, gt, gn, _, idx_dev, idx_host, copied, gsrc, gctrl = self._graph
        copied.synchronize()
        idx_host.copy_(order)
        idx_dev.copy_(idx_host, non_blocking=True)
        copied.record()
        torch.index_select(x, 0, idx_dev[0], out=gx)                # latents -> slots
        if gsrc is not None:
            torch.index_select(src.to(x), 0, idx_dev[0], out=gsrc)
        if gctrl is not None:
            torch.index_select(ctrl, 0, idx_dev[0], out=gctrl)
        gt.fill_(int(t))
        graph.replay()
        return torch.index_select(gn, 0, idx_dev[1])                # slots -> frames

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

    def _capture_chunk(self, key, x: torch.Tensor, src: Optional[torch.Tensor], ctrl: Optional[torch.Tensor]):
        """Capture the noise prediction of one chunk shaped like `x`; `key[1]` says whether it is the first chunk of a
        step, i.e. whether the blocks' stores are empty when it runs."""
        gx = x.clone()
        gsrc = None if src is None else src.to(x).clone()
        gctrl = None if ctrl is None else ctrl.clone()
        graph = torch.cuda.CUDAGraph()
        for g in self._block_generators():
            graph.register_generator_state(g)
        for st in self._stores:
            st.filled = not key[1]
        torch.cuda.synchronize(x.device)
        with torch.cuda.graph(graph):
            gn = self.pred_noise(gx, self._chunk_t, gsrc, gctrl)
        self._chunk_graphs[key] = (graph, gx, gn, gsrc, gctrl)
        return self._chunk_graphs[key]

    def _chunk_graph_noises(self, x: torch.Tensor, t: int, src: Optional[torch.Tensor] = None,
                            ctrl: Optional[torch.Tensor] = None) -> torch.Tensor:
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
        noises = torch.empty_like(x)
        for k, chunk in enumerate(chunks):
            lo, hi = int(chunk[0]), int(chunk[-1]) + 1
            key = (hi - lo, self.merge_global and k == 0, tuple(x.shape[1:]), inject)
            if self.pnp_f_t is not None:
                key = key + (conv,)
            entry = self._chunk_graphs.get(key)
            if entry is None:
                entry = self._capture_chunk(key, x[lo:hi], None if src is None else src[lo:hi],
                                            None if ctrl is None else ctrl[lo:hi])
            graph, gx, gn, gsrc, gctrl = entry
            gx.copy_(x[lo:hi])
            if gsrc is not None:
                gsrc.copy_(src[lo:hi])
            if gctrl is not None:
                gctrl.copy_(ctrl[lo:hi])
            graph.replay()
            noises[lo:hi].copy_(gn)
        return noises

    # one iteration of generate.py:211-224
    @torch.no_grad()
    def step(self, x: torch.Tensor, i: int) -> torch.Tensor:
        t = self.timesteps[i]
        src = None
        if self.source_latents is not None:                                 # generate.py:226-231 (pre_iter)
            pnp.register_time(self.unet, t, modules=self._pnp_targets)
            src = self.source_latents(t)
        ctrl = None
        if self.controlnet is not None:
            if len(self.control_images) != len(x):
                raise ValueError(f"control_images has {len(self.control_images)} frames, the latents {len(x)}")
            ctrl = self.control_images.to(x)                                # prepare_data's .to(self.init_noise)
        if self.chunk_graphs and self.merge_global and x.is_cuda and not self._stores:
            self._install_stores()
        if self.cuda_graph and x.is_cuda and self._eager_steps >= self.graph_warmup and self.chunk_graphs:
            noises = self._chunk_graph_noises(x, t, src, ctrl)
        elif self.cuda_graph and x.is_cuda and self._eager_steps >= self.graph_warmup and self.capture_global:
            noises = self._slot_noises(x, t, src, ctrl)
        elif self.cuda_graph and x.is_cuda and self._eager_steps >= self.graph_warmup:
            if self._graph is None or self._graph[4] != self._graph_key(x, t):
                self._capture(x, t, src, ctrl)
            graph, gx, gt, gn = self._graph[:4]
            gsrc, gctrl = self._graph[5:7]
            gx.copy_(x, non_blocking=True)
            if gsrc is not None:
                gsrc.copy_(src, non_blocking=True)
            if gctrl is not None:
                gctrl.copy_(ctrl, non_blocking=True)
            gt.fill_(int(t))
            graph.replay()
            noises = gn
        else:
            self._eager_steps += 1
            noises = self._all_noises(x, t, src, ctrl)
        x = self.pred_next_x(x, noises, i)
        if self.merge_global:
            self._reset_global()
        return x

    @torch.no_grad()
    def sample(self, x: torch.Tensor) -> torch.Tensor:
        for i in range(len(self.timesteps)):
            x = self.step(x, i)
        return x


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
    step is one replay, bit-identical to eager stepping."""

    def __init__(self, unet: torch.nn.Module, n_timesteps: int = 50, batch_size: int = 8,
                 save_steps: Optional[int] = None, save_intermediate: bool = True, cond: Optional[torch.Tensor] = None,
                 controlnet: Optional[torch.nn.Module] = None, control_images: Optional[torch.Tensor] = None,
                 control_scale: float = 1.0, cuda_graph: bool = False, graph_warmup: int = 2):
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
        self.unet = unet
        self.batch_size = batch_size
        self.cond = cond
        self.controlnet = controlnet
        self.control_images = control_images
        self.control_scale = control_scale
        self.cuda_graph = bool(cuda_graph)
        self.graph_warmup = int(graph_warmup)
        self.alphas_cumprod = ddim_alphas_cumprod()
        self.final_alpha_cumprod = self.alphas_cumprod[0]     # set_alpha_to_one=False in SD's config
        self.timesteps = ddim_timesteps(n_timesteps)[::-1]    # invert.py:120: reversed(scheduler.timesteps)
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
    def pred_noise(self, x: torch.Tensor, cond: Optional[torch.Tensor], t, ctrl: Optional[torch.Tensor] = None):
        kwargs = {}
        if ctrl is not None:                                                # utils/utils.py:280-295
            down, mid = self.controlnet(x, t, encoder_hidden_states=cond, controlnet_cond=ctrl, return_dict=False)
            down = [d * self.control_scale for d in down]
            mid *= self.control_scale
            kwargs = {"down_block_additional_residuals": down, "mid_block_additional_residual": mid}
        return self.unet(x, t, encoder_hidden_states=cond, **kwargs).sample

    def _batch_cond(self, lo: int, hi: int, flen: int) -> Optional[torch.Tensor]:
        if self.cond is None:
            return None
        if self.cond.shape[0] == 1:
            return self.cond.expand(hi - lo, -1, -1)
        if self.cond.shape[0] != flen:
            raise ValueError(f"cond has {self.cond.shape[0]} rows for {flen} frames (one per frame, or one for all)")
        return self.cond[lo:hi]

    def _all_noises(self, x: torch.Tensor, t, ctrl: Optional[torch.Tensor], out: Optional[torch.Tensor] = None):
        flen = len(x)
        noises = torch.empty_like(x) if out is None else out
        for lo in range(0, flen, self.batch_size):                         # invert.py:124-129
            hi = min(lo + self.batch_size, flen)
            noises[lo:hi] = self.pred_noise(x[lo:hi], self._batch_cond(lo, hi, flen), t,
                                            None if ctrl is None else ctrl[lo:hi])
        return noises

    def _device_tables(self, x: torch.Tensor):
        from . import ops
        coef = ops.ddim_table(self.coefficients(i) for i in range(len(self.timesteps))).to(x.device)
        slots = torch.tensor(self.slots, dtype=torch.int32, device=x.device)
        ts = torch.tensor(self.timesteps, dtype=torch.int64, device=x.device)
        step = torch.zeros(1, dtype=torch.int32, device=x.device)
        return coef, slots, ts, step

    @torch.no_grad()
    def invert(self, x: torch.Tensor) -> torch.Tensor:
        """Invert the clean latents x [F, 4, h, w] (invert.py:117-140).  Returns the final latents (the last entry of
        `trajectory`); `x` itself is not modified."""
        if x.dim() != 4:
            raise ValueError(f"latents must be [F, 4, h, w] (got {tuple(x.shape)})")
        ctrl = None
        if self.controlnet is not None:
            if len(self.control_images) != len(x):
                raise ValueError(f"control_images has {len(self.control_images)} frames, the latents {len(x)}")
            ctrl = self.control_images.to(x)
        if self.cond is not None:
            self._batch_cond(0, 0, len(x))                                 # check the row count up front
        kernel = x.is_cuda and x.dtype == torch.float16
        if self.cuda_graph and not kernel:
            raise ValueError("cuda_graph=True needs CUDA fp16 latents: the captured step updates them with KI")
        x = x.clone()
        traj = torch.empty((len(self.saved_timesteps),) + tuple(x.shape), dtype=x.dtype, device=x.device)
        scope = patch._unmerged_blocks() if self._patched() else contextlib.nullcontext()
        with scope:
            if kernel:
                self._invert_device(x, ctrl, traj)
            else:
                with torch.autocast(x.device.type, dtype=torch.float16, enabled=x.is_cuda):
                    for i, t in enumerate(self.timesteps):
                        x = self.pred_next_x(x, self._all_noises(x, t, ctrl), i)
                        if self.slots[i] >= 0:
                            traj[self.slots[i]] = x
        self.trajectory = traj
        return traj[-1]

    def _invert_device(self, x: torch.Tensor, ctrl: Optional[torch.Tensor], traj: torch.Tensor):
        from . import ops
        coef, slots, ts, step = self._device_tables(x)
        n = len(self.timesteps)
        eager = n if not self.cuda_graph else min(self.graph_warmup, n)
        with torch.autocast("cuda", dtype=torch.float16):
            for i in range(eager):
                eps = self._all_noises(x, self.timesteps[i], ctrl)
                ops.ddim_update(x, eps, coef, step, slots, traj)
                step.add_(1)
        if eager == n:
            return
        graph = torch.cuda.CUDAGraph()
        torch.cuda.synchronize(x.device)
        with torch.cuda.graph(graph), torch.autocast("cuda", dtype=torch.float16, cache_enabled=False):
            gt = torch.index_select(ts, 0, step)                          # the UNet's timestep input, [1]
            eps = self._all_noises(x, gt, ctrl)
            ops.ddim_update(x, eps, coef, step, slots, traj)
            step.add_(1)
        for _ in range(eager, n):
            graph.replay()
        torch.cuda.synchronize(x.device)
        del graph

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
