"""Minimal denoising driver around a patched UNet — the loop the metric "denoising steps/sec" counts.

Restates, on synthetic latents, the parts of the reference's Generator that sit around the hot path:
  get_chunks      generate.py:172-203   (frame chunking; order seq / rand / mix for global merging)
  ddim_sample     generate.py:205-224   (per step: every chunk's pred_noise, then the DDIM update)
  pred_noise      generate.py:238-279   (CFG batch cat([x, x]), UNet forward, guidance combine)
  pred_next_x     generate.py:281-311   (closed-form DDIM step)
  post_iter       generate.py:233-236   (reset global tokens after each step)
Text conditioning, VAE, ControlNet, PnP injection and file IO are outside the hot path and not restated.
"""
from __future__ import annotations

from typing import List, Optional

import numpy as np
import torch

from . import patch


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
                 chunk_graphs: bool = False):
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
        self-attention (KD) in every merged block, and no sharding."""
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
        self._chunk_graphs = {}     # (chunk length, first in step, frame shape) -> (CUDAGraph, static x, static noise)
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
    def pred_noise(self, x: torch.Tensor, t: int) -> torch.Tensor:
        flen = len(x)
        text = None if self.cond is None else self.cond.repeat_interleave(flen, dim=0)
        latent_model_input = torch.cat([x, x])                                # classifier-free guidance
        eps = self.unet(latent_model_input, t, encoder_hidden_states=text).sample
        noise_pred_uncond, noise_pred_cond = eps.chunk(2)
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

    def _all_noises(self, x: torch.Tensor, t) -> torch.Tensor:
        noises = torch.zeros_like(x)
        for chunk in self._step_chunks(len(x)):
            # chunks are contiguous frame ranges (possibly visited in another order): slice instead of indexing with
            # a host tensor, which would cost a synchronous host->device copy per chunk per step
            lo, hi = int(chunk[0]), int(chunk[-1]) + 1
            noises[lo:hi] = self.pred_noise(x[lo:hi], t)
        return noises

    def _block_generators(self) -> List[torch.Generator]:
        seen, gens = set(), []
        for m in self.unet.modules():
            g = getattr(m, "generator", None)
            if isinstance(g, torch.Generator) and g.device.type == "cuda" and id(g) not in seen:
                seen.add(id(g))
                gens.append(g)
        return gens

    def _capture(self, x: torch.Tensor, t: int):
        """Capture `_all_noises` for inputs shaped like `x` (called after the eager warm-up steps, so that every
        lazily created piece of state — generators forked by the hook, cached packed weights, the library handle,
        allocator pools — already exists)."""
        gx = x.clone()
        gt = torch.tensor(int(t), device=x.device, dtype=torch.long)      # the UNet's timestep input, set per replay
        graph = torch.cuda.CUDAGraph()
        for g in self._block_generators():
            graph.register_generator_state(g)
        torch.cuda.synchronize(x.device)
        with torch.cuda.graph(graph):
            gn = self._all_noises(gx, gt)
        self._graph = (graph, gx, gt, gn, tuple(x.shape))

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

    def _capture_slots(self, x: torch.Tensor, t: int):
        """Capture the noise prediction of one step over chunk slots (capture_global=True): slot k runs chunk k of the
        step's visiting order on gx[k * chunk_size:(k + 1) * chunk_size].  get_chunks is not called here, so capturing
        consumes no draw of the host RNG that eager stepping would not."""
        flen, cs = len(x), self.chunk_size
        if patch.GLOBAL_EXCHANGE != "recurrence":
            raise RuntimeError(f"capture_global=True needs patch.GLOBAL_EXCHANGE='recurrence' (got "
                               f"{patch.GLOBAL_EXCHANGE!r}): the cross-rank exchange is not captured")
        gx = x.clone()
        gt = torch.tensor(int(t), device=x.device, dtype=torch.long)
        graph = torch.cuda.CUDAGraph()
        for g in self._block_generators():
            graph.register_generator_state(g)
        patch.update_patch(self.unet, global_tokens=None)                # slot 0 starts the recurrence afresh
        torch.cuda.synchronize(x.device)
        with torch.cuda.graph(graph):
            gn = torch.zeros_like(gx)
            for k in range(flen // cs):
                gn[k * cs:(k + 1) * cs] = self.pred_noise(gx[k * cs:(k + 1) * cs], gt)
        idx_dev = torch.empty((2, flen), dtype=torch.int64, device=x.device)
        idx_host = torch.empty((2, flen), dtype=torch.int64).pin_memory()
        copied = torch.cuda.Event()          # the pinned buffer is rewritten only after its last upload has run
        self._graph = (graph, gx, gt, gn, tuple(x.shape), idx_dev, idx_host, copied)

    def _slot_noises(self, x: torch.Tensor, t: int) -> torch.Tensor:
        flen = len(x)
        if flen % self.chunk_size != 0:
            raise RuntimeError(f"capture_global=True needs a frame count divisible by chunk_size (got {flen} frames, "
                               f"chunk_size {self.chunk_size}): chunks of unequal length cannot share one graph")
        order = self.slot_index(self.get_chunks(flen), flen)        # the same host draws as eager stepping
        if self._graph is None or self._graph[4] != tuple(x.shape):
            self._capture_slots(x, t)
        graph, gx, gt, gn, _, idx_dev, idx_host, copied = self._graph
        copied.synchronize()
        idx_host.copy_(order)
        idx_dev.copy_(idx_host, non_blocking=True)
        copied.record()
        torch.index_select(x, 0, idx_dev[0], out=gx)                # latents -> slots
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
        for m in self.unet.modules():
            if type(m).__name__ == "ToMeBlock":
                m.global_tokens = patch.GlobalTokenStore(self.chunk_size)
                self._stores.append(m.global_tokens)

    def _reset_global(self):
        if self._stores:
            for st in self._stores:                                         # generate.py:233-236 on the stores
                st.reset()
        else:
            patch.update_patch(self.unet, global_tokens=None)               # generate.py:233-236

    def _capture_chunk(self, key, x: torch.Tensor):
        """Capture the noise prediction of one chunk shaped like `x`; `key[1]` says whether it is the first chunk of a
        step, i.e. whether the blocks' stores are empty when it runs."""
        gx = x.clone()
        graph = torch.cuda.CUDAGraph()
        for g in self._block_generators():
            graph.register_generator_state(g)
        for st in self._stores:
            st.filled = not key[1]
        torch.cuda.synchronize(x.device)
        with torch.cuda.graph(graph):
            gn = self.pred_noise(gx, self._chunk_t)
        self._chunk_graphs[key] = (graph, gx, gn)
        return self._chunk_graphs[key]

    def _chunk_graph_noises(self, x: torch.Tensor, t: int) -> torch.Tensor:
        flen = len(x)
        chunks = self.get_chunks(flen)                                      # the same host draws as eager stepping
        if not self._chunk_graphs:
            self._check_chunk_lengths(flen)                                 # before anything is captured
        if self._chunk_t is None:
            self._chunk_t = torch.tensor(int(t), device=x.device, dtype=torch.long)
        self._chunk_t.fill_(int(t))
        noises = torch.empty_like(x)
        for k, chunk in enumerate(chunks):
            lo, hi = int(chunk[0]), int(chunk[-1]) + 1
            key = (hi - lo, self.merge_global and k == 0, tuple(x.shape[1:]))
            entry = self._chunk_graphs.get(key)
            if entry is None:
                entry = self._capture_chunk(key, x[lo:hi])
            graph, gx, gn = entry
            gx.copy_(x[lo:hi])
            graph.replay()
            noises[lo:hi].copy_(gn)
        return noises

    # one iteration of generate.py:211-224
    @torch.no_grad()
    def step(self, x: torch.Tensor, i: int) -> torch.Tensor:
        t = self.timesteps[i]
        if self.chunk_graphs and self.merge_global and x.is_cuda and not self._stores:
            self._install_stores()
        if self.cuda_graph and x.is_cuda and self._eager_steps >= self.graph_warmup and self.chunk_graphs:
            noises = self._chunk_graph_noises(x, t)
        elif self.cuda_graph and x.is_cuda and self._eager_steps >= self.graph_warmup and self.capture_global:
            noises = self._slot_noises(x, t)
        elif self.cuda_graph and x.is_cuda and self._eager_steps >= self.graph_warmup:
            if self._graph is None or self._graph[4] != tuple(x.shape):
                self._capture(x, t)
            graph, gx, gt, gn = self._graph[:4]
            gx.copy_(x, non_blocking=True)
            gt.fill_(int(t))
            graph.replay()
            noises = gn
        else:
            self._eager_steps += 1
            noises = self._all_noises(x, t)
        x = self.pred_next_x(x, noises, i)
        if self.merge_global:
            self._reset_global()
        return x

    @torch.no_grad()
    def sample(self, x: torch.Tensor) -> torch.Tensor:
        for i in range(len(self.timesteps)):
            x = self.step(x, i)
        return x
