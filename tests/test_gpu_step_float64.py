"""Whole denoising and inversion steps against a float64 replay of the same step with the library's own merge decisions.
Needs an H100.

Below one block the suite holds every kernel to float64 (test_gpu_*_core) and test_gpu_block_core replays one patched
block stage by stage.  This file does the same for a whole step of ChunkedDenoiser / ChunkedInverter, so that a correct
kernel handed the wrong sample, chunk, frame or global-token slot by the Python layer fails a comparison:

  1. Record.  The step runs eagerly on CUDA fp16 with its call points wrapped (`_Recorder`, the pattern of
     test_gpu_block_core._Capture): the chunk spans of get_chunks; for every call of a patched block, keyed by module
     and call order, the plan's local map mu, its unmerge map pi, the global stage's map mu_g over [local | global] with
     the merged length M, the local unmerge map tau[:, :L] the global tokens are rewritten with, the coin, and whether
     PnP shares the source sample's queries and keys; the raw UNet output of every chunk and the step's x_{t-1}.  Two
     consecutive steps, so that the reset of the global tokens between steps is covered.

  2. Replay.  The models are copied to float64 before patching (copy.deepcopy(model).double(): exactly the fp16
     weights).  Every BasicTransformerBlock of the float64 copies is replaced by a closure that runs
     test_gpu_block_core._block64 with the maps of the same call; the global tokens are threaded through in float64
     (chunk k + 1 reads the float64 merged tokens of chunk k gathered with the recorded tau), never read from the fp16
     store.  Everything else runs as the float64 torch modules, PnP's torch forwards included, and each chunk's batch,
     guidance and DDIM update are ChunkedDenoiser.unet_output / guide / pred_next_x (ChunkedInverter.pred_noise /
     pred_next_x / sample_next_x) on the float64 models, with the chunk's rows of the per-frame inputs sliced here from
     the recorded spans.  The replay draws nothing: every draw comes from the recording.

  3. Compare.  Every sample of every chunk's raw UNet output (source, uncond, cond) separately, then x_{t-1}: max-norm
     error relative to max|ref| of that sample, against the case's level.

The last tests put one wiring error at a time into the Python layer of the library run and require the comparison that
names it to fail at ten times the case's level or more."""
import copy
import dataclasses
import time

import numpy as np
import pytest
import torch

import test_gpu_block_core as bc
import test_gpu_projection_core as pc
import test_gpu_rows_core as rc
import vidtome_b200
from vidtome_b200 import attention, driver, ops, patch, pnp
from vidtome_b200.driver import ChunkedDenoiser, ChunkedInverter
from vidtome_b200.skeleton import add_lora, make_controlnet, make_skeleton, pnp_attention_modules, pnp_conv_module

pytestmark = pytest.mark.gpu

SAMPLES = {1: ("eps",), 2: ("uncond", "cond"), 3: ("source", "uncond", "cond")}


class Mismatch(AssertionError):
    """A comparison above its level: `errors` {comparison: (largest error, where)} of every failing comparison."""

    def __init__(self, errors, levels):
        self.errors = errors
        super().__init__("; ".join(f"{k}: {e:.3e} at {w} > {levels[k]:.1e}" for k, (e, w) in errors.items()))


# ---------------------------------------------------------------------------------------------------------------------
# recording the library's step

def _clone(v):
    return v.detach().clone() if isinstance(v, torch.Tensor) else v


class _Recorder:
    """Wraps the call points of the Python layer (test_gpu_block_core._Capture's pattern) and keeps what the float64
    replay needs: `calls` {id(block): [one dict per call of its self-attention stage]}, `spans` (one list per
    get_chunks call), `outputs` (one dict per unet_output / pred_noise call) and `updates` (KI's x before and after)."""

    def __init__(self, mp):
        self.calls, self.spans, self.outputs, self.updates = {}, [], [], []
        self.cur = None
        self._wrap(mp, patch, "_self_attention_stage", self._stage)
        self._wrap(mp, patch, "build_merge_plan", self._plan)
        self._wrap(mp, patch, "_global_stage_store", lambda o, a, k: self._local_pi(o, a, k, 4))
        self._wrap(mp, patch, "_global_stage_device_coin", lambda o, a, k: self._local_pi(o, a, k, 3))
        self._wrap(mp, ops, "gather_rows", self._gather)
        self._wrap(mp, ops, "gather_rows_dev", self._gather)
        self._wrap(mp, ops, "unmerge_add", self._unmerge)
        self._wrap(mp, attention, "self_attention", self._attn)
        self._wrap(mp, ChunkedDenoiser, "get_chunks", self._chunks)
        self._wrap(mp, ChunkedDenoiser, "unet_output", self._unet_output)
        self._wrap(mp, ChunkedInverter, "pred_noise", self._pred_noise)
        self._wrap(mp, ops, "ddim_update", self._ddim_update)

    @staticmethod
    def _wrap(mp, owner, name, body):
        orig = getattr(owner, name)
        mp.setattr(owner, name, lambda *a, **k: body(orig, a, k))

    def _stage(self, orig, a, k):
        block = a[0]
        info = getattr(block, "_tome_info", None)
        call = {"plan": None, "glob": bool(info and info["args"]["merge_global"]),
                "rand": info["args"]["global_rand"] if info else None,
                "inject": bool(getattr(block.attn1, "_vtm_pnp", 0)) and pnp.injection_active(block.attn1)}
        self.calls.setdefault(id(block), []).append(call)
        self.cur = call
        try:
            return orig(*a, **k)
        finally:
            self.cur = None

    def _plan(self, orig, a, k):
        plan = orig(*a, **k)
        if plan is not None and self.cur is not None:
            M = plan.merged_tokens.shape[1] if plan.seq_len is None else int(plan.seq_len.item())
            coin = plan.coin if plan.coin is None or isinstance(plan.coin, float) else float(plan.coin.item())
            self.cur["plan"] = dict(B=plan.merged_tokens.shape[0], mu=_clone(plan.mu), pi=_clone(plan.pi), M=M,
                                    coin=coin, host_coin=isinstance(plan.coin, float))
        return plan

    def _local_pi(self, orig, a, k, at):
        if self.cur is not None:
            self.cur["pi_local"] = _clone(a[at])
        return orig(*a, **k)

    def _gather(self, orig, a, k):
        # the global stage's gather of the merged sequence from [local | global] (the local gathers pass ln= and out=)
        if self.cur is not None and "ln" not in k and "out" not in k:
            self.cur["mu_g"], self.cur["cat_len"] = _clone(a[1]), a[0].shape[1]
        return orig(*a, **k)

    def _unmerge(self, orig, a, k):
        if self.cur is not None and a[2] is None:                  # global tokens <- merged tokens at tau[:, :L]
            self.cur["tau"] = _clone(a[1])
        return orig(*a, **k)

    def _attn(self, orig, a, k):
        if self.cur is not None:
            self.cur["shared"] = bool(k.get("shared_qk", False))
        return orig(*a, **k)

    def _chunks(self, orig, a, k):
        chunks = orig(*a, **k)
        self.spans.append([(int(c[0]), int(c[-1]) + 1) for c in chunks])
        return chunks

    def _unet_output(self, orig, a, k):
        eps, samples = orig(*a, **k)
        self.outputs.append({"eps": _clone(eps), "samples": samples})
        return eps, samples

    def _pred_noise(self, orig, a, k):
        eps = orig(*a, **k)
        self.outputs.append({"eps": _clone(eps), "samples": 1})
        return eps

    def _ddim_update(self, orig, a, k):
        before = _clone(a[0])
        out = orig(*a, **k)
        self.updates.append((before, _clone(a[0])))
        return out


# ---------------------------------------------------------------------------------------------------------------------
# the float64 replay

def _block64_module_attn1(blk, h, ctx):
    """test_gpu_block_core._block64 unmerged, but with attn1 through the float64 module's own forward: PnP's torch
    forward, which injects the source frames' queries and keys by itself while its timestep is in the schedule."""
    hd = h.double()
    h1 = blk.attn1(bc._ln64(hd, blk.norm1)) + hd
    h2 = bc._attn64(blk.attn2, bc._ln64(h1, blk.norm2), ctx.double()) + h1
    a, g = bc._lin64(bc._ln64(h2, blk.norm3), blk.ff.proj).chunk(2, -1)
    return bc._lin64(a * pc._gelu64(g), blk.ff.out) + h2


class Replay:
    """Float64 copies of the models with every BasicTransformerBlock's forward replaced by the replay of the recorded
    calls of its fp16 twin, in call order (`calls`: _Recorder.calls, or {} for none: every block unmerged).  The global
    tokens of every block are threaded through in float64 (`stores`); reset() empties them, as the driver does after
    every step."""

    def __init__(self, models, models64, calls):
        self.queue = {k: list(v) for k, v in calls.items()}
        self.stores = {}
        self.blocks = 0
        for model, model64 in zip(models, models64):
            for m, m64 in zip(model.modules(), model64.modules()):
                if type(m64).__name__ == "BasicTransformerBlock":
                    m64.forward = self._forward(id(m), m64)
                    self.blocks += 1

    def reset(self):
        self.stores = {}

    def done(self):
        left = {k: len(v) for k, v in self.queue.items() if v}
        assert not left, f"recorded block calls the replay did not make: {left}"

    def _forward(self, key, blk):
        def forward(hidden_states, encoder_hidden_states=None, **kwargs):
            calls = self.queue.get(key)
            if key in self.queue:
                assert calls, "the replay calls a block more often than the library did"
            call = calls.pop(0) if calls else None
            plan = None if call is None else call["plan"]
            if plan is None:                          # a block that does not merge at this call
                if call is not None and call["inject"]:
                    return _block64_module_attn1(blk, hidden_states, encoder_hidden_states)
                return bc._block64(blk, hidden_states, encoder_hidden_states, None)
            maps = dict(B=plan["B"], mu=plan["mu"], pi=plan["pi"], shared=call.get("shared", False), mu_g=None, M=None,
                        store=None)
            if call["glob"]:
                self._global(blk, call, plan, maps, hidden_states)
            return bc._block64(blk, hidden_states, encoder_hidden_states, maps)
        return forward

    def _global(self, blk, call, plan, maps, h):
        """The global stage in float64 (patch.py:59-82): [local | global] gathered with the recorded mu_g, and the
        block's global tokens rewritten with the local rows of the merged tokens (tau)."""
        B, C = plan["B"], h.shape[-1]
        mu = plan["mu"]
        local = rc._gather(bc._ln64(h.double(), blk.norm1).reshape(B, -1, C), mu)
        L = local.shape[1]
        store = self.stores.get(id(blk))
        if store is None:
            # no global tokens (the first chunk of a step): the block keeps its local tokens
            if "mu_g" in call:
                # the library merged against global tokens the reference does not have; replay the local plan
                assert "pi_local" in call, "the library ran a global stage on the first chunk of a step"
                maps["pi"] = call["pi_local"]
            self.stores[id(blk)] = local
            return
        assert "mu_g" in call and "tau" in call, "the library ran no global stage where global tokens exist"
        mu_g = call["mu_g"].long()[:, :plan["M"]]
        Lg = call["cat_len"] - L
        if plan["host_coin"] and not np.float32(plan["coin"]) > np.float32(call["rand"]):    # patch.py:62, in fp32
            # [global | local] in the host-coin path (patch.py:68-71): as positions of [local | global]
            mu_g = torch.where(mu_g < Lg, mu_g + L, mu_g - Lg)
        if store.shape[1] < Lg:
            # a GlobalTokenStore's capacity: rows past its length must never be read
            pad = torch.full((B, Lg - store.shape[1], C), float("nan"), dtype=store.dtype, device=store.device)
            store = torch.cat([store, pad], 1)
        assert store.shape[1] == Lg, (store.shape, Lg)
        maps.update(mu_g=mu_g, M=plan["M"], store=store)
        merged = rc._gather(torch.cat([local, store], 1), mu_g)
        self.stores[id(blk)] = rc._gather(merged, call["tau"])


# ---------------------------------------------------------------------------------------------------------------------
# cases

@dataclasses.dataclass
class Case:
    level: float                  # max-norm error relative to max|ref|: 2x the largest measured on an H100
    x_level: float = None         # the level of x_{t-1} where it differs (default: `level`)
    frames: int = 8
    chunk: int = 4
    size: int = 16                # latent side
    glob: str = None              # global merging: None, "store" (GlobalTokenStore), "device" (DEVICE_COIN), "host"
    global_rand: float = 0.5
    random_chunks: bool = False
    pnp: bool = False             # PnP: [source | uncond | cond], align_batch, attention and conv injection
    control: str = None           # ControlNet: "unpatched", "patched" (include_control=True) or "served"
                                  # (FUSE_CONTROLNET_BLOCKS)
    depth: bool = False           # SD2-depth skeleton
    lora: str = None              # "diffusers" or "peft" on every projection
    unmerged_attention: bool = False   # FUSE_UNMERGED_ATTENTION with MAX_HEAD_DIM = 160
    invert: str = None            # "invert" or "reconstruct": ChunkedInverter
    steps: tuple = (0, 1)
    n_timesteps: int = 50
    np_seed: int = 2024


# Each level is 2x the largest error of the case over two runs on an H100 80GB (torch 2.11, CUDA 12.8), given in the
# comment with its comparison; the PnP cases, whose x_{t-1} is furthest, hold their UNet outputs to their own level.
# The errors, 0.96e-3 ... 3.6e-3, are about twice the one-block end-to-end errors of test_gpu_block_core (E2E_LEVEL):
# sixteen library blocks in a row plus the fp16 torch ops between them, each block's
# output rounded to fp16; x_{t-1} of the three-sample PnP cases is furthest, as guidance scales the difference of cond
# and uncond by 7.5.
CASES = {
    "local": Case(0.004),                                                                           # 1.92e-3 x_prev
    "local_t4096": Case(0.003, frames=4, size=64),                                                  # 1.48e-3 x_prev
    "global_store_local_src": Case(0.0034, frames=12, glob="store", global_rand=0.0),               # 1.67e-3 x_prev
    "global_store_global_src": Case(0.0036, frames=12, glob="store", global_rand=1.0),              # 1.76e-3 x_prev
    "global_device_coin": Case(0.0034, frames=12, glob="device"),                                   # 1.67e-3 x_prev
    "global_host_coin": Case(0.0034, frames=12, glob="host"),                                       # 1.67e-3 x_prev
    # np seed 3: a first chunk of 3 frames, then 4 and 3, in order
    "random_chunks": Case(0.0032, frames=10, glob="host", random_chunks=True, np_seed=3),           # 1.58e-3 x_prev
    # n_timesteps 4, pnp_attn_t = pnp_f_t = 0.5: step 1 inside both injection windows, step 2 past them
    # 1.48e-3 eps:uncond, 3.21e-3 x_prev
    "pnp": Case(0.003, 0.0065, pnp=True, glob="host", steps=(1, 2), n_timesteps=4),
    "control_unpatched": Case(0.0033, control="unpatched"),                                         # 1.63e-3 x_prev
    "control_patched": Case(0.0034, control="patched", glob="host"),                                # 1.66e-3 eps:cond
    "control_served": Case(0.0029, control="served"),                                               # 1.43e-3 x_prev
    "depth": Case(0.0029, depth=True),                                                              # 1.41e-3 eps:uncond
    # 1.74e-3 eps:source, 3.57e-3 x_prev
    "depth_pnp": Case(0.0035, 0.0072, depth=True, pnp=True, steps=(1, 2), n_timesteps=4),
    "lora_diffusers": Case(0.0044, lora="diffusers"),                                               # 2.20e-3 x_prev
    "lora_peft": Case(0.0044, lora="peft"),                                                         # 2.20e-3 x_prev
    # the 1280-channel blocks' attn1 through KD with the residual, PnP's source frames shared (shared_items)
    # 1.54e-3 eps:cond, 2.93e-3 x_prev
    "unmerged_attention_pnp": Case(0.0031, 0.0059, pnp=True, unmerged_attention=True, steps=(1, 2), n_timesteps=4),
    "invert": Case(0.002, frames=6, invert="invert", n_timesteps=2),                                # 9.60e-4 eps
    "invert_control": Case(0.0023, frames=6, invert="invert", control="served", n_timesteps=2),     # 1.13e-3 eps
    "reconstruct": Case(0.003, frames=6, invert="reconstruct", n_timesteps=2),                     # 1.49e-3 eps
}


class _Pipeline:
    """Name-only stand-ins: apply_patch(include_control=True) patches the `controlnet` of a
    StableDiffusionControlNetPipeline."""


class DiffusionPipeline(_Pipeline):
    pass


class StableDiffusionControlNetPipeline(DiffusionPipeline):
    def __init__(self, unet, controlnet):
        self.unet, self.controlnet = unet, controlnet


def _models(case):
    """(unet, controlnet or None) in fp16 on the GPU, unpatched, with LoRA when the case has it."""
    name = "sd21" if case.depth else "sd15"
    unet = make_skeleton(name, hot_path_only=False, device="cuda", pnp_conv=case.pnp,
                         transformer_io="linear" if case.depth else None, depth=case.depth)
    cn = make_controlnet(name, hot_path_only=False, device="cuda") if case.control else None
    if case.lora:
        add_lora(unet, 16, case.lora)
    return unet, cn


def _inputs(case):
    """Every input of the run: latents, text, source latents per timestep, control images, depth maps."""
    g = torch.Generator(device="cuda").manual_seed(5)
    cad = 1024 if case.depth else 768
    F, s = case.frames, case.size
    inp = {"x": torch.randn((F, 4, s, s), generator=g, device="cuda").half()}
    if case.invert:
        inp["cond"] = torch.randn((F, 77, cad), generator=g, device="cuda").half()
    else:
        inp["cond"] = torch.randn((3 if case.pnp else 2, 77, cad), generator=g, device="cuda").half()
    if case.control:
        inp["ctrl"] = torch.rand((F, 3, 8 * s, 8 * s), generator=g, device="cuda").half()
    if case.depth:
        inp["depth"] = torch.rand((F, 1, s, s), generator=g, device="cuda") * 2 - 1
    if case.pnp:
        inp["sources"] = {}
    return inp


def _source(inp, case):
    def load(t):
        if t not in inp["sources"]:
            gs = torch.Generator(device="cuda").manual_seed(int(t))
            inp["sources"][t] = torch.randn((case.frames, 4, case.size, case.size), generator=gs, device="cuda").half()
        return inp["sources"][t]
    return load


def _switches(mp, case):
    mp.setattr(patch, "DEVICE_COIN", case.glob == "device")
    mp.setattr(patch, "FUSE_CONTROLNET_BLOCKS", case.control == "served")
    mp.setattr(patch, "FUSE_UNMERGED_ATTENTION", case.unmerged_attention)
    mp.setattr(attention, "MAX_HEAD_DIM", 160 if case.unmerged_attention else 128)


def _denoiser(case, unet, cn, inp, fp64=False):
    kw = dict(n_timesteps=case.n_timesteps, chunk_size=case.chunk, cond=inp["cond"])
    if fp64:
        kw["cond"] = inp["cond"].double()
    else:
        kw.update(merge_global=case.glob is not None, randomize_chunks=case.random_chunks)
        if case.pnp:
            kw.update(source_latents=_source(inp, case), pnp_attn_t=0.5, pnp_f_t=0.5,
                      pnp_modules=pnp_attention_modules(unet), pnp_conv_modules=[pnp_conv_module(unet)])
        if case.depth:
            kw.update(depth=inp["depth"])
    if cn is not None:
        ctrl = inp["ctrl"].double() if fp64 else inp["ctrl"]
        kw.update(controlnet=cn, control_images=ctrl, control_scale=0.5)
    return ChunkedDenoiser(unet, **kw)


def _run_library(case, unet, cn, inp, mp, mutate=None):
    """The library's steps under a recorder; returns (recorder, [per step {i, t, x_in, x_out, spans, outputs}])."""
    merge_global = case.glob is not None
    if case.control == "patched":
        vidtome_b200.apply_patch(StableDiffusionControlNetPipeline(unet, cn), merge_global=merge_global,
                                 global_rand=case.global_rand, batch_size=2, include_control=True)
    else:
        vidtome_b200.apply_patch(unet, merge_global=merge_global, global_rand=case.global_rand,
                                 batch_size=3 if case.pnp else 2, align_batch=case.pnp)
    den = _denoiser(case, unet, cn, inp)
    if case.glob == "store":
        den._install_stores()
    _switches(mp, case)
    objs = dict(unet=unet, cn=cn, den=den)
    if mutate is not None:
        mutate(mp, objs)
    rec = _Recorder(mp)
    torch.manual_seed(2024)                      # the device RNG the blocks fork their generators from
    np.random.seed(case.np_seed)                 # get_chunks' host draws
    x, steps = inp["x"], []
    for i in case.steps:
        n_spans, n_out = len(rec.spans), len(rec.outputs)
        x_out = den.step(x, i)
        assert len(rec.spans) == n_spans + 1
        steps.append(dict(i=i, t=den.timesteps[i], x_in=x, x_out=x_out.clone(), spans=rec.spans[-1],
                          outputs=rec.outputs[n_out:]))
        x = x_out
    torch.cuda.synchronize()
    den.close()
    return rec, steps, den


def _rel(got, ref):
    assert torch.isfinite(got).all(), "non-finite library output"
    return ((got.double() - ref).abs().max() / ref.abs().max()).item()


def _replay_denoiser(case, models, models64, inp, rec, steps, den):
    """Every recorded step in float64 from the library's x_t; returns {comparison: (largest error, where)}."""
    unet64, cn64 = models64
    rep = Replay([m for m in models if m is not None], [m for m in models64 if m is not None], rec.calls)
    den64 = _denoiser(case, unet64, cn64, inp, fp64=True)
    targets = []
    if case.pnp:
        # PnP's torch forwards on the float64 modules, registered as the driver registers them
        targets = pnp_attention_modules(unet64) + [pnp_conv_module(unet64)]
        pnp.register_attention_control(unet64, den.pnp_schedule, 3, modules=targets[:-1])
        pnp.register_conv_control(unet64, den.pnp_conv_schedule, 3, modules=targets[-1:])
    errs = {}
    for st in steps:
        i, t = st["i"], st["t"]
        if targets:
            pnp.register_time(unet64, t, modules=targets)
        rep.reset()
        x64 = st["x_in"].double()
        full = {}                                  # the step's per-frame inputs, cast as the driver casts them
        if case.pnp:
            full["src"] = inp["sources"][t].double()
        if case.control:
            full["ctrl"] = inp["ctrl"].double()
        if case.depth:
            full["depth"] = inp["depth"].half().double()
        assert len(st["outputs"]) == len(st["spans"]), "one UNet output per chunk"
        assert sorted(f for lo, hi in st["spans"] for f in range(lo, hi)) == list(range(case.frames))
        out = torch.empty_like(x64)
        for k, ((lo, hi), got) in enumerate(zip(st["spans"], st["outputs"])):
            eps64, samples = den64.unet_output(x64[lo:hi], t, **{n: v[lo:hi] for n, v in full.items()})
            assert samples == got["samples"] and got["eps"].shape == eps64.shape
            for name, a, b in zip(SAMPLES[samples], got["eps"].chunk(samples), eps64.chunk(samples)):
                _note(errs, f"eps:{name}", _rel(a, b), f"step {i} chunk {k} frames {lo}:{hi}")
            out[lo:hi] = den64.pred_next_x(x64[lo:hi], den64.guide(eps64, samples), i)
        _note(errs, "x_prev", _rel(st["x_out"], out), f"step {i}")
    rep.done()
    return errs


def _note(errs, name, e, where):
    if name not in errs or e > errs[name][0]:
        errs[name] = (e, where)


def _run_inverter(case, unet, cn, inp, mp, mutate=None):
    vidtome_b200.apply_patch(unet, batch_size=2)           # a patched UNet inverts inside patch._unmerged_blocks()
    inv = ChunkedInverter(unet, n_timesteps=case.n_timesteps, batch_size=case.chunk, cond=inp["cond"], controlnet=cn,
                          control_images=inp.get("ctrl"), control_scale=0.5)
    _switches(mp, case)
    if mutate is not None:
        mutate(mp, dict(unet=unet, cn=cn, den=inv))
    rec = _Recorder(mp)
    if case.invert == "invert":
        inv.invert(inp["x"])
    else:
        inv.reconstruct(inp["x"])
    torch.cuda.synchronize()
    inv.close()
    return rec, None, inv


def _replay_inverter(case, models, models64, inp, rec, inv):
    unet64, cn64 = models64
    rep = Replay([m for m in models if m is not None], [m for m in models64 if m is not None], rec.calls)
    cond64 = inp["cond"].double()
    ctrl64 = inp["ctrl"].double() if case.control else None
    inv64 = ChunkedInverter(unet64, n_timesteps=case.n_timesteps, batch_size=case.chunk, cond=cond64, controlnet=cn64,
                            control_images=ctrl64, control_scale=0.5)
    ts = inv64.timesteps if case.invert == "invert" else inv64.sample_timesteps
    batches = [(lo, min(lo + case.chunk, case.frames)) for lo in range(0, case.frames, case.chunk)]
    assert len(rec.updates) == len(ts) and len(rec.outputs) == len(ts) * len(batches)
    errs = {}
    for i, (before, after) in enumerate(rec.updates):
        x64 = before.double()
        eps = torch.empty_like(x64)
        for k, (lo, hi) in enumerate(batches):
            frames = {} if ctrl64 is None else {"ctrl": ctrl64[lo:hi]}
            eps[lo:hi] = inv64.pred_noise(x64[lo:hi], cond64[lo:hi], ts[i], **frames)
            _note(errs, "eps:eps", _rel(rec.outputs[i * len(batches) + k]["eps"], eps[lo:hi]),
                  f"step {i} batch {k} frames {lo}:{hi}")
        ref = inv64.pred_next_x(x64, eps, i) if case.invert == "invert" else inv64.sample_next_x(x64, eps, i)
        _note(errs, "x_prev", _rel(after, ref), f"step {i}")
    rep.done()
    return errs


def _run(name, monkeypatch, mutate=None):
    """The library's steps of CASES[name] (with `mutate(mp, objects)` installed first), their float64 replay and the
    errors {comparison: (largest error, where)}."""
    case = CASES[name]
    torch.manual_seed(77)
    unet, cn = _models(case)
    models64 = (copy.deepcopy(unet).double(), None if cn is None else copy.deepcopy(cn).double())
    inp = _inputs(case)
    with monkeypatch.context() as mp:
        if case.invert:
            rec, steps, drv = _run_inverter(case, unet, cn, inp, mp, mutate)
        else:
            rec, steps, drv = _run_library(case, unet, cn, inp, mp, mutate)
    with torch.no_grad():
        if case.invert:
            return _replay_inverter(case, (unet, cn), models64, inp, rec, drv), rec
        return _replay_denoiser(case, (unet, cn), models64, inp, rec, steps, drv), rec


def _levels(name, errs):
    case = CASES[name]
    return {k: case.x_level if k == "x_prev" and case.x_level is not None else case.level for k in errs}


def _check(name, errs):
    levels = _levels(name, errs)
    bad = {k: v for k, v in errs.items() if v[0] > levels[k]}
    if bad:
        raise Mismatch(bad, levels)


# ---------------------------------------------------------------------------------------------------------------------
# the matrix

@pytest.mark.parametrize("name", list(CASES))
def test_step_matches_float64_replay(name, monkeypatch):
    case = CASES[name]
    t0 = time.perf_counter()
    errs, rec = _run(name, monkeypatch)
    calls = [c for v in rec.calls.values() for c in v]
    merged = [c for c in calls if c["plan"] is not None]
    if not case.invert:
        assert merged, "no block merged"
    if case.glob:
        staged = [c for c in merged if "mu_g" in c]
        assert staged, "no global stage ran"
        if case.glob == "store":
            assert all(c["plan"]["host_coin"] is False and "pi_local" in c for c in staged)
        if case.glob == "device":
            assert all(not c["plan"]["host_coin"] for c in staged), "the host coin ran with DEVICE_COIN"
        if case.glob == "host":
            assert all(c["plan"]["host_coin"] for c in staged)
        if case.global_rand in (0.0, 1.0):
            # the coin branch the case forces: coin > global_rand puts the local tokens in src
            assert all((c["plan"]["coin"] > case.global_rand) == (case.global_rand == 0.0) for c in staged)
    if case.pnp:
        assert any(c.get("shared") for c in merged), "no merged block shared the source sample's queries and keys"
    if case.unmerged_attention or case.invert:
        assert any(c["plan"] is None for c in calls)
    levels = _levels(name, errs)
    report = " ".join(f"{k}={e:.2e} (level {levels[k]:.1e})" for k, (e, _) in sorted(errs.items()))
    print(f"{name}: {report}; {time.perf_counter() - t0:.1f} s")
    _check(name, errs)


# ---------------------------------------------------------------------------------------------------------------------
# the harness catches wiring errors of the step

def _swap_guidance(mp, objs):
    """KS takes the cond sample as uncond and the uncond sample as cond."""
    orig = ops.cfg_ddim_update

    def mutated(x, eps, samples, guidance, coef, step, out):
        parts = list(eps.chunk(samples))
        parts[-2], parts[-1] = parts[-1], parts[-2]
        return orig(x, torch.cat(parts).contiguous(), samples, guidance, coef, step, out)
    mp.setattr(ops, "cfg_ddim_update", mutated)


def _controlnet_output(mp, objs, change):
    cn = objs["cn"]
    orig = cn.forward

    def mutated(*a, **k):
        down, mid = orig(*a, **k)
        return change(list(down), mid)
    mp.setattr(cn, "forward", mutated, raising=False)


def _roll_down_residuals(mp, objs):
    """Each down residual handed to the block after its own, within each resolution (rolled by one block)."""
    _controlnet_output(mp, objs, lambda d, m: ([d[1], d[0], d[3], d[2], d[5], d[4]], m))


def _control_scale_twice(mp, objs):
    s = objs["den"].control_scale
    _controlnet_output(mp, objs, lambda d, m: ([r * s for r in d], m * s))


def _depth_next_frame(mp, objs):
    """Each chunk's depth maps taken from the next frame."""
    mp.setattr(driver, "_rows", lambda frames, lo, hi: {k: (torch.roll(v, -1, 0) if k == "depth" else v)[lo:hi]
                                                         for k, v in frames.items()})


def _store_not_reset(mp, objs):
    mp.setattr(ChunkedDenoiser, "_reset_global", lambda self: None)


def _store_from_previous_chunk(mp, objs):
    """The global tokens keep the first chunk's: every later chunk reads tokens older than the previous chunk's."""
    orig = patch.GlobalTokenStore.write

    def mutated(self, rows):
        if not self.filled:
            orig(self, rows)
    mp.setattr(patch.GlobalTokenStore, "write", mutated)


MUTATIONS = {
    "guidance_uncond_cond_swapped": ("local", _swap_guidance, "x_prev"),
    "pnp_source_sample_1": ("pnp", bc._pnp_source_1, "eps:cond"),
    "controlnet_down_residuals_rolled": ("control_unpatched", _roll_down_residuals, "eps:cond"),
    "depth_from_next_frame": ("depth", _depth_next_frame, "eps:cond"),
    "global_store_not_reset": ("global_store_local_src", _store_not_reset, "eps:cond"),
    "global_store_from_older_chunk": ("global_store_local_src", _store_from_previous_chunk, "eps:cond"),
    "control_scale_twice": ("control_unpatched", _control_scale_twice, "eps:cond"),
}


@pytest.mark.parametrize("name", list(MUTATIONS))
def test_harness_catches(name, monkeypatch):
    case_key, mutate, comparison = MUTATIONS[name]
    errs, _ = _run(case_key, monkeypatch, mutate=mutate)
    level = _levels(case_key, errs)[comparison]
    e, where = errs[comparison]
    print(f"{name}: {comparison} {e:.3e} at {where} = {e / level:.0f} x the level of {case_key}")
    with pytest.raises(Mismatch) as info:
        _check(case_key, errs)
    assert comparison in info.value.errors and e >= 10 * level, f"{comparison}: {e:.3e} < 10 x {level:.1e}"
