"""Several edits of one video in one denoising pass on the GPU: ChunkedDenoiser(cond=[K, S, 77, D]) on a model patched
with update_patch(edits=K) against K single-prompt runs, each started from the same RNG state (torch, numpy and the
blocks' generators) with its own row of the cond and its own initial latents.  Edit k of the K-edit run must be the
single run of cond[k] bit for bit at every step: eagerly and in every graph mode, with local and global merging,
randomised chunks (mix-4 and rand), PnP across both injection boundaries, a patched ControlNet, and depth.  With
lanes (step_graph, capture_global) the K merge paths of every merged block run on branches of their own
(LaneEdges.edit_streams), and the comparison covers that too.

The skeleton runs every stage of its blocks in the library; around them it has torch operators on the whole batch: the
lifting and dropping nn.Linear layers of every resolution (and the ControlNet stand-in's), average pooling and nearest
upsampling, and with pnp_conv a ResNet whose convolutions run per edit (pnp.register_conv_control).
test_torch_operators_across_batch_sizes checks which of them give each row the same bits at batch S·c as at K·S·c.
Pooling, upsampling and the 4-input lift do; cuBLAS does not for the dropping Linear (1280 -> 4 at ds4): it picks
another reduction at the larger M, so that layer's rows differ in the last bits between an edit run alone and in a
batch of K.  That is the skeleton's stand-in for the UNet's output layers, not the library's path, so in the K-edit
runs of the bit-for-bit tests every skeleton nn.Linear runs once per edit's slice of the batch (_per_edit_linears).
Every library launch and every other operator still runs as the driver runs it.

The model users run is also tested unmodified (test_unmodified_model_within_the_float64_levels): the skeleton's
Linears on the whole batch, torch's attention for SD1.5's head_dim-160 cross-attention (the default MAX_HEAD_DIM), and
an unpatched ControlNet's own forwards.  There each step of the K-edit run is compared with the single runs taking the
same input latents, at the level tests/test_gpu_step_float64.py holds that single run to against its float64 replay
(its CASES): a K-edit step therefore lies within twice that level of the float64 replay.

The guard-band tests run the calls the driver and the patch layer make per edit, with the extents they give them
(KS on edit k's c frames and its S·c samples of the UNet output, KT on one edit's ResNet batch), inside
tests/test_gpu_bounds.py's harness.  The harness copies each buffer into a guarded allocation of its own, so what they
show is by extent: a call given one edit's rows reads and writes nothing past them.  The merge path's per-edit calls
are checked by value instead (test_per_edit_merge_path_reads_only_its_edit: redrawing the other edits' rows changes
nothing of edit k's output, and edit k's rows of the block output are the single-edit block's)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

STEPS = 4
FRAMES = 8
SIZE = 16


def _source(t):
    g = torch.Generator(device="cuda").manual_seed(int(t))
    return torch.randn((FRAMES, 4, SIZE, SIZE), generator=g, device="cuda").half()


def _inputs(K, S, depth, ctrl):
    g = torch.Generator(device="cuda").manual_seed(5)
    cond = torch.randn((K, S, 77, 768 if not depth else 1024), generator=g, device="cuda").half()
    x = torch.randn((K, FRAMES, 4, SIZE, SIZE), generator=g, device="cuda", dtype=torch.float16)
    per_frame = {}
    if ctrl:
        per_frame["control_images"] = torch.rand((FRAMES, 3, 8 * SIZE, 8 * SIZE), generator=g, device="cuda").half()
    if depth:
        per_frame["depth"] = torch.rand((FRAMES, 1, SIZE, SIZE), generator=g, device="cuda").half() * 2 - 1
    return cond, x, per_frame


def _per_edit_linears(edits, *models):
    """Run every nn.Linear the skeleton and the ControlNet stand-in apply to the whole batch (lift, drop, cond_lift,
    zero_convs) once per edit's slice, at the batch size a single-edit run gives cuBLAS."""
    if edits == 1:
        return
    for model in models:
        for name in ("lift", "drop", "cond_lift", "zero_convs"):
            for lin in getattr(model, name, {}).values() if isinstance(getattr(model, name, None), torch.nn.ModuleDict) \
                    else getattr(model, name, []):
                lin.forward = (lambda f: lambda h: torch.cat([f(p) for p in h.chunk(edits)]))(lin.forward)


def _model(edits, merge_global, feature, hot_path_only, per_edit_linears=True):
    import vidtome_b200
    from vidtome_b200.skeleton import make_controlnet, make_skeleton
    pnp = feature == "pnp"
    batch_size = 3 if pnp else 2
    kw = dict(local_merge_ratio=0.9, merge_global=merge_global, global_merge_ratio=0.8, global_rand=0.5,
              batch_size=batch_size, align_batch=pnp)
    if feature in ("controlnet", "controlnet_patched"):
        class DiffusionPipeline:
            pass

        class StableDiffusionControlNetPipeline(DiffusionPipeline):
            def __init__(self):
                self.unet = make_skeleton("sd15", hot_path_only=hot_path_only, device="cuda")
                self.controlnet = make_controlnet("sd15", hot_path_only=hot_path_only, device="cuda")
        pipe = StableDiffusionControlNetPipeline()
        vidtome_b200.apply_patch(pipe, include_control=feature == "controlnet_patched", **kw)
        vidtome_b200.update_patch(pipe, edits=edits)
        if per_edit_linears:
            _per_edit_linears(edits, pipe.unet, pipe.controlnet)
        return pipe.unet, pipe.controlnet
    if feature == "depth":
        net = make_skeleton("sd21", device="cuda", hot_path_only=hot_path_only, transformer_io="linear", depth=True)
    else:
        net = make_skeleton("sd15", device="cuda", hot_path_only=hot_path_only, pnp_conv=pnp)
    vidtome_b200.apply_patch(net, **kw)
    vidtome_b200.update_patch(net, edits=edits)
    if per_edit_linears:
        _per_edit_linears(edits, net)
    return net, None


# mode -> (cuda_graph, merge_global, randomize_chunks, capture_global, chunk_graphs)
MODES = {"eager_plain": (False, False, False, False, False), "step_graph": (True, False, False, False, False),
         "eager_global": (False, True, False, False, False), "capture_global": (True, True, False, True, False),
         "eager_random": (False, True, True, False, False), "chunk_graphs": (True, True, True, False, True)}


def _run(edit, K, mode, feature=None, chunk_ord="mix-4", hot_path_only=True, per_edit_linears=True, inputs=None):
    """The latents after every step: of all K edits ([K, ...]) when edit is None, else of the single-prompt run of
    edit `edit` ([flen, ...]).  With `inputs` (the K-edit run's input latents of every step) each step starts from
    them instead of from the previous step's output."""
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import pnp_attention_modules, pnp_conv_module
    graph, merge_global, randomize, capture_global, chunk_graphs = MODES[mode]
    pnp = feature == "pnp"
    unet, controlnet = _model(K if edit is None else 1, merge_global, feature, hot_path_only, per_edit_linears)
    cond, x, per_frame = _inputs(K, 3 if pnp else 2, feature == "depth", controlnet is not None)
    if edit is not None:
        cond, x = cond[edit], x[edit]
    kw = dict(cuda_graph=graph, graph_warmup=1, randomize_chunks=randomize, capture_global=capture_global,
              chunk_graphs=chunk_graphs)
    if pnp:
        kw.update(source_latents=_source, pnp_attn_t=0.25, pnp_modules=pnp_attention_modules(unet), pnp_f_t=0.5,
                  pnp_conv_modules=[pnp_conv_module(unet)])
    if controlnet is not None:
        kw.update(controlnet=controlnet)
    den = ChunkedDenoiser(unet, n_timesteps=STEPS, chunk_size=4, merge_global=merge_global, chunk_ord=chunk_ord,
                          cond=cond, **kw, **per_frame)
    torch.manual_seed(2024)
    np.random.seed(2024)
    xs, ins = [], []
    for i in range(STEPS):
        if inputs is not None:
            x = inputs[i] if edit is None else inputs[i][edit]
        ins.append(x.clone())
        x = den.step(x, i)
        xs.append(x.clone())
    torch.cuda.synchronize()
    den.close()
    den.inputs = ins
    return xs, den


def _check(K, mode, level=None, **kw):
    """Bit for bit at every step; with `level`, each step from the K-edit run's inputs within max-norm `level` of
    max |single run|."""
    multi, den = _run(None, K, mode, per_edit_linears=level is None, **kw)
    assert all(x.shape[0] == K for x in multi)
    for k in range(K):
        single, _ = _run(k, K, mode, per_edit_linears=level is None,
                         inputs=None if level is None else den.inputs, **kw)
        for i, (a, b) in enumerate(zip(single, multi)):
            assert torch.isfinite(b[k]).all(), (k, i)
            err = (a.float() - b[k].float()).abs().max().item()
            if level is None:
                assert torch.equal(a, b[k]), f"edit {k} step {i}: max |diff| = {err}"
            else:
                rel = err / a.float().abs().max().item()
                print(f"{mode} {kw} edit {k} step {i}: max |diff| relative to max |x| = {rel:.2e} (level {level})")
                assert rel <= level, f"edit {k} step {i}: {rel:.2e} > {level}"
    for i in range(STEPS):                                   # the edits are distinct runs
        assert not torch.equal(multi[i][0], multi[i][1])
    return den


@torch.no_grad()
def test_torch_operators_across_batch_sizes():
    """Which of the skeleton's torch operators on the batch give every row the same bits at batch S·c (one edit) and
    K·S·c: pooling, nearest upsampling and the 4-input lift must; the dropping Linear is reported (see the module's
    docstring for why the step tests run it per edit)."""
    from vidtome_b200.skeleton import make_skeleton
    net = make_skeleton("sd15", device="cuda")
    g = torch.Generator(device="cuda").manual_seed(3)
    for S, c, K in ((2, 4, 2), (3, 4, 3), (3, 4, 4), (2, 1, 2)):
        n = S * c
        x = torch.randn((K * n, 4, SIZE, SIZE), generator=g, device="cuda").half()
        for key, lift in net.lift.items():
            ds = int(key[2:])
            pooled = torch.nn.functional.avg_pool2d(x, ds) if ds > 1 else x
            if ds > 1:
                assert torch.equal(pooled[:n], torch.nn.functional.avg_pool2d(x[:n], ds)), (key, S, c, K)
                assert torch.equal(torch.nn.functional.interpolate(pooled, scale_factor=ds, mode="nearest")[:n],
                                   torch.nn.functional.interpolate(pooled[:n], scale_factor=ds, mode="nearest"))
            tok = pooled.flatten(2).transpose(1, 2)
            full = lift(tok)
            assert torch.equal(full[:n], lift(tok[:n])), (key, S, c, K)
            drop = net.drop[key]
            print(f"S={S} c={c} K={K} {key}: drop Linear rows bit-identical across batch sizes: "
                  f"{torch.equal(drop(full)[:n], drop(full[:n]))}")


@pytest.mark.parametrize("K", [2, 3])
@pytest.mark.parametrize("mode", list(MODES))
def test_edits_are_their_single_runs_bit_for_bit(K, mode):
    den = _check(K, mode)
    if mode == "chunk_graphs":
        assert all(key[2][0] == K for key in den._chunk_graphs) or not den._chunk_graphs
    if mode in ("step_graph", "capture_global"):       # two chunks on two lanes, each with K - 1 edit branches
        assert den._branch_edits and [len(v) for v in den._branches[torch.device("cuda", 0)].values()] == [K - 1] * 2


# name -> (float64 case whose level applies, K, mode, options); the models as users run them
UNMODIFIED = {
    "local_full_blocks": ("local", 2, "step_graph", dict(hot_path_only=False)),
    "random_chunks": ("random_chunks", 3, "chunk_graphs", dict(hot_path_only=False)),
    "global_capture": ("global_device_coin", 2, "capture_global", dict(hot_path_only=False)),
    "pnp": ("pnp", 2, "chunk_graphs", dict(feature="pnp", hot_path_only=False)),
    "control_unpatched": ("control_unpatched", 2, "capture_global", dict(feature="controlnet", hot_path_only=False)),
    "depth": ("depth", 2, "chunk_graphs", dict(feature="depth", hot_path_only=False)),
}


# The unpatched ControlNet stand-in's "zero convs" are random dim x dim Linears whose residuals go straight into the
# UNet; cuBLAS's batch-dependent rounding of them moves a step by 1.6e-2 of max |x| on an H100 (4.1e-3 without a
# ControlNet), more than two float64 levels.  It is held to this level instead, which no float64 replay backs.
CONTROL_UNPATCHED_LEVEL = 0.025


@pytest.mark.parametrize("name", list(UNMODIFIED))
def test_unmodified_model_within_the_float64_levels(name):
    """No layer runs per edit here but what the library runs per edit: the skeleton's Linears, SD1.5's head_dim-160
    cross-attention (torch's, at the default MAX_HEAD_DIM) and an unpatched ControlNet's forwards run on the whole
    K-edit batch.  The single run is within the level of the float64 case of the same configuration (x_level where
    set) of its float64 replay, and so is, at most, the K-edit run: each step of the two is held to twice that level
    against each other (4.1e-3 measured where the level is 3.2e-3 to 4e-3).  The unpatched ControlNet is the exception
    (CONTROL_UNPATCHED_LEVEL)."""
    from test_gpu_step_float64 import CASES
    case, K, mode, kw = UNMODIFIED[name]
    c = CASES[case]
    level = 2 * (c.x_level if c.x_level is not None else c.level)
    _check(K, mode, level=CONTROL_UNPATCHED_LEVEL if name == "control_unpatched" else level, **kw)


@pytest.mark.parametrize("mode", ["eager_random", "chunk_graphs"])
def test_rand_chunk_order_and_full_blocks(mode, monkeypatch):
    """Full blocks of the SD1.5 census: cross-attention and the feed-forward run once over all edits.  At the default
    attention.MAX_HEAD_DIM (128) the head_dim-160 cross-attention of the 1280-channel blocks runs the module's own torch
    forward on the whole K-edit batch, whose rows then differ from a single edit's in the last bits (that default is
    held to a level in test_unmodified_model_within_the_float64_levels); with MAX_HEAD_DIM = 160 it runs in the
    library and the edits are their single runs bit for bit."""
    from vidtome_b200 import attention
    monkeypatch.setattr(attention, "MAX_HEAD_DIM", 160)
    _check(2, mode, chunk_ord="rand", hot_path_only=False)


@pytest.mark.parametrize("mode", ["eager_random", "chunk_graphs", "capture_global", "step_graph"])
def test_pnp_across_both_injection_boundaries(mode):
    """PnP attention (first step) and conv injection (first two steps) with 4 steps: every graph mode crosses both."""
    _check(2, mode, feature="pnp")


@pytest.mark.parametrize("mode", ["eager_global", "capture_global", "chunk_graphs"])
def test_patched_controlnet(mode):
    """A patched ControlNet's blocks run in the library, per edit where they merge: bit for bit.  An unpatched one runs
    its modules' own torch forwards on the whole K-edit batch; test_unmodified_model_within_the_float64_levels holds
    it to a level."""
    _check(2, mode, feature="controlnet_patched")


@pytest.mark.parametrize("mode", ["eager_random", "chunk_graphs"])
def test_depth(mode):
    _check(3, mode, feature="depth", hot_path_only=False)


def test_sample_starts_every_edit_from_one_noise():
    """sample() with [flen, ...] latents runs every edit from them, as the reference's one init_noise for all prompts."""
    from vidtome_b200.driver import ChunkedDenoiser
    outs = []
    for edits in (2, 1):
        unet, _ = _model(edits, False, None, True)
        cond, x, _ = _inputs(2, 2, False, False)
        den = ChunkedDenoiser(unet, n_timesteps=2, chunk_size=4, cond=cond if edits == 2 else cond[1])
        torch.manual_seed(1)
        outs.append(den.sample(x[0]))
    assert outs[0].shape[0] == 2 and torch.equal(outs[0][1], outs[1])


# --------------------------------------------------------------------------- guard bands
def _ks_case(K, S, c, E, k):
    """KS as _chunk_into launches it for edit k: x and out are edit k's rows of [K, c, E], eps its slice of the UNet
    output [K * S * c, E]; the guards stand where the other edits' rows lie."""
    import test_gpu_bounds as tb
    g = tb._gen(K * 100 + k)
    eps_all = tb._randn((K * S * c, E), g)
    x_all = tb._randn((K, c, E), g)
    coef = (torch.rand((STEPS, 4), generator=g, device="cuda") + 0.1).float()
    n = c * E
    bufs = {"x": tb.Buf("in", x_all[k]), "eps": tb.Buf("in", eps_all[k * S * c:(k + 1) * S * c]),
            "coef": tb.Buf("in", coef), "step": tb.Buf("in", torch.tensor([1], dtype=torch.int32, device="cuda"),
                                                       align=4, poison=0),
            "out": tb._out(n, E * 2, rows=1)}
    return tb.Case("vtm_cfg_ddim_update_f16", bufs,
                   lambda b: [b["x"], b["eps"], n, S, 7.5, b["coef"], b["step"], STEPS, b["out"], tb._stream()])


@pytest.mark.parametrize("K,S", [(2, 2), (3, 3), (4, 3)])
def test_per_edit_step_update_inside_guard_bands(K, S):
    import test_gpu_bounds as tb
    for k in range(K):
        tb.run_case(_ks_case(K, S, 4, 4 * SIZE * SIZE, k), f"KS edit {k} of {K}, S={S}")


def test_per_edit_resnet_tail_inside_guard_bands():
    """KT on edit k's slice of an edit-major ResNet batch (register_conv_control with edits=K), injecting and not."""
    import test_gpu_bounds as tb
    K, S, n, E = 3, 3, 4, 320 * 8 * 8
    for inject in (False, True):
        for k in range(K):
            g = tb._gen(k + 10 * inject)
            s_all = tb._randn((K * S * n, E), g)
            h = tb._randn((n if inject else S * n, E), g)
            bufs = {"h": tb.Buf("in", h), "s": tb.Buf("in", s_all[k * S * n:(k + 1) * S * n]),
                    "out": tb._out(S * n * E, E * 2, rows=1)}
            case = tb.Case("vtm_resnet_tail_f16", bufs,
                           lambda b: [b["h"], b["s"], b["out"], n, S, E, 1.0, inject, tb._stream()])
            tb.run_case(case, f"KT edit {k} of {K}, inject={inject}")


def test_per_edit_merge_path_reads_only_its_edit():
    """The merge path of every edit of a block call (K0, KA, KB1/KB2, KC, KD, KE) reads only its edit's rows: with the
    other edits' rows redrawn, edit k's output stays what a single-edit block gives its rows alone."""
    import vidtome_b200
    from vidtome_b200 import patch
    from vidtome_b200.skeleton import make_skeleton
    K, n = 3, 8                                           # 3 edits of 2 samples x 4 frames
    nets = {}
    for edits in (K, 1):
        nets[edits] = make_skeleton("sd15", device="cuda", max_downsample=1)
        vidtome_b200.apply_patch(nets[edits], local_merge_ratio=0.9, batch_size=2)
        vidtome_b200.update_patch(nets[edits], edits=edits)
        nets[edits]._tome_info["size"] = (SIZE, SIZE)
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn((K * n, SIZE * SIZE, 320), generator=g, device="cuda").half()

    def stage(edits, rows):
        blk = nets[edits].blocks[0]
        blk.generator = torch.Generator(device="cuda").manual_seed(11)
        return patch._self_attention_stage(blk, rows, None, None, None, None, None)[0]
    for k in range(K):
        single = stage(1, x[k * n:(k + 1) * n])
        other = torch.randn_like(x, dtype=torch.float32).half() * 3
        other[k * n:(k + 1) * n] = x[k * n:(k + 1) * n]
        for rows in (x, other):
            got = stage(K, rows)[k * n:(k + 1) * n]
            assert torch.isfinite(got).all(), k
            assert torch.equal(got, single), k


def test_per_edit_plans_match_the_oracle_on_each_edit_alone():
    """compute_merge on a batch of K edits (exact-arithmetic tokens, a different video per edit): edit k's merged
    tokens and unmerge equal, bit for bit, the numpy oracle's compute_merge run on edit k's rows alone with the same
    draws, and every edit was given the first edit's draws."""
    from types import SimpleNamespace
    import vidtome_oracle as O
    from test_gpu_parity import _exact_video_fast
    from vidtome_b200 import patch
    K, B, F, T, C = 2, 2, 8, 256, 320
    rng = np.random.default_rng(7)
    videos = [_exact_video_fast(rng, B, F, T, C).reshape(B * F, T, C) for _ in range(K)]
    info = {"size": (16, 16), "hooks": [], "args": dict(max_downsample=2, generator=None, seed=123, batch_size=B,
            align_batch=False, merge_global=False, global_merge_ratio=0.8, local_merge_ratio=0.9, global_rand=0.5,
            target_stride=4, edits=K)}
    module = SimpleNamespace(generator=torch.Generator(device="cuda").manual_seed(3), global_tokens=None)
    m, u, merged = patch.compute_merge(module, torch.from_numpy(np.concatenate(videos)).cuda(), info)
    plans = m.plans
    assert len(plans) == K and all(p.randf == plans[0].randf for p in plans) and plans[0].randf
    out = u(merged).cpu().numpy()
    for k, (video, plan) in enumerate(zip(videos, plans)):
        draws = list(plan.randf)
        res = O.compute_merge(video, (16, 16), batch_size=B, local_merge_ratio=0.9, draw_randf=lambda s: draws.pop(0))
        assert not draws
        np.testing.assert_array_equal(plan.merged_tokens.cpu().numpy(), res.merged_tokens)
        np.testing.assert_array_equal(out[k * B * F:(k + 1) * B * F], res.unmerge(res.merged_tokens))
