"""DDIM inversion on the GPU: KI (`vtm_ddim_update_f16`) against torch's CUDA half ops, KD with the residual
(`vtm_attention_residual`) against KD + torch's add and against float64, and driver.ChunkedInverter on a patched
full-block SD1.5 skeleton: against an unpatched twin, from CUDA graphs against eager stepping (with and without a
patched ControlNet), and without side effects on a later PnP generation with global merging.  Needs an H100 (sm_90a)."""
import numpy as np
import pytest
import torch

from vidtome_b200 import ops

pytestmark = pytest.mark.gpu


# --------------------------------------------------------------------------- 1. KI
def _tables(inv, device="cuda"):
    coef = ops.ddim_table(inv.coefficients(i) for i in range(len(inv.timesteps))).to(device)
    return coef, torch.tensor(inv.slots, dtype=torch.int32, device=device)


@pytest.mark.parametrize("n,offsets", [(1, (0, 0, 0)), (7, (0, 0, 0)), (13, (1, 3, 5)), (4096, (0, 0, 0)),
                                       (4096, (2, 2, 2)), (4096, (0, 1, 0)), (4 * 64 * 64 * 32 + 5, (3, 3, 3)),
                                       (4 * 64 * 64 * 32, (0, 0, 7))])
def test_ddim_kernel_is_bit_identical_to_torch_for_all_50_steps(n, offsets):
    """x, eps and the trajectory at `offsets` elements past a 16-byte boundary; n not a multiple of 8 included."""
    from vidtome_b200.driver import ChunkedInverter
    from vidtome_b200.skeleton import make_skeleton
    inv = ChunkedInverter(make_skeleton("tiny", device="cpu", dtype=torch.float32), n_timesteps=50, save_steps=10)
    coef, slots = _tables(inv)
    g = torch.Generator(device="cuda").manual_seed(n)
    ox, oe, ot = offsets
    xbuf = torch.empty(n + 8, dtype=torch.float16, device="cuda")
    x = xbuf[ox:ox + n]
    x.copy_(torch.randn(n, generator=g, device="cuda"))
    ebuf = torch.empty(n + 8, dtype=torch.float16, device="cuda")
    n_slots = len(inv.saved_timesteps)
    tbuf = torch.full((n_slots * n + 8,), float("nan"), dtype=torch.float16, device="cuda")
    traj = tbuf[ot:ot + n_slots * n].view(n_slots, n)
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    want = x.clone()
    for i in range(50):
        eps = ebuf[oe:oe + n]
        eps.copy_(torch.randn(n, generator=g, device="cuda"))
        want = inv.pred_next_x(want, eps, i)                         # torch's CUDA half ops
        ops.ddim_update(x, eps, coef, step, slots, traj)
        step.add_(1)
        assert torch.equal(x, want), f"step {i}: max |diff| {(x.float() - want.float()).abs().max().item()}"
        if inv.slots[i] >= 0:
            assert torch.equal(traj[inv.slots[i]], want), i
    assert torch.isfinite(traj).all()                                 # every slot was written
    # a step past the table leaves x alone, and without a slot table nothing else is written
    before = x.clone()
    ops.ddim_update(x, eps, coef, step)
    assert torch.equal(x, before)


def test_ddim_kernel_sampling_coefficients_match_the_generation_update():
    """The same kernel with the sampling coefficients (a, b, c, d) = (sigma, mu, mu_prev, sigma_prev) gives
    ChunkedDenoiser.pred_next_x bit for bit."""
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton
    den = ChunkedDenoiser(make_skeleton("tiny", device="cpu", dtype=torch.float32), n_timesteps=50)
    rows = []
    for i, t in enumerate(den.timesteps):
        ap = den.alphas_cumprod[t]
        pp = den.alphas_cumprod[den.timesteps[i + 1]] if i < 49 else den.final_alpha_cumprod
        rows.append((float((1 - ap) ** 0.5), float(ap ** 0.5), float(pp ** 0.5), float((1 - pp) ** 0.5)))
    coef = ops.ddim_table(rows).cuda()
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn(3, 4, 9, 9, generator=g, device="cuda").half()
    want = x.clone()
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    for i in range(50):
        eps = torch.randn(3, 4, 9, 9, generator=g, device="cuda").half()
        want = den.pred_next_x(want, eps, i)
        ops.ddim_update(x, eps, coef, step)
        step.add_(1)
        assert torch.equal(x, want), i


# --------------------------------------------------------------------------- 2. KD with the residual
# (B, L, C, heads): SD1.5 ds1 / ds2 per-frame self-attention of 8 frames, SD2.1's 5 / 10 / 20 heads of 64, SD1.5 ds4 /
# ds8 at head_dim 160
SHAPES = [(8, 4096, 320, 8), (8, 1024, 640, 8), (8, 4096, 320, 5), (8, 1024, 640, 10), (8, 256, 1280, 20),
          (8, 256, 1280, 8), (8, 64, 1280, 8)]


def _lora(R, K, N, g):
    return ((torch.randn(R, K, generator=g, device="cuda") * 0.05).half(),
            (torch.randn(N, R, generator=g, device="cuda") * 0.05).half())


@pytest.mark.parametrize("lora", [False, True])
@pytest.mark.parametrize("B,L,C,H", SHAPES)
def test_attention_residual_is_kd_plus_torch_add(B, L, C, H, lora):
    g = torch.Generator(device="cuda").manual_seed(L + C + H)
    x = torch.randn(B, L, C, generator=g, device="cuda").half()
    resid = (torch.randn(B, L, C, generator=g, device="cuda") * 4).half()
    w_qkv = (torch.randn(3 * C, C, generator=g, device="cuda") * C ** -0.5).half()
    w_o = (torch.randn(C, C, generator=g, device="cuda") * C ** -0.5).half()
    b_o = (torch.randn(C, generator=g, device="cuda") * 0.1).half()
    kw = dict(lora_qkv=_lora(16, C, 3 * C, g), lora_o=_lora(8, C, C, g)) if lora else {}
    scale = (C // H) ** -0.5
    want = ops.attention(x, w_qkv, w_o, b_o, H, scale, **kw) + resid
    got = ops.attention_residual(x, w_qkv, w_o, b_o, H, scale, resid, **kw)
    assert torch.isfinite(got).all()
    assert torch.equal(got, want), f"max |diff| {(got.float() - want.float()).abs().max().item()}"


@pytest.mark.parametrize("name", ["random", "negative"])
@pytest.mark.parametrize("B,L,C,H", [s for s in SHAPES if s[2] // s[3] <= 128])
def test_attention_residual_against_float64(B, L, C, H, name):
    """The exact-arithmetic designs and per-element bound of test_gpu_attention_core (W_o = I, no bias) with a zero
    residual, so y = fp16(o) is held to the same bound."""
    from test_gpu_attention_core import _assert_within, _reference, _self_design, _self_qkv
    g = torch.Generator(device="cuda").manual_seed(B * L + C)
    x, w, scale = _self_design(name, B, L, C, H, g)
    q, k, v = _self_qkv(x, w, H)
    O, bound = _reference(q, k, v, scale)
    eye = torch.eye(C, dtype=torch.float16, device="cuda")
    y = ops.attention_residual(x, w, eye, None, H, scale, torch.zeros_like(x))
    torch.cuda.synchronize()
    _assert_within(y, O, bound, f"attention_residual {name} B={B} L={L} C={C} H={H}")


# --------------------------------------------------------------------------- 3. the inverter
FRAMES, SIZE = 11, 32


def _inputs(frames=FRAMES, size=SIZE, seed=3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(frames, 4, size, size, generator=g, device="cuda").half()
    cond = torch.randn(frames, 77, 768, generator=g, device="cuda").half()
    images = torch.rand(frames, 3, 8 * size, 8 * size, generator=g, device="cuda").half()
    return x, cond, images


def _patched(pnp_conv=False, batch_size=2, **kw):
    import vidtome_b200
    from vidtome_b200.skeleton import make_skeleton
    net = make_skeleton("sd15", hot_path_only=False, device="cuda", pnp_conv=pnp_conv)
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, batch_size=batch_size, **kw)
    return net


def test_one_step_noise_prediction_matches_an_unpatched_twin():
    from vidtome_b200 import attention, patch
    from vidtome_b200.driver import ChunkedInverter
    from vidtome_b200.skeleton import make_skeleton
    x, cond, _ = _inputs(frames=8)
    plain = make_skeleton("sd15", hot_path_only=False, device="cuda")
    net = _patched()
    calls = []
    inner = attention.self_attention_residual

    def counting(*a, **k):
        calls.append(a[1].shape)
        return inner(*a, **k)
    attention.self_attention_residual = counting
    try:
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            want = ChunkedInverter(plain, cond=cond).pred_noise(x, cond, 1)
            with patch._unmerged_blocks():
                got = ChunkedInverter(net, cond=cond).pred_noise(x, cond, 1)
    finally:
        attention.self_attention_residual = inner
    # every block with head_dim <= MAX_HEAD_DIM (SD1.5: the 10 blocks of 320 and 640 channels) ran KD-residual
    assert len(calls) == 10 and {s[1] for s in calls} == {SIZE * SIZE, SIZE * SIZE // 4}
    assert torch.isfinite(got).all()
    err = (got.float() - want.float()).abs().max().item()
    assert err <= 1e-2 * want.float().abs().max().item() + 1e-2, err


@pytest.mark.parametrize("control", [False, True])
def test_graph_trajectory_is_bit_identical_to_eager(control):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedInverter
    from vidtome_b200.skeleton import make_controlnet
    x, cond, images = _inputs()
    net = _patched()
    controlnet = None
    if control:
        controlnet = make_controlnet("sd15", hot_path_only=False, device="cuda")
        vidtome_b200.apply_patch(controlnet, local_merge_ratio=0.9, batch_size=2)
    kw = dict(n_timesteps=50, batch_size=4, cond=cond, controlnet=controlnet,
              control_images=images if control else None, control_scale=0.8)
    eager = ChunkedInverter(net, **kw)
    eager.invert(x)
    graph = ChunkedInverter(net, cuda_graph=True, graph_warmup=2, **kw)
    final = graph.invert(x)
    assert len(eager.saved_timesteps) == 50
    assert torch.isfinite(graph.trajectory).all()
    for k, t in enumerate(eager.saved_timesteps):
        a, b = eager.trajectory[k], graph.trajectory[k]
        assert torch.equal(a, b), f"t={t}: max |diff| {(a.float() - b.float()).abs().max().item()}"
    assert torch.equal(final, graph.trajectory[-1])
    assert not torch.equal(eager.trajectory[0], x)


def _snapshot(net):
    gens = {n: m.generator.get_state().clone() for n, m in net.named_modules() if hasattr(m, "generator")}
    toks = {n: m.global_tokens for n, m in net.named_modules() if hasattr(m, "global_tokens")}
    ts = {n: getattr(m, "t", None) for n, m in net.named_modules()
          if hasattr(m, "_vtm_pnp") or hasattr(m, "_vtm_pnp_conv")}
    return gens, toks, ts


def _generate(net, source, cond3, steps):
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import pnp_attention_modules, pnp_conv_module
    den = ChunkedDenoiser(net, n_timesteps=steps, chunk_size=4, merge_global=True, chunk_ord="mix-4", cond=cond3,
                          source_latents=source, pnp_attn_t=0.5, pnp_modules=pnp_attention_modules(net), pnp_f_t=0.8,
                          pnp_conv_modules=[pnp_conv_module(net)])
    return den


def test_inversion_has_no_side_effects_on_pnp_generation():
    from vidtome_b200.driver import ChunkedInverter
    steps, frames = 10, 8
    x0, cond, _ = _inputs(frames=frames, size=16, seed=5)
    g = torch.Generator(device="cuda").manual_seed(6)
    cond3 = torch.randn(3, 77, 768, generator=g, device="cuda").half()
    noise = torch.randn(frames, 4, 16, 16, generator=g, device="cuda").half()
    nets = [_patched(pnp_conv=True, batch_size=3, align_batch=True, merge_global=True) for _ in range(2)]
    holder = {}
    dens = [_generate(n, lambda t: holder["f"](t), cond3, steps) for n in nets]
    for net in nets:                                 # the blocks fork their generators and hold global tokens
        torch.cuda.manual_seed(17)
        with torch.no_grad():
            net(torch.zeros(3 * 4, 4, 16, 16, device="cuda", dtype=torch.float16), 981,
                encoder_hidden_states=cond3.repeat_interleave(4, 0))
    from vidtome_b200 import pnp
    pnp.register_time(nets[0], 981)
    pnp.register_time(nets[1], 981)
    before = _snapshot(nets[0])
    assert before[0] and before[1] and all(t == 981 for t in before[2].values())
    rng = torch.cuda.get_rng_state()
    inv = ChunkedInverter(nets[0], n_timesteps=steps, batch_size=3, cond=cond[:1])
    inv.invert(x0)
    assert torch.equal(torch.cuda.get_rng_state(), rng)
    after = _snapshot(nets[0])
    assert before[0].keys() == after[0].keys() and all(torch.equal(before[0][k], after[0][k]) for k in before[0])
    assert before[1].keys() == after[1].keys() and all(before[1][k] is after[1][k] for k in before[1])
    assert before[2] == after[2]
    # the same generation on the inverted model and on its twin, which never inverted, given the same trajectory
    traj = inv.trajectory.clone()
    holder["f"] = lambda t: traj[inv.saved_timesteps.index(int(t))]
    outs = []
    for den in dens:
        torch.manual_seed(2024)
        np.random.seed(2024)
        x = noise.clone()
        for i in range(steps):
            x = den.step(x, i)
        outs.append(x)
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0], outs[1]), f"max |diff| {(outs[0].float() - outs[1].float()).abs().max().item()}"
