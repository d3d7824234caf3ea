"""KS (vtm_cfg_ddim_update_f16), the sampling step's guidance combine and DDIM update in one kernel, on an H100:
  1. bit for bit against the torch ops it replaces (pred_noise's combine, then pred_next_x), NaN and inf included,
     for 2 and 3 samples, several guidance scales, every step of a 50-step table and an out-of-range step;
  2. every n up to a few vectors and odd element offsets, in place and out of place;
  3. guard bands (the harness of test_gpu_bounds.py);
  4. ChunkedDenoiser with driver.FUSE_STEP_UPDATE on against off, in every stepping mode and control: bit-identical
     latents, and a returned tensor that no later step changes;
  5. a replayed cuda_graph step launches nothing but fills outside the graph."""
import numpy as np
import pytest
import torch

import test_gpu_bounds as tb
from vidtome_b200 import driver, ops
from vidtome_b200.driver import ChunkedDenoiser

pytestmark = pytest.mark.gpu

GUIDANCE = [7.5, 1.0, 0.0, -2.0, 7.3]                  # 7.3 is not exact in fp32
SPECIAL = [65504.0, -65504.0, 6e-8, -6e-8, 3e-5, -1e-6, 0.0, -0.0, float("inf"), float("-inf"), float("nan")]


@pytest.fixture
def fuse():
    saved = driver.FUSE_STEP_UPDATE
    yield
    driver.FUSE_STEP_UPDATE = saved


def _halves(n, g, scale=2.0, special=0.05):
    """n fp16 values: normal * scale, with a fraction of adversarial values (±max, subnormals, ±0, ±inf, NaN)."""
    v = torch.randn(n, generator=g, device="cuda") * scale
    pick = torch.rand(n, generator=g, device="cuda") < special
    sp = torch.tensor(SPECIAL, device="cuda")[torch.randint(len(SPECIAL), (n,), generator=g, device="cuda")]
    return torch.where(pick, sp, v).half()


def _bits(t):
    return t.view(torch.int16)


def _want(den, x, eps, samples, guidance, i):
    u, c = eps.chunk(samples)[-2:]
    return den.pred_next_x(x, u + guidance * (c - u), i)


# --------------------------------------------------------------------------- 1. against the torch ops
@pytest.mark.parametrize("samples", [2, 3])
@pytest.mark.parametrize("guidance", GUIDANCE)
def test_matches_torch_ops_at_every_step(samples, guidance):
    den = ChunkedDenoiser(torch.nn.Identity(), n_timesteps=50)
    coef, step = den.step_tables("cuda")
    g = torch.Generator(device="cuda").manual_seed(samples * 100 + int(guidance * 10))
    n = 4 * 4 * 64 * 64 + 5
    x = _halves(n, g)
    eps = _halves(samples * n, g, scale=1.0)
    eps[(samples - 1) * n:(samples - 1) * n + 64] = 65504.0              # c - u overflows to inf against u = -65504
    eps[(samples - 2) * n:(samples - 2) * n + 64] = -65504.0
    out = torch.empty_like(x)
    for i in range(50):
        step.fill_(i)
        ops.cfg_ddim_update(x, eps, samples, guidance, coef, step, out)
        want = _want(den, x, eps, samples, guidance, i)
        assert torch.equal(_bits(out), _bits(want)), (i, int((_bits(out) != _bits(want)).sum()))
    assert torch.isnan(out).any() and torch.isinf(out).any()
    for s in (-1, 50):                                                   # out of range: nothing is written
        out.fill_(1.0)
        step.fill_(s)
        ops.cfg_ddim_update(x, eps, samples, guidance, coef, step, out)
        assert bool((out == 1.0).all()), s


# --------------------------------------------------------------------------- 2. lengths, offsets, in place
@pytest.mark.parametrize("inplace", [False, True])
def test_lengths_offsets_and_in_place(inplace):
    den = ChunkedDenoiser(torch.nn.Identity(), n_timesteps=50)
    coef, step = den.step_tables("cuda")
    step.fill_(17)
    g = torch.Generator(device="cuda").manual_seed(7 + inplace)
    lengths = list(range(1, 40)) + [8 * 129 + 7, 8 * 4096, 8 * 4096 + 3]
    for n in lengths:
        for off in [(0, 0, 0), (1, 1, 1), (3, 5, 7), (0, 2, 0), (8, 1, 8)]:
            samples = 3 if n % 2 else 2
            ox, oe, oo = off
            xbuf = _halves(n + 16, g)
            ebuf = _halves(samples * n + 16, g, scale=1.0)
            x, eps = xbuf[ox:ox + n], ebuf[oe:oe + samples * n]
            want = _want(den, x, eps, samples, 7.5, 17)
            if inplace:
                before = xbuf.clone()
                ops.cfg_ddim_update(x, eps, samples, 7.5, coef, step, x)
                got = x
                assert torch.equal(_bits(xbuf[:ox]), _bits(before[:ox]))
                assert torch.equal(_bits(xbuf[ox + n:]), _bits(before[ox + n:]))
            else:
                obuf = torch.full((n + 16,), 3.0, device="cuda", dtype=torch.float16)
                got = obuf[oo:oo + n]
                ops.cfg_ddim_update(x, eps, samples, 7.5, coef, step, got)
                assert bool((obuf[:oo] == 3.0).all()) and bool((obuf[oo + n:] == 3.0).all()), (n, off)
            assert torch.equal(_bits(got), _bits(want)), (n, off)


def test_wrapper_shape_and_overlap_checks():
    h = torch.zeros(2, 4, 8, device="cuda", dtype=torch.float16)
    coef, step = torch.zeros(3, 4, device="cuda"), torch.zeros(1, device="cuda", dtype=torch.int32)
    with pytest.raises(RuntimeError, match="samples"):
        ops.cfg_ddim_update(h, h, 2, 7.5, coef, step, h)
    with pytest.raises(RuntimeError, match="out"):
        ops.cfg_ddim_update(h, torch.cat([h, h]), 2, 7.5, coef, step, h[:1])
    buf = torch.zeros(2 * h.numel() + 8, device="cuda", dtype=torch.float16)
    with pytest.raises(RuntimeError, match="code -2"):                   # out partly over x
        ops.cfg_ddim_update(buf[:h.numel()].view_as(h), torch.cat([h, h]), 2, 7.5, coef, step,
                            buf[8:8 + h.numel()].view_as(h))
    eps = torch.zeros(2 * h.numel(), device="cuda", dtype=torch.float16)
    with pytest.raises(RuntimeError, match="code -2"):                   # out over eps
        ops.cfg_ddim_update(h, eps.view(4, 4, 8), 2, 7.5, coef, step, eps[:h.numel()].view_as(h))


# --------------------------------------------------------------------------- 3. guard bands
def _bounds_case(n, samples, step, aligns, inplace):
    g = tb._gen(n + 10 * samples + step)
    x, eps = tb._randn((n,), g), tb._randn((samples * n,), g)
    coef = ChunkedDenoiser(torch.nn.Identity(), n_timesteps=10).step_tables("cuda")[0].clone()
    in_range = 0 <= step < 10
    kept = None if in_range else torch.ones(n, dtype=torch.bool)
    ax, ae, ao = aligns
    bufs = {"x": tb.Buf("inout", x, align=ax, kept=kept) if inplace else tb.Buf("in", x, align=ax),
            "eps": tb.Buf("in", eps, align=ae), "coef": tb.Buf("in", coef),
            "step": tb.Buf("in", torch.tensor([step], dtype=torch.int32, device="cuda"), align=4, poison=0)}
    if not inplace:
        bufs["out"] = tb._out(n, n * 2, rows=1, align=ao, kept=kept)
    o = "x" if inplace else "out"
    return tb.Case("vtm_cfg_ddim_update_f16", bufs,
                   lambda b: [b["x"], b["eps"], n, samples, 7.5, b["coef"], b["step"], 10, b[o], tb._stream()],
                   errors=[(tb.VTM_E_NULL, {8: None}), (tb.VTM_E_NULL, {5: None}), (tb.VTM_E_SHAPE, {3: 4}),
                           (tb.VTM_E_SHAPE, {2: 0})])


# (n, samples, step, (x, eps, out) offsets from a 256-byte boundary, in place)
BOUNDS = [(4096 + 5, 2, 0, (16, 16, 16), False), (1001, 3, 3, (2, 4, 6), False), (1, 2, 9, (2, 2, 2), True),
          (777, 3, 10, (16, 18, 16), False), (777, 2, -1, (2, 2, 2), True), (4 * 64 * 64, 3, 4, (18, 18, 18), True),
          (4 * 64 * 64, 2, 5, (16, 16, 16), False)]

# The entry point's cases for test_gpu_bounds.REGISTRY (tests/test_bounds_cpu.py checks that the registry names every
# compute entry point of the C-ABI)
tb.REGISTRY.setdefault("vtm_cfg_ddim_update_f16", []).extend(
    (f"n={n} samples={s} step={st} align={al} inplace={ip}", (lambda a=(n, s, st, al, ip): _bounds_case(*a)))
    for n, s, st, al, ip in BOUNDS)


@pytest.mark.parametrize("n,samples,step,aligns,inplace", BOUNDS)
def test_guard_bands(n, samples, step, aligns, inplace):
    tb.run_case(_bounds_case(n, samples, step, aligns, inplace),
                f"vtm_cfg_ddim_update_f16 n={n} samples={samples} step={step} align={aligns} inplace={inplace}")




# --------------------------------------------------------------------------- 4. the step driver, on against off
STEPS, FRAMES, SIZE = 6, 8, 32
MODES = ["eager", "cuda_graph", "capture_global", "chunk_graphs", "pnp", "controlnet", "depth", "odd_size"]


def _run(mode, fuse):
    """STEPS steps of one configuration with FUSE_STEP_UPDATE = fuse; returns every step's returned tensor together
    with a copy taken when it was returned."""
    import vidtome_b200
    from vidtome_b200.skeleton import make_controlnet, make_skeleton, pnp_attention_modules, pnp_conv_module
    driver.FUSE_STEP_UPDATE = fuse
    torch.manual_seed(77)
    name, frames, size, chunk = "sd21", FRAMES, SIZE, 4
    pnp = mode == "pnp"
    if mode == "odd_size":                  # 3 * 4 * 15 * 15 halves per chunk: n % 8 != 0 and odd chunk offsets
        name, frames, size, chunk = "sd15", 7, 15, 3
        net = make_skeleton(name, hot_path_only=False, max_downsample=1, device="cuda")
    else:
        net = make_skeleton(name, hot_path_only=False, device="cuda", pnp_conv=pnp, depth=mode == "depth")
        vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=mode in ("capture_global", "chunk_graphs"),
                                 global_merge_ratio=0.8, global_rand=0.5, batch_size=3 if pnp else 2, align_batch=True)
    cad = 1024 if name == "sd21" else 768
    g = torch.Generator(device="cuda").manual_seed(5)
    kw = dict(cuda_graph=mode != "eager", graph_warmup=2, chunk_size=chunk,
              cond=torch.randn((3 if pnp else 2, 77, cad), generator=g, device="cuda").half())
    if mode == "capture_global":
        kw.update(merge_global=True, chunk_ord="mix-4", capture_global=True)
    if mode == "chunk_graphs":
        kw.update(merge_global=True, chunk_ord="rand", randomize_chunks=True, chunk_graphs=True, graph_warmup=1)
    if mode == "controlnet":
        cnet = make_controlnet(name, hot_path_only=False, device="cuda")
        images = torch.rand((frames, 3, 8 * size, 8 * size), generator=g, device="cuda").half()
        kw.update(controlnet=cnet, control_images=images, control_scale=0.8)
    if mode == "depth":
        kw.update(depth=torch.rand((frames, 1, size, size), generator=g, device="cuda") * 2 - 1)
    if pnp:
        sources = {}

        def source(t):
            if t not in sources:
                gs = torch.Generator(device="cuda").manual_seed(int(t))
                sources[t] = torch.randn((frames, 4, size, size), generator=gs, device="cuda").half()
            return sources[t]
        kw.update(source_latents=source, pnp_attn_t=0.5, pnp_modules=pnp_attention_modules(net), pnp_f_t=0.8,
                  pnp_conv_modules=[pnp_conv_module(net)])
    den = ChunkedDenoiser(net, n_timesteps=STEPS, **kw)
    x = torch.randn((frames, 4, size, size), generator=g, device="cuda", dtype=torch.float16)
    torch.manual_seed(2024)
    np.random.seed(2024)
    xs = []
    for i in range(STEPS):
        x = den.step(x, i)
        xs.append((x, x.clone()))
    torch.cuda.synchronize()
    den.close()
    return xs


@pytest.mark.parametrize("mode", MODES)
def test_driver_fused_update_is_bit_identical(fuse, mode):
    on = _run(mode, True)
    off = _run(mode, False)
    for i, ((a, a_then), (b, b_then)) in enumerate(zip(on, off)):
        assert torch.isfinite(a).all(), i
        assert torch.equal(a, a_then) and torch.equal(b, b_then), f"step {i}: a later step changed a returned tensor"
        assert torch.equal(_bits(a), _bits(b)), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"


# --------------------------------------------------------------------------- 5. what a replayed step launches
ARITHMETIC = {"aten::mul", "aten::sub", "aten::add", "aten::div", "aten::rsub"}


def _launches(den, x, i):
    """(kernel launches, graph launches, aten op counts) of one step, from the runtime calls torch.profiler records."""
    from collections import Counter
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        den.step(x, i)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    return (sum(n.startswith("cudaLaunchKernel") for n in names), names.count("cudaGraphLaunch"),
            Counter(n for n in names if n.startswith("aten::")))


def test_replayed_step_launches_only_fills(fuse):
    """Outside the graph a fused replayed step launches fills only: the timestep and step index, and the seed / offset
    fills torch issues for every generator registered with the graph.  The copies in and out are memcpys.  Off, the
    torch update's six half ops follow the replay, and there is no step index to fill."""
    import vidtome_b200
    from vidtome_b200.skeleton import make_skeleton
    torch.manual_seed(3)
    net = make_skeleton("sd15", hot_path_only=True, device="cuda")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, batch_size=2)
    x = torch.randn((16, 4, 64, 64), device="cuda", dtype=torch.float16)
    counts = {}
    for fuse_on in (True, False):
        driver.FUSE_STEP_UPDATE = fuse_on
        den = ChunkedDenoiser(net, n_timesteps=50, chunk_size=16, cuda_graph=True)
        for i in range(4):                                   # 2 eager steps, the capture, a replay
            den.step(x, i)
        counts[fuse_on] = _launches(den, x, 4)
        den.close()
    kernels, graphs, aten = counts[True]
    assert graphs == 1
    assert kernels == aten["aten::fill_"] >= 2, counts[True]
    assert not set(aten) & ARITHMETIC, aten
    kernels_off, graphs_off, aten_off = counts[False]
    assert graphs_off == 1 and aten_off["aten::fill_"] == aten["aten::fill_"] - 1, counts[False]
    assert kernels_off == aten_off["aten::fill_"] + 6, counts[False]
    assert {"aten::mul", "aten::sub", "aten::add", "aten::div"} <= set(aten_off), aten_off
