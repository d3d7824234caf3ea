"""PnP's conv-feature injection on the GPU: the residual-tail kernel (KT) against torch's tail bit for bit, the library
ResNet path against the reference's forward in torch ops at SD1.5's up_blocks[1].resnets[1] shape and against the
fixture of the reference's conv_forward, and ChunkedDenoiser(pnp_f_t=...) eager and from every graph mode across the
three injection phases."""
import os

import numpy as np
import pytest
import torch

from vidtome_b200 import ops, pnp

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pnp_conv_forward.npz")


# --------------------------------------------------------------------------- 1. the tail kernel
def _torch_tail(h, shortcut, n, num_inputs, osf, inject):
    """utils/pnp_utils.py:146-162 on the GPU."""
    h = h.clone()
    if inject:
        h[n:2 * n] = h[:n]
        if num_inputs > 2:
            h[2 * n:3 * n] = h[:n]
    return (shortcut + h) / osf


def _view(buf, off, shape):
    """A contiguous tensor of `shape` starting `off` elements into `buf` (to move it off a 16-byte boundary)."""
    numel = int(np.prod(shape))
    return buf[off:off + numel].view(shape)


def _check(n, num_inputs, E, osf, inject, offs=(0, 0, 0), g=None):
    B = n * num_inputs
    shape = (B, E)
    bufs = [torch.empty(B * E + 8, dtype=torch.float16, device="cuda") for _ in range(3)]
    h, s, out = (_view(b, o, shape) for b, o in zip(bufs, offs))
    h.copy_(torch.randn(shape, generator=g, device="cuda") * 3)
    s.copy_(torch.randn(shape, generator=g, device="cuda") * 3)
    if E > 4:                                     # values whose sum leaves fp16's range
        h[:, 1] = 60000.0
        s[:, 1] = 20000.0
        h[:, 2] = -60000.0
        s[:, 2] = -30000.0
    want = _torch_tail(h, s, n, num_inputs, osf, inject)
    outs = [out]
    if inject:                                    # h holding only the source samples
        outs.append(torch.empty_like(out))
    for o in outs:
        o.fill_(float("nan"))
    ops.resnet_tail(h, s, num_inputs, osf, inject, out=out)
    if inject:
        ops.resnet_tail(h[:n].contiguous(), s, num_inputs, osf, inject, out=outs[1])
    torch.cuda.synchronize()
    for o in outs:
        same = (o.view(torch.int16) == want.view(torch.int16)) | (o.isnan() & want.isnan())
        assert bool(same.all()), (n, num_inputs, E, osf, inject, offs, int((~same).sum()))
        assert not o.isnan().any() or want.isnan().any()


def test_torch_divides_by_multiplying_with_the_fp32_reciprocal():
    """KT copies torch's rounding of `half / python float`: a multiplication by the fp32 reciprocal of the divisor."""
    g = torch.Generator(device="cuda").manual_seed(1)
    x = (torch.randn(1 << 20, generator=g, device="cuda") * 100).half()
    for osf in (1.0, 2.0, 2.0 ** -0.5, 3.0, 0.3):
        inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(osf, dtype=torch.float32)
        by_mul = (x.float() * inv.item()).half()
        assert torch.equal((x / osf).view(torch.int16), by_mul.view(torch.int16)), osf


@pytest.mark.parametrize("num_inputs", [2, 3])
@pytest.mark.parametrize("inject", [False, True])
def test_tail_kernel_is_bit_identical_to_torch(num_inputs, inject):
    g = torch.Generator(device="cuda").manual_seed(10 * num_inputs + inject)
    elems = [1, 2, 3, 5, 7, 8, 9, 15, 16, 17, 23, 24, 25, 63, 64, 65, 255, 256, 257, 1000, 1001, 4097]
    for n in (1, 2, 3, 4, 5, 7, 8, 16):
        for E in elems:
            for osf in (1.0, 2.0, 2.0 ** -0.5):
                _check(n, num_inputs, E, osf, inject, g=g)
    # SD1.5's up_blocks[1] at 512x512 (1280 x 16 x 16) and a large odd sample
    for n in (1, 4, 16):
        for E in (1280 * 16 * 16, 1280 * 16 * 16 + 3):
            _check(n, num_inputs, E, 2.0 ** -0.5 if n == 4 else 1.0, inject, g=g)


@pytest.mark.parametrize("inject", [False, True])
def test_tail_kernel_off_the_16_byte_boundary(inject):
    g = torch.Generator(device="cuda").manual_seed(3 + inject)
    for offs in [(1, 1, 1), (3, 3, 3), (7, 7, 7), (0, 1, 0), (1, 0, 0), (0, 0, 5), (2, 6, 4), (4, 4, 0)]:
        for n, E in ((1, 9), (2, 64), (3, 17), (4, 1000), (5, 8), (16, 1281)):
            for num_inputs in (2, 3):
                _check(n, num_inputs, E, 2.0, inject, offs=offs, g=g)


def test_tail_kernel_refuses_bad_arguments_on_the_device():
    s = torch.zeros(6, 8, dtype=torch.float16, device="cuda")
    with pytest.raises(RuntimeError, match="num_inputs"):
        ops.resnet_tail(s, s, 4, 1.0, False)
    with pytest.raises(RuntimeError, match="does not fit"):
        ops.resnet_tail(s[:2], s, 3, 1.0, False)                  # h holds the source samples only while injecting
    with pytest.raises(RuntimeError, match="code -6"):
        ops.resnet_tail(s, s, 3, 0.0, False)


# --------------------------------------------------------------------------- 2. the ResNet
def _sd15_resnet(seed=0):
    from vidtome_b200.skeleton import ResnetBlock2D
    torch.manual_seed(seed)
    return ResnetBlock2D(2560, 1280, temb_channels=1280).to(device="cuda", dtype=torch.float16).eval()


def _inputs(B, seed=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((B, 2560, 16, 16), generator=g, device="cuda").half()
    temb = torch.randn((B, 1280), generator=g, device="cuda").half()
    return x, temb


@torch.no_grad()
def test_source_branch_on_the_source_third_matches_the_full_batch():
    """The library path runs norm1 ... conv2 on the n source samples only while injecting; GroupNorm is per sample, so
    only the convolutions' algorithm choice for batch n against batch 3n could change the source rows."""
    resnet = _sd15_resnet()
    for n in (1, 4, 16):
        x, _ = _inputs(3 * n, seed=n)
        full = resnet.conv2(resnet.nonlinearity(resnet.norm2(resnet.conv1(resnet.nonlinearity(resnet.norm1(x))))))
        src = x[:n]
        third = resnet.conv2(resnet.nonlinearity(resnet.norm2(resnet.conv1(resnet.nonlinearity(resnet.norm1(src))))))
        diff = (full[:n].float() - third.float()).abs().max().item()
        print(f"n={n}: source branch on batch {n} vs {3 * n}: max |diff| = {diff}, bit-identical: "
              f"{torch.equal(full[:n], third)}")
        torch.testing.assert_close(third, full[:n], rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("num_inputs", [2, 3])
@torch.no_grad()
def test_library_resnet_against_the_torch_forward_at_sd15_shape(num_inputs):
    resnet = _sd15_resnet()
    n = 4
    x, temb = _inputs(num_inputs * n)
    pnp.register_conv_control(None, [981], num_inputs, modules=[resnet])
    calls = []
    inner = ops.resnet_tail

    def counting(*a, **k):
        calls.append((a[2], a[4]))                    # (num_inputs, inject)
        return inner(*a, **k)
    for t, inject in ((961, False), (981, True), (1000, True)):
        pnp.register_time(None, t, modules=[resnet])
        assert pnp.conv_eligible(resnet, x, temb)
        want = pnp._conv_torch_forward(resnet, num_inputs, x, temb)
        ops.resnet_tail = counting
        try:
            got = resnet(x, temb)
        finally:
            ops.resnet_tail = inner
        assert calls[-1] == (num_inputs, inject)
        if not inject:
            assert torch.equal(got, want)
        else:
            diff = (got.float() - want.float()).abs().max().item()
            print(f"num_inputs={num_inputs} t={t}: library vs torch forward, injected: max |diff| = {diff}, "
                  f"bit-identical: {torch.equal(got, want)}")
            torch.testing.assert_close(got, want, rtol=2e-3, atol=4e-3)
    assert len(calls) == 3


@pytest.mark.parametrize("name", ["b3_inject", "b3_plain", "b2_inject", "b2_plain", "b3_t1000", "b3_none"])
@torch.no_grad()
def test_library_resnet_against_the_reference_fixture(name):
    from test_pnp_conv_cpu import _fixture_resnet
    g = np.load(GOLD)
    resnet = _fixture_resnet(g, name).to(device="cuda", dtype=torch.float16)
    sched = None if bool(g[f"{name}.sched_none"]) else [int(v) for v in g[f"{name}.sched"]]
    pnp.register_conv_control(None, sched, int(g[f"{name}.num_inputs"]), modules=[resnet])
    pnp.register_time(None, int(g[f"{name}.t"]), modules=[resnet])
    x = torch.from_numpy(g[f"{name}.x"]).to("cuda", torch.float16)
    temb = torch.from_numpy(g[f"{name}.temb"]).to("cuda", torch.float16)
    assert pnp.conv_eligible(resnet, x, temb)
    before = ops.STATS.launches
    y = resnet(x, temb)
    assert ops.STATS.launches == before + 1                            # one KT launch
    want = torch.from_numpy(g[f"{name}.out"])
    torch.testing.assert_close(y.float().cpu(), want, rtol=1e-2, atol=2e-2)


# --------------------------------------------------------------------------- 3. the driver
STEPS = 8              # pnp_attn_t 0.25, pnp_f_t 0.75: steps 0-1 both injections, 2-5 conv only, 6-7 neither


def _run(mode, pnp_f_t=0.75, frames=8, size=16):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton, pnp_attention_modules, pnp_conv_module
    torch.manual_seed(77)
    net = make_skeleton("sd15", device="cuda", pnp_conv=True)
    merge_global = mode not in ("step_graph", "eager_plain")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=merge_global, global_merge_ratio=0.8,
                             global_rand=0.5, batch_size=3, align_batch=True)
    g = torch.Generator(device="cuda").manual_seed(5)
    cond = torch.randn((3, 77, 768), generator=g, device="cuda").half()
    sources = {}

    def source(t):
        if t not in sources:
            gs = torch.Generator(device="cuda").manual_seed(int(t))
            sources[t] = torch.randn((frames, 4, size, size), generator=gs, device="cuda").half()
        return sources[t]
    graph = not mode.startswith("eager")
    kw = dict(cuda_graph=graph, graph_warmup=1)
    if mode in ("chunk_graphs", "eager_random"):
        kw.update(randomize_chunks=True, chunk_graphs=graph)
    if mode in ("capture_global", "eager_global"):
        kw.update(capture_global=graph)
    den = ChunkedDenoiser(net, n_timesteps=STEPS, chunk_size=4, merge_global=merge_global, chunk_ord="mix-4",
                          cond=cond, source_latents=source, pnp_attn_t=0.25, pnp_modules=pnp_attention_modules(net),
                          pnp_f_t=pnp_f_t, pnp_conv_modules=None if pnp_f_t is None else [pnp_conv_module(net)], **kw)
    x = torch.randn((frames, 4, size, size), generator=g, device="cuda", dtype=torch.float16)
    torch.manual_seed(2024)
    np.random.seed(2024)
    xs, keys = [], []
    for i in range(STEPS):
        x = den.step(x, i)
        xs.append(x.clone())
        keys.append(sorted(den._chunk_graphs) if mode == "chunk_graphs" else
                    (den._graph.key if graph and den._graph is not None else None))
    torch.cuda.synchronize()
    return xs, keys, den


@pytest.mark.parametrize("mode,eager_mode", [("step_graph", "eager_plain"), ("capture_global", "eager_global"),
                                             ("chunk_graphs", "eager_random")])
def test_driver_graph_modes_are_bit_identical_to_eager_over_the_three_phases(mode, eager_mode):
    calls = []
    inner = ops.resnet_tail

    def counting(*a, **k):
        calls.append(bool(a[4]))
        return inner(*a, **k)
    ops.resnet_tail = counting
    try:
        eager, _, den_e = _run(eager_mode)
    finally:
        ops.resnet_tail = inner
    assert den_e.pnp_schedule == den_e.timesteps[:2] and den_e.pnp_conv_schedule == den_e.timesteps[:6]
    assert calls and any(calls) and not all(calls), "the library ResNet path did not run in both states"
    graph, keys, den = _run(mode)
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(b).all(), i
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"
    if mode == "chunk_graphs":
        assert any(k[3] and k[4] for k in keys[1]), "no doubly injected chunk graph was captured"
        assert keys[2] and not any(k[3] for k in keys[2]), "attention-injected chunk graphs outlived their schedule"
        assert any(k[4] for k in keys[5]), "no conv-injected chunk graph was captured"
        assert keys[-1] and not any(k[3] or k[4] for k in keys[-1]), "injected chunk graphs outlived the schedule"
    else:
        assert [k[1:] for k in keys[1:]] == [(i < 2, i < 6) for i in range(1, STEPS)], keys


def test_conv_injection_changes_the_latents():
    with_conv, _, _ = _run("eager_plain")
    without, _, den = _run("eager_plain", pnp_f_t=None)
    assert den._graph_key(with_conv[0], den.timesteps[0]) == (tuple(with_conv[0].shape), True)
    assert not torch.equal(with_conv[0], without[0])
