"""PnP's conv-feature injection, host side: pnp.register_conv_control's torch forward against the reference's own
conv_forward (tests/golden/pnp_conv_forward.npz), the conv schedules against the reference's init_pnp
(tests/golden/pnp_conv_schedules.npz; both written by tests/make_golden_pnp_conv.py), the targets, the marker and every
case that keeps a call off the library path, the driver's graph keys over the three injection phases, and the library
entry point's argument checks, which return before any CUDA call."""
import ctypes
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from test_pnp_driver_cpu import StandInUNet

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _fixture_resnet(g, name):
    from vidtome_b200.skeleton import ResnetBlock2D
    w = {k[len(name) + 3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith(f"{name}.w.")}
    cin, cout = w["conv1.weight"].shape[1], w["conv1.weight"].shape[0]
    resnet = ResnetBlock2D(cin, cout, temb_channels=w["time_emb_proj.weight"].shape[1],
                           groups=int(g[f"{name}.groups"]), output_scale_factor=float(g[f"{name}.osf"]))
    resnet.load_state_dict(w)
    return resnet.eval()


@pytest.mark.parametrize("name", ["b3_inject", "b3_plain", "b2_inject", "b2_plain", "b3_t1000", "b3_none"])
def test_torch_forward_matches_reference_conv_forward(name):
    from vidtome_b200 import pnp
    g = np.load(os.path.join(GOLD, "pnp_conv_forward.npz"))
    resnet = _fixture_resnet(g, name)
    sched = None if bool(g[f"{name}.sched_none"]) else [int(v) for v in g[f"{name}.sched"]]
    pnp.register_conv_control(None, sched, int(g[f"{name}.num_inputs"]), modules=[resnet])
    pnp.register_time(None, int(g[f"{name}.t"]), modules=[resnet])
    x, temb = torch.from_numpy(g[f"{name}.x"]), torch.from_numpy(g[f"{name}.temb"])
    assert pnp.conv_ineligibility(resnet, x, temb) == "device"             # CPU: the torch forward
    with torch.no_grad():
        y = resnet(x, temb)
    np.testing.assert_allclose(y.numpy(), g[f"{name}.out"], rtol=1e-5, atol=1e-5)
    inject = name.endswith(("inject", "t1000"))
    assert pnp.injection_active(resnet) == inject
    # with injection the residual branch of every sample is the source's: out * osf - shortcut is periodic in n
    ni = int(g[f"{name}.num_inputs"])
    n = x.shape[0] // ni
    with torch.no_grad():
        branch = y.double() * float(g[f"{name}.osf"]) - resnet.conv_shortcut(x).double()
    same = torch.allclose(branch[n:2 * n], branch[:n], atol=1e-4)
    assert same == inject


def test_conv_schedule_matches_reference_init_pnp():
    from vidtome_b200.skeleton import ResnetBlock2D
    from vidtome_b200.driver import ChunkedDenoiser
    g = np.load(os.path.join(GOLD, "pnp_conv_schedules.npz"))
    for case in range(int(g["cases"])):
        n, frac = int(g[f"sched{case}_n"]), float(g[f"sched{case}_frac"])
        resnet = ResnetBlock2D(32, 16, temb_channels=8, groups=4)
        den = ChunkedDenoiser(StandInUNet(), n_timesteps=n, cond=torch.randn(3, 77, 16), source_latents=lambda t: None,
                              pnp_modules=[], pnp_f_t=frac, pnp_conv_modules=[resnet])
        assert den.pnp_conv_schedule == [int(v) for v in g[f"sched{case}"]], case
        assert resnet._vtm_pnp_conv == int(g["num_inputs"]) == 3
        assert list(resnet.injection_schedule) == den.pnp_conv_schedule
        for t in den.timesteps:
            assert den.conv_injecting(t) == (t in den.pnp_conv_schedule)


def test_targets_marker_and_register_time():
    from vidtome_b200 import pnp
    from vidtome_b200.skeleton import ResnetBlock2D, make_skeleton, pnp_conv_module
    resnets = [[ResnetBlock2D(32, 16, temb_channels=8, groups=4) for _ in range(3)] for _ in range(4)]
    unet = SimpleNamespace(up_blocks=[SimpleNamespace(resnets=r) for r in resnets])
    model = SimpleNamespace(unet=unet)
    assert pnp._conv_targets(model, None) == [resnets[1][1]]            # utils/pnp_utils.py:169
    pnp.register_conv_control(model, [981, 961], num_inputs=3)
    target = resnets[1][1]
    assert target._vtm_pnp_conv == 3 and target.injection_schedule == [981, 961]
    assert target.forward._vtm_pnp_conv_forward
    assert not any(hasattr(r, "_vtm_pnp_conv") for row in resnets for r in row if r is not target)
    # register_time reaches the marked ResNets as well as the attention modules (utils/pnp_utils.py:23-24)
    net = make_skeleton("sd15", device="cpu", dtype=torch.float32, pnp_conv=True)
    pnp.register_conv_control(net, [981], num_inputs=3, modules=[pnp_conv_module(net)])
    pnp.register_attention_control(net, [981], num_inputs=3, modules=[net.blocks[8].attn1])
    pnp.register_time(net, 981)
    assert net.resnet.t == 981 and net.blocks[8].attn1.t == 981
    assert pnp.injection_active(net.resnet)
    pnp.register_time(net, 1000)                                         # the t == 1000 clause
    assert pnp.injection_active(net.resnet)
    pnp.register_time(net, 961)
    assert not pnp.injection_active(net.resnet)


def test_every_fallback_case():
    from vidtome_b200 import pnp
    from vidtome_b200.skeleton import ResnetBlock2D

    def fresh(num_inputs=3):
        r = ResnetBlock2D(32, 16, temb_channels=8, groups=4)
        pnp.register_conv_control(None, [981], num_inputs, modules=[r])
        return r.eval()
    x, temb = torch.randn(6, 32, 4, 4), torch.randn(6, 8)
    assert pnp.conv_ineligibility(fresh(), x, temb) == "device"        # otherwise eligible: CPU fp32
    assert pnp.conv_ineligibility(fresh(), x.half(), temb.half()) == "device"
    assert pnp.conv_ineligibility(fresh(), x, None) == "device"
    assert pnp.conv_ineligibility(fresh(4), x[:4], temb[:4]) == "num_inputs"
    assert pnp.conv_ineligibility(ResnetBlock2D(32, 16, 8, groups=4), x, temb) == "num_inputs"   # not marked
    assert pnp.conv_ineligibility(fresh(), x[:5], temb[:5]) == "batch"
    assert pnp.conv_ineligibility(fresh(), x[:0], temb[:0]) == "batch"
    assert pnp.conv_ineligibility(fresh(), x.flatten(2), temb) == "batch"
    assert pnp.conv_ineligibility(fresh(), x.to(memory_format=torch.channels_last), temb) == "layout"
    for attr, value, why in (("upsample", torch.nn.Identity(), "resample"), ("downsample", torch.nn.Identity(), "resample"),
                             ("time_embedding_norm", "scale_shift", "time_embedding_norm")):
        r = fresh()
        setattr(r, attr, value)
        assert pnp.conv_ineligibility(r, x, temb) == why
    r = fresh()
    r.dropout = torch.nn.Dropout(0.1).eval()
    assert pnp.conv_ineligibility(r, x, temb) == "device"              # eval mode: inactive
    r.train()
    assert pnp.conv_ineligibility(r, x, temb) == "dropout"
    assert pnp.conv_ineligibility(fresh(), x, temb[:2]) == "temb"
    assert pnp.conv_ineligibility(fresh(), x, temb[:1]) == "device"
    for sub in ("norm1", "conv1", "conv2", "conv_shortcut", "time_emb_proj"):
        r = fresh()
        getattr(r, sub).register_forward_hook(lambda *a: None)
        assert pnp.conv_ineligibility(r, x, temb) == "hooks", sub
        r = fresh()
        getattr(r, sub).register_forward_pre_hook(lambda *a: None)
        assert pnp.conv_ineligibility(r, x, temb) == "hooks", sub
    r = fresh()
    r.register_forward_hook(lambda *a: None)                            # on the ResNet itself: runs around both paths
    assert pnp.conv_ineligibility(r, x, temb) == "device"


def _denoiser(**kw):
    from vidtome_b200.driver import ChunkedDenoiser
    return ChunkedDenoiser(StandInUNet(), cond=torch.randn(3, 77, 16), source_latents=lambda t: None, pnp_modules=[],
                           **kw)


def test_graph_keys_over_the_three_phases():
    from vidtome_b200.skeleton import ResnetBlock2D
    r = ResnetBlock2D(32, 16, temb_channels=8, groups=4)
    den = _denoiser(n_timesteps=8, pnp_attn_t=0.25, pnp_f_t=0.75, pnp_conv_modules=[r])
    x = torch.zeros(4, 4, 8, 8)
    phases = []
    for i, t in enumerate(den.timesteps):
        key = den._graph_key(x, t)
        assert key == (tuple(x.shape), i < 2, i < 6), (i, key)
        assert den.injecting(t) == (i < 2) and den.conv_injecting(t) == (i < 6)
        phases.append(key[1:])
    assert sorted(set(phases)) == [(False, False), (False, True), (True, True)]
    # a conv schedule shorter than the attention one gives the fourth combination
    den = _denoiser(n_timesteps=8, pnp_attn_t=0.5, pnp_f_t=0.25, pnp_conv_modules=[r])
    assert [den._graph_key(x, t)[1:] for t in den.timesteps[:4]] == [(True, True)] * 2 + [(True, False)] * 2


@pytest.mark.parametrize("n,frac", [(50, 0.5), (6, 0.5), (8, 0.25)])
def test_without_pnp_f_t_nothing_changes(n, frac):
    from vidtome_b200.skeleton import ResnetBlock2D
    r = ResnetBlock2D(32, 16, temb_channels=8, groups=4)
    den = _denoiser(n_timesteps=n, pnp_attn_t=frac)
    x = torch.zeros(4, 4, 8, 8)
    k = int(n * frac)
    for i, t in enumerate(den.timesteps):
        assert den._graph_key(x, t) == (tuple(x.shape), i < k)
        assert not den.conv_injecting(t)
    assert den.pnp_f_t is None and den.pnp_conv_schedule == [] and not hasattr(r, "_vtm_pnp_conv")
    # the same steps, the same noise predictions, with and without an (unused) conv module around
    torch.manual_seed(5)
    x = torch.randn(6, 4, 8, 8)
    src = torch.randn(6, 4, 8, 8)
    outs = []
    for kw in ({}, {"pnp_conv_modules": [r]}):
        from vidtome_b200.driver import ChunkedDenoiser
        d = ChunkedDenoiser(StandInUNet(), n_timesteps=4, chunk_size=4, cond=torch.ones(3, 77, 16),
                            source_latents=lambda t: src, pnp_modules=[], **kw)
        y = x
        for i in range(4):
            y = d.step(y, i)
        outs.append(y)
    assert torch.equal(outs[0], outs[1])
    with pytest.raises(ValueError, match="needs source_latents"):
        ChunkedDenoiser(StandInUNet(), pnp_f_t=0.8)
    with pytest.raises(ValueError, match="pnp_conv_modules"):
        _denoiser(pnp_f_t=0.8)


def test_skeleton_stand_in_resnet():
    from vidtome_b200 import pnp
    from vidtome_b200.skeleton import PNP_CONV_POSITION, make_skeleton, pnp_conv_module
    plain = make_skeleton("sd15", device="cpu", dtype=torch.float32)
    net = make_skeleton("sd15", device="cpu", dtype=torch.float32, pnp_conv=True)
    assert plain.resnet is None
    with pytest.raises(ValueError, match="no stand-in ResNet"):
        pnp_conv_module(plain)
    # the option draws its weights after all others: the rest of the skeleton is unchanged
    sd, sd_plain = net.state_dict(), plain.state_dict()
    assert set(sd) - set(sd_plain) == {k for k in sd if k.startswith("resnet.")}
    assert all(torch.equal(sd[k], v) for k, v in sd_plain.items())
    r = pnp_conv_module(net)
    C = net.census[PNP_CONV_POSITION].dim
    assert (r.conv1.in_channels, r.conv1.out_channels, r.conv_shortcut.out_channels) == (2 * C, C, C) == (2560, 1280, 1280)
    for attr in ("norm1", "nonlinearity", "upsample", "downsample", "conv1", "time_emb_proj", "time_embedding_norm",
                 "norm2", "dropout", "conv2", "conv_shortcut", "output_scale_factor"):
        assert hasattr(r, attr), attr
    with pytest.raises(ValueError, match="census block 8"):
        make_skeleton("sd15", device="cpu", dtype=torch.float32, max_downsample=2, pnp_conv=True)
    with pytest.raises(ValueError, match="census block 8"):
        make_skeleton("tiny", device="cpu", dtype=torch.float32, pnp_conv=True)
    # the ResNet runs in the forward, sees the timestep, and its injection reaches the prediction
    torch.manual_seed(0)
    lat = torch.randn(3, 4, 16, 16)
    with torch.no_grad():
        a = plain(lat, 981).sample
        b = net(lat, 981).sample
        c = net(lat, 1).sample
        pnp.register_conv_control(net, [981], num_inputs=3, modules=[r])
        pnp.register_time(net, 981)
        seen = []
        r.register_forward_pre_hook(lambda m, args: seen.append(args))
        d = net(lat, 981).sample
    assert not torch.equal(a, b) and not torch.equal(b, c) and not torch.equal(b, d)
    # the skeleton hands the ResNet what a diffusers UNet does (contiguous NCHW, [B, temb] embedding): on the CPU only
    # the device keeps the call off the library path
    (x, temb), = seen
    assert x.shape == (3, 2560, 4, 4) and x.is_contiguous() and temb.shape == (3, 1280)
    assert pnp.conv_ineligibility(r, x, temb) == "device"


def test_library_entry_point_argument_errors():
    from vidtome_b200 import _lib
    lib = _lib.load()
    fn = lib.vtm_resnet_tail_f16
    assert fn is not None
    p = 0x10000                                                 # never dereferenced: every call below is refused first
    E_NULL, E_SHAPE, E_UNSUP = -1, -2, -6
    assert fn(None, p, p, 2, 3, 100, 1.0, 1, None) == E_NULL
    assert fn(p, None, p, 2, 3, 100, 1.0, 1, None) == E_NULL
    assert fn(p, p, None, 2, 3, 100, 1.0, 1, None) == E_NULL
    assert fn(p, p, p, 0, 3, 100, 1.0, 1, None) == E_SHAPE
    assert fn(p, p, p, 2, 0, 100, 1.0, 1, None) == E_SHAPE
    assert fn(p, p, p, 2, 3, 0, 1.0, 1, None) == E_SHAPE
    assert fn(p, p, p, 2, 3, -5, 1.0, 1, None) == E_SHAPE
    assert fn(p, p, p, 2, 4, 100, 1.0, 1, None) == E_UNSUP
    assert fn(p, p, p, 2, 3, 100, 1.0, 2, None) == E_UNSUP
    assert fn(p, p, p, 2, 3, 100, 0.0, 1, None) == E_UNSUP
    assert fn(p, p, p, 2, 3, 100, float("inf"), 1, None) == E_UNSUP
    assert fn(p, p, p, 2, 3, 100, float("nan"), 1, None) == E_UNSUP
    assert fn(p + 1, p, p, 2, 3, 100, 1.0, 1, None) == E_SHAPE         # fp16 pointers are 2-byte aligned
    assert fn(p, p, p + 1, 2, 3, 100, 1.0, 1, None) == E_SHAPE
    assert fn(p, p, p, 1 << 30, 3, 1 << 62, 1.0, 0, None) == E_SHAPE  # element count overflows int64
    assert lib.vtm_error_string(E_UNSUP).decode()
    assert isinstance(fn.argtypes[6], type) and fn.argtypes[6] is ctypes.c_float


def test_ops_wrapper_refuses_cpu_and_bad_shapes():
    from vidtome_b200 import ops
    h = torch.zeros(6, 4, 2, 2, dtype=torch.float16)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.resnet_tail(h, h, 3, 1.0, True)
