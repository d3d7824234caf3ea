"""DDIM inversion, host side: driver.ChunkedInverter on the unpatched tiny CPU skeleton against the reference's own
`Inverter.ddim_inversion` (tests/golden/inversion_*.npz, written by tests/make_golden_inversion.py), the kept-timestep
set, `source_latents`, the argument errors, the unmerged-block context's switches, and the two new library entry
points' argument checks, which return before any CUDA call."""
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["f11_b4_s50", "f11_b4_s50_final", "f11_b4_s20_save5", "f6_b4_s10_control"]


def _tiny():
    from vidtome_b200.skeleton import make_controlnet, make_skeleton
    return (make_skeleton("tiny", hot_path_only=False, device="cpu", dtype=torch.float32),
            make_controlnet("tiny", hot_path_only=False, device="cpu", dtype=torch.float32))


def _inverter(g, unet, controlnet, **kw):
    from vidtome_b200.driver import ChunkedInverter
    seed = torch.from_numpy(g["cond_seed"])
    cond = seed.repeat(1, 1, 768 // seed.shape[-1])
    control = bool(g["control"])
    return ChunkedInverter(unet, n_timesteps=int(g["steps"]), batch_size=int(g["batch_size"]),
                           save_steps=int(g["save_steps"]), save_intermediate=bool(g["save_intermediate"]), cond=cond,
                           controlnet=controlnet if control else None,
                           control_images=torch.from_numpy(g["images"]) if control else None,
                           control_scale=float(g["control_scale"]), **kw)


@pytest.mark.parametrize("name", CASES)
def test_inverter_matches_reference_ddim_inversion(name):
    g = np.load(os.path.join(GOLD, f"inversion_{name}.npz"))
    unet, controlnet = _tiny()
    inv = _inverter(g, unet, controlnet)
    x = torch.from_numpy(g["x"])
    final = inv.invert(x)
    assert torch.equal(x, torch.from_numpy(g["x"]))                  # the input is not modified
    assert inv.saved_timesteps == [int(t) for t in g["saved"]]       # exactly the reference's files
    want = torch.from_numpy(g["latents"])
    assert inv.trajectory.shape == want.shape
    for k in range(len(want)):                                       # test_host_cpu's pred_next_x tolerance
        err = (inv.trajectory[k] - want[k]).abs().max().item()
        assert err <= 2e-3 * want[k].abs().max().item() + 1e-3, (k, err)
    assert torch.equal(final, inv.trajectory[-1])
    load = inv.source_latents()
    for k, t in enumerate(inv.saved_timesteps):
        assert torch.equal(load(t), inv.trajectory[k])
    sub = inv.source_latents([1, 3])
    assert torch.equal(sub(inv.saved_timesteps[-1]), inv.trajectory[-1][[1, 3]])


def test_save_schedule_and_missing_timestep():
    from vidtome_b200.driver import ChunkedInverter, ddim_timesteps
    unet, _ = _tiny()
    inv = ChunkedInverter(unet, n_timesteps=20, save_steps=5, batch_size=4, cond=torch.zeros(1, 77, 768))
    assert inv.timesteps == ddim_timesteps(20)[::-1]
    assert inv.saved_timesteps == [1, 201, 401, 601, 801, 951]
    assert [inv.timesteps[i] for i, s in enumerate(inv.slots) if s >= 0] == inv.saved_timesteps
    assert ChunkedInverter(unet, n_timesteps=20, save_intermediate=False).saved_timesteps == [951]
    with pytest.raises(RuntimeError, match="invert"):
        inv.source_latents()
    inv.invert(torch.randn(3, 4, 4, 4))
    with pytest.raises(KeyError, match="timestep 51"):
        inv.source_latents()(51)


def test_inverter_cpu_steps_are_the_torch_restatement():
    """Every step is pred_next_x on the UNet's prediction: one step by hand equals the first kept latents."""
    from vidtome_b200.driver import ChunkedInverter
    unet, _ = _tiny()
    torch.manual_seed(3)
    x, cond = torch.randn(5, 4, 4, 4), torch.randn(1, 77, 768)
    inv = ChunkedInverter(unet, n_timesteps=10, batch_size=2, cond=cond)
    inv.invert(x)
    with torch.no_grad():
        eps = torch.cat([unet(x[lo:lo + 2], 1, encoder_hidden_states=cond.expand(len(x[lo:lo + 2]), -1, -1)).sample
                         for lo in range(0, 5, 2)])
    assert torch.equal(inv.trajectory[0], inv.pred_next_x(x, eps, 0))
    a, b, c, d = inv.coefficients(0)
    ac = inv.alphas_cumprod
    assert (a, b) == (float((1 - ac[0]) ** 0.5), float(ac[0] ** 0.5))    # i = 0: final_alpha_cumprod
    assert (c, d) == (float(ac[1] ** 0.5), float((1 - ac[1]) ** 0.5))


def test_argument_errors():
    from vidtome_b200.driver import ChunkedInverter
    unet, controlnet = _tiny()
    with pytest.raises(ValueError, match="n_timesteps"):
        ChunkedInverter(unet, n_timesteps=0)
    with pytest.raises(ValueError, match="batch_size"):
        ChunkedInverter(unet, batch_size=0)
    with pytest.raises(ValueError, match="save_steps"):
        ChunkedInverter(unet, save_steps=0)
    with pytest.raises(ValueError, match="go together"):
        ChunkedInverter(unet, controlnet=controlnet)
    with pytest.raises(ValueError, match="control_images"):
        ChunkedInverter(unet, controlnet=controlnet, control_images=torch.zeros(2, 1, 8, 8))
    with pytest.raises(ValueError, match="cond"):
        ChunkedInverter(unet, cond=torch.zeros(2, 76, 768))
    with pytest.raises(ValueError, match="graph_warmup"):
        ChunkedInverter(unet, cuda_graph=True, graph_warmup=0)
    x = torch.zeros(3, 4, 4, 4)
    with pytest.raises(ValueError, match="cond has 2 rows for 3 frames"):
        ChunkedInverter(unet, cond=torch.zeros(2, 77, 768)).invert(x)
    with pytest.raises(ValueError, match="control_images has 2 frames"):
        ChunkedInverter(unet, controlnet=controlnet, control_images=torch.zeros(2, 3, 8, 8)).invert(x)
    with pytest.raises(ValueError, match="CUDA fp16"):
        ChunkedInverter(unet, cuda_graph=True).invert(x)
    with pytest.raises(ValueError, match=r"\[F, 4, h, w\]"):
        ChunkedInverter(unet).invert(x[0])


def test_unmerged_context_switches_hooks_and_injection():
    """Inside _unmerged_blocks() the model and block pre-hooks record nothing and fork no generator, and PnP's injection
    test is off whatever `t` holds; outside, everything is as before."""
    from vidtome_b200 import patch, pnp
    from vidtome_b200.skeleton import make_skeleton, pnp_attention_modules
    unet = make_skeleton("sd15", device="cpu", dtype=torch.float32, max_downsample=1)
    patch.apply_patch(unet, batch_size=3, align_batch=True)
    mods = pnp_attention_modules(unet)
    pnp.register_attention_control(unet, [981], 3, modules=mods)
    pnp.register_time(unet, 981, modules=mods)
    assert all(pnp.injection_active(m) for m in mods)
    with patch._unmerged_blocks():
        assert patch.unmerged_active()
        assert not any(pnp.injection_active(m) for m in mods)
        for _, m in unet.named_modules():
            for h in m._forward_pre_hooks.values():
                h(m, (torch.zeros(1, 4, 8, 8),))
        assert unet._tome_info["size"] is None
        assert not any(hasattr(m, "generator") for m in unet.modules())
        with patch._unmerged_blocks():                                # nests
            assert patch.unmerged_active()
        assert patch.unmerged_active()
    assert not patch.unmerged_active()
    assert all(pnp.injection_active(m) and m.t == 981 for m in mods)


def test_library_entry_points_argument_errors():
    from vidtome_b200 import _lib
    lib = _lib.load()
    p = 0x10000                                                  # never dereferenced: every call below is refused first
    E_NULL, E_SHAPE, E_WS, E_UNSUP = -1, -2, -4, -6
    ddim = lib.vtm_ddim_update_f16
    #          x     eps   n    coef  slot  step  steps traj  n_slots stream
    assert ddim(None, p, 100, p, p, p, 50, p, 3, None) == E_NULL
    assert ddim(p, None, 100, p, p, p, 50, p, 3, None) == E_NULL
    assert ddim(p, p, 100, None, p, p, 50, p, 3, None) == E_NULL
    assert ddim(p, p, 100, p, p, None, 50, p, 3, None) == E_NULL
    assert ddim(p, p, 100, p, p, p, 50, None, 3, None) == E_NULL          # a slot table needs the trajectory
    assert ddim(p, p, 0, p, p, p, 50, p, 3, None) == E_SHAPE
    assert ddim(p, p, -7, p, p, p, 50, p, 3, None) == E_SHAPE
    assert ddim(p, p, 100, p, p, p, 0, p, 3, None) == E_SHAPE
    assert ddim(p, p, 100, p, p, p, 50, p, 0, None) == E_SHAPE
    assert ddim(p, p, 100, p, p, p, 50, p, -1, None) == E_SHAPE
    assert ddim(p + 1, p, 100, p, p, p, 50, p, 3, None) == E_SHAPE        # fp16 pointers are 2-byte aligned
    assert ddim(p, p + 1, 100, p, p, p, 50, p, 3, None) == E_SHAPE
    assert ddim(p, p, 100, p, p, p, 50, p + 1, 3, None) == E_SHAPE
    assert ddim(p, p, 100, p + 8, p, p, 50, p, 3, None) == E_SHAPE        # the table is read as float4
    assert ddim(p, p, 100, p, p, p + 2, 50, p, 3, None) == E_SHAPE
    assert ddim(p, p, 100, p, p + 2, p, 50, p, 3, None) == E_SHAPE
    assert ddim(p, p, 1 << 62, p, p, p, 50, p, 8, None) == E_SHAPE        # trajectory size overflows int64
    att = lib.vtm_attention_residual
    ws = lib.vtm_attention_workspace_bytes(2, 64, 320, 8)
    #         x  wqkv wo  bo  resid lq    lo    B  L   C    heads scale y  ws  bytes stream
    assert att(p, p, p, None, None, None, None, 2, 64, 320, 8, 0.1, p, p, ws, None) == E_NULL
    assert att(None, p, p, None, p, None, None, 2, 64, 320, 8, 0.1, p, p, ws, None) == E_NULL
    assert att(p, p, p, None, p, None, None, 2, 64, 320, 8, 0.1, None, p, ws, None) == E_NULL
    assert att(p, p, p, None, p, None, None, 0, 64, 320, 8, 0.1, p, p, ws, None) == E_SHAPE
    assert att(p, p, p, None, p, None, None, 2, 64, 320, 7, 0.1, p, p, ws, None) == E_SHAPE
    assert att(p, p, p, None, p, None, None, 2, 64, 320, 64, 0.1, p, p, ws, None) == E_SHAPE   # head_dim 5
    assert att(p, p, p, None, p, None, None, 2, 64, 1344, 7, 0.1, p, p, 1 << 40, None) == E_UNSUP  # head_dim 192
    assert att(p, p, p, None, p, None, None, 2, 64, 320, 8, 0.1, p, p, ws - 1, None) == E_WS
    lora = _lib.VtmLora(p, p, 8)
    wl = lib.vtm_attention_lora_workspace_bytes(2, 64, 320, 8, 0, 8)
    assert wl > ws
    assert att(p, p, p, None, p, None, lora, 2, 64, 320, 8, 0.1, p, p, ws, None) == E_WS


def test_ops_wrappers_refuse_cpu_and_bad_shapes():
    from vidtome_b200 import ops
    h = torch.zeros(2, 4, 8, dtype=torch.float16)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.attention_residual(h, h, h, None, 1, 1.0, h)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.ddim_update(h, h, torch.zeros(1, 4), torch.zeros(1, dtype=torch.int32))
