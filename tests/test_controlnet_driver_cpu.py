"""ControlNet control in the step driver (ChunkedDenoiser(controlnet=..., control_images=...)), host side: the noise
prediction against the reference's own pred_noise / get_controlnet_kwargs (tests/golden/callers_pred_noise_controlnet.npz,
written by tests/make_golden_controlnet.py), the calls it issues, the refusals, the skeleton ControlNet's residuals, and
the reach of the global-token stores and resets into a patched ControlNet."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "callers_pred_noise_controlnet.npz")


class StandInControlNet(torch.nn.Module):
    """Deterministic ControlNet stand-in that records its calls and the residual tensors it returns.  Every residual row
    depends on its own latent, text row, control image, batch position and the timestep."""

    def __init__(self):
        super().__init__()
        self.calls = []
        self.returned = []              # (down list, mid) as returned, the objects themselves
        self.returned_values = []       # their values at return time

    def forward(self, sample, timestep, encoder_hidden_states=None, controlnet_cond=None, return_dict=True):
        self.calls.append(dict(sample=sample, t=int(timestep), text=encoder_hidden_states, cond=controlnet_cond.clone(),
                               return_dict=return_dict))
        n, _, h, w = sample.shape
        wgt = 1 + 0.5 * torch.arange(n, dtype=sample.dtype) / n
        img = F.avg_pool2d(controlnet_cond.mean(dim=1, keepdim=True), controlnet_cond.shape[-1] // w)
        base = sample * wgt[:, None, None, None] + img + float(timestep) * 1e-3
        if encoder_hidden_states is not None:
            base = base + 0.25 * encoder_hidden_states.mean(dim=(1, 2))[:, None, None, None]
        down = [base * 0.5, base.flip(-1) - 0.1]
        mid = base.mean(dim=1, keepdim=True) * 2
        self.returned.append((list(down), mid))
        self.returned_values.append(([d.clone() for d in down], mid.clone()))
        return down, mid


class StandInUNet(torch.nn.Module):
    """Deterministic UNet stand-in taking the additional residuals; records its calls."""

    def __init__(self):
        super().__init__()
        self.calls = []

    def forward(self, sample, t, encoder_hidden_states=None, down_block_additional_residuals=None,
                mid_block_additional_residual=None):
        self.calls.append(dict(sample=sample, t=int(t), text=encoder_hidden_states,
                               down=down_block_additional_residuals, mid=mid_block_additional_residual))
        n = sample.shape[0]
        wgt = 1 + 0.25 * torch.arange(n, dtype=sample.dtype) / n
        eps = sample * wgt[:, None, None, None] + float(t) * 1e-3
        if encoder_hidden_states is not None:
            eps = eps + 0.5 * encoder_hidden_states.mean(dim=(1, 2))[:, None, None, None]
        if down_block_additional_residuals is not None:
            for k, d in enumerate(down_block_additional_residuals):
                eps = eps + (k + 1) * 0.1 * d
        if mid_block_additional_residual is not None:
            eps = eps + 0.3 * mid_block_additional_residual
        return SimpleNamespace(sample=eps)


def _denoiser(ctrl, cond=None, **kw):
    from vidtome_b200.driver import ChunkedDenoiser
    cond = torch.randn(2, 77, 16) if cond is None else cond
    return ChunkedDenoiser(StandInUNet(), cond=cond, controlnet=StandInControlNet(), control_images=ctrl, **kw)


def test_pred_noise_matches_reference():
    g = np.load(GOLD)
    x, cond, ctrl = (torch.from_numpy(g[k]) for k in ("x", "cond", "ctrl"))
    lo, hi, t, scale = int(g["lo"]), int(g["hi"]), int(g["t"]), float(g["control_scale"])
    den = _denoiser(ctrl, cond=cond, guidance_scale=float(g["guidance_scale"]), control_scale=scale)
    out = den.pred_noise(x[lo:hi], t, ctrl=ctrl[lo:hi])
    np.testing.assert_array_equal(out.numpy(), g["out"])

    n = hi - lo
    (cn,), (un,) = den.controlnet.calls, den.unet.calls
    # the ControlNet sees the UNet's batch [x | x] and text, and the chunk's control images once per CFG sample
    assert cn["sample"] is un["sample"] and torch.equal(un["sample"], torch.cat([x[lo:hi], x[lo:hi]]))
    assert cn["text"] is un["text"] and torch.equal(un["text"], cond.repeat_interleave(n, dim=0))
    assert torch.equal(cn["cond"], torch.cat([ctrl[lo:hi]] * 2))
    assert cn["t"] == un["t"] == t and cn["return_dict"] is False
    # down residuals scaled out of place, the mid residual in place, each exactly once
    (down_ret, mid_ret), = den.controlnet.returned
    (down_val, mid_val), = den.controlnet.returned_values
    assert len(un["down"]) == len(down_ret)
    for passed, ret, val in zip(un["down"], down_ret, down_val):
        assert passed is not ret and torch.equal(ret, val)
        assert torch.equal(passed, val * scale)
    assert un["mid"] is mid_ret and torch.equal(mid_ret, mid_val * scale)


def test_eager_step_gives_each_chunk_its_control_images():
    torch.manual_seed(3)
    flen = 6
    x = torch.randn(flen, 4, 8, 8)
    ctrl = torch.randn(flen, 3, 16, 16)
    den = _denoiser(ctrl, n_timesteps=3, chunk_size=4, control_scale=0.5)
    for i in range(len(den.timesteps)):
        before = len(den.controlnet.calls)
        x = den.step(x, i)
        calls = den.controlnet.calls[before:]
        assert [c["sample"].shape[0] for c in calls] == [8, 4]            # chunks of 4 and 2 frames, 2 samples each
        for c, (lo, hi) in zip(calls, [(0, 4), (4, 6)]):
            assert torch.equal(c["cond"], ctrl[lo:hi].repeat(2, 1, 1, 1))
            assert c["t"] == den.timesteps[i]
    assert len(den.unet.calls) == len(den.controlnet.calls) == 6


def test_without_controlnet_the_unet_gets_no_residual_keywords():
    from vidtome_b200.driver import ChunkedDenoiser
    den = ChunkedDenoiser(StandInUNet(), cond=torch.randn(2, 77, 16))
    den.pred_noise(torch.randn(4, 4, 8, 8), 981)
    assert den.unet.calls[-1]["down"] is None and den.unet.calls[-1]["mid"] is None


def test_refusals():
    from vidtome_b200.driver import ChunkedDenoiser
    ctrl = torch.randn(6, 3, 16, 16)
    with pytest.raises(ValueError, match="exclusive"):
        ChunkedDenoiser(StandInUNet(), cond=torch.randn(3, 77, 16), source_latents=lambda t: None, pnp_modules=[],
                        controlnet=StandInControlNet(), control_images=ctrl)
    with pytest.raises(ValueError, match="go together"):
        ChunkedDenoiser(StandInUNet(), controlnet=StandInControlNet())
    with pytest.raises(ValueError, match="go together"):
        ChunkedDenoiser(StandInUNet(), control_images=ctrl)
    with pytest.raises(ValueError, match=r"\[flen, 3, H, W\]"):
        _denoiser(torch.randn(6, 1, 16, 16))
    den = _denoiser(ctrl, chunk_size=4)
    for flen in (5, 7):
        with pytest.raises(ValueError, match="control_images has 6 frames, the latents"):
            den.step(torch.randn(flen, 4, 8, 8), 0)
    assert not den.unet.calls and not den.controlnet.calls


def _skeletons(name="sd15", **kw):
    from vidtome_b200.skeleton import make_controlnet, make_skeleton
    return (make_skeleton(name, device="cpu", dtype=torch.float32, **kw),
            make_controlnet(name, device="cpu", dtype=torch.float32))


def test_skeleton_controlnet_residuals_match_the_unet_encoder_blocks():
    unet, cn = _skeletons()
    assert cn.census_index == list(range(7)) and cn.census == unet.census[:7]
    torch.manual_seed(0)
    x = torch.randn(4, 4, 16, 16)
    img = torch.rand(4, 3, 128, 128)
    down, mid = cn(x, 981, controlnet_cond=img, return_dict=False)
    assert len(down) == 6
    shapes = [(4, (16 // s.downsample) ** 2, s.dim) for s in unet.census[:7]]
    assert [tuple(d.shape) for d in down] + [tuple(mid.shape)] == shapes
    assert all(d.abs().max() > 0 for d in down) and mid.abs().max() > 0     # non-zero "zero convs"
    # the residuals reach the prediction; all-zero residuals leave it bit-identical
    plain = unet(x, 981).sample
    assert not torch.equal(unet(x, 981, down_block_additional_residuals=down,
                                mid_block_additional_residual=mid).sample, plain)
    zeros = unet(x, 981, down_block_additional_residuals=[torch.zeros_like(d) for d in down],
                 mid_block_additional_residual=torch.zeros_like(mid)).sample
    assert torch.equal(zeros, plain)
    # the control image matters
    down2, mid2 = cn(x, 981, controlnet_cond=img.flip(-1), return_dict=False)
    assert not torch.equal(mid, mid2)


def test_skeleton_unet_refuses_residuals_that_do_not_match_its_blocks():
    unet, cn = _skeletons()
    x = torch.randn(2, 4, 16, 16)
    down, mid = cn(x, 1, controlnet_cond=torch.rand(2, 3, 16, 16), return_dict=False)
    with pytest.raises(ValueError, match="5 residuals for the UNet's 6 down blocks"):
        unet(x, 1, down_block_additional_residuals=down[:5], mid_block_additional_residual=mid)
    with pytest.raises(ValueError, match="shape"):
        unet(x, 1, down_block_additional_residuals=down[::-1], mid_block_additional_residual=mid)
    with pytest.raises(ValueError, match="shape"):
        unet(x, 1, down_block_additional_residuals=down, mid_block_additional_residual=mid[:, :1])
    # a UNet without the deepest blocks has fewer down blocks and no mid block
    small, _ = _skeletons(max_downsample=2)
    with pytest.raises(ValueError, match="6 residuals for the UNet's 4 down blocks"):
        small(x, 1, down_block_additional_residuals=down)
    with pytest.raises(ValueError, match="no mid block"):
        small(x, 1, mid_block_additional_residual=mid)
    # a ControlNet of another census
    tiny_cn = _skeletons("tiny")[1]
    tdown, tmid = tiny_cn(x, 1, controlnet_cond=torch.rand(2, 3, 16, 16), return_dict=False)
    with pytest.raises(ValueError, match="down blocks"):
        unet(x, 1, down_block_additional_residuals=tdown, mid_block_additional_residual=tmid)
    with pytest.raises(ValueError, match="whole multiple"):
        cn(x, 1, controlnet_cond=torch.rand(2, 3, 24, 24))


def _pipeline(include_control):
    import vidtome_b200
    unet, cn = _skeletons("tiny")

    class DiffusionPipeline:
        pass

    class StableDiffusionControlNetPipeline(DiffusionPipeline):
        def __init__(self):
            self.unet, self.controlnet = unet, cn
    pipe = StableDiffusionControlNetPipeline()
    vidtome_b200.apply_patch(pipe, merge_global=True, include_control=include_control)
    return pipe


@pytest.mark.parametrize("include_control", [False, True])
def test_stores_and_global_reset_reach_the_patched_controlnet(include_control):
    from vidtome_b200 import patch
    from vidtome_b200.driver import ChunkedDenoiser
    pipe = _pipeline(include_control)
    cn_blocks = [m for m in pipe.controlnet.modules() if type(m).__name__ == "ToMeBlock"]
    assert len(cn_blocks) == (3 if include_control else 0)
    den = ChunkedDenoiser(pipe.unet, chunk_size=4, merge_global=True, controlnet=pipe.controlnet,
                          control_images=torch.zeros(8, 3, 16, 16))
    # update_patch(pipe, global_tokens=None) after each step reaches both models
    blocks = [m for net in (pipe.unet, pipe.controlnet) for m in net.modules() if hasattr(m, "_tome_info")]
    for m in blocks:
        m.global_tokens = torch.zeros(1)
    den._reset_global()
    assert all(m.global_tokens is None for m in blocks)
    # every ToMeBlock of both models gets a store, and resetting empties each one
    den._install_stores()
    unet_blocks = [m for m in pipe.unet.modules() if type(m).__name__ == "ToMeBlock"]
    assert len(den._stores) == len(unet_blocks) + len(cn_blocks) == 4 + len(cn_blocks)
    assert all(isinstance(b.global_tokens, patch.GlobalTokenStore) and b.global_tokens in den._stores
               for b in unet_blocks + cn_blocks)
    for st in den._stores:
        st.filled = True
    den._reset_global()
    assert not any(st.filled for st in den._stores)
