"""SD2-depth in the step driver and the inverter (ChunkedDenoiser(depth=...), ChunkedInverter(depth=...)), host side:
the noise prediction with and without PnP against the reference's own Generator.pred_noise, the inversion trajectory
against its own Inverter.ddim_inversion (tests/golden/depth_*.npz, written by tests/make_golden_depth.py), the depth
maps each chunk gets when chunks are visited out of order, the depth skeleton, and the refusals."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _depth_skeleton():
    from vidtome_b200.skeleton import make_skeleton
    return make_skeleton("tiny", hot_path_only=False, device="cpu", dtype=torch.float32, depth=True)


def _cond(seed: np.ndarray) -> torch.Tensor:
    seed = torch.from_numpy(seed)
    return seed.repeat(1, 1, 768 // seed.shape[-1])


class RecordingUNet(torch.nn.Module):
    """A 5-channel UNet stand-in that records every sample it gets; its prediction mixes the latent and depth channels."""

    in_channels = 5

    def __init__(self):
        super().__init__()
        self.calls = []

    def forward(self, sample, t, encoder_hidden_states=None, **kwargs):
        self.calls.append(sample.clone())
        return SimpleNamespace(sample=sample[:, :4] * 0.5 + sample[:, 4:] * 0.25 + float(t) * 1e-4)


@pytest.mark.parametrize("pnp", [False, True])
def test_pred_noise_matches_reference(pnp):
    from vidtome_b200.driver import ChunkedDenoiser
    g = np.load(os.path.join(GOLD, "depth_pred_noise.npz"))
    x, src, depth = (torch.from_numpy(g[k]) for k in ("x", "src", "depth"))
    cond3 = _cond(g["cond_seed"])
    lo, hi, t = int(g["lo"]), int(g["hi"]), int(g["t"])
    den = ChunkedDenoiser(_depth_skeleton(), cond=cond3 if pnp else cond3[1:],
                          guidance_scale=float(g["guidance_scale"]), depth=depth)
    out = den.pred_noise(x[lo:hi], t, src[lo:hi] if pnp else None, depth=depth[lo:hi])
    want = torch.from_numpy(g["out_pnp" if pnp else "out_plain"])
    torch.testing.assert_close(out, want, rtol=1e-5, atol=1e-5 * want.abs().max().item())
    # the depth channel matters: other maps give another prediction
    other = den.pred_noise(x[lo:hi], t, src[lo:hi] if pnp else None, depth=-depth[lo:hi])
    assert (other - want).abs().max() > 1e-2 * want.abs().max()


def test_pred_noise_batch_layout():
    """generate.py:256-262: the depth maps repeated over [source | x | x] and appended as channel 4."""
    from vidtome_b200.driver import ChunkedDenoiser
    torch.manual_seed(0)
    x, src, depth = torch.randn(3, 4, 8, 8), torch.randn(3, 4, 8, 8), torch.randn(3, 1, 8, 8)
    den = ChunkedDenoiser(RecordingUNet(), depth=depth)
    den.pred_noise(x, 981, depth=depth)
    den.pred_noise(x, 981, src, depth=depth)
    plain, pnp = den.unet.calls
    assert torch.equal(plain, torch.cat([torch.cat([x, x]), depth.repeat(2, 1, 1, 1)], dim=1))
    assert torch.equal(pnp, torch.cat([torch.cat([src, x, x]), depth.repeat(3, 1, 1, 1)], dim=1))


def test_inverter_matches_reference_ddim_inversion():
    from vidtome_b200.driver import ChunkedInverter
    g = np.load(os.path.join(GOLD, "depth_inversion_f11_b4.npz"))
    x, depth = torch.from_numpy(g["x"]), torch.from_numpy(g["depth"])
    inv = ChunkedInverter(_depth_skeleton(), n_timesteps=int(g["steps"]), batch_size=int(g["batch_size"]),
                          cond=_cond(g["cond_seed"]), depth=depth)
    assert len(x) % inv.batch_size != 0                               # the last batch is ragged
    final = inv.invert(x)
    assert torch.equal(x, torch.from_numpy(g["x"]))
    assert inv.saved_timesteps == [int(t) for t in g["saved"]]
    want = torch.from_numpy(g["latents"])
    assert inv.trajectory.shape == want.shape                        # 4 latent channels
    for k in range(len(want)):                                       # test_inversion_cpu's tolerance
        err = (inv.trajectory[k] - want[k]).abs().max().item()
        assert err <= 2e-3 * want[k].abs().max().item() + 1e-3, (k, err)
    assert torch.equal(final, inv.trajectory[-1])
    # without the depth maps' contribution the trajectory is another one
    other = ChunkedInverter(_depth_skeleton(), n_timesteps=int(g["steps"]), batch_size=int(g["batch_size"]),
                            cond=_cond(g["cond_seed"]), depth=torch.zeros_like(depth))
    other.invert(x)
    assert (other.trajectory[-1] - want[-1]).abs().max() > 1e-2


def test_inverter_batches_get_their_own_depth():
    from vidtome_b200.driver import ChunkedInverter
    torch.manual_seed(1)
    x, depth = torch.randn(7, 4, 4, 4), torch.randn(7, 1, 4, 4)
    inv = ChunkedInverter(RecordingUNet(), n_timesteps=2, batch_size=3, depth=depth)
    inv.invert(x)
    calls = inv.unet.calls
    assert [len(c) for c in calls] == [3, 3, 1] * 2
    for c, lo in zip(calls, [0, 3, 6] * 2):
        assert c.shape[1] == 5 and torch.equal(c[:, 4:], depth[lo:lo + len(c)])
    assert torch.equal(calls[0][:, :4], x[:3])


@pytest.mark.parametrize("order", ["reversed", "permuted"])
def test_eager_step_gives_each_chunk_its_frames_depth(order):
    from vidtome_b200.driver import ChunkedDenoiser
    flen = 10
    torch.manual_seed(5)
    np.random.seed(5)
    depth = torch.randn(flen, 1, 8, 8)
    kw = (dict(randomize_chunks=True) if order == "reversed" else dict(merge_global=True, chunk_ord="rand"))
    den = ChunkedDenoiser(RecordingUNet(), n_timesteps=8, chunk_size=4, depth=depth, **kw)
    x = torch.randn(flen, 4, 8, 8)
    out_of_order = False
    for i in range(len(den.timesteps)):
        before = len(den.unet.calls)
        x_in = x
        x = den.step(x, i)
        los = []
        for sample in den.unet.calls[before:]:
            n = len(sample) // 2
            lo, = [f for f in range(flen) if torch.equal(x_in[f], sample[0, :4])]
            los.append(lo)
            assert torch.equal(sample[:n, :4], x_in[lo:lo + n]) and torch.equal(sample[n:, :4], sample[:n, :4])
            assert torch.equal(sample[:, 4:], depth[lo:lo + n].repeat(2, 1, 1, 1)), (i, lo)
        lens = [len(s) // 2 for s in den.unet.calls[before:]]
        assert sorted(f for lo, n in zip(los, lens) for f in range(lo, lo + n)) == list(range(flen))
        out_of_order |= los != sorted(los)
    assert out_of_order, "no step visited its chunks out of order"


def test_depth_skeleton():
    from vidtome_b200.skeleton import make_skeleton
    net = _depth_skeleton()
    assert (net.in_channels, net.out_channels) == (5, 4)
    plain = make_skeleton("tiny", hot_path_only=False, device="cpu", dtype=torch.float32)
    assert (plain.in_channels, plain.out_channels) == (4, 4)
    # the blocks are drawn before the lift, so they are the same as the plain skeleton's
    for a, b in zip(net.blocks.parameters(), plain.blocks.parameters()):
        assert torch.equal(a, b)
    torch.manual_seed(2)
    x, d = torch.randn(2, 4, 8, 8), torch.randn(2, 1, 8, 8)
    cond = torch.randn(2, 77, 768)
    with torch.no_grad():
        eps = net(torch.cat([x, d], dim=1), 981, encoder_hidden_states=cond).sample
        eps2 = net(torch.cat([x, -d], dim=1), 981, encoder_hidden_states=cond).sample
    assert eps.shape == x.shape and not torch.equal(eps, eps2)


def test_denoiser_refusals():
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton
    with pytest.raises(ValueError, match=r"\[flen, 1, h, w\]"):
        ChunkedDenoiser(RecordingUNet(), depth=torch.zeros(6, 8, 8))
    with pytest.raises(ValueError, match=r"\[flen, 1, h, w\]"):
        ChunkedDenoiser(RecordingUNet(), depth=torch.zeros(6, 3, 8, 8))
    with pytest.raises(ValueError, match="depth and controlnet are exclusive"):
        ChunkedDenoiser(RecordingUNet(), depth=torch.zeros(6, 1, 8, 8), controlnet=torch.nn.Identity(),
                        control_images=torch.zeros(6, 3, 64, 64))
    den = ChunkedDenoiser(RecordingUNet(), chunk_size=4, depth=torch.zeros(6, 1, 8, 8))
    for shape in ((5, 4, 8, 8), (7, 4, 8, 8), (6, 4, 8, 4), (6, 4, 16, 16)):
        with pytest.raises(ValueError, match="one map per frame"):
            den.step(torch.randn(shape), 0)
    plain = make_skeleton("tiny", device="cpu", dtype=torch.float32)            # 4 input channels
    with pytest.raises(ValueError, match="takes 4 input channels"):
        ChunkedDenoiser(plain, chunk_size=4, depth=torch.zeros(6, 1, 8, 8)).step(torch.randn(6, 4, 8, 8), 0)
    diffusers_like = RecordingUNet()
    diffusers_like.config = SimpleNamespace(in_channels=9)                      # unet.config.in_channels wins
    with pytest.raises(ValueError, match="takes 9 input channels"):
        ChunkedDenoiser(diffusers_like, depth=torch.zeros(6, 1, 8, 8)).step(torch.randn(6, 4, 8, 8), 0)
    assert not den.unet.calls and not diffusers_like.calls


def test_inverter_refusals():
    from vidtome_b200.driver import ChunkedInverter
    from vidtome_b200.skeleton import make_skeleton
    with pytest.raises(ValueError, match=r"\[flen, 1, h, w\]"):
        ChunkedInverter(RecordingUNet(), depth=torch.zeros(6, 8, 8))
    with pytest.raises(ValueError, match=r"\[flen, 1, h, w\]"):
        ChunkedInverter(RecordingUNet(), depth=torch.zeros(6, 2, 8, 8))
    with pytest.raises(ValueError, match="depth and controlnet are exclusive"):
        ChunkedInverter(RecordingUNet(), depth=torch.zeros(6, 1, 8, 8), controlnet=torch.nn.Identity(),
                        control_images=torch.zeros(6, 3, 64, 64))
    inv = ChunkedInverter(RecordingUNet(), n_timesteps=2, depth=torch.zeros(6, 1, 8, 8))
    for shape in ((5, 4, 8, 8), (7, 4, 8, 8), (6, 4, 4, 8)):
        with pytest.raises(ValueError, match="one map per frame"):
            inv.invert(torch.randn(shape))
    plain = make_skeleton("tiny", device="cpu", dtype=torch.float32)
    with pytest.raises(ValueError, match="takes 4 input channels"):
        ChunkedInverter(plain, n_timesteps=2, depth=torch.zeros(6, 1, 8, 8)).invert(torch.randn(6, 4, 8, 8))
    assert not inv.unet.calls
