"""PnP control in the step driver (ChunkedDenoiser(source_latents=...)), host side: the noise prediction and the
injection schedule against the reference's own pred_noise / init_pnp (tests/golden/callers_pred_noise_pnp.npz, written
by tests/make_golden_pnp.py), the graph key of every step, and the constructor's refusals."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "callers_pred_noise_pnp.npz")


class StandInUNet(torch.nn.Module):
    """Deterministic UNet stand-in: every output row depends on its own latent, its own text row, its position in the
    batch and the timestep, so that a wrong batch order, conditioning or guidance split shows in the result."""

    def __init__(self, batch_size=3, align_batch=True):
        super().__init__()
        self._tome_info = {"args": {"batch_size": batch_size, "align_batch": align_batch}}
        self.calls = []

    def forward(self, sample, t, encoder_hidden_states=None, **kwargs):
        self.calls.append((sample.clone(), int(t), encoder_hidden_states))
        n = sample.shape[0]
        w = 1 + 0.25 * torch.arange(n, dtype=sample.dtype) / n
        eps = sample * w[:, None, None, None] + float(t) * 1e-3
        if encoder_hidden_states is not None:
            eps = eps + 0.5 * encoder_hidden_states.mean(dim=(1, 2))[:, None, None, None]
        return SimpleNamespace(sample=eps)


def _denoiser(unet=None, cond=None, src=None, **kw):
    from vidtome_b200.driver import ChunkedDenoiser
    unet = StandInUNet() if unet is None else unet
    cond = torch.randn(3, 77, 16) if cond is None else cond
    return ChunkedDenoiser(unet, cond=cond, source_latents=src if callable(src) else (lambda t: src), **kw)


def test_pred_noise_matches_reference():
    g = np.load(GOLD)
    x, cond, src = (torch.from_numpy(g[k]) for k in ("x", "cond", "src"))
    lo, hi, t = int(g["lo"]), int(g["hi"]), int(g["t"])
    den = _denoiser(cond=cond, src=src, guidance_scale=float(g["guidance_scale"]), pnp_modules=[])
    out = den.pred_noise(x[lo:hi], t, src[lo:hi])
    np.testing.assert_array_equal(out.numpy(), g["out"])
    sample, _, text = den.unet.calls[-1]
    n = hi - lo
    assert torch.equal(sample, torch.cat([src[lo:hi], x[lo:hi], x[lo:hi]]))
    assert torch.equal(text, cond.repeat_interleave(n, dim=0))


@pytest.mark.parametrize("case", range(5))
def test_schedule_matches_reference_init_pnp(case):
    from vidtome_b200.skeleton import Attention
    g = np.load(GOLD)
    n, frac = int(g[f"sched{case}_n"]), float(g[f"sched{case}_frac"])
    attn = Attention(32, 2, 16)
    den = _denoiser(n_timesteps=n, pnp_attn_t=frac, pnp_modules=[attn])
    assert den.pnp_schedule == [int(v) for v in g[f"sched{case}"]]
    assert attn._vtm_pnp == int(g["num_inputs"]) == 3
    assert list(attn.injection_schedule) == den.pnp_schedule


@pytest.mark.parametrize("n,frac", [(50, 0.5), (6, 0.5), (10, 0.35), (50, 0.0), (50, -0.2), (4, 1.0)])
def test_graph_key_follows_the_schedule(n, frac):
    den = _denoiser(n_timesteps=n, pnp_attn_t=frac, pnp_modules=[])
    x = torch.zeros(4, 4, 8, 8)
    k = int(n * frac)
    for i, t in enumerate(den.timesteps):
        want = 0 <= k and i < k
        assert den.injecting(t) == want, (i, t)
        assert den._graph_key(x, t) == (tuple(x.shape), want)
    # without PnP nothing is ever injected
    from vidtome_b200.driver import ChunkedDenoiser
    plain = ChunkedDenoiser(StandInUNet(), n_timesteps=n)
    assert not any(plain.injecting(t) for t in plain.timesteps)


def test_eager_step_feeds_source_latents_of_the_step():
    from vidtome_b200.skeleton import Attention
    torch.manual_seed(3)
    flen = 6
    x = torch.randn(flen, 4, 8, 8)
    srcs = {}

    def source(t):
        srcs[t] = torch.full((flen, 4, 8, 8), float(t) / 1000)
        return srcs[t]
    attn = Attention(32, 2, 16)
    den = _denoiser(src=source, n_timesteps=4, pnp_attn_t=0.5, chunk_size=4, pnp_modules=[attn])
    for i in range(len(den.timesteps)):
        t = den.timesteps[i]
        before = len(den.unet.calls)
        x = den.step(x, i)
        assert attn.t == t
        calls = den.unet.calls[before:]
        assert [c[0].shape[0] for c in calls] == [12, 6]                 # chunks of 4 and 2 frames, 3 samples each
        lo = 0
        for sample, tt, text in calls:
            m = sample.shape[0] // 3
            assert tt == t and text.shape == (3 * m, 77, 16)
            assert torch.equal(sample[:m], srcs[t][lo:lo + m])
            assert torch.equal(sample[m:2 * m], sample[2 * m:])
            lo += m
    assert set(srcs) == set(den.timesteps)


def test_refusals():
    with pytest.raises(ValueError, match="batch_size=3 and align_batch=True"):
        _denoiser(unet=StandInUNet(batch_size=2), pnp_modules=[])
    with pytest.raises(ValueError, match="batch_size=3 and align_batch=True"):
        _denoiser(unet=StandInUNet(align_batch=False), pnp_modules=[])
    bare = StandInUNet()
    del bare._tome_info
    with pytest.raises(ValueError, match="batch_size=3 and align_batch=True"):
        _denoiser(unet=bare, pnp_modules=[])
    for cond in (torch.randn(2, 77, 16), torch.randn(3, 76, 16), torch.randn(3, 77)):
        with pytest.raises(ValueError, match=r"cond = \[3, 77, D\]"):
            _denoiser(cond=cond, pnp_modules=[])
    from vidtome_b200.driver import ChunkedDenoiser
    with pytest.raises(ValueError, match=r"cond = \[3, 77, D\]"):
        ChunkedDenoiser(StandInUNet(), source_latents=lambda t: None, pnp_modules=[])
    # the refusals of the graph modes stay as they are
    with pytest.raises(ValueError, match="shard=True"):
        _denoiser(pnp_modules=[], cuda_graph=True, chunk_graphs=True, shard=True)


def test_skeleton_pnp_targets_are_the_reference_decoder_blocks():
    from vidtome_b200.skeleton import make_skeleton, pnp_attention_modules
    net = make_skeleton("sd15", device="cpu", dtype=torch.float32)
    mods = pnp_attention_modules(net)
    assert mods == [net.blocks[i].attn1 for i in range(8, 16)]
    dims = [m.to_q.weight.shape[0] for m in mods]
    assert dims == [1280] * 2 + [640] * 3 + [320] * 3                   # up_blocks[1].attentions[1, 2], [2], [3]
    small = make_skeleton("sd15", device="cpu", dtype=torch.float32, max_downsample=2)
    assert [m.to_q.weight.shape[0] for m in pnp_attention_modules(small)] == [640] * 3 + [320] * 3
    assert pnp_attention_modules(make_skeleton("tiny", device="cpu", dtype=torch.float32)) == []
