"""KS, the sampling step's fused guidance combine and DDIM update, host side: ChunkedDenoiser's coefficient table against
the floats pred_next_x takes, the argument checks of vtm_cfg_ddim_update_f16 (which return before any CUDA call), and
which steps take the kernel path, with the ops calls stubbed in torch."""
from types import SimpleNamespace

import pytest
import torch

from vidtome_b200 import _lib, driver, ops
from vidtome_b200.driver import ChunkedDenoiser


class _Record:
    """Stands in for the latents and the noise in pred_next_x and records the python floats it is combined with."""

    def __init__(self, log):
        self.log = log

    def _scalar(self, v):
        assert isinstance(v, float)
        self.log.append(v)
        return self

    __rmul__ = __truediv__ = _scalar

    def __sub__(self, other):
        return self

    __add__ = __sub__


@pytest.mark.parametrize("n_timesteps", [10, 20, 50])
def test_coefficient_table_is_pred_next_x_floats(n_timesteps):
    den = ChunkedDenoiser(torch.nn.Identity(), n_timesteps=n_timesteps)
    coef, step = den.step_tables("cpu")
    assert coef.shape == (n_timesteps, 4) and coef.dtype == torch.float32
    assert step.dtype == torch.int32 and step.numel() == 1
    for i in range(n_timesteps):
        log = []
        den.pred_next_x(_Record(log), _Record(log), i)
        sigma, mu, mu_prev, sigma_prev = log                 # in pred_next_x's order of use
        assert den.coefficients(i) == (sigma, mu, mu_prev, sigma_prev)
        want = torch.tensor([sigma, 1.0 / mu, mu_prev, sigma_prev], dtype=torch.float32)
        assert torch.equal(coef[i], want), i
    ac = den.alphas_cumprod
    assert den.coefficients(n_timesteps - 1)[2] == float(den.final_alpha_cumprod ** 0.5) == float(ac[0] ** 0.5)
    assert den.step_tables("cpu")[0] is coef                 # made once: captured graphs hold its address


def test_entry_point_argument_errors():
    lib = _lib.load()
    ks = lib.vtm_cfg_ddim_update_f16
    p, q = 0x10000, 0x40000                                   # never dereferenced: every call below is refused first
    E_NULL, E_SHAPE = -1, -2
    #         x     eps   n    samples g    coef  step  steps out   stream
    assert ks(None, p, 100, 2, 7.5, p, p, 50, q, None) == E_NULL
    assert ks(p, None, 100, 2, 7.5, p, p, 50, q, None) == E_NULL
    assert ks(p, p, 100, 2, 7.5, None, p, 50, q, None) == E_NULL
    assert ks(p, p, 100, 2, 7.5, p, None, 50, q, None) == E_NULL
    assert ks(q, p, 100, 2, 7.5, p, p, 50, None, None) == E_NULL
    for samples in (-1, 0, 1, 4):
        assert ks(q, p, 100, samples, 7.5, p, p, 50, q, None) == E_SHAPE, samples
    assert ks(q, p, 0, 2, 7.5, p, p, 50, q, None) == E_SHAPE
    assert ks(q, p, -8, 3, 7.5, p, p, 50, q, None) == E_SHAPE
    assert ks(q, p, 100, 2, 7.5, p, p, 0, q, None) == E_SHAPE
    assert ks(q, p, 1 << 62, 3, 7.5, p, p, 50, q, None) == E_SHAPE         # eps's size overflows int64
    assert ks(q + 1, p, 100, 2, 7.5, p, p, 50, q + 1, None) == E_SHAPE      # fp16 pointers are 2-byte aligned
    assert ks(q, p + 1, 100, 2, 7.5, p, p, 50, q, None) == E_SHAPE
    assert ks(q, p, 100, 2, 7.5, p, p, 50, q + 1, None) == E_SHAPE
    assert ks(q, p, 100, 2, 7.5, p + 8, p, 50, q, None) == E_SHAPE          # the table is read as float4
    assert ks(q, p, 100, 2, 7.5, p + 4, p, 50, q, None) == E_SHAPE
    assert ks(q, p, 100, 2, 7.5, p, p + 2, 50, q, None) == E_SHAPE
    # out is x itself or apart from x and eps
    assert ks(q, p, 100, 2, 7.5, p, p, 50, q + 2, None) == E_SHAPE
    assert ks(q + 2, p, 100, 2, 7.5, p, p, 50, q, None) == E_SHAPE
    assert ks(q, p, 100, 2, 7.5, p, p, 50, p + 398, None) == E_SHAPE       # the last element of eps's 2 * 100
    assert ks(q, p, 100, 3, 7.5, p, p, 50, p + 400, None) == E_SHAPE       # inside eps's third block
    assert ks(p, p, 100, 2, 7.5, p, p, 50, p, None) == E_SHAPE             # in place on eps


def test_ops_wrapper_refuses_cpu_tensors():
    h = torch.zeros(2, 4, 8, dtype=torch.float16)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.cfg_ddim_update(h, torch.cat([h, h]), 2, 7.5, torch.zeros(1, 4), torch.zeros(1, dtype=torch.int32), h)


def _fake(is_cuda=True, dtype=torch.float16, contiguous=True):
    return SimpleNamespace(is_cuda=is_cuda, dtype=dtype, is_contiguous=lambda: contiguous)


def test_which_steps_fuse_the_update(monkeypatch):
    den = ChunkedDenoiser(torch.nn.Identity())
    sharded = ChunkedDenoiser(torch.nn.Identity(), shard=True)
    monkeypatch.setattr(driver, "FUSE_STEP_UPDATE", True)
    assert den._fuses_update(_fake())
    assert not sharded._fuses_update(_fake())                                # other ranks' frames: out of scope
    assert not den._fuses_update(_fake(is_cuda=False))
    assert not den._fuses_update(torch.zeros(2, 4, 8, 8, dtype=torch.float16))     # CPU latents
    for dtype in (torch.float32, torch.bfloat16, torch.float64):
        assert not den._fuses_update(_fake(dtype=dtype))
    assert not den._fuses_update(_fake(contiguous=False))
    monkeypatch.setattr(driver, "FUSE_STEP_UPDATE", False)
    assert not den._fuses_update(_fake())


class _Unet(torch.nn.Module):
    """A UNet stand-in whose output differs per sample and per frame, in `out_dtype`."""

    def __init__(self, out_dtype):
        super().__init__()
        self.out_dtype = out_dtype

    def forward(self, x, t, encoder_hidden_states=None, **kw):
        ramp = torch.arange(1, len(x) + 1, dtype=torch.float32).view(-1, 1, 1, 1)
        return SimpleNamespace(sample=(x.float() * 0.25 + ramp * 0.125 - float(t) / 1000).to(self.out_dtype))


def _steps(den, x, steps):
    out = []
    for i in range(steps):
        x = den.step(x, i)
        out.append(x)
    return out


@pytest.mark.parametrize("eps_dtype", [torch.float16, torch.float32])
def test_eager_fused_step_calls_the_kernel_per_chunk(monkeypatch, eps_dtype):
    """With the fused path forced on CPU and the kernels stubbed by torch ops, every chunk's rows go through KS (fp16 UNet
    output) or the torch guidance combine and KI (other dtypes), at the step index step() set, and the latents equal
    the torch path's bit for bit."""
    calls = []

    def ks(x, eps, samples, guidance, coef, step, out):
        s = int(step[0])
        calls.append(("KS", len(x), samples, s, eps.dtype))
        u, c = eps.chunk(samples)[-2:]
        out.copy_(den.pred_next_x(x, u + guidance * (c - u), s))

    def ki(x, eps, coef, step):
        s = int(step[0])
        calls.append(("KI", len(x), None, s, eps.dtype))
        x.copy_(den.pred_next_x(x, eps, s))

    torch.manual_seed(0)
    x0 = torch.randn(6, 4, 4, 4).half()
    monkeypatch.setattr(driver, "FUSE_STEP_UPDATE", False)
    den = ChunkedDenoiser(_Unet(eps_dtype), n_timesteps=5, chunk_size=4)
    want = _steps(den, x0, 3)
    monkeypatch.setattr(driver, "FUSE_STEP_UPDATE", True)
    monkeypatch.setattr(ChunkedDenoiser, "_fuses_update", lambda self, x: driver.FUSE_STEP_UPDATE)
    monkeypatch.setattr(ops, "cfg_ddim_update", ks)
    monkeypatch.setattr(ops, "ddim_update", ki)
    den = ChunkedDenoiser(_Unet(eps_dtype), n_timesteps=5, chunk_size=4)
    got = _steps(den, x0, 3)
    kind = "KS" if eps_dtype == torch.float16 else "KI"
    want_dtype = torch.float16                                               # KI gets the noise in the latents' dtype
    assert calls == [(kind, n, 2 if kind == "KS" else None, i, eps_dtype if kind == "KS" else want_dtype)
                     for i in range(3) for n in (4, 2)]
    for a, b in zip(want, got):
        assert torch.equal(a, b)
    calls.clear()
    monkeypatch.setattr(driver, "FUSE_STEP_UPDATE", False)                   # read at every eager step
    den.step(x0, 3)
    assert calls == []
