"""CPU emulation of GegluEpi's gelu (`gelu_x2` in csrc/linear.cu) over every finite fp16 gate.  The coefficients are read
from the source, so a refit is checked here before it reaches a GPU: every gate must be within one ulp of the correctly
rounded gelu, and zero wherever that is zero, allowing for ex2.approx's relative error of 2^-22 either way.  The
non-finite gates give what float64's g * Phi(g) and torch's erf form of gelu give: +inf at +inf, NaN at -inf and NaN."""
import os
import re

import pytest
import torch

SRC = os.path.join(os.path.dirname(__file__), "..", "vidtome_b200", "csrc", "linear.cu")


def _gelu_polynomial_source():
    """The coefficients and Horner steps of the polynomial: gelu_x2's body up to the ex2 of its result."""
    src = open(SRC).read()
    body = src[src.index("void gelu_x2("):]
    return body[:body.index("ex2_approx(")]


def _coefficients():
    body = _gelu_polynomial_source()
    coefs = [float(torch.tensor(float(c)).float()) for c in re.findall(r"(-?[0-9][0-9.e+-]*)f\b", body)]
    assert len(coefs) >= 3 and coefs[-1] == -1.0, coefs
    return coefs


def _f32(x):
    return x.float().double()


def _emulate(g, coefs, ex2_rel):
    """The kernel's fp32 steps for fp16 gates g (float64 tensor): FMAs rounded once, ex2 scaled by (1 + ex2_rel)."""
    t = g.abs()
    p = torch.full_like(t, coefs[0])
    for c in coefs[1:]:
        p = _f32(p * t + c)
    assert torch.isfinite(p[torch.isfinite(g)]).all(), "the polynomial overflows fp32"
    h = _f32(torch.exp2(p) * (1 + ex2_rel))
    gh = _f32(g * h)
    return torch.where(g >= 0, torch.where(h == 0, g, _f32(g - gh)), gh).float().half()


def _ordered(h):
    b = h.view(torch.int16).int()
    return torch.where(b < 0, -(b & 0x7FFF), b)


@pytest.mark.parametrize("ex2_rel", (0.0, 2.0 ** -22, -2.0 ** -22))
def test_gelu_polynomial_fit_within_one_ulp(ex2_rel):
    coefs = _coefficients()
    h = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16)
    g = h[torch.isfinite(h)].double()
    ref = (g * torch.special.ndtr(g)).numpy().astype("float16")   # numpy rounds float64 -> fp16 once
    ref = torch.from_numpy(ref)
    y = _emulate(g, coefs, ex2_rel)
    dist = (_ordered(y) - _ordered(ref)).abs()
    i = int(dist.argmax())
    assert dist[i] <= 1, f"gelu({g[i].item()!r}) = {y[i].item()!r}, correctly rounded {ref[i].item()!r}"
    # the flushed negative tail (near g = 0 a zero result sits at a rounding midpoint, where ex2's error decides)
    tail = (ref == 0) & (g < -1)
    assert (y[tail] == 0).all(), f"non-zero gelu at g = {g[tail][y[tail] != 0][:4].tolist()}"


def test_gelu_non_finite_gates():
    """g = +inf takes the positive branch with h = 0 and returns g itself (g - g h would be inf - NaN); -inf and NaN
    give NaN.  The kernel's branch on h == 0 is read from the source, so the emulation cannot drift from it."""
    src = open(SRC).read()
    body = src[src.index("void gelu_x2("):]
    assert "h0 == 0.f ? g0 : g0 - gh0" in body[:body.index("struct GegluEpi")], "gelu_x2's positive branch changed"
    g = torch.tensor([float("inf"), float("-inf"), float("nan")], dtype=torch.float64)
    y = _emulate(g, _coefficients(), 0.0).double()
    ref = g * torch.special.ndtr(g)
    assert y[0].item() == float("inf") and ref[0].item() == float("inf")
    assert torch.isnan(y[1:]).all() and torch.isnan(ref[1:]).all()
