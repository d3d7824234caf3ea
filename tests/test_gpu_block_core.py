"""The patched BasicTransformerBlock stage by stage against float64, with the block's own merge plan replayed, at the
production shapes of SD1.5 and SD2.1 and along every path the Python layer wires (merged, global stage, PnP, LoRA,
unmerged, Transformer2DModel).  Needs an H100.

The kernels are held to float64 one by one elsewhere (test_gpu_attention_core, test_gpu_projection_core,
test_gpu_rows_core, test_gpu_lora, test_gpu_transformer_io).  What this file checks is the composition: which rows each
kernel reads, which weight slice, bias, LoRA pair and residual it gets, which sample PnP shares, how many rows of a
capacity-sized buffer are live.  One call of a patched block runs with its call points wrapped (`_Capture`); every
stage's fp16 inputs and output are recorded, and each stage is compared with float64 from its own captured input:

    S0  GroupNorm -> tokens, proj_in             (Transformer2DModel entry)
    S1  norm1 fused into the merge gather        LN(h) at the plan's mu (and, with global tokens, its global map)
    S2  attn1 (KD / shared / device length)      softmax attention with the module's projections and LoRA
    S3  unmerge + residual (KE)                  RN16(attn[pi] + h), bit for bit
    S4  norm2 + attn2 + residual                 LN, then cross-attention over the context
    S5  norm3 + feed-forward + residual          LN, then GEGLU with the exact-erf gelu
    S6  proj_out storing NCHW + residual         (Transformer2DModel exit)

Bounds.  Every fp16 value a kernel stores is modelled as a storage point: its float64 centre is RN16 of the exact
value of the library's dataflow at that point, and its error is the distance to the furthest fp16 value the kernel may
store there, RN16 of the exact value +- the accumulated error bound (`_interval`).  The error bounds are the forward-error
forms of the core tests: c(K) sum |a||w| for the wgmma GEMMs (test_gpu_projection_core._linear_bound), the flash
kernel's bound relative to P|V| (test_gpu_attention_core._reference), the LayerNorm's delta
(test_gpu_rows_core._ln_reference); an upstream error e reaches a downstream value through |W| e.  A stage output must
lie in [RN16(z - e), RN16(z + e)] element by element, z the float64 value and e its bound: no max-norm tolerance.

Then the chain: each stage's captured input is bit-identical to the previous stage's captured output and the block's
return value is the last stage's output, so nothing runs between the stages unseen; and the whole block is recomputed
in float64 from its fp16 input with the plan's maps, reported as max-norm error relative to max|ref|.

The last tests put one deliberate wiring error at a time into the Python layer and require the stage check that names
it to fail."""
import contextlib
import dataclasses
import time

import pytest
import torch

import test_gpu_attention_core as ac
import test_gpu_projection_core as pc
import test_gpu_rows_core as rc
import test_gpu_transformer_io as tio
import vidtome_b200
from vidtome_b200 import attention, feedforward, lora, ops, patch, pnp
from vidtome_b200 import skeleton
from vidtome_b200.skeleton import (BasicTransformerBlock, LoRACompatibleLinear, ModelMixin, PeftLoraLinear,
                                   Transformer2DModel, add_lora)

pytestmark = pytest.mark.gpu

U = 2.0 ** -24             # unit roundoff of fp32
GELU_LIPSCHITZ = 1.13      # max |gelu'(x)| = 1.1289 (at x = sqrt(2))
STAGES = ("S0", "S1", "S2", "S3", "S4", "S5", "S6", "chain", "E2E")

# End-to-end max-norm error relative to max|ref|: 4.5e-4 ... 8.5e-4 over the cases below on an H100 (largest: sd21_h20_ds2,
# 8.54e-4), set mostly by the final fp16 rounding of outputs near max|ref|.  The bound leaves a margin of 2.3x.
E2E_LEVEL = 2e-3


class StageError(AssertionError):
    """One or more stage checks failed; `stage` is the first in STAGES order."""

    def __init__(self, failures):
        self.failures = failures
        self.stage = min(failures, key=lambda f: STAGES.index(f[0]))[0]
        super().__init__("\n".join(f"{s}: {m}" for s, m in failures))


# ---------------------------------------------------------------------------------------------------------------------
# float64 storage points and projections

def _interval(z, e):
    """The fp16 value a kernel stores for an fp32 result within e of z: (RN16(z), the furthest it can be from it)."""
    v, lo, hi = pc._round16(z), pc._round16(z - e), pc._round16(z + e)
    return v, torch.maximum(hi - v, v - lo)


def _terms(m):
    """(W, b, [(A, B, s), ...]) of a projection as its module defines it: an nn.Linear, diffusers' LoRACompatibleLinear
    (s = network_alpha / rank) or peft's lora.Linear (s = scaling[name] per active adapter).  Read here from the
    modules themselves, not through vidtome_b200.lora, so that the library's reading of them is under test."""
    if type(m) is torch.nn.Conv2d:                      # a 1x1 convolution: the Linear it computes
        return m.weight.view(m.weight.shape[0], -1), m.bias, []
    if isinstance(m, PeftLoraLinear):
        ads = [(m.lora_A[n].weight, m.lora_B[n].weight, m.scaling[n]) for n in m.active_adapters if n in m.lora_A]
        return m.base_layer.weight, m.base_layer.bias, ads
    if isinstance(m, LoRACompatibleLinear) and m.lora_layer is not None:
        ly = m.lora_layer
        s = 1.0 if ly.network_alpha is None else ly.network_alpha / ly.rank
        return m.weight, m.bias, [(ly.down.weight, ly.up.weight, s)]
    assert type(m) in (torch.nn.Linear, LoRACompatibleLinear), type(m)
    return m.weight, m.bias, []


def _stack(parts):
    """The terms of projections sharing one GEMM (q | k | v, or k | v): weights stacked, each adapter's up matrix
    padded with zero rows to the GEMM's width."""
    N = sum(w.shape[0] for w, _, _ in parts)
    W = torch.cat([w for w, _, _ in parts])
    b = None
    if any(p[1] is not None for p in parts):
        b = torch.cat([p[1] if p[1] is not None else torch.zeros_like(p[0][:, 0]) for p in parts])
    ads, n0 = [], 0
    for w, _, a in parts:
        for A, B, s in a:
            Bp = torch.zeros((N, B.shape[1]), dtype=B.dtype, device=B.device)
            Bp[n0:n0 + w.shape[0]] = B
            ads.append((A, Bp, s))
        n0 += w.shape[0]
    return W, b, ads


def _proj(x, ex, terms):
    """The library's projection of an fp16 operand known to lie within ex of x (float64 [M, K]; ex None: exactly x):
    T = RN16(x D^T) for the stacked LoRA down matrices D = RN16(A) (lora.pack), then the fp32 sum
    [x | T] [W | U]^T + b with U = RN16(fp32(s B)).  Returns (z, e): z the float64 value of that sum at the centres,
    e a bound on the distance of the kernel's fp32 result from z (before its fp16 rounding)."""
    W, b, ads = terms
    W = W.double()
    ax = x.abs() if ex is None else x.abs() + ex
    z = x @ W.t()
    e = 0.0 if ex is None else ex @ W.abs().t()
    a_cols, w_cols = [ax], [W.abs()]
    if ads:
        D = torch.cat([A.detach().half().double() for A, _, _ in ads])
        Uu = torch.cat([(B.detach().float() * s).half().double() for _, B, s in ads], 1)
        zT = x @ D.t()
        eT = pc._linear_bound(ax, D, None, zT)
        if ex is not None:
            eT = eT + ex @ D.abs().t()
        T, errT = _interval(zT, eT)
        z = z + T @ Uu.t()
        e = e + errT @ Uu.abs().t()
        a_cols.append(T.abs() + errT)
        w_cols.append(Uu.abs())
    e = e + pc._linear_bound(torch.cat(a_cols, 1), torch.cat(w_cols, 1), None, z)
    if b is not None:
        z = z + b.double()
        e = e + U * (z.abs() + e)
    return z, e


def _flash(q, eq, k, ek, v, ev, H, scale, shared=False):
    """softmax(q k^T scale) v per head in float64 at the centres q, k, v ([B, L, C], fp16 values) and a bound on the
    flash kernel's fp16 output for inputs within eq, ek, ev of them.  The kernel's own bound on its actual inputs is
    test_gpu_attention_core._reference's, which takes S = q k^T as exact; here S carries its fp32 wgmma error
    c(d) sum |q||k| and the inputs their deviations, so every score is within E_ij = scale (|q| ek + eq |k| + eq ek
    + c(d) |q||k|) of the centre's.  Scores off by at most E_i (the row's largest) move each weight by a factor within
    exp(+-2 E_i): with g = expm1(2 E_i) the output moves by at most g P|V| + (1 + g) P ev, and the kernel's bound grows
    by at most the factor 1 + g.  Returns (O, bound), each [B, Lq, C]."""
    B, Lq, C = q.shape
    Lk = k.shape[1]
    qh, eqh, kh, ekh, vh, evh = (ac._heads(t, H) for t in (q, eq, k, ek, v, ev))
    O, bnd = ac._reference(qh, kh, vh, scale, qk_shared=shared)
    if shared:
        qh, eqh = qh[:1].expand_as(qh), eqh[:1].expand_as(eqh)
        kh, ekh = kh[:1].expand_as(kh), ekh[:1].expand_as(ekh)
    d = qh.shape[-1]
    c = -(-d // 16) * 2.0 ** -23
    a = torch.cat([qh.abs(), eqh], -1)
    bm = torch.cat([ekh + c * kh.abs(), kh.abs() + ekh], -1).transpose(-1, -2)
    kt = kh.transpose(-1, -2)
    va = vh.abs()
    rows = max(1, (1 << 25) // (B * H * Lk))
    out = []
    for i0 in range(0, Lq, rows):
        sl = slice(i0, i0 + rows)
        s = (qh[:, :, sl] @ kt) * scale
        w = torch.exp(s - s.amax(-1, keepdim=True))
        l = w.sum(-1, keepdim=True)
        pv = (w @ va) / l
        pe = (w @ evh) / l
        g = torch.expm1(2 * abs(scale) * (a[:, :, sl] @ bm).amax(-1, keepdim=True))
        out.append((1 + g) * (bnd[:, :, sl] + pe) + g * (pv + pe))
    bound = torch.cat(out, 2)
    merge = lambda t: t.transpose(1, 2).reshape(B, Lq, C)
    return merge(O), merge(bound)


def _self_attention_bound(attn, x, shared=False):
    """attn1 on x [B, L, C] fp16: (z, e) of the out projection (before its fp16 rounding)."""
    B, L, C = x.shape
    z, e = _proj(x.double().reshape(B * L, C), None, _stack([_terms(attn.to_q), _terms(attn.to_k), _terms(attn.to_v)]))
    qkv, eqkv = (t.view(B, L, 3, C) for t in _interval(z, e))
    O, eo = _flash(qkv[:, :, 0], eqkv[:, :, 0], qkv[:, :, 1], eqkv[:, :, 1], qkv[:, :, 2], eqkv[:, :, 2],
                   int(attn.heads), float(attn.scale), shared)
    z, e = _proj(O.reshape(B * L, C), eo.reshape(B * L, C), _terms(attn.to_out[0]))
    return z.view(B, L, C), e.view(B, L, C)


def _cross_attention_bound(attn, x, ctx):
    B, L, C = x.shape
    Lk, Cc = ctx.shape[1:]
    zq, eq = _proj(x.double().reshape(B * L, C), None, _terms(attn.to_q))
    q, eq = (t.view(B, L, C) for t in _interval(zq, eq))
    zkv, ekv = _proj(ctx.double().reshape(B * Lk, Cc), None, _stack([_terms(attn.to_k), _terms(attn.to_v)]))
    kv, ekv = (t.view(B, Lk, 2, C) for t in _interval(zkv, ekv))
    O, eo = _flash(q, eq, kv[:, :, 0], ekv[:, :, 0], kv[:, :, 1], ekv[:, :, 1], int(attn.heads), float(attn.scale))
    z, e = _proj(O.reshape(B * L, C), eo.reshape(B * L, C), _terms(attn.to_out[0]))
    return z.view(B, L, C), e.view(B, L, C)


def _ff_bound(ff, n3):
    """GEGLU feed-forward on n3 [M, C] fp16: [a | g] stored in fp16 (GegluEpi), gelu(g) stored in fp16 within one ulp of
    the correctly rounded value (test_gpu_projection_core.test_geglu_gelu_exhaustive), their product stored in fp16,
    then the output projection.  Returns (z, e) of the output projection."""
    z, e = _proj(n3.double(), None, _terms(ff.proj))
    inner = z.shape[1] // 2
    a, ea = _interval(z[:, :inner], e[:, :inner])
    g, eg = _interval(z[:, inner:], e[:, inner:])
    G, eG = _interval(pc._gelu64(g), GELU_LIPSCHITZ * eg)
    eG = eG + pc._ulp16(G.abs() + eG)
    u, eu = _interval(a * G, G.abs() * ea + a.abs() * eG + ea * eG)
    return _proj(u, eu, _terms(ff.out))


def _within(y, z, e, what, resid=None):
    """y (fp16) in [RN16(z - e), RN16(z + e)], or with a residual added in the epilogue (fp16(fp16(acc) + resid), as
    the residual GEMMs round) in [RN16(RN16(z - e) + r), RN16(RN16(z + e) + r)].  Returns the largest |y - centre|
    relative to e + half an ulp (+ half an ulp of the sum with a residual): the fraction of the bound used."""
    lo, hi = pc._round16(z - e), pc._round16(z + e)
    used = e + pc._ulp16(z.abs() + e) / 2
    if resid is not None:
        r = resid.double()
        lo, hi = pc._round16(lo + r), pc._round16(hi + r)
        z = z + r
        used = used + pc._ulp16(z.abs() + e) / 2
    yd = y.double()
    bad = ~((yd >= lo) & (yd <= hi))
    if bad.any():
        i = tuple(torch.nonzero(bad)[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside [RN16(z - e), RN16(z + e)]; "
                             f"first at {i}: y = {yd[i].item()!r}, interval [{lo[i].item()!r}, {hi[i].item()!r}], "
                             f"z = {z[i].item()!r}")
    return ((yd - z).abs() / used).max().item()


# ---------------------------------------------------------------------------------------------------------------------
# float64 block

def _lin64(x, m):
    W, b, ads = _terms(m)
    y = x @ W.double().t()
    if b is not None:
        y = y + b.double()
    for A, B, s in ads:
        y = y + s * ((x @ A.double().t()) @ B.double().t())
    return y


def _ln64(x, norm):
    return torch.nn.functional.layer_norm(x, x.shape[-1:], norm.weight.double(),
                                          None if norm.bias is None else norm.bias.double(), norm.eps)


def _attn64(attn, x, ctx=None, shared=False):
    kv = x if ctx is None else ctx
    H = int(attn.heads)
    q, k, v = (ac._heads(_lin64(t, m), H) for t, m in ((x, attn.to_q), (kv, attn.to_k), (kv, attn.to_v)))
    if shared:
        q, k = q[:1].expand_as(q), k[:1].expand_as(k)
    B, _, L, _ = q.shape
    rows = max(1, (1 << 25) // (B * H * k.shape[2]))
    o = torch.cat([torch.softmax((q[:, :, i:i + rows] @ k.transpose(-1, -2)) * attn.scale, -1) @ v
                   for i in range(0, L, rows)], 2)
    return _lin64(o.transpose(1, 2).reshape(B, L, -1), attn.to_out[0])


def _block64(blk, h, ctx, maps):
    """The block in float64 from its input h [(B F), T, C] (fp16, or float64 inside the float64 Transformer2DModel),
    with the plan's maps (None: unmerged)."""
    hd = h.double()
    n1 = _ln64(hd, blk.norm1)
    if maps is None:
        h1 = _attn64(blk.attn1, n1) + hd
    else:
        B = maps["B"]
        merged = rc._gather(n1.reshape(B, -1, n1.shape[-1]), maps["mu"])
        if maps.get("mu_g") is not None:
            cat = torch.cat([merged, maps["store"].double()], 1)
            merged = rc._gather(cat, maps["mu_g"][:, :maps["M"]])
        a = _attn64(blk.attn1, merged, shared=maps["shared"])
        h1 = rc._gather(a, maps["pi"]).reshape(h.shape) + hd
    h2 = _attn64(blk.attn2, _ln64(h1, blk.norm2), ctx.double()) + h1
    up = _lin64(_ln64(h2, blk.norm3), blk.ff.proj)
    a, g = up.chunk(2, -1)
    return _lin64(a * pc._gelu64(g), blk.ff.out) + h2


def _group_norm64(x, norm):
    n, C, hh, ww = x.shape
    G = norm.num_groups
    xd = x.double().view(n, G, -1)
    mean, var = xd.mean(-1, keepdim=True), xd.var(-1, unbiased=False, keepdim=True)
    t = ((xd - mean) / torch.sqrt(var + norm.eps)).view(n, C, hh * ww)
    return t * norm.weight.double()[:, None] + norm.bias.double()[:, None]


# ---------------------------------------------------------------------------------------------------------------------
# capture

def _snap(v):
    return v.detach().clone() if isinstance(v, torch.Tensor) else v


def _bits(t):
    return t.detach().contiguous().view(torch.int16).flatten()


class _Capture:
    """Wraps the call points of the Python layer and records every call's arguments and result (tensors cloned)."""

    POINTS = ((patch, "build_merge_plan", "plan"), (attention, "self_attention", "attn1"),
              (attention, "self_attention_residual", "attn1r"), (patch.MergePlan, "unmerge_add", "unmerge"),
              (attention, "cross_attention_residual", "attn2"), (ops, "layer_norm", "ln"),
              (feedforward, "feed_forward_residual", "ff"), (ops, "group_norm_tokens", "gn"), (ops, "linear", "proj_in"),
              (ops, "linear_nchw_residual", "proj_out"), (ops, "gather_rows_dev", "gather_dev"),
              (skeleton.Attention, "forward", "module_attn"))

    def __init__(self, mp):
        self.rec = {key: [] for _, _, key in self.POINTS}
        for owner, name, key in self.POINTS:
            self._wrap(mp, owner, name, key)

    def _wrap(self, mp, owner, name, key):
        orig = getattr(owner, name)
        rec = self.rec[key]

        def wrapper(*args, **kwargs):
            entry = {"args": [_snap(a) for a in args], "kwargs": {k: _snap(v) for k, v in kwargs.items()}}
            out = orig(*args, **kwargs)
            if key == "plan" and out is not None:
                entry["plan"] = dataclasses.replace(out, merged_tokens=_snap(out.merged_tokens), pi=_snap(out.pi),
                                                    mu=_snap(out.mu), seq_len=_snap(out.seq_len), coin=_snap(out.coin))
            entry["out"] = _snap(out) if key != "plan" else None
            rec.append(entry)
            return out
        mp.setattr(owner, name, wrapper)

    def one(self, key):
        assert len(self.rec[key]) == 1, f"{key}: {len(self.rec[key])} calls, expected one"
        return self.rec[key][0]

    def ln_of(self, norm):
        hits = [e for e in self.rec["ln"] if e["args"][1][0].data_ptr() == norm.weight.data_ptr()]
        assert len(hits) == 1, f"{len(hits)} LayerNorm calls with the weight of {norm}"
        return hits[0]


# ---------------------------------------------------------------------------------------------------------------------
# cases

@dataclasses.dataclass
class Case:
    C: int
    heads: int
    latent: int                   # latent side; the block runs at latent / ds
    ds: int
    frames: int
    batch: int = 2
    cad: int = 768                # context width
    lora: str = None
    ratio: float = 0.9
    max_downsample: int = 2
    wide: bool = True             # attention.MAX_HEAD_DIM = 160
    path: str = "merged"          # merged, unmerged, global, pnp
    global_rand: float = 0.5
    t2d: str = None               # Transformer2DModel around the block: "conv" or "linear"
    seed: int = 0

    @property
    def T(self):
        return (self.latent // self.ds) ** 2


CASES = {
    # SD1.5: 8 heads of 40 / 80 / 160
    "sd15_c320_ds1": Case(320, 8, 64, 1, frames=8),
    "sd15_c640_ds2": Case(640, 8, 64, 2, frames=4),
    "sd15_c1280_ds4": Case(1280, 8, 64, 4, frames=8, max_downsample=8),
    "sd15_c1280_ds8": Case(1280, 8, 64, 8, frames=8, max_downsample=8),
    # head_dim 160 above the default MAX_HEAD_DIM (128): attn1 and attn2 run their module forwards (torch), the merge,
    # the unmerge and the feed-forward run in the library
    "sd15_c1280_ds4_default_limit": Case(1280, 8, 64, 4, frames=8, max_downsample=8, wide=False),
    # SD2.1: heads of 64, 1024-wide context
    "sd21_h5_ds1": Case(320, 5, 96, 1, frames=2, batch=1, cad=1024),
    "sd21_h10_ds2": Case(640, 10, 96, 2, frames=4, cad=1024),
    "sd21_h20_ds2": Case(1280, 20, 96, 2, frames=2, cad=1024),
    # chunk shapes
    "frames8_b2": Case(320, 8, 32, 1, frames=8),
    "frames5": Case(640, 8, 32, 2, frames=5),
    "frames1": Case(320, 8, 32, 1, frames=1),
    "ratio1": Case(320, 8, 32, 1, frames=4, ratio=1.0),
    # global stage through a GlobalTokenStore, both coin branches: coin > 0 (local tokens src), coin <= 1 (global src)
    "global_local_src": Case(320, 8, 16, 1, frames=4, path="global", global_rand=0.0),
    "global_global_src": Case(320, 8, 16, 1, frames=4, path="global", global_rand=1.0),
    # PnP: three aligned samples, sample 0's attention map shared
    "pnp": Case(320, 8, 32, 1, frames=4, batch=3, path="pnp"),
    # LoRA on attn1 / attn2 / ff
    "lora_diffusers": Case(320, 8, 32, 1, frames=4, lora="diffusers"),
    "lora_peft": Case(640, 8, 32, 2, frames=4, lora="peft"),
    # unmerged (inversion): norm1 -> KD with the residual in its out projection
    "unmerged": Case(640, 8, 32, 1, frames=2, path="unmerged"),
    # Transformer2DModel around the block
    "t2d_conv": Case(320, 8, 32, 1, frames=4, t2d="conv"),
    "t2d_linear": Case(640, 10, 24, 1, frames=2, cad=1024, t2d="linear"),
}


def _make(case):
    """(net, block): a patched one-block model with parameters drawn so that every bias, affine and eps takes a visible
    part: biases of std 0.5, LayerNorm affines around (1, 0) and eps of 1e-3, 2e-2, 5e-3 (so that an eps mixed up with
    another norm's, or with the 1e-5 default, moves the normalised rows by far more than an fp16 rounding)."""
    torch.manual_seed(case.seed + case.C + case.heads)
    blk = BasicTransformerBlock(case.C, case.heads, case.cad, hot_path_only=False)
    with torch.no_grad():
        for name, p in blk.named_parameters():
            if name.endswith("bias"):
                p.normal_(0.0, 0.5)
        for norm, eps in ((blk.norm1, 1e-3), (blk.norm2, 2e-2), (blk.norm3, 5e-3)):
            norm.weight.normal_(1.0, 0.2)
            norm.eps = eps
        if case.path == "global":
            # every live key scores well below zero against every query, so that a key read past the live length
            # (a zero row, score 0) would take most of each softmax
            blk.attn1.to_q.weight.mul_(2.0)
            blk.attn1.to_k.weight.copy_(-blk.attn1.to_q.weight)

    class Net(ModelMixin):
        def __init__(self):
            super().__init__()
            self.block = blk
            self.wrap = None if case.t2d is None else Transformer2DModel(case.C, blk,
                                                                         use_linear_projection=case.t2d == "linear")

        def forward(self, latent, x, ctx):                  # the model's pre-hook reads the latent size from `latent`
            if self.wrap is not None:
                return self.wrap(x, encoder_hidden_states=ctx).sample
            return self.block(x, encoder_hidden_states=ctx)

    net = Net().cuda().half().eval()
    if case.lora:
        add_lora(net, 16, case.lora)
    vidtome_b200.apply_patch(net, local_merge_ratio=case.ratio, batch_size=case.batch, max_downsample=case.max_downsample,
                             merge_global=case.path == "global", global_merge_ratio=0.8, global_rand=case.global_rand,
                             align_batch=case.path == "pnp")
    if case.path == "global":
        blk.global_tokens = patch.GlobalTokenStore(case.frames + 2)
    if case.path == "pnp":
        pnp.register_attention_control(net, [981], case.batch, modules=[blk.attn1])
        pnp.register_time(net, 981, modules=[blk.attn1])
    return net, blk


def _inputs(case, g):
    """Video-like fp16 hidden states: one direction common to every token, one pattern per sample repeated over the
    frames, and per-frame noise; a random context per frame."""
    n = case.batch * case.frames
    base = torch.randn((case.batch, 1, case.T, case.C), generator=g, device="cuda")
    dc = torch.randn((case.C,), generator=g, device="cuda")
    h = dc + base + 0.5 * torch.randn((case.batch, case.frames, case.T, case.C), generator=g, device="cuda")
    h = h.reshape(n, case.T, case.C).half()
    ctx = torch.randn((n, 77, case.cad), generator=g, device="cuda").half()
    if case.t2d is not None:
        side = case.latent // case.ds
        h = h.transpose(1, 2).reshape(n, case.C, side, side).contiguous()
    return h, ctx


def _latent(case):
    """A stand-in latent of the case's size: the model's pre-hook reads only its spatial shape."""
    return torch.empty((1, 4, case.latent, case.latent), dtype=torch.float16, device="cuda")


# ---------------------------------------------------------------------------------------------------------------------
# the stage checks

def _run(name, monkeypatch, mutate=None, report=None):
    """Runs one call of the patched block of CASES[name] under capture and checks every stage.  mutate(mp, blk) installs a
    wiring error first.  Raises StageError naming the failing stages; returns {stage: slack} otherwise."""
    case = CASES[name]
    net, blk = _make(case)
    g = torch.Generator(device="cuda").manual_seed(case.seed + 17)
    h, ctx = _inputs(case, g)
    store = None
    with monkeypatch.context() as mp:
        mp.setattr(attention, "MAX_HEAD_DIM", 160 if case.wide else 128)
        if mutate is not None:
            mutate(mp, blk)
        with torch.no_grad():
            if case.path == "global":
                # the first chunk fills the store; the second runs the global stage against it
                torch.manual_seed(case.seed)
                net(_latent(case), *_inputs(case, g))
                store = blk.global_tokens
                live = int(store.length.item())
                assert store.filled and live < store.cap
                store.tokens[:, live:] = float("nan")           # rows past the live length must never be read
                store_before = store.tokens.clone()
            torch.manual_seed(case.seed + 1)
            rec = _Capture(mp)
            with patch._unmerged_blocks() if case.path == "unmerged" else contextlib.nullcontext():
                out = net(_latent(case), h, ctx)
        torch.cuda.synchronize()
    failures, slack = [], {}

    def check(stage, fn):
        try:
            r = fn()
            if r is not None:
                slack[stage] = max(slack.get(stage, 0.0), r)
        except (AssertionError, pytest.fail.Exception) as e:
            failures.append((stage, str(e).splitlines()[0] if str(e) else repr(e)))

    C = case.C
    what = lambda s: f"{name} {s}"

    # ---------------------------------------------------------------- S0 / S6: the Transformer2DModel entry and exit
    if case.t2d is not None:
        gn, pin, pout = rec.one("gn"), rec.one("proj_in"), rec.one("proj_out")
        wrap = net.wrap

        def s0():
            x = gn["args"][0]
            want = _group_norm64(x, wrap.norm).transpose(1, 2)
            n, _, hh, ww = x.shape
            G = wrap.norm.num_groups
            xd = x.double().view(n, G, -1)
            mean = xd.mean(-1)
            var = xd.var(-1, unbiased=False)
            rstd = 1 / torch.sqrt(var + wrap.norm.eps)
            # the statistics' error bounds of test_gpu_transformer_io._check_stats, then the normalisation's fp32 steps
            steps = tio._stats_steps(xd.shape[-1], n * G)
            e_mean = steps * 4 * U * xd.abs().amax(-1) + U * mean.abs()
            e_var = steps * 8 * U * var + 4 * (xd - mean[..., None]).abs().amax(-1) * e_mean + e_mean ** 2
            e_rstd = 0.5 * rstd ** 3 * e_var * 1.01 + 4 * U * rstd
            cpg = C // G
            rep = lambda t: t.repeat_interleave(cpg, 1)[:, :, None]
            t = (x.double().view(n, C, -1) - rep(mean)) * rep(rstd)
            gam = wrap.norm.weight.double().abs()[None, :, None]
            e = gam * (rep(e_mean) * rep(rstd) + (t.abs() / rep(rstd)) * rep(e_rstd))
            e = (e + 2 * U * t.abs() * gam + U * want.transpose(1, 2).abs()) * 1.01
            r = _within(gn["out"], want, e.transpose(1, 2), what("S0 GroupNorm -> tokens"))
            z, e2 = _proj(gn["out"].double().reshape(-1, C), None, _terms(wrap.proj_in))
            return max(r, _within(pin["out"], z, e2, what("S0 proj_in")))

        def s6():
            t, w, b, x, hw = pout["args"]
            z, e = _proj(t.double(), None, _terms(wrap.proj_out))
            n = x.shape[0]
            z, e = (v.view(n, -1, C).transpose(1, 2).reshape(x.shape) for v in (z, e))
            return _within(pout["out"], z, e, what("S6 proj_out + residual"), resid=x)
        check("S0", s0)
        check("S6", s6)

    # ------------------------------------------------------------------------------------------- the block's stages
    plan_e = rec.rec["plan"][0] if rec.rec["plan"] else None
    plan = None if plan_e is None else plan_e["plan"]
    if case.path == "unmerged":
        assert plan_e is None, "a merge plan was built inside _unmerged_blocks()"
        ln1, a1 = rec.ln_of(blk.norm1), rec.one("attn1r")
        h_in = ln1["args"][0].view(-1, case.T, C)
        check("S1", lambda: rc._check_ln(ln1["out"], ln1["args"][0], (blk.norm1.weight, blk.norm1.bias, blk.norm1.eps),
                                         what("S1 norm1")) and None)

        def s2u():
            z, e = _self_attention_bound(blk.attn1, a1["args"][1])
            return _within(a1["out"], z, e, what("S2 attn1 + residual"), resid=a1["args"][2])
        check("S2", s2u)
        h1 = a1["out"]
    else:
        assert plan is not None, "no merge plan"
        h_in = plan_e["args"][1]
        B = plan.merged_tokens.shape[0]
        table = h_in.reshape(B, -1, C)
        n1 = (blk.norm1.weight, blk.norm1.bias, blk.norm1.eps)
        M = plan.merged_tokens.shape[1] if plan.seq_len is None else int(plan.seq_len.item())
        mu_g = None
        if case.path == "global":
            gd = rec.one("gather_dev")
            mu_g = gd["args"][1].long().expand(B, -1)
            assert int(gd["args"][2].item()) == M
            assert (plan.coin.item() > case.global_rand) == (case.global_rand < 0.5), "not the intended coin branch"

        def s1():
            src = rc._gather(table, plan.mu)
            y = plan.merged_tokens
            if mu_g is None:
                rc._check_ln(y, src, n1, what("S1 norm1 + merge gather"))
                return None
            L = src.shape[1]
            x = rc._gather(torch.cat([src, store_before], 1), mu_g[:, :M])
            loc = (mu_g[:, :M] < L)
            rc._check_ln(y[:, :M][loc], x[loc], n1, what("S1 norm1 + merge gather, local rows"))
            assert torch.equal(_bits(y[:, :M][~loc]), _bits(x[~loc])), what("S1 global rows are not the stored rows")
            assert (_bits(y[:, M:]) == 0).all(), what("S1 rows past the merged length are not +0")
        check("S1", s1)

        if case.wide or C // case.heads <= 128:
            a1 = rec.one("attn1")
            assert all(e["args"][0] is not blk.attn1 for e in rec.rec["module_attn"]), "attn1 ran its module forward"
            shared = bool(a1["kwargs"].get("shared_qk", False))
            assert shared == (case.path == "pnp"), f"shared_qk = {shared}"
            assert (a1["kwargs"].get("seq_len") is None) == (plan.seq_len is None)

            def s2():
                assert torch.equal(_bits(a1["args"][1]), _bits(plan.merged_tokens)), "KD's input is not the plan's"
                z, e = _self_attention_bound(blk.attn1, a1["args"][1][:, :M], shared)
                return _within(a1["out"][:, :M], z, e, what("S2 attn1"))
            check("S2", s2)
            y1 = a1["out"]
        else:
            # head_dim 160 above MAX_HEAD_DIM: attn1 runs its module forward (torch), which is what S2 then is
            mods = [e for e in rec.rec["module_attn"] if e["args"][0] is blk.attn1]
            assert len(mods) == 1 and not rec.rec["attn1"], "attn1 did not run its module forward"
            y1 = mods[0]["out"]

            def s2t():
                assert torch.equal(_bits(mods[0]["args"][1]), _bits(plan.merged_tokens))
                with torch.no_grad():
                    again = type(blk.attn1).forward(blk.attn1, mods[0]["args"][1])
                assert torch.equal(_bits(again), _bits(y1)), "attn1's module forward is not torch's"
            check("S2", s2t)

        un = rec.one("unmerge")

        def s3():
            pi = plan.pi.long()
            assert int(pi.max()) < M, "the unmerge map reads rows past the merged length"
            assert torch.equal(_bits(un["args"][1]), _bits(y1)), "KE's input is not attn1's output"
            resid = h_in.reshape(B, -1, C)
            want = rc._sum16(rc._gather(un["args"][1], pi), resid)
            rc._assert_same(un["out"].reshape(B, -1, C), want, what("S3 unmerge + residual"))
        check("S3", s3)
        h1 = un["out"]

    # norm2 + attn2 + residual
    if case.wide or C // case.heads <= 128:
        ln2, a2 = rec.ln_of(blk.norm2), rec.one("attn2")
        check("S4", lambda: rc._check_ln(ln2["out"], ln2["args"][0], (blk.norm2.weight, blk.norm2.bias, blk.norm2.eps),
                                         what("S4 norm2")) and None)

        def s4():
            _, x, c, r = a2["args"]
            z, e = _cross_attention_bound(blk.attn2, x, c)
            return _within(a2["out"], z, e, what("S4 attn2 + residual"), resid=r)
        check("S4", s4)
        h2 = a2["out"]
        chain4 = [("norm2 input", ln2["args"][0], h1), ("attn2 queries", a2["args"][1], ln2["out"]),
                  ("attn2 residual", a2["args"][3], h1), ("attn2 context", a2["args"][2], ctx)]
    else:
        mods = [e for e in rec.rec["module_attn"] if e["args"][0] is blk.attn2]
        assert len(mods) == 1 and not rec.rec["attn2"], "attn2 did not run its module forward"

        def s4t():
            with torch.no_grad():
                want = type(blk.attn2).forward(blk.attn2, blk.norm2(h1), encoder_hidden_states=ctx) + h1
            assert torch.equal(_bits(want), _bits(ff_e["args"][3])), "norm2 + attn2 + residual is not torch's"
        ff_e = rec.one("ff")
        check("S4", s4t)
        h2 = ff_e["args"][3]
        chain4 = []

    # norm3 + feed-forward + residual
    ff_e = rec.one("ff")
    ln3 = rec.ln_of(blk.norm3)
    check("S5", lambda: rc._check_ln(ln3["out"], ln3["args"][0], (blk.norm3.weight, blk.norm3.bias, blk.norm3.eps),
                                     what("S5 norm3")) and None)

    def s5():
        z, e = _ff_bound(blk.ff, ln3["out"])
        hs = ff_e["args"][3]
        return _within(ff_e["out"].reshape(-1, C), z, e, what("S5 feed-forward + residual"), resid=hs.reshape(-1, C))
    check("S5", s5)
    h3 = ff_e["out"]

    # ------------------------------------------------------------------------------------------------------ chain
    def chain():
        links = list(chain4) + [("feed-forward input", ff_e["args"][3], h2), ("norm3 input", ln3["args"][0], h2)]
        if case.path != "unmerged":
            links += [("unmerge residual", un["args"][2], h_in)]
        else:
            links += [("attn1 residual", a1["args"][2], h_in), ("attn1 input", a1["args"][1], ln1["out"])]
        if case.t2d is None:
            links += [("block input", h_in, h), ("block output", out, h3)]
        else:
            links += [("proj_in input", pin["args"][0], gn["out"]), ("block input", h_in, pin["out"]),
                      ("proj_out input", pout["args"][0], h3), ("proj_out residual", pout["args"][3], h),
                      ("GroupNorm input", gn["args"][0], h), ("wrapper output", out, pout["out"])]
        for name, got, want in links:
            assert got.numel() == want.numel() and torch.equal(_bits(got), _bits(want)), f"{name} differs"
    check("chain", chain)

    # ------------------------------------------------------------------------------------------------ end to end
    rel = None

    def e2e():
        nonlocal rel
        maps = None
        if case.path != "unmerged":
            maps = dict(B=B, mu=plan.mu, pi=plan.pi, shared=case.path == "pnp", mu_g=mu_g, M=M,
                        store=store_before if case.path == "global" else None)
        if case.t2d is None:
            ref = _block64(blk, h, ctx, maps)
        else:
            wrap = net.wrap
            n, _, hh, ww = h.shape
            tok = _group_norm64(h, wrap.norm).transpose(1, 2)
            t = _block64(blk, _lin64(tok, wrap.proj_in), ctx, maps)
            ref = _lin64(t, wrap.proj_out).transpose(1, 2).reshape(h.shape) + h.double()
        assert torch.isfinite(out).all(), "non-finite output"
        rel = (out.double() - ref).abs().max().item() / ref.abs().max().item()
        assert rel <= E2E_LEVEL, f"{name} end to end: max-norm error {rel:.3e} of max|ref| > {E2E_LEVEL:.1e}"
    check("E2E", e2e)
    if report is not None:
        report.update(slack=slack, e2e=rel)
    if failures:
        raise StageError(failures)
    return slack


# ---------------------------------------------------------------------------------------------------------------------
# the matrix

@pytest.mark.parametrize("name", list(CASES))
def test_block_stages(name, monkeypatch):
    case = CASES[name]
    t0 = time.perf_counter()
    report = {}
    calls = {}
    orig = ops.attention

    def counting(*a, **k):
        calls["kd"] = calls.get("kd", 0) + 1
        return orig(*a, **k)
    monkeypatch.setattr(ops, "attention", counting)
    _run(name, monkeypatch, report=report)
    if case.path != "unmerged":
        # the library's KD ran for this block (no fallback): one call (two for the global stage: the store fill too);
        # none where head_dim 160 is above MAX_HEAD_DIM
        want = 0 if not case.wide and case.C // case.heads > 128 else 2 if case.path == "global" else 1
        assert calls.get("kd", 0) == want, calls
    slack = " ".join(f"{s}={v:.2f}" for s, v in sorted(report["slack"].items()))
    print(f"{name}: end-to-end max-norm error {report['e2e']:.3e} of max|ref|; largest |y - z| / (e + ulp / 2) "
          f"per stage: {slack}; {time.perf_counter() - t0:.1f} s")


# ---------------------------------------------------------------------------------------------------------------------
# the harness catches wiring errors

def _roll_pi(mp, blk):
    orig = patch.MergePlan.unmerge_add

    def mutated(self, y, h):
        pi = self.pi.expand(y.shape[0], -1).clone()
        pi[1] = torch.roll(pi[1], 1)
        return orig(dataclasses.replace(self, pi=pi.contiguous()), y, h)
    mp.setattr(patch.MergePlan, "unmerge_add", mutated)


def _drop_b_o(mp, blk):
    orig = ops.attention
    mp.setattr(ops, "attention", lambda x, w_qkv, w_o, b_o, *a, **k: orig(x, w_qkv, w_o, None, *a, **k))


def _lora_scale_1(mp, blk):
    orig = lora._adapter
    mp.setattr(lora, "_adapter", lambda a, b, s, w: orig(a, b, 1.0, w))


def _seq_len_plus_1(mp, blk):
    orig = attention.self_attention

    def mutated(attn, x, shared_qk=False, seq_len=None):
        return orig(attn, x, shared_qk=shared_qk, seq_len=None if seq_len is None else seq_len + 1)
    mp.setattr(attention, "self_attention", mutated)


def _pnp_source_1(mp, blk):
    orig = attention.self_attention

    def mutated(attn, x, shared_qk=False, seq_len=None):
        if not shared_qk:
            return orig(attn, x, shared_qk=shared_qk, seq_len=seq_len)
        perm = [1, 0] + list(range(2, x.shape[0]))          # its own inverse
        return orig(attn, x[perm].contiguous(), shared_qk=True, seq_len=seq_len)[perm].contiguous()
    mp.setattr(attention, "self_attention", mutated)


def _norm2_eps(mp, blk):
    orig = patch._fusable_layer_norm

    def mutated(norm, x):
        r = orig(norm, x)
        return (r[0], r[1], 1e-5) if r is not None and norm is blk.norm2 else r
    mp.setattr(patch, "_fusable_layer_norm", mutated)


MUTATIONS = {
    "pi_rolled_for_item_1": ("sd15_c640_ds2", _roll_pi, "S3"),
    "kd_without_b_o": ("sd15_c640_ds2", _drop_b_o, "S2"),
    "lora_scale_1": ("lora_peft", _lora_scale_1, "S2"),
    "seq_len_plus_1": ("global_local_src", _seq_len_plus_1, "S2"),
    "pnp_source_sample_1": ("pnp", _pnp_source_1, "S2"),
    "norm2_eps_1e-5": ("sd15_c640_ds2", _norm2_eps, "S4"),
}


@pytest.mark.parametrize("name", list(MUTATIONS))
def test_harness_catches(name, monkeypatch):
    case_key, mutate, stage = MUTATIONS[name]
    with pytest.raises(StageError) as info:
        _run(case_key, monkeypatch, mutate=mutate)
    assert info.value.stage == stage, f"first failing stage {info.value.stage}, expected {stage}:\n{info.value}"
