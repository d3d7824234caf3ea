"""LoRA-adapted projections, host side (no GPU): which wrapped layers the library reads (lora.linear_parts), the
stacked down / up matrices (lora.pack) against the modules' own forward in float64, the caches on the modules, and the
dispatch rules that let LoRA-adapted attention and feed-forward modules run in the library."""
import copy

import pytest
import torch
import torch.nn as nn

from vidtome_b200 import attention, feedforward, lora, patch
from vidtome_b200.skeleton import (Attention, BasicTransformerBlock, LoRACompatibleLinear, LoRALinearLayer,
                                   PeftLoraLinear, add_lora)


def _block(seed=0, dtype=torch.float16):
    torch.manual_seed(seed)
    return BasicTransformerBlock(64, 2, cross_attention_dim=32, hot_path_only=False).to(dtype)


def _peft(K=64, N=48, names=(("a", 8, 4.0),), dtype=torch.float16, adapter_dtype=None, seed=0):
    torch.manual_seed(seed)
    m = PeftLoraLinear(nn.Linear(K, N).to(dtype))
    for name, r, alpha in names:
        m.update_layer(name, r, alpha)
        nn.init.normal_(m.lora_B[name].weight)
    m.lora_A.to(adapter_dtype or dtype)
    m.lora_B.to(adapter_dtype or dtype)
    return m


def _diffusers(K=64, N=48, r=8, alpha=4.0, dtype=torch.float16, adapter_dtype=None, seed=0):
    torch.manual_seed(seed)
    layer = LoRALinearLayer(K, N, r, network_alpha=alpha)
    nn.init.normal_(layer.up.weight)
    m = LoRACompatibleLinear(K, N, lora_layer=layer).to(dtype)
    layer.to(adapter_dtype or dtype)
    return m


# ---------------------------------------------------------------------------------------------------------------------
# recognition and refusal

def test_plain_linear_has_no_adapters():
    m = nn.Linear(16, 24)
    w, b, ads = lora.linear_parts(m)
    assert w is m.weight and b is m.bias and ads == []
    assert lora.pack([lora.linear_parts(m)], "cpu") is None


def test_diffusers_form():
    m = _diffusers(alpha=4.0)
    w, b, ads = lora.linear_parts(m)
    assert w is m.weight and b is m.bias and len(ads) == 1
    A, B, s = ads[0]
    assert A is m.lora_layer.down.weight and B is m.lora_layer.up.weight and s == 4.0 / 8
    m.lora_layer.network_alpha = None
    assert lora.linear_parts(m)[2][0][2] == 1.0
    m.lora_layer = None
    assert lora.linear_parts(m)[2] == []


def test_peft_form_and_adapter_selection():
    m = _peft(names=(("a", 8, 4.0), ("b", 16, 32.0), ("c", 8, 8.0)))
    m.set_adapter(["a", "b", "missing"])                # a name without weights in this layer is skipped, as peft does
    w, b, ads = lora.linear_parts(m)
    assert w is m.base_layer.weight and b is m.base_layer.bias
    assert [(A.shape[0], s) for A, _, s in ads] == [(8, 0.5), (16, 2.0)]
    m._disable_adapters = True
    assert lora.linear_parts(m)[2] == []
    m._disable_adapters = False
    m.merged_adapters = ["a"]
    assert lora.linear_parts(m)[2] == []
    m._disable_adapters = True                          # peft unmerges out of the base weight first: not ours to compute
    assert lora.linear_parts(m) is None


def _refused(m, what):
    assert lora.linear_parts(m) is None, what


def test_refusals():
    m = _peft(); m.use_dora["a"] = True; _refused(m, "DoRA")
    m = _peft(); m.lora_bias["a"] = True; _refused(m, "lora_bias flag")
    m = _peft(); m.lora_B["a"] = nn.Linear(8, 48, bias=True).half(); _refused(m, "lora_B with a bias")
    m = _peft(); m.lora_dropout["a"] = nn.Dropout(0.1); m.train(); _refused(m, "dropout in training")
    m = _peft(); m.lora_dropout["a"] = nn.Dropout(0.1); m.eval()
    assert lora.linear_parts(m) is not None, "inactive dropout"
    m = _peft(); m.fan_in_fan_out = True; _refused(m, "fan_in_fan_out")
    m = _peft(); m.base_layer = LoRACompatibleLinear(64, 48).half(); _refused(m, "base layer not an exact Linear")
    for sub in ("self", "base", "A", "B", "drop"):
        for kind in ("hook", "pre_hook", "forward"):
            m = _peft()
            tgt = {"self": m, "base": m.base_layer, "A": m.lora_A["a"], "B": m.lora_B["a"], "drop": m.lora_dropout["a"]}[sub]
            if kind == "hook":
                tgt.register_forward_hook(lambda mod, i, o: o)
            elif kind == "pre_hook":
                tgt.register_forward_pre_hook(lambda mod, i: None)
            else:
                tgt.forward = lambda *a, **k: None
            _refused(m, f"peft {kind} on {sub}")
    for sub in ("self", "layer", "down", "up"):
        m = _diffusers()
        tgt = {"self": m, "layer": m.lora_layer, "down": m.lora_layer.down, "up": m.lora_layer.up}[sub]
        tgt.register_forward_hook(lambda mod, i, o: o)
        _refused(m, f"diffusers hook on {sub}")
    m = _diffusers(); m.lora_layer = nn.Linear(64, 48); _refused(m, "lora_layer not a LoRALinearLayer")
    m = _diffusers(); m.lora_layer.up = nn.Linear(8, 48, bias=True).half(); _refused(m, "up with a bias")
    m = nn.Linear(8, 8); m.register_forward_hook(lambda mod, i, o: o); _refused(m, "Linear with a hook")

    class Other(nn.Linear):                             # a Linear subclass that is neither form
        pass
    _refused(Other(8, 8), "other Linear subclass")


def test_lora_attn_processor_stays_refused():
    """diffusers <= 0.20 put the LoRA into the attention processor; that form is not read."""
    a = _block().attn1

    class LoRAAttnProcessor:
        pass
    a.processor = LoRAAttnProcessor()
    assert not patch._plain_attention_module(a)
    assert not attention.cross_attention_eligible(a, torch.empty(1, 4, 64, dtype=torch.float16))


# ---------------------------------------------------------------------------------------------------------------------
# packing against the modules' forward in float64

def _check_pack(layers, x):
    """y = x W^T + b + (x D^T) U^T from the packs, in float64, against the layers' own float64 forward, concatenated.
    The packs round A (fp32 adapters; fp16 ones exactly) and s B to fp16 once each, so the gap is bounded by
    |x| |D - A|^T |U|^T + |x A^T| |U - s B|^T, each rounding at most half an fp16 spacing."""
    parts = [lora.linear_parts(m) for m in layers]
    assert all(p is not None for p in parts)
    packed = lora.pack(parts, "cpu")
    x64 = x.double()
    want = torch.cat([copy.deepcopy(m).double()(x64) for m in layers], dim=-1)
    w = torch.cat([p[0] for p in parts], dim=0).double()
    y = x64 @ w.t()
    b = [p[1].double() if p[1] is not None else torch.zeros(p[0].shape[0], dtype=torch.float64) for p in parts]
    y = y + torch.cat(b)
    if packed is None:
        assert all(not p[2] for p in parts)
        torch.testing.assert_close(y, want, rtol=0, atol=1e-12)
        return y
    down, up = packed
    assert down.dtype == up.dtype == torch.float16 and down.shape[0] % 8 == 0 and up.shape[1] == down.shape[0]
    t = x64 @ down.double().t()
    y = y + t @ up.double().t()
    # exact A and s B in float64, for the bound
    exact_down = torch.zeros(down.shape, dtype=torch.float64)
    exact_up = torch.zeros(up.shape, dtype=torch.float64)
    r0 = n0 = 0
    for wgt, _, ads in parts:
        for A, B, s in ads:
            exact_down[r0:r0 + A.shape[0]] = A.double()
            if A.dtype == torch.float16:
                assert torch.equal(down[r0:r0 + A.shape[0]].double(), A.double()), "fp16 A rows must be packed exactly"
            exact_up[n0:n0 + wgt.shape[0], r0:r0 + A.shape[0]] = B.double() * s
            r0 += A.shape[0]
        n0 += wgt.shape[0]
    half_ulp = torch.finfo(torch.float16).eps / 2
    err_down = (down.double() - exact_down).abs()
    err_up = (up.double() - exact_up).abs()
    assert (err_down <= half_ulp * exact_down.abs() + 2.0 ** -25).all(), "A rounded more than once"
    assert (err_up <= half_ulp * exact_up.abs() + 2.0 ** -25).all(), "s B rounded more than once"
    bound = (x64.abs() @ err_down.t()) @ up.double().abs().t() + (x64 @ exact_down.t()).abs() @ err_up.t()
    bound = bound + 1e-9 * (want.abs() + 1)
    gap = (y - want).abs()
    assert (gap <= bound).all(), f"gap {gap.max().item()} over bound {bound[gap > bound][:4].tolist()}"
    return y


def _x(K=64, M=37, seed=1, dtype=torch.float16):
    return torch.randn((M, K), generator=torch.Generator().manual_seed(seed)).to(dtype)


@pytest.mark.parametrize("adapter_dtype", [torch.float16, torch.float32])
def test_pack_diffusers(adapter_dtype):
    m = _diffusers(adapter_dtype=adapter_dtype)
    _check_pack([m], _x())


@pytest.mark.parametrize("adapter_dtype", [torch.float16, torch.float32])
def test_pack_peft_multiple_adapters(adapter_dtype):
    m = _peft(names=(("a", 8, 4.0), ("b", 12, 3.0), ("c", 8, 8.0)), adapter_dtype=adapter_dtype)
    m.set_adapter(["b", "a"])
    if adapter_dtype == torch.float32:
        assert not torch.equal(m.lora_A["a"].weight, m.lora_A["a"].weight.half().float()), "A must not be fp16 values"
    _check_pack([m], _x())                              # R = 20, padded to 24


@pytest.mark.parametrize("form", ["diffusers", "peft"])
def test_pack_qkv_subset(form):
    """LoRA on to_q and to_v only: U is block-diagonal with the k rows zero."""
    blk = add_lora(_block(), 8, form, targets=("to_q", "to_v"))
    a = blk.attn1
    assert type(a.to_k) is nn.Linear
    _check_pack([a.to_q, a.to_k, a.to_v], _x())
    parts = [lora.linear_parts(m) for m in (a.to_q, a.to_k, a.to_v)]
    down, up = lora.pack(parts, "cpu")
    assert down.shape == (16, 64) and up.shape == (192, 16)
    assert not up[64:128].any() and not up[:64, 8:].any() and not up[128:, :8].any()


@pytest.mark.parametrize("form", ["diffusers", "peft"])
def test_pack_every_projection_of_a_block(form):
    blk = add_lora(_block(), 8, form)
    x = _x()
    ctx = _x(K=32, seed=2)
    _check_pack([blk.attn1.to_q, blk.attn1.to_k, blk.attn1.to_v], x)
    _check_pack([blk.attn1.to_out[0]], x)
    _check_pack([blk.attn2.to_q], x)
    _check_pack([blk.attn2.to_k, blk.attn2.to_v], ctx)
    _check_pack([blk.ff.proj], x)
    _check_pack([blk.ff.out], _x(K=256, seed=3))


def test_pack_geglu_up_interleaved():
    """The GEGLU pack's up matrix is interleaved like the weight rows (ops.interleave_geglu)."""
    from vidtome_b200 import ops
    blk = add_lora(_block(), 8, "peft", targets=("ff",))
    w_il, b_il, w_o, b_o = feedforward._packed(blk.ff, blk.ff.proj, blk.ff.out)
    lora_1, lora_2 = feedforward._packed_lora(blk.ff, blk.ff.proj, blk.ff.out)
    parts = lora.linear_parts(blk.ff.proj)
    down, up = lora.pack([parts], "cpu")
    assert torch.equal(lora_1[0], down) and torch.equal(lora_1[1], ops.interleave_geglu(up, None)[0])
    assert torch.equal(w_il, ops.interleave_geglu(parts[0], None)[0])
    assert lora_2 is not None and lora_2[1].shape == (64, 8)


# ---------------------------------------------------------------------------------------------------------------------
# caches

def test_cache_refreshes():
    blk = add_lora(_block(), 8, "peft")
    a = blk.attn1
    like = torch.empty(0)
    first = attention._packed(a, like)
    assert first[3] is not None and first[4] is not None
    assert attention._packed(a, like)[3] is first[3]                # unchanged: cached

    a.to_q.scaling["default"] = 2.0                                           # rescale
    second = attention._packed(a, like)
    assert second[3] is not first[3] and not torch.equal(second[3][1], first[3][1])

    a.to_q.update_layer("extra", 8, 8.0)                                      # another active adapter
    third = attention._packed(a, like)
    assert third[3][0].shape[0] == 32

    a.to_q.set_adapter("default")                                             # adapter set
    fourth = attention._packed(a, like)
    assert fourth[3][0].shape[0] == 24

    with torch.no_grad():                                                     # a weight, in place
        a.to_v.lora_B["default"].weight.mul_(2)
    fifth = attention._packed(a, like)
    assert torch.equal(fifth[3][1][128:, 16:].float(), fourth[3][1][128:, 16:].float() * 2)
    assert torch.equal(fifth[3][1][:128], fourth[3][1][:128])

    for m in (a.to_q, a.to_k, a.to_v, a.to_out[0]):                           # everything disabled: no packs
        m._disable_adapters = True
    plain = attention._packed(a, like)
    assert plain[3] is None and plain[4] is None
    assert len(attention._packed_weights(a, like)) == 3 and attention._packed_lora(a, like) == (None, None)
    assert torch.equal(plain[0], torch.cat([a.to_q.base_layer.weight, a.to_k.base_layer.weight,
                                            a.to_v.base_layer.weight]))


def test_cross_attention_and_ff_caches_refresh():
    blk = add_lora(_block(), 8, "diffusers")
    ff = blk.ff
    first = feedforward._packed_all(ff, ff.proj, ff.out)
    ff.proj.lora_layer.network_alpha = 2.0
    second = feedforward._packed_all(ff, ff.proj, ff.out)
    assert not torch.equal(first[4][1], second[4][1])
    assert len(feedforward._packed(ff, ff.proj, ff.out)) == 4
    assert feedforward._packed_lora(ff, ff.proj, ff.out)[0] is second[4]
    ff.proj.lora_layer = None
    assert feedforward._packed_all(ff, ff.proj, ff.out)[4] is None


# ---------------------------------------------------------------------------------------------------------------------
# dispatch

@pytest.mark.parametrize("form", ["diffusers", "peft"])
def test_kd_accepts_lora_attention(form):
    blk = add_lora(_block(), 8, form)
    assert patch._plain_attention_module(blk.attn1)
    blk.attn1.to_k.register_forward_hook(lambda m, i, o: o)
    assert not patch._plain_attention_module(blk.attn1)


def test_kd_refuses_lora_with_bias_on_qkv():
    blk = _block()
    blk.attn1.to_q = PeftLoraLinear(nn.Linear(64, 64, bias=True).half())
    blk.attn1.to_q.update_layer("a", 8, 8.0)
    assert not patch._plain_attention_module(blk.attn1)


def test_stock_modules_still_refused_without_lora_fields():
    """Linear subclasses or wrappers that are not one of the two LoRA forms still fall back."""
    a = Attention(64, 2, 32)

    class LoRACompatibleLinearNoLayer(nn.Linear):
        def forward(self, x):
            return super().forward(x) + 1.0
    LoRACompatibleLinearNoLayer.__name__ = "LoRACompatibleLinear"
    a.to_q = LoRACompatibleLinearNoLayer(64, 64, bias=False)
    assert not patch._plain_attention_module(a)


def test_new_symbols_exported():
    from vidtome_b200 import _lib
    lib = _lib.load()
    for name in ("vtm_linear_lora_f16", "vtm_linear_geglu_lora_f16", "vtm_attention_lora", "vtm_cross_attention_lora",
                 "vtm_linear_lora_workspace_bytes", "vtm_attention_lora_workspace_bytes",
                 "vtm_cross_attention_lora_workspace_bytes"):
        assert hasattr(lib, name), name
    assert lib.vtm_linear_lora_workspace_bytes(100, 16) == 3200
    assert lib.vtm_linear_lora_workspace_bytes(100, 0) == 0
    base = lib.vtm_attention_workspace_bytes(2, 100, 320, 8)
    assert lib.vtm_attention_lora_workspace_bytes(2, 100, 320, 8, 0, 0) == base
    assert lib.vtm_attention_lora_workspace_bytes(2, 100, 320, 8, 24, 8) == base + 2 * 100 * 24 * 2
    xbase = lib.vtm_cross_attention_workspace_bytes(2, 100, 77, 320, 8)
    assert lib.vtm_cross_attention_lora_workspace_bytes(2, 100, 77, 320, 8, 0, 0, 0) == xbase
    assert lib.vtm_cross_attention_lora_workspace_bytes(2, 100, 77, 320, 8, 8, 16, 24) == xbase + (200 * 24 + 154 * 16) * 2


def test_lora_calls_fail_without_a_device():
    """No CPU fallback: with no CUDA device the entry points report an error (after argument checks)."""
    from vidtome_b200 import _lib
    lib = _lib.load()
    bad = _lib.VtmLora(None, None, 8)
    assert lib.vtm_linear_lora_f16(1, 1, None, None, 0, bad, 8, 8, 8, 1, 8, 1, 1 << 20, None) == -1
    odd = _lib.VtmLora(1, 1, 12)
    assert lib.vtm_linear_lora_f16(1, 1, None, None, 0, odd, 8, 8, 8, 1, 8, 1, 1 << 20, None) == -2
    ok = _lib.VtmLora(16, 16, 8)
    assert lib.vtm_linear_lora_f16(1, 1, None, None, 0, ok, 8, 8, 8, 1, 8, 16, 16, None) == -4
    assert lib.vtm_linear_lora_f16(1, 1, None, None, 0, ok, 8, 8, 8, 1, 8, 8, 1 << 20, None) == -2   # unaligned T
    # every argument is checked before the first launch (here a launch would report a CUDA error instead)
    ws = 1 << 20
    assert lib.vtm_linear_lora_f16(16, 16, None, None, 0, ok, 8, 12, 8, 16, 16, 16, ws, None) == -2      # N % 8
    assert lib.vtm_linear_lora_f16(16, 16, None, None, 0, ok, 8, 8, 8, 16, 4, 16, ws, None) == -2        # ldd < N
    assert lib.vtm_linear_lora_f16(16, 16, None, 16, 4, ok, 8, 8, 8, 16, 8, 16, ws, None) == -2          # ldr < N
    assert lib.vtm_linear_lora_f16(16, 16, None, None, 0, ok, 8, 8, 8, None, 8, 16, ws, None) == -1      # no output
    assert lib.vtm_linear_geglu_lora_f16(16, 16, None, ok, 8, 96, 8, 16, 48, 16, ws, None) == -2         # N % 64
    assert lib.vtm_linear_geglu_lora_f16(16, 16, None, ok, 8, 64, 8, 16, 16, 16, ws, None) == -2         # ldd < N / 2
