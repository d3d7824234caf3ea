"""The blocks of an unpatched ControlNet in the library (patch.FUSE_CONTROLNET_BLOCKS, patch.serve_unmerged): each stage of
a served block against float64 within the forward-error intervals of test_gpu_block_core, the whole ControlNet against
its torch forward, the step driver in every graph mode and the inverter's captured step against eager, a step free of
torch attention and reproducible across processes, and the switch off.  Needs an H100 (sm_90a)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import test_gpu_block_core as bc
import test_gpu_rows_core as rc
import test_gpu_transformer_io as tio
import vidtome_b200
from vidtome_b200 import attention, patch
from vidtome_b200.skeleton import BasicTransformerBlock, Transformer2DModel, make_controlnet, make_skeleton

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def switch():
    saved = patch.FUSE_CONTROLNET_BLOCKS, patch.FUSE_UNMERGED_ATTENTION, attention.MAX_HEAD_DIM
    yield
    patch.FUSE_CONTROLNET_BLOCKS, patch.FUSE_UNMERGED_ATTENTION, attention.MAX_HEAD_DIM = saved


# ---------------------------------------------------------------------------------- 1. stage bounds of a served block
# (C, heads, side of the block's token grid, items, context width, wrapper form, MAX_HEAD_DIM)
STAGE_CASES = {
    "sd15_c320_conv": (320, 8, 32, 4, 768, "conv", 128),
    "sd15_c640_conv": (640, 8, 32, 4, 768, "conv", 128),
    "sd15_c1280_conv_wide": (1280, 8, 16, 8, 768, "conv", 160),
    "sd15_c1280_conv_default_limit": (1280, 8, 16, 8, 768, "conv", 128),
    "sd15_mid_conv_wide": (1280, 8, 8, 8, 768, "conv", 160),
    "sd21_h10_linear": (640, 10, 24, 4, 1024, "linear", 128),
    "sd21_h20_linear": (1280, 20, 16, 4, 1024, "linear", 128),
}


def _served_wrapper(C, heads, cad, form, seed=0):
    """A served Transformer2DModel around one full block, with every bias, affine and eps taking a visible part (as
    test_gpu_block_core._make draws them)."""
    torch.manual_seed(seed + C + heads)
    blk = BasicTransformerBlock(C, heads, cad, hot_path_only=False)
    with torch.no_grad():
        for name, p in blk.named_parameters():
            if name.endswith("bias"):
                p.normal_(0.0, 0.5)
        for norm, eps in ((blk.norm1, 1e-3), (blk.norm2, 2e-2), (blk.norm3, 5e-3)):
            norm.weight.normal_(1.0, 0.2)
            norm.eps = eps
    wrap = Transformer2DModel(C, blk, use_linear_projection=form == "linear").cuda().half().eval()
    return patch.serve_unmerged(wrap), blk


@pytest.mark.parametrize("name", list(STAGE_CASES))
def test_served_block_stages_against_float64(switch, monkeypatch, name):
    C, heads, side, n, cad, form, limit = STAGE_CASES[name]
    wrap, blk = _served_wrapper(C, heads, cad, form)
    wide = C // heads <= limit
    g = torch.Generator(device="cuda").manual_seed(17)
    h = torch.randn((n, C, side, side), generator=g, device="cuda").half()
    ctx = torch.randn((n, 77, cad), generator=g, device="cuda").half()
    patch.FUSE_CONTROLNET_BLOCKS = True
    with monkeypatch.context() as mp:
        mp.setattr(attention, "MAX_HEAD_DIM", limit)
        rec = bc._Capture(mp)
        with torch.no_grad():
            out = wrap(h, encoder_hidden_states=ctx).sample
        torch.cuda.synchronize()
    assert not rec.rec["plan"], "a served block built a merge plan"
    failures = []

    def check(stage, fn):
        try:
            fn()
        except AssertionError as e:
            failures.append((stage, str(e).splitlines()[0]))

    what = lambda s: f"{name} {s}"                                            # noqa: E731
    gn, pin, pout = rec.one("gn"), rec.one("proj_in"), rec.one("proj_out")

    def s0():                                           # the Transformer2DModel entry: proj_in from the GroupNorm rows
        z, e = bc._proj(gn["out"].double().reshape(-1, C), None, bc._terms(wrap.proj_in))
        bc._within(pin["out"], z, e, what("S0 proj_in"))
        # the GroupNorm's interval: test_gpu_block_core's S0 (the statistics' bounds of test_gpu_transformer_io, then
        # the normalisation's fp32 steps)
        x = gn["args"][0]
        want = bc._group_norm64(x, wrap.norm).transpose(1, 2)
        G = wrap.norm.num_groups
        xd = x.double().view(n, G, -1)
        mean, var = xd.mean(-1), xd.var(-1, unbiased=False)
        rstd = 1 / torch.sqrt(var + wrap.norm.eps)
        steps = tio._stats_steps(xd.shape[-1], n * G)
        e_mean = steps * 4 * bc.U * xd.abs().amax(-1) + bc.U * mean.abs()
        e_var = steps * 8 * bc.U * var + 4 * (xd - mean[..., None]).abs().amax(-1) * e_mean + e_mean ** 2
        e_rstd = 0.5 * rstd ** 3 * e_var * 1.01 + 4 * bc.U * rstd
        rep = lambda t: t.repeat_interleave(C // G, 1)[:, :, None]              # noqa: E731
        t = (x.double().view(n, C, -1) - rep(mean)) * rep(rstd)
        gam = wrap.norm.weight.double().abs()[None, :, None]
        e = gam * (rep(e_mean) * rep(rstd) + (t.abs() / rep(rstd)) * rep(e_rstd))
        e = (e + 2 * bc.U * t.abs() * gam + bc.U * want.transpose(1, 2).abs()) * 1.01
        bc._within(gn["out"], want, e.transpose(1, 2), what("S0 GroupNorm -> tokens"))
    check("S0", s0)

    def s6():                                           # the exit: proj_out storing NCHW + residual
        t, w, b, x, hw = pout["args"]
        z, e = bc._proj(t.double(), None, bc._terms(wrap.proj_out))
        z, e = (v.view(n, -1, C).transpose(1, 2).reshape(x.shape) for v in (z, e))
        bc._within(pout["out"], z, e, what("S6 proj_out + residual"), resid=x)
    check("S6", s6)

    h_in = pin["out"].view(n, side * side, C)
    if wide:                                            # norm1 -> KD with the residual in its out projection
        ln1, a1 = rec.ln_of(blk.norm1), rec.one("attn1r")
        assert not [e for e in rec.rec["module_attn"] if e["args"][0] is blk.attn1], "attn1 ran its module forward"
        check("S1", lambda: rc._check_ln(ln1["out"], ln1["args"][0], (blk.norm1.weight, blk.norm1.bias, blk.norm1.eps),
                                         what("S1 norm1")) and None)

        def s2():
            z, e = bc._self_attention_bound(blk.attn1, a1["args"][1])
            bc._within(a1["out"], z, e, what("S2 attn1 + residual"), resid=a1["args"][2])
        check("S2", s2)
        h1 = a1["out"]
        links = [("attn1 input", a1["args"][1], ln1["out"]), ("attn1 residual", a1["args"][2], h_in),
                 ("norm1 input", ln1["args"][0], h_in)]
        ln2, a2 = rec.ln_of(blk.norm2), rec.one("attn2")
        check("S4", lambda: rc._check_ln(ln2["out"], ln2["args"][0], (blk.norm2.weight, blk.norm2.bias, blk.norm2.eps),
                                         what("S4 norm2")) and None)

        def s4():
            _, x, c, r = a2["args"]
            z, e = bc._cross_attention_bound(blk.attn2, x, c)
            bc._within(a2["out"], z, e, what("S4 attn2 + residual"), resid=r)
        check("S4", s4)
        h2 = a2["out"]
        links += [("norm2 input", ln2["args"][0], h1), ("attn2 queries", a2["args"][1], ln2["out"]),
                  ("attn2 residual", a2["args"][3], h1), ("attn2 context", a2["args"][2], ctx)]
    else:
        # head_dim above MAX_HEAD_DIM: attn1 and attn2 run their module forwards (torch), the rest the library
        mods = [e for e in rec.rec["module_attn"] if e["args"][0] in (blk.attn1, blk.attn2)]
        assert len(mods) == 2 and not rec.rec["attn1r"] and not rec.rec["attn2"], "the attention left its modules"
        ff_e = rec.one("ff")
        h2 = ff_e["args"][3]

        def s24():
            with torch.no_grad():
                h1 = type(blk.attn1).forward(blk.attn1, blk.norm1(h_in)) + h_in
                want = type(blk.attn2).forward(blk.attn2, blk.norm2(h1), encoder_hidden_states=ctx) + h1
            assert torch.equal(bc._bits(want), bc._bits(h2)), what("S2/S4: the modules' path is not torch's")
        check("S4", s24)
        links = []

    ff_e, ln3 = rec.one("ff"), rec.ln_of(blk.norm3)
    check("S5", lambda: rc._check_ln(ln3["out"], ln3["args"][0], (blk.norm3.weight, blk.norm3.bias, blk.norm3.eps),
                                     what("S5 norm3")) and None)

    def s5():
        z, e = bc._ff_bound(blk.ff, ln3["out"])
        hs = ff_e["args"][3]
        bc._within(ff_e["out"].reshape(-1, C), z, e, what("S5 feed-forward + residual"), resid=hs.reshape(-1, C))
    check("S5", s5)

    def chain():
        for label, got, want in links + [("feed-forward input", ff_e["args"][3], h2), ("norm3 input", ln3["args"][0], h2),
                                         ("proj_in input", pin["args"][0], gn["out"]), ("GroupNorm input", gn["args"][0], h),
                                         ("proj_out input", pout["args"][0], ff_e["out"]),
                                         ("proj_out residual", pout["args"][3], h), ("output", out, pout["out"])]:
            assert got.numel() == want.numel() and torch.equal(bc._bits(got), bc._bits(want)), f"{label} differs"
    check("chain", chain)

    def e2e():
        tok = bc._group_norm64(h, wrap.norm).transpose(1, 2)
        t = bc._block64(blk, bc._lin64(tok, wrap.proj_in), ctx, None)
        ref = bc._lin64(t, wrap.proj_out).transpose(1, 2).reshape(h.shape) + h.double()
        assert torch.isfinite(out).all()
        rel = (out.double() - ref).abs().max().item() / ref.abs().max().item()
        assert rel <= bc.E2E_LEVEL, what(f"end to end: {rel:.3e} of max|ref|")
    check("E2E", e2e)
    assert not failures, failures


# ------------------------------------------------------------------------------------- 2. the whole ControlNet forward
# max-norm difference of every residual from the torch forward, relative to its max|.|: both are fp16 computations of
# the same function, the library's with fp32 softmax and fused roundings
WHOLE_LEVEL = 1e-2


@pytest.mark.parametrize("name,io", [("sd15", "conv"), ("sd21", "linear"), ("sd15", None)])
def test_whole_controlnet_matches_its_torch_forward(switch, name, io):
    attention.MAX_HEAD_DIM = 160
    cn = make_controlnet(name, hot_path_only=False, device="cuda", transformer_io=io)
    cad = 1024 if name == "sd21" else 768
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn((8, 4, 32, 32), generator=g, device="cuda").half()
    ctx = torch.randn((8, 77, cad), generator=g, device="cuda").half()
    ctrl = torch.rand((8, 3, 256, 256), generator=g, device="cuda").half()
    calls = {"kd": 0}
    inner = attention.self_attention_residual

    def counting(*a, **k):
        calls["kd"] += 1
        return inner(*a, **k)
    with torch.no_grad():
        want = cn(x, 981, encoder_hidden_states=ctx, controlnet_cond=ctrl)
        patch.serve_unmerged(cn)
        patch.FUSE_CONTROLNET_BLOCKS = True
        attention.self_attention_residual = counting
        try:
            got = cn(x, 981, encoder_hidden_states=ctx, controlnet_cond=ctrl)
        finally:
            attention.self_attention_residual = inner
    assert calls["kd"] == len(cn.blocks)
    for i, (a, b) in enumerate(zip(list(got[0]) + [got[1]], list(want[0]) + [want[1]])):
        assert torch.isfinite(a).all(), i
        rel = (a.float() - b.float()).abs().max().item() / b.float().abs().max().item()
        assert 0 < rel <= WHOLE_LEVEL, (i, rel)


# ------------------------------------------------------------------------------------------------- 3-6. the drivers
STEPS, FRAMES, SIZE = 4, 8, 32


def _run(name, mode, on, steps=STEPS, fuse_unmerged=False, cn=None, keep=None):
    """Latents after every step of a ControlNet-controlled ChunkedDenoiser: UNet patched, ControlNet unpatched."""
    from vidtome_b200.driver import ChunkedDenoiser
    patch.FUSE_CONTROLNET_BLOCKS = on
    patch.FUSE_UNMERGED_ATTENTION = fuse_unmerged
    io = "linear" if name == "sd21" else "conv"
    torch.manual_seed(77)
    unet = make_skeleton(name, hot_path_only=False, device="cuda", transformer_io=io)
    cn = make_controlnet(name, hot_path_only=False, device="cuda", transformer_io=io) if cn is None else cn
    merge_global = mode not in ("step_graph", "eager_plain")
    vidtome_b200.apply_patch(unet, local_merge_ratio=0.9, merge_global=merge_global, global_merge_ratio=0.8,
                             global_rand=0.5, batch_size=2)
    cad = 1024 if name == "sd21" else 768
    g = torch.Generator(device="cuda").manual_seed(5)
    graph = not mode.startswith("eager")
    kw = dict(cuda_graph=graph, graph_warmup=1)
    if mode in ("chunk_graphs", "eager_random"):
        kw.update(randomize_chunks=True, chunk_graphs=graph)
    if mode in ("capture_global", "eager_global"):
        kw.update(capture_global=graph)
    cond = torch.randn((2, 77, cad), generator=g, device="cuda").half()
    images = torch.rand((FRAMES, 3, 8 * SIZE, 8 * SIZE), generator=g, device="cuda").half()
    den = ChunkedDenoiser(unet, n_timesteps=steps, chunk_size=4, merge_global=merge_global, chunk_ord="mix-4",
                          cond=cond, controlnet=cn, control_images=images, control_scale=0.8, **kw)
    x = torch.randn((FRAMES, 4, SIZE, SIZE), generator=g, device="cuda", dtype=torch.float16)
    torch.manual_seed(2024)
    np.random.seed(2024)
    xs = []
    for i in range(steps):
        x = den.step(x, i)
        xs.append(x.clone())
        if keep is not None:
            keep.append(patch.is_served(cn))
    torch.cuda.synchronize()
    den.close()
    return xs


class _CountKD:
    def __init__(self, monkeypatch):
        self.n = 0
        inner = attention.self_attention_residual

        def counting(*a, **k):
            self.n += 1
            return inner(*a, **k)
        monkeypatch.setattr(attention, "self_attention_residual", counting)


@pytest.mark.parametrize("name", ["sd15", "sd21"])
@pytest.mark.parametrize("mode,eager_mode", [("step_graph", "eager_plain"), ("capture_global", "eager_global"),
                                             ("chunk_graphs", "eager_random")])
def test_driver_graph_modes_are_bit_identical_to_eager(switch, monkeypatch, name, mode, eager_mode):
    attention.MAX_HEAD_DIM = 160
    count = _CountKD(monkeypatch)
    served = []
    eager = _run(name, eager_mode, True, keep=served)
    assert count.n > 0 and all(served), "the ControlNet's blocks did not run in the library"
    graph = _run(name, mode, True)
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(b).all(), i
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"
    off = _run(name, eager_mode, False)
    for i, (a, b) in enumerate(zip(eager, off)):
        err = (a.float() - b.float()).abs().max().item()
        assert err <= 2e-2 * b.float().abs().max().item() + 2e-2, (i, err)


@pytest.mark.parametrize("name", ["sd15", "sd21"])
def test_inverter_captured_step_is_bit_identical_to_eager(switch, monkeypatch, name):
    from vidtome_b200.driver import ChunkedInverter
    attention.MAX_HEAD_DIM = 160
    patch.FUSE_CONTROLNET_BLOCKS = True
    count = _CountKD(monkeypatch)
    io = "linear" if name == "sd21" else "conv"
    cad = 1024 if name == "sd21" else 768
    unet = make_skeleton(name, hot_path_only=False, device="cuda", transformer_io=io)
    vidtome_b200.apply_patch(unet, local_merge_ratio=0.9, batch_size=2)
    cn = make_controlnet(name, hot_path_only=False, device="cuda", transformer_io=io)
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn((6, 4, SIZE, SIZE), generator=g, device="cuda").half()
    cond = torch.randn((6, 77, cad), generator=g, device="cuda").half()
    images = torch.rand((6, 3, 8 * SIZE, 8 * SIZE), generator=g, device="cuda").half()
    trajs = []
    for graph in (False, True):
        inv = ChunkedInverter(unet, n_timesteps=5, batch_size=4, cond=cond, controlnet=cn, control_images=images,
                              control_scale=0.8, cuda_graph=graph, graph_warmup=1)
        inv.invert(x)
        assert patch.is_served(cn)
        trajs.append(inv.trajectory.clone())
        inv.close()
        assert not patch.is_served(cn)
    assert count.n > 0
    assert torch.isfinite(trajs[1]).all()
    assert torch.equal(trajs[0], trajs[1]), (trajs[0].float() - trajs[1].float()).abs().max().item()


@pytest.mark.parametrize("name", ["sd15", "sd21"])
def test_no_torch_attention_is_left_in_a_controlnet_step(switch, monkeypatch, name):
    attention.MAX_HEAD_DIM = 160
    calls = {"sdpa": 0}
    sdpa = torch.nn.functional.scaled_dot_product_attention

    def counting_sdpa(*a, **k):
        calls["sdpa"] += 1
        return sdpa(*a, **k)
    monkeypatch.setattr(torch.nn.functional, "scaled_dot_product_attention", counting_sdpa)
    _run(name, "eager_global", True, steps=2, fuse_unmerged=True)
    assert calls["sdpa"] == 0, calls
    _run(name, "eager_global", False, steps=2, fuse_unmerged=True)     # the ControlNet's modules call it, switch off
    assert calls["sdpa"] > 0, calls


_CHILD = """
import sys, numpy as np, torch
sys.path[:0] = [{root!r}, {tests!r}, {oracle!r}]
import test_gpu_controlnet_blocks as t
from vidtome_b200 import attention
attention.MAX_HEAD_DIM = 160
xs = t._run({name!r}, "eager_global", True, steps=3, fuse_unmerged=True)
np.save({out!r}, torch.stack(xs).cpu().numpy())
"""


@pytest.mark.parametrize("name", ["sd15", "sd21"])
def test_two_processes_give_bit_identical_latents(tmp_path, name):
    outs = []
    for k in range(2):
        out = str(tmp_path / f"x{k}.npy")
        code = _CHILD.format(root=ROOT, tests=os.path.join(ROOT, "tests"), oracle=os.path.join(ROOT, "oracle"), name=name,
                             out=out)
        r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        outs.append(np.load(out))
    assert np.isfinite(outs[0]).all()
    diff = np.abs(outs[0].astype(np.float32) - outs[1].astype(np.float32))
    assert np.array_equal(outs[0], outs[1]), f"max |diff| {diff.max()} at step {np.argwhere(diff > 0)[0][0]}"


@pytest.mark.parametrize("name", ["sd15", "sd21"])
def test_switch_off_is_the_parent_path(switch, name):
    """With the switch off nothing is swapped and the latents are those of the modules' own forwards; a ControlNet that
    was served and is stepped with the switch off again gives the same latents bit for bit."""
    attention.MAX_HEAD_DIM = 160
    io = "linear" if name == "sd21" else "conv"
    cn = make_controlnet(name, hot_path_only=False, device="cuda", transformer_io=io)
    before = {n: type(m) for n, m in cn.named_modules()}
    served = []
    off = _run(name, "eager_global", False, cn=cn, keep=served)
    assert not any(served) and {n: type(m) for n, m in cn.named_modules()} == before
    on = _run(name, "eager_global", True, cn=cn)
    assert any(not torch.equal(a, b) for a, b in zip(off, on)), "the switch changed nothing"
    patch.serve_unmerged(cn)                                             # served, switch off: the modules' forwards
    again = _run(name, "eager_global", False, cn=cn)
    patch.unserve_unmerged(cn)
    assert {n: type(m) for n, m in cn.named_modules()} == before
    for i, (a, b) in enumerate(zip(off, again)):
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"
