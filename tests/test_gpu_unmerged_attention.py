"""The self-attention of blocks that do not merge, in the library during generation (patch.FUSE_UNMERGED_ATTENTION):
`vtm_attention_residual_ex` against `vtm_attention_residual`, against per-frame compositions of
`vtm_attention_ex(VTM_ATTN_SHARED_QK)` and against float64, its memory behaviour inside guard bands, a PnP-marked block
against the module's torch forward, and the step driver with the switch on.  Needs an H100 (sm_90a)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import test_gpu_attention_core as core
import test_gpu_attention_wide as wide
import test_gpu_bounds as tb
from vidtome_b200 import _lib, attention, ops, patch, pnp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHARED_QK = 1


@pytest.fixture
def switch():
    saved = patch.FUSE_UNMERGED_ATTENTION, attention.MAX_HEAD_DIM
    yield
    patch.FUSE_UNMERGED_ATTENTION, attention.MAX_HEAD_DIM = saved


def _lora(R, K, N, g):
    return ((torch.randn(R, K, generator=g, device="cuda") * 0.05).half(),
            (torch.randn(N, R, generator=g, device="cuda") * 0.05).half())


def _residual_ex(x, w_qkv, w_o, b_o, H, scale, resid, flags, items, lora_qkv=None, lora_o=None):
    """vtm_attention_residual_ex through the C-ABI, workspace filled with 0xFF bytes and the output with NaN."""
    lib = _lib.load()
    B, L, C = x.shape
    dq, rq = ops._lora_arg(lora_qkv, C, 3 * C, "qkv")
    do, ro = ops._lora_arg(lora_o, C, C, "out")
    ws_bytes = lib.vtm_attention_lora_workspace_bytes(B, L, C, H, rq, ro)
    ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device="cuda")
    y = torch.full_like(x, float("nan"))
    rc = lib.vtm_attention_residual_ex(x.data_ptr(), w_qkv.data_ptr(), w_o.data_ptr(), ops._ptr(b_o), resid.data_ptr(),
                                       ops._lora_ref(dq), ops._lora_ref(do), B, L, C, H, float(scale), flags, items,
                                       y.data_ptr(), ws.data_ptr(), ws_bytes, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, rc
    return y


def _weights(C, g):
    return ((torch.randn(3 * C, C, generator=g, device="cuda") * C ** -0.5).half(),
            (torch.randn(C, C, generator=g, device="cuda") * C ** -0.5).half(),
            (torch.randn(C, generator=g, device="cuda") * 0.1).half())


# --------------------------------------------------------------------------- 1. flags == 0 is vtm_attention_residual
# (B, L, C, heads): SD2.1 512² / 768² ds4 per-frame items (2 or 3 inputs x 16 frames), SD1.5 ds4 / ds8 at head_dim 160,
# ragged lengths
SHAPES = [(32, 256, 1280, 20), (48, 256, 1280, 20), (32, 576, 1280, 20), (32, 256, 1280, 8), (48, 64, 1280, 8),
          (6, 144, 640, 10), (4, 576, 320, 8), (6, 1, 1280, 8)]


@pytest.mark.parametrize("lora", [False, True])
@pytest.mark.parametrize("B,L,C,H", SHAPES)
def test_unshared_is_bit_identical_to_attention_residual(B, L, C, H, lora):
    g = torch.Generator(device="cuda").manual_seed(B + L + C + H)
    x = torch.randn(B, L, C, generator=g, device="cuda").half()
    resid = (torch.randn(B, L, C, generator=g, device="cuda") * 4).half()
    w_qkv, w_o, b_o = _weights(C, g)
    kw = dict(lora_qkv=_lora(16, C, 3 * C, g), lora_o=_lora(8, C, C, g)) if lora else {}
    scale = (C // H) ** -0.5
    want = ops.attention_residual(x, w_qkv, w_o, b_o, H, scale, resid, **kw)
    for items in (0, 1, 7):                                   # ignored without the flag
        got = _residual_ex(x, w_qkv, w_o, b_o, H, scale, resid, 0, items, **kw)
        assert torch.equal(got, want), f"items={items}: max |diff| {(got.float() - want.float()).abs().max().item()}"


# --------------------------------------------------------------------------- 2. shared, by frame
def _composition(x, w_qkv, w_o, b_o, H, scale, resid, n, lora_qkv=None, lora_o=None):
    """For every frame f < n: items {f + j n} through vtm_attention_ex(VTM_ATTN_SHARED_QK), then torch's half add."""
    B, L, C = x.shape
    out = torch.empty_like(x)
    for f in range(n):
        idx = torch.arange(f, B, n, device="cuda")
        y = ops.attention(x[idx].contiguous(), w_qkv, w_o, b_o, H, scale, shared_qk=True, lora_qkv=lora_qkv,
                          lora_o=lora_o)
        out[idx] = y + resid[idx]
    return out


CASES = [(ni, n, d) for ni in (2, 3) for n in (1, 4, 16) for d in (40, 64, 80, 160)]


@pytest.mark.parametrize("num_inputs,n,d", CASES)
def test_shared_by_frame_is_the_per_frame_composition(num_inputs, n, d):
    """head_dim 40 / 64 / 80 / 160: groups of up to 4 / 2 / 2 / 1 inputs per CTA, ragged at 3 inputs."""
    B, H = num_inputs * n, max(1, 640 // d // 2)
    C, L = d * H, 193
    g = torch.Generator(device="cuda").manual_seed(num_inputs * 1000 + n * 10 + d)
    x = torch.randn(B, L, C, generator=g, device="cuda").half()
    resid = (torch.randn(B, L, C, generator=g, device="cuda") * 4).half()
    w_qkv, w_o, b_o = _weights(C, g)
    scale = d ** -0.5
    for lora in (False, True):
        kw = dict(lora_qkv=_lora(16, C, 3 * C, g), lora_o=_lora(8, C, C, g)) if lora else {}
        want = _composition(x, w_qkv, w_o, b_o, H, scale, resid, n, **kw)
        got = _residual_ex(x, w_qkv, w_o, b_o, H, scale, resid, SHARED_QK, n, **kw)
        assert torch.isfinite(got).all()
        assert torch.equal(got, want), f"lora={lora}: max |diff| {(got.float() - want.float()).abs().max().item()}"
        assert torch.equal(ops.attention_residual(x, w_qkv, w_o, b_o, H, scale, resid, shared_items=n, **kw), want)
    # the item layout matters: a different period gives a different result unless the batch is one frame
    if n > 1:
        other = _residual_ex(x, w_qkv, w_o, b_o, H, scale, resid, SHARED_QK, 1)
        assert not torch.equal(other, want)


@pytest.mark.parametrize("name", ["random", "negative"])
@pytest.mark.parametrize("num_inputs,n,d", [(ni, n, d) for ni in (2, 3) for n in (1, 4, 16) for d in (40, 64, 80, 160)
                                            if n * ni * d <= 3 * 16 * 80])
def test_shared_by_frame_against_float64(num_inputs, n, d, name):
    """utils/pnp_utils.py:47-95 in float64 (q, k of item b mod n, `attn.repeat(num_inputs, 1, 1)`), on the exact
    designs of test_gpu_attention_core with W_o = I, no bias and a zero residual, held to its bound."""
    B, H, L = num_inputs * n, 2, 129
    g = torch.Generator(device="cuda").manual_seed(n * 7 + d + num_inputs)
    x, w, scale = core._self_design(name, B, L, d * H, H, g)
    q, k, v = wide._self_qkv(x, w, H)
    q, k = q[:n].repeat(num_inputs, 1, 1, 1), k[:n].repeat(num_inputs, 1, 1, 1)
    O, bound = core._reference(q, k, v, scale)
    eye = torch.eye(d * H, dtype=torch.float16, device="cuda")
    y = _residual_ex(x, w, eye, None, H, scale, torch.zeros_like(x), SHARED_QK, n)
    torch.cuda.synchronize()
    core._assert_within(y, O, bound, f"shared by frame {name} num_inputs={num_inputs} n={n} d={d}")


# --------------------------------------------------------------------------- 3. guard bands
def _bounds_case(B, L, d, H, n, lora=None, name="random"):
    x, w, wo, scale, g = tb._self_inputs(name, B, L, d, H, seed=B * L + d + n)
    C = d * H
    Rq, Ro = lora or (0, 0)
    lib = _lib.load()
    ws_bytes = lib.vtm_attention_lora_workspace_bytes(B, L, C, H, Rq, Ro)
    DP = tb._dp(d)
    slab = B * H * L * DP * 2                               # bytes of one of q, k, v for all items
    ws_kept = torch.zeros(ws_bytes, dtype=torch.bool)
    for j in range(2):                                      # q and k of items n .. B - 1 are left as they were
        ws_kept[j * slab + n * H * L * DP * 2:(j + 1) * slab] = True
    bufs = {"x": tb.Buf("in", x), "w": tb.Buf("in", w), "wo": tb.Buf("in", wo), "bo": tb.Buf("in", tb._randn((C,), g)),
            "r": tb.Buf("in", tb._randn(x.shape, g)), "y": tb._out(B * L * C, C * 2), "ws": tb._ws(ws_bytes, kept=ws_kept)}
    if lora:
        for k, (R, N) in (("q", (Rq, 3 * C)), ("o", (Ro, C))):
            bufs["d" + k], bufs["u" + k] = tb.Buf("in", tb._randn((R, C), g, 0.05)), tb.Buf("in", tb._randn((N, R), g, 0.05))

    def args(b):
        lq, lo = ((_lib.VtmLora(b["dq"], b["uq"], Rq), _lib.VtmLora(b["do"], b["uo"], Ro)) if lora else (None, None))
        return [b["x"], b["w"], b["wo"], b["bo"], b["r"], tb._ref(lq), tb._ref(lo), B, L, C, H, scale, SHARED_QK, n,
                b["y"], b["ws"], ws_bytes, tb._stream()]
    errs = [(tb.VTM_E_NULL, {4: None}), (tb.VTM_E_SHAPE, {13: 0}), (tb.VTM_E_UNSUPPORTED, {12: 3})]
    if B > 1:
        errs.append((tb.VTM_E_SHAPE, {13: B + 1}))
    return tb.Case("vtm_attention_residual_ex", bufs, args, ws="ws", ws_arg=16, errors=errs)


# (B, L, d, H, n, lora): ragged groups at 3 inputs, head_dim classes 40 / 80 / 128 / 160, one frame and many
BOUNDS = [(6, 65, 40, 2, 2, None), (9, 193, 80, 2, 3, None), (12, 129, 64, 4, 4, (16, 8)), (4, 1000, 160, 2, 2, None),
          (3, 1, 128, 2, 1, None), (48, 64, 160, 2, 16, (8, 200))]

# The entry point's cases for test_gpu_bounds.REGISTRY (tests/test_bounds_cpu.py checks that the registry names every
# compute entry point of the C-ABI)
tb.REGISTRY.setdefault("vtm_attention_residual_ex", []).extend(
    (f"B={B} L={L} d={d} H={H} items={n} lora={lo}", (lambda a=(B, L, d, H, n, lo): _bounds_case(*a)))
    for B, L, d, H, n, lo in BOUNDS)


@pytest.mark.parametrize("B,L,d,H,n,lora", BOUNDS)
def test_guard_bands(B, L, d, H, n, lora):
    case = _bounds_case(B, L, d, H, n, lora)
    tb.run_case(case, f"vtm_attention_residual_ex B={B} L={L} d={d} H={H} items={n} lora={lora}")


# --------------------------------------------------------------------------- 4. one PnP-marked block
@pytest.mark.parametrize("name,d", [("sd21", 64), ("sd15", 160)])
def test_pnp_block_matches_the_module_forward(switch, name, d):
    from vidtome_b200.skeleton import BasicTransformerBlock
    attention.MAX_HEAD_DIM = 160
    torch.manual_seed(4)
    C, heads, frames, T = 1280, 1280 // d, 4, 64
    blk = BasicTransformerBlock(C, heads, hot_path_only=True).cuda().half()
    blk.__class__ = patch.make_diffusers_tome_block(blk.__class__)
    blk._tome_info = {"size": (32, 32), "hooks": [], "args": dict(
        max_downsample=2, generator=None, seed=123, batch_size=3, align_batch=True, merge_global=False,
        global_merge_ratio=0.8, local_merge_ratio=0.9, global_rand=0.5, target_stride=4)}
    pnp.register_attention_control(None, [981], 3, modules=[blk.attn1])
    x = torch.randn(3 * frames, T, C, device="cuda").half()
    for t in (981, 500):
        pnp.register_time(None, t, modules=[blk.attn1])
        with torch.no_grad():
            patch.FUSE_UNMERGED_ATTENTION = False
            want = blk(x)
            patch.FUSE_UNMERGED_ATTENTION = True
            got = blk(x)
        assert torch.isfinite(got).all()
        err = (got.float() - want.float()).abs().max().item()
        assert err <= 4e-3 * want.float().abs().max().item(), (t, err)
        if t == 981:                                     # injecting: the uncond and cond frames share the source maps
            shared = got - x
            assert not torch.equal(shared[frames:2 * frames], shared[:frames])


# --------------------------------------------------------------------------- 5-7. the step driver
STEPS, FRAMES, SIZE = 4, 8, 32


def _run(name, mode, fuse, control=False, steps=STEPS):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_controlnet, make_skeleton, pnp_attention_modules, pnp_conv_module
    patch.FUSE_UNMERGED_ATTENTION = fuse
    torch.manual_seed(77)
    net = make_skeleton(name, hot_path_only=False, device="cuda", pnp_conv=not control)
    merge_global = mode not in ("step_graph", "eager_plain")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=merge_global, global_merge_ratio=0.8,
                             global_rand=0.5, batch_size=2 if control else 3, align_batch=True)
    cad = 1024 if name == "sd21" else 768
    g = torch.Generator(device="cuda").manual_seed(5)
    graph = not mode.startswith("eager")
    kw = dict(cuda_graph=graph, graph_warmup=1)
    if mode in ("chunk_graphs", "eager_random"):
        kw.update(randomize_chunks=True, chunk_graphs=graph)
    if mode in ("capture_global", "eager_global"):
        kw.update(capture_global=graph)
    if control:
        cnet = make_controlnet(name, hot_path_only=False, device="cuda")
        vidtome_b200.apply_patch(cnet, local_merge_ratio=0.9, batch_size=2)
        cond = torch.randn((2, 77, cad), generator=g, device="cuda").half()
        images = torch.rand((FRAMES, 3, 8 * SIZE, 8 * SIZE), generator=g, device="cuda").half()
        kw.update(controlnet=cnet, control_images=images, control_scale=0.8)
    else:
        cond = torch.randn((3, 77, cad), generator=g, device="cuda").half()
        sources = {}

        def source(t):
            if t not in sources:
                gs = torch.Generator(device="cuda").manual_seed(int(t))
                sources[t] = torch.randn((FRAMES, 4, SIZE, SIZE), generator=gs, device="cuda").half()
            return sources[t]
        kw.update(source_latents=source, pnp_attn_t=0.5, pnp_modules=pnp_attention_modules(net), pnp_f_t=0.8,
                  pnp_conv_modules=[pnp_conv_module(net)])
    den = ChunkedDenoiser(net, n_timesteps=steps, chunk_size=4, merge_global=merge_global, chunk_ord="mix-4",
                          cond=cond, **kw)
    x = torch.randn((FRAMES, 4, SIZE, SIZE), generator=g, device="cuda", dtype=torch.float16)
    torch.manual_seed(2024)
    np.random.seed(2024)
    xs = []
    for i in range(steps):
        x = den.step(x, i)
        xs.append(x.clone())
    torch.cuda.synchronize()
    return xs


class _Count:
    """Counts the library's residual self-attention calls by their shared_items."""

    def __init__(self, monkeypatch):
        self.calls = []
        inner = attention.self_attention_residual

        def counting(attn, x, resid, shared_items=None):
            self.calls.append(shared_items)
            return inner(attn, x, resid, shared_items=shared_items)
        monkeypatch.setattr(attention, "self_attention_residual", counting)


@pytest.mark.parametrize("name", ["sd21", "sd15"])
@pytest.mark.parametrize("mode,eager_mode", [("step_graph", "eager_plain"), ("capture_global", "eager_global"),
                                             ("chunk_graphs", "eager_random")])
def test_driver_graph_modes_are_bit_identical_to_eager(switch, monkeypatch, name, mode, eager_mode):
    attention.MAX_HEAD_DIM = 160
    count = _Count(monkeypatch)
    eager = _run(name, eager_mode, True)
    shared = [c for c in count.calls if c is not None]
    assert shared and None in count.calls, "the shared and the plain path did not both run"
    assert set(shared) <= set(range(1, FRAMES + 1)), set(shared)          # frames of a chunk
    graph = _run(name, mode, True)
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(b).all(), i
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"
    off = _run(name, eager_mode, False)
    for i, (a, b) in enumerate(zip(eager, off)):
        err = (a.float() - b.float()).abs().max().item()
        assert err <= 2e-2 * b.float().abs().max().item() + 2e-2, (i, err)


@pytest.mark.parametrize("name", ["sd21", "sd15"])
def test_driver_with_controlnet_graph_is_bit_identical_to_eager(switch, name):
    attention.MAX_HEAD_DIM = 160
    eager = _run(name, "eager_plain", True, control=True, steps=3)
    graph = _run(name, "step_graph", True, control=True, steps=3)
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(b).all(), i
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"


@pytest.mark.parametrize("name", ["sd21", "sd15"])
def test_no_torch_attention_is_left_in_a_step(switch, monkeypatch, name):
    attention.MAX_HEAD_DIM = 160
    calls = {"sdpa": 0, "pnp": 0}
    sdpa = torch.nn.functional.scaled_dot_product_attention

    def counting_sdpa(*a, **k):
        calls["sdpa"] += 1
        return sdpa(*a, **k)
    monkeypatch.setattr(torch.nn.functional, "scaled_dot_product_attention", counting_sdpa)
    torch_forward = pnp._torch_forward

    def counting_torch_forward(attn, num_inputs):
        fwd = torch_forward(attn, num_inputs)

        def forward(*a, **k):
            calls["pnp"] += 1
            return fwd(*a, **k)
        forward._vtm_pnp_forward = True
        return forward
    monkeypatch.setattr(pnp, "_torch_forward", counting_torch_forward)
    _run(name, "eager_plain", True, steps=2)
    assert calls == {"sdpa": 0, "pnp": 0}, calls
    _run(name, "eager_plain", False, steps=2)                 # the counters see the module path with the switch off
    assert calls["sdpa"] > 0 and calls["pnp"] > 0, calls


_CHILD = """
import sys, numpy as np, torch
sys.path[:0] = [{root!r}, {tests!r}, {oracle!r}]
import test_gpu_unmerged_attention as t
from vidtome_b200 import attention
attention.MAX_HEAD_DIM = 160
xs = t._run({name!r}, "eager_global", True, steps=3)
np.save({out!r}, torch.stack(xs).cpu().numpy())
"""


@pytest.mark.parametrize("name", ["sd21", "sd15"])
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
