"""The flash-attention kernel at head_dim 136-160 (KS = 9 and 10 k-steps, rows padded to 192 halfs, three TMA boxes)
and SD1.5's 1280-channel blocks (8 heads of 160) running attention in the library once `attention.MAX_HEAD_DIM` is
160.  Needs an H100 (sm_90a).

Kernel checks use the method of test_gpu_attention_core.py (its designs, reference and bound are imported from there):
tokens on a 1/8 grid and signed-permutation projections make q, k and v exact, W_o = I, the workspace is filled with
0xFF bytes and the output with NaN.  Restated for d <= 160: q and k are bounded by 4, so S = q k^T has |S| <= 16 * 160
< 2^12 on a 2^-6 grid, 18 significant bits, and is exact in fp32 whatever the order of the k-steps.  The bound of
`_reference` does not depend on d otherwise: its accumulation terms count the 64-key tiles (P V) and the row sums
(l), both the same as at d <= 128, so it holds unchanged."""
import os
import subprocess
import sys

import pytest
import torch

import test_gpu_attention_core as core
from vidtome_b200 import _lib

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIDE = (136, 144, 152, 160)
LENGTHS = (1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 1000)


@pytest.fixture
def wide_limit():
    from vidtome_b200 import attention
    saved = attention.MAX_HEAD_DIM
    attention.MAX_HEAD_DIM = 160
    yield
    attention.MAX_HEAD_DIM = saved


# ---------------------------------------------------------------------------------------------------------------------
# kernel against float64

def _check_exact(q, k, v):
    assert q.shape[-1] <= 160
    for name, t in (("q", q), ("k", k)):
        assert torch.equal(t * 8, torch.round(t * 8)), f"{name} is off the 1/8 grid"
        assert t.abs().max().item() <= 4, f"|{name}| > 4: q k^T may round in fp32"
    assert torch.equal(v.half().double(), v), "v is not exact in fp16"


def _run_probe(name, B, Lq, Lk, d, H, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    Q, K, V, scale = core._probe_design(name, B, Lq, Lk, d * H, H, g)
    q, k, v = core._heads(Q, H), core._heads(K, H), core._heads(V, H)
    _check_exact(q, k, v)
    O, bound = core._reference(q, k, v, scale)
    y = core._cross_probe(Q, K, V, H, scale)
    core._assert_within(y, O, bound, f"cross probe {name} B={B} Lq={Lq} Lk={Lk} d={d} H={H}")


def _self_qkv(x, w, H):
    C = x.shape[-1]
    xd = x.double()
    q, k, v = (core._heads(xd @ w[i * C:(i + 1) * C].double().t(), H) for i in range(3))
    _check_exact(q, k, v)
    return q, k, v


def _run_self(name, B, L, d, H, seed, flags=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x, w, scale = core._self_design(name, B, L, d * H, H, g)
    q, k, v = _self_qkv(x, w, H)
    O, bound = core._reference(q, k, v, scale, qk_shared=bool(flags & 1))
    y = core._self_attention(x, w, H, scale, flags=flags)
    core._assert_within(y, O, bound, f"self-attention {name} B={B} L={L} d={d} H={H} flags={flags}")


def _bh(i, one):
    """(B, H) cycling through a covering set; a length-1 case needs B >= 2 and H >= 2."""
    cycle = ((2, 2), (3, 3), (2, 3)) if one else ((1, 1), (2, 2), (3, 3), (1, 2), (2, 3), (3, 1))
    return cycle[i % len(cycle)]


@pytest.mark.parametrize("d", WIDE)
@pytest.mark.parametrize("L", LENGTHS)
def test_self_attention_wide(L, d):
    B, H = _bh(LENGTHS.index(L) + WIDE.index(d), L == 1)
    for name in core.SELF_DESIGNS:
        _run_self(name, B, L, d, H, seed=7 * L + d)


@pytest.mark.parametrize("d", WIDE)
@pytest.mark.parametrize("L", LENGTHS)
def test_cross_probe_wide(L, d):
    """Queries and keys of the same length, then the text-context lengths below."""
    B, H = _bh(LENGTHS.index(L) + WIDE.index(d), L == 1)
    for name in core.PROBE_DESIGNS:
        _run_probe(name, B, L, L, d, H, seed=11 * L + d)


@pytest.mark.parametrize("d", WIDE)
@pytest.mark.parametrize("Lq,Lk", [(193, 77), (1000, 77), (65, 7), (1, 77), (256, 77), (64, 77)])
def test_cross_probe_context_lengths(Lq, Lk, d):
    B, H = (2, 2) if Lq == 1 else (3, 2)
    for name in core.PROBE_DESIGNS:
        _run_probe(name, B, Lq, Lk, d, H, seed=1000 * Lq + Lk + d)


@pytest.mark.parametrize("d", WIDE)
@pytest.mark.parametrize("L", (1, 65, 193, 1000))
def test_shared_qk_wide(L, d):
    """VTM_ATTN_SHARED_QK at B = 1..4: q and k of sample 0 for every sample (one CTA per sample at KS >= 6)."""
    for B in (1, 2, 3, 4):
        for name in core.SELF_DESIGNS:
            _run_self(name, B, L, d, 2, seed=L + d + B, flags=1)


@pytest.mark.parametrize("d", WIDE)
@pytest.mark.parametrize("n", (1, 63, 64, 65, 193, 449))
def test_device_length_wide(n, d):
    """vtm_attention_dev at a capacity of 449 rows with the first n valid; rows past n hold +-1000.  Rows < n meet the
    bound and equal vtm_attention_ex at L = n bit for bit."""
    cap, B, H = 449, 2, 2
    for name in core.SELF_DESIGNS:
        g = torch.Generator(device="cuda").manual_seed(n + d)
        x, w, scale = core._self_design(name, B, n, d * H, H, g)
        big = (torch.randint(0, 2, (B, cap - n, d * H), generator=g, device="cuda") * 2000 - 1000).half()
        xc = torch.cat([x, big], 1).contiguous()
        q, k, v = _self_qkv(x, w, H)
        O, bound = core._reference(q, k, v, scale)
        y = core._self_attention(xc, w, H, scale, len_dev=torch.tensor([n], dtype=torch.int32, device="cuda"))
        core._assert_within(y[:, :n], O, bound, f"device length {name} n={n} d={d}")
        assert torch.equal(y[:, :n], core._self_attention(x, w, H, scale)), f"{name} n={n} d={d}"


def test_head_dim_168_is_unsupported():
    lib = _lib.load()
    B, L, H, d = 1, 64, 2, 168
    C = H * d
    ws_bytes = lib.vtm_attention_workspace_bytes(B, L, C, H)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device="cuda")
    x = torch.zeros((B, L, C), dtype=torch.float16, device="cuda")
    w = torch.zeros((3 * C, C), dtype=torch.float16, device="cuda")
    y = torch.empty_like(x)
    rc = lib.vtm_attention_ex(x.data_ptr(), w.data_ptr(), w.data_ptr(), None, B, L, C, H, 1.0, 0, y.data_ptr(),
                              ws.data_ptr(), ws_bytes, core._stream())
    assert rc == -6                                               # VTM_E_UNSUPPORTED


# ---------------------------------------------------------------------------------------------------------------------
# SD1.5 blocks at C = 1280

class _Counter:
    """Class-level counting wrapper on skeleton.Attention.forward: counts the modules that run their own forward, by
    head_dim and kind (an instance hook would itself make the module ineligible for the library)."""

    def __init__(self, monkeypatch):
        from vidtome_b200 import skeleton
        self.calls = []
        orig = skeleton.Attention.forward
        counter = self

        def forward(mod, hidden_states, encoder_hidden_states=None, *args, **kwargs):
            d = mod.to_q.weight.shape[0] // mod.heads
            counter.calls.append((d, encoder_hidden_states is not None))
            return orig(mod, hidden_states, encoder_hidden_states, *args, **kwargs)
        monkeypatch.setattr(skeleton.Attention, "forward", forward)


def _sd15_full(max_downsample, frames=4, size=64, seed=3):
    import vidtome_b200
    from vidtome_b200.skeleton import make_skeleton
    net = make_skeleton("sd15", device="cuda", hot_path_only=False, max_downsample=max_downsample, seed=seed)
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, batch_size=2, max_downsample=max_downsample)
    g = torch.Generator(device="cuda").manual_seed(seed)
    lat = torch.randn((2 * frames, 4, size, size), generator=g, device="cuda", dtype=torch.float16)
    ctx = torch.randn((2 * frames, 77, 768), generator=g, device="cuda", dtype=torch.float16)
    return net, lat, ctx


def _fp32_attention(attn, x, ctx=None):
    """attn(x, ctx) in fp32 from the module's fp16 weights."""
    c = x if ctx is None else ctx
    B, L, C = x.shape
    h = attn.heads
    q = (x.float() @ attn.to_q.weight.float().t()).view(B, L, h, -1).transpose(1, 2)
    k = (c.float() @ attn.to_k.weight.float().t()).view(B, c.shape[1], h, -1).transpose(1, 2)
    v = (c.float() @ attn.to_v.weight.float().t()).view(B, c.shape[1], h, -1).transpose(1, 2)
    o = torch.nn.functional.scaled_dot_product_attention(q, k, v, scale=attn.scale).transpose(1, 2).reshape(B, L, C)
    return o @ attn.to_out[0].weight.float().t() + attn.to_out[0].bias.float()


@pytest.mark.parametrize("max_downsample", (4, 8))
def test_sd15_blocks_run_attention_in_the_library(max_downsample, wide_limit, monkeypatch):
    """SD1.5 ds4 (and ds8) blocks patched with max_downsample 4 / 8 and the limit at 160: every attn1 on merged tokens
    runs KD and every attn2 runs vtm_cross_attention, each within 1e-3 * max |ref| of fp32 torch attention on the same
    inputs, and no module runs its own forward.  At the default limit the d = 160 modules do."""
    from vidtome_b200 import attention
    net, lat, ctx = _sd15_full(max_downsample)
    kd, xa = [], []
    self_attention, cross_residual = attention.self_attention, attention.cross_attention_residual

    def rec_self(attn, x, shared_qk=False, seq_len=None):
        y = self_attention(attn, x, shared_qk=shared_qk, seq_len=seq_len)
        kd.append((attn, x.clone(), y.clone()))
        return y

    def rec_cross(attn, x, c, resid):
        y = cross_residual(attn, x, c, resid)
        xa.append((attn, x.clone(), c, resid.clone(), y.clone()))
        return y
    monkeypatch.setattr(attention, "self_attention", rec_self)
    monkeypatch.setattr(attention, "cross_attention_residual", rec_cross)
    count = _Counter(monkeypatch)
    with torch.no_grad():
        out = net(lat, 0, encoder_hidden_states=ctx).sample
    assert torch.isfinite(out).all()
    assert count.calls == [], count.calls
    wide_kd = [r for r in kd if r[0].heads * 160 == r[0].to_q.weight.shape[0]]
    wide_xa = [r for r in xa if r[0].heads * 160 == r[0].to_q.weight.shape[0]]
    n_wide = sum(1 for s in net.census if s.dim == 1280)
    assert len(wide_kd) == n_wide and len(wide_xa) == n_wide, (len(wide_kd), len(wide_xa), n_wide)
    with torch.no_grad():
        for attn, x, y in wide_kd:
            ref = _fp32_attention(attn, x)
            assert (y.float() - ref).abs().max().item() <= 1e-3 * ref.abs().max().item()
        for attn, x, c, resid, y in wide_xa:
            assert c.shape[1] == 77
            ref = _fp32_attention(attn, x, c) + resid.float()
            assert (y.float() - ref).abs().max().item() <= 1e-3 * ref.abs().max().item()

    # the default limit: the same network sends its d = 160 modules back to their own forward
    attention.MAX_HEAD_DIM = 128
    count.calls.clear()
    with torch.no_grad():
        net(lat, 0, encoder_hidden_states=ctx)
    assert sorted(set(count.calls)) == [(160, False), (160, True)]
    assert len(count.calls) == 2 * n_wide


# ---------------------------------------------------------------------------------------------------------------------
# the step driver

def _driver_steps(cuda_graph, steps=5, frames=8, size=32):
    """Latents of `steps` ChunkedDenoiser steps on the full SD1.5 skeleton patched with max_downsample = 8."""
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton
    torch.manual_seed(77)
    net = make_skeleton("sd15", device="cuda", hot_path_only=False)
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, batch_size=2, max_downsample=8)
    g = torch.Generator(device="cuda").manual_seed(5)
    cond = torch.randn((2, 77, 768), generator=g, device="cuda").half()
    den = ChunkedDenoiser(net, n_timesteps=50, chunk_size=4, cond=cond, cuda_graph=cuda_graph, graph_warmup=2)
    x = torch.randn((frames, 4, size, size), generator=g, device="cuda", dtype=torch.float16)
    xs = []
    for i in range(steps):
        x = den.step(x, i)
        xs.append(x.clone())
    torch.cuda.synchronize()
    return xs, den


def test_driver_graph_is_bit_identical_to_eager(wide_limit, monkeypatch):
    count = _Counter(monkeypatch)
    eager, _ = _driver_steps(False)
    assert count.calls == [], "a module ran its own attention"
    graph, den = _driver_steps(True)
    assert den._graph is not None, "the graph was never captured"
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(a).all(), i
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"


def _pnp_run(chunk_graphs, steps=6, frames=8, size=32):
    import numpy as np
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton, pnp_attention_modules
    torch.manual_seed(77)
    net = make_skeleton("sd15", device="cuda", max_downsample=4)           # PnP targets at C 1280, 640 and 320
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=True, global_merge_ratio=0.8, global_rand=0.5,
                             batch_size=3, align_batch=True, max_downsample=4)
    g = torch.Generator(device="cuda").manual_seed(5)
    cond = torch.randn((3, 77, 768), generator=g, device="cuda").half()
    sources = {}

    def source(t):
        if t not in sources:
            gs = torch.Generator(device="cuda").manual_seed(int(t))
            sources[t] = torch.randn((frames, 4, size, size), generator=gs, device="cuda").half()
        return sources[t]
    mods = pnp_attention_modules(net)
    den = ChunkedDenoiser(net, n_timesteps=steps, chunk_size=4, merge_global=True, chunk_ord="mix-4", cond=cond,
                          source_latents=source,
                          pnp_attn_t=0.5, pnp_modules=mods, cuda_graph=chunk_graphs, graph_warmup=1,
                          randomize_chunks=True, chunk_graphs=chunk_graphs)
    x = torch.randn((frames, 4, size, size), generator=g, device="cuda", dtype=torch.float16)
    torch.manual_seed(2024)
    np.random.seed(2024)
    xs, keys = [], []
    for i in range(steps):
        x = den.step(x, i)
        xs.append(x.clone())
        keys.append(sorted(den._chunk_graphs) if chunk_graphs else None)
    torch.cuda.synchronize()
    return xs, keys, mods


def test_pnp_chunk_graphs_bit_identical_to_eager_with_wide_modules(wide_limit, monkeypatch):
    """PnP with max_downsample = 4 and global merging: the injected d = 160 modules of up_blocks[1] run KD with the
    shared map inside their merged blocks (under the chunk graphs on the GlobalTokenStore's device length), and chunk
    graphs equal eager stepping across the injection boundary."""
    from vidtome_b200 import attention
    shared, device_length = [], []
    self_attention = attention.self_attention

    def rec(attn, x, shared_qk=False, seq_len=None):
        if attn.to_q.weight.shape[0] == 160 * attn.heads:
            shared.append(shared_qk)
            device_length.append(seq_len is not None)
        return self_attention(attn, x, shared_qk=shared_qk, seq_len=seq_len)
    monkeypatch.setattr(attention, "self_attention", rec)
    count = _Counter(monkeypatch)
    eager, _, mods = _pnp_run(False)
    assert any(m.to_q.weight.shape[0] == 160 * m.heads for m in mods)
    assert True in shared and False in shared, "the d = 160 modules never ran KD with and without injection"
    assert count.calls == [], "a module ran its own attention"
    graph, keys, _ = _pnp_run(True)
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(b).all(), i
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"
    assert any(k[3] for k in keys[2]), "no injected chunk graph was captured"
    assert any(device_length), "the d = 160 modules never ran on a device-length token set"


_CHILD = r"""
import sys, torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
from vidtome_b200 import attention
attention.MAX_HEAD_DIM = 160
import test_gpu_attention_wide as t
xs, _ = t._driver_steps(False, steps=3)
torch.save([x.cpu() for x in xs], sys.argv[2])
"""


def test_eager_steps_identical_across_processes(tmp_path):
    """Two processes run the same eager steps from the same seeds with no torch attention left in the step; their
    latents are bit-identical."""
    outs = []
    for i in range(2):
        path = str(tmp_path / f"latents{i}.pt")
        r = subprocess.run([sys.executable, "-c", _CHILD, ROOT, path], cwd=ROOT, capture_output=True, text=True,
                           timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        outs.append(torch.load(path))
    for i, (a, b) in enumerate(zip(*outs)):
        assert torch.isfinite(a.float()).all(), i
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"
