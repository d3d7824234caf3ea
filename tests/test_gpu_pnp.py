"""PnP on the GPU: the grouped shared-map flash kernel (one CTA serves several samples with one attention map) against
the per-sample kernel, and ChunkedDenoiser(source_latents=...) eager and from every graph mode."""
import numpy as np
import pytest
import torch

from vidtome_b200 import _lib

pytestmark = pytest.mark.gpu

SHARED_QK = 1


# --------------------------------------------------------------------------- 1. kernel bit-identity
def _stream():
    return torch.cuda.current_stream().cuda_stream


def _attention(x, w_qkv, heads, flags, len_dev=None):
    """vtm_attention_ex / vtm_attention_dev with W_o = I, no bias, a 0xFF (fp16 NaN) workspace and a NaN output."""
    lib = _lib.load()
    B, L, C = x.shape
    ws_bytes = lib.vtm_attention_workspace_bytes(B, L, C, heads)
    ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device="cuda")
    y = torch.full_like(x, float("nan"))
    wo = torch.eye(C, dtype=torch.float16, device="cuda")
    scale = (C // heads) ** -0.5
    if len_dev is None:
        _lib.check(lib.vtm_attention_ex(x.data_ptr(), w_qkv.data_ptr(), wo.data_ptr(), None, B, L, C, heads, scale,
                                        flags, y.data_ptr(), ws.data_ptr(), ws_bytes, _stream()), "vtm_attention_ex")
    else:
        _lib.check(lib.vtm_attention_dev(x.data_ptr(), w_qkv.data_ptr(), wo.data_ptr(), None, B, L, C, heads, scale,
                                         flags, len_dev.data_ptr(), y.data_ptr(), ws.data_ptr(), ws_bytes, _stream()),
                   "vtm_attention_dev")
    torch.cuda.synchronize()
    return y


def _split_problem(B, L, d, seed):
    """Two heads of head_dim d.  q / k rows of W_qkv read only the first half of the channels, v rows only the second
    half; every sample has the first half of sample 0.  The per-sample kernel then computes exactly the shared
    semantics.  Returns (x with equal first halves, x whose other samples' first halves differ, W_qkv)."""
    heads, C = 2, 2 * d
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = torch.randn((3 * C, C), generator=g, device="cuda") * (C // 2) ** -0.5
    w[:2 * C, C // 2:] = 0
    w[2 * C:, :C // 2] = 0
    x = torch.randn((B, L, C), generator=g, device="cuda").half()
    x[:, :, :C // 2] = x[:1, :, :C // 2]
    other = x.clone()
    other[1:, :, :C // 2] = torch.randn((B - 1, L, C // 2), generator=g, device="cuda").half()
    return x, other, w.half(), heads


@pytest.mark.parametrize("d", list(range(8, 129, 8)))
def test_shared_kernel_is_bit_identical_to_per_sample_kernel(d):
    for B in (1, 2, 3, 4):
        for L in (1, 63, 64, 65, 191, 192, 193, 3001):
            x, other, w, heads = _split_problem(B, L, d, seed=1000 * d + 10 * B + L)
            want = _attention(x, w, heads, 0)
            assert torch.isfinite(want).all(), (B, L)
            for inp in (x, other) if B > 1 else (x,):
                got = _attention(inp, w, heads, SHARED_QK)
                assert torch.equal(got, want), (B, L, (got.float() - want.float()).abs().max().item())


@pytest.mark.parametrize("d", list(range(8, 129, 8)))
def test_shared_kernel_with_device_length(d):
    cap, n = 300, 193
    for B in (1, 2, 3, 4):
        x, other, w, heads = _split_problem(B, cap, d, seed=7 * d + B)
        len_dev = torch.tensor([n], dtype=torch.int32, device="cuda")
        want = _attention(x[:, :n].contiguous(), w, heads, 0)
        for inp in (x, other) if B > 1 else (x,):
            got = _attention(inp, w, heads, SHARED_QK, len_dev=len_dev)
            assert torch.equal(got[:, :n], want), B


# --------------------------------------------------------------------------- 2. the driver
STEPS = 6              # pnp_attn_t 0.5: steps 0-2 inject, 3-5 do not


def _run(mode, frames=8, size=16, record=None):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton, pnp_attention_modules
    torch.manual_seed(77)
    net = make_skeleton("sd15", device="cuda", max_downsample=2)           # PnP targets at C 640 and 320
    merge_global = mode not in ("step_graph", "eager_plain")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=merge_global, global_merge_ratio=0.8,
                             global_rand=0.5, batch_size=3, align_batch=True)
    g = torch.Generator(device="cuda").manual_seed(5)
    cond = torch.randn((3, 77, 768), generator=g, device="cuda").half()
    sources = {}

    def source(t):
        if t not in sources:
            gs = torch.Generator(device="cuda").manual_seed(int(t))
            sources[t] = torch.randn((frames, 4, size, size), generator=gs, device="cuda").half()
        return sources[t]
    graph = not mode.startswith("eager")
    kw = dict(cuda_graph=graph, graph_warmup=1)
    if mode in ("chunk_graphs", "eager_random"):
        kw.update(randomize_chunks=True, chunk_graphs=graph)
    if mode in ("capture_global", "eager_global"):
        kw.update(capture_global=graph)
    den = ChunkedDenoiser(net, n_timesteps=STEPS, chunk_size=4, merge_global=merge_global, chunk_ord="mix-4",
                          cond=cond, source_latents=source, pnp_attn_t=0.5, pnp_modules=pnp_attention_modules(net), **kw)
    if record is not None:
        def hook(module, args, kwargs):
            record.append((args[0].clone(), kwargs.get("encoder_hidden_states")))
        net.register_forward_pre_hook(hook, with_kwargs=True)
    x = torch.randn((frames, 4, size, size), generator=g, device="cuda", dtype=torch.float16)
    torch.manual_seed(2024)
    np.random.seed(2024)
    xs, keys = [], []
    for i in range(STEPS):
        x = den.step(x, i)
        xs.append(x.clone())
        keys.append(sorted(den._chunk_graphs) if mode == "chunk_graphs" else
                    (den._graph[4] if graph and den._graph is not None else None))
    torch.cuda.synchronize()
    return xs, keys, den, sources


@pytest.mark.parametrize("mode,eager_mode", [("step_graph", "eager_plain"), ("capture_global", "eager_global"),
                                             ("chunk_graphs", "eager_random")])
def test_driver_graph_modes_are_bit_identical_to_eager_across_the_injection_boundary(mode, eager_mode):
    eager, _, den_e, _ = _run(eager_mode)
    assert den_e.pnp_schedule == den_e.timesteps[:3]
    graph, keys, den, _ = _run(mode)
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(b).all(), i
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"
    if mode == "chunk_graphs":
        assert any(k[3] for k in keys[2]), "no injected chunk graph was captured"
        assert keys[-1] and not any(k[3] for k in keys[-1]), "injected chunk graphs outlived the schedule"
    else:
        assert keys[2][1] is True and keys[-1][1] is False, keys


def test_unet_sees_source_then_cfg_batch_with_three_row_conditioning():
    record = []
    _, _, den, sources = _run("eager_random", record=record)
    assert record
    cond = den.cond
    for sample, text in record:
        m = sample.shape[0] // 3
        assert sample.shape[0] == 3 * m and text.shape == (3 * m, 77, 768)
        assert torch.equal(sample[m:2 * m], sample[2 * m:])
        assert torch.equal(text, cond.repeat_interleave(m, dim=0))
        assert any(torch.equal(sample[:m], s[lo:lo + m]) for s in sources.values() for lo in range(len(s) - m + 1))
