"""SD2-depth on the GPU: ChunkedDenoiser(depth=...) and ChunkedInverter(depth=...) on the SD2.1-census depth skeleton
(5 input channels, linear Transformer2DModel IO, cross-attention and feed-forward) in CUDA fp16, patched with
apply_patch.  Every graph mode gives latents bit-identical to eager stepping with a distinct depth map per frame, the
depth maps reach the model in each mode, PnP with conv injection combines with depth, and the captured inversion step
gives the eager trajectory."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

STEPS = 6                 # one eager warm-up step, then five from graphs
SIZE = 16                 # latent 16 x 16


def _depth(frames, flip=False):
    g = torch.Generator(device="cuda").manual_seed(9)
    d = (torch.rand((frames, 1, SIZE, SIZE), generator=g, device="cuda") * 2 - 1)      # prepare_depth's range, fp32
    return d.flip(0) if flip else d


def _run(mode, frames=8, flip=False, pnp=False):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton, pnp_attention_modules, pnp_conv_module
    torch.manual_seed(77)
    net = make_skeleton("sd21", device="cuda", hot_path_only=False, transformer_io="linear", depth=True, pnp_conv=pnp)
    merge_global = mode in ("capture_global", "eager_global", "chunk_graphs", "eager_flamingo")
    bs = 3 if pnp else 2
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=merge_global, global_merge_ratio=0.9,
                             global_rand=0.5, batch_size=bs, align_batch=pnp)
    g = torch.Generator(device="cuda").manual_seed(5)
    cond = torch.randn((bs, 77, 1024), generator=g, device="cuda").half()
    graph = not mode.startswith("eager")
    kw = dict(cuda_graph=graph, graph_warmup=1, chunk_ord="mix-4")
    if mode in ("chunk_graphs", "eager_flamingo"):                   # configs/flamingo.yaml
        kw.update(randomize_chunks=True, chunk_graphs=graph, chunk_ord="rand")
    if mode in ("capture_global", "eager_global"):
        kw.update(capture_global=graph)
    if pnp:
        sources = {}

        def source(t):
            if t not in sources:
                gs = torch.Generator(device="cuda").manual_seed(int(t))
                sources[t] = torch.randn((frames, 4, SIZE, SIZE), generator=gs, device="cuda").half()
            return sources[t]
        kw.update(source_latents=source, pnp_attn_t=0.5, pnp_modules=pnp_attention_modules(net), pnp_f_t=0.8,
                  pnp_conv_modules=[pnp_conv_module(net)])
    den = ChunkedDenoiser(net, n_timesteps=STEPS, chunk_size=4, merge_global=merge_global, cond=cond,
                          depth=_depth(frames, flip), **kw)
    x = torch.randn((frames, 4, SIZE, SIZE), generator=g, device="cuda", dtype=torch.float16)
    torch.manual_seed(2024)              # the device RNG the blocks fork from
    np.random.seed(2024)                 # the host draws of get_chunks
    xs = []
    for i in range(STEPS):
        x = den.step(x, i)
        xs.append(x.clone())
    torch.cuda.synchronize()
    return xs, den


def _assert_identical(eager, graph):
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(b).all(), i
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"


@pytest.mark.parametrize("mode,eager_mode,frames", [("step_graph", "eager_plain", 8),
                                                    ("capture_global", "eager_global", 8),
                                                    ("chunk_graphs", "eager_flamingo", 10)])
def test_graph_modes_bit_identical_to_eager_and_depth_reaches_the_model(mode, eager_mode, frames):
    eager, _ = _run(eager_mode, frames)
    graph, den = _run(mode, frames)
    if mode == "chunk_graphs":
        assert den._chunk_graphs, "no chunk graph was captured"
    else:
        assert den._graph is not None
    _assert_identical(eager, graph)
    # the same frames' depth maps in another order give other latents, eagerly and from graphs
    eager_flip, _ = _run(eager_mode, frames, flip=True)
    graph_flip, _ = _run(mode, frames, flip=True)
    assert not torch.equal(eager[0], eager_flip[0])
    assert not torch.equal(graph[-1], graph_flip[-1])
    _assert_identical(eager_flip, graph_flip)


def test_pnp_with_depth_bit_identical_to_eager():
    eager, den_e = _run("eager_plain", pnp=True)
    assert den_e.pnp_schedule == den_e.timesteps[:3] and den_e.pnp_conv_schedule == den_e.timesteps[:4]
    graph, den = _run("step_graph", pnp=True)
    assert den._graph[4] == (tuple(graph[0].shape), False, False)       # the last step's key: neither injection
    _assert_identical(eager, graph)


def test_inverter_graph_bit_identical_to_eager_with_a_ragged_batch():
    import vidtome_b200
    from vidtome_b200.driver import ChunkedInverter
    from vidtome_b200.skeleton import make_skeleton
    net = make_skeleton("sd21", device="cuda", hot_path_only=False, transformer_io="linear", depth=True)
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, batch_size=2)
    g = torch.Generator(device="cuda").manual_seed(3)
    frames = 10
    x = torch.randn((frames, 4, SIZE, SIZE), generator=g, device="cuda").half()
    cond = torch.randn((frames, 77, 1024), generator=g, device="cuda").half()
    kw = dict(n_timesteps=8, batch_size=4, cond=cond)
    eager = ChunkedInverter(net, depth=_depth(frames), **kw)
    eager.invert(x)
    graph = ChunkedInverter(net, cuda_graph=True, graph_warmup=2, depth=_depth(frames), **kw)
    graph.invert(x)
    assert graph.trajectory.shape[2] == 4
    assert torch.isfinite(graph.trajectory).all()
    assert torch.equal(eager.trajectory, graph.trajectory)
    flipped = ChunkedInverter(net, cuda_graph=True, graph_warmup=2, depth=_depth(frames, flip=True), **kw)
    flipped.invert(x)
    assert not torch.equal(flipped.trajectory[-1], graph.trajectory[-1])
