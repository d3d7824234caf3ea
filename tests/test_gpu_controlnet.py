"""ControlNet control on the GPU: ChunkedDenoiser(controlnet=..., control_images=...) on sd15 skeletons (skeleton.
make_controlnet for the ControlNet) with 4-frame chunks, eager and from every graph mode, with the ControlNet left
unpatched (the reference's default) and patched through apply_patch(include_control=True)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

STEPS = 7              # graph_warmup 2: steps 0-1 eager, capture at step 2, replays after


def _pipeline(include_control, merge_global, hot_path_only=True):
    import vidtome_b200
    from vidtome_b200.skeleton import make_controlnet, make_skeleton

    class DiffusionPipeline:
        pass

    class StableDiffusionControlNetPipeline(DiffusionPipeline):
        def __init__(self):
            self.unet = make_skeleton("sd15", hot_path_only=hot_path_only, device="cuda")
            self.controlnet = make_controlnet("sd15", hot_path_only=hot_path_only, device="cuda")
    pipe = StableDiffusionControlNetPipeline()
    vidtome_b200.apply_patch(pipe, local_merge_ratio=0.9, merge_global=merge_global, global_merge_ratio=0.8,
                             global_rand=0.5, batch_size=2, include_control=include_control)
    return pipe


# mode -> (graph, merge_global, randomize_chunks)
MODES = {"eager_plain": (False, False, False), "step_graph": (True, False, False),
         "eager_global": (False, True, False), "capture_global": (True, True, False),
         "eager_random": (False, True, True), "chunk_graphs": (True, True, True),
         "eager_random_local": (False, False, True), "chunk_graphs_local": (True, False, True)}


def _run(mode, include_control, scale=1.0, with_controlnet=True, frames=8, size=16, steps=STEPS, hook=None):
    from vidtome_b200.driver import ChunkedDenoiser
    graph, merge_global, randomize = MODES[mode]
    torch.manual_seed(77)
    pipe = _pipeline(include_control, merge_global)
    g = torch.Generator(device="cuda").manual_seed(5)
    cond = torch.randn((2, 77, 768), generator=g, device="cuda").half()
    ctrl = torch.rand((frames, 3, 8 * size, 8 * size), generator=g, device="cuda").half()
    kw = dict(cuda_graph=graph, graph_warmup=2, randomize_chunks=randomize)
    if graph and randomize:
        kw.update(chunk_graphs=True)
    elif graph and merge_global:
        kw.update(capture_global=True)
    if with_controlnet:
        kw.update(controlnet=pipe.controlnet, control_images=ctrl, control_scale=scale)
    den = ChunkedDenoiser(pipe.unet, n_timesteps=50, chunk_size=4, merge_global=merge_global, chunk_ord="mix-4",
                          cond=cond, **kw)
    if hook is not None:
        hook(den, pipe)
    x = torch.randn((frames, 4, size, size), generator=g, device="cuda", dtype=torch.float16)
    torch.manual_seed(2024)
    np.random.seed(2024)
    xs = []
    for i in range(steps):
        x = den.step(x, i)
        xs.append(x.clone())
    torch.cuda.synchronize()
    return xs, den, pipe


@pytest.mark.parametrize("include_control", [False, True])
def test_residuals_change_the_prediction(include_control):
    one, _, _ = _run("eager_plain", include_control, scale=1.0, steps=2)
    zero, _, _ = _run("eager_plain", include_control, scale=0.0, steps=2)
    none, _, _ = _run("eager_plain", include_control, with_controlnet=False, steps=2)
    for a in one + zero:
        assert torch.isfinite(a).all()
    assert not torch.equal(one[-1], zero[-1])
    for a, b in zip(zero, none):
        assert torch.equal(a, b), (a.float() - b.float()).abs().max().item()


@pytest.mark.parametrize("include_control", [False, True])
@pytest.mark.parametrize("mode,eager_mode", [("step_graph", "eager_plain"), ("capture_global", "eager_global"),
                                             ("chunk_graphs", "eager_random"),
                                             ("chunk_graphs_local", "eager_random_local")])
def test_graph_modes_are_bit_identical_to_eager(mode, eager_mode, include_control):
    eager, _, _ = _run(eager_mode, include_control)
    graph, den, pipe = _run(mode, include_control)
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(b).all(), i
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"
    cn_gens = {id(m.generator) for m in pipe.controlnet.modules() if type(m).__name__ == "ToMeBlock"}
    assert len(cn_gens) == (7 if include_control else 0)
    assert cn_gens <= {id(g) for g in den._block_generators()}
    if mode == "chunk_graphs":
        assert den._chunk_graphs


def _cn_blocks(pipe):
    return [m for m in pipe.controlnet.modules() if type(m).__name__ == "ToMeBlock"]


@pytest.mark.parametrize("mode", ["eager_global", "chunk_graphs"])
def test_global_reset_between_steps_reaches_the_controlnet(mode):
    """The first ControlNet call of every step finds its blocks' global tokens empty, the later ones find them set:
    the reset after each step reaches the patched ControlNet (update_patch eagerly, the stores under chunk_graphs).
    The hook runs on the two eager warm-up steps only (a graph replay runs no Python)."""
    seen = []

    def hook(den, pipe):
        def pre(module, args):
            g = getattr(module, "global_tokens", None)
            seen.append(g is not None and getattr(g, "filled", True))
        _cn_blocks(pipe)[0].register_forward_pre_hook(pre)
    _, den, pipe = _run(mode, True, steps=2, hook=hook)
    if mode == "eager_global":                                  # 2 steps of two 4-frame chunks
        assert seen == [False, True] * 2, seen
        assert all(b.global_tokens is None for b in _cn_blocks(pipe))
    else:                                                       # 2 steps of 2 or 3 chunks (random first chunk)
        firsts = [i for i, s in enumerate(seen) if not s]
        assert len(firsts) == 2 and firsts[0] == 0 and firsts[1] >= 2, seen
        stores = [b.global_tokens for b in _cn_blocks(pipe)]
        assert len(stores) == 7 and all(any(st is s for s in den._stores) for st in stores)
        assert not any(st.filled for st in den._stores)


def test_controlnet_blocks_draw_from_their_own_generators():
    states = []

    def hook(den, pipe):
        def post(module, args, out):
            states.append([b.generator.get_state().clone() for b in _cn_blocks(pipe)])
        pipe.controlnet.register_forward_hook(post)
    _, den, pipe = _run("eager_plain", True, steps=2, hook=hook)
    blocks = _cn_blocks(pipe)
    unet_gens = {id(m.generator) for m in pipe.unet.modules() if type(m).__name__ == "ToMeBlock"}
    assert len({id(b.generator) for b in blocks}) == 7 and not unet_gens & {id(b.generator) for b in blocks}
    assert all(b.generator.device.type == "cuda" for b in blocks)
    # the merged ControlNet blocks (ds 1 and 2: the first four) advance their generators call by call
    for a, b in zip(states, states[1:]):
        assert all(not torch.equal(sa, sb) for sa, sb in zip(a[:4], b[:4]))


@pytest.mark.parametrize("include_control", [False, True])
def test_c3_hot_workload_graph_equals_eager(include_control):
    """BASELINE config 3 shape with the ControlNet branch: 32 frames of 512x512 (latent 64) in 4-frame chunks, local 0.9
    + global 0.8, eager against capture_global over the warm-up/capture boundary."""
    eager, _, _ = _run("eager_global", include_control, frames=32, size=64, steps=4)
    graph, _, _ = _run("capture_global", include_control, frames=32, size=64, steps=4)
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(b).all(), i
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"
