"""patch.FUSE_CONTROLNET_BLOCKS and patch.serve_unmerged / unserve_unmerged without a GPU: the class swap and its undo on
the skeleton ControlNet, what serving leaves untouched (parameters, generators, global tokens, hooks), the refusal of
patched models, the step drivers' lazy serving, and which forward each served module takes, with the library calls
replaced by recorders (the eligibility tests read shapes, types and flags, never the device)."""
import pytest
import torch

import vidtome_b200
from vidtome_b200 import attention, feedforward, ops, patch, transformer2d
from vidtome_b200.driver import ChunkedDenoiser, ChunkedInverter
from vidtome_b200.skeleton import Attention, BasicTransformerBlock, Transformer2DModel, make_controlnet


@pytest.fixture
def switch():
    saved = patch.FUSE_CONTROLNET_BLOCKS, patch.FUSE_TRANSFORMER_IO, attention.MAX_HEAD_DIM
    yield
    patch.FUSE_CONTROLNET_BLOCKS, patch.FUSE_TRANSFORMER_IO, attention.MAX_HEAD_DIM = saved


def _classes(net):
    return {name: type(m) for name, m in net.named_modules()}


def _cn(transformer_io="conv", hot_path_only=False):
    return make_controlnet("tiny", hot_path_only=hot_path_only, device="cpu", dtype=torch.float32,
                           transformer_io=transformer_io)


def test_switch_is_off_by_default():
    assert patch.FUSE_CONTROLNET_BLOCKS is False


@pytest.mark.parametrize("transformer_io", [None, "conv", "linear"])
def test_serve_swaps_the_classes_and_unserve_restores_them(transformer_io):
    cn = _cn(transformer_io)
    before = _classes(cn)
    state = {k: v.clone() for k, v in cn.state_dict().items()}
    assert patch.serve_unmerged(cn) is cn
    assert patch.is_served(cn) and not patch.is_patched(cn)
    served = _classes(cn)
    for name, m in cn.named_modules():
        if before[name] is BasicTransformerBlock:
            assert type(m).__name__ == "UnmergedBlock" and m._parent is BasicTransformerBlock
            assert isinstance(m, BasicTransformerBlock)
        elif before[name] is Transformer2DModel:
            assert type(m).__name__ == "UnmergedTransformer2D" and m._parent is Transformer2DModel
        else:
            assert served[name] is before[name], name
    assert sum(type(m).__name__ == "UnmergedBlock" for m in cn.modules()) == len(cn.blocks)
    assert sum(type(m).__name__ == "UnmergedTransformer2D" for m in cn.modules()) == (
        0 if transformer_io is None else len(cn.blocks))
    # the parameters and buffers are the model's own, under the same names
    after = cn.state_dict()
    assert list(after) == list(state)
    assert all(after[k].data_ptr() == cn.state_dict()[k].data_ptr() and torch.equal(after[k], state[k]) for k in state)
    # serving again changes nothing
    patch.serve_unmerged(cn)
    assert _classes(cn) == served
    assert patch.unserve_unmerged(cn) is cn
    assert _classes(cn) == before and not patch.is_served(cn)
    assert all(torch.equal(cn.state_dict()[k], state[k]) for k in state)


def test_serving_adds_no_state_and_draws_nothing(switch):
    cn = _cn()
    attrs = {name: set(vars(m)) for name, m in cn.named_modules()}
    patch.serve_unmerged(cn)
    patch.FUSE_CONTROLNET_BLOCKS = True
    cpu_state = torch.get_rng_state()
    g = torch.Generator().manual_seed(0)
    x = torch.randn((2, 4, 8, 8), generator=g)
    ctx = torch.randn((2, 77, 768), generator=g)
    ctrl = torch.rand((2, 3, 64, 64), generator=g)
    with torch.no_grad():
        cn(x, 10, encoder_hidden_states=ctx, controlnet_cond=ctrl)
    assert torch.equal(torch.get_rng_state(), cpu_state)
    for name, m in cn.named_modules():
        assert set(vars(m)) == attrs[name], name                    # no generator, global_tokens or _tome_info
        assert not hasattr(m, "generator") and not hasattr(m, "global_tokens") and not hasattr(m, "_tome_info")
        assert not m._forward_pre_hooks and not m._forward_hooks, name


def _pipeline(transformer_io="conv"):
    class DiffusionPipeline:
        pass

    class StableDiffusionControlNetPipeline(DiffusionPipeline):       # apply_patch matches the class name
        def __init__(self):
            self.unet = make_controlnet("tiny", device="cpu", dtype=torch.float32)
            self.controlnet = _cn(transformer_io)
    return StableDiffusionControlNetPipeline()


def test_a_patched_model_is_refused():
    pipe = _pipeline()
    vidtome_b200.apply_patch(pipe, include_control=True)
    patched = _classes(pipe.controlnet)
    with pytest.raises(ValueError, match="apply_patch"):
        patch.serve_unmerged(pipe.controlnet)
    with pytest.raises(ValueError, match="remove_patch"):
        patch.unserve_unmerged(pipe.controlnet)
    assert _classes(pipe.controlnet) == patched
    # include_control=False leaves the ControlNet unpatched: it may be served
    pipe = _pipeline()
    vidtome_b200.apply_patch(pipe)
    assert not patch.is_patched(pipe.controlnet)
    patch.serve_unmerged(pipe.controlnet)
    with pytest.raises(ValueError):
        patch.serve_unmerged(pipe.unet)


def test_a_removed_patch_may_be_served():
    cn = _cn()
    before = _classes(cn)
    vidtome_b200.apply_patch(cn)
    vidtome_b200.remove_patch(cn)
    assert _classes(cn) == before and not patch.is_patched(cn)
    patch.serve_unmerged(cn)
    patch.unserve_unmerged(cn)
    assert _classes(cn) == before


@pytest.mark.parametrize("on", [False, True])
def test_served_model_on_cpu_computes_its_own_forward(switch, on):
    """Off the device every served module runs its own forward, bit for bit, whatever the switch."""
    cn = _cn()
    g = torch.Generator().manual_seed(1)
    x = torch.randn((2, 4, 8, 8), generator=g)
    ctx = torch.randn((2, 77, 768), generator=g)
    ctrl = torch.rand((2, 3, 64, 64), generator=g)
    with torch.no_grad():
        down, mid = cn(x, 10, encoder_hidden_states=ctx, controlnet_cond=ctrl)
        patch.serve_unmerged(cn)
        patch.FUSE_CONTROLNET_BLOCKS = on
        down2, mid2 = cn(x, 10, encoder_hidden_states=ctx, controlnet_cond=ctrl)
    assert torch.equal(mid, mid2) and all(torch.equal(a, b) for a, b in zip(down, down2))


# ------------------------------------------------------------------------------------------------ the drivers
def _driver_inputs():
    g = torch.Generator().manual_seed(3)
    return (torch.randn((4, 4, 8, 8), generator=g), torch.rand((4, 3, 64, 64), generator=g),
            torch.randn((2, 77, 768), generator=g))


@pytest.mark.parametrize("on", [False, True])
def test_denoiser_serves_lazily_and_close_restores(switch, on):
    unet = vidtome_b200.skeleton.make_skeleton("tiny", device="cpu", dtype=torch.float32)
    cn = _cn(None)
    before = _classes(cn)
    x, images, cond = _driver_inputs()
    patch.FUSE_CONTROLNET_BLOCKS = on
    den = ChunkedDenoiser(unet, n_timesteps=2, chunk_size=2, cond=cond, controlnet=cn, control_images=images)
    assert _classes(cn) == before                                   # nothing happens before the first step
    den.step(x, 0)
    assert patch.is_served(cn) is on
    den.close()
    assert _classes(cn) == before
    den.step(x, 1)                                                  # serves again after close()
    assert patch.is_served(cn) is on
    den.close()


def test_denoiser_leaves_a_served_or_patched_controlnet_alone(switch):
    patch.FUSE_CONTROLNET_BLOCKS = True
    unet = vidtome_b200.skeleton.make_skeleton("tiny", device="cpu", dtype=torch.float32)
    x, images, cond = _driver_inputs()
    cn = patch.serve_unmerged(_cn(None))
    served = _classes(cn)
    den = ChunkedDenoiser(unet, n_timesteps=2, chunk_size=2, cond=cond, controlnet=cn, control_images=images)
    den.step(x, 0)
    den.close()
    assert _classes(cn) == served                                   # the caller's serving outlives the driver
    pipe = _pipeline(None)
    vidtome_b200.apply_patch(pipe, include_control=True, batch_size=2, max_downsample=0)   # no block merges on the CPU
    patched = _classes(pipe.controlnet)
    den = ChunkedDenoiser(unet, n_timesteps=2, chunk_size=2, cond=cond, controlnet=pipe.controlnet,
                          control_images=images)
    den.step(x, 0)
    den.close()
    assert _classes(pipe.controlnet) == patched


@pytest.mark.parametrize("on", [False, True])
def test_inverter_serves_lazily_and_close_restores(switch, on):
    unet = vidtome_b200.skeleton.make_skeleton("tiny", device="cpu", dtype=torch.float32)
    cn = _cn(None)
    before = _classes(cn)
    x, images, cond = _driver_inputs()
    patch.FUSE_CONTROLNET_BLOCKS = on
    inv = ChunkedInverter(unet, n_timesteps=2, batch_size=2, cond=cond[:1], controlnet=cn, control_images=images)
    assert _classes(cn) == before
    inv.invert(x)
    assert patch.is_served(cn) is on
    inv.close()
    assert _classes(cn) == before


# ------------------------------------------------------------------------------------------------ dispatch
class Recorder:
    """Stands in for the library calls and for the modules' own forwards; `calls` lists (what, batch)."""

    def __init__(self, monkeypatch):
        self.calls = []
        monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
        monkeypatch.setattr(ops, "layer_norm", lambda x, ln: x)
        monkeypatch.setattr(attention, "self_attention_residual", self.rec("attn1_library", 2))
        monkeypatch.setattr(attention, "cross_attention_residual", self.rec("attn2_library", 3))
        monkeypatch.setattr(feedforward, "feed_forward_residual", self.rec("ff_library", 3))
        monkeypatch.setattr(transformer2d, "library_forward", self.wrapper_library)
        monkeypatch.setattr(Attention, "forward", self.module_attention)
        monkeypatch.setattr(patch, "build_merge_plan", self.plan)
        block_forward = BasicTransformerBlock.forward
        wrapper_forward = Transformer2DModel.forward

        def own_block(blk, x, *a, **k):
            self.calls.append(("block_own", x.shape[0]))
            return block_forward(blk, x, *a, **k)

        def own_wrapper(w, x, *a, **k):
            self.calls.append(("wrapper_own", x.shape[0]))
            return wrapper_forward(w, x, *a, **k)
        monkeypatch.setattr(BasicTransformerBlock, "forward", own_block)
        monkeypatch.setattr(Transformer2DModel, "forward", own_wrapper)

    def rec(self, what, resid_arg):
        """A library call whose argument `resid_arg` is the residual: recorded by its batch, returns residual + 1."""
        def fn(*args, **kwargs):
            self.calls.append((what, args[resid_arg].shape[0]))
            return args[resid_arg] + 1
        return fn

    def plan(self, *a, **k):
        raise AssertionError("a served block built a merge plan")

    def module_attention(self, x, encoder_hidden_states=None, attention_mask=None, **kw):
        self.calls.append(("attn_module", x.shape[0]))
        return torch.zeros_like(x)

    def wrapper_library(self, module, x, **kwargs):
        self.calls.append(("wrapper_library", x.shape[0]))
        if not kwargs.get("return_dict", True):
            return (x + 1,)
        return transformer2d.Transformer2DModelOutput(sample=x + 1)


def _served_block(dim=320, heads=8, hot_path_only=False):
    torch.manual_seed(0)
    blk = BasicTransformerBlock(dim, heads, hot_path_only=hot_path_only).half().eval()
    blk.__class__ = patch.make_unmerged_block(blk.__class__)
    return blk


def _x(B, tokens=16, dim=320, dtype=torch.float16):
    return torch.randn(B, tokens, dim).to(dtype)


def _ctx(B):
    return torch.randn(B, 77, 768).half()


LIBRARY = [("attn1_library", 4), ("attn2_library", 4), ("ff_library", 4)]


def test_switch_off_runs_the_block_class_forward(switch, monkeypatch):
    rec = Recorder(monkeypatch)
    blk = _served_block()
    blk(_x(4), encoder_hidden_states=_ctx(4))
    assert rec.calls == [("block_own", 4), ("attn_module", 4), ("attn_module", 4)]


def test_switch_on_runs_every_stage_in_the_library(switch, monkeypatch):
    rec = Recorder(monkeypatch)
    patch.FUSE_CONTROLNET_BLOCKS = True
    blk = _served_block()
    x = _x(4)
    y = blk(x, encoder_hidden_states=_ctx(4), timestep=None)
    assert rec.calls == LIBRARY
    assert torch.equal(y, x + 1 + 1 + 1)
    # the hot-path-only block (no attn2, no ff) stops after the self-attention
    rec.calls.clear()
    blk = _served_block(hot_path_only=True)
    blk(x)
    assert rec.calls == [("attn1_library", 4)]


@pytest.mark.parametrize("call", ["mask", "encoder_mask", "cross_kwargs", "positional", "unknown_kwarg", "fp32",
                                  "ada", "ada_zero", "only_cross", "old_flags", "training"])
def test_ineligible_calls_run_the_block_class_forward(switch, monkeypatch, call):
    rec = Recorder(monkeypatch)
    patch.FUSE_CONTROLNET_BLOCKS = True
    blk = _served_block(hot_path_only=True)
    x, kw, args = _x(4), {}, ()
    if call == "mask":
        kw["attention_mask"] = torch.zeros(4, 16, 16).half()
    elif call == "encoder_mask":
        kw["encoder_attention_mask"] = torch.zeros(4, 1, 77).half()
    elif call == "cross_kwargs":
        kw["cross_attention_kwargs"] = {"scale": 1.0}
    elif call == "positional":
        args = (None,)
    elif call == "unknown_kwarg":
        kw["added_cond_kwargs"] = None
    elif call == "fp32":
        x = _x(4, dtype=torch.float32)
        blk.float()
    elif call == "ada":
        blk.use_ada_layer_norm = True
    elif call == "ada_zero":
        blk.use_ada_layer_norm_zero = True
    elif call == "only_cross":
        blk.only_cross_attention = True
    elif call == "old_flags":
        del blk.use_ada_layer_norm
    elif call == "training":
        blk.train()
    try:
        blk(x, *args, **kw)
    except Exception:
        pass                       # the own forward may not take what it is given; where it went is what counts
    assert rec.calls[:1] == [("block_own", 4)], rec.calls
    assert not [c for c in rec.calls if c[0].endswith("_library")], rec.calls


def test_ineligible_stages_run_their_modules(switch, monkeypatch):
    rec = Recorder(monkeypatch)
    patch.FUSE_CONTROLNET_BLOCKS = True
    # head_dim 160 above MAX_HEAD_DIM: attn1 and attn2 run their modules, the feed-forward the library
    blk = _served_block(dim=1280, heads=8)
    x, ctx = _x(4, dim=1280), _ctx(4)
    blk(x, encoder_hidden_states=ctx)
    assert rec.calls == [("attn_module", 4), ("attn_module", 4), ("ff_library", 4)]
    attention.MAX_HEAD_DIM = 160
    rec.calls.clear()
    blk(x, encoder_hidden_states=ctx)
    assert rec.calls == LIBRARY
    # a forward hook on attn1, a norm1 that is not a plain LayerNorm: attn1's module, the rest in the library
    blk = _served_block()
    handle = blk.attn1.register_forward_hook(lambda *a: None)
    rec.calls.clear()
    blk(_x(4), encoder_hidden_states=_ctx(4))
    assert rec.calls == [("attn_module", 4)] + LIBRARY[1:]
    handle.remove()

    class Norm(torch.nn.LayerNorm):
        pass
    norm = Norm(320).half()
    norm.load_state_dict(blk.norm1.state_dict())
    blk.norm1 = norm
    rec.calls.clear()
    blk(_x(4), encoder_hidden_states=_ctx(4))
    assert rec.calls == [("attn_module", 4)] + LIBRARY[1:]
    # a feed-forward that is not the stock GEGLU runs its module
    blk = _served_block()
    blk.ff = torch.nn.Sequential(torch.nn.Linear(320, 320)).half()
    rec.calls.clear()
    blk(_x(4), encoder_hidden_states=_ctx(4))
    assert rec.calls == LIBRARY[:2]


def _served_wrapper(linear=False):
    torch.manual_seed(0)
    blk = BasicTransformerBlock(320, 8, hot_path_only=True)
    w = Transformer2DModel(320, blk, use_linear_projection=linear).half().eval()
    patch.serve_unmerged(w)
    return w


@pytest.mark.parametrize("linear", [False, True])
def test_wrapper_dispatch(switch, monkeypatch, linear):
    rec = Recorder(monkeypatch)
    w = _served_wrapper(linear)
    x = torch.randn(2, 320, 4, 4).half()
    w(x)                                                            # switch off: the class's own forward
    assert rec.calls == [("wrapper_own", 2), ("block_own", 2), ("attn_module", 2)]
    patch.FUSE_CONTROLNET_BLOCKS = True
    rec.calls.clear()
    out = w(x, return_dict=False)[0]
    assert rec.calls == [("wrapper_library", 2)] and torch.equal(out, x + 1)
    # FUSE_TRANSFORMER_IO off, a hook on proj_in, an fp32 input, a keyword library_forward does not restate: its own
    for case in ("io_off", "hook", "fp32", "kwarg"):
        rec.calls.clear()
        kw, xin, handle = {}, x, None
        if case == "io_off":
            patch.FUSE_TRANSFORMER_IO = False
        elif case == "hook":
            handle = w.proj_in.register_forward_hook(lambda *a: None)
        elif case == "fp32":
            xin = x.float()
        else:
            kw["added_cond_kwargs"] = None
        try:
            w(xin, **kw)
        except Exception:
            pass
        assert rec.calls[:1] == [("wrapper_own", 2)], (case, rec.calls)
        patch.FUSE_TRANSFORMER_IO = True
        if handle is not None:
            handle.remove()
