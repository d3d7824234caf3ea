"""Host side of the Transformer2DModel entry / exit path, without a GPU: the exported symbols, the grid planner of the
statistics kernel restated, the skeleton's stand-in wrapper against the written-out formula, the patch lifecycle, and
every reason `transformer2d.ineligibility` gives."""
import json
import os

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import vidtome_b200
from vidtome_b200 import _lib, patch, transformer2d
from vidtome_b200.skeleton import (BasicTransformerBlock, LoRACompatibleLinear, ModelMixin, Transformer2DModel,
                                   make_controlnet, make_skeleton)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_new_symbols_are_exported():
    lib = _lib.load()
    for name in ("vtm_group_norm_stats_workspace_bytes", "vtm_group_norm_stats_f16", "vtm_group_norm_tokens_f16",
                 "vtm_linear_nchw_residual_f16"):
        assert name in _lib.SIGNATURES and getattr(lib, name) is not None
    assert lib.vtm_version() == 100
    # argument checks come before any CUDA call
    assert lib.vtm_group_norm_stats_f16(None, 1, 32, 1, 32, 1e-6, None, None, 0, None) == -1
    assert lib.vtm_group_norm_tokens_f16(None, None, None, None, 1, 32, 1, 32, None, None) == -1
    assert lib.vtm_linear_nchw_residual_f16(None, None, None, None, 1, 1, 8, 8, None, None) == -1


def _split(runs, R):
    """transformer_io.cu: pieces per run."""
    if R <= 2048 or runs >= 512 or R <= 8192:
        return 1
    return min(-(-R // 8192), -(-512 // runs))


def test_stats_planner_reaches_every_branch_the_gpu_test_claims():
    lib = _lib.load()
    HWS = (1, 2, 7, 8, 9, 63, 64, 144, 256, 576, 1024, 4096, 9216)
    kinds = set()
    for cpg in range(1, 41):
        for HW in HWS:
            n = 1 + (cpg + HW) % 3
            runs, R = 32 * n, cpg * HW
            S = _split(runs, R)
            want = 0 if S == 1 else runs * S * 12
            assert lib.vtm_group_norm_stats_workspace_bytes(n, 32 * cpg, HW, 32) == want, (cpg, HW, n)
            kinds.add("warp" if R <= 2048 else "cta" if S == 1 else "split")
    assert kinds == {"warp", "cta", "split"}
    assert lib.vtm_group_norm_stats_workspace_bytes(1, 320, 9216, 32) == 32 * 12 * 12        # S = 12, 384 CTAs
    assert lib.vtm_group_norm_stats_workspace_bytes(32, 320, 4096, 32) == 0                  # 1024 runs: one CTA each
    assert lib.vtm_group_norm_stats_workspace_bytes(1, 33, 4, 32) == 0                       # groups do not divide C


@pytest.mark.parametrize("form", ["conv", "linear"])
def test_stand_in_forward_is_the_written_out_formula(form):
    torch.manual_seed(0)
    C, h, w = 64, 5, 3
    block = BasicTransformerBlock(C, 2, hot_path_only=True)
    m = Transformer2DModel(C, block, use_linear_projection=form == "linear").eval()
    x = torch.randn(3, C, h, w)
    Transformer2DModel.torch_calls = 0
    with torch.no_grad():
        got = m(x).sample
        assert Transformer2DModel.torch_calls == 1
        y = F.group_norm(x, 32, m.norm.weight, m.norm.bias, 1e-6)
        w_in, w_out = m.proj_in.weight.view(C, C), m.proj_out.weight.view(C, C)
        if form == "conv":
            t = F.conv2d(y, m.proj_in.weight, m.proj_in.bias).permute(0, 2, 3, 1).reshape(3, h * w, C)
        else:
            t = F.linear(y.permute(0, 2, 3, 1).reshape(3, h * w, C), w_in, m.proj_in.bias)
        t = block(t)
        if form == "conv":
            o = F.conv2d(t.reshape(3, h, w, C).permute(0, 3, 1, 2), m.proj_out.weight, m.proj_out.bias)
        else:
            o = F.linear(t, w_out, m.proj_out.bias).reshape(3, h, w, C).permute(0, 3, 1, 2)
        torch.testing.assert_close(got, o + x, rtol=1e-5, atol=1e-5)
        assert m(x, return_dict=False)[0].shape == x.shape


@pytest.mark.parametrize("make", [make_skeleton, make_controlnet])
@pytest.mark.parametrize("io", ["conv", "linear"])
def test_option_leaves_existing_parameters_bit_identical(make, io):
    kw = dict(device="cpu", dtype=torch.float32)
    if make is make_skeleton:
        kw["pnp_conv"] = False
    a, b = make("tiny", **kw), make("tiny", transformer_io=io, **kw)
    sa, sb = a.state_dict(), b.state_dict()
    assert set(sa) < set(sb) and all(k.startswith("wrappers.") for k in set(sb) - set(sa))
    assert all(torch.equal(sa[k], sb[k]) for k in sa)
    assert [n for n, _ in a.named_modules()] == [n for n, _ in make("tiny", transformer_io=None, **kw).named_modules()]
    with pytest.raises(ValueError):
        make("tiny", transformer_io="patches", **kw)


def test_skeleton_with_pnp_conv_keeps_the_resnet_weights():
    a = make_skeleton("sd15", device="cpu", dtype=torch.float32, pnp_conv=True, max_downsample=None)
    b = make_skeleton("sd15", device="cpu", dtype=torch.float32, pnp_conv=True, transformer_io="conv")
    sa, sb = a.state_dict(), b.state_dict()
    assert all(torch.equal(sa[k], sb[k]) for k in sa)


def _pipe(io):
    class DiffusionPipeline:
        pass

    class StableDiffusionControlNetPipeline(DiffusionPipeline):
        pass
    pipe = StableDiffusionControlNetPipeline()
    pipe.unet = make_skeleton("tiny", device="cpu", dtype=torch.float32, transformer_io=io)
    pipe.controlnet = make_controlnet("tiny", device="cpu", dtype=torch.float32, transformer_io=io)
    return pipe


def _classes(net):
    return [type(m).__name__ for m in net.modules()]


@pytest.mark.parametrize("include_control", [False, True])
def test_apply_and_remove_swap_and_restore_the_wrapper_class(include_control):
    pipe = _pipe("conv")
    before_u, before_c = _classes(pipe.unet), _classes(pipe.controlnet)
    vidtome_b200.apply_patch(pipe, include_control=include_control)
    assert all(type(m).__name__ == "ToMeTransformer2D" and m._parent is Transformer2DModel for m in pipe.unet.wrappers)
    assert all(not hasattr(m, "_tome_info") for m in pipe.unet.wrappers)
    want = "ToMeTransformer2D" if include_control else "Transformer2DModel"
    assert all(type(m).__name__ == want for m in pipe.controlnet.wrappers)
    vidtome_b200.update_patch(pipe, marker=1)
    assert all(not hasattr(m, "marker") for m in pipe.unet.wrappers)
    assert all(hasattr(m, "marker") for m in pipe.unet.blocks)
    keys = set(vidtome_b200.collect_from_patch(pipe, attr="marker"))
    assert not any("wrappers" in k for k in keys)
    vidtome_b200.remove_patch(pipe)
    assert _classes(pipe.unet) == before_u
    # the reference's lifecycle asymmetry: remove_patch on a pipeline does not reach pipe.controlnet
    assert (_classes(pipe.controlnet) == before_c) == (not include_control)
    vidtome_b200.remove_patch(pipe.controlnet)
    assert _classes(pipe.controlnet) == before_c


def test_model_without_wrappers_is_patched_as_before():
    net = make_skeleton("tiny", device="cpu", dtype=torch.float32)
    vidtome_b200.apply_patch(net)
    names = {type(m).__name__ for m in net.modules()}
    assert "ToMeTransformer2D" not in names and "ToMeBlock" in names
    assert [n for n, m in net.named_modules() if hasattr(m, "_tome_info")] == [""] + [f"blocks.{i}" for i in range(4)]
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "lifecycle_controlnet.json")))
    assert golden                                     # the fixture the lifecycle tests hold the patch to is untouched
    vidtome_b200.remove_patch(net)


class _Net(ModelMixin):
    def __init__(self, wrapper):
        super().__init__()
        self.attn = wrapper

    def forward(self, x, *a, **k):
        return self.attn(x, return_dict=False)[0]


def _fresh(form="conv", C=64):
    torch.manual_seed(1)
    return Transformer2DModel(C, BasicTransformerBlock(C, 2, hot_path_only=True),
                              use_linear_projection=form == "linear").eval()


def _reasons():
    x = torch.randn(2, 64, 4, 4)

    def vectorized(m): m.is_input_vectorized = True
    def patches(m): m.is_input_patches = True
    def layer_norm(m): m.norm = nn.LayerNorm(4)
    def no_affine(m): m.norm = nn.GroupNorm(32, 64, affine=False)
    def conv3(m): m.proj_in = nn.Conv2d(64, 64, 3, padding=1)
    def lora(m): m.proj_out = LoRACompatibleLinear(64, 64)
    def mixed(m): m.proj_out = nn.Linear(64, 64)
    def hook(m): m.proj_in.register_forward_hook(lambda *a: None)
    def train(m): m.train()
    return [("input_variant", vectorized, x), ("input_variant", patches, x), ("shape", None, x[0]),
            ("layout", None, x.permute(0, 1, 3, 2)), ("norm", layer_norm, x), ("norm", no_affine, x),
            ("norm", None, torch.randn(2, 96, 4, 4)), ("projection", conv3, x), ("projection", lora, x),
            ("projection", mixed, x), ("hooks", hook, x), ("training", train, x), ("device", None, x)]


@pytest.mark.parametrize("case", range(13))
def test_every_ineligibility_reason_and_its_torch_fallback(case):
    reason, change, x = _reasons()[case]
    m = _fresh("linear" if reason == "projection" and case == 8 else "conv")
    if change is not None:
        change(m)
    assert transformer2d.ineligibility(m, x) == reason
    if reason in ("shape", "norm") and change is None or case in (4, 7, 9):
        return                                        # the torch forward itself cannot run on this input / module
    net = _Net(m)
    vidtome_b200.apply_patch(net, max_downsample=0)   # no block is merged: the patched block runs on the CPU
    assert type(net.attn).__name__ == "ToMeTransformer2D" and patch.FUSE_TRANSFORMER_IO
    Transformer2DModel.torch_calls = 0
    out = net(x)
    assert Transformer2DModel.torch_calls == 1 and out.shape == x.shape
    vidtome_b200.remove_patch(net)
    assert type(net.attn) is Transformer2DModel


def test_eligible_module_is_only_held_back_by_the_device():
    """On a CPU tensor everything but the last check passes; the same module with CUDA fp16 tensors is eligible."""
    m = _fresh()
    assert transformer2d.ineligibility(m, torch.randn(2, 64, 4, 4)) == "device"
    assert transformer2d.LIBRARY_KWARGS == set(
        Transformer2DModel.forward.__code__.co_varnames[2:Transformer2DModel.forward.__code__.co_argcount])
