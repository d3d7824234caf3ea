"""The float64 replay of test_gpu_step_float64 on the CPU with merging off: every block replaced by
test_gpu_block_core._block64 with no maps must give the unpatched float64 model's output, for the UNet, the ControlNet
and the SD2-depth UNet, so that the replay machinery is the model's own forward before any GPU result is read."""
import copy

import pytest
import torch

import test_gpu_step_float64 as sf
from vidtome_b200.skeleton import make_controlnet, make_skeleton


def _pair(model):
    """(the unpatched float64 model, a float64 copy with every block replayed without maps)."""
    plain = copy.deepcopy(model).double()
    replayed = copy.deepcopy(model).double()
    rep = sf.Replay([replayed], [replayed], {})
    assert rep.blocks == sum(type(m).__name__ == "BasicTransformerBlock" for m in plain.modules()) > 0
    return plain, replayed


def _assert_close(got, want):
    # test_gpu_block_core._attn64 takes softmax(q k^T scale) v in its own order of float64 operations, the skeleton's
    # Attention torch's scaled_dot_product_attention: the two agree to a few float64 roundings (7.4e-16 of max|ref| at
    # most, torch 2.11 on x86), not bit for bit
    rel = ((got - want).abs().max() / want.abs().max()).item()
    print(f"replay against the model's forward: {rel:.2e} of max|ref|")
    assert rel <= 1e-14, rel


@pytest.mark.parametrize("name", ["sd15", "sd21_depth"])
def test_unet_replay_is_the_model_forward(name):
    depth = name == "sd21_depth"
    net = make_skeleton("sd21" if depth else "sd15", hot_path_only=False, device="cpu", dtype=torch.float32,
                        transformer_io="linear" if depth else None, depth=depth, pnp_conv=not depth)
    plain, replayed = _pair(net)
    g = torch.Generator().manual_seed(0)
    x = torch.randn((2, 5 if depth else 4, 8, 8), generator=g, dtype=torch.float64)
    ctx = torch.randn((2, 77, 1024 if depth else 768), generator=g, dtype=torch.float64)
    with torch.no_grad():
        want = plain(x, 501, encoder_hidden_states=ctx).sample
        got = replayed(x, 501, encoder_hidden_states=ctx).sample
    _assert_close(got, want)


def test_controlnet_replay_is_the_model_forward():
    cn = make_controlnet("sd15", hot_path_only=False, device="cpu", dtype=torch.float32)
    plain, replayed = _pair(cn)
    g = torch.Generator().manual_seed(1)
    x = torch.randn((2, 4, 8, 8), generator=g, dtype=torch.float64)
    ctx = torch.randn((2, 77, 768), generator=g, dtype=torch.float64)
    img = torch.rand((2, 3, 64, 64), generator=g, dtype=torch.float64)
    with torch.no_grad():
        want = plain(x, 501, encoder_hidden_states=ctx, controlnet_cond=img)
        got = replayed(x, 501, encoder_hidden_states=ctx, controlnet_cond=img)
    for a, b in zip(list(got[0]) + [got[1]], list(want[0]) + [want[1]]):
        _assert_close(a, b)
