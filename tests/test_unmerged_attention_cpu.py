"""patch.FUSE_UNMERGED_ATTENTION without a GPU: the binding of `vtm_attention_residual_ex`, its argument errors (returned
before anything touches a device), and which path ToMeBlock.forward takes for a block that does not merge, with the
library calls replaced by recorders (the eligibility tests read shapes, types and flags, never the device)."""
import pytest
import torch

from vidtome_b200 import _lib, attention, ops, patch, pnp
from vidtome_b200.skeleton import Attention, BasicTransformerBlock

E_NULL, E_SHAPE, E_WS, E_UNSUP = -1, -2, -4, -6
SHARED_QK = 1


def test_symbol_is_bound_with_the_declared_argtypes():
    lib = _lib.load()
    fn = lib.vtm_attention_residual_ex
    res, args = _lib.SIGNATURES["vtm_attention_residual_ex"]
    assert fn.restype is res and list(fn.argtypes) == list(args)
    assert len(args) == 18 and args[12] is _lib._i32 and args[13] is _lib._i32      # flags, qk_items
    # the older entry point keeps its signature
    assert len(_lib.SIGNATURES["vtm_attention_residual"][1]) == 16


def test_argument_errors_without_a_device():
    lib = _lib.load()
    att = lib.vtm_attention_residual_ex
    p = 0x10000                                                  # never dereferenced: every call below is refused first
    ws = lib.vtm_attention_workspace_bytes(6, 64, 320, 8)
    #          x  wqkv wo  bo    resid lq    lo    B  L   C    heads scale flags      items y  ws  bytes  stream
    assert att(p, p, p, None, p, None, None, 6, 64, 320, 8, 0.1, SHARED_QK, 4, p, p, ws, None) == E_SHAPE  # 6 % 4
    assert att(p, p, p, None, p, None, None, 6, 64, 320, 8, 0.1, SHARED_QK, 0, p, p, ws, None) == E_SHAPE
    assert att(p, p, p, None, p, None, None, 6, 64, 320, 8, 0.1, SHARED_QK, -2, p, p, ws, None) == E_SHAPE
    assert att(p, p, p, None, p, None, None, 6, 64, 320, 8, 0.1, 2, 2, p, p, ws, None) == E_UNSUP
    assert att(p, p, p, None, p, None, None, 6, 64, 320, 8, 0.1, SHARED_QK | 4, 2, p, p, ws, None) == E_UNSUP
    assert att(p, p, p, None, None, None, None, 6, 64, 320, 8, 0.1, SHARED_QK, 2, p, p, ws, None) == E_NULL
    assert att(p, p, p, None, None, None, None, 6, 64, 320, 8, 0.1, 0, 0, p, p, ws, None) == E_NULL
    # valid period, workspace one byte short: the checks above are the only ones qk_items takes part in
    assert att(p, p, p, None, p, None, None, 6, 64, 320, 8, 0.1, SHARED_QK, 3, p, p, ws - 1, None) == E_WS
    assert att(p, p, p, None, p, None, None, 6, 64, 320, 8, 0.1, SHARED_QK, 6, p, p, ws - 1, None) == E_WS
    # flags == 0 ignores qk_items
    assert att(p, p, p, None, p, None, None, 6, 64, 320, 8, 0.1, 0, 0, p, p, ws - 1, None) == E_WS
    assert att(p, p, p, None, p, None, None, 6, 64, 320, 8, 0.1, 0, 4, p, p, ws - 1, None) == E_WS
    lora = _lib.VtmLora(p, p, 8)
    assert att(p, p, p, None, p, None, lora, 6, 64, 320, 8, 0.1, SHARED_QK, 3, p, p, ws, None) == E_WS


# ------------------------------------------------------------------------------------------------ dispatch
SIZE = 16                     # latent 16 x 16: 256 tokens per frame at downsample 1, 64 at 2, 16 at 4


class Recorder:
    """Stands in for the library calls and for attn1's own forward; `calls` lists (what, batch, shared_items)."""

    def __init__(self, monkeypatch):
        self.calls = []
        monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
        monkeypatch.setattr(ops, "layer_norm", lambda x, ln: x)
        monkeypatch.setattr(attention, "self_attention_residual", self.residual)
        monkeypatch.setattr(Attention, "forward", self.module_forward)
        monkeypatch.setattr(patch, "build_merge_plan", self.plan)

    def plan(self, module, x, info, ln=None):
        # a merged block's plan needs the device: recorded, and declined, so that its attn1 runs the module
        self.calls.append(("plan", x.shape[0], None))
        return None

    def residual(self, attn, x, resid, shared_items=None):
        self.calls.append(("library", x.shape[0], shared_items))
        return resid + 1

    def module_forward(self, x, encoder_hidden_states=None, attention_mask=None, **kw):
        self.calls.append(("module", x.shape[0], None))
        return torch.zeros_like(x)

    def what(self):
        return [c for c in self.calls if c[0] != "plan"]


def _block(dim=320, heads=8, max_downsample=2):
    torch.manual_seed(0)
    blk = BasicTransformerBlock(dim, heads, hot_path_only=True).half()
    blk.__class__ = patch.make_diffusers_tome_block(blk.__class__)
    blk._tome_info = {"size": (SIZE, SIZE), "hooks": [], "args": dict(
        max_downsample=max_downsample, generator=None, seed=123, batch_size=3, align_batch=True, merge_global=False,
        global_merge_ratio=0.8, local_merge_ratio=0.9, global_rand=0.5, target_stride=4)}
    blk.generator = torch.Generator().manual_seed(5)
    return blk


def _x(B, tokens, dim=320):
    return torch.randn(B, tokens, dim).half()


@pytest.fixture
def switch():
    saved = patch.FUSE_UNMERGED_ATTENTION, attention.MAX_HEAD_DIM
    yield
    patch.FUSE_UNMERGED_ATTENTION, attention.MAX_HEAD_DIM = saved


def _mark(blk, rec, num_inputs=3):
    """PnP control on attn1 at t = 981, inside the schedule; its torch forward replaced by a recorder."""
    pnp.register_attention_control(None, [981, 961], num_inputs, modules=[blk.attn1])
    pnp.register_time(None, 981, modules=[blk.attn1])

    def recorded(x, *a, **k):
        rec.calls.append(("pnp_module", x.shape[0], None))
        return torch.zeros_like(x)
    recorded._vtm_pnp_forward = True
    blk.attn1.forward = recorded


def test_switch_off_unmerged_block_calls_the_module_as_before(switch, monkeypatch):
    rec = Recorder(monkeypatch)
    assert patch.FUSE_UNMERGED_ATTENTION is False
    blk = _block()
    x = _x(12, SIZE * SIZE // 16)                       # downsample 4 > max_downsample 2
    blk(x)
    assert rec.what() == [("module", 12, None)]
    assert ("plan", 12, None) in rec.calls               # the merge plan is asked, and declines


def test_switch_on_unmerged_block_takes_the_residual_path(switch, monkeypatch):
    rec = Recorder(monkeypatch)
    patch.FUSE_UNMERGED_ATTENTION = True
    blk = _block()
    x = _x(12, SIZE * SIZE // 16)
    state = blk.generator.get_state().clone()
    y = blk(x)
    assert rec.calls == [("library", 12, None)]          # no merge plan, nothing drawn
    assert torch.equal(blk.generator.get_state(), state)
    assert torch.equal(y, x + 1)


def test_switch_on_merged_block_never_takes_it(switch, monkeypatch):
    rec = Recorder(monkeypatch)
    patch.FUSE_UNMERGED_ATTENTION = True
    blk = _block()
    for tokens in (SIZE * SIZE, SIZE * SIZE // 4):       # downsample 1 and 2
        rec.calls.clear()
        blk(_x(12, tokens))
        assert rec.what() == [("module", 12, None)], tokens
        assert rec.calls[0] == ("plan", 12, None)
    # downsample 4 merges once max_downsample is 4
    blk._tome_info["args"]["max_downsample"] = 4
    rec.calls.clear()
    blk(_x(12, SIZE * SIZE // 16))
    assert rec.what() == [("module", 12, None)]


@pytest.mark.parametrize("num_inputs", [2, 3])
def test_pnp_module_shares_by_frame_only_while_injecting(switch, monkeypatch, num_inputs):
    rec = Recorder(monkeypatch)
    patch.FUSE_UNMERGED_ATTENTION = True
    blk = _block()
    _mark(blk, rec, num_inputs=num_inputs)
    B = num_inputs * 4
    x = _x(B, SIZE * SIZE // 16)
    blk(x)                                                # t = 981 is in the schedule
    assert rec.calls == [("library", B, 4)]
    rec.calls.clear()
    pnp.register_time(None, 500, modules=[blk.attn1])    # outside the schedule
    blk(x)
    assert rec.calls == [("library", B, None)]
    rec.calls.clear()
    pnp.register_time(None, 1000, modules=[blk.attn1])   # t == 1000 always injects (utils/pnp_utils.py:58)
    blk(x)
    assert rec.calls == [("library", B, 4)]
    rec.calls.clear()
    patch.FUSE_UNMERGED_ATTENTION = False                 # switch off: PnP's own forward, as before
    blk(x)
    assert rec.what() == [("pnp_module", B, None)]


def test_pnp_inside_unmerged_blocks_never_shares(switch, monkeypatch):
    rec = Recorder(monkeypatch)
    blk = _block()
    _mark(blk, rec)
    for on in (False, True):
        patch.FUSE_UNMERGED_ATTENTION = on
        rec.calls.clear()
        with patch._unmerged_blocks():
            blk(_x(12, SIZE * SIZE))                      # even a block that would merge
        assert rec.calls == [("library", 12, None)], on


def test_indivisible_batch_keeps_the_module_forward(switch, monkeypatch):
    rec = Recorder(monkeypatch)
    patch.FUSE_UNMERGED_ATTENTION = True
    blk = _block()
    _mark(blk, rec, num_inputs=3)
    blk(_x(8, SIZE * SIZE // 16))                         # 8 % 3 != 0 while injecting
    assert rec.what() == [("pnp_module", 8, None)]
    rec.calls.clear()
    pnp.register_time(None, 500, modules=[blk.attn1])    # not injecting: no period needed
    blk(_x(8, SIZE * SIZE // 16))
    assert rec.calls == [("library", 8, None)]


def test_wide_heads_and_non_plain_modules_keep_the_module_forward(switch, monkeypatch):
    rec = Recorder(monkeypatch)
    patch.FUSE_UNMERGED_ATTENTION = True
    blk = _block(dim=1280, heads=8)                       # head_dim 160
    x = _x(6, SIZE * SIZE // 16, dim=1280)
    blk(x)
    assert rec.what() == [("module", 6, None)]
    attention.MAX_HEAD_DIM = 160
    rec.calls.clear()
    blk(x)
    assert rec.calls == [("library", 6, None)]
    # a forward hook makes attn1 a module KD could not replace
    handle = blk.attn1.register_forward_hook(lambda *a: None)
    rec.calls.clear()
    blk(x)
    assert rec.what() == [("module", 6, None)]
    handle.remove()
    # an attention mask or cross_attention_kwargs keep the module too
    rec.calls.clear()
    blk(x, cross_attention_kwargs={"scale": 1.0})
    assert rec.what() == [("module", 6, None)]


def test_gate_is_the_merge_plans_gate():
    info = {"size": (64, 64), "args": {"max_downsample": 2}}
    for tokens, merges in ((4096, True), (1024, True), (256, False), (64, False)):
        assert patch.block_merges(torch.empty(1, tokens, 8), info) is merges
    info["args"]["max_downsample"] = 4
    assert patch.block_merges(torch.empty(1, 256, 8), info) and not patch.block_merges(torch.empty(1, 64, 8), info)
