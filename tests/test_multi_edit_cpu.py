"""Several edits of one video in one pass, host side: the edit-major batch the driver builds against the batches of K
single-prompt drivers, the per-edit slicing and shared draws of the patch layer, the per-edit PnP items, graph keys,
and the refusals.  Stand-in modules as in the other *_cpu.py tests; the kernels run in tests/test_gpu_multi_edit.py."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from vidtome_b200 import patch, pnp, utils
from vidtome_b200.driver import ChunkedDenoiser


class StandInUNet(torch.nn.Module):
    """Every output row depends on its own latent, its own text row and the timestep (not on its position), so that a
    K-edit batch must give each edit exactly its single run's rows."""

    def __init__(self, batch_size=2, align_batch=False, edits=None, in_channels=4):
        super().__init__()
        self._tome_info = {"args": {"batch_size": batch_size, "align_batch": align_batch}}
        if edits is not None:
            self._tome_info["args"]["edits"] = edits
        self.in_channels = in_channels
        self.calls = []

    def forward(self, sample, t, encoder_hidden_states=None, **kwargs):
        self.calls.append((sample.clone(), encoder_hidden_states))
        eps = sample[:, :4] * 1.25 + float(t) * 1e-3 + sample[:, 4:].sum(1, keepdim=True)
        if encoder_hidden_states is not None:
            eps = eps + 0.5 * encoder_hidden_states.mean(dim=(1, 2))[:, None, None, None]
        return SimpleNamespace(sample=eps)


def _cond(K, S, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((K, S, 77, 16), generator=g)


def _src(t):
    return torch.full((6, 4, 8, 8), float(t) * 1e-3)


@pytest.mark.parametrize("K", [1, 2, 3])
@pytest.mark.parametrize("pnp_on,depth", [(False, False), (True, False), (False, True), (True, True)])
def test_edit_major_batch_is_the_single_batches_in_edit_order(K, pnp_on, depth):
    S = 3 if pnp_on else 2
    cond = _cond(K, S)
    g = torch.Generator().manual_seed(1)
    x = torch.randn((K, 6, 4, 8, 8), generator=g)
    dmap = torch.rand((6, 1, 8, 8), generator=g) if depth else None
    kw = dict(source_latents=_src, pnp_modules=[]) if pnp_on else {}
    multi = ChunkedDenoiser(StandInUNet(S, pnp_on, edits=K, in_channels=5 if depth else 4), cond=cond, depth=dmap,
                            **kw)
    lo, hi = 1, 5
    frames = {"depth": dmap[lo:hi]} if depth else {}
    src = _src(981)[lo:hi] if pnp_on else None
    got = multi.pred_noise(x[:, lo:hi], 981, src=src, **frames)
    sample, text = multi.unet.calls[-1]
    assert sample.shape[0] == K * S * (hi - lo) and text.shape[0] == sample.shape[0]
    for k in range(K):
        one = ChunkedDenoiser(StandInUNet(S, pnp_on, in_channels=5 if depth else 4), cond=cond[k], depth=dmap, **kw)
        want = one.pred_noise(x[k, lo:hi], 981, src=src, **frames)
        s1, t1 = one.unet.calls[-1]
        n = S * (hi - lo)
        assert torch.equal(sample[k * n:(k + 1) * n], s1)
        assert torch.equal(text[k * n:(k + 1) * n], t1)
        assert torch.equal(got[k], want)


def test_eager_step_of_k_edits_is_k_single_steps():
    K = 3
    cond = _cond(K, 2)
    x = torch.randn((K, 6, 4, 8, 8), generator=torch.Generator().manual_seed(2))
    multi = ChunkedDenoiser(StandInUNet(edits=K), n_timesteps=5, chunk_size=4, cond=cond, randomize_chunks=True)
    np.random.seed(3)
    torch.manual_seed(3)
    got = multi.step(x, 0)
    for k in range(K):
        one = ChunkedDenoiser(StandInUNet(), n_timesteps=5, chunk_size=4, cond=cond[k], randomize_chunks=True)
        np.random.seed(3)
        torch.manual_seed(3)
        assert torch.equal(got[k], one.step(x[k], 0))


def test_step_draws_the_chunks_once_whatever_k():
    """get_chunks' numpy and torch draws are issued once per step, as by one run."""
    states = []
    for K in (None, 1, 4):
        cond = _cond(1, 2)[0] if K is None else _cond(K, 2)
        den = ChunkedDenoiser(StandInUNet(edits=K), n_timesteps=5, chunk_size=4, cond=cond, randomize_chunks=True,
                              merge_global=True, chunk_ord="mix-4")
        x = torch.zeros((6, 4, 8, 8) if K is None else (K, 6, 4, 8, 8))
        np.random.seed(7)
        torch.manual_seed(7)
        den.step(x, 0)
        states.append((np.random.get_state()[1][:4].tolist(), np.random.get_state()[2], torch.rand(1).item()))
    assert states[0] == states[1] == states[2]


def test_sample_takes_one_noise_for_every_edit():
    K = 2
    cond = _cond(K, 2)
    x = torch.randn((6, 4, 8, 8), generator=torch.Generator().manual_seed(4))
    got = ChunkedDenoiser(StandInUNet(edits=K), n_timesteps=2, chunk_size=4, cond=cond).sample(x)
    assert got.shape == (K, 6, 4, 8, 8)
    for k in range(K):
        assert torch.equal(got[k], ChunkedDenoiser(StandInUNet(), n_timesteps=2, chunk_size=4, cond=cond[k]).sample(x))


def test_graph_keys_carry_k():
    for K in (1, 2, 4):
        den = ChunkedDenoiser(StandInUNet(edits=K), cond=_cond(K, 2))
        x = torch.zeros((K, 8, 4, 8, 8))
        assert den._graph_key(x, 981) == ((K, 8, 4, 8, 8), False)
        assert den._flen(x) == 8 and den._frame_rows(x, 2, 6).shape == (K, 4, 4, 8, 8)
    single = ChunkedDenoiser(StandInUNet(), cond=_cond(1, 2)[0])
    assert single._graph_key(torch.zeros(8, 4, 8, 8), 981) == ((8, 4, 8, 8), False)


def test_refusals():
    with pytest.raises(ValueError, match="shard=True"):
        ChunkedDenoiser(StandInUNet(edits=2), cond=_cond(2, 2), shard=True)
    with pytest.raises(ValueError, match="edits=1"):
        ChunkedDenoiser(StandInUNet(), cond=_cond(2, 2))
    with pytest.raises(ValueError, match="edits=3"):
        ChunkedDenoiser(StandInUNet(edits=3), cond=_cond(2, 2))
    with pytest.raises(ValueError, match="edits=2"):
        ChunkedDenoiser(StandInUNet(edits=2), cond=_cond(2, 2)[0])
    with pytest.raises(ValueError, match=r"\[K, S, 77, D\]"):
        ChunkedDenoiser(StandInUNet(edits=2), cond=torch.zeros(2, 4, 77, 16))
    with pytest.raises(ValueError, match="PnP"):
        ChunkedDenoiser(StandInUNet(3, True, edits=2), cond=_cond(2, 2), source_latents=_src, pnp_modules=[])
    den = ChunkedDenoiser(StandInUNet(edits=2), cond=_cond(2, 2))
    with pytest.raises(ValueError, match="latents of 2 edits"):
        den.step(torch.zeros(6, 4, 8, 8), 0)
    with pytest.raises(ValueError, match="latents of 2 edits"):
        den.step(torch.zeros(3, 6, 4, 8, 8), 0)
    for bad in (0, -1, 1.5, True):
        with pytest.raises(ValueError, match="positive int"):
            patch.update_patch(StandInUNet(), edits=bad)


def test_reference_pnp_forward_is_refused_with_several_edits():
    from vidtome_b200.skeleton import Attention
    attn = Attention(32, 2, 16)
    unet = StandInUNet(3, True, edits=2)
    unet.extra = attn
    attn.injection_schedule = [981]
    attn.forward = lambda *a, **k: None                      # the reference's closure stands in
    with pytest.raises(ValueError, match="reference's PnP forward"):
        ChunkedDenoiser(unet, cond=_cond(2, 3), source_latents=_src, pnp_modules=[])
    assert patch._reference_pnp_forward(attn)
    pnp.register_attention_control(None, [981], 3, modules=[attn])
    assert not patch._reference_pnp_forward(attn)


def test_update_patch_stores_edits_as_a_patch_argument():
    unet = StandInUNet()
    assert patch.edits_of(unet) == 1 and "edits" not in unet._tome_info["args"]
    patch.update_patch(unet, edits=3)
    assert patch.edits_of(unet) == 3 and not hasattr(unet, "edits")
    assert patch.edits_of(torch.nn.Linear(2, 2)) == 1


# ------------------------------------------------------------------------------------------- the patch layer
class StandInBlock(torch.nn.Module):
    """What _self_attention_stage reads of a ToMeBlock, with a CPU generator."""
    _vtm_unmerged = False
    use_ada_layer_norm = False
    use_ada_layer_norm_zero = False

    def __init__(self, edits, batch_size=2):
        super().__init__()
        self._tome_info = {"args": {"batch_size": batch_size, "edits": edits}, "size": (4, 4)}
        self.attn1 = torch.nn.Identity()
        self.generator = torch.Generator().manual_seed(5)


def _recording_stage(monkeypatch, draws_per_call=2):
    """Replace the single-edit stage by one that records its rows and draws like build_merge_plan (one randint per
    level, one coin), through patch._draw."""
    seen = []

    def stage(block, h, *rest):
        vals = [patch._draw(lambda: utils.draw_randf(block.generator, 4, 8)) for _ in range(draws_per_call)]
        vals.append(patch._draw(lambda: utils.draw_coin(block.generator, on_device=False)))
        g = block.global_tokens
        block.global_tokens = h[:1].clone() if g is None else g + 1
        seen.append((h.clone(), vals, g))
        return h * 2, None
    monkeypatch.setattr(patch, "_edit_self_attention", stage)
    return seen


def test_one_edit_takes_the_single_path(monkeypatch):
    seen = _recording_stage(monkeypatch)
    blk = StandInBlock(1)
    blk.global_tokens = None
    x = torch.randn(8, 16, 4)
    out, _ = patch._self_attention_stage(blk, x, None, None, None, None, None)
    assert len(seen) == 1 and torch.equal(seen[0][0], x) and torch.equal(out, 2 * x)
    assert patch._SHARED_DRAWS is None and torch.is_tensor(blk.global_tokens)


@pytest.mark.parametrize("K", [2, 3, 4])
def test_edits_run_on_their_slices_with_shared_draws(monkeypatch, K):
    seen = _recording_stage(monkeypatch)
    blk = StandInBlock(K)
    ref = torch.Generator().manual_seed(5)
    want = [utils.draw_randf(ref, 4, 8), utils.draw_randf(ref, 4, 8), utils.draw_coin(ref, on_device=False)]
    x = torch.randn(K * 8, 16, 4)
    out, _ = patch._self_attention_stage(blk, x, None, None, None, None, None)
    assert torch.equal(out, 2 * x)
    assert [torch.equal(h, x[k * 8:(k + 1) * 8]) for k, (h, _, _) in enumerate(seen)] == [True] * K
    assert all(vals == want for _, vals, _ in seen)                          # every edit gets the same draws
    assert blk.generator.get_state().equal(ref.get_state())                  # drawn once, whatever K is
    # each edit keeps its own global tokens across calls
    assert isinstance(blk.global_tokens, list) and len(blk.global_tokens) == K
    assert all(torch.equal(g, x[k * 8:k * 8 + 1]) for k, g in enumerate(blk.global_tokens))
    seen.clear()
    patch._self_attention_stage(blk, x, None, None, None, None, None)
    assert all(torch.equal(g, x[k * 8:k * 8 + 1]) for k, (_, _, g) in enumerate(seen))
    patch.update_patch(blk, global_tokens=None)
    seen.clear()
    patch._self_attention_stage(blk, x, None, None, None, None, None)
    assert all(g is None for _, _, g in seen)


def test_an_edit_drawing_differently_is_an_error(monkeypatch):
    calls = []

    def stage(block, h, *rest):
        calls.append(1)
        for _ in range(len(calls)):                                          # edit k draws k + 1 times
            patch._draw(lambda: utils.draw_randf(block.generator, 4, 8))
        return h, None
    monkeypatch.setattr(patch, "_edit_self_attention", stage)
    with pytest.raises(RuntimeError, match="drew more"):
        patch._self_attention_stage(StandInBlock(2), torch.zeros(16, 4, 2), None, None, None, None, None)
    assert patch._SHARED_DRAWS is None


def test_bad_batches_and_global_tokens_are_refused(monkeypatch):
    _recording_stage(monkeypatch)
    blk = StandInBlock(3)
    with pytest.raises(ValueError, match="not 3 edits"):
        patch._self_attention_stage(blk, torch.zeros(8, 4, 2), None, None, None, None, None)
    blk.global_tokens = torch.zeros(1, 2, 2)
    with pytest.raises(ValueError, match="list of 3"):
        patch._self_attention_stage(blk, torch.zeros(12, 4, 2), None, None, None, None, None)


def test_pnp_items_are_counted_within_each_edit(monkeypatch):
    """With K edits of [source | uncond | cond] x c frames, every edit's stage sees 3c items, of which the first c lead
    (item b takes the map of item b mod c), as in a single-edit run."""
    from vidtome_b200.skeleton import Attention
    attn = Attention(32, 2, 16)
    pnp.register_attention_control(None, [981], 3, modules=[attn])
    pnp.register_time(None, 981, modules=[attn])
    shared = []

    def stage(block, h, *rest):
        shared.append(patch._pnp_shared_items(block.attn1, h.shape[0]))
        return h, None
    monkeypatch.setattr(patch, "_edit_self_attention", stage)
    blk = StandInBlock(2, batch_size=3)
    blk.attn1 = attn
    c = 4
    patch._self_attention_stage(blk, torch.zeros(2 * 3 * c, 16, 32), None, None, None, None, None)
    assert shared == [c, c]
    assert patch._pnp_shared_items(attn, 2 * 3 * c) == 2 * c                 # not what a whole-batch split would give


def test_conv_injection_runs_per_edit():
    """register_conv_control with edits=K runs the ResNet once per edit's slice: each edit's uncond and cond samples
    take their own source samples' features."""
    from vidtome_b200.skeleton import ResnetBlock2D
    torch.manual_seed(0)
    resnet = ResnetBlock2D(32, 32, temb_channels=8).eval()
    K, n = 2, 2
    x = torch.randn(K * 3 * n, 32, 4, 4)
    temb = torch.randn(K * 3 * n, 8)
    pnp.register_conv_control(None, [981], 3, modules=[resnet], edits=K)
    pnp.register_time(None, 981, modules=[resnet])
    with torch.no_grad():
        got = resnet(x, temb)
        for k in range(K):
            rows = slice(k * 3 * n, (k + 1) * 3 * n)
            want = pnp._conv_torch_forward(resnet, 3, x[rows], temb[rows])
            assert torch.equal(got[rows], want), k


def test_lane_edges_keep_one_recurrence_per_edit_and_branch_each_lane():
    """In a lane capture, edit k's global stage waits only on edit k's store of the previous chunk, and the block's
    edits 1..K-1 run on the side streams made for the current lane."""
    made = []

    class Ev:
        def __init__(self):
            self.records, self.waited = [], 0
            made.append(self)

        def record(self, stream):
            self.records.append(stream)

    class Stream:
        def __init__(self, handle):
            self.cuda_stream, self.waits = handle, []

        def wait_event(self, ev):
            self.waits.append(ev)

    lane = Stream(7)
    side = [Stream(8), Stream(9)]
    blk = torch.nn.Linear(1, 1)
    edges = patch.LaneEdges([blk], event=Ev, current_stream=lambda: lane, branches={7: side})
    assert edges.edit_streams(3) == [lane] + side and edges.edit_streams(4) is None
    tokens = SimpleNamespace(record_stream=lambda s: None)
    for k in range(2):
        patch._EDIT = k
        try:
            edges.wait(blk, tokens)                      # nothing recorded yet: no wait
            edges.record(blk)
            edges.wait(blk, tokens)
        finally:
            patch._EDIT = None
    assert len(made) == 3 and len(lane.waits) == 2 and lane.waits[0] is not lane.waits[1]
    assert {id(blk), (id(blk), 0), (id(blk), 1)} == set(edges.events)


def test_conv_injection_reads_the_edits_at_every_call():
    """register_conv_control before update_patch(edits=K): the ResNet still runs per edit, and inside inversion
    (_unmerged_blocks) it takes the whole batch as one run."""
    from vidtome_b200.skeleton import ResnetBlock2D
    torch.manual_seed(0)
    resnet = ResnetBlock2D(32, 32, temb_channels=8).eval()
    unet = StandInUNet(3)
    unet.resnet = resnet
    pnp.register_conv_control(unet, [981], 3, modules=[resnet])
    pnp.register_time(None, 981, modules=[resnet])
    patch.update_patch(unet, edits=2)
    x, temb = torch.randn(12, 32, 4, 4), torch.randn(12, 8)
    with torch.no_grad():
        got = resnet(x, temb)
        for k in range(2):
            assert torch.equal(got[6 * k:6 * (k + 1)], pnp._conv_torch_forward(resnet, 3, x[6 * k:6 * (k + 1)],
                                                                              temb[6 * k:6 * (k + 1)]))
        with patch._unmerged_blocks():
            assert resnet(x[:9], temb[:9]).shape[0] == 9     # an inversion batch, not divisible by the edits
