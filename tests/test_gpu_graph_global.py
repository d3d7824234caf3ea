"""Global merging with the coin on the device (vtm_split_t.coin_dev, patch.DEVICE_COIN) and captured in the CUDA-graph
step driver (ChunkedDenoiser(capture_global=True)).  The device coin keeps the two token sets in one storage order,
cat = [local | global], and lets the coin pick which half is src; everything here checks that this computes what the
reference's coin-ordered concatenation computes, bit for bit."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _info(B, hw, **kw):
    args = dict(max_downsample=2, generator=None, seed=123, batch_size=B, align_batch=False, merge_global=True,
                global_merge_ratio=0.8, local_merge_ratio=0.9, global_rand=0.5, target_stride=4)
    args.update(kw)
    return {"size": (hw, hw), "hooks": [], "args": args}


# --------------------------------------------------------------------------- 1. the split itself
@pytest.mark.parametrize("B,L,C,align", [(2, 40, 64, False), (3, 40, 64, True), (2, 5325, 320, False),
                                         (3, 5325, 320, True)])
def test_coin_split_equals_the_concatenation_order(B, L, C, align):
    from vidtome_b200 import merge, ops
    from vidtome_b200._lib import VtmSplit
    g = torch.Generator(device="cuda").manual_seed(L + B)
    loc = torch.randn((B, L, C), generator=g, device="cuda").half()
    glo = torch.randn((B, L, C), generator=g, device="cuda").half()
    cat = torch.cat([loc, glo], dim=1)
    ref = VtmSplit.prefix(2 * L, L)
    r = torch.arange(2 * L, device="cuda")
    for coin_v, thr in ((0.75, 0.5), (0.25, 0.5), (0.5, 0.5)):
        swapped = not (coin_v > thr)
        tokens = torch.cat([glo, loc], dim=1) if swapped else cat           # the reference's order (patch.py:63-71)
        conc = (r + L) % (2 * L) if swapped else r                          # storage position -> concatenation position
        sp = VtmSplit.prefix_coin(L, torch.tensor([coin_v], device="cuda"), thr)
        assert ops.split_counts(sp) == (L, L)
        a0, b0 = ops.normalize_split(tokens, None, ref)
        a1, b1 = ops.normalize_split(cat, None, sp)
        assert torch.equal(a0, a1) and torch.equal(b0, b1), (coin_v, thr)
        m0 = merge.match_level(tokens, None, ref, 0.8, align)
        m1 = merge.match_level(cat, None, sp, 0.8, align)
        assert torch.equal(m0.keys, m1.keys) and torch.equal(m0.edge, m1.edge)
        mu0, pi0 = ops.compose_maps(ref, m0.r, m0.keys, m0.edge, m0.rank, None, None, 0, 2 * L)
        mu1, pi1 = ops.compose_maps(sp, m1.r, m1.keys, m1.edge, m1.rank, None, None, 0, 2 * L)
        assert torch.equal(conc[mu1.long()], mu0.long())
        assert torch.equal(pi1, pi0[:, conc])
        assert torch.equal(ops.gather_rows(cat, mu1), ops.gather_rows(tokens, mu0))
        y0 = ops.merge_reduce(tokens, ref, m0.r, m0.keys, m0.edge, "mean")
        y1 = ops.merge_reduce(cat, sp, m1.r, m1.keys, m1.edge, "mean")
        assert torch.equal(y0, y1)
    coin = torch.tensor([0.9], device="cuda")
    with pytest.raises(RuntimeError):
        ops.split_counts(VtmSplit(1, 2 * L + 1, 0, 0, 0, 0, 0, L, None, coin.data_ptr(), 0.5))


# --------------------------------------------------------------------------- 2. the global stage under capture
def test_captured_global_stage_replays_like_eager():
    from vidtome_b200 import patch
    B, F, hw, C = 2, 4, 8, 128
    info = _info(B, hw)
    gx = torch.Generator(device="cuda").manual_seed(3)
    xs = [torch.randn((B * F, hw * hw, C), generator=gx, device="cuda").half() for _ in range(2)]
    n = 12

    eager_mod = SimpleNamespace(generator=torch.Generator(device="cuda").manual_seed(7), global_tokens=None)
    want = []
    for _ in range(n):
        eager_mod.global_tokens = None
        patch.build_merge_plan(eager_mod, xs[0], info)
        p1 = patch.build_merge_plan(eager_mod, xs[1], info)
        want.append((p1.merged_tokens.clone(), p1.pi.clone(), eager_mod.global_tokens.clone(), p1.coin))
    coins = [w[3] for w in want]
    assert min(coins) <= 0.5 < max(coins), coins                         # both sides of global_rand occur

    gen = torch.Generator(device="cuda").manual_seed(7)
    mod = SimpleNamespace(generator=gen, global_tokens=None)
    graph = torch.cuda.CUDAGraph()
    graph.register_generator_state(gen)
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        patch.build_merge_plan(mod, xs[0], info)
        p1 = patch.build_merge_plan(mod, xs[1], info)
        stored = mod.global_tokens
    assert isinstance(p1.coin, torch.Tensor)
    for k in range(n):
        graph.replay()
        torch.cuda.synchronize()
        merged, pi, glob, coin = want[k]
        assert float(p1.coin.item()) == coin, k
        assert torch.equal(p1.merged_tokens, merged), k
        assert torch.equal(p1.pi, pi), k
        assert torch.equal(stored, glob), k


def test_capture_refuses_unequal_token_sets():
    from vidtome_b200 import patch
    B, hw, C = 2, 8, 128
    info = _info(B, hw)
    gx = torch.Generator(device="cuda").manual_seed(4)
    x4 = torch.randn((B * 4, hw * hw, C), generator=gx, device="cuda").half()
    x2 = torch.randn((B * 2, hw * hw, C), generator=gx, device="cuda").half()
    gen = torch.Generator(device="cuda").manual_seed(1)
    mod = SimpleNamespace(generator=gen, global_tokens=None)
    patch.build_merge_plan(mod, x4, info)                                  # stores 4 frames' worth of tokens
    graph = torch.cuda.CUDAGraph()
    graph.register_generator_state(gen)
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="divisible"):
        with torch.cuda.graph(graph):
            patch.build_merge_plan(mod, x2, info)


# --------------------------------------------------------------------------- 3. reference fixtures, device coin
class Replay:
    """Feed recorded torch.randint / torch.rand values to the code under test (as tests/test_gpu_parity.py does)."""

    def __init__(self, monkeypatch, randint=(), rand=()):
        self.ri, self.rr = [int(v) for v in randint], [float(v) for v in rand]
        monkeypatch.setattr(torch, "randint", self._randint)
        monkeypatch.setattr(torch, "rand", self._rand)

    def _randint(self, lo, hi, size, generator=None, device=None, **kw):
        v = self.ri.pop(0)
        assert lo <= v < hi
        return torch.full(tuple(size), v, dtype=torch.int64, device=device)

    def _rand(self, *size, generator=None, device=None, **kw):
        return torch.full((1,), self.rr.pop(0), dtype=torch.float32, device=device)

    def done(self):
        return not self.ri and not self.rr


@pytest.mark.parametrize("name", ["compute_merge_exact_global", "compute_merge_exact_global_align",
                                  "compute_merge_exact_global_rand0", "compute_merge_exact_global_rand1"])
def test_compute_merge_with_device_coin_bit_exact_vs_reference(name, monkeypatch):
    from vidtome_b200 import patch
    monkeypatch.setattr(patch, "DEVICE_COIN", True)
    g = np.load(os.path.join(GOLD, name + ".npz"))
    info = {"size": tuple(int(v) for v in g["size"]), "hooks": [], "args": dict(
        max_downsample=int(g["arg_max_downsample"]), generator=None, seed=123, batch_size=int(g["batch_size"]),
        align_batch=bool(g["arg_align_batch"]), merge_global=bool(g["arg_merge_global"]),
        global_merge_ratio=float(g["arg_global_merge_ratio"]), local_merge_ratio=float(g["arg_local_merge_ratio"]),
        global_rand=float(g["arg_global_rand"]), target_stride=int(g["arg_target_stride"]))}
    module = SimpleNamespace(generator=torch.Generator(device="cuda").manual_seed(0), global_tokens=None)
    device_coins = 0
    for i in range(int(g["n_chunks"])):
        rp = Replay(monkeypatch, randint=g[f"randint{i}"], rand=g[f"rand{i}"])
        x = torch.from_numpy(g[f"x{i}"]).cuda()
        m, u, merged = patch.compute_merge(module, x, info)
        assert rp.done(), "different number of random draws than the reference"
        device_coins += isinstance(m.plan.coin, torch.Tensor)
        np.testing.assert_array_equal(merged.cpu().numpy(), g[f"merged{i}"])
        np.testing.assert_array_equal(u(merged).cpu().numpy(), g[f"back{i}"])
        if f"global{i}" in g.files:
            np.testing.assert_array_equal(module.global_tokens.cpu().numpy(), g[f"global{i}"])
    assert device_coins >= 1, "the device-coin branch never ran"


# --------------------------------------------------------------------------- 4./5. the driver, graph vs eager
def _run(graph: bool, steps: int, chunk_ord: str, frames: int = 16, size: int = 16, name: str = "tiny"):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton
    torch.manual_seed(77)
    net = make_skeleton(name, device="cuda")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=True, global_merge_ratio=0.8, batch_size=2)
    den = ChunkedDenoiser(net, n_timesteps=50, chunk_size=4, merge_global=True, chunk_ord=chunk_ord,
                          cuda_graph=graph, capture_global=graph, graph_warmup=2)
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn((frames, 4, size, size), generator=g, device="cuda", dtype=torch.float16)
    torch.manual_seed(2024)              # host draws of get_chunks and the device RNG the blocks fork from
    xs = []
    for i in range(steps):
        x = den.step(x, i)
        xs.append(x.clone())
    torch.cuda.synchronize()
    return xs, den


@pytest.mark.parametrize("chunk_ord", ["seq", "rand", "mix-4"])
def test_driver_graph_with_global_merging_is_bit_identical_to_eager(chunk_ord):
    eager, _ = _run(False, 7, chunk_ord)
    graph, den = _run(True, 7, chunk_ord)
    assert den._graph is not None, "the graph was never captured"
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(a).all()
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"
    assert not torch.equal(graph[3], graph[4])


def test_driver_graph_with_global_merging_full_size():
    """BASELINE config 3's shape: SD1.5 skeleton at 512x512 (latent 64), 32 frames in chunks of 4."""
    eager, _ = _run(False, 4, "mix-4", frames=32, size=64, name="sd15")
    graph, den = _run(True, 4, "mix-4", frames=32, size=64, name="sd15")
    assert den._graph is not None
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(b).all()
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"


# --------------------------------------------------------------------------- 6. refusals
def test_driver_refuses_unequal_chunks_before_capture():
    with pytest.raises(RuntimeError, match="divisible by chunk_size"):
        _run(True, 3, "seq", frames=18)


def test_driver_refuses_collective_exchange_before_capture(monkeypatch):
    from vidtome_b200 import patch
    monkeypatch.setattr(patch, "GLOBAL_EXCHANGE", "allgather")
    with pytest.raises(RuntimeError, match="recurrence"):
        _run(True, 3, "seq")
