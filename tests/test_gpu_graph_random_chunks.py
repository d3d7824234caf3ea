"""The reference's randomised chunking (random first chunk length, reversed half the time) replayed from CUDA graphs:
ChunkedDenoiser(chunk_graphs=True) captures one graph per chunk length, and the global stage runs on a GlobalTokenStore
whose coin-dependent counts (Ns, Nd, r, the merged length M) stay on the device (vtm_split_t mode 2).  Everything here
checks that this computes, bit for bit, what the same work computes with the counts known on the host."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# --------------------------------------------------------------------------- 0. the RNG premise, checked first
def test_generator_shared_by_several_graphs_draws_like_eager():
    """One generator registered with several graphs: replays in any order advance it exactly as eager draws do."""
    def draws(g, n):
        return [torch.rand(n, generator=g, device="cuda"), torch.randint(0, 4, (1,), generator=g, device="cuda")]

    sizes = (1, 3, 2)
    order = [0, 1, 1, 2, 0, 2, 2, 1, 0, 0]
    eager_g = torch.Generator(device="cuda").manual_seed(11)
    want = [[t.clone() for t in draws(eager_g, sizes[k])] for k in order]

    g = torch.Generator(device="cuda").manual_seed(11)
    graphs, outs = [], []
    for n in sizes:
        graph = torch.cuda.CUDAGraph()
        graph.register_generator_state(g)
        torch.cuda.synchronize()
        with torch.cuda.graph(graph):
            out = draws(g, n)
        graphs.append(graph)
        outs.append(out)
    for i, k in enumerate(order):
        graphs[k].replay()
        torch.cuda.synchronize()
        for a, b in zip(outs[k], want[i]):
            assert torch.equal(a, b), (i, k)
    after_eager = torch.rand(4, generator=eager_g, device="cuda")
    assert torch.equal(torch.rand(4, generator=g, device="cuda"), after_eager)


# --------------------------------------------------------------------------- 1. the device-count global stage
def _tokens(shape, gen, exact):
    if exact:   # small integers: exact products and many ties, which exercise the first-index rule
        return torch.randint(-2, 3, shape, generator=gen, device="cuda").half()
    return torch.randn(shape, generator=gen, device="cuda").half()


def _attn_weights(C, gen):
    w_qkv = (torch.randn((3 * C, C), generator=gen, device="cuda") * C ** -0.5).half()
    w_o = (torch.randn((C, C), generator=gen, device="cuda") * C ** -0.5).half()
    b_o = (torch.randn((C,), generator=gen, device="cuda") * 0.1).half()
    return w_qkv, w_o, b_o


@pytest.mark.parametrize("B,L,Lg,C,align,exact", [
    (2, 40, 25, 64, False, False), (2, 25, 40, 64, True, False), (3, 40, 40, 64, False, True),
    (2, 31, 57, 64, False, True),
    (2, 5325, 4096, 320, False, False), (2, 5325, 4506, 320, True, False), (2, 5325, 4916, 320, False, True)])
def test_store_stage_matches_the_host_count_path(B, L, Lg, C, align, exact):
    from vidtome_b200 import merge, ops
    from vidtome_b200._lib import VtmSplit
    gen = torch.Generator(device="cuda").manual_seed(L * 7 + Lg)
    cap = max(L, Lg) + 13                                          # the store may be larger than both sets
    loc = _tokens((B, L, C), gen, exact)
    glo = _tokens((B, Lg, C), gen, exact)
    store = torch.randn((B, cap, C), generator=gen, device="cuda").half()   # stale rows past Lg
    store[:, :Lg] = glo
    cat = torch.cat([loc, store], dim=1)
    glen = torch.tensor([Lg], dtype=torch.int32, device="cuda")
    heads = C // 64
    w_qkv, w_o, b_o = _attn_weights(C, gen)
    ratio = 0.8
    for thr in (0.0, 1.0):                                         # coin 0.5: local is src, then global is src
        coin = torch.tensor([0.5], device="cuda")
        swapped = not (0.5 > thr)
        tokens = torch.cat([glo, loc], dim=1) if swapped else torch.cat([loc, glo], dim=1)
        src_len, off = (Lg, Lg) if swapped else (L, 0)
        ref = VtmSplit.prefix(L + Lg, src_len)
        m0 = merge.match_level(tokens, None, ref, ratio, align)
        mu0, tau0 = ops.compose_maps(ref, m0.r, m0.keys, m0.edge, m0.rank, None, None, 0, L + Lg)
        merged0 = ops.gather_rows(tokens, mu0)
        glob0 = ops.unmerge_add(merged0, tau0[:, off:off + L].contiguous(), None)
        M = merged0.shape[1]

        sp = VtmSplit.prefix_coin_dev(L, glen, cap, coin, thr)
        m1 = merge.match_level_dev(cat, sp, ratio, align)
        assert m1.counts.tolist() == [m0.Ns, m0.Nd, m0.r, M], thr
        Ns = m0.Ns
        assert torch.equal(m1.keys[:, :Ns], m0.keys) and torch.equal(m1.edge[:, :Ns], m0.edge), thr
        assert torch.equal(m1.rank[:, :Ns], m0.rank), thr
        mu1, tau1 = ops.compose_maps_dev(sp, m1.counts, m1.keys, m1.edge, m1.rank, None, L + cap)
        # storage position -> concatenation position
        r = torch.arange(L + Lg, device="cuda")
        conc = torch.where(r < L, r + Lg, r - L) if swapped else r
        assert torch.equal(conc[mu1[:, :M].long()], mu0.long()), thr
        assert torch.equal(tau1[:, :L + Lg], tau0[:, conc]), thr
        merged1 = ops.gather_rows_dev(cat, mu1, m1.counts[3:4])
        assert torch.equal(merged1[:, :M], merged0), thr
        assert not merged1[:, M:].any(), thr
        glob1 = ops.unmerge_add(merged1, tau1[:, :L], None)
        assert torch.equal(glob1, glob0), thr
        # the composed unmerge map of the local tokens
        pi = torch.randint(0, L, (1 if align else B, 3 * L), generator=gen, device="cuda").to(torch.int32)
        pi0 = torch.gather(tau0, 1, (pi.long() + off)).to(torch.int32)
        _, pi1 = ops.compose_maps_dev(sp, m1.counts, m1.keys, m1.edge, m1.rank, pi, pi.shape[1])
        assert torch.equal(pi1, pi0), thr
        # KD on the capacity-sized merged tokens with the length on the device
        y0 = ops.attention(merged0.contiguous(), w_qkv, w_o, b_o, heads, 0.125)
        y1 = ops.attention(merged1, w_qkv, w_o, b_o, heads, 0.125, seq_len=m1.counts[3:4])
        assert torch.equal(y1[:, :M], y0), thr


# --------------------------------------------------------------------------- 2. reference fixtures through the store
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
def test_compute_merge_through_the_store_bit_exact_vs_reference(name, monkeypatch):
    from vidtome_b200 import patch
    g = np.load(os.path.join(GOLD, name + ".npz"))
    info = {"size": tuple(int(v) for v in g["size"]), "hooks": [], "args": dict(
        max_downsample=int(g["arg_max_downsample"]), generator=None, seed=123, batch_size=int(g["batch_size"]),
        align_batch=bool(g["arg_align_batch"]), merge_global=bool(g["arg_merge_global"]),
        global_merge_ratio=float(g["arg_global_merge_ratio"]), local_merge_ratio=float(g["arg_local_merge_ratio"]),
        global_rand=float(g["arg_global_rand"]), target_stride=int(g["arg_target_stride"]))}
    n = int(g["n_chunks"])
    frames = max(g[f"x{i}"].shape[0] // int(g["batch_size"]) for i in range(n))
    store = patch.GlobalTokenStore(frames)
    module = SimpleNamespace(generator=torch.Generator(device="cuda").manual_seed(0), global_tokens=store)
    device_counts = 0
    for i in range(n):
        rp = Replay(monkeypatch, randint=g[f"randint{i}"], rand=g[f"rand{i}"])
        x = torch.from_numpy(g[f"x{i}"]).cuda()
        m, u, merged = patch.compute_merge(module, x, info)
        assert rp.done(), "different number of random draws than the reference"
        want = g[f"merged{i}"]
        M = want.shape[1]
        if m.plan.seq_len is not None:
            device_counts += 1
            assert int(m.plan.seq_len.item()) == M
            assert not merged[:, M:].any()
        np.testing.assert_array_equal(merged[:, :M].cpu().numpy(), want)
        np.testing.assert_array_equal(u(merged).cpu().numpy(), g[f"back{i}"])
        if f"global{i}" in g.files:
            Lst = int(store.length.item())
            np.testing.assert_array_equal(store.tokens[:, :Lst].cpu().numpy(), g[f"global{i}"])
    assert device_counts >= 1, "the device-count global stage never ran"


# --------------------------------------------------------------------------- 3. KD with a device length
@pytest.mark.parametrize("C,heads,M,cap", [(320, 5, 200, 256), (320, 5, 130, 600), (128, 2, 64, 64),
                                           (640, 8, 1000, 1400), (320, 5, 5325, 9000)])
def test_attention_with_device_length_equals_host_length(C, heads, M, cap):
    from vidtome_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(M + C)
    B = 2
    x = torch.zeros((B, cap, C), dtype=torch.float16, device="cuda")
    x[:, :M] = torch.randn((B, M, C), generator=gen, device="cuda").half()
    w_qkv, w_o, b_o = _attn_weights(C, gen)
    y0 = ops.attention(x[:, :M].contiguous(), w_qkv, w_o, b_o, heads, (C // heads) ** -0.5)
    y1 = ops.attention(x, w_qkv, w_o, b_o, heads, (C // heads) ** -0.5, seq_len=torch.tensor([M], dtype=torch.int32,
                                                                                               device="cuda"))
    assert torch.isfinite(y0).all()
    assert torch.equal(y1[:, :M], y0)


# --------------------------------------------------------------------------- 4. the driver, chunk graphs vs eager
def _run(graph: bool, steps: int, chunk_ord: str, merge_global: bool, frames: int, size: int = 16,
         name: str = "tiny", record=None):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton
    torch.manual_seed(77)
    net = make_skeleton(name, device="cuda")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=merge_global, global_merge_ratio=0.8,
                             batch_size=2)
    den = ChunkedDenoiser(net, n_timesteps=50, chunk_size=4, merge_global=merge_global, chunk_ord=chunk_ord,
                          randomize_chunks=True, cuda_graph=graph, chunk_graphs=graph, graph_warmup=2)
    if record is not None:
        get_chunks = den.get_chunks

        def recorded(flen):
            chunks = get_chunks(flen)
            record["first"].add(len(chunks[0]))
            return chunks
        den.get_chunks = recorded
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn((frames, 4, size, size), generator=g, device="cuda", dtype=torch.float16)
    torch.manual_seed(2024)              # the device RNG the blocks fork from
    np.random.seed(2024)                 # the host draws of get_chunks (first chunk length, reversal)
    xs = []
    for i in range(steps):
        x = den.step(x, i)
        xs.append(x.clone())
    torch.cuda.synchronize()
    return xs, den


def _compare(chunk_ord, merge_global, frames, steps, monkeypatch, **kw):
    from vidtome_b200 import patch
    record = {"first": set(), "coins": []}
    draw_coin = patch.draw_coin

    def recorded_coin(generator, on_device=None):
        c = draw_coin(generator, on_device=on_device)
        if isinstance(c, float):
            record["coins"].append(c)
        return c
    monkeypatch.setattr(patch, "draw_coin", recorded_coin)
    eager, _ = _run(False, steps, chunk_ord, merge_global, frames, record=record, **kw)
    monkeypatch.setattr(patch, "draw_coin", draw_coin)
    graph, den = _run(True, steps, chunk_ord, merge_global, frames, **kw)
    assert den._chunk_graphs, "no graph was captured"
    assert len(record["first"]) >= 2, record["first"]
    if merge_global:
        assert min(record["coins"]) <= 0.5 < max(record["coins"]), "both coin outcomes must occur"
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(b).all()
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"
    return den


@pytest.mark.parametrize("chunk_ord,merge_global,frames", [("seq", True, 16), ("rand", True, 18), ("mix-4", True, 30),
                                                           ("mix-4", False, 18), ("seq", False, 30)])
def test_driver_chunk_graphs_with_random_chunks_are_bit_identical_to_eager(chunk_ord, merge_global, frames, monkeypatch):
    den = _compare(chunk_ord, merge_global, frames, 8, monkeypatch)
    assert len(den._chunk_graphs) <= 2 * den.chunk_size


def test_driver_chunk_graphs_full_size(monkeypatch):
    """BASELINE config 3 with the reference's chunking: SD1.5 skeleton at 512x512 (latent 64), 32 frames, chunk_size 4
    with a random first chunk, mix-4 order, local 0.9 + global 0.8."""
    _compare("mix-4", True, 32, 4, monkeypatch, size=64, name="sd15")


# --------------------------------------------------------------------------- 5. refusals
def test_store_refuses_other_merge_exchange_and_simt_modes(monkeypatch):
    from vidtome_b200 import merge, ops, patch
    from vidtome_b200._lib import VtmSplit
    L, Lg, cap, C = 40, 30, 48, 64
    cat = torch.randn((2, L + cap, C), device="cuda").half()
    sp = VtmSplit.prefix_coin_dev(L, torch.tensor([Lg], dtype=torch.int32, device="cuda"), cap,
                                  torch.tensor([0.7], device="cuda"), 0.5)
    m = merge.match_level_dev(cat, sp, 0.8, False)
    with pytest.raises(RuntimeError, match="inconsistent vtm_split_t"):
        ops.merge_reduce(cat, sp, 0, m.keys, m.edge, "mean")          # reductions have no device-count path
    with pytest.raises(RuntimeError, match="inconsistent vtm_split_t"):
        ops.compose_maps(sp, 0, m.keys, m.edge, m.rank, None, None, 0, L + cap)
    a, b = ops.normalize_split(cat, None, sp)
    with pytest.raises(RuntimeError, match="SIMT twin"):
        ops.sim_argmax(a, b, False, simt=True, counts=m.counts)

    info = {"size": (8, 8), "hooks": [], "args": dict(
        max_downsample=2, generator=None, seed=123, batch_size=2, align_batch=False, merge_global=True,
        global_merge_ratio=0.8, local_merge_ratio=0.9, global_rand=0.5, target_stride=4)}
    x = torch.randn((8, 64, C), device="cuda").half()
    mod = SimpleNamespace(generator=torch.Generator(device="cuda").manual_seed(1), global_tokens=patch.GlobalTokenStore(4))
    monkeypatch.setattr(patch, "GLOBAL_EXCHANGE", "allgather")
    with pytest.raises(RuntimeError, match="recurrence"):
        patch.build_merge_plan(mod, x, info)


def test_driver_refuses_draw_dependent_chunk_lengths():
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton
    net = make_skeleton("tiny", device="cuda")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=True, batch_size=2)
    den = ChunkedDenoiser(net, chunk_size=8, merge_global=True, randomize_chunks=True, cuda_graph=True,
                          chunk_graphs=True, graph_warmup=1)
    x = torch.randn((16, 4, 16, 16), device="cuda", dtype=torch.float16)
    x = den.step(x, 0)                                                 # eager warm-up: any chunk length runs
    with pytest.raises(RuntimeError, match=r"\[5, 6, 7\].*depend on the frame draw"):
        den.step(x, 1)
    assert not den._chunk_graphs
