"""Host side of replaying the reference's randomised chunking from CUDA graphs (no GPU needed): the vtm_split_t layout
with the mode-2 tail, its argument checks and capacity counts, ChunkedDenoiser(chunk_graphs=True)'s constructor rules,
the chunk lengths it refuses, and the host draws of get_chunks in both modes."""
import ctypes

import numpy as np
import pytest
import torch


def _skeleton():
    from vidtome_b200.skeleton import make_skeleton
    return make_skeleton("tiny", device="cpu", dtype=torch.float32)


def test_split_layout_appends_the_device_count_tail():
    from vidtome_b200._lib import VtmSplit, VtmSplitDev
    assert ctypes.sizeof(VtmSplit) == 56                      # modes 0 and 1 keep the shorter form
    assert VtmSplitDev.glob_len_dev.offset == 56 and VtmSplitDev.glob_cap.offset == 64
    assert ctypes.sizeof(VtmSplitDev) == 72
    old = VtmSplitDev(1, 100, 0, 0, 0, 0, 0, 37)              # the 8-value positional form still works
    assert (old.mode, old.N, old.src_len) == (1, 100, 37) and not old.glob_len_dev and old.glob_cap == 0


def test_device_count_split_counts_are_capacities():
    from vidtome_b200 import _lib
    from vidtome_b200._lib import VtmSplitDev
    lib = _lib.load()
    ns, nd = ctypes.c_int32(), ctypes.c_int32()
    coin, glen = ctypes.c_void_p(0x1000).value, ctypes.c_void_p(0x2000).value    # never dereferenced on the host
    for L, cap in ((40, 25), (25, 40), (40, 40)):
        ok = VtmSplitDev(2, L + cap, 0, 0, 0, 0, 0, L, None, coin, 0.5, glen, cap)
        assert lib.vtm_split_counts(ctypes.byref(ok), ctypes.byref(ns), ctypes.byref(nd)) == 0
        assert (ns.value, nd.value) == (max(L, cap), max(L, cap))
    bad = [VtmSplitDev(2, 41 + 25, 0, 0, 0, 0, 0, 40, None, coin, 0.5, glen, 25),     # N != L + cap
           VtmSplitDev(2, 65, 0, 0, 0, 0, 0, 40, None, None, 0.5, glen, 25),          # no coin
           VtmSplitDev(2, 65, 0, 0, 0, 0, 0, 40, None, coin, 0.5, None, 25),          # no length
           VtmSplitDev(2, 40, 0, 0, 0, 0, 0, 40, None, coin, 0.5, glen, 0)]           # no capacity
    for sp in bad:
        assert lib.vtm_split_counts(ctypes.byref(sp), ctypes.byref(ns), ctypes.byref(nd)) == -3
    # the device counts exist only for mode 2 (refused on the host, before any launch)
    plain = VtmSplitDev(1, 65, 0, 0, 0, 0, 0, 40)
    assert lib.vtm_split_counts_dev(ctypes.byref(plain), 0.8, ctypes.c_void_p(0x3000), None) == -3


def test_prefix_coin_dev_checks_its_arguments():
    from vidtome_b200._lib import VtmSplit
    ln = torch.zeros(1, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="float32 CUDA tensor"):
        VtmSplit.prefix_coin_dev(64, ln, 80, torch.zeros(1), 0.5)          # CPU coin
    with pytest.raises(RuntimeError, match="float32 CUDA tensor"):
        VtmSplit.prefix_coin_dev(64, ln, 80, 0.7, 0.5)                     # host float


def test_chunk_graphs_constructor_rules():
    from vidtome_b200.driver import ChunkedDenoiser
    net = _skeleton()
    den = ChunkedDenoiser(net, chunk_size=4, merge_global=True, randomize_chunks=True, cuda_graph=True,
                          chunk_graphs=True)
    assert den.chunk_graphs and not den._chunk_graphs
    ChunkedDenoiser(net, chunk_size=4, merge_global=False, randomize_chunks=True, cuda_graph=True, chunk_graphs=True)
    with pytest.raises(ValueError, match="chunk_graphs"):
        ChunkedDenoiser(net, merge_global=True, chunk_graphs=True)                         # nothing to capture
    with pytest.raises(ValueError, match="chunk_graphs"):
        ChunkedDenoiser(net, merge_global=True, cuda_graph=True, capture_global=True, chunk_graphs=True)
    with pytest.raises(ValueError, match="shard"):
        ChunkedDenoiser(net, cuda_graph=True, chunk_graphs=True, shard=True)
    with pytest.raises(ValueError, match="graph_warmup"):
        ChunkedDenoiser(net, merge_global=True, cuda_graph=True, chunk_graphs=True, graph_warmup=0)
    # the refusals that existed before stay
    with pytest.raises(ValueError):
        ChunkedDenoiser(net, merge_global=True, cuda_graph=True, capture_global=True, randomize_chunks=True)
    with pytest.raises(ValueError):
        ChunkedDenoiser(net, cuda_graph=True, randomize_chunks=True)
    with pytest.raises(ValueError):
        ChunkedDenoiser(net, merge_global=True, cuda_graph=True)


def test_draw_dependent_chunk_lengths():
    from vidtome_b200.driver import ChunkedDenoiser
    assert ChunkedDenoiser.draw_dependent_lengths(4, 4) == []
    assert ChunkedDenoiser.draw_dependent_lengths(8, 4) == [5, 6, 7]
    assert ChunkedDenoiser.draw_dependent_lengths(16, 4) == [5, 6, 7, 9, 10, 11, 13, 14, 15]
    assert ChunkedDenoiser.draw_dependent_lengths(8, 2) == [3, 5, 6, 7]


def test_possible_chunk_lengths_cover_every_draw():
    from vidtome_b200.driver import ChunkedDenoiser
    net = _skeleton()
    for randomize in (True, False):
        den = ChunkedDenoiser(net, chunk_size=4, merge_global=True, chunk_ord="mix-4", randomize_chunks=randomize)
        for flen in (3, 16, 18, 30):
            seen = set()
            np.random.seed(flen)
            torch.manual_seed(flen)
            for _ in range(200):
                chunks = den.get_chunks(flen)
                assert sorted(int(i) for c in chunks for i in c) == list(range(flen))
                seen |= {len(c) for c in chunks}
            assert seen <= set(den.possible_lengths(flen)), (randomize, flen)
            if randomize and flen >= 8:
                assert set(den.possible_lengths(flen)) == set(range(1, 5))
    assert ChunkedDenoiser(net, chunk_size=4).possible_lengths(18) == [2, 4]


@pytest.mark.parametrize("merge_global", [True, False])
def test_get_chunks_consumes_the_same_host_draws_in_both_modes(merge_global):
    """On CPU tensors the chunk-graph denoiser steps eagerly: same latents and the same numpy / torch host RNG state."""
    from vidtome_b200.driver import ChunkedDenoiser
    net = _skeleton()
    kw = dict(n_timesteps=10, chunk_size=4, merge_global=merge_global, chunk_ord="mix-4", randomize_chunks=True)
    ref = ChunkedDenoiser(net, **kw)
    den = ChunkedDenoiser(net, cuda_graph=True, chunk_graphs=True, graph_warmup=1, **kw)
    x0 = torch.randn(18, 4, 8, 8, generator=torch.Generator().manual_seed(0))
    outs, states = [], []
    for d in (ref, den):
        np.random.seed(3)
        torch.manual_seed(4)
        x = x0
        for i in range(3):
            x = d.step(x, i)
        outs.append(x)
        states.append((np.random.rand(), float(torch.rand(1))))
    assert not den._chunk_graphs
    assert torch.equal(outs[0], outs[1])
    assert states[0] == states[1]
