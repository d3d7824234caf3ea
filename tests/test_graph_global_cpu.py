"""Host side of capturing global merging in a CUDA graph (no GPU needed): the vtm_split_t layout with the device coin,
VtmSplit.prefix_coin's argument checks, the coin split's count rule, ChunkedDenoiser(capture_global=True)'s
constructor rules and eager stepping on CPU tensors, and the slot index of every chunk order."""
import ctypes

import numpy as np
import pytest
import torch


def _skeleton():
    from vidtome_b200.skeleton import make_skeleton
    return make_skeleton("tiny", device="cpu", dtype=torch.float32)


def test_split_layout_appends_the_coin_at_the_tail():
    from vidtome_b200._lib import VtmSplit
    offs = {name: getattr(VtmSplit, name).offset for name, _ in VtmSplit._fields_}
    assert [offs[n] for n in ("mode", "N", "unm_pre", "F", "tnum", "stride", "randf", "src_len")] == list(range(0, 32, 4))
    assert offs["randf_dev"] == 32 and offs["coin_dev"] == 40 and offs["coin_threshold"] == 48
    assert ctypes.sizeof(VtmSplit) == 56
    old = VtmSplit(1, 100, 0, 0, 0, 0, 0, 37)                 # the 8-value positional form still works
    assert (old.mode, old.N, old.src_len) == (1, 100, 37)
    assert not old.randf_dev and not old.coin_dev and old.coin_threshold == 0.0


def test_coin_split_counts_need_equal_halves():
    from vidtome_b200 import _lib
    from vidtome_b200._lib import VtmSplit
    lib = _lib.load()
    ns, nd = ctypes.c_int32(), ctypes.c_int32()
    fake = ctypes.c_void_p(0x1000).value                     # never dereferenced by the host helper
    ok = VtmSplit(1, 2 * 70, 0, 0, 0, 0, 0, 70, None, fake, 0.5)
    assert lib.vtm_split_counts(ctypes.byref(ok), ctypes.byref(ns), ctypes.byref(nd)) == 0
    assert (ns.value, nd.value) == (70, 70)
    for N, src_len in ((150, 70), (140, 60), (0, 0)):
        bad = VtmSplit(1, N, 0, 0, 0, 0, 0, src_len, None, fake, 0.5)
        assert lib.vtm_split_counts(ctypes.byref(bad), ctypes.byref(ns), ctypes.byref(nd)) == -3, (N, src_len)
    # without a coin the same unequal split is a plain prefix split
    plain = VtmSplit(1, 150, 0, 0, 0, 0, 0, 70, None, None, 0.5)
    assert lib.vtm_split_counts(ctypes.byref(plain), ctypes.byref(ns), ctypes.byref(nd)) == 0
    assert (ns.value, nd.value) == (70, 80)


def test_prefix_coin_checks_its_arguments():
    from vidtome_b200._lib import VtmSplit
    with pytest.raises(RuntimeError, match="float32 CUDA tensor"):
        VtmSplit.prefix_coin(64, torch.zeros(1), 0.5)                       # CPU tensor
    with pytest.raises(RuntimeError, match="float32 CUDA tensor"):
        VtmSplit.prefix_coin(64, 0.7, 0.5)                                  # host float
    with pytest.raises(RuntimeError, match="float32 CUDA tensor"):
        VtmSplit.prefix_coin(64, torch.zeros(2, dtype=torch.int32), 0.5)
    assert ctypes.sizeof(VtmSplit.prefix(10, 5)) == 56


def test_capture_global_constructor_rules():
    from vidtome_b200.driver import ChunkedDenoiser
    net = _skeleton()
    den = ChunkedDenoiser(net, chunk_size=4, merge_global=True, cuda_graph=True, capture_global=True)
    assert den.capture_global and den._graph is None
    with pytest.raises(ValueError, match="cuda_graph"):
        ChunkedDenoiser(net, merge_global=True, cuda_graph=True)             # without the new keyword: refused as before
    with pytest.raises(ValueError):
        ChunkedDenoiser(net, merge_global=True, cuda_graph=True, capture_global=True, randomize_chunks=True)
    with pytest.raises(ValueError):
        ChunkedDenoiser(net, merge_global=True, cuda_graph=True, capture_global=True, shard=True)
    with pytest.raises(ValueError, match="capture_global"):
        ChunkedDenoiser(net, merge_global=True, capture_global=True)         # nothing to capture


def test_capture_global_steps_eagerly_on_cpu_tensors():
    from vidtome_b200.driver import ChunkedDenoiser
    net = _skeleton()
    ref = ChunkedDenoiser(net, n_timesteps=10, chunk_size=4, merge_global=True, chunk_ord="mix-4")
    den = ChunkedDenoiser(net, n_timesteps=10, chunk_size=4, merge_global=True, chunk_ord="mix-4", cuda_graph=True,
                          capture_global=True, graph_warmup=1)
    x0 = torch.randn(8, 4, 8, 8, generator=torch.Generator().manual_seed(0))
    outs = []
    for d in (ref, den):
        torch.manual_seed(4)
        x = x0
        for i in range(3):
            x = d.step(x, i)
        outs.append(x)
    assert den._graph is None
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("chunk_ord", ["seq", "rand", "mix", "mix-4"])
def test_slot_index_round_trips(chunk_ord):
    from vidtome_b200.driver import ChunkedDenoiser
    den = ChunkedDenoiser(_skeleton(), chunk_size=4, merge_global=True, chunk_ord=chunk_ord)
    flen = 32
    x = torch.arange(flen * 3, dtype=torch.float32).reshape(flen, 3)
    for seed in range(6):
        torch.manual_seed(seed)
        chunks = den.get_chunks(flen)
        idx = ChunkedDenoiser.slot_index(chunks, flen)
        assert idx.shape == (2, flen) and idx.dtype == torch.int64
        slots = x[idx[0]]
        for k, c in enumerate(chunks):                      # slot k holds chunk k of the visiting order
            assert torch.equal(slots[4 * k:4 * k + 4], x[c])
        assert torch.equal(slots[idx[1]], x)                # and the inverse puts every frame back
        assert torch.equal(idx[0][idx[1]], torch.arange(flen))
    with pytest.raises(RuntimeError):
        ChunkedDenoiser.slot_index([torch.arange(0, 4), torch.arange(4, 6)], 6)


def test_draw_coin_consumes_the_reference_draw_on_cpu():
    from vidtome_b200 import utils
    g1 = torch.Generator().manual_seed(9)
    g2 = torch.Generator().manual_seed(9)
    want = [float(torch.rand(1, generator=g1)) for _ in range(4)]
    got = [utils.draw_coin(g2) for _ in range(4)]
    assert got == want and all(isinstance(v, float) for v in got)
    with pytest.raises(RuntimeError, match="CUDA generator"):
        utils.draw_coin(g2, on_device=True)
    assert np.isfinite(got).all()
