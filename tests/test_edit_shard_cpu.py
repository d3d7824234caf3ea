"""Edits of a multi-prompt generation split over the ranks, host side: the partition of dist.shard_edits and the
all-gather of dist.gather_edits over gloo worlds of 2 and 3 spawned processes; ChunkedDenoiser(cond=[K, S, 77, D],
shard=True) on a stand-in UNet that draws from torch's default generator at every call, whose gathered result must be
the unsharded K-edit run's bit for bit; and every refusal, each raised on every rank so that none is left waiting.
The library's merge path runs in tests/test_gpu_edit_shard.py."""
import os
import socket
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

STEPS, FRAMES = 4, 6


class DrawingUNet(torch.nn.Module):
    """Every output row depends on its own latent, its own text row and the timestep, plus one value drawn from the
    default generator per call and shared by the whole batch, as a block's draws are shared by all edits."""

    def __init__(self, edits):
        super().__init__()
        self._tome_info = {"args": {"batch_size": 2, "align_batch": False, "edits": edits}}

    def forward(self, sample, t, encoder_hidden_states=None, **kwargs):
        eps = sample * 0.9 + float(t) * 1e-3 + 1e-2 * torch.rand(())
        return SimpleNamespace(sample=eps + 0.5 * encoder_hidden_states.mean(dim=(1, 2))[:, None, None, None])


def _cond(K):
    return torch.randn((K, 2, 77, 16), generator=torch.Generator().manual_seed(11))


def _noise(K):
    return torch.randn((K, FRAMES, 4, 4, 4), generator=torch.Generator().manual_seed(12))


def _denoiser(K, edits, shard, **kw):
    from vidtome_b200.driver import ChunkedDenoiser
    kw = dict(dict(n_timesteps=STEPS, chunk_size=4, merge_global=True, chunk_ord="mix-4", randomize_chunks=True), **kw)
    return ChunkedDenoiser(DrawingUNet(edits), cond=_cond(K), shard=shard, **kw)


def _seed(seed=2024):
    torch.manual_seed(seed)
    np.random.seed(seed)


# --------------------------------------------------------------------------- the partition
@pytest.mark.parametrize("K", [2, 3, 5])
@pytest.mark.parametrize("world", [1, 2, 3])
def test_shard_edits_partitions_the_edits(K, world):
    from vidtome_b200 import dist as vd
    parts = [vd.shard_edits(K, r, world) for r in range(world)]
    assert sorted(k for p in parts for k in p) == list(range(K))
    for r, p in enumerate(parts):
        assert p == list(range(r, K, world))
    assert vd.shard_edits(K) == list(range(K))                         # one process runs every edit


def test_gather_edits_single_process_is_identity():
    from vidtome_b200 import dist as vd
    t = torch.randn(3, 5, 2)
    assert vd.gather_edits(t, 3) is t


def test_shard_without_a_process_group_is_refused():
    assert not dist.is_initialized()
    with pytest.raises(ValueError, match="process group"):
        _denoiser(2, 1, True)


def test_unsharded_refusal_names_the_edits():
    with pytest.raises(ValueError, match="the cond has 2 edit"):
        _denoiser(2, 1, False)


# --------------------------------------------------------------------------- gloo worlds
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _raises_everywhere(fn, match):
    """fn() must raise ValueError matching `match` here; a barrier afterwards shows no rank was left in a collective."""
    try:
        fn()
    except ValueError as e:
        assert match in str(e), str(e)
    else:
        raise AssertionError(f"not refused: {match}")
    dist.barrier()


def _worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from vidtome_b200 import dist as vd, patch
        for K in (2, 3, 5):
            if K < world:
                continue
            mine = vd.shard_edits(K)
            full = torch.arange(K * 6, dtype=torch.float32).view(K, 2, 3) * 1.5
            got = vd.gather_edits(full[mine].clone(), K)
            assert torch.equal(got, full), (K, world, rank)
        if world == 3:
            _raises_everywhere(lambda: _denoiser(2, 1, True), "at most 2 ranks")
            return
        results = {}
        # the whole job: K = 3 over 2 ranks, rank 0 runs edits 0 and 2, rank 1 edit 1 (K_r == 1)
        for name, start in (("all_rows", _noise(3)), ("own_rows", _noise(3)[vd.shard_edits(3)]),
                            ("one_noise", _noise(3)[0])):
            den = _denoiser(3, len(vd.shard_edits(3)), True)
            assert den.edits == len(vd.shard_edits(3)) and den.cond.shape[0] == den.edits and not den.shard
            _seed()
            results[name] = den.sample(start)
        den = _denoiser(3, len(vd.shard_edits(3)), True)
        _seed()
        results["steps"] = [den.step(_noise(3)[vd.shard_edits(3)], i) for i in range(2)]
        torch.save(results, os.path.join(out_dir, f"rank{rank}.pt"))
        # refusals, each on both ranks
        K_r = len(vd.shard_edits(3))
        _raises_everywhere(lambda: _denoiser(3, K_r + 1, True), f"this rank runs {K_r} of the 3 edits")
        for key, kw, x in (("edits", {}, None), ("latents", {}, _noise(2)[:, :4 + 2 * rank]),
                           ("n_timesteps", dict(n_timesteps=STEPS + rank), None),
                           ("mode", dict(chunk_size=4 - rank), None), ("rng", {}, None), ("exchange", {}, None)):
            K = 2 + rank if key == "edits" else 2
            den = _denoiser(K, 1, True, **kw)
            _seed(2024 + rank if key == "rng" else 2024)
            saved = patch.GLOBAL_EXCHANGE
            if key == "exchange" and rank == 1:
                patch.GLOBAL_EXCHANGE = "allgather"
            try:
                _raises_everywhere(lambda: den.sample(_noise(K) if x is None else x), f"disagree on {key}")
            finally:
                patch.GLOBAL_EXCHANGE = saved
        patch.GLOBAL_EXCHANGE = "allgather"
        try:
            _raises_everywhere(lambda: _denoiser(2, 1, True), "GLOBAL_EXCHANGE='recurrence'")
        finally:
            patch.GLOBAL_EXCHANGE = "recurrence"
        with open(os.path.join(out_dir, f"done{rank}"), "w"):
            pass
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_world(tmp_path, world):
    """gather_edits for K in (2, 3, 5) over the world; with world 2 a sharded K = 3 generation (every form of the
    initial latents, and step() on the rank's rows) against the unsharded run, and the refusals; with world 3 the
    refusal of more ranks than edits."""
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    if world == 3:
        return
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        want = {}
        for name, start in (("all_rows", _noise(3)), ("one_noise", _noise(3)[0])):
            _seed()
            want[name] = _denoiser(3, 3, False).sample(start)
        want["own_rows"] = want["all_rows"]
        den = _denoiser(3, 3, False)
        _seed()
        steps = [den.step(_noise(3), i) for i in range(2)]
    finally:
        torch.set_num_threads(threads)
    assert not torch.equal(want["all_rows"][0], want["all_rows"][1])
    for rank, rows in ((0, [0, 2]), (1, [1])):
        assert os.path.exists(tmp_path / f"done{rank}")
        got = torch.load(tmp_path / f"rank{rank}.pt")
        for name in ("all_rows", "own_rows", "one_noise"):
            assert got[name].shape == (3, FRAMES, 4, 4, 4), (rank, name)
            assert torch.equal(got[name], want[name]), (rank, name)
        for a, b in zip(got["steps"], steps):
            assert torch.equal(a, b[rows]), rank
