"""Reconstruction and sharded inversion, host side: ChunkedInverter.reconstruct() on the tiny CPU skeleton against the
reference's own `Inverter.ddim_sample` (tests/golden/recon_*.npz, written by tests/make_golden_recon.py); the batch
partition of dist.shard_batches; world-2 gloo jobs whose invert() and reconstruct() are bit-identical to one process's,
over even and ragged batch counts, more ranks than batches, per-frame cond, ControlNet and depth; a sharded trajectory
feeding sharded PnP generation without a further collective; and the argument errors."""
import os
import socket
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RECON = ["f8_b4_plain", "f11_b4_ragged", "f11_b4_cond", "f6_b4_control"]


def _tiny(depth=False):
    from vidtome_b200.skeleton import make_controlnet, make_skeleton
    return (make_skeleton("tiny", hot_path_only=False, device="cpu", dtype=torch.float32, depth=depth),
            make_controlnet("tiny", hot_path_only=False, device="cpu", dtype=torch.float32))


# --------------------------------------------------------------------------- reconstruct() against the reference
@pytest.mark.parametrize("name", RECON)
def test_reconstruct_matches_reference_ddim_sample(name):
    from vidtome_b200.driver import ChunkedInverter
    g = np.load(os.path.join(GOLD, f"recon_{name}.npz"))
    unet, controlnet = _tiny()
    seed = torch.from_numpy(g["cond_seed"])
    control = bool(g["control"])
    inv = ChunkedInverter(unet, n_timesteps=int(g["steps"]), batch_size=int(g["batch_size"]),
                          cond=seed.repeat(1, 1, 768 // seed.shape[-1]), controlnet=controlnet if control else None,
                          control_images=torch.from_numpy(g["images"]) if control else None,
                          control_scale=float(g["control_scale"]))
    x = torch.from_numpy(g["x"])
    out = inv.reconstruct(x)
    assert torch.equal(x, torch.from_numpy(g["x"]))                  # the input is not modified
    want = torch.from_numpy(g["out"])
    assert out.shape == want.shape
    err = (out - want).abs().max().item()                            # test_inversion_cpu's tolerance
    assert err <= 2e-3 * want.abs().max().item() + 1e-3, err
    assert inv.trajectory is None                                     # reconstruct() keeps no trajectory


def test_reconstruct_steps_and_default_input():
    """Forward timesteps; step i is sample_next_x on the UNet's prediction, with the sampling coefficients (those of
    ChunkedDenoiser, final_alpha_cumprod at the last step); reconstruct() defaults to the final inverted latents."""
    from vidtome_b200.driver import ChunkedDenoiser, ChunkedInverter
    unet, _ = _tiny()
    torch.manual_seed(5)
    x, cond = torch.randn(5, 4, 4, 4), torch.randn(1, 77, 768)
    inv = ChunkedInverter(unet, n_timesteps=10, batch_size=2, cond=cond)
    den = ChunkedDenoiser(unet, n_timesteps=10)
    assert inv.sample_timesteps == den.timesteps == inv.timesteps[::-1]
    assert [inv.sample_coefficients(i) for i in range(10)] == [den.coefficients(i) for i in range(10)]
    one = ChunkedInverter(unet, n_timesteps=1, batch_size=2, cond=cond)
    with torch.no_grad():
        eps = torch.cat([unet(x[lo:lo + 2], 1, encoder_hidden_states=cond.expand(len(x[lo:lo + 2]), -1, -1)).sample
                         for lo in range(0, 5, 2)])
    assert one.sample_timesteps == [1]
    assert torch.equal(one.reconstruct(x), one.sample_next_x(x, eps, 0))
    a, b, c, d = one.sample_coefficients(0)
    ac = one.alphas_cumprod
    assert (c, d) == (float(ac[0] ** 0.5), float((1 - ac[0]) ** 0.5))    # the last step: final_alpha_cumprod
    final = inv.invert(x)
    assert torch.equal(inv.reconstruct(), inv.reconstruct(final))


def test_reconstruct_argument_errors():
    from vidtome_b200.driver import ChunkedInverter
    unet, controlnet = _tiny()
    x = torch.zeros(3, 4, 4, 4)
    with pytest.raises(RuntimeError, match="invert"):
        ChunkedInverter(unet).reconstruct()
    with pytest.raises(ValueError, match=r"\[F, 4, h, w\]"):
        ChunkedInverter(unet).reconstruct(x[0])
    with pytest.raises(ValueError, match="cond has 2 rows for 3 frames"):
        ChunkedInverter(unet, cond=torch.zeros(2, 77, 768)).reconstruct(x)
    with pytest.raises(ValueError, match="control_images has 2 frames"):
        ChunkedInverter(unet, controlnet=controlnet, control_images=torch.zeros(2, 3, 8, 8)).reconstruct(x)
    with pytest.raises(ValueError, match="CUDA fp16"):
        ChunkedInverter(unet, cuda_graph=True).reconstruct(x)
    assert not dist.is_initialized()
    with pytest.raises(ValueError, match="process group"):
        ChunkedInverter(unet, shard=True)


# --------------------------------------------------------------------------- the partition
@pytest.mark.parametrize("flen,batch_size", [(8, 2), (11, 4), (3, 4), (1, 1), (16, 8), (17, 8), (40, 3)])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_shard_batches_partitions_the_unsharded_batches(flen, batch_size, world):
    from vidtome_b200 import dist as vd
    unsharded = [(lo, min(lo + batch_size, flen)) for lo in range(0, flen, batch_size)]
    parts = [vd.shard_batches(flen, batch_size, r, world) for r in range(world)]
    assert sorted(b for p in parts for b in p) == unsharded
    for r, p in enumerate(parts):
        assert p == unsharded[r::world]
        assert all(hi - lo == batch_size for lo, hi in p[:-1])          # only a rank's last batch may be ragged
    assert vd.shard_batches(flen, batch_size) == unsharded             # one process takes every batch


# --------------------------------------------------------------------------- world-2 gloo jobs
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


class StandInUNet(torch.nn.Module):
    """A PnP-patched UNet stand-in whose every output row depends on its own sample, text row and the timestep."""

    def __init__(self):
        super().__init__()
        self._tome_info = {"args": {"batch_size": 3, "align_batch": True}}

    def forward(self, sample, t, encoder_hidden_states=None, **kwargs):
        eps = sample * 0.9 + float(t) * 1e-3
        return SimpleNamespace(sample=eps + 0.5 * encoder_hidden_states.mean(dim=(1, 2))[:, None, None, None])


# (name, frames, batch_size, per-frame cond, controlnet, depth)
CASES = [
    ("even", 8, 2, False, False, False),
    ("ragged", 11, 4, False, False, False),
    ("one_batch", 3, 4, False, False, False),        # world 2 > 1 batch: rank 1 runs nothing
    ("cond", 7, 2, True, False, False),
    ("control", 6, 2, True, True, False),
    ("depth", 5, 2, True, False, True),
]
STEPS, GEN_STEPS = 6, 3


def _case(name, frames, batch_size, per_frame, control, depth, shard):
    from vidtome_b200.driver import ChunkedInverter
    unet, controlnet = _tiny(depth=depth)
    g = torch.Generator().manual_seed(frames * 10 + batch_size)
    x = torch.randn(frames, 4, 4, 4, generator=g)
    cond = torch.randn(frames if per_frame else 1, 77, 768, generator=g)
    images = torch.rand(frames, 3, 8, 8, generator=g)
    maps = torch.rand(frames, 1, 4, 4, generator=g) * 2 - 1
    inv = ChunkedInverter(unet, n_timesteps=STEPS, batch_size=batch_size, cond=cond,
                          controlnet=controlnet if control else None, control_images=images if control else None,
                          control_scale=0.7, depth=maps if depth else None, shard=shard)
    final = inv.invert(x)
    assert torch.equal(final, inv.trajectory[-1])
    return inv, {"traj": inv.trajectory, "recon": inv.reconstruct()}


def _generate(source, frames, shard):
    """Sharded PnP generation (chunks i % world == rank) from a trajectory's source_latents."""
    from vidtome_b200.driver import ChunkedDenoiser
    g = torch.Generator().manual_seed(77)
    cond3, x = torch.randn(3, 77, 16, generator=g), torch.randn(frames, 4, 4, 4, generator=g)
    den = ChunkedDenoiser(StandInUNet(), n_timesteps=STEPS, chunk_size=4, cond=cond3, source_latents=source,
                          pnp_modules=[], shard=shard)
    for i in range(GEN_STEPS):
        x = den.step(x, i)
    return x


def _refuse(*a, **k):
    raise AssertionError("a collective after the inversion's gather")


def _worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        for case in CASES:
            inv, out = _case(*case, shard=True)
            torch.save(out, os.path.join(out_dir, f"{case[0]}_{rank}.pt"))
            if case[0] == "ragged":
                # the gathered trajectory feeds sharded generation on every rank with no further collective
                saved = {k: getattr(dist, k) for k in ("all_gather", "all_gather_into_tensor", "all_gather_object",
                                                      "all_reduce", "broadcast", "barrier")}
                for k in saved:
                    setattr(dist, k, _refuse)
                try:
                    gen = _generate(inv.source_latents(), case[1], shard=True)
                finally:
                    for k, f in saved.items():
                        setattr(dist, k, f)
                torch.save(gen, os.path.join(out_dir, f"gen_{rank}.pt"))
    finally:
        dist.destroy_process_group()


def test_two_rank_gloo_is_bit_identical_to_one_process(tmp_path):
    threads = torch.get_num_threads()
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    torch.set_num_threads(1)
    try:
        for case in CASES:
            inv, want = _case(*case, shard=False)
            for rank in range(2):
                got = torch.load(tmp_path / f"{case[0]}_{rank}.pt")
                for k in ("traj", "recon"):
                    assert got[k].shape == want[k].shape, (case[0], rank, k)
                    assert torch.equal(got[k], want[k]), (case[0], rank, k)
            if case[0] == "ragged":
                gen = _generate(inv.source_latents(), case[1], shard=False)
                for rank, frames in ((0, list(range(0, 4)) + list(range(8, 11))), (1, list(range(4, 8)))):
                    got = torch.load(tmp_path / f"gen_{rank}.pt")
                    assert torch.equal(got[frames], gen[frames]), rank       # the rank's chunks
    finally:
        torch.set_num_threads(threads)


def test_gather_batches_single_process_is_identity():
    from vidtome_b200 import dist as vd
    t = torch.randn(3, 5, 2)
    assert vd.gather_batches(t, 5, 2, frame_dim=1) is t
