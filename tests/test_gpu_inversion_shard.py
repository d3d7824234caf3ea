"""Reconstruction and sharded inversion on the GPU: ChunkedInverter.reconstruct() through KI against the torch
restatement of the sampling step on CUDA fp16, from CUDA graphs against eager stepping (with and without a ControlNet),
and two gloo ranks sharing the one GPU whose trajectory and reconstruction, eager and from graphs, are bit-identical to
the unsharded run's: wholly when every attention runs in the library (attention.MAX_HEAD_DIM = 160), and in each rank's
own frames at the default limit, where torch's SDPA computes the other rank's.  The ranks are spawned processes, joined
with a timeout.  Needs an H100 (sm_90a)."""
import os
import socket
import time

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

FRAMES, SIZE, STEPS = 11, 16, 20


def _inputs(frames=FRAMES, size=SIZE, seed=13):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(frames, 4, size, size, generator=g, device="cuda").half()
    cond = torch.randn(frames, 77, 768, generator=g, device="cuda").half()
    images = torch.rand(frames, 3, 8 * size, 8 * size, generator=g, device="cuda").half()
    return x, cond, images


def _models(control):
    import vidtome_b200
    from vidtome_b200.skeleton import make_controlnet, make_skeleton
    net = make_skeleton("sd15", hot_path_only=False, device="cuda")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, batch_size=2)
    controlnet = None
    if control:
        controlnet = make_controlnet("sd15", hot_path_only=False, device="cuda")
        vidtome_b200.apply_patch(controlnet, local_merge_ratio=0.9, batch_size=2)
    return net, controlnet


def _kw(cond, images, controlnet, batch_size=4):
    return dict(n_timesteps=STEPS, batch_size=batch_size, cond=cond, controlnet=controlnet,
                control_images=images if controlnet is not None else None, control_scale=0.8)


def _diff(a, b):
    return (a.float() - b.float()).abs().max().item()


def test_reconstruct_kernel_is_bit_identical_to_the_torch_restatement():
    """KI with the sampling table gives, step by step, what sample_next_x gives on the same noise predictions."""
    from vidtome_b200 import patch
    from vidtome_b200.driver import ChunkedInverter
    x, cond, _ = _inputs()
    net, _ = _models(False)
    inv = ChunkedInverter(net, n_timesteps=STEPS, batch_size=4, cond=cond)
    got = inv.reconstruct(x)
    want = x.clone()
    with torch.no_grad(), patch._unmerged_blocks(), torch.autocast("cuda", dtype=torch.float16):
        for i, t in enumerate(inv.sample_timesteps):
            eps = torch.empty_like(want)                                # the UNet's output, stored as the latents
            for lo in range(0, FRAMES, 4):
                eps[lo:lo + 4] = inv.pred_noise(want[lo:lo + 4], cond[lo:lo + 4], t)
            want = inv.sample_next_x(want, eps, i)
    assert torch.isfinite(got).all() and got.dtype == torch.float16
    assert torch.equal(got, want), f"max |diff| {_diff(got, want)}"
    assert not torch.equal(got, x)


@pytest.mark.parametrize("control", [False, True])
def test_reconstruct_graph_is_bit_identical_to_eager(control):
    from vidtome_b200.driver import ChunkedInverter
    x, cond, images = _inputs()
    net, controlnet = _models(control)
    kw = _kw(cond, images, controlnet)
    eager = ChunkedInverter(net, **kw)
    graph = ChunkedInverter(net, cuda_graph=True, graph_warmup=2, **kw)
    eager.invert(x)
    graph.invert(x)
    assert torch.equal(eager.trajectory, graph.trajectory)
    a, b = eager.reconstruct(), graph.reconstruct()
    assert torch.isfinite(a).all()
    assert torch.equal(a, b), f"max |diff| {_diff(a, b)}"
    assert torch.equal(graph.reconstruct(x), eager.reconstruct(x))     # an explicit input, which stays as it was
    assert torch.equal(x, _inputs()[0])


# --------------------------------------------------------------------------- two gloo ranks on one GPU
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _stage_through_host(real):
    def staged(out, inp, group=None, async_op=False):
        host = torch.empty(out.shape, dtype=out.dtype)
        real(host, inp.cpu(), group=group)
        out.copy_(host)
    return staged


def _worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from vidtome_b200 import attention, dist as vd
        from vidtome_b200.driver import ChunkedInverter
        staged = False
        try:                                            # gloo's all-gather of CUDA tensors
            probe = torch.full((2,), float(rank), device="cuda")
            got = torch.empty(2 * world, device="cuda")
            dist.all_gather_into_tensor(got, probe)
            assert got.tolist() == [float(r) for r in range(world) for _ in range(2)]
        except RuntimeError:
            dist.all_gather_into_tensor = _stage_through_host(dist.all_gather_into_tensor)
            staged = True
        results = {"staged": staged}
        x, cond, images = _inputs()
        # batch_size 4 over 11 frames: 3 batches, the last one ragged; rank 0 runs batches 0 and 2, rank 1 batch 1
        mine = [f for lo, hi in vd.shard_batches(FRAMES, 4) for f in range(lo, hi)]
        for head_dim in (160, 128):
            # 160: every attention of SD1.5 runs in the library, which computes a batch the same way in every process;
            # 128 (the default): the 1280-channel blocks run torch's SDPA, whose result may differ between processes
            # in the last bits (DESIGN §7), so only this rank's own frames are held to bit identity
            attention.MAX_HEAD_DIM = head_dim
            for control in (False, True):
                net, controlnet = _models(control)
                kw = _kw(cond, images, controlnet)
                for graph in (False, True):
                    gkw = dict(cuda_graph=graph, graph_warmup=2)
                    one = ChunkedInverter(net, **kw, **gkw)
                    one.invert(x)
                    want = one.reconstruct()
                    sh = ChunkedInverter(net, shard=True, **kw, **gkw)
                    final = sh.invert(x)
                    got = sh.reconstruct()
                    assert torch.equal(final, sh.trajectory[-1])
                    key = f"head_dim{head_dim}_control{int(control)}_graph{int(graph)}"
                    results[key] = {"own_traj": torch.equal(sh.trajectory[:, mine], one.trajectory[:, mine]),
                                    "own_recon": torch.equal(got[mine], want[mine]),
                                    "traj": torch.equal(sh.trajectory, one.trajectory),
                                    "recon": torch.equal(got, want), "finite": bool(torch.isfinite(got).all()),
                                    "traj_diff": _diff(sh.trajectory, one.trajectory), "recon_diff": _diff(got, want),
                                    "traj_max": one.trajectory.float().abs().max().item(),
                                    "recon_max": want.float().abs().max().item()}
        # more ranks than batches: 3 frames in one batch, rank 1 runs nothing and still joins the gathers
        attention.MAX_HEAD_DIM = 160
        net, _ = _models(False)
        kw = _kw(cond[:3], None, None)
        one = ChunkedInverter(net, **kw)
        one.invert(x[:3])
        sh = ChunkedInverter(net, shard=True, cuda_graph=True, **kw)
        sh.invert(x[:3])
        results["one_batch"] = {"traj": torch.equal(sh.trajectory, one.trajectory),
                                "recon": torch.equal(sh.reconstruct(), one.reconstruct())}
        torch.save(results, os.path.join(out_dir, f"rank{rank}.pt"))
    finally:
        dist.destroy_process_group()


def test_two_gloo_ranks_are_bit_identical_to_one_rank(tmp_path):
    ctx = mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=False,
                             start_method="spawn")
    deadline = time.monotonic() + 900
    try:
        while not ctx.join(timeout=5):
            if time.monotonic() > deadline:
                raise TimeoutError("the two ranks did not finish within 900 s")
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.kill()
            p.join()
    for rank in range(2):
        res = torch.load(tmp_path / f"rank{rank}.pt")
        print(f"rank {rank}: all-gather staged through host memory: {res.pop('staged')}")
        for key, r in res.items():
            print(rank, key, r)
            if key.startswith("head_dim128"):
                # the other rank's frames of the trajectory within fp16 noise; the reconstruction of those frames starts
                # from latents that differ already, so only its own frames are compared
                assert r["own_traj"] and r["own_recon"] and r["finite"], (rank, key, r)
                assert r["traj_diff"] <= 2e-2 * r["traj_max"] + 2e-2, (rank, key, r)
            else:
                assert all(v for k, v in r.items() if isinstance(v, bool)), (rank, key, r)
