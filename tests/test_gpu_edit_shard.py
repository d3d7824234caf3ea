"""Edits of a multi-prompt generation split over the ranks, on the GPU: two gloo ranks sharing the one H100 run
ChunkedDenoiser(cond=[K, S, 77, D], shard=True) for K in (2, 3) (with K = 3 rank 0 runs edits 0 and 2, rank 1 edit 1
alone): eagerly with global merging and randomised chunks, from the lane-captured step of cuda_graph=True, with
capture_global=True and with chunk_graphs=True; with PnP across both injection boundaries, a patched ControlNet and
depth.  The models and inputs are tests/test_gpu_multi_edit.py's, whose skeleton Linears run once per edit's slice there
and here, so every operator gives a row the same bits whatever the number of edits in the batch.

Every rank also runs the unsharded K-edit run itself.  Each edit of the result sample() gathers on a rank must be, bit
for bit, that edit of the unsharded run made in the process of the rank that computed it.  The reference is taken per
process because the unsharded run itself is not bit-identical between two processes on the same GPU: with merging, one
edit of a run can differ in the last bits of some elements (7.8e-3 in latents of magnitude about 4 on an H100), while
repeated runs in one process are bit-identical.  The cause is not identified; the test prints, per case, whether the
two ranks' unsharded runs agree.

With the skeleton's Linears on the whole batch (the model users run) a rank's batch of K_r edits is not the unsharded
run's K: each step of a rank's edits, from the unsharded run's inputs, is held to the level test_gpu_multi_edit.py holds
a K-edit step to against single runs.  One NCCL world of one rank runs the sharded path with a real NCCL group.  The
ranks are spawned processes, joined with a timeout.  Needs an H100 (sm_90a)."""
import os
import socket
import time

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_gpu_multi_edit import MODES, STEPS, _inputs, _model, _source

pytestmark = pytest.mark.gpu

# name -> (K, mode of test_gpu_multi_edit.MODES, feature, hot_path_only)
CASES = {f"{mode}_{K}": (K, mode, None, True) for K in (2, 3)
         for mode in ("eager_random", "step_graph", "capture_global", "chunk_graphs")}
CASES.update({
    "pnp_capture_global_2": (2, "capture_global", "pnp", True),
    "pnp_chunk_graphs_3": (3, "chunk_graphs", "pnp", True),
    "pnp_step_graph_3": (3, "step_graph", "pnp", True),
    "controlnet_capture_global_2": (2, "capture_global", "controlnet_patched", True),
    "controlnet_chunk_graphs_3": (3, "chunk_graphs", "controlnet_patched", True),
    "depth_eager_random_3": (3, "eager_random", "depth", False),
    "depth_chunk_graphs_2": (2, "chunk_graphs", "depth", False),
})
# the unmodified model, with the float64 case whose level applies (test_gpu_multi_edit.UNMODIFIED["local_full_blocks"])
LEVEL_CASE, LEVEL_K, LEVEL_MODE, LEVEL_FLOAT64 = "unmodified_step_graph_3", 3, "step_graph", "local"


def _run(K, mode, feature, hot_path_only, shard, per_edit_linears=True, inputs=None):
    """sample() of all K edits, or with `inputs` (the unsharded run's input latents of every step) the output of every
    step taken from them: [K, ...] per step unsharded, the rank's [K_r, ...] sharded."""
    from vidtome_b200 import dist as vd
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import pnp_attention_modules, pnp_conv_module
    graph, merge_global, randomize, capture_global, chunk_graphs = MODES[mode]
    rows = vd.shard_edits(K) if shard else list(range(K))
    pnp = feature == "pnp"
    unet, controlnet = _model(len(rows), merge_global, feature, hot_path_only, per_edit_linears)
    cond, x, per_frame = _inputs(K, 3 if pnp else 2, feature == "depth", controlnet is not None)
    kw = dict(cuda_graph=graph, graph_warmup=1, randomize_chunks=randomize, capture_global=capture_global,
              chunk_graphs=chunk_graphs)
    if pnp:
        kw.update(source_latents=_source, pnp_attn_t=0.25, pnp_modules=pnp_attention_modules(unet), pnp_f_t=0.5,
                  pnp_conv_modules=[pnp_conv_module(unet)])
    if controlnet is not None:
        kw.update(controlnet=controlnet)
    den = ChunkedDenoiser(unet, n_timesteps=STEPS, chunk_size=4, merge_global=merge_global, chunk_ord="mix-4",
                          cond=cond, shard=shard, **kw, **per_frame)
    torch.manual_seed(2024)
    np.random.seed(2024)
    if inputs is None:
        out = den.sample(x)
    else:
        ins, out = [], []
        for i in range(STEPS):
            x = x if inputs is True else inputs[i][rows]
            ins.append(x.clone())
            x = den.step(x, i)
            out.append(x.clone())
        out = (ins, out)
    torch.cuda.synchronize()
    den.close()
    return out


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


def _worker(rank, world, port, out_dir, backend):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(0)
    if backend == "nccl":
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", 0))
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from vidtome_b200 import dist as vd
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
        names = ["capture_global_2"] if backend == "nccl" else list(CASES)
        for name in names:
            results[name] = {"unsharded": _run(*CASES[name], shard=False).cpu(),
                             "sharded": _run(*CASES[name], shard=True).cpu()}
        if backend == "gloo":
            ins, want = _run(LEVEL_K, LEVEL_MODE, None, False, False, per_edit_linears=False, inputs=True)
            got = _run(LEVEL_K, LEVEL_MODE, None, False, True, per_edit_linears=False, inputs=ins)[1]
            rows = vd.shard_edits(LEVEL_K)
            results[LEVEL_CASE] = [((a.float() - b[rows].float()).abs().max() / b[rows].float().abs().max()).item()
                                   for a, b in zip(got, want)]
        torch.save(results, os.path.join(out_dir, f"{backend}{rank}.pt"))
    finally:
        dist.destroy_process_group()


def _spawn(world, out_dir, backend):
    ctx = mp.start_processes(_worker, args=(world, _free_port(), out_dir, backend), nprocs=world, join=False,
                             start_method="spawn")
    deadline = time.monotonic() + 900
    try:
        while not ctx.join(timeout=5):
            if time.monotonic() > deadline:
                raise TimeoutError(f"the {world} rank(s) did not finish within 900 s")
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.kill()
            p.join()


def test_sharded_edits_are_the_unsharded_run(tmp_path):
    """Every edit of the result each rank gathers is, bit for bit, the unsharded run's edit computed in the process of
    the rank that ran it (see the module's doc for why not across processes); the level case within its level."""
    from test_gpu_step_float64 import CASES as FLOAT64
    from vidtome_b200 import dist as vd
    _spawn(2, str(tmp_path), "gloo")
    _spawn(1, str(tmp_path), "nccl")
    c = FLOAT64[LEVEL_FLOAT64]
    level = 2 * (c.x_level if c.x_level is not None else c.level)
    bad = []
    for backend, world in (("gloo", 2), ("nccl", 1)):
        res = [torch.load(tmp_path / f"{backend}{rank}.pt") for rank in range(world)]
        for rank, r in enumerate(res):
            print(f"{backend} rank {rank}: all-gather staged through host memory: {r.pop('staged')}")
            for step, rel in enumerate(r.pop(LEVEL_CASE, [])):
                print(f"{LEVEL_CASE} rank {rank} step {step}: max |diff| relative to max |x| = {rel:.2e} "
                      f"(level {level})")
                if not rel <= level:
                    bad.append((backend, rank, LEVEL_CASE, step, rel))
        for name in res[0]:
            K = CASES[name][0]
            want = [r[name]["unsharded"] for r in res]
            assert all(w.shape[0] == K and torch.isfinite(w).all() for w in want), name
            assert not torch.equal(want[0][0], want[0][1]), name            # the edits are distinct runs
            if world > 1:
                print(f"{name}: the unsharded runs of the two processes bit-identical: {torch.equal(*want)}")
            for rank, r in enumerate(res):
                got = r[name]["sharded"]
                for owner in range(world):
                    rows = vd.shard_edits(K, owner, world)
                    same = got.shape == want[owner].shape and torch.equal(got[rows], want[owner][rows])
                    print(f"{backend} rank {rank} {name}: edits {rows} bit-identical to rank {owner}'s unsharded "
                          f"run: {same}")
                    if not same:
                        bad.append((backend, rank, name, owner))
    assert not bad, bad
