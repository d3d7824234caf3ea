"""Sharded DDIM inversion and reconstruction (driver.ChunkedInverter(shard=True)): steps per second of invert() and
reconstruct(), and the time of the one all-gather that ends each, against the unsharded inverter in the same process.

    python tools/inversion_shard_bench.py                                    # one GPU: world 1
    torchrun --nproc-per-node N tools/inversion_shard_bench.py --gpus N      # N GPUs, NCCL

Workload: the full-block skeleton (SD1.5 by default) patched and run unmerged through the library, --frames frames of
64 x 64 latents (512² video), batch_size 8, 50 steps, every timestep kept, one CUDA graph per step after 2 eager steps
(--eager: no graph).  Two arms alternate over --rounds rounds after a warm-up round: `unsharded` (shard=False, every
batch on this GPU: the path without sharding) and `sharded` (shard=True: this rank's batches, then the gather).  Every
time comes from CUDA events between barriers, the maximum over ranks of the median over rounds.  The gather is also
timed alone on the trajectory's local slab (--iters calls).  The run checks that both arms give bit-identical
trajectories and reconstructions.  Rank 0 prints one JSON line, with the card name and power limit read in the same run.

On one GPU the sharded arm runs every batch, so it measures what sharding costs when it cannot help; the speed-up over
N GPUs needs N GPUs.
"""
from __future__ import annotations

import argparse
import json
import os
import socket
import statistics
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.global_graph_bench import card  # noqa: E402


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _init(gpus: int):
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world != gpus:
        raise SystemExit(f"--gpus {gpus} needs {gpus} processes (torchrun --nproc-per-node {gpus}); got {world}")
    local = int(os.environ.get("LOCAL_RANK", "0"))
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    if "RANK" not in os.environ:                     # one process: a world-1 group, so that shard=True can run
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(_free_port()), RANK="0", WORLD_SIZE="1")
    dist.init_process_group("nccl", device_id=dev)
    return dev


def _max_over_ranks(v: float) -> float:
    t = torch.tensor([v], dtype=torch.float64, device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def _timed(fn):
    dist.barrier()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    out = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e), out


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--model", default="sd15")
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--size", type=int, default=64, help="latent side (64 = 512x512 video)")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--eager", action="store_true", help="no CUDA graphs")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("inversion_shard_bench needs a CUDA device")
    _init(args.gpus)
    import vidtome_b200
    from vidtome_b200 import dist as vd
    from vidtome_b200.driver import ChunkedInverter
    from vidtome_b200.skeleton import make_skeleton
    cad = 1024 if args.model == "sd21" else 768
    g = torch.Generator(device="cuda").manual_seed(1)                  # the same inputs on every rank
    x = torch.randn(args.frames, 4, args.size, args.size, generator=g, device="cuda").half()
    cond = torch.randn(args.frames, 77, cad, generator=g, device="cuda").half()
    torch.manual_seed(0)
    net = make_skeleton(args.model, hot_path_only=False, device="cuda")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, batch_size=2)
    kw = dict(n_timesteps=args.steps, batch_size=args.batch, cond=cond, cuda_graph=not args.eager, graph_warmup=2)
    arms = {"unsharded": ChunkedInverter(net, **kw), "sharded": ChunkedInverter(net, shard=True, **kw)}
    times = {k: {"invert": [], "reconstruct": []} for k in arms}
    outs = {}
    for r in range(args.rounds + 1):                 # round 0 warms up both arms
        for k, inv in arms.items():
            ms_inv, _ = _timed(lambda: inv.invert(x))
            ms_rec, rec = _timed(lambda: inv.reconstruct())
            if r:
                times[k]["invert"].append(ms_inv)
                times[k]["reconstruct"].append(ms_rec)
            outs[k] = (inv.trajectory, rec)
    same = {"trajectory": bool(torch.equal(outs["sharded"][0], outs["unsharded"][0])),
            "reconstruction": bool(torch.equal(outs["sharded"][1], outs["unsharded"][1]))}
    # the gather alone, on a slab shaped like this rank's part of the trajectory
    mine = sum(hi - lo for lo, hi in vd.shard_batches(args.frames, args.batch))
    local = arms["sharded"].trajectory[:, :mine].contiguous()
    vd.gather_batches(local, args.frames, args.batch, 1)
    ms_gather, _ = _timed(lambda: [vd.gather_batches(local, args.frames, args.batch, 1) for _ in range(args.iters)])
    res = {}
    for k, tt in times.items():
        ms = {p: _max_over_ranks(statistics.median(v)) for p, v in tt.items()}
        res[k] = {"invert_ms": round(ms["invert"], 1), "reconstruct_ms": round(ms["reconstruct"], 1),
                  "invert_steps_per_s": round(args.steps / ms["invert"] * 1e3, 2),
                  "reconstruct_steps_per_s": round(args.steps / ms["reconstruct"] * 1e3, 2)}
    gather_ms = _max_over_ranks(ms_gather / args.iters)
    if dist.get_rank() == 0:
        name, power = card()
        print(json.dumps({"card": name, "power_limit": power, "world": dist.get_world_size(), "model": args.model,
                          "frames": args.frames, "latent": args.size, "batch_size": args.batch, "steps": args.steps,
                          "graph": not args.eager, "rounds": args.rounds, "arms": res,
                          "gather_ms": round(gather_ms, 3),
                          "gather_local_bytes": local.numel() * local.element_size(),
                          "sharded_equals_unsharded": same}))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
