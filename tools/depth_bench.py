"""SD2-depth (ChunkedDenoiser(depth=...), ChunkedInverter(depth=...)): step rates eager against CUDA graphs on the
workload of the reference's configs/flamingo.yaml.

Model: the SD2.1-census depth skeleton (make_skeleton("sd21", depth=True): 5 input channels, 4 out), full blocks
(cross-attention over a 1024-wide text context and the GEGLU feed-forward), linear Transformer2DModel IO, CUDA fp16,
patched with local merging 0.9 and global merging 0.9 (global_rand 0.5).  --frames frames of 512x512 video (64 x 64
latents), one depth map per frame.

Generation: chunk_size 4 with the reference's randomised chunks (random first chunk, reversed half the time),
merge_global, chunk_ord "rand", classifier-free guidance (B = 2).  Two denoisers on two identical skeletons, eager and
chunk_graphs=True, first step the same seeded latents with the same host draws --check-steps times and their latents
are compared bit for bit; then --rounds timed rounds alternate them, --steps steps each.
Inversion: --frames frames in batches of 8, 50 steps, eager (KI update) against cuda_graph=True; the trajectories are
compared bit for bit, then --rounds timed rounds alternate the two.
Input assembly: the depth maps' share of a step, timed alone: `cat([x | x], depth.repeat(2))` on dim 1 at one chunk's
shape, times the chunks of a step.

Every time comes from CUDA events; medians over rounds are reported.  One JSON line goes to stdout, with the card name
and power limit read in the same run.

    python tools/depth_bench.py --steps 20 --rounds 3
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.global_graph_bench import card  # noqa: E402

CHUNK = 4
N_TIMESTEPS = 50


def _model():
    import vidtome_b200
    from vidtome_b200.skeleton import make_skeleton
    torch.manual_seed(123)
    net = make_skeleton("sd21", hot_path_only=False, transformer_io="linear", depth=True, device="cuda")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=True, global_merge_ratio=0.9, global_rand=0.5,
                             batch_size=2)
    return net


def _inputs(frames: int, size: int):
    g = torch.Generator(device="cuda").manual_seed(5)
    cond = torch.randn((2, 77, 1024), generator=g, device="cuda", dtype=torch.float16)
    depth = torch.rand((frames, 1, size, size), generator=g, device="cuda") * 2 - 1
    x = torch.randn((frames, 4, size, size), generator=g, device="cuda", dtype=torch.float16)
    return cond, depth, x


def _timed(fn) -> float:
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


@torch.no_grad()
def generation(frames: int, size: int, steps: int, rounds: int, check_steps: int) -> dict:
    from vidtome_b200.driver import ChunkedDenoiser
    cond, depth, x0 = _inputs(frames, size)
    arms = {}
    for name, kw in (("eager", {}), ("chunk_graphs", {"cuda_graph": True, "chunk_graphs": True})):
        arms[name] = ChunkedDenoiser(_model(), n_timesteps=N_TIMESTEPS, chunk_size=CHUNK, merge_global=True,
                                     chunk_ord="rand", randomize_chunks=True, cond=cond, depth=depth, graph_warmup=2,
                                     **kw)
    state, finals = {}, {}
    for name, den in arms.items():
        torch.manual_seed(2024)              # the device RNG the blocks fork from
        np.random.seed(2024)                 # the host draws of get_chunks
        x = x0.clone()
        for i in range(check_steps):
            x = den.step(x, i)
        torch.cuda.synchronize()
        state[name], finals[name] = [x, check_steps], x
    same = bool(torch.equal(finals["eager"], finals["chunk_graphs"]))
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for name, den in arms.items():
            st = state[name]

            def run():
                for _ in range(steps):
                    st[0] = den.step(st[0], st[1] % N_TIMESTEPS)
                    st[1] += 1
            times[name].append(_timed(run) / steps)
    ms = {k: statistics.median(v) for k, v in times.items()}
    return {"frames": frames, "latent": size, "chunk_size": CHUNK, "steps_timed": steps, "rounds": rounds,
            "ms_per_step": {k: round(v, 2) for k, v in ms.items()},
            "steps_per_s": {k: round(1000.0 / v, 3) for k, v in ms.items()},
            "graph_speedup": round(ms["eager"] / ms["chunk_graphs"], 3),
            "chunk_graphs_captured": len(arms["chunk_graphs"]._chunk_graphs),
            "graph_equals_eager_after_check_steps": same, "check_steps": check_steps}


@torch.no_grad()
def inversion(frames: int, size: int, batch: int, rounds: int) -> dict:
    from vidtome_b200.driver import ChunkedInverter
    net = _model()
    _, depth, x = _inputs(frames, size)
    g = torch.Generator(device="cuda").manual_seed(7)
    cond = torch.randn((frames, 77, 1024), generator=g, device="cuda", dtype=torch.float16)
    kw = dict(n_timesteps=N_TIMESTEPS, batch_size=batch, cond=cond, depth=depth)
    arms = {"eager": ChunkedInverter(net, **kw), "graph": ChunkedInverter(net, cuda_graph=True, graph_warmup=2, **kw)}
    times = {k: [] for k in arms}
    for r in range(rounds + 1):                      # round 0 warms up both arms
        for name, inv in arms.items():
            ms = _timed(lambda: inv.invert(x))
            if r:
                times[name].append(ms / N_TIMESTEPS)
    same = bool(torch.equal(arms["eager"].trajectory, arms["graph"].trajectory))
    ms = {k: statistics.median(v) for k, v in times.items()}
    return {"frames": frames, "latent": size, "batch_size": batch, "steps": N_TIMESTEPS, "rounds": rounds,
            "ms_per_step": {k: round(v, 2) for k, v in ms.items()},
            "steps_per_s": {k: round(1000.0 / v, 3) for k, v in ms.items()},
            "graph_speedup": round(ms["eager"] / ms["graph"], 3), "graph_equals_eager": same}


@torch.no_grad()
def input_assembly(frames: int, size: int, iters: int, rounds: int) -> dict:
    """The concatenation ChunkedDenoiser.pred_noise adds for depth, at one chunk's shape (generate.py:256-262)."""
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn((CHUNK, 4, size, size), generator=g, device="cuda", dtype=torch.float16)
    depth = torch.rand((CHUNK, 1, size, size), generator=g, device="cuda").half()
    lmi = torch.cat([x, x])

    def run():
        for _ in range(iters):
            torch.cat([lmi, depth.repeat(2, 1, 1, 1).to(x)], dim=1)
    run()
    per_call = statistics.median(_timed(run) / iters for _ in range(rounds))
    chunks = -(-frames // CHUNK)
    return {"ms_per_call": round(per_call, 4), "chunks_per_step": chunks,
            "ms_per_step": round(per_call * chunks, 3)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--size", type=int, default=64, help="latent side (64 = 512x512 video)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--check-steps", type=int, default=6)
    ap.add_argument("--inv-batch", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("depth_bench needs a CUDA device")
    name, power = card()
    gen = generation(args.frames, args.size, args.steps, args.rounds, args.check_steps)
    asm = input_assembly(args.frames, args.size, 200, args.rounds)
    asm["share_of_eager_step"] = round(asm["ms_per_step"] / gen["ms_per_step"]["eager"], 4)
    res = {"card": name, "power_limit": power, "generation": gen, "input_assembly": asm,
           "inversion": inversion(args.frames, args.size, args.inv_batch, args.rounds)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
