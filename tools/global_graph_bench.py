"""Step rate of chunked sampling with global token merging, eager vs CUDA-graph stepping (BASELINE config 3).

Workload: the SD1.5 skeleton at 512x512 (latent 64), 32 frames in chunks of 4 visited in "mix-4" order, local merging
0.9 + global merging 0.8 with global_rand 0.5, classifier-free guidance (B = 2).  "hot" runs the merge + self-attention
path only (as bench.py's hot workload); "full" adds cross-attention over a [2, 77, 768] text context and the
feed-forward.

The eager and the graph denoiser drive two identical skeletons.  Both first step the same seeded latents
--check-steps times, and the final latents are compared bit for bit.  Then --rounds timed rounds alternate eager and
graph, --steps steps each, timed with CUDA events.  One JSON line goes to stdout, with the card name and power limit
read in the same run.

--profile DIR instead runs torch.profiler over a few steps of each and writes the per-kernel tables to DIR: where a
step's time goes (device-busy time against wall time per step).

    python tools/global_graph_bench.py --workload hot --steps 20 --rounds 3
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FRAMES, CHUNK, LATENT = 32, 4, 64


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[0].split(",")]
        return name, power
    except Exception as e:                      # report, do not guess
        return torch.cuda.get_device_name(), f"unknown ({type(e).__name__})"


def make(kind: str, graph: bool):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton
    torch.manual_seed(123)
    net = make_skeleton("sd15", hot_path_only=(kind == "hot"), device="cuda")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=True, global_merge_ratio=0.8, global_rand=0.5,
                             batch_size=2)
    cond = None
    if kind != "hot":
        gc = torch.Generator(device="cuda").manual_seed(5)
        cond = torch.randn((2, 77, 768), generator=gc, device="cuda", dtype=torch.float16)
    return ChunkedDenoiser(net, n_timesteps=50, chunk_size=CHUNK, merge_global=True, chunk_ord="mix-4", cond=cond,
                           cuda_graph=graph, capture_global=graph, graph_warmup=2)


class Chain:
    """One denoiser stepping its own latents; step i of the chain uses DDIM step i % 50."""

    def __init__(self, den, x0):
        self.den, self.x, self.i = den, x0.clone(), 0

    def step(self):
        self.x = self.den.step(self.x, self.i % 50)
        self.i += 1


def timed(chain: Chain, steps: int) -> float:
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        chain.step()
    e.record()
    torch.cuda.synchronize()
    return steps / (s.elapsed_time(e) / 1e3)


def profile(chains, steps: int, out_dir: str):
    from torch.profiler import ProfilerActivity, profile as tprof
    os.makedirs(out_dir, exist_ok=True)
    res = {}
    for name, ch in chains.items():
        torch.cuda.synchronize()
        with tprof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(steps):
                ch.step()
            e.record()
            torch.cuda.synchronize()
        wall = s.elapsed_time(e) / steps
        ka = p.key_averages()
        busy_us = sum(k.self_device_time_total for k in ka if k.device_type.name == "CUDA") / steps
        top = sorted((k for k in ka if k.self_device_time_total > 0), key=lambda k: -k.self_device_time_total)[:15]
        with open(os.path.join(out_dir, f"{name}_kernels.txt"), "w") as f:
            f.write(ka.table(sort_by="self_cuda_time_total", row_limit=40))
        res[name] = {"ms_per_step_profiled": round(wall, 3), "device_busy_ms_per_step": round(busy_us / 1e3, 3),
                     "busy_frac": round(busy_us / 1e3 / wall, 3),
                     "top": [(k.key[:60], round(k.self_device_time_total / steps / 1e3, 3), k.count // steps)
                             for k in top]}
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", choices=("hot", "full"), default="hot")
    ap.add_argument("--steps", type=int, default=20, help="timed steps per round and mode")
    ap.add_argument("--rounds", type=int, default=3, help="alternating eager / graph rounds")
    ap.add_argument("--check-steps", type=int, default=6, help="steps compared bit for bit (2 eager + capture + replays)")
    ap.add_argument("--warmup", type=int, default=3, help="untimed steps of each chain after the check")
    ap.add_argument("--profile", metavar="DIR", default=None, help="profile a few steps of each mode instead of timing")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("global_graph_bench.py needs a CUDA device")
    name, power = card()

    g = torch.Generator(device="cuda").manual_seed(123)
    x0 = torch.randn((FRAMES, 4, LATENT, LATENT), generator=g, device="cuda", dtype=torch.float16)
    chains = {}
    for mode in ("eager", "graph"):
        chains[mode] = Chain(make(args.workload, mode == "graph"), x0)
        torch.manual_seed(2024)           # the same host (chunk order) and device (block generators) draws
        for _ in range(args.check_steps):
            chains[mode].step()
    torch.cuda.synchronize()
    identical = torch.equal(chains["eager"].x, chains["graph"].x)
    finite = bool(torch.isfinite(chains["graph"].x).all())
    for ch in chains.values():
        for _ in range(args.warmup):
            ch.step()

    line = {"tool": "global_graph_bench", "workload": args.workload, "card": name, "power_limit": power,
            "frames": FRAMES, "chunk_size": CHUNK, "latent": LATENT, "chunk_ord": "mix-4", "local_ratio": 0.9,
            "global_ratio": 0.8, "global_rand": 0.5, "batch": 2, "check_steps": args.check_steps,
            "latents_bit_identical": identical, "finite": finite}
    if args.profile:
        line["profile"] = profile(chains, max(2, min(args.steps, 5)), args.profile)
    else:
        rates = {"eager": [], "graph": []}
        for _ in range(args.rounds):
            for mode in ("eager", "graph"):
                rates[mode].append(round(timed(chains[mode], args.steps), 2))
        line.update({"steps_per_round": args.steps, "rounds": args.rounds,
                     "eager_steps_per_s": rates["eager"], "graph_steps_per_s": rates["graph"],
                     "eager_range": [min(rates["eager"]), max(rates["eager"])],
                     "graph_range": [min(rates["graph"]), max(rates["graph"])],
                     "speedup_median": round(sorted(rates["graph"])[len(rates["graph"]) // 2]
                                             / sorted(rates["eager"])[len(rates["eager"]) // 2], 3)})
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
