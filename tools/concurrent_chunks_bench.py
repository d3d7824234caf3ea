"""Step rate of a captured chunked step with its chunks on one stream against several lanes (driver.LANES).

Workloads, on the SD1.5 skeleton at 512x512 (latent 64), 32 frames:
  c3-hot / c3-full   BASELINE config 3: 4-frame chunks in "mix-4" order, local 0.9 + global 0.8 (global_rand 0.5),
                     capture_global=True; "hot" is the merge + self-attention path only, "full" adds cross-attention
                     over a [2, 77, 768] text context and the feed-forward
  c3-pnp             c3-full with PnP (batch 3: source | uncond | cond), timed inside the attention-injection schedule
                     (pnp_attn_t 0.5 of 50 steps), so that every timed step replays the same graph
  local-4 / local-8  local merging 0.9 only, cuda_graph=True, 4- and 8-frame chunks, full blocks

Every arm (1 lane, and each count of --lanes) drives its own skeleton built from the same seed.  All arms first step
the same seeded latents --check-steps times (eager warm-up, capture, replays); their latents must then be bit-equal.
Then --rounds timed rounds alternate the arms, --steps steps each, timed with CUDA events.  Reported per arm: the
median steps/s with min and max, and the graph's memory pool (bytes reserved by its segments).  One JSON line per
workload goes to stdout, with the card's name, power limit and max SM clock read in the same run.

    python tools/concurrent_chunks_bench.py --workloads c3-hot c3-full --lanes 2 3 4
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

FRAMES, LATENT, N_STEPS = 32, 64, 50
WORKLOADS = ("c3-hot", "c3-full", "c3-pnp", "local-4", "local-8")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [s.strip() for s in out[0].split(",")]
        return name, power, clock
    except Exception as e:                      # report, do not guess
        return torch.cuda.get_device_name(), f"unknown ({type(e).__name__})", "unknown"


def make(workload: str, lanes: int):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton, pnp_attention_modules
    torch.manual_seed(123)
    pnp = workload == "c3-pnp"
    local = workload.startswith("local")
    net = make_skeleton("sd15", hot_path_only=(workload == "c3-hot"), device="cuda")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=not local, global_merge_ratio=0.8,
                             global_rand=0.5, batch_size=3 if pnp else 2, align_batch=pnp)
    gc = torch.Generator(device="cuda").manual_seed(5)
    cond = None
    if workload != "c3-hot":
        cond = torch.randn((3 if pnp else 2, 77, 768), generator=gc, device="cuda", dtype=torch.float16)
    kw = {}
    if pnp:
        sources = {}

        def source(t):
            if t not in sources:
                gs = torch.Generator(device="cuda").manual_seed(int(t))
                sources[t] = torch.randn((FRAMES, 4, LATENT, LATENT), generator=gs, device="cuda").half()
            return sources[t]
        kw.update(source_latents=source, pnp_attn_t=0.5, pnp_modules=pnp_attention_modules(net))
    chunk = int(workload.split("-")[1]) if local else 4
    den = ChunkedDenoiser(net, n_timesteps=N_STEPS, chunk_size=chunk, merge_global=not local, chunk_ord="mix-4",
                          cond=cond, cuda_graph=True, capture_global=not local, graph_warmup=2, **kw)
    den._lane_count = lanes                 # the arm's lane count instead of driver.LANES
    return den


class Chain:
    """One denoiser stepping its own latents over DDIM steps `first`, first + 1, ..., cycling below `end`."""

    def __init__(self, den, x0, first=0, end=N_STEPS):
        self.den, self.x, self.first, self.end, self.n = den, x0.clone(), first, end, 0

    def step(self):
        self.x = self.den.step(self.x, self.first + self.n % (self.end - self.first))
        self.n += 1


def timed(chain: Chain, steps: int) -> float:
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        chain.step()
    e.record()
    torch.cuda.synchronize()
    return steps / (s.elapsed_time(e) / 1e3)


def pool_bytes(graph) -> int:
    """Bytes reserved by the segments of the graph's private memory pool."""
    pool, segs = tuple(graph.pool()), torch.cuda.memory_snapshot()
    if not any("segment_pool_id" in seg for seg in segs):
        return None
    return sum(seg["total_size"] for seg in segs if tuple(seg.get("segment_pool_id", ())) == pool)


def run(workload: str, lanes, rounds: int, steps: int, check_steps: int):
    import numpy as np
    g = torch.Generator(device="cuda").manual_seed(123)
    x0 = torch.randn((FRAMES, 4, LATENT, LATENT), generator=g, device="cuda", dtype=torch.float16)
    end = 25 if workload == "c3-pnp" else N_STEPS      # PnP: inside the injection schedule, one graph key
    arms = {}
    for n in [1] + list(lanes):
        arms[n] = Chain(make(workload, n), x0, end=end)
        torch.manual_seed(2024)
        np.random.seed(2024)
        for _ in range(check_steps):
            arms[n].step()
    torch.cuda.synchronize()
    identical = all(torch.equal(arms[1].x, ch.x) for ch in arms.values())
    rates = {n: [] for n in arms}
    for _ in range(rounds):
        for n, ch in arms.items():
            rates[n].append(round(timed(ch, steps), 2))
    out = {}
    for n, ch in arms.items():
        r = sorted(rates[n])
        out[str(n)] = {"lane_count": ch.den._lane_count,
                       "steps_per_s_median": r[len(r) // 2], "min": r[0], "max": r[-1], "all": rates[n],
                       "pool_MiB": None}
        size = pool_bytes(ch.den._graph.graph)
        if size is not None:
            out[str(n)]["pool_MiB"] = round(size / 2 ** 20, 1)
    base = out["1"]["steps_per_s_median"]
    for n in lanes:
        out[str(n)]["speedup_median"] = round(out[str(n)]["steps_per_s_median"] / base, 3)
    return {"latents_bit_identical": identical, "finite": bool(torch.isfinite(arms[1].x).all()), "arms": out,
            "max_allocated_GiB": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workloads", nargs="+", choices=WORKLOADS, default=list(WORKLOADS))
    ap.add_argument("--lanes", nargs="+", type=int, default=[2, 3, 4], help="lane counts set against one lane")
    ap.add_argument("--steps", type=int, default=20, help="timed steps per round and arm")
    ap.add_argument("--rounds", type=int, default=5, help="rounds alternating the arms")
    ap.add_argument("--check-steps", type=int, default=5, help="steps compared bit for bit (2 eager + capture + replays)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("concurrent_chunks_bench.py needs a CUDA device")
    name, power, clock = card()
    for w in args.workloads:
        torch.cuda.reset_peak_memory_stats()
        line = {"tool": "concurrent_chunks_bench", "workload": w, "card": name, "power_limit": power,
                "max_sm_clock": clock, "frames": FRAMES, "latent": LATENT, "steps_per_round": args.steps,
                "rounds": args.rounds}
        line.update(run(w, args.lanes, args.rounds, args.steps, args.check_steps))
        print(json.dumps(line), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
