"""Step rate of chunked sampling with the reference's randomised chunking, eager vs one CUDA graph per chunk
(ChunkedDenoiser(chunk_graphs=True)), and with fixed chunking, one graph per chunk vs one graph per step
(capture_global=True).

Workload: BASELINE config 3 with the reference's chunking: the SD1.5 skeleton at 512x512 (latent 64), 32 frames,
chunk_size 4 with a random first chunk of 1..4 frames and the chunk list reversed half the time (generate.py:172-203),
"mix-4" order, local merging 0.9 + global merging 0.8 with global_rand 0.5, classifier-free guidance (B = 2).  "hot" runs
the merge + self-attention path only (as bench.py's hot workload); "full" adds cross-attention over a [2, 77, 768] text
context and the feed-forward.

Four denoisers drive four identical skeletons: random chunking eager ("rand_eager") and from chunk graphs
("rand_chunk_graphs"), fixed chunking from chunk graphs ("fixed_chunk_graphs") and from one graph per step
("fixed_step_graph").  Each pair first steps the same seeded latents with the same host draws --check-steps times and
its final latents are compared bit for bit.  Then --rounds timed rounds alternate the four, --steps steps each, timed
with CUDA events.  One JSON line goes to stdout, with the card name and power limit read in the same run.

    python tools/random_chunk_graph_bench.py --workload hot --steps 20 --rounds 3
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.global_graph_bench import CHUNK, FRAMES, LATENT, Chain, card, timed  # noqa: E402

MODES = {                                  # name -> (randomize_chunks, ChunkedDenoiser graph keywords)
    "rand_eager": (True, {}),
    "rand_chunk_graphs": (True, {"cuda_graph": True, "chunk_graphs": True}),
    "fixed_chunk_graphs": (False, {"cuda_graph": True, "chunk_graphs": True}),
    "fixed_step_graph": (False, {"cuda_graph": True, "capture_global": True}),
}
PAIRS = (("rand_eager", "rand_chunk_graphs"), ("fixed_chunk_graphs", "fixed_step_graph"))


def make(kind: str, mode: str):
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
    randomize, kw = MODES[mode]
    return ChunkedDenoiser(net, n_timesteps=50, chunk_size=CHUNK, merge_global=True, chunk_ord="mix-4", cond=cond,
                           randomize_chunks=randomize, graph_warmup=2, **kw)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", choices=("hot", "full"), default="hot")
    ap.add_argument("--steps", type=int, default=20, help="timed steps per round and mode")
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of the four modes")
    ap.add_argument("--check-steps", type=int, default=8, help="steps compared bit for bit within each pair")
    ap.add_argument("--warmup", type=int, default=6, help="untimed steps of each chain after the check (captures)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("random_chunk_graph_bench.py needs a CUDA device")
    name, power = card()

    g = torch.Generator(device="cuda").manual_seed(123)
    x0 = torch.randn((FRAMES, 4, LATENT, LATENT), generator=g, device="cuda", dtype=torch.float16)
    chains = {}
    for mode in MODES:
        chains[mode] = Chain(make(args.workload, mode), x0)
        np.random.seed(2024)              # the same host draws (first chunk, reversal, chunk order) within each pair
        torch.manual_seed(2024)           # and the same device draws (block generators)
        for _ in range(args.check_steps):
            chains[mode].step()
    torch.cuda.synchronize()
    identical = {f"{a}=={b}": torch.equal(chains[a].x, chains[b].x) for a, b in PAIRS}
    finite = all(bool(torch.isfinite(ch.x).all()) for ch in chains.values())
    for ch in chains.values():
        for _ in range(args.warmup):
            ch.step()

    rates = {m: [] for m in MODES}
    for _ in range(args.rounds):
        for mode in MODES:
            rates[mode].append(round(timed(chains[mode], args.steps), 2))

    def med(v):
        return sorted(v)[len(v) // 2]
    line = {"tool": "random_chunk_graph_bench", "workload": args.workload, "card": name, "power_limit": power,
            "frames": FRAMES, "chunk_size": CHUNK, "latent": LATENT, "chunk_ord": "mix-4", "local_ratio": 0.9,
            "global_ratio": 0.8, "global_rand": 0.5, "batch": 2, "check_steps": args.check_steps,
            "latents_bit_identical": identical, "finite": finite, "steps_per_round": args.steps,
            "rounds": args.rounds, "steps_per_s": rates,
            "graphs_captured": {m: len(chains[m].den._chunk_graphs) for m in MODES if "chunk" in m},
            "rand_speedup_median": round(med(rates["rand_chunk_graphs"]) / med(rates["rand_eager"]), 3),
            "fixed_chunk_vs_step_graph_median": round(med(rates["fixed_chunk_graphs"]) / med(rates["fixed_step_graph"]),
                                                      3)}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
