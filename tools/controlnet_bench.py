"""Step rate of ControlNet-controlled chunked sampling (BASELINE config 3 with the ControlNet branch), eager against
each CUDA-graph mode of the step driver.

Workload: the SD1.5 skeleton and its ControlNet stand-in (skeleton.make_controlnet: the encoder half of the census) at
512x512 (latent 64), 32 frames with [32, 3, 512, 512] control images, chunks of 4 visited in "mix-4" order, local
merging 0.9 + global merging 0.8 with global_rand 0.5, classifier-free guidance (B = 2), control_scale 1.0.  "hot" runs
the merge + self-attention path only (as bench.py's hot workload); "full" adds cross-attention over a [2, 77, 768] text
context and the feed-forward, in the UNet and the ControlNet.  --include-control patches the ControlNet's blocks too
(apply_patch(include_control=True) on a StableDiffusionControlNetPipeline); by default they stay unpatched, as in the
reference's generation.

Four denoisers drive four identical pipelines: "eager", "capture_global" (one graph per step over chunk slots),
"chunk_graphs" (one graph per chunk) and "capture_global_no_controlnet" (the same workload without the ControlNet
branch: what the branch costs).  Each first steps the same seeded latents --check-steps times, and the final latents of
each graph mode are compared bit for bit with eager's.  Then --rounds timed rounds alternate the modes, --steps steps
each, timed with CUDA events.  One JSON line goes to stdout, with the card name and power limit read in the same run.

    python tools/controlnet_bench.py --workload hot --steps 20 --rounds 3
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from global_graph_bench import Chain, card, timed  # noqa: E402

FRAMES, CHUNK, LATENT = 32, 4, 64
MODES = ("eager", "capture_global", "chunk_graphs", "capture_global_no_controlnet")


def make(kind: str, mode: str, include_control: bool, control_images: torch.Tensor):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_controlnet, make_skeleton

    class DiffusionPipeline:
        pass

    class StableDiffusionControlNetPipeline(DiffusionPipeline):       # apply_patch matches the class name
        def __init__(self):
            self.unet = make_skeleton("sd15", hot_path_only=(kind == "hot"), device="cuda")
            self.controlnet = make_controlnet("sd15", hot_path_only=(kind == "hot"), device="cuda")

    torch.manual_seed(123)
    pipe = StableDiffusionControlNetPipeline()
    vidtome_b200.apply_patch(pipe, local_merge_ratio=0.9, merge_global=True, global_merge_ratio=0.8, global_rand=0.5,
                             batch_size=2, include_control=include_control)
    cond = None
    if kind != "hot":
        gc = torch.Generator(device="cuda").manual_seed(5)
        cond = torch.randn((2, 77, 768), generator=gc, device="cuda", dtype=torch.float16)
    kw = {}
    if mode != "eager":
        kw.update(cuda_graph=True, graph_warmup=2, chunk_graphs=(mode == "chunk_graphs"),
                  capture_global=(mode != "chunk_graphs"))
    if mode != "capture_global_no_controlnet":
        kw.update(controlnet=pipe.controlnet, control_images=control_images, control_scale=1.0)
    return ChunkedDenoiser(pipe.unet, n_timesteps=50, chunk_size=CHUNK, merge_global=True, chunk_ord="mix-4",
                           cond=cond, **kw)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", choices=("hot", "full"), default="hot")
    ap.add_argument("--include-control", action="store_true", help="patch the ControlNet's blocks too")
    ap.add_argument("--steps", type=int, default=20, help="timed steps per round and mode")
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds over the modes")
    ap.add_argument("--check-steps", type=int, default=6, help="steps compared bit for bit (2 eager + capture + replays)")
    ap.add_argument("--warmup", type=int, default=3, help="untimed steps of each chain after the check")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("controlnet_bench.py needs a CUDA device")
    name, power = card()

    g = torch.Generator(device="cuda").manual_seed(123)
    x0 = torch.randn((FRAMES, 4, LATENT, LATENT), generator=g, device="cuda", dtype=torch.float16)
    ctrl = torch.rand((FRAMES, 3, 8 * LATENT, 8 * LATENT), generator=g, device="cuda", dtype=torch.float16)
    chains = {}
    for mode in MODES:
        chains[mode] = Chain(make(args.workload, mode, args.include_control, ctrl), x0)
        torch.manual_seed(2024)           # the same host (chunk order) and device (block generators) draws
        for _ in range(args.check_steps):
            chains[mode].step()
    torch.cuda.synchronize()
    identical = {m: torch.equal(chains["eager"].x, chains[m].x) for m in ("capture_global", "chunk_graphs")}
    finite = all(bool(torch.isfinite(ch.x).all()) for ch in chains.values())
    for ch in chains.values():
        for _ in range(args.warmup):
            ch.step()

    rates = {m: [] for m in MODES}
    for _ in range(args.rounds):
        for mode in MODES:
            rates[mode].append(round(timed(chains[mode], args.steps), 2))
    med = {m: sorted(r)[len(r) // 2] for m, r in rates.items()}
    line = {"tool": "controlnet_bench", "workload": args.workload, "include_control": args.include_control,
            "card": name, "power_limit": power, "frames": FRAMES, "chunk_size": CHUNK, "latent": LATENT,
            "chunk_ord": "mix-4", "local_ratio": 0.9, "global_ratio": 0.8, "global_rand": 0.5, "batch": 2,
            "control_scale": 1.0, "check_steps": args.check_steps, "latents_bit_identical": identical,
            "finite": finite, "steps_per_round": args.steps, "rounds": args.rounds,
            "steps_per_s": rates, "ranges": {m: [min(r), max(r)] for m, r in rates.items()},
            "speedup_median": {m: round(med[m] / med["eager"], 3) for m in ("capture_global", "chunk_graphs")},
            "controlnet_cost_median": round(med["capture_global_no_controlnet"] / med["capture_global"], 3)}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
