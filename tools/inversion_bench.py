"""DDIM inversion (driver.ChunkedInverter): the reference's inversion on the unpatched model against the patched model
run unmerged through the library, eager and from CUDA graphs; and KD with the residual against the module's forward.

Part 1: the full-block skeleton (SD1.5, then SD2.1), --frames frames of 512x512 video (64 x 64 latents, the reference's
default frame_range of 32 frames), batch_size 8, 50 steps, every timestep kept.  Three arms alternate in one process over
--rounds rounds: `torch` (the unpatched skeleton: its own forward, torch SDPA, and the torch-op update), `eager` (the
same weights patched: unmerged blocks through KD-residual, XA and the GEGLU feed-forward, and KI) and `graph` (the
patched model, one CUDA graph per step after 2 eager steps).  The run checks that the graph and eager trajectories are
bit-identical and reports the largest difference of the final latents between `torch` and `eager`.
Part 2: one unmerged block's self-attention with its residual at the per-frame shapes of SD1.5's ds1 and ds2 blocks
(8 frames x 4096 tokens x 320 channels, 8 x 1024 x 640), `attn1(norm1(h)) + h` through the module's forward (torch
SDPA) against vtm_attention_residual (both after the same LayerNorm).

Every time comes from CUDA events; the median over rounds is reported.  One JSON line goes to stdout, with the card
name and power limit read in the same run.

    python tools/inversion_bench.py --rounds 3
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.global_graph_bench import card  # noqa: E402


def _event_ms(fn) -> float:
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    out = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e), out


@torch.no_grad()
def inversion_part(name: str, frames: int, size: int, batch: int, steps: int, rounds: int) -> dict:
    import vidtome_b200
    from vidtome_b200.driver import ChunkedInverter
    from vidtome_b200.skeleton import make_skeleton
    cad = 1024 if name == "sd21" else 768
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(frames, 4, size, size, generator=g, device="cuda").half()
    cond = torch.randn(frames, 77, cad, generator=g, device="cuda").half()
    plain = make_skeleton(name, hot_path_only=False, device="cuda")
    patched = make_skeleton(name, hot_path_only=False, device="cuda")
    vidtome_b200.apply_patch(patched, local_merge_ratio=0.9, batch_size=2)
    kw = dict(n_timesteps=steps, batch_size=batch, cond=cond)
    arms = {"torch": ChunkedInverter(plain, **kw), "eager": ChunkedInverter(patched, **kw),
            "graph": ChunkedInverter(patched, cuda_graph=True, graph_warmup=2, **kw)}
    times = {k: [] for k in arms}
    finals = {}
    for r in range(rounds + 1):                      # round 0 warms up every arm
        for k, inv in arms.items():
            ms, out = _event_ms(lambda: inv.invert(x))
            if r:
                times[k].append(ms)
            finals[k] = out
    same = bool(torch.equal(arms["graph"].trajectory, arms["eager"].trajectory))
    diff = (finals["torch"].float() - finals["eager"].float()).abs().max().item()
    med = {k: statistics.median(v) for k, v in times.items()}
    return {"model": name, "frames": frames, "latent": size, "batch_size": batch, "steps": steps,
            "ms": {k: round(v, 1) for k, v in med.items()},
            "speedup_vs_torch": {k: round(med["torch"] / med[k], 3) for k in ("eager", "graph")},
            "graph_equals_eager": same, "final_max_abs_diff_torch_vs_library": diff,
            "final_max_abs": finals["torch"].float().abs().max().item()}


@torch.no_grad()
def attention_part(rounds: int, iters: int) -> list:
    from vidtome_b200 import attention, ops, patch
    from vidtome_b200.skeleton import BasicTransformerBlock
    out = []
    for B, L, C, H in ((8, 4096, 320, 8), (8, 1024, 640, 8)):
        torch.manual_seed(C)
        blk = BasicTransformerBlock(C, H, 768, hot_path_only=True).to("cuda", torch.float16).eval()
        h = torch.randn(B, L, C, device="cuda").half()
        ln = patch._fusable_layer_norm(blk.norm1, h)
        n1 = ops.layer_norm(h.view(-1, C), ln).view(B, L, C)
        arms = {"module": lambda: blk.attn1(n1) + h, "library": lambda: attention.self_attention_residual(blk.attn1, n1, h)}
        for fn in arms.values():
            fn()
        times = {k: [] for k in arms}
        for _ in range(rounds):
            for k, fn in arms.items():
                times[k].append(_event_ms(lambda: [fn() for _ in range(iters)])[0] / iters)
        med = {k: statistics.median(v) for k, v in times.items()}
        diff = (arms["module"]().float() - arms["library"]().float()).abs().max().item()
        flops = 4.0 * B * L * L * C + 8.0 * B * L * C * C
        out.append({"B": B, "L": L, "C": C, "heads": H, "ms": {k: round(v, 3) for k, v in med.items()},
                    "speedup": round(med["module"] / med["library"], 3),
                    "library_tflops": round(flops / med["library"] / 1e9, 1), "max_abs_diff": diff})
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--size", type=int, default=64, help="latent side (64 = 512x512 video)")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--models", default="sd15,sd21")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("inversion_bench needs a CUDA device")
    res = {"card": card(), "attention": attention_part(args.rounds, args.iters),
           "inversion": [inversion_part(m, args.frames, args.size, args.batch, args.steps, args.rounds)
                         for m in args.models.split(",")]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
