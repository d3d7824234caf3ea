"""The self-attention of blocks that do not merge, during generation: the module's own forward against the library
(patch.FUSE_UNMERGED_ATTENTION, vtm_attention_residual_ex).

Part 1 (kernel level): `attn1(norm1(h)) + h` of one unmerged block at per-frame shapes, after the same LayerNorm, the
module's forward (skeleton Attention: torch SDPA; while injecting, PnP's torch forward pnp._torch_forward with
num_inputs 3) against attention.self_attention_residual (shared_items = B / num_inputs while injecting).  The arms
alternate, the L2 is flushed (a 256 MB write) before every timed call, and each call is timed with CUDA events.
Shapes: SD2.1 512² ds4 (B = 2 x 16 or 3 x 16 items, L 256, C 1280, 20 heads of 64), SD2.1 768² ds4 (L 576), SD1.5 ds4
and ds8 (C 1280, 8 heads of 160, L 256 / 64) at attention.MAX_HEAD_DIM = 160.
Part 2 (step level): the dog config's workload on the SD2.1 full-block skeleton (32 frames at 512², chunk 4, mix-4,
merge_global, PnP with pnp_attn_t 0.5 and pnp_f_t 0.8, chunk_graphs) with the switch on against off, and the same on
SD1.5 with MAX_HEAD_DIM = 160 in both arms.  The arms alternate over --rounds rounds of --steps steps each; a step's
time comes from CUDA events, after 2 warm-up steps.

Median and min-max are reported; one JSON line goes to stdout, with the card name and power limit read in the same run.

    python tools/unmerged_attention_bench.py --reps 30 --rounds 2 --steps 10
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


def _stats(ts):
    return {"median_ms": round(statistics.median(ts), 4), "min_ms": round(min(ts), 4), "max_ms": round(max(ts), 4)}


@torch.no_grad()
def kernel_part(reps: int) -> list:
    from vidtome_b200 import attention, ops, pnp
    from vidtome_b200.skeleton import BasicTransformerBlock
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows = []
    # (label, items, L, C, heads, num_inputs)
    shapes = [("sd21 512 ds4 cfg", 32, 256, 1280, 20, 2), ("sd21 512 ds4 pnp", 48, 256, 1280, 20, 3),
              ("sd21 768 ds4 pnp", 48, 576, 1280, 20, 3), ("sd15 ds4 pnp", 48, 256, 1280, 8, 3),
              ("sd15 ds8 pnp", 48, 64, 1280, 8, 3)]
    attention.MAX_HEAD_DIM = 160
    for label, B, L, C, H, ni in shapes:
        torch.manual_seed(0)
        blk = BasicTransformerBlock(C, H, hot_path_only=True).cuda().half()
        h = torch.randn(B, L, C, device="cuda").half()
        n1 = blk.norm1(h)
        inject_modes = (False, True) if ni == 3 else (False,)
        for inject in inject_modes:
            if inject:
                fwd = pnp._torch_forward(blk.attn1, ni)
                pnp.register_time(None, 1000, modules=[blk.attn1])       # t == 1000 always injects
                blk.attn1.injection_schedule = [1000]
                module = lambda: fwd(n1) + h                              # noqa: E731
                library = lambda: attention.self_attention_residual(blk.attn1, n1, h, shared_items=B // ni)  # noqa
            else:
                module = lambda: blk.attn1(n1) + h                        # noqa: E731
                library = lambda: attention.self_attention_residual(blk.attn1, n1, h)   # noqa: E731
            arms = {"module": module, "library": library}
            times = {k: [] for k in arms}
            outs = {k: f() for k, f in arms.items()}                      # warm-up, and the outputs compared
            for _ in range(reps):
                for k, f in arms.items():
                    flush.fill_(1)
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    s.record()
                    f()
                    e.record()
                    torch.cuda.synchronize()
                    times[k].append(s.elapsed_time(e))
            diff = (outs["module"].float() - outs["library"].float()).abs().max().item()
            rows.append({"shape": label, "B": B, "L": L, "C": C, "heads": H, "inject": inject,
                         "module": _stats(times["module"]), "library": _stats(times["library"]),
                         "speedup": round(statistics.median(times["module"]) / statistics.median(times["library"]), 3),
                         "max_abs_diff": diff})
            print(json.dumps(rows[-1]), file=sys.stderr)
    return rows


@torch.no_grad()
def step_part(name: str, frames: int, size: int, steps: int, rounds: int) -> dict:
    import numpy as np
    import vidtome_b200
    from vidtome_b200 import attention, patch
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton, pnp_attention_modules, pnp_conv_module
    attention.MAX_HEAD_DIM = 160 if name == "sd15" else 128
    cad = 1024 if name == "sd21" else 768
    g = torch.Generator(device="cuda").manual_seed(5)
    cond = torch.randn((3, 77, cad), generator=g, device="cuda").half()
    x0 = torch.randn((frames, 4, size, size), generator=g, device="cuda").half()
    src = torch.randn((frames, 4, size, size), generator=g, device="cuda").half()
    times = {False: [], True: []}
    finals = {}
    for _ in range(rounds):
        for fuse in (False, True):
            patch.FUSE_UNMERGED_ATTENTION = fuse
            torch.manual_seed(77)
            net = make_skeleton(name, hot_path_only=False, device="cuda", pnp_conv=True)
            vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=True, global_merge_ratio=0.8,
                                     global_rand=0.5, batch_size=3, align_batch=True)
            den = ChunkedDenoiser(net, n_timesteps=steps, chunk_size=4, merge_global=True, chunk_ord="mix-4",
                                  cond=cond, source_latents=lambda t: src, pnp_attn_t=0.5,
                                  pnp_modules=pnp_attention_modules(net), pnp_f_t=0.8,
                                  pnp_conv_modules=[pnp_conv_module(net)], randomize_chunks=True, cuda_graph=True,
                                  chunk_graphs=True, graph_warmup=2)
            torch.manual_seed(2024)
            np.random.seed(2024)
            x = x0.clone()
            for i in range(steps):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                x = den.step(x, i)
                e.record()
                torch.cuda.synchronize()
                if i >= 2:
                    times[fuse].append(s.elapsed_time(e))
            finals[fuse] = x
            del den, net
            torch.cuda.empty_cache()
    patch.FUSE_UNMERGED_ATTENTION = False
    off, on = statistics.median(times[False]), statistics.median(times[True])
    diff = (finals[True].float() - finals[False].float()).abs().max().item()
    return {"model": name, "frames": frames, "latent": size, "steps": steps, "off": _stats(times[False]),
            "on": _stats(times[True]), "speedup": round(off / on, 3), "final_max_abs_diff": diff,
            "final_max_abs": finals[False].float().abs().max().item()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--size", type=int, default=64)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("unmerged_attention_bench: needs a CUDA device")
    name, power = card()
    res = {"gpu": name, "power_limit": power, "kernel": kernel_part(args.reps), "step": []}
    for model in ("sd21", "sd15"):
        res["step"].append(step_part(model, args.frames, args.size, args.steps, args.rounds))
        print(json.dumps(res["step"][-1]), file=sys.stderr)
    line = json.dumps(res)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
