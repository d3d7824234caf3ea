"""The transformer blocks of an unpatched ControlNet: their modules' own forwards against the library
(patch.FUSE_CONTROLNET_BLOCKS, patch.serve_unmerged).

Part 1 (block level): one Transformer2DModel with its BasicTransformerBlock (SD1.5, conv proj_in / proj_out, full
block: self-attention, cross-attention over a [B, 77, 768] context, GEGLU feed-forward), served, called with the switch
off (the modules' forwards: GroupNorm, 1x1 convs, torch SDPA, ...) and on (GroupNorm -> tokens, KD with the residual,
cross-attention, GEGLU, proj_out storing NCHW).  Shapes of the SD1.5 ControlNet at 512² with chunk 4 (B = 8 items: 4
frames x CFG): ds1 320 ch / 4096 tokens, ds2 640 / 1024, ds4 1280 / 256, mid 1280 / 64.  The arms alternate, the L2 is
flushed (a 256 MB write) before every timed call, and each call is timed with CUDA events.
Part 2 (ControlNet branch): one call of the SD1.5 ControlNet stand-in (skeleton.make_controlnet, full blocks, conv
wrappers) on the batch of one UNet call, switch off against on.
Part 3 (step level): BASELINE config 3's workload of tools/controlnet_bench.py (SD1.5 skeleton + ControlNet, 32 frames at
512², chunk 4, mix-4, merge_global; --workload full or hot, --io none or conv wrappers) in capture_global mode, one
pipeline captured with the switch off and one with it on, their replays alternating over --rounds rounds of --steps
steps.

attention.MAX_HEAD_DIM is --max-head-dim (default 160) in every arm, so that the 1280-channel blocks (8 heads of 160)
can run in the library; FUSE_UNMERGED_ATTENTION stays off.  Medians with min-max; one JSON line goes to stdout, with
the card name and power limit read in the same run.  --profile DIR adds a torch.profiler table of both arms of every
block shape (run on its own: tracing slows the host).

    python tools/controlnet_blocks_bench.py --reps 30 --rounds 3 --steps 10
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

from global_graph_bench import Chain, card, timed  # noqa: E402

FRAMES, CHUNK, LATENT = 32, 4, 64
# (label, channels, tokens per item) at SD1.5 512², B = 8
SHAPES = [("ds1", 320, 4096), ("ds2", 640, 1024), ("ds4", 1280, 256), ("mid", 1280, 64)]
B = 8


def _stats(ts):
    return {"median_ms": round(statistics.median(ts), 4), "min_ms": round(min(ts), 4), "max_ms": round(max(ts), 4)}


def _wrapper(C: int):
    from vidtome_b200 import patch
    from vidtome_b200.skeleton import BasicTransformerBlock, Transformer2DModel
    torch.manual_seed(C)
    blk = BasicTransformerBlock(C, 8, 768, hot_path_only=False)
    w = Transformer2DModel(C, blk).cuda().half().eval()
    return patch.serve_unmerged(w)


def _event_time(fn, flush=None) -> float:
    if flush is not None:
        flush.fill_(1)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


@torch.no_grad()
def block_part(reps: int, profile_dir=None) -> list:
    from vidtome_b200 import patch
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows = []
    for label, C, T in SHAPES:
        w = _wrapper(C)
        side = int(T ** 0.5)
        g = torch.Generator(device="cuda").manual_seed(1)
        x = torch.randn((B, C, side, side), generator=g, device="cuda").half()
        ctx = torch.randn((B, 77, 768), generator=g, device="cuda").half()
        run = lambda: w(x, encoder_hidden_states=ctx, return_dict=False)[0]      # noqa: E731
        outs, times = {}, {False: [], True: []}
        for on in (False, True):                                 # warm-up: module loads, packed weights
            patch.FUSE_CONTROLNET_BLOCKS = on
            for _ in range(3):
                outs[on] = run()
        torch.cuda.synchronize()
        for _ in range(reps):
            for on in (False, True):
                patch.FUSE_CONTROLNET_BLOCKS = on
                times[on].append(_event_time(run, flush))
        ref = outs[False].float()
        err = (outs[True].float() - ref).abs().max().item() / ref.abs().max().item()
        mod, lib = _stats(times[False]), _stats(times[True])
        rows.append({"shape": label, "B": B, "C": C, "tokens": T, "module": mod, "library": lib,
                     "speedup_median": round(mod["median_ms"] / lib["median_ms"], 3), "rel_max_diff": float(f"{err:.3e}")})
        if profile_dir:
            rows[-1]["profile"] = _profile(run, f"{label}", profile_dir)
        patch.FUSE_CONTROLNET_BLOCKS = False
    return rows


def _profile(run, label, out_dir):
    from torch.profiler import ProfilerActivity, profile as tprof
    from vidtome_b200 import patch
    os.makedirs(out_dir, exist_ok=True)
    res = {}
    for on in (False, True):
        patch.FUSE_CONTROLNET_BLOCKS = on
        torch.cuda.synchronize()
        with tprof(activities=[ProfilerActivity.CUDA]) as p:
            for _ in range(10):
                run()
            torch.cuda.synchronize()
        arm = "library" if on else "module"
        table = p.key_averages().table(sort_by="cuda_time_total", row_limit=15)
        with open(os.path.join(out_dir, f"controlnet_blocks_{label}_{arm}.txt"), "w") as f:
            f.write(table)
        res[arm] = [{"kernel": k.key[:80], "cuda_us_per_call": round(k.device_time_total / 10, 1)}
                    for k in sorted(p.key_averages(), key=lambda k: -k.device_time_total)[:6]]
    patch.FUSE_CONTROLNET_BLOCKS = False
    return res


@torch.no_grad()
def branch_part(reps: int) -> dict:
    from vidtome_b200 import patch
    from vidtome_b200.skeleton import make_controlnet
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    cn = patch.serve_unmerged(make_controlnet("sd15", hot_path_only=False, device="cuda", transformer_io="conv"))
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn((B, 4, LATENT, LATENT), generator=g, device="cuda").half()
    ctx = torch.randn((B, 77, 768), generator=g, device="cuda").half()
    ctrl = torch.rand((B, 3, 8 * LATENT, 8 * LATENT), generator=g, device="cuda").half()
    run = lambda: cn(x, 981, encoder_hidden_states=ctx, controlnet_cond=ctrl)  # noqa: E731
    times, outs = {False: [], True: []}, {}
    for on in (False, True):
        patch.FUSE_CONTROLNET_BLOCKS = on
        for _ in range(3):
            outs[on] = run()
    for _ in range(reps):
        for on in (False, True):
            patch.FUSE_CONTROLNET_BLOCKS = on
            times[on].append(_event_time(run, flush))
    patch.FUSE_CONTROLNET_BLOCKS = False
    errs = [((a.float() - b.float()).abs().max() / b.float().abs().max()).item()
            for a, b in zip(list(outs[True][0]) + [outs[True][1]], list(outs[False][0]) + [outs[False][1]])]
    mod, lib = _stats(times[False]), _stats(times[True])
    return {"B": B, "latent": LATENT, "module": mod, "library": lib,
            "speedup_median": round(mod["median_ms"] / lib["median_ms"], 3),
            "rel_max_diff_residuals": float(f"{max(errs):.3e}")}


def _denoiser(on: bool, ctrl: torch.Tensor, workload: str, io):
    import vidtome_b200
    from vidtome_b200 import patch
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_controlnet, make_skeleton
    torch.manual_seed(123)
    hot = workload == "hot"
    unet = make_skeleton("sd15", hot_path_only=hot, device="cuda", transformer_io=io)
    cn = make_controlnet("sd15", hot_path_only=hot, device="cuda", transformer_io=io)
    vidtome_b200.apply_patch(unet, local_merge_ratio=0.9, merge_global=True, global_merge_ratio=0.8, global_rand=0.5,
                             batch_size=2)
    cond = None
    if not hot:
        gc = torch.Generator(device="cuda").manual_seed(5)
        cond = torch.randn((2, 77, 768), generator=gc, device="cuda", dtype=torch.float16)
    patch.FUSE_CONTROLNET_BLOCKS = on
    return ChunkedDenoiser(unet, n_timesteps=50, chunk_size=CHUNK, merge_global=True, chunk_ord="mix-4", cond=cond,
                           cuda_graph=True, capture_global=True, graph_warmup=2, controlnet=cn, control_images=ctrl,
                           control_scale=1.0)


@torch.no_grad()
def step_part(rounds: int, steps: int, workload: str, io) -> dict:
    from vidtome_b200 import patch
    g = torch.Generator(device="cuda").manual_seed(123)
    x0 = torch.randn((FRAMES, 4, LATENT, LATENT), generator=g, device="cuda", dtype=torch.float16)
    ctrl = torch.rand((FRAMES, 3, 8 * LATENT, 8 * LATENT), generator=g, device="cuda", dtype=torch.float16)
    chains = {}
    for on in (False, True):
        # each pipeline is captured with its own switch state; its replays do not read the switch
        chains[on] = Chain(_denoiser(on, ctrl, workload, io), x0)
        torch.manual_seed(2024)
        for _ in range(5):                                       # 2 eager, the capture, 2 replays
            chains[on].step()
    patch.FUSE_CONTROLNET_BLOCKS = False
    torch.cuda.synchronize()
    diff = (chains[True].x.float() - chains[False].x.float()).abs().max().item()
    rates = {False: [], True: []}
    for _ in range(rounds):
        for on in (False, True):
            rates[on].append(round(timed(chains[on], steps), 3))
    med = {on: statistics.median(r) for on, r in rates.items()}
    return {"workload": f"C3 {workload}, capture_global", "transformer_io": io, "frames": FRAMES, "chunk_size": CHUNK, "latent": LATENT,
            "steps_per_s": {"off": rates[False], "on": rates[True]},
            "median": {"off": med[False], "on": med[True]},
            "range": {"off": [min(rates[False]), max(rates[False])], "on": [min(rates[True]), max(rates[True])]},
            "speedup_median": round(med[True] / med[False], 3), "latents_max_abs_diff_after_5_steps": diff,
            "finite": bool(torch.isfinite(chains[True].x).all())}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=30, help="timed calls per arm and block shape")
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of the step part")
    ap.add_argument("--steps", type=int, default=10, help="steps per round and arm")
    ap.add_argument("--max-head-dim", type=int, default=160)
    ap.add_argument("--parts", default="block,branch,step")
    ap.add_argument("--workload", choices=("hot", "full"), default="full", help="step part: tools/controlnet_bench.py's")
    ap.add_argument("--io", choices=("none", "conv"), default="none",
                    help="step part: Transformer2DModel wrappers around the blocks (none, as tools/controlnet_bench.py)")
    ap.add_argument("--profile", default=None, help="write torch.profiler tables of the block part here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("controlnet_blocks_bench.py needs a CUDA device")
    from vidtome_b200 import attention, patch
    attention.MAX_HEAD_DIM = args.max_head_dim
    patch.FUSE_UNMERGED_ATTENTION = False
    name, power = card()
    parts = args.parts.split(",")
    line = {"tool": "controlnet_blocks_bench", "card": name, "power_limit": power, "max_head_dim": args.max_head_dim}
    if "block" in parts:
        line["blocks"] = block_part(args.reps, args.profile)
    if "branch" in parts:
        line["controlnet_branch"] = branch_part(args.reps)
    if "step" in parts:
        line["step"] = step_part(args.rounds, args.steps, args.workload, None if args.io == "none" else args.io)
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
