"""PnP's conv-feature injection: the library ResNet path against the reference's forward, the residual-tail kernel (KT)
against torch's four tail ops, and a PnP driver step with and without the conv injection.

Part 1: SD1.5's up_blocks[1].resnets[1] at 512x512 (2560 -> 1280 channels, 16 x 16, temb 1280), 3 samples (source,
uncond, cond) of n = 4 and n = 16 frames, injecting and not: the reference's conv_forward in torch ops
(pnp._conv_torch_forward) against the library path (pnp.conv_library_forward: norm1 ... conv2 on the source third only
while injecting, then KT).  Also whether the two give the same bits.
Part 2: the tail alone at the same shapes, injecting: torch's two slice copies, add and divide (the reference's ops)
against one KT launch; bytes/s from the algorithmic traffic of each (19 n E and 7 n E halfs, E = C H W).
Part 3: a PnP driver step (chunk graphs, the reference's default config: pnp_attn_t 0.5, random chunking, mix-4, local
0.9 + global 0.8 merging) on the SD1.5 skeleton with the stand-in ResNet, latent 64, --frames frames: the steps in
which only the conv injection is active (25-39 of 50), with pnp_f_t = 0.8 and with pnp_f_t off (the ResNet then runs
its plain full-batch forward).

Every time comes from CUDA events; the implementations alternate over --rounds rounds and the median is reported.
One JSON line goes to stdout, with the card name and power limit read in the same run.

    python tools/pnp_conv_bench.py --rounds 5
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


def timed(fn, iters: int) -> float:
    """ms per call of fn over `iters` back-to-back calls."""
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def alternate(fns: dict, rounds: int, iters: int) -> dict:
    for fn in fns.values():                      # warm-up: cuDNN autotuning, allocator
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            times[k].append(timed(fn, iters))
    return {k: statistics.median(v) for k, v in times.items()}


@torch.no_grad()
def resnet_part(rounds: int, iters: int):
    from vidtome_b200 import pnp
    from vidtome_b200.skeleton import ResnetBlock2D
    torch.manual_seed(0)
    resnet = ResnetBlock2D(2560, 1280, temb_channels=1280).to(device="cuda", dtype=torch.float16).eval()
    pnp.register_conv_control(None, [981], 3, modules=[resnet])
    out = []
    for n in (4, 16):
        g = torch.Generator(device="cuda").manual_seed(n)
        x = torch.randn((3 * n, 2560, 16, 16), generator=g, device="cuda").half()
        temb = torch.randn((3 * n, 1280), generator=g, device="cuda").half()
        for t, inject in ((981, True), (961, False)):
            pnp.register_time(None, t, modules=[resnet])
            ref = pnp._conv_torch_forward(resnet, 3, x, temb)
            lib = pnp.conv_library_forward(resnet, x, temb)
            ms = alternate({"reference": lambda: pnp._conv_torch_forward(resnet, 3, x, temb),
                            "library": lambda: pnp.conv_library_forward(resnet, x, temb)}, rounds, iters)
            out.append({"n": n, "batch": 3 * n, "inject": inject, "reference_ms": round(ms["reference"], 4),
                        "library_ms": round(ms["library"], 4), "speedup": round(ms["reference"] / ms["library"], 3),
                        "bit_identical": bool(torch.equal(ref, lib)),
                        "max_abs_diff": float((ref.float() - lib.float()).abs().max())})
        # the cuDNN question on its own: the source rows of the branch on batch n against batch 3n
        branch = lambda z: resnet.conv2(resnet.nonlinearity(resnet.norm2(                          # noqa: E731
            resnet.conv1(resnet.nonlinearity(resnet.norm1(z))))))
        out[-1]["source_branch_batch_n_vs_3n_bit_identical"] = bool(torch.equal(branch(x)[:n], branch(x[:n])))
    return out


@torch.no_grad()
def tail_part(rounds: int, iters: int):
    from vidtome_b200 import ops
    out = []
    E = 1280 * 16 * 16
    for n in (4, 16):
        g = torch.Generator(device="cuda").manual_seed(n)
        h = torch.randn((3 * n, 1280, 16, 16), generator=g, device="cuda").half()
        s = torch.randn_like(h)
        osf = 1.0
        dst = torch.empty_like(h)

        def reference():
            h[n:2 * n] = h[:n]
            h[2 * n:3 * n] = h[:n]
            return (s + h) / osf

        def kernel():
            return ops.resnet_tail(h, s, 3, osf, True, out=dst)
        ms = alternate({"torch": reference, "kt": kernel}, rounds, iters)
        out.append({"n": n, "sample_elems": E, "torch_us": round(ms["torch"] * 1e3, 2), "kt_us": round(ms["kt"] * 1e3, 2),
                    "torch_GBps": round(19 * n * E * 2 / (ms["torch"] * 1e-3) / 1e9, 1),
                    "kt_GBps": round(7 * n * E * 2 / (ms["kt"] * 1e-3) / 1e9, 1),
                    "bit_identical": bool(torch.equal(reference(), kernel()))})
    return out


def make_denoiser(pnp_f_t, frames: int, sources):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton, pnp_attention_modules, pnp_conv_module
    torch.manual_seed(123)
    net = make_skeleton("sd15", device="cuda", pnp_conv=True)
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=True, global_merge_ratio=0.8, global_rand=0.5,
                             batch_size=3, align_batch=True)
    gc = torch.Generator(device="cuda").manual_seed(5)
    cond = torch.randn((3, 77, 768), generator=gc, device="cuda", dtype=torch.float16)
    return ChunkedDenoiser(net, n_timesteps=50, chunk_size=4, merge_global=True, chunk_ord="mix-4", cond=cond,
                           randomize_chunks=True, cuda_graph=True, chunk_graphs=True, graph_warmup=2,
                           source_latents=sources.__getitem__, pnp_attn_t=0.5, pnp_modules=pnp_attention_modules(net),
                           pnp_f_t=pnp_f_t, pnp_conv_modules=None if pnp_f_t is None else [pnp_conv_module(net)])


def driver_part(rounds: int, frames: int):
    from vidtome_b200.driver import ddim_timesteps
    sources = {}
    for t in ddim_timesteps(50):
        g = torch.Generator(device="cuda").manual_seed(int(t))
        sources[t] = torch.randn((frames, 4, 64, 64), generator=g, device="cuda", dtype=torch.float16)
    g = torch.Generator(device="cuda").manual_seed(7)
    x0 = torch.randn((frames, 4, 64, 64), generator=g, device="cuda", dtype=torch.float16)
    dens = {"pnp_f_t_0.8": make_denoiser(0.8, frames, sources), "pnp_f_t_off": make_denoiser(None, frames, sources)}
    steps = range(25, 40)                         # attention injection over, conv injection on (with pnp_f_t 0.8)
    times = {k: [] for k in dens}
    for r in range(rounds + 1):
        for k, den in dens.items():
            torch.manual_seed(r)
            np.random.seed(r)
            x = x0
            ev = []
            for i in ([0, 1, 2] if r == 0 else []):             # warm-up: eager steps, then the captures
                x = den.step(x, i)
            for i in steps:
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                x = den.step(x, i)
                e.record()
                ev.append((s, e))
            torch.cuda.synchronize()
            if r > 0:                                            # round 0 captures the graphs
                times[k].extend(s.elapsed_time(e) for s, e in ev)
    out = {k: {"step_ms_median": round(statistics.median(v), 3),
               "steps_per_s": round(1e3 / statistics.median(v), 2)} for k, v in times.items()}
    out["conv_injecting"] = [dens["pnp_f_t_0.8"].conv_injecting(dens["pnp_f_t_0.8"].timesteps[i]) for i in steps][0]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--frames", type=int, default=16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pnp_conv_bench: needs a CUDA device")
    name, power = card()
    res = {"tool": "pnp_conv_bench", "card": name, "power_limit": power,
           # a tail call takes tens of microseconds: 100x the calls, so that each timed window lasts tens of ms
           "resnet": resnet_part(args.rounds, args.iters), "tail": tail_part(args.rounds, args.iters * 100),
           "driver": driver_part(args.rounds, args.frames), "frames": args.frames}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
