"""PnP generation (the reference's default config) in the step driver: eager vs one CUDA graph per chunk, and the
flash kernel's time per shared (PnP-injected) self-attention call.

Workload: configs/default.yaml of the reference on the SD1.5 skeleton at 512x512 (latent 64): 32 frames, chunk_size 4
with a random first chunk, "mix-4" order, local merging 0.9 + global merging 0.8 with global_rand 0.5, align_batch,
three samples per UNet call (source, uncond, cond), 50 timesteps with pnp_attn_t 0.5 (the first 25 steps take the
decoder self-attention map from the source sample).  "hot" runs the merge + self-attention path only; "full" adds
cross-attention over the [3, 77, 768] text context and the feed-forward.

Part 1: an eager and a chunk-graph denoiser drive two identical skeletons over the same 50 steps with the same host
draws; the latents after every step are compared bit for bit.  Then --rounds timed passes of 50 steps alternate the two.
Every step is timed with CUDA events; steps/s is reported from the median step time of the injected and of the
non-injected steps (the median leaves out the few steps that capture a graph).

Part 2: the shapes of the shared KD calls of one injected step are recorded; each is timed in a child process per
library build (--prev-lib: another build of the same library, loaded through VIDTOME_B200_LIB), the builds alternated
--ab-rounds times.  torch.profiler gives the flash kernel's device time per call.

One JSON line goes to stdout, with the card name and power limit read in the same run.

    python tools/pnp_bench.py --workload hot --rounds 2 [--prev-lib build/prev/libvidtome_b200.so]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.global_graph_bench import CHUNK, FRAMES, LATENT, card  # noqa: E402

STEPS = 50


def make(kind: str, graph: bool, sources):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton, pnp_attention_modules
    torch.manual_seed(123)
    net = make_skeleton("sd15", hot_path_only=(kind == "hot"), device="cuda")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=True, global_merge_ratio=0.8, global_rand=0.5,
                             batch_size=3, align_batch=True)
    gc = torch.Generator(device="cuda").manual_seed(5)
    cond = torch.randn((3, 77, 768), generator=gc, device="cuda", dtype=torch.float16)
    return ChunkedDenoiser(net, n_timesteps=STEPS, chunk_size=CHUNK, merge_global=True, chunk_ord="mix-4", cond=cond,
                           randomize_chunks=True, cuda_graph=graph, chunk_graphs=graph, graph_warmup=2,
                           source_latents=sources.__getitem__, pnp_attn_t=0.5, pnp_modules=pnp_attention_modules(net))


def make_sources():
    from vidtome_b200.driver import ddim_timesteps
    out = {}
    for t in ddim_timesteps(STEPS):
        g = torch.Generator(device="cuda").manual_seed(int(t))
        out[t] = torch.randn((FRAMES, 4, LATENT, LATENT), generator=g, device="cuda", dtype=torch.float16)
    return out


def run_pass(den, x, seed, times=None):
    """50 steps from x with the host draws seeded; per-step event times (ms) appended to `times`."""
    torch.manual_seed(seed)
    np.random.seed(seed)
    xs = []
    ev = []
    for i in range(STEPS):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        x = den.step(x, i)
        e.record()
        ev.append((s, e))
        xs.append(x)
    torch.cuda.synchronize()
    if times is not None:
        times.append([s.elapsed_time(e) for s, e in ev])
    return xs


def driver_part(kind: str, rounds: int):
    sources = make_sources()
    g = torch.Generator(device="cuda").manual_seed(7)
    x0 = torch.randn((FRAMES, 4, LATENT, LATENT), generator=g, device="cuda", dtype=torch.float16)
    dens = {"eager": make(kind, False, sources), "chunk_graphs": make(kind, True, sources)}
    n_inj = len(dens["eager"].pnp_schedule)
    # pass 0: warm-up, captures, and the bit-identity check
    ref = run_pass(dens["eager"], x0, 2024)
    got = run_pass(dens["chunk_graphs"], x0, 2024)
    identical = all(torch.equal(a, b) for a, b in zip(ref, got))
    times = {k: [] for k in dens}
    for r in range(rounds):
        for k in dens:
            run_pass(dens[k], x0, 3000 + r, times[k])
    out = {"bit_identical_50_steps": identical, "injected_steps": n_inj}
    for k, ts in times.items():
        inj = [t for row in ts for t in row[:n_inj]]
        rest = [t for row in ts for t in row[n_inj:]]
        out[k] = {"injected_steps_per_s": round(1e3 / statistics.median(inj), 2),
                  "plain_steps_per_s": round(1e3 / statistics.median(rest), 2),
                  "pass_s_median": round(statistics.median(sum(row) for row in ts) / 1e3, 3)}
    # the shapes of the shared KD calls of one injected eager step
    from vidtome_b200 import attention as A
    shapes = []
    inner = A.ops.attention

    def recording(x, w_qkv, w_o, b_o, heads, scale, shared_qk=False, seq_len=None):
        if shared_qk:
            n = int(seq_len.item()) if seq_len is not None else None
            shapes.append((tuple(x.shape), int(heads), n))
        return inner(x, w_qkv, w_o, b_o, heads, scale, shared_qk=shared_qk, seq_len=seq_len)
    A.ops.attention = recording
    try:
        torch.manual_seed(1)
        np.random.seed(1)
        dens["eager"].step(x0, 0)
    finally:
        A.ops.attention = inner
    torch.cuda.synchronize()
    return out, sorted(set(shapes), key=str)


def kernel_child(shapes, iters: int):
    """Device time per shared KD call (flash kernel and whole call) at each shape, with this process's library."""
    from torch.profiler import ProfilerActivity, profile
    from vidtome_b200 import ops
    res = []
    for (B, L, C), heads, n in shapes:
        g = torch.Generator(device="cuda").manual_seed(L + C)
        x = torch.randn((B, L, C), generator=g, device="cuda", dtype=torch.float16)
        w_qkv = (torch.randn((3 * C, C), generator=g, device="cuda") * C ** -0.5).half()
        w_o = (torch.randn((C, C), generator=g, device="cuda") * C ** -0.5).half()
        b_o = torch.zeros(C, device="cuda", dtype=torch.float16)
        seq = None if n is None else torch.tensor([n], dtype=torch.int32, device="cuda")
        scale = (C // heads) ** -0.5
        for _ in range(5):
            ops.attention(x, w_qkv, w_o, b_o, heads, scale, shared_qk=True, seq_len=seq)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                ops.attention(x, w_qkv, w_o, b_o, heads, scale, shared_qk=True, seq_len=seq)
            torch.cuda.synchronize()
        flash = total = 0.0
        for ev in prof.key_averages():               # CUDA activity only: the kernels of the KD calls
            dt = ev.device_time_total
            total += dt
            if "flash_attn_kernel" in ev.key:
                flash += dt
        res.append({"B": B, "L": L, "C": C, "heads": heads, "seq_len": n,
                    "flash_us_per_call": round(flash / iters, 2), "kd_kernels_us_per_call": round(total / iters, 2)})
    return res


def kernel_part(shapes, prev_lib, ab_rounds: int, iters: int):
    builds = {"this": None}
    if prev_lib:
        builds["prev"] = os.path.abspath(prev_lib)
    runs = {k: [] for k in builds}
    for _ in range(ab_rounds):
        for name, lib in builds.items():
            env = dict(os.environ)
            env.pop("VIDTOME_B200_LIB", None)
            if lib:
                env["VIDTOME_B200_LIB"] = lib
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--kernel-child", json.dumps(shapes),
                                "--iters", str(iters)], env=env, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"kernel child ({name}) failed:\n{r.stderr[-4000:]}")
            runs[name].append(json.loads(r.stdout.strip().splitlines()[-1]))
    out = []
    for i, shp in enumerate(shapes):
        row = dict(runs["this"][0][i])
        for name in builds:
            row[f"flash_us_{name}"] = [run[i]["flash_us_per_call"] for run in runs[name]]
            row[f"kd_us_{name}"] = [run[i]["kd_kernels_us_per_call"] for run in runs[name]]
        del row["flash_us_per_call"], row["kd_kernels_us_per_call"]
        out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=("hot", "full"), default="hot")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--prev-lib", default=None)
    ap.add_argument("--ab-rounds", type=int, default=2)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--kernel-child", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pnp_bench: needs a CUDA device")
    if args.kernel_child is not None:
        shapes = [(tuple(s[0]), s[1], s[2]) for s in json.loads(args.kernel_child)]
        print(json.dumps(kernel_child(shapes, args.iters)))
        return
    name, power = card()
    drv, shapes = driver_part(args.workload, args.rounds)
    kern = kernel_part(shapes, args.prev_lib, args.ab_rounds, args.iters)
    print(json.dumps({"tool": "pnp_bench", "workload": args.workload, "card": name, "power_limit": power,
                      "frames": FRAMES, "latent": LATENT, "chunk_size": CHUNK, "driver": drv, "shared_kd_calls": kern}))


if __name__ == "__main__":
    main()
