"""driver.FUSE_STEP_UPDATE on against off: time per sampling step with the guidance combine and DDIM update fused into
KS (ops.cfg_ddim_update, inside the captured step) against the torch ops they replace (pred_noise's combine and
pred_next_x after the replay).

Workloads, each with two denoisers, one per switch value, alternated round by round in this process on one card.  Each
arm has its own patched skeleton, built from the same seed: a denoiser with global merging installs its own token stores
in the blocks, so two arms on one model would read each other's stores.  Both arms first step the same seeded latents
with the same host and device draws, and their latents are compared bit for bit before the timed rounds.
  config2   bench.py's headline: SD1.5 hot-path skeleton, local merging 0.9, 16 frames of 64 x 64 latents in one chunk,
            CFG batch 2; eager stepping and cuda_graph replay.
  config3   the chunk_graphs workload (tools/random_chunk_graph_bench.py): SD1.5 hot-path skeleton, local 0.9 and
            global 0.8 merging, 32 frames in chunks of 4 with the reference's randomised chunking, chunk_ord "mix-4",
            cuda_graph + chunk_graphs.
Per round and arm: device time per step from CUDA events around --steps steps, and host time per step from
time.perf_counter around the same loop without a synchronise (the time step() takes to issue its work).  Medians,
spreads and whether every round's on-arm beat its off-arm are reported.
kernel    KS alone against the torch ops it replaces (the combine's 3 ops and pred_next_x's 6) at 4, 16 and 64 frames of
            4 x 64 x 64 latents: CUDA events around each call, the L2 flushed (a 256 MB write) before each, medians.

One JSON line on stdout, with the card's name, power limit and SM clocks read in the same run.

    python tools/step_update_bench.py --steps 50 --rounds 5
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return dict(zip(q.split(","), [s.strip() for s in out[0].split(",")]))
    except Exception as e:                      # report, do not guess
        return {"name": torch.cuda.get_device_name(), "error": type(e).__name__}


def _model(name: str, merge_global: bool):
    import vidtome_b200
    from vidtome_b200.skeleton import make_skeleton
    torch.manual_seed(123)
    net = make_skeleton(name, hot_path_only=True, device="cuda")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, batch_size=2, merge_global=merge_global,
                             global_merge_ratio=0.8, global_rand=0.5)
    return net


def _arms(config: str, graph: bool):
    from vidtome_b200.driver import ChunkedDenoiser
    if config == "config2":
        name, merge_global, frames = "sd15", False, 16
        kw = dict(chunk_size=16, cuda_graph=graph)
    else:
        name, merge_global, frames = "sd15", True, 32
        kw = dict(chunk_size=4, merge_global=True, chunk_ord="mix-4", randomize_chunks=True, cuda_graph=True,
                  chunk_graphs=True)
    return {fuse: ChunkedDenoiser(_model(name, merge_global), n_timesteps=50, **kw) for fuse in (True, False)}, frames


@torch.no_grad()
def stepping(config: str, graph: bool, steps: int, rounds: int) -> dict:
    from vidtome_b200 import driver
    arms, frames = _arms(config, graph)
    # config3 draws its chunk lengths: enough warm-up steps that the chunk graphs of most (length, first chunk) keys are
    # captured before the timed rounds
    warm = 6 if config == "config2" else 24
    g = torch.Generator(device="cuda").manual_seed(5)
    x0 = torch.randn((frames, 4, 64, 64), generator=g, device="cuda", dtype=torch.float16)
    state = {}
    for fuse, den in arms.items():                         # warm-up: eager steps, captures, replays
        driver.FUSE_STEP_UPDATE = fuse
        np.random.seed(2024)                               # the same host draws (chunking, chunk order)
        torch.manual_seed(2024)                            # and the same device draws (block generators)
        x = x0.clone()
        for i in range(warm):
            x = den.step(x, i)
        state[fuse] = [x, warm]
    torch.cuda.synchronize()
    equal = bool(torch.equal(state[True][0], state[False][0]))
    dev = {k: [] for k in arms}
    host = {k: [] for k in arms}
    for _ in range(rounds):
        for fuse, den in arms.items():
            driver.FUSE_STEP_UPDATE = fuse
            st = state[fuse]
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            s.record()
            for _ in range(steps):
                st[0] = den.step(st[0], st[1] % 50)
                st[1] += 1
            e.record()
            t1 = time.perf_counter()
            torch.cuda.synchronize()
            dev[fuse].append(s.elapsed_time(e) / steps)
            host[fuse].append((t1 - t0) * 1e3 / steps)
    driver.FUSE_STEP_UPDATE = True

    def summary(v):
        return {"median": round(statistics.median(v), 4), "min": round(min(v), 4), "max": round(max(v), 4)}
    return {"frames": frames, "steps_per_round": steps, "rounds": rounds, "latents_equal_after_warmup": equal,
            "chunk_graphs_captured": {"on": len(arms[True]._chunk_graphs), "off": len(arms[False]._chunk_graphs)},
            "device_ms_per_step": {"on": summary(dev[True]), "off": summary(dev[False])},
            "host_ms_per_step": {"on": summary(host[True]), "off": summary(host[False])},
            "device_on_faster_every_round": all(a < b for a, b in zip(dev[True], dev[False])),
            "host_on_faster_every_round": all(a < b for a, b in zip(host[True], host[False])),
            "device_saving_ms": round(statistics.median(dev[False]) - statistics.median(dev[True]), 4),
            "host_saving_ms": round(statistics.median(host[False]) - statistics.median(host[True]), 4)}


@torch.no_grad()
def kernel(frames: int, iters: int) -> dict:
    from vidtome_b200 import ops
    from vidtome_b200.driver import ChunkedDenoiser
    den = ChunkedDenoiser(torch.nn.Identity(), n_timesteps=50)
    coef, step = den.step_tables("cuda")
    step.fill_(10)
    n = frames * 4 * 64 * 64
    g = torch.Generator(device="cuda").manual_seed(frames)
    x = torch.randn((frames, 4, 64, 64), generator=g, device="cuda").half()
    eps = torch.randn((2 * frames, 4, 64, 64), generator=g, device="cuda").half()
    out = torch.empty_like(x)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def fused():
        ops.cfg_ddim_update(x, eps, 2, 7.5, coef, step, out)

    def torch_ops():
        u, c = eps.chunk(2)
        den.pred_next_x(x, u + 7.5 * (c - u), 10)

    res = {}
    for name, fn in (("KS", fused), ("torch", torch_ops)):
        fn()
        ts = []
        for _ in range(iters):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            torch.cuda.synchronize()
            ts.append(s.elapsed_time(e) * 1e3)
        res[name] = round(statistics.median(ts), 2)
    # bytes: KS reads x, u, c and writes out; torch: 3 + 6 ops of 2 reads (or 1) and 1 write each
    ks_bytes = 4 * 2 * n
    return {"frames": frames, "elements": n, "us": res, "ks_bytes": ks_bytes,
            "ks_GBps": round(ks_bytes / (res["KS"] * 1e-6) / 1e9, 1), "speedup": round(res["torch"] / res["KS"], 2)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("step_update_bench needs a CUDA device")
    res = {"card": card()}
    res["config2_graph"] = stepping("config2", True, args.steps, args.rounds)
    res["config2_eager"] = stepping("config2", False, max(5, args.steps // 5), args.rounds)
    res["config3_chunk_graphs"] = stepping("config3", True, max(5, args.steps // 5), args.rounds)
    res["kernel"] = [kernel(f, args.iters) for f in (4, 16, 64)]
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
