"""Head_dim 160 (SD1.5's 1280-channel blocks, 8 heads): the library against each module's own forward.

Prints one JSON line per measurement, after a line naming the device, its power limit and SM clocks:
- `kd`: KD (QKV projection, flash kernel, out projection: ops.attention) against the module's forward (cuBLAS
  projections + torch SDPA) on the merged tokens of a ds4 (B = 2, L = 641) and a ds8 (B = 2, L = 161) block; `flash_ms`
  is the flash kernel alone (torch.profiler, in a pass of its own after the timed rounds);
- `xa`: cross-attention with the residual (ops.cross_attention) against the module's forward plus the residual, 32
  items of 256 (ds4) or 64 (ds8) queries over 77 context rows;
- `step`: the full SD1.5 skeleton (cross-attention and feed-forward) on a 16-frame chunk at 512x512 (latents
  [16, 4, 64, 64], CFG batch 2), patched with max_downsample 4 or 8, one ChunkedDenoiser(cuda_graph=True) step per
  replay, with `attention.MAX_HEAD_DIM` at 128 (d = 160 modules run their own forward) and at 160.
Every arm is timed with CUDA events, L2 flushed (a 256 MiB write) before each call of the kernel-level arms; the arms of
a comparison alternate round by round and each figure is the median (with min and max) of at least `--iters` samples.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vidtome_b200 import attention, ops  # noqa: E402

_flush = None


def flush_l2():
    global _flush
    if _flush is None:
        _flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    _flush.fill_(1)


def timed_ms(fn, flush=True):
    if flush:
        flush_l2()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def alternate(arms, iters, warmup=3, flush=True):
    """{name: [ms, ...]}: the arms run in turn, `iters` rounds, after `warmup` untimed rounds."""
    for _ in range(warmup):
        for fn in arms.values():
            fn()
    out = {k: [] for k in arms}
    for _ in range(iters):
        for k, fn in arms.items():
            out[k].append(timed_ms(fn, flush))
    return out


def summary(ts):
    return {"median": round(statistics.median(ts), 4), "min": round(min(ts), 4), "max": round(max(ts), 4), "n": len(ts)}


def device_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        pl, cmax, cnow = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
        info.update({"power_limit": pl, "max_sm_clock": cmax, "sm_clock_idle": cnow})
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        info["power_limit"] = "unknown (nvidia-smi unavailable)"
    return info


def sm_clock_now():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def flash_kernel_ms(fn, calls=10):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            flush_l2()
            fn()
        torch.cuda.synchronize()
    us = [e.device_time_total for e in prof.key_averages() if "flash_attn_kernel" in e.key]
    return sum(us) / calls / 1e3 if us else float("nan")


def module(C=1280, heads=8, cross=None, seed=0):
    from vidtome_b200.skeleton import Attention
    torch.manual_seed(seed)
    return Attention(C, heads, C // heads, cross_attention_dim=cross).half().cuda().eval()


def bench_kd(name, B, L, iters):
    attn = module()
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn((B, L, 1280), generator=g, device="cuda").half()
    w_qkv, w_o, b_o = attention._packed_weights(attn, x)
    kd = lambda: ops.attention(x, w_qkv, w_o, b_o, attn.heads, attn.scale)  # noqa: E731
    torch_fwd = lambda: attn(x)  # noqa: E731
    with torch.no_grad():
        err = (kd().float() - torch_fwd().float()).abs().max().item()
        ts = alternate({"kd": kd, "torch": torch_fwd}, iters)
        fl = flash_kernel_ms(kd)
    print(json.dumps({"what": "kd", "shape": name, "B": B, "L": L, "C": 1280, "heads": 8, "kd_ms": summary(ts["kd"]),
                      "torch_ms": summary(ts["torch"]), "flash_ms": round(fl, 4),
                      "speedup": round(statistics.median(ts["torch"]) / statistics.median(ts["kd"]), 3),
                      "max_abs_diff": err, "sm_clock_after": sm_clock_now()}), flush=True)


def bench_xa(name, B, Lq, iters, Lk=77):
    attn = module(cross=768)
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn((B, Lq, 1280), generator=g, device="cuda").half()
    ctx = torch.randn((B, Lk, 768), generator=g, device="cuda").half()
    resid = torch.randn((B, Lq, 1280), generator=g, device="cuda").half()
    xa = lambda: attention.cross_attention_residual(attn, x, ctx, resid)  # noqa: E731
    torch_fwd = lambda: attn(x, encoder_hidden_states=ctx) + resid  # noqa: E731
    with torch.no_grad():
        err = (xa().float() - torch_fwd().float()).abs().max().item()
        ts = alternate({"xa": xa, "torch": torch_fwd}, iters)
        fl = flash_kernel_ms(xa)
    print(json.dumps({"what": "xa", "shape": name, "B": B, "Lq": Lq, "Lk": Lk, "C": 1280, "heads": 8,
                      "xa_ms": summary(ts["xa"]), "torch_ms": summary(ts["torch"]), "flash_ms": round(fl, 4),
                      "speedup": round(statistics.median(ts["torch"]) / statistics.median(ts["xa"]), 3),
                      "max_abs_diff": err, "sm_clock_after": sm_clock_now()}), flush=True)


def bench_step(max_downsample, iters, steps_per_sample=5):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton
    frames = 16
    g = torch.Generator(device="cuda").manual_seed(5)
    cond = torch.randn((2, 77, 768), generator=g, device="cuda").half()
    x0 = torch.randn((frames, 4, 64, 64), generator=g, device="cuda", dtype=torch.float16)
    arms = {}
    for limit in (128, 160):
        attention.MAX_HEAD_DIM = limit
        net = make_skeleton("sd15", hot_path_only=False, device="cuda")
        vidtome_b200.apply_patch(net, local_merge_ratio=0.9, batch_size=2, max_downsample=max_downsample)
        den = ChunkedDenoiser(net, n_timesteps=50, chunk_size=frames, cond=cond, cuda_graph=True)
        state = {"x": x0.clone(), "i": 0}
        for _ in range(3):                                   # two eager steps, then the capture
            state["x"] = den.step(state["x"], state["i"])
            state["i"] += 1
        assert den._graph is not None

        def run(den=den, state=state, limit=limit):
            attention.MAX_HEAD_DIM = limit
            for _ in range(steps_per_sample):
                state["x"] = den.step(state["x"], state["i"] % 40 + 3)
                state["i"] += 1
        arms[f"limit{limit}"] = run
    ts = alternate(arms, iters, warmup=1, flush=False)
    attention.MAX_HEAD_DIM = 128
    row = {"what": "step", "workload": "sd15 full, 16 frames 512x512, CFG 2", "max_downsample": max_downsample}
    for k, v in ts.items():
        per = [t / steps_per_sample for t in v]
        row[k + "_ms_per_step"] = summary(per)
        row[k + "_steps_per_s"] = round(1e3 / statistics.median(per), 2)
    row["sm_clock_after"] = sm_clock_now()
    print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=15)
    ap.add_argument("--no-step", action="store_true", help="kernel-level arms only")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wide_head_bench needs a CUDA device")
    print(json.dumps(device_info()), flush=True)
    bench_kd("ds4", 2, 641, args.iters)
    bench_kd("ds8", 2, 161, args.iters)
    bench_xa("ds4", 32, 256, args.iters)
    bench_xa("ds8", 32, 64, args.iters)
    if not args.no_step:
        bench_step(4, args.iters)
        bench_step(8, args.iters)


if __name__ == "__main__":
    main()
