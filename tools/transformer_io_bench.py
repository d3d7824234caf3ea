"""Measures the Transformer2DModel entry / exit path of the library against the stand-in's torch forward.

(a) per wrapper shape of SD1.5 at 512 x 512 and SD2.1 at 768 x 768 (16 frames x CFG 2 = 32 items), both projection
    forms: entry (GroupNorm -> projected tokens) and exit (tokens -> NCHW + residual), library against torch, the arms
    alternated call by call with the L2 flushed before each, CUDA events, median and min-max; plus the achieved bytes/s
    of the two GroupNorm kernels against their algorithmic bytes;
(b) the whole step on make_skeleton("sd15", hot_path_only=False, transformer_io="conv") under
    ChunkedDenoiser(cuda_graph=True), patch.FUSE_TRANSFORMER_IO on against off on two identical pipelines, alternated.
The default path (bench.py's headline, which has no wrappers) is compared between two builds by running bench.py with
VIDTOME_B200_LIB pointing at each.  Prints the device name, power limit and clocks it ran under; changes nothing.

    python tools/transformer_io_bench.py [--reps 15] [--steps 6] [--skip-step]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

ITEMS = 32
SHAPES = [("sd15-512", "conv", 320, 64), ("sd15-512", "conv", 640, 32), ("sd15-512", "conv", 1280, 16),
          ("sd15-512", "conv", 1280, 8), ("sd21-768", "linear", 320, 96), ("sd21-768", "linear", 640, 48),
          ("sd21-768", "linear", 1280, 24), ("sd21-768", "linear", 1280, 12)]


def device_report():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = "nvidia-smi unavailable"
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": f"{q}: {out}"}


def timed(fns, reps, flush):
    """Alternates the callables call by call; per callable the list of times in ms."""
    times = [[] for _ in fns]
    for r in range(reps + 2):
        for k, fn in enumerate(fns):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            if r >= 2:                       # two warm-up rounds per shape
                times[k].append(a.elapsed_time(b))
    return times


def summary(ts):
    return {"median_ms": round(statistics.median(ts), 4), "min_ms": round(min(ts), 4), "max_ms": round(max(ts), 4),
            "n": len(ts)}


def per_shape(reps):
    from vidtome_b200 import ops
    from vidtome_b200.skeleton import Transformer2DModel
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")           # larger than the 50 MB L2
    rows = []
    for name, form, C, side in SHAPES:
        HW = side * side
        torch.manual_seed(0)
        m = Transformer2DModel(C, torch.nn.Identity(), use_linear_projection=form == "linear").cuda().half().eval()
        x = torch.randn(ITEMS, C, side, side, device="cuda").half()
        tok = torch.randn(ITEMS, HW, C, device="cuda").half()
        gn = (m.norm.weight, m.norm.bias, m.norm.eps, m.norm.num_groups)
        w_in, w_out = m.proj_in.weight.view(C, C), m.proj_out.weight.view(C, C)

        def lib_entry():
            return ops.linear(ops.group_norm_tokens(x, gn).view(-1, C), w_in, m.proj_in.bias)

        def torch_entry():
            h = m.norm(x)
            if form == "conv":
                return m.proj_in(h).permute(0, 2, 3, 1).reshape(ITEMS, HW, C)
            return m.proj_in(h.permute(0, 2, 3, 1).reshape(ITEMS, HW, C))

        def lib_exit():
            return ops.linear_nchw_residual(tok.view(-1, C), w_out, m.proj_out.bias, x, (side, side))

        def torch_exit():
            if form == "conv":
                return m.proj_out(tok.reshape(ITEMS, side, side, C).permute(0, 3, 1, 2).contiguous()) + x
            return m.proj_out(tok).reshape(ITEMS, side, side, C).permute(0, 3, 1, 2).contiguous() + x

        def stats_only():
            return ops.group_norm_stats(x, 32, 1e-6)
        st = stats_only()
        y = torch.empty(ITEMS, HW, C, device="cuda", dtype=torch.float16)
        from vidtome_b200 import _lib
        lib = _lib.load()

        def tokens_only():
            _lib.check(lib.vtm_group_norm_tokens_f16(x.data_ptr(), st.data_ptr(), gn[0].data_ptr(), gn[1].data_ptr(),
                                                     ITEMS, C, HW, 32, y.data_ptr(), ops._stream()), "tokens")
        with torch.no_grad():
            t = timed([lib_entry, torch_entry, lib_exit, torch_exit, stats_only, tokens_only], reps, flush)
        nbytes = 2.0 * ITEMS * C * HW
        row = {"model": name, "form": form, "C": C, "HW": HW, "activation_MB": round(nbytes / 1e6, 2),
               "entry_lib": summary(t[0]), "entry_torch": summary(t[1]), "exit_lib": summary(t[2]),
               "exit_torch": summary(t[3]), "stats": summary(t[4]), "tokens": summary(t[5]),
               "stats_GBps": round(nbytes / statistics.median(t[4]) / 1e6, 1),
               "tokens_GBps": round(2 * nbytes / statistics.median(t[5]) / 1e6, 1)}
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def whole_step(reps, steps):
    import numpy as np
    import vidtome_b200
    from vidtome_b200 import patch
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton
    frames, size = 16, 64
    dens = []
    for on in (True, False):
        net = make_skeleton("sd15", hot_path_only=False, device="cuda", transformer_io="conv")
        vidtome_b200.apply_patch(net, local_merge_ratio=0.9, batch_size=2)
        g = torch.Generator(device="cuda").manual_seed(5)
        cond = torch.randn((2, 77, 768), generator=g, device="cuda").half()
        den = ChunkedDenoiser(net, n_timesteps=50, chunk_size=16, chunk_ord="mix-4", cond=cond, cuda_graph=True,
                              graph_warmup=1)
        x = torch.randn((frames, 4, size, size), generator=g, device="cuda", dtype=torch.float16)
        dens.append([den, x, on, 0])
    times = {True: [], False: []}
    torch.manual_seed(1)
    np.random.seed(1)
    for r in range(reps + 3):
        for d in dens:
            den, x, on, i = d
            patch.FUSE_TRANSFORMER_IO = on          # read while the step is captured (the first steps), not at replay
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(steps):
                x = den.step(x, i % 50)
                i += 1
            b.record()
            torch.cuda.synchronize()
            d[1], d[3] = x, i
            if r >= 3:
                times[on].append(a.elapsed_time(b) / steps)
    patch.FUSE_TRANSFORMER_IO = True
    row = {"whole_step_ms_per_step": {"fused_on": summary(times[True]), "fused_off": summary(times[False])},
           "frames": frames, "latent": size, "steps_per_sample": steps}
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--skip-step", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("transformer_io_bench: needs a CUDA device (nothing is measured without one)")
    print(json.dumps(device_report()), flush=True)
    per_shape(args.reps)
    if not args.skip_step:
        whole_step(args.reps, args.steps)


if __name__ == "__main__":
    main()
