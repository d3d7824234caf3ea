"""Row kernels K0 (normalise + split, with and without the fused LayerNorm) and KC (merge gather, same), and KE for
comparison, at the level shapes of bench.py's headline step; plus a per-kernel breakdown of that step's device time.

    python tools/row_kernel_bench.py [--libs OLD.so NEW.so] [--rounds 2] [--profile] [--out DIR]

`--libs`: time each library in its own process (VIDTOME_B200_LIB), alternating between them `--rounds` times, so two
builds are compared in one session on the same card; without it the library of this tree is timed.  Each line gives
the algorithmic bytes (every row read once and written once, plus the map) over the kernel's device time per launch
(torch.profiler), and a SHA-256 digest of the kernel's outputs on seeded inputs, so that two builds can also be checked
for bit-identical results.
`--profile`: a torch.profiler pass (CUDA activities) over replays of the headline step
(ChunkedDenoiser(cuda_graph=True), SD1.5 skeleton, 16 frames, ratio 0.9), with the device time per step grouped by
kernel family.  The card's name, power limit and SM clock are printed first and last.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B = 2
# (name, N0 level-0 rows per sample, C, level-2 rows per sample, level-2 carried tokens, merged length)
BLOCKS = [("ds1", 65536, 320, 21300, 4916, 10241), ("ds2", 16384, 640, 5325, 1229, 2561)]
F, STRIDE, RANDF = 16, 4, 1
L2_BYTES = 50 << 20


def card():
    import torch
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        smi = r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        smi = "nvidia-smi not available"
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q + ": " + smi}


def digest(*ts):
    import torch
    h = hashlib.sha256()
    for t in ts:
        h.update(t.contiguous().view(-1).view(torch.uint8).cpu().numpy().tobytes())
    return h.hexdigest()[:16]


def kernel_ms(fns, kernel, reps=24):
    """Device time per launch of `kernel` (a substring of its name), from torch.profiler: the closures (over different
    buffers, together larger than L2) launched back to back round-robin.  The kernel's own duration, so host overhead
    between the short launches does not enter it."""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    for f in fns:
        f()
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(reps):
            fns[i % len(fns)]()
        torch.cuda.synchronize()
    evs = [e for e in prof.key_averages() if kernel in e.key]
    n = sum(e.count for e in evs)
    if n < reps // 2:   # the profiler may miss the first launch or two of a window
        raise RuntimeError(f"expected {reps} launches of {kernel}, the profile has {n}")
    return sum(e.device_time_total for e in evs) / n / 1e3


def replicas(nbytes):
    return max(2, min(8, -(-4 * L2_BYTES // max(nbytes, 1))))


def worker():
    import torch
    from vidtome_b200 import ops
    from vidtome_b200._lib import LIB_PATH, VtmSplit
    torch.cuda.init()
    lib = os.path.basename(os.path.dirname(LIB_PATH)) + "/" + os.path.basename(LIB_PATH)
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, N0, C, L2, unm2, M in BLOCKS:
        T = N0 // F
        ln_mod = torch.nn.LayerNorm(C).cuda().half()
        with torch.no_grad():
            ln_mod.weight.copy_(1 + 0.1 * torch.randn(C, generator=g, device="cuda"))
            ln_mod.bias.copy_(0.1 * torch.randn(C, generator=g, device="cuda"))
        ln = (ln_mod.weight.data, ln_mod.bias.data, ln_mod.eps)
        R = replicas(2 * B * N0 * C)
        xs = [(torch.randn((B, N0, C), generator=g, device="cuda") * 3 + 0.5).half() for _ in range(R)]
        # level 2 reads the level-0 table through a row map (per sample, or one map for all under align_batch)
        maps = [torch.stack([torch.randperm(N0, generator=g, device="cuda")[:L2] for _ in range(B)]).int()
                for _ in range(R)]
        levels = [("L1", VtmSplit.local(N0, 0, F, STRIDE, RANDF), None, N0),
                  ("L2", VtmSplit.local(L2, unm2, (L2 - unm2) // T, STRIDE, RANDF), maps, L2)]
        for lvl, sp, mp, rows in levels:
            for use_ln in (False, True):
                for align in ((False, True) if mp is not None else (False,)):
                    def call(i, sp=sp, mp=mp, use_ln=use_ln, align=align):
                        m = None if mp is None else (mp[i][:1] if align else mp[i])
                        return ops.normalize_split(xs[i], m, sp, ln if use_ln else None)
                    byts = 4.0 * B * rows * C + (4.0 * B * rows if mp is not None else 0.0)
                    ms = kernel_ms([(lambda i=i: call(i)) for i in range(R)], "normalize_split_kernel")
                    print(json.dumps({"lib": lib, "kernel": "K0", "shape": f"{name} {lvl}", "B": B, "rows": rows,
                                      "C": C, "ln": use_ln, "align_batch": align, "ms": round(ms, 4),
                                      "GBs": round(byts / ms / 1e6, 1), "digest": digest(*call(0))}), flush=True)
        mus = [torch.stack([torch.randperm(N0, generator=g, device="cuda")[:M] for _ in range(B)]).int()
               for _ in range(R)]
        for use_ln in (True, False):
            def kc(i, use_ln=use_ln):
                return ops.gather_rows(xs[i], mus[i], ln=ln if use_ln else None)
            byts = 4.0 * B * M * C + 4.0 * B * M
            ms = kernel_ms([(lambda i=i: kc(i)) for i in range(R)], "gather_rows_kernel")
            print(json.dumps({"lib": lib, "kernel": "KC", "shape": f"{name} merged", "B": B, "rows": M, "C": C,
                              "ln": use_ln, "ms": round(ms, 4), "GBs": round(byts / ms / 1e6, 1),
                              "digest": digest(kc(0))}), flush=True)
        ys = [ops.gather_rows(xs[i], mus[i]) for i in range(R)]
        pis = [torch.randint(0, M, (B, N0), generator=g, device="cuda", dtype=torch.int32) for _ in range(R)]

        def ke(i):
            return ops.unmerge_add(ys[i], pis[i], xs[i])
        byts = 2.0 * B * (M + 2 * N0) * C + 4.0 * B * N0
        ms = kernel_ms([(lambda i=i: ke(i)) for i in range(R)], "gather_rows_kernel")
        print(json.dumps({"lib": lib, "kernel": "KE", "shape": f"{name} unmerge", "B": B, "rows": N0, "C": C,
                          "ms": round(ms, 4), "GBs": round(byts / ms / 1e6, 1), "digest": digest(ke(0))}), flush=True)
        del xs, maps, mus, ys, pis
        torch.cuda.empty_cache()


GROUPS = [("KA", ("sim_argmax", "ArgmaxEpi")), ("flash", ("flash_attn",)), ("K0", ("normalize_split",)),
          ("KE", ("gather_rows_kernel<(int)8, (int)5, (bool)1", "gather_rows_kernel<(int)16, (int)5, (bool)1",
                  "gather_rows_kernel<8, 5, true", "gather_rows_kernel<16, 5, true")),
          ("KC", ("gather_rows",)), ("KB1", ("radix", "topr")), ("projection GEMMs", ("gemm_kernel",)),
          ("memset", ("memset", "Memset")), ("library, other", ("vtm::",))]


def group_of(name):
    for g, keys in GROUPS:
        if any(k in name for k in keys):
            return g
    return "torch / other"


def profile(out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile

    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton
    sys.path.insert(0, ROOT)
    torch.manual_seed(123)
    dev = torch.device("cuda", 0)
    net = make_skeleton("sd15", hot_path_only=True, device=dev)
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, batch_size=2, merge_global=False)
    den = ChunkedDenoiser(net, n_timesteps=50, chunk_size=16, cuda_graph=True)
    g = torch.Generator(device=dev).manual_seed(123)
    x = torch.randn((16, 4, 64, 64), generator=g, device=dev, dtype=torch.float16)
    for i in range(8):
        x = den.step(x, i)
    torch.cuda.synchronize()
    steps = 5
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(steps):
        x = den.step(x, i)
    e.record()
    torch.cuda.synchronize()
    step_ms = s.elapsed_time(e) / steps
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(steps):
            x = den.step(x, i)
        torch.cuda.synchronize()
    per_kernel = {}
    for ev in prof.key_averages():
        t = ev.device_time_total
        if t > 0:
            per_kernel[ev.key] = per_kernel.get(ev.key, 0.0) + t / steps / 1e3
    groups = {}
    for k, ms in per_kernel.items():
        grp = group_of(k)
        groups[grp] = groups.get(grp, 0.0) + ms
    total = sum(groups.values())
    by_time = sorted(groups.items(), key=lambda kv: -kv[1])
    print(json.dumps({"profile": "headline step, cuda_graph replay", "step_ms_unprofiled": round(step_ms, 3),
                      "kernel_ms_per_step": round(total, 3),
                      "groups_ms_per_step": {k: round(v, 3) for k, v in by_time}}), flush=True)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "profile_kernels.json"), "w") as f:
            json.dump({k: round(v, 4) for k, v in sorted(per_kernel.items(), key=lambda kv: -kv[1])}, f, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", nargs="+", default=None)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="directory for the profile's per-kernel table")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        worker()
        return
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("row_kernel_bench.py needs a CUDA device")
    print(json.dumps(card()), flush=True)
    if args.profile:
        profile(args.out)
    libs = args.libs or [None]
    for _ in range(args.rounds):
        for lib in libs:
            env = dict(os.environ)
            if lib:
                env["VIDTOME_B200_LIB"] = os.path.abspath(lib)
            subprocess.run([sys.executable, os.path.abspath(__file__), "--worker"], env=env, check=True)
    print(json.dumps(card()), flush=True)


if __name__ == "__main__":
    main()
