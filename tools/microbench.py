"""Kernel microbench (BASELINE.json configs[4]): sim+argmax sweep and the HBM-bound row kernels.

Prints one JSON line per (kernel, shape): CUDA-event time (median of `--iters` after warm-up, L2 flushed
between iterations by writing a 256 MiB buffer), achieved TFLOP/s or GB/s and the fraction of the measured
peak in MEASURED_PEAKS.json (else the H100 SXM data-sheet figures).  `--quick` runs only the BASELINE config-2 shapes;
`--ka-only` only the KA (similarity + arg-max) shapes; `--kd-only` only the two KD (merged-token self-attention)
shapes.

The KA line also gives `l2_fill_MB`: the operand bytes the kernel's tiling loads into shared memory (computed from the
shapes, the tile sizes and the work split of csrc/sim_argmax.cu), and `l2_fill_TBs`, those bytes over the kernel time.

The KD line also gives the flash-attention kernel's own time (`flash_ms`, mean over a torch.profiler pass that follows
the timed window, with L2 flushed before every call as in the timed window) and `flash_over_mufu_floor`: that time over
the least time the SM's exponential units need for the B·H·L² ex2 of the softmax, at 16 ex2 per clock per SM and the SM
clock read from nvidia-smi right after the timed window (`sm_clock_mhz`; the device's maximum clock when nvidia-smi is
not available).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vidtome_b200 import ops  # noqa: E402
from vidtome_b200._lib import VtmSplit  # noqa: E402


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d["hbm_gbs"], d["bf16_tflops"], "measured"
    return 3350.0, 989.0, "fallback"


_flush = None


def flush_l2():
    global _flush
    if _flush is None:
        _flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    _flush.fill_(1)


def time_ms(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        flush_l2()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def time_rotating_ms(fns, reps=12, warmup=3):
    """Device time per call for short kernels: `fns` are equivalent closures over DIFFERENT buffers (together larger
    than L2), launched back to back `reps` times round-robin between two events, so that neither host launch
    latency nor L2 residency of the previous call's data enters the figure."""
    for _ in range(warmup):
        for f in fns:
            f()
    ts = []
    for _ in range(5):
        flush_l2()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        for i in range(reps):
            fns[i % len(fns)]()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e) / reps)
    ts.sort()
    return ts[len(ts) // 2]


def ka_l2_fill_bytes(B, Ns, Nd, C, sms):
    """Operand bytes KA moves from L2 (or HBM) into shared memory, mirroring ka::Items / ka::Layout in sim_argmax.cu:
    128 x 256 tiles, 64-column K chunks, the src block loaded once per work item when it fits in shared memory next to
    three 256 x 64 dst stages (else once per tile), each dst tile once per CTA."""
    BM, BN, BK, target = 128, 256, 64, 8
    kp = -(-C // BK) * BK
    m_tiles, n_tiles = -(-Ns // BM), -(-Nd // BN)
    resident = kp // BK <= 8 and 1024 + 224 + BM * kp * 2 + 3 * BN * BK * 2 <= 227 * 1024
    s = 1
    while m_tiles * B * s < target * sms and s * 2 <= n_tiles:
        s *= 2
    tps = -(-n_tiles // s)
    n_splits = -(-n_tiles // tps)
    a_loads = m_tiles * B * (n_splits if resident else n_tiles)
    return 2.0 * kp * (a_loads * BM + m_tiles * B * n_tiles * BN)


def bench_sim_argmax(B, Ns, Nd, C, align, iters):
    hbm, tf, src = peaks()
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.randn((B, Ns, C), generator=g, device="cuda").half()
    b = torch.randn((B, Nd, C), generator=g, device="cuda").half()
    med, best = time_ms(lambda: ops.sim_argmax(a, b, align), iters)
    flops = 2.0 * B * Ns * Nd * C
    byts = 2.0 * B * (Ns + Nd) * C + 8.0 * (1 if align else B) * Ns
    fill = ka_l2_fill_bytes(B, Ns, Nd, C, torch.cuda.get_device_properties(0).multi_processor_count)
    print(json.dumps({"kernel": "KA sim_argmax", "B": B, "Ns": Ns, "Nd": Nd, "C": C,
                      "align": align, "ms": round(med, 4), "ms_best": round(best, 4),
                      "tflops": round(flops / med / 1e9, 1), "frac_tensor_peak": round(flops / med / 1e9 / tf, 3),
                      "eff_GBs": round(byts / med / 1e6, 1), "l2_fill_MB": round(fill / 1e6, 1),
                      "l2_fill_TBs": round(fill / med / 1e9, 2), "peak": src}), flush=True)


def bench_rows(B, F, T, C, iters):
    hbm, tf, src = peaks()
    N = F * T
    g = torch.Generator(device="cuda").manual_seed(0)
    R = 4   # replicas: 4 x (84 MB in + 84 MB out) >> 50 MB L2
    xs = [torch.randn((B, N, C), generator=g, device="cuda").half() for _ in range(R)]
    sp = VtmSplit.local(N, 0, F, 4, 1)
    med = time_rotating_ms([(lambda x=x: ops.normalize_split(x, None, sp)) for x in xs])
    byts = 4.0 * B * N * C
    print(json.dumps({"kernel": "K0 normalize_split", "B": B, "N": N, "C": C, "ms": round(med, 4),
                      "GBs": round(byts / med / 1e6, 1), "frac_hbm": round(byts / med / 1e6 / hbm, 3), "peak": src}), flush=True)
    ln = torch.nn.LayerNorm(C).cuda().half()
    med = time_rotating_ms([(lambda x=x: ops.normalize_split(x, None, sp, ln=(ln.weight.data, ln.bias.data, ln.eps))) for x in xs])
    print(json.dumps({"kernel": "K0 normalize_split + fused LayerNorm", "B": B, "N": N, "C": C, "ms": round(med, 4),
                      "GBs": round(byts / med / 1e6, 1), "frac_hbm": round(byts / med / 1e6 / hbm, 3), "peak": src}), flush=True)
    L = int(0.156 * N)
    mus = [torch.randint(0, N, (B, L), device="cuda", dtype=torch.int32) for _ in range(R)]
    med = time_rotating_ms([(lambda x=x, m=m: ops.gather_rows(x, m)) for x, m in zip(xs, mus)])
    byts = 4.0 * B * L * C + 4.0 * B * L
    print(json.dumps({"kernel": "KC gather_rows", "B": B, "L": L, "C": C, "ms": round(med, 4),
                      "GBs": round(byts / med / 1e6, 1), "frac_hbm": round(byts / med / 1e6 / hbm, 3), "peak": src}), flush=True)
    ys = [ops.gather_rows(x, m) for x, m in zip(xs, mus)]
    pis = [torch.randint(0, L, (B, N), device="cuda", dtype=torch.int32) for _ in range(R)]
    med = time_rotating_ms([(lambda y=y, p=p, x=x: ops.unmerge_add(y, p, x)) for y, p, x in zip(ys, pis, xs)])
    byts = 2.0 * B * (L + 2 * N) * C + 4.0 * B * N
    print(json.dumps({"kernel": "KE unmerge_add", "B": B, "N": N, "L": L, "C": C, "ms": round(med, 4),
                      "GBs": round(byts / med / 1e6, 1), "frac_hbm": round(byts / med / 1e6 / hbm, 3), "peak": src}), flush=True)
    Ns = 3 * N // 4
    kks = [torch.randint(0, 2 ** 40, (B, Ns), device="cuda", dtype=torch.int64) for _ in range(2)]
    med = time_rotating_ms([(lambda k=k: ops.topr_sort(k)) for k in kks])
    print(json.dumps({"kernel": "KB1 topr_sort", "Bp": B, "Ns": Ns, "ms": round(med, 4)}), flush=True)


def bench_linear(M, N, K, iters):
    hbm, tf, src = peaks()
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.randn((M, K), generator=g, device="cuda").half()
    w = torch.randn((N, K), generator=g, device="cuda").half()
    med, _ = time_ms(lambda: ops.linear(a, w), iters)
    med_t, _ = time_ms(lambda: torch.nn.functional.linear(a, w), iters)
    flops = 2.0 * M * N * K
    print(json.dumps({"kernel": "linear_f16", "M": M, "N": N, "K": K, "ms": round(med, 4),
                      "tflops": round(flops / med / 1e9, 1), "cublas_ms": round(med_t, 4),
                      "cublas_tflops": round(flops / med_t / 1e9, 1)}), flush=True)


def sm_clock_mhz():
    """Current SM clock of device 0 from nvidia-smi (read right after a timed window, i.e. the clock under load), else
    the device's maximum SM clock."""
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0]), "nvidia-smi"
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return torch.cuda.get_device_properties(0).clock_rate / 1e3, "max"


def flash_kernel_ms(fn, calls=10):
    """Mean device time per call of the flash-attention kernel over `calls` calls of fn, from torch.profiler, with L2
    flushed before every call as in time_ms."""
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


def bench_attention(B, L, C, heads, iters, kernel=False):
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((B, L, C), generator=g, device="cuda").half()
    ws = [(torch.randn((C, C), generator=g, device="cuda") / C ** 0.5).half() for _ in range(4)]
    wqkv = torch.cat(ws[:3], 0).contiguous()
    bo = torch.zeros(C, device="cuda").half()
    d = C // heads
    kd = lambda: ops.attention(x, wqkv, ws[3], bo, heads, d ** -0.5)  # noqa: E731
    med, _ = time_ms(kd, iters)
    clock, clock_src = sm_clock_mhz() if kernel else (None, None)

    def sdpa():
        q, k, v = [torch.nn.functional.linear(x, w).view(B, L, heads, d).transpose(1, 2) for w in ws[:3]]
        o = torch.nn.functional.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, L, C)
        return torch.nn.functional.linear(o, ws[3], bo)
    med_t, _ = time_ms(sdpa, iters)
    flops = 4.0 * B * L * L * C + 8.0 * B * L * C * C
    row = {"kernel": "KD attention (qkv+flash+out)", "B": B, "L": L, "C": C, "heads": heads,
           "ms": round(med, 4), "tflops": round(flops / med / 1e9, 1), "torch_sdpa_path_ms": round(med_t, 4),
           "speedup_vs_torch": round(med_t / med, 2)}
    if kernel:
        fl = flash_kernel_ms(kd)
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        mufu_ms = B * heads * float(L) * L / (16.0 * sms * clock * 1e3)
        row.update({"flash_ms": round(fl, 4), "sm_clock_mhz": clock, "sm_clock_src": clock_src,
                    "mufu_floor_ms": round(mufu_ms, 4), "flash_over_mufu_floor": round(fl / mufu_ms, 2)})
    print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--ka-only", action="store_true")
    ap.add_argument("--kd-only", action="store_true")
    args = ap.parse_args()
    torch.cuda.init()
    if args.kd_only:
        from vidtome_b200._lib import LIB_PATH
        print(json.dumps({"device": torch.cuda.get_device_name(0), "lib": LIB_PATH}), flush=True)
        bench_attention(2, 10241, 320, 8, args.iters, kernel=True)
        bench_attention(2, 2561, 640, 8, args.iters, kernel=True)
        return
    # BASELINE config 2 shapes (SURVEY App. B): ds1 level 1/2, ds2 level 1/2
    for (Ns, Nd, C) in [(49152, 16384, 320), (12288, 9012, 320), (12288, 4096, 640), (3072, 2253, 640)]:
        bench_sim_argmax(2, Ns, Nd, C, False, args.iters)
    bench_sim_argmax(2, 49152, 16384, 320, True, args.iters)
    if args.ka_only:
        return
    bench_rows(2, 16, 4096, 320, args.iters)
    bench_rows(2, 16, 1024, 640, args.iters)
    bench_attention(2, 10241, 320, 8, args.iters)
    bench_attention(2, 2561, 640, 8, args.iters)
    bench_linear(20482, 960, 320, args.iters)
    bench_linear(5122, 1920, 640, args.iters)
    if args.quick:
        return
    for N in (4096, 8192, 16384, 32768, 65536):
        for C in (320, 640, 1280):
            for B in (1, 2):
                bench_sim_argmax(B, 3 * N // 4, N // 4, C, False, args.iters)
            bench_sim_argmax(2, 3 * N // 4, N // 4, C, True, args.iters)


if __name__ == "__main__":
    main()
