"""LoRA-adapted generation at C2 (SD1.5 skeleton, 16 frames at 512x512, local merge ratio 0.9, CFG batch 2): the library
with LoRA against the same model with the library's attention and feed-forward switched off (the modules' own forward
for every LoRA-wrapped layer) and against the library without LoRA; plus the projection GEMMs with and without the
LoRA K tail, and (with --baseline-lib) the plain projections of this build against another build of the library.

Arms, per rank (adapters on every attention projection, and on both feed-forward layers in the full workload):
  "lib_lora"  — patched model with LoRA, library attention / cross-attention / feed-forward (the K tail);
  "off_lora"  — the same model with attention.ENABLED, patch.FUSE_CROSS_ATTENTION and patch.FUSE_FEED_FORWARD False;
  "lib_plain" — the patched model without LoRA.
Each timed sample is --iters UNet forwards bracketed by CUDA events; --rounds rounds alternate the arms and the medians
are reported.  "hot" is bench.py's hot workload (blocks without attn2 / ff); "full" adds cross-attention and the
feed-forward.  Projection timings: QKV (M = merged rows of ds1, N = 3C, K = C), GEGLU (M = frames x tokens, N = 8C,
K = C) and FF output (N = C, K = 4C, residual) at C = 320, each with the T launch included when R > 0.  One JSON line
goes to stdout with the card name and power limit read in the same run.

    python tools/lora_bench.py --workload full --ranks 8,32,128 --rounds 5
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from global_graph_bench import card  # noqa: E402

FRAMES, LATENT, BATCH = 16, 64, 2


def _events_ms(fn, iters: int) -> float:
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def _median(v):
    v = sorted(v)
    return v[len(v) // 2]


def models(workload: str, ranks, form: str):
    import copy

    import vidtome_b200
    from vidtome_b200.skeleton import add_lora, make_skeleton
    base = make_skeleton("sd15", hot_path_only=(workload == "hot"), device="cuda")
    nets = {0: base}
    for r in ranks:
        nets[r] = add_lora(copy.deepcopy(base), r, form, seed=r)
    for net in nets.values():
        vidtome_b200.apply_patch(net, local_merge_ratio=0.9, batch_size=BATCH)
    return nets


def forward_fn(net, lat, cond, library: bool):
    from vidtome_b200 import attention, patch

    def run():
        attention.ENABLED = patch.FUSE_CROSS_ATTENTION = patch.FUSE_FEED_FORWARD = library
        with torch.no_grad():
            net(lat, 0, encoder_hidden_states=cond)
    return run


def projection_timings(ranks, iters: int, rounds: int, baseline_lib):
    """Median ms of the projection GEMMs per rank (0 = the entry point without LoRA), and of the plain projections in
    this build and in `baseline_lib` (alternating)."""
    from vidtome_b200 import _lib, ops
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(1)
    Cc = 320
    shapes = {"qkv": (BATCH * 10241, 3 * Cc, Cc), "geglu": (BATCH * FRAMES * 4096, 8 * Cc, Cc),
              "ff_out": (BATCH * FRAMES * 4096, Cc, 4 * Cc)}
    stream = torch.cuda.current_stream().cuda_stream
    bufs = {}
    for name, (M, N, K) in shapes.items():
        a = torch.randn((M, K), generator=g, device="cuda").half()
        w = (torch.randn((N, K), generator=g, device="cuda") / K ** 0.5).half()
        b = torch.randn((N,), generator=g, device="cuda").half()
        d = torch.empty((M, N // 2 if name == "geglu" else N), dtype=torch.float16, device="cuda")
        resid = torch.randn((M, N), generator=g, device="cuda").half() if name == "ff_out" else None
        bufs[name] = (M, N, K, a, w, b, d, resid)

    def plain_call(L, name):
        M, N, K, a, w, b, d, resid = bufs[name]
        if name == "geglu":
            return lambda: L.vtm_linear_geglu_f16(a.data_ptr(), w.data_ptr(), b.data_ptr(), M, N, K, d.data_ptr(), N // 2,
                                                  stream)
        if name == "ff_out":
            return lambda: L.vtm_linear_residual_f16(a.data_ptr(), w.data_ptr(), b.data_ptr(), resid.data_ptr(), N, M, N,
                                                     K, d.data_ptr(), N, stream)
        return lambda: L.vtm_linear_f16(a.data_ptr(), w.data_ptr(), b.data_ptr(), M, N, K, d.data_ptr(), N, stream)

    def lora_call(name, R):
        M, N, K, a, w, b, d, resid = bufs[name]
        down = (torch.randn((R, K), generator=g, device="cuda") / K ** 0.5).half()
        up = (torch.randn((N, R), generator=g, device="cuda") * 0.1).half()
        desc = _lib.VtmLora(down.data_ptr(), up.data_ptr(), R)
        ws_bytes = lib.vtm_linear_lora_workspace_bytes(M, R)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
        keep = (down, up, ws, desc)
        if name == "geglu":
            def f():
                _lib.check(lib.vtm_linear_geglu_lora_f16(a.data_ptr(), w.data_ptr(), b.data_ptr(), C.byref(keep[3]), M,
                                                         N, K, d.data_ptr(), N // 2, ws.data_ptr(), ws_bytes, stream), "geglu")
        else:
            def f():
                _lib.check(lib.vtm_linear_lora_f16(a.data_ptr(), w.data_ptr(), b.data_ptr(), None if resid is None
                                                   else resid.data_ptr(), N, C.byref(keep[3]), M, N, K, d.data_ptr(), N,
                                                   ws.data_ptr(), ws_bytes, stream), "linear")
        return f

    calls = {(n, 0): plain_call(lib, n) for n in shapes}
    for n in shapes:
        for r in ranks:
            calls[(n, r)] = lora_call(n, r)
    base_calls = {}
    if baseline_lib:
        bl = C.CDLL(baseline_lib)
        for fname in ("vtm_linear_f16", "vtm_linear_geglu_f16", "vtm_linear_residual_f16"):
            fn = getattr(bl, fname)
            fn.restype, fn.argtypes = _lib.SIGNATURES[fname]
        base_calls = {n: plain_call(bl, n) for n in shapes}
    for fn in list(calls.values()) + list(base_calls.values()):
        _events_ms(fn, 3)
    samples = {k: [] for k in calls}
    ab = {n: {"this": [], "baseline": []} for n in base_calls}
    for i in range(rounds):
        for k, fn in calls.items():
            samples[k].append(_events_ms(fn, iters))
        for n, fn in base_calls.items():
            # the two builds alternate, and which of them goes first alternates from round to round
            order = (("baseline", fn), ("this", calls[(n, 0)]))
            for which, f in order if i % 2 == 0 else order[::-1]:
                ab[n][which].append(_events_ms(f, iters))
    proj = {n: {str(r): round(_median(samples[(n, r)]), 4) for r in [0] + list(ranks)} for n in shapes}
    spread = {n: {str(r): [round(min(samples[(n, r)]), 4), round(max(samples[(n, r)]), 4)] for r in [0] + list(ranks)}
              for n in shapes}
    plain_ab = {n: {k: {"median": round(_median(v), 4), "range": [round(min(v), 4), round(max(v), 4)]}
                    for k, v in d.items()} for n, d in ab.items()}
    return {"shapes_MNK": shapes, "ms": proj, "ms_range": spread, "plain_this_vs_baseline_ms": plain_ab or "not measured"}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", choices=("hot", "full"), default="full")
    ap.add_argument("--ranks", default="8,32,128")
    ap.add_argument("--form", choices=("peft", "diffusers"), default="peft")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3, help="UNet forwards per timed sample")
    ap.add_argument("--proj-iters", type=int, default=20, help="GEMM calls per timed projection sample")
    ap.add_argument("--baseline-lib", default=None, help="another build of libvidtome_b200.so for the plain A/B")
    ap.add_argument("--skip-model", action="store_true", help="projection timings only")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lora_bench.py needs a CUDA device")
    name, power = card()
    ranks = [int(r) for r in args.ranks.split(",") if r]
    line = {"tool": "lora_bench", "workload": args.workload, "form": args.form, "card": name, "power_limit": power,
            "frames": FRAMES, "latent": LATENT, "batch": BATCH, "local_ratio": 0.9, "ranks": ranks}
    if not args.skip_model:
        from vidtome_b200 import attention, patch
        nets = models(args.workload, ranks, args.form)
        g = torch.Generator(device="cuda").manual_seed(3)
        lat = torch.randn((BATCH * FRAMES, 4, LATENT, LATENT), generator=g, device="cuda").half()
        cond = None
        if args.workload == "full":
            cond = torch.randn((BATCH * FRAMES, 77, 768), generator=g, device="cuda").half()
        arms = {}
        for r in ranks:
            arms[f"lib_lora_r{r}"] = forward_fn(nets[r], lat, cond, True)
            arms[f"off_lora_r{r}"] = forward_fn(nets[r], lat, cond, False)
        arms["lib_plain"] = forward_fn(nets[0], lat, cond, True)
        saved = (attention.ENABLED, patch.FUSE_CROSS_ATTENTION, patch.FUSE_FEED_FORWARD)
        try:
            for fn in arms.values():
                _events_ms(fn, 1)
            times = {k: [] for k in arms}
            for _ in range(args.rounds):
                for k, fn in arms.items():
                    times[k].append(_events_ms(fn, args.iters))
        finally:
            attention.ENABLED, patch.FUSE_CROSS_ATTENTION, patch.FUSE_FEED_FORWARD = saved
        med = {k: round(_median(v), 3) for k, v in times.items()}
        line.update({"forward_ms_median": med, "forward_ms_range": {k: [round(min(v), 3), round(max(v), 3)]
                                                                    for k, v in times.items()},
                     "lib_lora_over_off_lora": {str(r): round(med[f"lib_lora_r{r}"] / med[f"off_lora_r{r}"], 3)
                                                for r in ranks},
                     "lib_lora_over_lib_plain": {str(r): round(med[f"lib_lora_r{r}"] / med["lib_plain"], 3)
                                                 for r in ranks}})
        del nets
        torch.cuda.empty_cache()
    line["projections"] = projection_timings(ranks, args.proj_iters, args.rounds, args.baseline_lib)
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
