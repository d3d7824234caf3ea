"""Steps per second per edit of K edits of one video in one denoising pass (ChunkedDenoiser(cond=[K, S, 77, D])) against
K separate single-prompt runs, with the graph memory each needs.

Workloads, 32 frames at 512x512 (latent 64), 4-frame chunks, local 0.9 + global 0.8 (global_rand 0.5), full blocks:
  dog   the reference's two-prompt config (configs/dog.yaml): the SD2.1 skeleton with PnP attention and conv injection
        (pnp_attn_t 0.5, pnp_f_t 0.8, `pnp_conv=True`), randomised chunks in "mix-4" order, from chunk_graphs=True;
        timed inside both injection windows, so that every timed step replays graphs of one phase
  c3    BASELINE config 3 on the SD1.5 skeleton with a [2, 77, 768] text context: fixed chunks in "mix-4" order,
        capture_global=True

Every arm (K = 1 and each count of --edits) drives its own skeleton built from the same seed, with the first K rows
of one cond and of one set of initial latents.  K separate runs cost K times the K = 1 arm's step time, so the K = 1
arm's steps/s is the per-edit rate of separate runs.  All arms first step --check-steps times from the same RNG state
(eager warm-up, captures, replays), and so does a single-prompt run of every edit k from its own cond row and initial
latents.  Reported: max |x_k - single_k| / max |single_k| for every edit k of every arm after those steps.
The skeleton's torch layers run on the whole K-edit batch here, as a user runs them, so small differences
are expected (tests/test_gpu_multi_edit.py holds them to the float64 step levels).  --rounds
timed rounds then alternate the arms, --steps steps each, timed with CUDA events.  Reported per arm: the median
steps/s with min and max, the same per edit, the speedup per edit over K = 1, and the bytes reserved by its graphs'
private memory pools.  One JSON line per workload goes to stdout, with the card's name, power limit and max SM clock
read in the same run.

    python tools/multi_edit_bench.py --workloads dog c3 --edits 2 4

--shard runs the edits split over the ranks of a torch.distributed job instead (ChunkedDenoiser(cond=[K, ...],
shard=True): rank r runs edits k % world == r).  Start it with torchrun, one rank per GPU; every rank builds two arms
per edit count K, the unsharded K-edit run and its sharded share of the edits, steps both --check-steps times from the
same RNG state (reporting max |x - unsharded| / max |unsharded| over its own edits), then times --rounds rounds of
--steps steps each, the ranks aligned by a barrier before every round.  Each rank prints one JSON line per workload and
K with its steps/s in both arms.  With one rank the two arms run the same K edits, so the line shows what the sharded
path costs on its own; the speed-up over N GPUs is that of N ranks' lines.

    torchrun --nproc-per-node 4 tools/multi_edit_bench.py --shard --workloads dog --edits 4
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from concurrent_chunks_bench import Chain, card, pool_bytes, timed  # noqa: E402

FRAMES, LATENT, N_STEPS = 32, 64, 50
WORKLOADS = ("dog", "c3")
MAX_EDITS = 4


def make(workload: str, K: int, edit: int = 0, shard: bool = False):
    """The arm of K edits (K = 1: the single-prompt run of edit `edit`); with `shard` this rank's share of K edits."""
    import vidtome_b200
    from vidtome_b200 import dist as vd
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton, pnp_attention_modules, pnp_conv_module
    torch.manual_seed(123)
    dog = workload == "dog"
    net = make_skeleton("sd21" if dog else "sd15", hot_path_only=False, device="cuda", pnp_conv=dog)
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=True, global_merge_ratio=0.8, global_rand=0.5,
                             batch_size=3 if dog else 2, align_batch=dog)
    vidtome_b200.update_patch(net, edits=len(vd.shard_edits(K)) if shard else K)
    gc = torch.Generator(device="cuda").manual_seed(5)
    cond = torch.randn((MAX_EDITS, 3 if dog else 2, 77, 1024 if dog else 768), generator=gc, device="cuda",
                       dtype=torch.float16)
    cond = cond[:K] if K > 1 else cond
    kw = dict(capture_global=True)
    if dog:
        sources = {}

        def source(t):
            if t not in sources:
                gs = torch.Generator(device="cuda").manual_seed(int(t))
                sources[t] = torch.randn((FRAMES, 4, LATENT, LATENT), generator=gs, device="cuda").half()
            return sources[t]
        kw = dict(chunk_graphs=True, randomize_chunks=True, source_latents=source, pnp_attn_t=0.5,
                  pnp_modules=pnp_attention_modules(net), pnp_f_t=0.8, pnp_conv_modules=[pnp_conv_module(net)])
    return ChunkedDenoiser(net, n_timesteps=N_STEPS, chunk_size=4, merge_global=True, chunk_ord="mix-4",
                           cond=cond if K > 1 else cond[edit], cuda_graph=True, graph_warmup=2, shard=shard, **kw)


def graph_pool_mib(den):
    graphs = [g.graph for g in den._chunk_graphs.values()] + ([den._graph.graph] if den._graph is not None else [])
    sizes = [pool_bytes(g) for g in graphs]
    return None if not sizes or None in sizes else round(sum(sizes) / 2 ** 20, 1)


def run(workload: str, edits, rounds: int, steps: int, check_steps: int):
    import numpy as np
    g = torch.Generator(device="cuda").manual_seed(123)
    x0 = torch.randn((MAX_EDITS, FRAMES, 4, LATENT, LATENT), generator=g, device="cuda", dtype=torch.float16)
    end = 25 if workload == "dog" else N_STEPS          # dog: inside both PnP injection windows
    arms = {}
    for K in [1] + list(edits):
        arms[K] = Chain(make(workload, K), x0[:K] if K > 1 else x0[0], end=end)
        torch.manual_seed(2024)
        np.random.seed(2024)
        for _ in range(check_steps):
            arms[K].step()
    singles = [arms[1].x]
    for k in range(1, max(edits)):                   # the single-prompt run of every further edit, checked only
        ch = Chain(make(workload, 1, edit=k), x0[k], end=end)
        torch.manual_seed(2024)
        np.random.seed(2024)
        for _ in range(check_steps):
            ch.step()
        singles.append(ch.x)
        del ch
    torch.cuda.synchronize()
    ref = arms[1].x
    diff = {str(K): [round(float((ch.x[k].float() - singles[k].float()).abs().max()
                                 / singles[k].float().abs().max()), 6) for k in range(K)]
            for K, ch in arms.items() if K > 1}
    rates = {K: [] for K in arms}
    for _ in range(rounds):
        for K, ch in arms.items():
            rates[K].append(timed(ch, steps))
    out = {}
    for K, ch in arms.items():
        r = sorted(rates[K])
        out[str(K)] = {"steps_per_s_median": round(r[len(r) // 2], 2), "min": round(r[0], 2),
                       "max": round(r[-1], 2), "edit_steps_per_s_median": round(K * r[len(r) // 2], 2),
                       "edit_min": round(K * r[0], 2), "edit_max": round(K * r[-1], 2),
                       "graph_pool_MiB": graph_pool_mib(ch.den)}
    base = out["1"]["edit_steps_per_s_median"]
    for K in edits:
        out[str(K)]["speedup_per_edit_median"] = round(out[str(K)]["edit_steps_per_s_median"] / base, 3)
    return {"edit_rel_diff_to_single_run": diff, "finite": bool(torch.isfinite(ref).all()), "arms": out,
            "max_allocated_GiB": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}


def run_shard(workload: str, K: int, rounds: int, steps: int, check_steps: int):
    """This rank's steps/s of the unsharded K-edit run and of its share of the sharded one (see the module's doc)."""
    import numpy as np
    import torch.distributed as dist
    from vidtome_b200 import dist as vd
    rows = vd.shard_edits(K)
    g = torch.Generator(device="cuda").manual_seed(123)
    x0 = torch.randn((K, FRAMES, 4, LATENT, LATENT), generator=g, device="cuda", dtype=torch.float16)
    end = 25 if workload == "dog" else N_STEPS
    arms = {"unsharded": Chain(make(workload, K), x0, end=end),
            "sharded": Chain(make(workload, K, shard=True), x0[rows], end=end)}
    for ch in arms.values():
        torch.manual_seed(2024)
        np.random.seed(2024)
        for _ in range(check_steps):
            ch.step()
    torch.cuda.synchronize()
    ref = arms["unsharded"].x[rows].float()
    diff = round(float((arms["sharded"].x.float() - ref).abs().max() / ref.abs().max()), 6)
    rates = {name: [] for name in arms}
    for _ in range(rounds):
        for name, ch in arms.items():
            dist.barrier()
            rates[name].append(timed(ch, steps))
    out = {"rank": vd.rank(), "world": vd.world(), "edits": K, "rank_edits": rows,
           "rel_diff_to_unsharded": diff, "finite": bool(torch.isfinite(arms["sharded"].x).all())}
    for name, r in rates.items():
        r = sorted(r)
        out[name] = {"steps_per_s_median": round(r[len(r) // 2], 2), "min": round(r[0], 2), "max": round(r[-1], 2)}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workloads", nargs="+", choices=WORKLOADS, default=list(WORKLOADS))
    ap.add_argument("--edits", nargs="+", type=int, default=[2, 4], help="edit counts set against one edit")
    ap.add_argument("--steps", type=int, default=8, help="timed steps per round and arm")
    ap.add_argument("--rounds", type=int, default=5, help="rounds alternating the arms")
    ap.add_argument("--check-steps", type=int, default=6,
                    help="steps from the same RNG state before the comparison (2 eager + captures + replays)")
    ap.add_argument("--shard", action="store_true", help="split the edits over the ranks of a torchrun job")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multi_edit_bench.py needs a CUDA device")
    if any(not 1 < K <= MAX_EDITS for K in args.edits):
        raise SystemExit(f"--edits: counts from 2 to {MAX_EDITS}")
    name, power, clock = card()
    if args.shard:
        import torch.distributed as dist
        local = int(os.environ.get("LOCAL_RANK", 0))
        torch.cuda.set_device(local)
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29511")
        dist.init_process_group("nccl", rank=int(os.environ.get("RANK", 0)),
                                world_size=int(os.environ.get("WORLD_SIZE", 1)),
                                device_id=torch.device("cuda", local))
        try:
            for w in args.workloads:
                for K in args.edits:
                    line = {"tool": "multi_edit_bench", "leg": "shard", "workload": w, "card": name,
                            "power_limit": power, "max_sm_clock": clock, "frames": FRAMES, "latent": LATENT,
                            "steps_per_round": args.steps, "rounds": args.rounds}
                    line.update(run_shard(w, K, args.rounds, args.steps, args.check_steps))
                    print(json.dumps(line), flush=True)
                    torch.cuda.empty_cache()
        finally:
            dist.destroy_process_group()
        return
    for w in args.workloads:
        torch.cuda.reset_peak_memory_stats()
        line = {"tool": "multi_edit_bench", "workload": w, "card": name, "power_limit": power,
                "max_sm_clock": clock, "frames": FRAMES, "latent": LATENT, "steps_per_round": args.steps,
                "rounds": args.rounds}
        line.update(run(w, args.edits, args.rounds, args.steps, args.check_steps))
        print(json.dumps(line), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
