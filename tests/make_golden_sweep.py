"""Generate tests/golden/sweep_*.npz: the reference's compute_merge (vidtome/patch.py:14-91) across its argument space.

Run in the build container only (`python tests/make_golden_sweep.py`), as tests/make_golden.py: it imports the
reference from its tree, runs `vidtome.patch.compute_merge` on the CPU over a chain of chunks on ONE module (so the
global-token recurrence of patch.py:59-82 runs), and stores per chunk the input x{i}, every draw (randint{i}, rand{i}),
the merged tokens, back = u(merged) and module.global_tokens, in make_golden's compute_merge format.  Where the
reference raises, refused{i} holds the exception's type name and the chain stops; where it would loop forever
(target_stride 1 on several frames: every frame is dst, patch.py:44 never ends) refused{i} is "nonterminating".

Tokens are the exact family (make_golden.exact_video_tokens) with nnz in {4, 16, 64} nonzeros of +-1/4, so norms,
normalised values and scores are exact on any device.  The grid puts every value of every axis into some case:
latents (4,4) (6,10) (5,7) (9,16) (7,12) at ds1 and ds2 and (5,5) at ds4, max_downsample 1 / 2 / 4 (with layers the
reference skips), batch_size 1 / 2 / 3 with align_batch off and on, frames per chunk 1..16 with target_stride 1, 2, 3, 4,
8 (F % stride != 0 with both dst-frame counts drawn, forced where needed), local_merge_ratio 0 .. 1, and global merging
over equal and ragged chains with global_merge_ratio 0 (refused), 0.5, 0.8, 1.0 and global_rand 0, 0.1, 0.5, 1 and 0.3 /
0.8 with the coin forced to exactly fp32(global_rand) (and, as a companion, the next float above it).  Forced values
replace what the reference's torch.rand / torch.randint returned after the real draw advanced the generator, and the
Recorder stores them, so a replay feeds the same values.

The sweep has its own RNG seed and writes only sweep_* files: every fixture of the other generators stays as it is.
"""
from __future__ import annotations

import contextlib
import math
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import Recorder, exact_video_tokens, ref_patch, save, t2n  # noqa: E402

SEED = 20260917
MAX_DRAWS_PER_CALL = 64      # a terminating compute_merge draws at most log2(F) + 2 values


class NonTermination(Exception):
    pass


@contextlib.contextmanager
def forced_draws(randint: list, coin=None):
    """Installed outside the Recorder, so that it records what the reference saw.  Every draw still advances the
    generator; while the list `randint` is not empty, randint results are replaced by its values (popped), and with
    `coin` every torch.rand result is that fp32 value."""
    ri = randint
    real_ri, real_r = torch.randint, torch.rand
    count = [0]

    def randint_(*a, **k):
        out = real_ri(*a, **k)
        count[0] += 1
        if count[0] > MAX_DRAWS_PER_CALL:
            raise NonTermination()
        if ri:
            v = ri.pop(0)
            assert a[0] <= v < a[1], (v, a)
            out = torch.full_like(out, v)
        return out

    def rand_(*a, **k):
        out = real_r(*a, **k)
        return out if coin is None else torch.full_like(out, coin)

    torch.randint, torch.rand = randint_, rand_
    try:
        yield
    finally:
        torch.randint, torch.rand = real_ri, real_r


def level_tokens(size, ds):
    """Tokens per frame of the UNet layer that downsamples the latent `size` ds times (ceil per halving)."""
    h, w = size
    for _ in range(int(math.log2(ds))):
        h, w = -(-h // 2), -(-w // 2)
    return h * w


def run_case(name, rng, *, size, ds, B, chunks, C=64, nnz=16, seed=0, randint=(), coin=None, **args):
    T = level_tokens(size, ds)
    module = SimpleNamespace(generator=torch.Generator(device="cpu").manual_seed(seed), global_tokens=None)
    info = {"size": size, "hooks": [], "args": dict(
        max_downsample=2, generator=None, seed=123, batch_size=B, align_batch=False, merge_global=False,
        global_merge_ratio=0.8, local_merge_ratio=0.9, global_rand=0.5, target_stride=4)}
    info["args"].update(args)
    out = {"n_chunks": len(chunks), "size": np.array(size), "batch_size": B, "nnz": nnz, "ds": ds}
    out.update({f"arg_{k}": v for k, v in info["args"].items() if k != "generator"})
    forced = list(randint)
    for i, F in enumerate(chunks):
        x = exact_video_tokens(rng, B, F, T, C, nnz=nnz, flips=min(6, nnz // 2)).reshape(B * F, T, C)
        out[f"x{i}"] = x
        xt = torch.from_numpy(x)
        rec = Recorder()
        try:
            with forced_draws(forced, coin), rec:
                m, u, merged = ref_patch.compute_merge(module, xt, info)
                back = u(merged)
        except NonTermination:
            out[f"refused{i}"] = "nonterminating"
            break
        except Exception as e:  # noqa: BLE001  (the reference's refusal is recorded, whatever it is)
            out[f"refused{i}"] = type(e).__name__
        # the draws made, up to a refusal too
        out[f"randint{i}"] = np.array(rec.randint, dtype=np.int64)
        out[f"rand{i}"] = np.array(rec.rand, dtype=np.float64)
        if f"refused{i}" in out:
            break
        out[f"merged{i}"] = t2n(merged)
        out[f"back{i}"] = t2n(back)
        if module.global_tokens is not None:
            out[f"global{i}"] = t2n(module.global_tokens)
    save("sweep_" + name, **out)


def f32_above(v):
    return float(np.nextafter(np.float32(v), np.float32(np.inf)))


def main():
    rng = np.random.default_rng(SEED)
    torch.manual_seed(SEED)
    seeds = iter(range(1000, 2000))

    def c(name, **kw):
        run_case(name, rng, seed=next(seeds), **kw)

    G = dict(merge_global=True)

    # ---- latent size x level, batch_size x align_batch, frames x stride, local ratio (one chunk each)
    c("sq4_ds1_b2_f8", size=(4, 4), ds=1, B=2, chunks=[8])
    c("sq4_ds2_b1_align_f5_s3", size=(4, 4), ds=2, B=1, chunks=[5], align_batch=True, target_stride=3,
      local_merge_ratio=0.5, nnz=4)
    c("sq4_ds1_md1_f4", size=(4, 4), ds=1, B=2, chunks=[4], max_downsample=1)
    c("r6x10_ds1_b3_f7_r095", size=(6, 10), ds=1, B=3, chunks=[7], local_merge_ratio=0.95)
    c("r6x10_ds2_b3_align_f9_s8", size=(6, 10), ds=2, B=3, chunks=[9], align_batch=True, target_stride=8)
    c("r5x7_ds1_b1_f12_s2_r01", size=(5, 7), ds=1, B=1, chunks=[12], target_stride=2, local_merge_ratio=0.1)
    c("r5x7_ds2_md1_skip", size=(5, 7), ds=2, B=2, chunks=[4], max_downsample=1)
    c("r5x7_ds2_b2_align_f3_s2_r1", size=(5, 7), ds=2, B=2, chunks=[3], align_batch=True, target_stride=2,
      local_merge_ratio=1.0)
    c("r9x16_ds1_c320_f2", size=(9, 16), ds=1, B=1, chunks=[2], C=320, nnz=64)
    c("r9x16_ds2_b2_f5_nnz4", size=(9, 16), ds=2, B=2, chunks=[5], nnz=4)
    c("r7x12_ds1_b2_align_f3_s3_r05", size=(7, 12), ds=1, B=2, chunks=[3], align_batch=True, target_stride=3,
      local_merge_ratio=0.5, nnz=64)
    c("r7x12_ds2_b3_align_f16", size=(7, 12), ds=2, B=3, chunks=[16], align_batch=True)
    c("o5x5_ds4_md4_f8_s2", size=(5, 5), ds=4, B=2, chunks=[8], max_downsample=4, target_stride=2, nnz=4)
    c("o5x5_ds4_md2_skip", size=(5, 5), ds=4, B=2, chunks=[8], max_downsample=2)
    c("sq4_ds2_f2_r01_r0", size=(4, 4), ds=2, B=2, chunks=[2], local_merge_ratio=0.1, nnz=4)   # Ns = 4: r = 0
    c("sq4_ds1_f5_ratio0", size=(4, 4), ds=1, B=2, chunks=[5], local_merge_ratio=0.0)          # no draw
    c("sq4_ds1_b1_f1", size=(4, 4), ds=1, B=1, chunks=[1])
    c("sq4_ds1_f1_s1", size=(4, 4), ds=1, B=2, chunks=[1], target_stride=1)
    c("sq4_ds1_f3_s1_nonterminating", size=(4, 4), ds=1, B=2, chunks=[3], target_stride=1)
    # F % stride != 0: both dst-frame counts of the first level (randf 0 -> 2 dst frames, the last value -> 1)
    c("r6x10_ds2_f7_s4_rf0", size=(6, 10), ds=2, B=2, chunks=[7], randint=[0])
    c("r6x10_ds2_f7_s4_rf3", size=(6, 10), ds=2, B=2, chunks=[7], randint=[3])
    c("r7x12_ds2_b1_f5_s4_rf0", size=(7, 12), ds=2, B=1, chunks=[5], randint=[0], nnz=64)
    c("r7x12_ds2_b1_f5_s4_rf2", size=(7, 12), ds=2, B=1, chunks=[5], randint=[2], nnz=64)

    # ---- global stage: equal and ragged chains
    c("g_sq4_444", size=(4, 4), ds=1, B=2, chunks=[4, 4, 4], **G)
    c("g_r6x10_ds2_b3_align_344_g05_r01", size=(6, 10), ds=2, B=3, chunks=[3, 4, 4], align_batch=True,
      global_merge_ratio=0.5, global_rand=0.1, **G)
    c("g_r5x7_ds2_b1_443_g1_r0", size=(5, 7), ds=2, B=1, chunks=[4, 4, 3], global_merge_ratio=1.0,
      global_rand=0.0, **G)
    c("g_sq4_b2_align_414_r1", size=(4, 4), ds=1, B=2, chunks=[4, 1, 4], align_batch=True, global_rand=1.0, **G)
    c("g_r6x10_ds2_144", size=(6, 10), ds=2, B=2, chunks=[1, 4, 4], nnz=4, **G)
    c("g_r7x12_ds2_b1_1212_s8", size=(7, 12), ds=2, B=1, chunks=[12, 12], target_stride=8, **G)
    c("g_sq4_b2_169_r095", size=(4, 4), ds=1, B=2, chunks=[16, 9], local_merge_ratio=0.95, global_merge_ratio=0.5,
      **G)
    c("g_sq4_b3_33_ratio0", size=(4, 4), ds=1, B=3, chunks=[3, 3], local_merge_ratio=0.0, **G)
    c("g_r9x16_ds2_b2_22_s2", size=(9, 16), ds=2, B=2, chunks=[2, 2], target_stride=2, **G)
    c("g_sq4_44_gratio0_refused", size=(4, 4), ds=1, B=2, chunks=[4, 4], global_merge_ratio=0.0, **G)
    # the coin exactly at fp32(global_rand), which lies above global_rand (0.3, 0.8), and the next float above it
    c("g_sq4_444_rand03_at", size=(4, 4), ds=1, B=2, chunks=[4, 4, 4], global_rand=0.3,
      coin=float(np.float32(0.3)), **G)
    c("g_sq4_444_rand03_above", size=(4, 4), ds=1, B=2, chunks=[4, 4, 4], global_rand=0.3, coin=f32_above(0.3), **G)
    c("g_r6x10_ds2_b3_align_344_rand08_at", size=(6, 10), ds=2, B=3, chunks=[3, 4, 4], align_batch=True,
      global_rand=0.8, coin=float(np.float32(0.8)), **G)
    c("g_r6x10_ds2_b3_align_344_rand08_above", size=(6, 10), ds=2, B=3, chunks=[3, 4, 4], align_batch=True,
      global_rand=0.8, coin=f32_above(0.8), **G)
    # a draw-dependent chunk whose draw is not randf = 0 merges to MORE tokens than randf = 0 does: 10 frames of 84
    # tokens at stride 4 give 161 local tokens for randf 2 or 3 and 160 for randf 0 or 1 (a store sized at randf = 0
    # would refuse the first chunk).  Generated last, so that every case above stays byte-identical.
    c("g_r7x12_ds1_1010_rf2", size=(7, 12), ds=1, B=2, chunks=[10, 10], randint=[2, 0, 3, 1], **G)


if __name__ == "__main__":
    main()
