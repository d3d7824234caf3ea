"""Pins the numpy oracle's compute_merge against the reference across its argument space: every sweep_* fixture of
tests/make_golden_sweep.py (latent shapes and levels, batch sizes with and without align_batch, frame counts and
strides, local and global ratios, equal and ragged chunk chains, the global coin at fp32(global_rand)) replayed with
the recorded draws.  Bit for bit in the merged tokens, the unmerge and the global tokens, the same number of draws, and
a refusal wherever the reference refused.  CPU only; tests/test_gpu_merge_sweep.py replays the same fixtures through the
library."""
import glob
import os

import numpy as np
import pytest

import vidtome_oracle as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SWEEP = sorted(os.path.basename(p)[len("sweep_"):-len(".npz")] for p in glob.glob(os.path.join(GOLD, "sweep_*.npz")))

# what the reference did -> what the code under test must raise.  "nonterminating": target_stride 1 on several frames
# makes every frame dst, so the reference's level loop (patch.py:44) never ends; the oracle and the library refuse.
REFUSALS = {"ValueError": ValueError, "nonterminating": ValueError}


def load(name):
    return np.load(os.path.join(GOLD, f"sweep_{name}.npz"))


def merge_args(g):
    """The reference's tome_info["args"] of a fixture, as keyword arguments of oracle.compute_merge."""
    return dict(batch_size=int(g["batch_size"]), local_merge_ratio=float(g["arg_local_merge_ratio"]),
                max_downsample=int(g["arg_max_downsample"]), target_stride=int(g["arg_target_stride"]),
                align_batch=bool(g["arg_align_batch"]), merge_global=bool(g["arg_merge_global"]),
                global_merge_ratio=float(g["arg_global_merge_ratio"]), global_rand=float(g["arg_global_rand"]))


def chunks(g):
    """(index, x, randint draws, rand draws, refusal or None) for each chunk the reference was given; a refused chunk
    comes with the draws the reference made before it raised (none where it would not have terminated)."""
    for i in range(int(g["n_chunks"])):
        if f"x{i}" not in g.files:
            return
        refused = str(g[f"refused{i}"]) if f"refused{i}" in g.files else None
        ri = [int(v) for v in g[f"randint{i}"]] if f"randint{i}" in g.files else []
        rr = [float(v) for v in g[f"rand{i}"]] if f"rand{i}" in g.files else []
        yield i, g[f"x{i}"], ri, rr, refused
        if refused is not None:
            return


def test_sweep_fixtures_present():
    assert len(SWEEP) >= 38
    assert sum("rand03_at" in n or "rand08_at" in n for n in SWEEP) == 2


@pytest.mark.parametrize("name", SWEEP)
def test_oracle_compute_merge_matches_reference_sweep(name):
    g = load(name)
    glob_tokens = None
    for i, x, ri, rr, refused in chunks(g):
        kw = dict(global_tokens=glob_tokens, draw_randf=lambda s: ri.pop(0), draw_coin=lambda: rr.pop(0),
                  **merge_args(g))
        if refused is not None:
            with pytest.raises(REFUSALS[refused]):
                O.compute_merge(x, tuple(g["size"]), **kw)
            return
        res = O.compute_merge(x, tuple(g["size"]), **kw)
        assert not ri and not rr, f"chunk {i}: the oracle consumed a different number of draws than the reference"
        np.testing.assert_array_equal(res.merged_tokens, g[f"merged{i}"], err_msg=f"chunk {i}: merged")
        np.testing.assert_array_equal(res.unmerge(res.merged_tokens), g[f"back{i}"], err_msg=f"chunk {i}: back")
        glob_tokens = res.global_tokens
        if f"global{i}" in g.files:
            np.testing.assert_array_equal(glob_tokens, g[f"global{i}"], err_msg=f"chunk {i}: global tokens")
        else:
            assert glob_tokens is None


@pytest.mark.parametrize("grand", [0.0, 0.1, 0.3, 0.5, 0.6, 0.7, 0.8, 0.9, 1.0])
def test_coin_rule_is_torchs_fp32_comparison(grand):
    """patch.py:62 `torch.rand(1) > global_rand`: the library's host rule (utils.coin_above) decides as torch does at
    fp32(global_rand) and at its neighbours, also where that float lies above global_rand (0.1, 0.3, 0.6, 0.8)."""
    import torch
    from vidtome_b200.utils import coin_above
    f = np.float32(grand)
    for c in (np.nextafter(f, np.float32(-1)), f, np.nextafter(f, np.float32(2))):
        want = bool(torch.tensor([float(c)], dtype=torch.float32) > grand)
        assert coin_above(float(c), grand) == want, (grand, float(c))


@pytest.mark.parametrize("F,T,ratio,stride", [(10, 84, 0.9, 4), (10, 1024, 0.9, 4), (7, 12, 0.5, 4), (12, 24, 0.95, 8),
                                              (9, 15, 0.9, 3), (6, 40, 0.1, 4), (5, 16, 1.0, 4), (8, 16, 0.0, 4)])
def test_store_capacity_is_the_longest_local_set_over_every_draw(F, T, ratio, stride):
    """patch.local_merged_len, which sizes a GlobalTokenStore, against the oracle's local merged length under every
    sequence of draws: equal to the longest.  randf = 0 is not always the longest: (10, 84, 0.9, 4) gives 160 tokens for
    a first draw of 0 or 1 and 161 for 2 or 3."""
    from vidtome_b200.patch import local_merged_len
    x = np.random.default_rng(0).standard_normal((F, T, 8)).astype(np.float16)
    args = dict(batch_size=1, local_merge_ratio=ratio, target_stride=stride, max_downsample=1)

    def longest(prefix):
        strides = []

        def draw(s):
            strides.append(s)
            return prefix[len(strides) - 1] if len(strides) <= len(prefix) else 0

        n = O.compute_merge(x, (1, T), draw_randf=draw, **args).merged_tokens.shape[1]
        if len(strides) > len(prefix):
            return max(longest(prefix + [v]) for v in range(strides[len(prefix)]))
        return n

    assert local_merged_len(F, T, dict(local_merge_ratio=ratio, target_stride=stride)) == longest([])
