"""The merge plan (patch.compute_merge / build_merge_plan) against the reference across its argument space.

1. Every sweep_* fixture of tests/make_golden_sweep.py (the reference's compute_merge over chains of chunks on one
   module) replayed with the recorded draws through the library on CUDA fp16, in each execution form of the global
   stage: (a) eager with the host coin; (b) patch.DEVICE_COIN, the mode-1 split, which takes equal halves only (a block
   whose sets differ keeps the host coin, as documented); (c) a GlobalTokenStore as module.global_tokens with max_frames
   = the chain's largest chunk, the mode-2 device counts.  Bit for bit: merged, back = u(merged), the global tokens
   after every chunk and the number of draws; a refusal exactly where the reference refused.
2. The patched block's unmerge + residual (plan.unmerge_add) on a non-square fixture against the oracle.
3. A hypothesis fuzz beyond the grid: larger latents (up to 24 x 40), C up to 640, ragged chains, coins at and next to
   fp32(global_rand); identical draws go to form (a) and to oracle.compute_merge, which must agree bit for bit.
"""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from hypothesis import HealthCheck, given, note, settings, strategies as st

import test_oracle_sweep_cpu as S
import vidtome_oracle as O
from test_gpu_graph_global import Replay

pytestmark = pytest.mark.gpu

GLOBAL = [n for n in S.SWEEP if bool(S.load(n)["arg_merge_global"])]


def _info(size, args):
    a = dict(args)
    a.update(generator=None, seed=123)
    return {"size": tuple(int(v) for v in size), "hooks": [], "args": a}


def _fixture_info(g):
    return _info(g["size"], S.merge_args(g))


def _valid(merged, plan):
    """The merged sequence: a GlobalTokenStore stage sizes the tensor for capacity, the first seq_len rows valid."""
    if plan is not None and plan.seq_len is not None:
        return merged[:, :int(plan.seq_len.item())]
    return merged


def _global_tokens(module):
    from vidtome_b200.patch import GlobalTokenStore
    g = module.global_tokens
    if isinstance(g, GlobalTokenStore):
        return g.tokens[:, :int(g.length.item())] if g.filled else None
    return g


# --------------------------------------------------------------------------- 1. every fixture, every form
def _replay_fixture(name, form, monkeypatch):
    from vidtome_b200 import patch
    g = S.load(name)
    info = _fixture_info(g)
    B = int(g["batch_size"])
    if form == "device_coin":
        monkeypatch.setattr(patch, "DEVICE_COIN", True)
    module = SimpleNamespace(generator=torch.Generator(device="cuda").manual_seed(0), global_tokens=None)
    if form == "store":
        frames = [g[f"x{i}"].shape[0] // B for i in range(int(g["n_chunks"])) if f"x{i}" in g.files]
        module.global_tokens = patch.GlobalTokenStore(max(frames))
    device_coins = 0
    for i, x, ri, rr, refused in S.chunks(g):
        rp = Replay(monkeypatch, randint=ri, rand=rr)
        xt = torch.from_numpy(x).cuda()
        if refused is not None:
            with pytest.raises(S.REFUSALS[refused]):
                patch.compute_merge(module, xt, info)
            return device_coins
        m, u, merged = patch.compute_merge(module, xt, info)
        plan = getattr(m, "plan", None)
        assert rp.done(), f"chunk {i}: a different number of random draws than the reference"
        device_coins += plan is not None and isinstance(plan.coin, torch.Tensor)
        np.testing.assert_array_equal(_valid(merged, plan).cpu().numpy(), g[f"merged{i}"], err_msg=f"chunk {i}")
        np.testing.assert_array_equal(u(merged).cpu().numpy(), g[f"back{i}"], err_msg=f"chunk {i}")
        glob = _global_tokens(module)
        if f"global{i}" in g.files:
            np.testing.assert_array_equal(glob.cpu().numpy(), g[f"global{i}"], err_msg=f"chunk {i}")
        else:
            assert glob is None
    return device_coins


@pytest.mark.parametrize("name", S.SWEEP)
def test_host_coin_matches_reference_sweep(name, monkeypatch):
    _replay_fixture(name, "host", monkeypatch)


@pytest.mark.parametrize("name", GLOBAL)
def test_device_coin_matches_reference_sweep(name, monkeypatch):
    coins = _replay_fixture(name, "device_coin", monkeypatch)
    # the mode-1 split runs at every global stage whose local set is as long as the stored one (the global tokens after
    # chunk i are chunk i's local set), e.g. at the third chunk of the (3, 4, 4) chains, where the boundary coin meets
    # the kernels' fp32 threshold
    g = S.load(name)
    equal = sum(f"global{i - 1}" in g.files and f"global{i}" in g.files
                and g[f"global{i - 1}"].shape[1] == g[f"global{i}"].shape[1] for i in range(1, int(g["n_chunks"])))
    assert coins == equal, f"the device-coin branch ran {coins} times, expected {equal}"


@pytest.mark.parametrize("name", GLOBAL)
def test_global_token_store_matches_reference_sweep(name, monkeypatch):
    coins = _replay_fixture(name, "store", monkeypatch)
    g = S.load(name)
    stages = sum(f"global{i}" in g.files for i in range(1, int(g["n_chunks"])))
    assert coins == stages, f"the store's global stage ran {coins} times, expected {stages}"


# --------------------------------------------------------------------------- 2. non-square block tail
def test_non_square_unmerge_add_with_residual_matches_oracle():
    """patch.py:168-169 (u_a(attn_output) + hidden_states) on the 6 x 10 latent with three align-free samples: one KE
    pass against the oracle's unmerge and an fp16 add.  Exact-family values, so every sum is exact."""
    from vidtome_b200 import patch
    g = S.load("r6x10_ds1_b3_f7_r095")
    x, ri = g["x0"], [int(v) for v in g["randint0"]]
    module = SimpleNamespace(generator=torch.Generator(device="cuda").manual_seed(0), global_tokens=None)
    draws = list(ri)
    with pytest.MonkeyPatch.context() as mp:
        Replay(mp, randint=ri)
        plan = patch.build_merge_plan(module, torch.from_numpy(x).cuda(), _fixture_info(g))
    res = O.compute_merge(x, tuple(g["size"]), draw_randf=lambda s: draws.pop(0), **S.merge_args(g))
    rng = np.random.default_rng(5)
    y = (rng.integers(-64, 64, size=res.merged_tokens.shape) / 64).astype(np.float16)
    got = plan.unmerge_add(torch.from_numpy(y).cuda(), torch.from_numpy(x).cuda()).cpu().numpy()
    want = (res.unmerge(y).astype(np.float32) + x.astype(np.float32)).astype(np.float16)
    np.testing.assert_array_equal(got, want)


def _balanced_video_tokens(rng, B, F, T, C, nnz=16):
    """Exact-family tokens whose rows all have mean 0 and the same variance (nnz / 2 entries of +1/4 and of -1/4; each
    frame swaps the signs of a few +/- pairs), so that a LayerNorm with unit affine scales every row by the same factor:
    the normalised rows keep the family's exact ties, and any two correct implementations take the same decisions."""
    x = np.zeros((B, F, T, C), dtype=np.float16)
    for b in range(B):
        for t in range(T):
            cols = rng.choice(C, size=nnz, replace=False)
            signs = np.repeat(np.array([0.25, -0.25], dtype=np.float16), nnz // 2)
            for f in range(F):
                s = signs.copy()
                for _ in range(rng.integers(0, 4)):
                    i, j = rng.choice(np.nonzero(s > 0)[0]), rng.choice(np.nonzero(s < 0)[0])
                    s[i], s[j] = s[j], s[i]
                x[b, f, t, cols] = s
    return x.reshape(B * F, T, C)


def test_non_square_patched_block_self_attention_matches_oracle_block():
    """patch.py:139-169 on the 6 x 10 latent (T = 60), three samples of 7 frames, ratio 0.95: the patched block's whole
    self-attention section (norm1 fused into the merge kernels, the merge plan, attn1 on the merged tokens, the unmerge
    with the residual) against oracle.tome_block_self_attention with the same draws.  The decisions are exact (balanced
    tokens), so the outputs differ only by the attention's fp16 rounding."""
    import vidtome_b200
    from vidtome_b200 import patch
    from vidtome_b200.skeleton import BasicTransformerBlock, ModelMixin
    B, F, size, C, heads = 3, 7, (6, 10), 64, 2
    torch.manual_seed(11)
    blk = BasicTransformerBlock(C, heads, hot_path_only=True)

    class Net(ModelMixin):
        def __init__(self):
            super().__init__()
            self.block = blk

    net = Net().cuda().half().eval()
    vidtome_b200.apply_patch(net, local_merge_ratio=0.95, batch_size=B)
    blk._tome_info["size"] = size                          # what the model's pre-hook reads from the latent
    blk.generator = torch.Generator(device="cuda").manual_seed(0)
    x = _balanced_video_tokens(np.random.default_rng(7), B, F, size[0] * size[1], C)
    draws = [0, 1]                                         # 7 frames, stride 4: randf 0 (two dst frames), then 1 of 2
    sd = {k: v.float().cpu().numpy().astype(np.float16) for k, v in blk.state_dict().items()}
    with pytest.MonkeyPatch.context() as mp, torch.no_grad():
        rp = Replay(mp, randint=draws)                     # a copy: `draws` is left for the oracle
        got, _ = patch._self_attention_stage(blk, torch.from_numpy(x).cuda(), None, None, None, None, None)
        assert rp.done()
    want, res = O.tome_block_self_attention(
        x, size, sd["norm1.weight"], sd["norm1.bias"], sd["attn1.to_q.weight"], sd["attn1.to_k.weight"],
        sd["attn1.to_v.weight"], sd["attn1.to_out.0.weight"], sd["attn1.to_out.0.bias"], heads, batch_size=B,
        local_merge_ratio=0.95, draw_randf=lambda s: draws.pop(0))
    got = got.float().cpu().numpy()
    want = want.astype(np.float32)
    err = np.abs(got - want)
    assert got.shape == want.shape and res.merged_tokens.shape[1] < F * size[0] * size[1]
    assert err.max() <= 4e-3 * np.abs(want).max(), (err.max(), np.abs(want).max())


# --------------------------------------------------------------------------- 3. fuzz: library vs oracle
def _exact_video_tokens(rng, B, F, T, C, nnz):
    """Exact-family tokens (tests/make_golden.py): nnz entries of +-1/4 per base token, a few sign flips per frame."""
    base = np.zeros((B, 1, T, C), dtype=np.float16)
    cols = np.argsort(rng.random((B, T, C)), axis=-1)[..., :nnz]
    np.put_along_axis(base[:, 0], cols, rng.choice(np.array([-0.25, 0.25], dtype=np.float16), size=(B, T, nnz)), -1)
    x = np.repeat(base, F, axis=1)
    flips = rng.integers(0, nnz, size=(B, F, T, min(6, nnz // 2)))
    fc = np.take_along_axis(np.broadcast_to(cols[:, None], (B, F, T, nnz)), flips, -1)
    np.put_along_axis(x, fc, -np.take_along_axis(x, fc, -1), axis=-1)
    return x.reshape(B * F, T, C)


@st.composite
def configs(draw):
    h, w = draw(st.integers(1, 24)), draw(st.integers(1, 40))
    ds = draw(st.sampled_from([1, 2, 4]))
    hh, ww = h, w
    for _ in range(int(math.log2(ds))):
        hh, ww = -(-hh // 2), -(-ww // 2)
    T = hh * ww
    C = 8 * draw(st.integers(1, 80))
    nnz = draw(st.sampled_from([n for n in (4, 16, 64) if n <= C]))
    B = draw(st.integers(1, 3))
    fmax = max(1, min(16, 3_000_000 // (B * T * C)))
    merge_global = draw(st.booleans())
    n_chunks = draw(st.integers(2, 3)) if merge_global else 1
    grand = draw(st.sampled_from([0.0, 0.1, 0.3, 0.5, 0.6, 0.8, 1.0]))
    return dict(size=(h, w), T=T, C=C, nnz=nnz, B=B, chunks=[draw(st.integers(1, fmax)) for _ in range(n_chunks)],
                seed=draw(st.integers(0, 2 ** 31 - 1)),
                coins=draw(st.lists(st.sampled_from(["at", "above", "below", "uniform"]), min_size=3, max_size=3)),
                args=dict(batch_size=B, max_downsample=draw(st.sampled_from([1, 2, 4])),
                          target_stride=draw(st.integers(2, 8)), align_batch=draw(st.booleans()),
                          local_merge_ratio=draw(st.sampled_from([0.0, 0.1, 0.5, 0.9, 0.95, 1.0])
                                                 | st.floats(0.01, 1.0)),
                          merge_global=merge_global,
                          global_merge_ratio=draw(st.sampled_from([0.5, 0.8, 1.0]) | st.floats(0.01, 1.0)),
                          global_rand=grand))


def _coin(kind, grand, rng):
    f = np.float32(grand)
    if kind == "at":
        return float(f)
    if kind in ("above", "below"):
        return float(np.nextafter(f, np.float32(np.inf if kind == "above" else -np.inf)))
    return float(np.float32(rng.random()))


@settings(max_examples=150, derandomize=True, database=None, deadline=None,
          suppress_health_check=[HealthCheck.too_slow, HealthCheck.data_too_large])
@given(cfg=configs())
def test_fuzz_library_matches_oracle(cfg):
    """Form (a), and with global merging form (c) too: a GlobalTokenStore sized for the chain's largest chunk must hold
    the local set of every chunk whatever its draws, and compute what the host coin computes."""
    from vidtome_b200 import patch
    note(f"configuration: {cfg}")
    args, B = cfg["args"], cfg["B"]
    rng = np.random.default_rng(cfg["seed"])
    info = _info(cfg["size"], args)
    modules = {"host": SimpleNamespace(generator=torch.Generator(device="cuda").manual_seed(0), global_tokens=None)}
    if args["merge_global"]:
        modules["store"] = SimpleNamespace(generator=torch.Generator(device="cuda").manual_seed(0),
                                           global_tokens=patch.GlobalTokenStore(max(cfg["chunks"])))
    glob = None
    for i, F in enumerate(cfg["chunks"]):
        x = _exact_video_tokens(rng, B, F, cfg["T"], cfg["C"], cfg["nnz"])
        randfs, coins = [], []

        def draw_randf(s):
            randfs.append(int(rng.integers(0, s)))
            return randfs[-1]

        def draw_coin():
            coins.append(_coin(cfg["coins"][i], args["global_rand"], rng))
            return coins[-1]

        try:
            res = O.compute_merge(x, cfg["size"], global_tokens=glob, draw_randf=draw_randf, draw_coin=draw_coin,
                                  **args)
        except ValueError:
            for form, module in modules.items():
                with pytest.MonkeyPatch.context() as mp:
                    Replay(mp, randint=randfs, rand=coins)
                    with pytest.raises(ValueError):
                        patch.compute_merge(module, torch.from_numpy(x).cuda(), info)
            return
        glob = res.global_tokens
        for form, module in modules.items():
            with pytest.MonkeyPatch.context() as mp:
                rp = Replay(mp, randint=randfs, rand=coins)
                m, u, merged = patch.compute_merge(module, torch.from_numpy(x).cuda(), info)
                assert rp.done(), f"{form}, chunk {i}: a different number of draws than the oracle"
            plan = getattr(m, "plan", None)
            np.testing.assert_array_equal(_valid(merged, plan).cpu().numpy(), res.merged_tokens,
                                          err_msg=f"{form}, chunk {i}: merged")
            np.testing.assert_array_equal(u(merged).cpu().numpy(), res.unmerge(res.merged_tokens),
                                          err_msg=f"{form}, chunk {i}: back")
            got = _global_tokens(module)
            if glob is None:
                assert got is None, f"{form}, chunk {i}"
            else:
                np.testing.assert_array_equal(got.cpu().numpy(), glob, err_msg=f"{form}, chunk {i}: global")
