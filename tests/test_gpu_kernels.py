"""Parity of each CUDA kernel (through the C-ABI) against the numpy oracle.  Needs an H100 (sm_90a)."""
import numpy as np
import pytest
import torch

import vidtome_oracle as O

pytestmark = pytest.mark.gpu


def _ops():
    from vidtome_b200 import ops
    return ops


def _split(N, unm_pre, F, stride, randf):
    from vidtome_b200._lib import VtmSplit
    return VtmSplit.local(N, unm_pre, F, stride, randf)


def _ulp_diff_f16(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    def ordered(x):
        u = x.view(np.uint16).astype(np.int32)
        return np.where(u & 0x8000, 0x8000 - (u & 0x7FFF), 0x8000 + u)
    return np.abs(ordered(a) - ordered(b))


def _exact_tokens(rng, shape, nnz=64, val=0.125):
    """Rows with exactly `nnz` entries of +-val: every dot product is an integer multiple of val^2 that
    is exact in fp32 in any summation order and exactly representable in fp16 -> scores (and their many
    ties) are bit-identical on every device."""
    B, N, C = shape
    x = np.zeros(shape, dtype=np.float16)
    for b in range(B):
        for i in range(N):
            cols = rng.choice(C, size=nnz, replace=False)
            x[b, i, cols] = rng.choice([-val, val], size=nnz)
    return x


def _oracle_node(a: np.ndarray, b: np.ndarray, align: bool):
    s = O.scores_matmul(a, b)
    if align:
        s = np.concatenate([s[i] for i in range(s.shape[0])], axis=-1)[None]
    idx = s.argmax(-1)
    mx = np.take_along_axis(s, idx[..., None], -1)[..., 0]
    return s, mx, idx


# --------------------------------------------------------------------------- K0
@pytest.mark.parametrize("N,unm_pre,F,stride,randf,C", [
    (4 * 96, 0, 4, 4, 2, 320),
    (5 * 64 + 37, 37, 5, 4, 1, 640),      # ragged F, carried unmerged tokens
    (2 * 50 + 11, 11, 2, 2, 0, 1280),
])
def test_normalize_split(N, unm_pre, F, stride, randf, C):
    ops = _ops()
    rng = np.random.default_rng(0)
    B = 2
    x = rng.standard_normal((B, N, C)).astype(np.float16)
    a_idx, b_idx, _, _ = O.split_indices_randframe(N, F, unm_pre, stride, randf)
    xn = O.normalize_rows(x)
    a, b = ops.normalize_split(torch.from_numpy(x).cuda(), None, _split(N, unm_pre, F, stride, randf))
    a, b = a.cpu().numpy(), b.cpu().numpy()
    assert a.shape == (B, len(a_idx), C) and b.shape == (B, len(b_idx), C)
    for got, want in ((a, xn[:, a_idx]), (b, xn[:, b_idx])):
        d = _ulp_diff_f16(got, want)
        # the fp32 sum of squares is order dependent: a row whose norm sits on an fp16 rounding boundary
        # may differ by one ulp; everything else must be identical
        assert d.max() <= 1
        assert (d > 0).mean() < 5e-3


def test_normalize_split_rowmap():
    ops = _ops()
    rng = np.random.default_rng(1)
    B, N0, C = 2, 300, 320
    x = rng.standard_normal((B, N0, C)).astype(np.float16)
    N, unm_pre, F = 2 * 60 + 20, 20, 2
    rowmap = np.stack([rng.permutation(N0)[:N] for _ in range(B)]).astype(np.int32)
    seq = np.take_along_axis(x, rowmap[:, :, None].astype(np.int64), axis=1)
    a_idx, b_idx, _, _ = O.split_indices_randframe(N, F, unm_pre, 4, 1)
    xn = O.normalize_rows(seq)
    a, b = ops.normalize_split(torch.from_numpy(x).cuda(), torch.from_numpy(rowmap).cuda(),
                               _split(N, unm_pre, F, 4, 1))
    assert _ulp_diff_f16(a.cpu().numpy(), xn[:, a_idx]).max() <= 1
    assert _ulp_diff_f16(b.cpu().numpy(), xn[:, b_idx]).max() <= 1


# --------------------------------------------------------------------------- KA
@pytest.mark.parametrize("B,Ns,Nd,C,align", [
    (1, 128, 256, 64, False),      # exactly one tile, one K chunk
    (2, 300, 700, 320, False),     # ragged tiles
    (2, 300, 700, 320, True),
    (3, 1000, 2500, 640, True),    # PnP-like batch of 3
    (2, 515, 5000, 320, False),    # many dst tiles -> split dst sweeps + atomic combine
    (1, 130, 257, 72, False),      # K tail (72 = 64 + 8), 1-row / 1-column tails
])
def test_sim_argmax_bit_exact_on_exact_inputs(B, Ns, Nd, C, align):
    ops = _ops()
    rng = np.random.default_rng(B * 1000 + Ns)
    nnz = min(64, C // 2)
    a = _exact_tokens(rng, (B, Ns, C), nnz=nnz)
    b = _exact_tokens(rng, (B, Nd, C), nnz=nnz)
    _, mx, idx = _oracle_node(a, b, align)
    keys = ops.sim_argmax(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda(), align)
    score, arg = ops.keys_to_score_arg(keys)
    np.testing.assert_array_equal(score.cpu().numpy().view(np.uint16), mx.view(np.uint16))
    np.testing.assert_array_equal(arg.cpu().numpy(), idx)


@pytest.mark.parametrize("align", [False, True])
def test_sim_argmax_equal_maxima_across_dst_ranges(align):
    """The epilogue filters on the maximum other dst ranges have already published.  Every dst row here occurs
    many times across the whole sweep (and in both samples), so the winning score is tied across work items that
    run in arbitrary order: the smallest dst index must still win, bit for bit."""
    ops = _ops()
    rng = np.random.default_rng(11)
    B, Ns, Nd, C = 2, 700, 6144, 320
    a = _exact_tokens(rng, (B, Ns, C))
    pool = _exact_tokens(rng, (1, 96, C))[0]
    pick = rng.integers(0, 96, size=(B, Nd))
    b = pool[pick]
    if align:
        b[1] = b[0][::-1]                      # the same rows again in the second sample, other order
    _, mx, idx = _oracle_node(a, b, align)
    keys = ops.sim_argmax(torch.from_numpy(a).cuda(), torch.from_numpy(np.ascontiguousarray(b)).cuda(), align)
    score, arg = ops.keys_to_score_arg(keys)
    np.testing.assert_array_equal(score.cpu().numpy().view(np.uint16), mx.view(np.uint16))
    np.testing.assert_array_equal(arg.cpu().numpy(), idx)


def test_sim_argmax_nonpositive_and_zero_scores():
    """Rows whose best score is negative, +0 or -0 (threshold stepping around zero, merge.py:112 semantics)."""
    ops = _ops()
    rng = np.random.default_rng(12)
    B, Ns, Nd, C = 1, 260, 2304, 128
    b = np.abs(_exact_tokens(rng, (B, Nd, C, ), nnz=48))
    a = -np.abs(_exact_tokens(rng, (B, Ns, C), nnz=48))   # every score <= 0; supports overlap, so most are < 0
    a[0, :40] = 0                                         # all scores +0 for these src rows
    for zero_rows in (False, True):
        if zero_rows:
            b[0, 1500::211] = 0                           # late zero dst rows: -0 beats the negative scores so far
        a16, b16 = a.astype(np.float16), b.astype(np.float16)
        s, mx, idx = _oracle_node(a16, b16, False)
        assert zero_rows or (mx[0, 40:] < 0).all()
        keys = ops.sim_argmax(torch.from_numpy(a16).cuda(), torch.from_numpy(b16).cuda(), False)
        score, arg = ops.keys_to_score_arg(keys)
        assert np.array_equal(score.cpu().numpy().astype(np.float32), mx.astype(np.float32))     # -0 == +0
        np.testing.assert_array_equal(arg.cpu().numpy(), idx)


def test_sim_argmax_matches_simt_twin_at_config_size():
    """C3 ds1 level shape (Ns=12288, Nd=4096, C=320): tensor-core kernel vs CUDA-core twin."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(3)
    B, Ns, Nd, C = 2, 12288, 4096, 320
    a = torch.randn((B, Ns, C), generator=g, device="cuda", dtype=torch.float32)
    b = torch.randn((B, Nd, C), generator=g, device="cuda", dtype=torch.float32)
    a = (a / a.norm(dim=-1, keepdim=True)).half()
    b = (b / b.norm(dim=-1, keepdim=True)).half()
    k1 = ops.sim_argmax(a, b, False)
    k2 = ops.sim_argmax(a, b, False, simt=True)
    s1, a1 = ops.keys_to_score_arg(k1)
    s2, a2 = ops.keys_to_score_arg(k2)
    assert _ulp_diff_f16(s1.cpu().numpy(), s2.cpu().numpy()).max() <= 1
    assert (a1 == a2).float().mean().item() > 0.98
    # where they differ, the full-precision score of both picks must be within fp16 rounding of each other
    diff = (a1 != a2).nonzero()
    if len(diff):
        bi, ri = diff[:, 0], diff[:, 1]
        sa = (a[bi, ri].float() * b[bi, a1[bi, ri]].float()).sum(-1)
        sb = (a[bi, ri].float() * b[bi, a2[bi, ri]].float()).sum(-1)
        assert (sa - sb).abs().max().item() < 2e-3


# --------------------------------------------------------------------------- KB1
@pytest.mark.parametrize("Bp,Ns", [(1, 1), (1, 1000), (2, 1024), (2, 5000), (3, 12288)])
def test_topr_sort_is_stable_descending(Bp, Ns):
    ops = _ops()
    rng = np.random.default_rng(Ns)
    vals = rng.choice(np.array([-1.0, -0.5, 0.0, 0.25, 0.5, 0.75, 0.999, 1.0], dtype=np.float16), size=(Bp, Ns))
    vals[:, ::7] = rng.standard_normal((Bp, len(range(0, Ns, 7)))).astype(np.float16)
    hb = vals.view(np.uint16).astype(np.uint64)
    hb = np.where(hb == 0x8000, 0, hb)
    ordered = np.where(hb & 0x8000, hb ^ 0xFFFF, hb | 0x8000)
    arg = rng.integers(0, 1000, size=(Bp, Ns)).astype(np.uint64)
    keys = (ordered << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - arg)
    edge, rank = ops.topr_sort(torch.from_numpy(keys.view(np.int64)).cuda())
    want = O.stable_argsort_desc(vals)
    np.testing.assert_array_equal(edge.cpu().numpy(), want)
    inv = np.empty_like(want)
    for b in range(Bp):
        inv[b, want[b]] = np.arange(Ns)
    np.testing.assert_array_equal(rank.cpu().numpy(), inv)


# --------------------------------------------------------------------------- KC / KE
@pytest.mark.parametrize("shared_map", [False, True])
def test_gather_and_unmerge_add(shared_map):
    ops = _ops()
    rng = np.random.default_rng(5)
    B, N, L, C = 2, 777, 301, 320
    x = rng.standard_normal((B, N, C)).astype(np.float16)
    mb = 1 if shared_map else B
    mu = rng.integers(0, N, size=(mb, L)).astype(np.int32)
    y = ops.gather_rows(torch.from_numpy(x).cuda(), torch.from_numpy(mu).cuda())
    want = np.take_along_axis(x, np.broadcast_to(mu, (B, L))[:, :, None].astype(np.int64), axis=1)
    np.testing.assert_array_equal(y.cpu().numpy(), want)

    pi = rng.integers(0, L, size=(mb, N)).astype(np.int32)
    resid = rng.standard_normal((B, N, C)).astype(np.float16)
    out = ops.unmerge_add(y, torch.from_numpy(pi).cuda(), torch.from_numpy(resid).cuda())
    g = np.take_along_axis(want, np.broadcast_to(pi, (B, N))[:, :, None].astype(np.int64), axis=1)
    np.testing.assert_array_equal(out.cpu().numpy(), (g.astype(np.float32) + resid.astype(np.float32)).astype(np.float16))
    out2 = ops.unmerge_add(y, torch.from_numpy(pi).cuda(), None)
    np.testing.assert_array_equal(out2.cpu().numpy(), g)


# --------------------------------------------------------------------------- projection GEMM
@pytest.mark.parametrize("M,N,K,bias", [(128, 256, 64, False), (1000, 960, 320, False), (333, 320, 320, True),
                                        (2561, 1920, 640, True)])
def test_linear_f16(M, N, K, bias):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(M)
    a = torch.randn((M, K), generator=g, device="cuda").half()
    w = (torch.randn((N, K), generator=g, device="cuda") / K ** 0.5).half()
    bb = torch.randn((N,), generator=g, device="cuda").half() if bias else None
    d = ops.linear(a, w, bb)
    ref = a.float() @ w.float().t()
    if bias:
        ref = ref + bb.float()
    err = (d.float() - ref).abs().max().item()
    assert err <= 1e-3 * max(1.0, ref.abs().max().item()) + 1e-3  # fp16 output rounding, rel 1e-3


# --------------------------------------------------------------------------- fused LayerNorm (norm1)
@pytest.mark.parametrize("C", [320, 640, 1280, 128])
def test_fused_layernorm_in_k0_and_kc(C):
    """K0 / KC with norm1 fused == torch LayerNorm (fp16, the module the reference calls at patch.py:146)
    followed by the plain kernels; at most one fp16 ulp apart (different fp32 summation order)."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(C)
    B, F, T = 2, 4, 96
    N = F * T
    x = (torch.randn((B, N, C), generator=g, device="cuda") * 2 + 0.3).half()
    ln = torch.nn.LayerNorm(C).cuda().half()
    with torch.no_grad():
        ln.weight.copy_(1 + 0.2 * torch.randn(C, generator=g, device="cuda"))
        ln.bias.copy_(0.1 * torch.randn(C, generator=g, device="cuda"))
        y = ln(x)
    sp = _split(N, 0, F, 4, 1)
    a0, b0 = ops.normalize_split(y, None, sp)
    a1, b1 = ops.normalize_split(x, None, sp, ln=(ln.weight.data, ln.bias.data, ln.eps))
    for got, want in ((a1, a0), (b1, b0)):
        d = _ulp_diff_f16(got.cpu().numpy(), want.cpu().numpy())
        assert d.max() <= 2 and (d > 0).mean() < 0.02
    mu = torch.randint(0, N, (B, 123), generator=g, device="cuda", dtype=torch.int32)
    m0 = ops.gather_rows(y, mu)
    m1 = ops.gather_rows(x, mu, ln=(ln.weight.data, ln.bias.data, ln.eps))
    d = _ulp_diff_f16(m1.cpu().numpy(), m0.cpu().numpy())
    assert d.max() <= 1 and (d > 0).mean() < 0.01


# --------------------------------------------------------------------------- feed-forward GEMMs (f3)
@pytest.mark.parametrize("M,K,inner", [(256, 64, 128), (1000, 320, 1280), (4099, 640, 2560)])
def test_linear_geglu_and_residual(M, K, inner):
    """GEGLU projection with the gate fused into the epilogue, and the output projection with bias + residual, against
    the unfused fp16 torch ops (F.linear -> chunk -> a * gelu(g); F.linear + h): same rounding points, so agreement is
    at the level of one fp16 ulp of the result."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(M)
    a = torch.randn((M, K), generator=g, device="cuda").half()
    w = (torch.randn((2 * inner, K), generator=g, device="cuda") / K ** 0.5).half()
    b = (0.1 * torch.randn((2 * inner,), generator=g, device="cuda")).half()
    wi, bi = ops.interleave_geglu(w, b)
    u = ops.linear_geglu(a, wi, bi)
    proj = torch.nn.functional.linear(a, w, b)
    h, gate = proj.chunk(2, dim=-1)
    want = h * torch.nn.functional.gelu(gate)
    ref32 = (a.float() @ w.float().t() + b.float())
    r_h, r_g = ref32.chunk(2, dim=-1)
    ref = r_h * torch.nn.functional.gelu(r_g)
    scale = ref.abs().max().item()
    assert (u.float() - ref).abs().max().item() <= 2e-3 * scale            # vs exact arithmetic
    assert (u.float() - want.float()).abs().max().item() <= 2e-3 * scale   # vs torch's fp16 pipeline
    w2 = (torch.randn((K, inner), generator=g, device="cuda") / inner ** 0.5).half()
    b2 = (0.1 * torch.randn((K,), generator=g, device="cuda")).half()
    resid = torch.randn((M, K), generator=g, device="cuda").half()
    out = ops.linear_residual(u, w2, b2, resid)
    want2 = torch.nn.functional.linear(u, w2, b2) + resid
    ref2 = u.float() @ w2.float().t() + b2.float() + resid.float()
    s2 = ref2.abs().max().item()
    assert (out.float() - ref2).abs().max().item() <= 2e-3 * s2
    assert (out.float() - want2.float()).abs().max().item() <= 2e-3 * s2


def test_feed_forward_fast_path_matches_module():
    """feedforward.feed_forward_residual == h + ff(norm3(h)) of the module (both stand-in layouts: the skeleton's
    GEGLUFeedForward and diffusers' FeedForward.net = [GEGLU, Dropout, Linear])."""
    from vidtome_b200 import feedforward, patch
    from vidtome_b200.skeleton import GEGLUFeedForward
    torch.manual_seed(0)
    dim = 320

    class GEGLU(torch.nn.Module):
        def __init__(self, dim_in, dim_out):
            super().__init__()
            self.proj = torch.nn.Linear(dim_in, dim_out * 2)

        def forward(self, x):
            h, gate = self.proj(x).chunk(2, dim=-1)
            return h * torch.nn.functional.gelu(gate)

    class FeedForward(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.net = torch.nn.ModuleList([GEGLU(dim, 4 * dim), torch.nn.Dropout(0.0), torch.nn.Linear(4 * dim, dim)])

        def forward(self, x):
            for m in self.net:
                x = m(x)
            return x

    for ff in (GEGLUFeedForward(dim), FeedForward()):
        ff = ff.cuda().half().eval()
        norm = torch.nn.LayerNorm(dim).cuda().half()
        with torch.no_grad():
            norm.weight.add_(0.1 * torch.randn_like(norm.weight))
            norm.bias.add_(0.1 * torch.randn_like(norm.bias))
        h = torch.randn((6, 500, dim), device="cuda").half()
        parts = feedforward.geglu_parts(ff)
        assert parts is not None
        ln = patch._fusable_layer_norm(norm, h)
        with torch.no_grad():
            got = feedforward.feed_forward_residual(ff, parts, ln, h)
            want = ff(norm(h)) + h
            ref = ff.float()(norm.float()(h.float())) + h.float()
        s = ref.abs().max().item()
        assert (got.float() - ref).abs().max().item() <= 2e-3 * s
        assert (got.float() - want.float()).abs().max().item() <= 3e-3 * s
    # anything non-stock is refused
    ff = GEGLUFeedForward(dim).cuda().half()
    ff.register_forward_hook(lambda m, i, o: o)
    assert feedforward.geglu_parts(ff) is None
