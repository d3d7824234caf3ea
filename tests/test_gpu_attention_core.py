"""The flash-attention kernel behind KD (`vtm_attention_ex`, `vtm_attention_dev`, `VTM_ATTN_SHARED_QK`) and
`vtm_cross_attention`, against float64 softmax attention, with a per-element tolerance relative to the attention output
itself.  Needs an H100 (sm_90a).

Inputs are chosen so that the flash kernel's roundings are the only approximation left:
- tokens lie on a 1/8 grid, and the projection weights are signed permutation matrices, so q, k and v are copies of
  input values: exact in fp16 and in fp32 whatever the GEMM's summation order;
- q and k are bounded by 4, so S = q k^T (|S| <= 128 * 16 = 2^11 on a 2^-6 grid: 17 significant bits) is exact in fp32;
- W_o = I and no bias, so y = fp16(o) exactly.

Cross-attention serves as a fully controllable probe of the kernel: with Cctx = 2C, W_q = I, W_k = [I | 0] and
W_v = [0 | I], Q comes from x and K, V from the two halves of ctx, three independent designs.  Self-attention uses
signed permutations that take a head's q, k and v from the input blocks of heads h, h + 1 and h + 2.

Every call goes through the C-ABI with the workspace filled with 0xFF bytes (fp16 NaN) and the output with NaN, so any
workspace element the kernels read without having written it, and any output element left unwritten, shows as NaN."""
import math

import pytest
import torch

from vidtome_b200 import _lib

pytestmark = pytest.mark.gpu

LOG2E = 1.0 / math.log(2.0)
LENGTHS = (1, 2, 3, 63, 64, 65, 127, 128, 129, 191, 192, 193, 1000)


# ---------------------------------------------------------------------------------------------------------------------
# reference and tolerance

def _ulp16(x):
    """Spacing of fp16 numbers at |x| (2^-24 in the subnormal range)."""
    e = torch.floor(torch.log2(x.abs().clamp(min=2.0 ** -14)))
    return torch.exp2(e - 10)


def _check_exact(q, k, v):
    """q, k, v [B, H, L, d] float64 as the kernel sees them.  Asserts the limits that make them and S = q k^T exact."""
    assert q.shape[-1] <= 128
    for name, t in (("q", q), ("k", k)):
        assert torch.equal(t * 8, torch.round(t * 8)), f"{name} is off the 1/8 grid"
        assert t.abs().max().item() <= 4, f"|{name}| > 4: q k^T may round in fp32"
    assert torch.equal(v.half().double(), v), "v is not exact in fp16"


def _reference(q, k, v, scale, qk_shared=False):
    """O = softmax(q k^T * scale) v in float64 and the per-element bound on |y - O| for the kernel's output y.

    q [B, H, Lq, d], k, v [B, H, Lk, d] float64, exact as _check_exact requires.  With qk_shared, q and k of sample 0
    serve every sample (VTM_ATTN_SHARED_QK).  Returns (O, bound), each [B, H, Lq, d].

    Bound.  In log2 units t_j = s_j * scale * log2(e) and w_j = 2^(t_j - max t) (so the largest w is 1, l = sum w >= 1),
    O = sum w_j v_j / l.  The kernel's roundings, as relative errors of the weights and sums:
    - scale * log2(e) is rounded to fp32 (with scale itself): a factor (1 + eta), |eta| <= 3 * 2^-24, common to every
      key, so the exponent t_j - m is off by eta * |t_j - m|; the product s_j * scale_log2 and the subtraction of the
      running maximum m each round once: 2^-24 * (|t_j| + |m|) + 2^-24 * |t_j - m|.  With T = max |t| <= 512 and only
      keys with |t_j - m| < 64 carrying weight above 2^-64, the weights are off by at most
      ln 2 * (2^-23 * T + 2^-22 * 64) < 2^-13.8;
    - ex2.approx: relative error below 2^-21; flushed subnormal results lose at most 2^-126 each;
    - P is rounded to fp16 for the P V wgmma, while l sums the unrounded P.  The kernel rounds p = w * 2^(max t - m_tile)
      >= w (m_tile the running maximum) and scales the result back by the later alphas, so the error of one key is at
      most min(w, max(2^-11 w, 2^-25)) <= 2^-11 w + min(w, 2^-25) in units of the final weights;
    - fp32 accumulation: O += P V through the wgmma accumulator (4 k-steps and one alpha rescale per 64-key tile) and l
      through one thread's chain (about 10 roundings per tile).  At Lk <= 16384 (256 tiles) these stay below
      (5 + 10) * 256 * 2^-24 < 2^-12 relative to sum w |v| / l;
    - O * (1 / l) in fp32 (two roundings), then one final rounding to fp16: half an fp16 ulp of the result.
    Relative weight errors act on the numerator sum w v and on l alike, so they cost twice their size in units of
    P|V| = sum w |v| / l (which bounds |O|).  Summed, relative to P|V|:
    2^-11 + 2 * 2^-13.8 + 2 * 2^-21 + 2^-12 + 2^-22 < 1.8 * 2^-11 < 2 * 2^-11, so

        |y - O| <= 2 * 2^-11 * P|V|  +  sum min(w_j, 2^-25) |v_j| / l  +  ulp16(O)

    per element, where the last term holds the final rounding (half an ulp) and the slack when O is near a binade edge.
    Nothing in it depends on the size of other elements of y."""
    B, H, Lq, d = q.shape
    Lk = k.shape[2]
    assert Lk <= 16384
    tl = float(scale) * LOG2E
    if qk_shared:
        q, k = q[:1].expand(B, -1, -1, -1), k[:1].expand(B, -1, -1, -1)
    kt = k.transpose(-1, -2)
    va = v.abs()
    rows = max(1, (1 << 25) // (B * H * Lk))
    outs, bounds = [], []
    for i0 in range(0, Lq, rows):
        t = (q[:, :, i0:i0 + rows] @ kt) * tl
        assert t.abs().max().item() <= 512, "scores beyond the bound's range"
        w = torch.exp2(t - t.amax(-1, keepdim=True))
        l = w.sum(-1, keepdim=True)
        o = (w @ v) / l
        pv = (w @ va) / l
        sub = (w.clamp(max=2.0 ** -25) @ va) / l
        outs.append(o)
        bounds.append(2 * 2.0 ** -11 * pv + sub + _ulp16(o))
    return torch.cat(outs, 2), torch.cat(bounds, 2)


def _heads(t, H):
    """[B, L, C] -> [B, H, L, d] float64."""
    B, L, C = t.shape
    return t.double().view(B, L, H, C // H).transpose(1, 2)


def _assert_within(y, O, bound, what):
    """y [B, L, C] kernel output; O, bound [B, H, L, d]."""
    yh = _heads(y, O.shape[1])
    assert torch.isfinite(yh).all(), f"{what}: non-finite output at {torch.nonzero(~torch.isfinite(yh))[:4].tolist()}"
    ratio = (yh - O).abs() / bound
    worst = ratio.max().item()
    if worst > 1:
        i = tuple(torch.nonzero(ratio == ratio.max())[0].tolist())
        pytest.fail(f"{what}: |y - O| = {abs(yh[i] - O[i]).item():.3e} exceeds the bound {bound[i].item():.3e} "
                    f"at (b, h, row, col) = {i}: y = {yh[i].item()!r}, O = {O[i].item()!r} ({worst:.2f} x bound)")


# ---------------------------------------------------------------------------------------------------------------------
# C-ABI calls with a poisoned workspace

def _stream():
    return torch.cuda.current_stream().cuda_stream


def _poisoned(nbytes):
    return torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")


def _eye(C):
    return torch.eye(C, dtype=torch.float16, device="cuda")


def _self_attention(x, w_qkv, heads, scale, flags=0, len_dev=None):
    """vtm_attention_ex (or vtm_attention_dev with len_dev) with W_o = I, no bias, a 0xFF workspace, a NaN output."""
    lib = _lib.load()
    B, L, C = x.shape
    ws_bytes = lib.vtm_attention_workspace_bytes(B, L, C, heads)
    ws = _poisoned(ws_bytes)
    y = torch.full_like(x, float("nan"))
    wo = _eye(C)
    if len_dev is None:
        _lib.check(lib.vtm_attention_ex(x.data_ptr(), w_qkv.data_ptr(), wo.data_ptr(), None, B, L, C, heads,
                                        float(scale), flags, y.data_ptr(), ws.data_ptr(), ws_bytes, _stream()),
                   "vtm_attention_ex")
    else:
        _lib.check(lib.vtm_attention_dev(x.data_ptr(), w_qkv.data_ptr(), wo.data_ptr(), None, B, L, C, heads,
                                         float(scale), flags, len_dev.data_ptr(), y.data_ptr(), ws.data_ptr(),
                                         ws_bytes, _stream()), "vtm_attention_dev")
    torch.cuda.synchronize()
    return y


def _cross_probe(Q, K, V, heads, scale):
    """vtm_cross_attention with W_q = I, W_k = [I | 0], W_v = [0 | I] (ctx = [K | V]), W_o = I, no bias or residual:
    the flash kernel on exactly Q, K, V."""
    lib = _lib.load()
    B, Lq, C = Q.shape
    Lk = K.shape[1]
    ctx = torch.cat([K, V], -1).contiguous()
    w_q, w_kv = _eye(C), _eye(2 * C)
    ws_bytes = lib.vtm_cross_attention_workspace_bytes(B, Lq, Lk, C, heads)
    ws = _poisoned(ws_bytes)
    y = torch.full_like(Q, float("nan"))
    _lib.check(lib.vtm_cross_attention(Q.data_ptr(), ctx.data_ptr(), w_q.data_ptr(), w_kv.data_ptr(), w_q.data_ptr(),
                                       None, None, B, Lq, Lk, C, 2 * C, heads, float(scale), y.data_ptr(),
                                       ws.data_ptr(), ws_bytes, _stream()), "vtm_cross_attention")
    torch.cuda.synchronize()
    return y


# ---------------------------------------------------------------------------------------------------------------------
# designs

def _grid(shape, g, lo, hi):
    """Uniform multiples of 1/8 in [lo, hi], fp16."""
    return (torch.randint(int(lo * 8), int(hi * 8) + 1, shape, generator=g, device="cuda") / 8).half()


def _ramp(n, rising):
    """n keys' values on the 1/8 grid from -4 to 4 (or 4 to -4): the maximum moves in every 64-key tile."""
    r = torch.round((torch.arange(n, device="cuda", dtype=torch.float64) * 8 / max(n - 1, 1) - 4) * 8) / 8
    return (r if rising else -r).half()


def _probe_design(name, B, Lq, Lk, C, H, g):
    """(Q [B, Lq, C], K [B, Lk, C], V [B, Lk, C], scale) for the cross-attention probe."""
    d = C // H
    V = _grid((B, Lk, C), g, -4, 4)
    if name == "random":
        return _grid((B, Lq, C), g, -2, 2), _grid((B, Lk, C), g, -2, 2), V, d ** -0.5
    if name == "uniform":                       # scale 0: O = the mean of V over exactly the valid keys
        return _grid((B, Lq, C), g, -4, 4), _grid((B, Lk, C), g, -4, 4), V + 64, 0.0
    if name == "offset":                        # a large common offset: an error in l shows directly in O
        return _grid((B, Lq, C), g, -1, 1), _grid((B, Lk, C), g, -1, 1), V + 64, d ** -0.5
    Q = torch.zeros((B, Lq, H, d), dtype=torch.float16, device="cuda")
    K = torch.zeros((B, Lk, H, d), dtype=torch.float16, device="cuda")
    if name == "onehot":
        # each query's designated key scores 16 against 0 for every other key (46 in log2 units at scale 2); the
        # designated keys sit at 0, 63, 64, a middle tile and Lk - 1, each on its own coordinate
        targets = sorted({j for j in (0, 63, 64, Lk // 2, Lk - 1) if j < Lk})
        for c, j in enumerate(targets):
            K[:, j, :, c] = 4
        for b in range(B):
            for h in range(H):
                c = (torch.arange(Lq, device="cuda") + b + 2 * h) % len(targets)
                Q[b, :, h].scatter_(-1, c.view(Lq, 1), 4.0)
        return Q.view(B, Lq, C), K.view(B, Lk, C), V, 2.0
    slope = (1 + torch.arange(Lq, device="cuda") % 4).half()
    if name in ("rising", "falling"):           # t = 1.44 * scale * (1..4) * ramp: |t| <= 23 rising, 92 falling
        Q[..., 0] = slope.view(1, Lq, 1)
        K[..., 0] = _ramp(Lk, name == "rising").view(1, Lk, 1)
        return Q.view(B, Lq, C), K.view(B, Lk, C), V, 1.0 if name == "rising" else 4.0
    if name == "negative":                      # every valid score in [-369, -69] log2 units; keys past Lk score 0
        Q[..., 0] = slope.view(1, Lq, 1)
        K[..., 0] = _grid((B, Lk, H), g, -4, -3)
        return Q.view(B, Lq, C), K.view(B, Lk, C), V, 16.0
    raise ValueError(name)


PROBE_DESIGNS = ("onehot", "uniform", "rising", "falling", "negative", "offset", "random")


def _signed_perm(C, H, shift, sign, g):
    """[C, C] fp16: output head h takes a random signed permutation of input head (h + shift) % H's columns
    (sign=+1/-1: all signs that; 0: random signs)."""
    d = C // H
    W = torch.zeros((C, C), dtype=torch.float64, device="cuda")
    for h in range(H):
        src = ((h + shift) % H) * d
        perm = torch.randperm(d, generator=g, device="cuda")
        s = (torch.randint(0, 2, (d,), generator=g, device="cuda") * 2 - 1).double() if sign == 0 else \
            torch.full((d,), float(sign), dtype=torch.float64, device="cuda")
        W[h * d + torch.arange(d, device="cuda"), src + perm] = s
    assert torch.equal((W != 0).sum(1), torch.ones(C, dtype=torch.long, device="cuda"))
    return W.half()


def _self_design(name, B, L, C, H, g):
    """(x [B, L, C], W_qkv [3C, C], scale) for self-attention."""
    d = C // H
    if name == "random":
        x = _grid((B, L, C), g, -2, 2)
        signs, scale = (0, 0, 0), d ** -0.5
    elif name == "uniform":                     # scale 0: O = the mean of v (all in [3, 4]) over the valid keys
        x = _grid((B, L, C), g, 3, 4)
        signs, scale = (0, 0, 1), 0.0
    elif name == "negative":                    # q in [3, 4], k in [-4, -3]: every valid score < 0, |t| up to 400
        x = _grid((B, L, C), g, 3, 4)
        signs, scale = (1, -1, 1), 400 / (16 * d * LOG2E)
    else:
        raise ValueError(name)
    w = torch.cat([_signed_perm(C, H, s, sg, g) for s, sg in zip((0, 1, 2), signs)], 0).contiguous()
    return x, w, scale


SELF_DESIGNS = ("random", "uniform", "negative")


def _self_qkv(x, w, H):
    C = x.shape[-1]
    xd = x.double()
    q, k, v = (_heads(xd @ w[i * C:(i + 1) * C].double().t(), H) for i in range(3))
    _check_exact(q, k, v)
    return q, k, v


def _run_probe(name, B, Lq, Lk, d, H, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    Q, K, V, scale = _probe_design(name, B, Lq, Lk, d * H, H, g)
    q, k, v = _heads(Q, H), _heads(K, H), _heads(V, H)
    _check_exact(q, k, v)
    O, bound = _reference(q, k, v, scale)
    y = _cross_probe(Q, K, V, H, scale)
    _assert_within(y, O, bound, f"cross probe {name} B={B} Lq={Lq} Lk={Lk} d={d} H={H}")


def _run_self(name, B, L, d, H, seed, flags=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x, w, scale = _self_design(name, B, L, d * H, H, g)
    q, k, v = _self_qkv(x, w, H)
    O, bound = _reference(q, k, v, scale, qk_shared=bool(flags & 1))
    y = _self_attention(x, w, H, scale, flags=flags)
    _assert_within(y, O, bound, f"self-attention {name} B={B} L={L} d={d} H={H} flags={flags}")


# ---------------------------------------------------------------------------------------------------------------------
# shapes

HEAD_DIMS = tuple(range(8, 129, 8))                 # KS 1..8, CW 3 and 2, DP 64 and 128, one and two TMA atoms


@pytest.mark.parametrize("name", PROBE_DESIGNS)
@pytest.mark.parametrize("d", HEAD_DIMS)
def test_cross_probe_head_dims(d, name):
    _run_probe(name, 2, 193, 129, d, 3, seed=d)


@pytest.mark.parametrize("name", SELF_DESIGNS)
@pytest.mark.parametrize("d", HEAD_DIMS)
def test_self_attention_head_dims(d, name):
    _run_self(name, 2, 193, d, 3, seed=d)


def _bh(i, d, one):
    """(B, H) for the i-th length at head_dim d, cycling through a covering set; a length-1 case needs B >= 2 and H >= 2
    (with H = 1 the slots of a misplaced row can coincide with the right ones)."""
    cycle = ((2, 2), (3, 5), (2, 5), (3, 2)) if one else ((1, 1), (2, 2), (3, 5), (1, 2), (2, 5), (3, 1))
    return cycle[(3 * i + (40, 80, 128).index(d)) % len(cycle)]


_CROSS_LENGTHS = sorted({(lq, 129) for lq in LENGTHS} | {(193, lk) for lk in LENGTHS + (77,)})


@pytest.mark.parametrize("d", (40, 80, 128))
@pytest.mark.parametrize("Lq,Lk", _CROSS_LENGTHS)
def test_cross_probe_lengths(Lq, Lk, d):
    B, H = _bh(_CROSS_LENGTHS.index((Lq, Lk)), d, min(Lq, Lk) == 1)
    for name in PROBE_DESIGNS:
        _run_probe(name, B, Lq, Lk, d, H, seed=1000 * Lq + Lk)


@pytest.mark.parametrize("d", (40, 80, 128))
@pytest.mark.parametrize("L", LENGTHS)
def test_self_attention_lengths(L, d):
    B, H = _bh(LENGTHS.index(L), d, L == 1)
    for name in SELF_DESIGNS:
        _run_self(name, B, L, d, H, seed=L)


@pytest.mark.parametrize("name", ("random", "negative"))
def test_self_attention_full_size_c2_ds1(name):
    """BASELINE config 2, ds1 merged length: B = 2, L = 10241, C = 320, 8 heads of 40."""
    _run_self(name, 2, 10241, 40, 8, seed=7)


@pytest.mark.parametrize("L,d", [(1, 40), (65, 40), (193, 128), (1000, 80)])
def test_shared_qk(L, d):
    """VTM_ATTN_SHARED_QK: q and k of sample 0 for every sample, v of each sample."""
    for name in SELF_DESIGNS:
        _run_self(name, 3, L, d, 2, seed=L + d, flags=1)


@pytest.mark.parametrize("d,B,H", [(40, 2, 2), (80, 2, 5), (128, 3, 2)])
@pytest.mark.parametrize("n", (1, 63, 64, 65, 193, 449))
def test_device_length(n, d, B, H):
    """vtm_attention_dev at a capacity of 449 rows with the first n valid: rows past n hold +-1000, which would win
    every softmax if they took part.  Rows < n meet the bound against the reference at L = n and equal
    vtm_attention_ex at L = n bit for bit."""
    cap = 449
    for name in SELF_DESIGNS:
        g = torch.Generator(device="cuda").manual_seed(n + d)
        x, w, scale = _self_design(name, B, n, d * H, H, g)
        big = (torch.randint(0, 2, (B, cap - n, d * H), generator=g, device="cuda") * 2000 - 1000).half()
        xc = torch.cat([x, big], 1).contiguous()
        q, k, v = _self_qkv(x, w, H)
        O, bound = _reference(q, k, v, scale)
        y = _self_attention(xc, w, H, scale, len_dev=torch.tensor([n], dtype=torch.int32, device="cuda"))
        _assert_within(y[:, :n], O, bound, f"device length {name} n={n} d={d}")
        assert torch.equal(y[:, :n], _self_attention(x, w, H, scale)), f"{name} n={n} d={d}"


def test_block_cross_attention_one_token_context():
    """A patched block whose attn2 gets a 1-token context: the fast path (vtm_cross_attention, K and V projected from
    one row per item) equals the module path."""
    import vidtome_b200
    from vidtome_b200 import attention, patch
    from vidtome_b200.skeleton import make_skeleton
    outs = []
    for fast in (True, False):
        patch.FUSE_CROSS_ATTENTION = fast
        try:
            net = make_skeleton("tiny", device="cuda", hot_path_only=False, seed=11)
            vidtome_b200.apply_patch(net, batch_size=2, max_downsample=0)
            torch.manual_seed(2); torch.cuda.manual_seed(2)
            lat = torch.randn(2 * 4, 4, 16, 16, device="cuda", dtype=torch.float16)
            ctx = torch.randn(2 * 4, 1, 768, device="cuda", dtype=torch.float16)
            assert all(attention.cross_attention_eligible(b.attn2, ctx) for b in net.blocks)
            with torch.no_grad():
                outs.append(net(lat, 0, encoder_hidden_states=ctx).sample.float())
        finally:
            patch.FUSE_CROSS_ATTENTION = True
    assert torch.isfinite(outs[0]).all()
    err = (outs[0] - outs[1]).abs().max().item()
    assert err <= 3e-3 * outs[1].abs().max().item()
