"""LoRA-adapted projections on the H100: the GEMMs' K tail against float64 references bit for bit, R = 0 / NULL against
the entry points without LoRA, LoRA-adapted attention and feed-forward modules against their own math, a patched
SD1.5 skeleton with adapters on every projection, and CUDA-graph stepping with LoRA against eager stepping.

Exact inputs (as in test_gpu_projection_core.py): x on a 1/8 grid, W on a 1/16 grid, the bias on the 2^-7 grid; every row
of the down matrix D holds 8 non-zeros of +-1/16 or +-1/8, so that T = x D^T is a multiple of 2^-7 below 8 in
magnitude and exact in fp16; U on a 1/16 grid with |u| <= 1.  Every product is then a multiple of 2^-11 and, with
sum |x w| + |b| + sum |t u| < 2^13, every partial sum is exact in fp32: the kernels' only approximations left are their
fp16 roundings, so outputs are compared bit for bit with float64 results rounded once."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

import test_gpu_projection_core as pc
from vidtome_b200 import _lib, ops

pytestmark = pytest.mark.gpu

RANKS = (8, 56, 64, 72, 200)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ref(desc):
    return None if desc is None else C.byref(desc)


def _tail(R, K, N, g):
    """D [R, K] with 8 non-zeros per row (fewer when K < 8) and U [N, R] on the 1/16 grid, |u| <= 1."""
    nz = min(8, K)
    idx = torch.rand((R, K), generator=g, device="cuda").argsort(1)[:, :nz]
    mag = torch.randint(1, 3, (R, nz), generator=g, device="cuda").double() / 16
    sgn = torch.randint(0, 2, (R, nz), generator=g, device="cuda").double() * 2 - 1
    D = torch.zeros((R, K), dtype=torch.float64, device="cuda").scatter_(1, idx, mag * sgn).half()
    U = pc._grid((N, R), 1 / 16, 1, g)
    return D, U


def _exact_lora(x, w, b, D, U):
    """x W^T + b + T U^T in float64 with T = x D^T, asserting the conditions under which the kernels are exact."""
    x64, w64 = x.double(), w.double()
    T = x64 @ D.double().t()
    assert torch.equal(T * 128, torch.round(T * 128)) and T.abs().max().item() < 8, "T not exact in fp16"
    S = x64.abs() @ w64.abs().t() + T.abs() @ U.double().abs().t()
    r = x64 @ w64.t() + T @ U.double().t()
    if b is not None:
        S = S + b.double().abs()
        r = r + b.double()
    assert S.max().item() < 2.0 ** 13, "partial sums may round in fp32"
    return r


def _linear_lora(a, w, b, D, U, ldd, resid=None, ldr=0, desc_r=None):
    """vtm_linear_lora_f16 into a guarded output; D = None passes a NULL descriptor, desc_r = 0 an empty one."""
    lib = _lib.load()
    M, K = a.shape
    N = w.shape[0]
    d = pc._guarded(M, N, ldd)
    if D is None:
        desc, R = (None, 0) if desc_r is None else (_lib.VtmLora(None, None, 0), 0)
    else:
        R = D.shape[0]
        desc = _lib.VtmLora(D.data_ptr(), U.data_ptr(), R)
    ws_bytes = lib.vtm_linear_lora_workspace_bytes(M, R)
    ws = torch.full((max(ws_bytes, 16),), 0xFF, dtype=torch.uint8, device="cuda")
    _lib.check(lib.vtm_linear_lora_f16(a.data_ptr(), w.data_ptr(), pc._ptr(b), pc._ptr(resid), ldr, _ref(desc), M, N, K,
                                       d.data_ptr(), ldd, ws.data_ptr(), ws_bytes, _stream()), "vtm_linear_lora_f16")
    torch.cuda.synchronize()
    what = f"linear lora M={M} N={N} K={K} R={R} ldd={ldd} resid={resid is not None}"
    pc._check_guards(d, M, N, what)
    return d[:M, :N], what


def _geglu_lora(a, w_il, b_il, D, U_il, ldd):
    lib = _lib.load()
    M, K = a.shape
    N = w_il.shape[0]
    d = pc._guarded(M, N // 2, ldd)
    desc = None if D is None else _lib.VtmLora(D.data_ptr(), U_il.data_ptr(), D.shape[0])
    R = 0 if D is None else D.shape[0]
    ws_bytes = lib.vtm_linear_lora_workspace_bytes(M, R)
    ws = torch.full((max(ws_bytes, 16),), 0xFF, dtype=torch.uint8, device="cuda")
    _lib.check(lib.vtm_linear_geglu_lora_f16(a.data_ptr(), w_il.data_ptr(), pc._ptr(b_il), _ref(desc), M, N, K,
                                             d.data_ptr(), ldd, ws.data_ptr(), ws_bytes, _stream()),
               "vtm_linear_geglu_lora_f16")
    torch.cuda.synchronize()
    what = f"geglu lora M={M} N={N} K={K} R={R} ldd={ldd}"
    pc._check_guards(d, M, N // 2, what)
    return d[:M, :N // 2], what


# ---------------------------------------------------------------------------------------------------------------------
# store and residual epilogues, exact

LINEAR_CASES = ([(161, 136, 200, R) for R in RANKS] +
                [(33, 72, 24, 56), (1, 264, 8, 200), (4099, 320, 320, 64), (129, 8, 136, 72), (65, 200, 72, 8),
                 (257, 1280, 640, 64)])


@pytest.mark.parametrize("M,N,K,R", LINEAR_CASES)
def test_linear_lora_exact(M, N, K, R):
    g = torch.Generator(device="cuda").manual_seed(M + N + K + R)
    a, w, b = pc._exact_inputs(M, N, K, g)
    D, U = _tail(R, K, N, g)
    r = _exact_lora(a, w, b, D, U)
    y, what = _linear_lora(a, w, b, D, U, ldd=N + 24)
    pc._assert_equal(y, pc._round16(r), what)
    ldr = N + 8
    resid = torch.full((M, ldr), float("nan"), dtype=torch.float16, device="cuda")
    resid[:, :N] = (torch.randn((M, N), generator=g, device="cuda") * 64).half()
    y2, what2 = _linear_lora(a, w, b, D, U, ldd=N, resid=resid, ldr=ldr)
    pc._assert_equal(y2, pc._round16(pc._round16(r) + resid[:, :N].double()), what2)


# ---------------------------------------------------------------------------------------------------------------------
# GEGLU epilogue, exact

@pytest.mark.parametrize("inner,R", [(32, 8), (96, 72), (160, 200), (1280, 64), (1312, 56)])
def test_geglu_lora_exact(inner, R):
    M, K = pc.RAGGED_M, pc.RAGGED_K
    g = torch.Generator(device="cuda").manual_seed(inner + R)
    a, w, b = pc._exact_inputs(M, 2 * inner, K, g)
    w[inner:] = pc._grid((inner, K), 1 / 16, max(1, round(48 / (1.78 * K) ** 0.5)) / 16, g)
    D, U = _tail(R, K, 2 * inner, g)
    wi, bi = ops.interleave_geglu(w, b)
    ui, _ = ops.interleave_geglu(U, None)
    y, what = _geglu_lora(a, wi, bi, D, ui, ldd=inner + 8)
    r = pc._round16(_exact_lora(a, w, b, D, U))
    want, alt, near = pc._geglu_reference(r[:, :inner], r[:, inner:])
    yd = y.double()
    ok = (yd == want) | (near & (yd == alt))
    assert ok.all(), f"{what}: {int((~ok).sum())} elements differ"


# ---------------------------------------------------------------------------------------------------------------------
# head-split epilogue (self: plain, shared, device length; cross: q and kv), exact

def _attn_lora(x, w_qkv, w_o, b_o, lq, lo, H, flags=0, len_dev=None, scale=0.0, ws_fill=0xFF):
    lib = _lib.load()
    B, L, Cc = x.shape
    rq = 0 if lq is None else lq[0].shape[0]
    ro = 0 if lo is None else lo[0].shape[0]
    dq = None if lq is None else _lib.VtmLora(lq[0].data_ptr(), lq[1].data_ptr(), rq)
    do = None if lo is None else _lib.VtmLora(lo[0].data_ptr(), lo[1].data_ptr(), ro)
    ws_bytes = lib.vtm_attention_lora_workspace_bytes(B, L, Cc, H, rq, ro)
    ws = torch.full((ws_bytes,), ws_fill, dtype=torch.uint8, device="cuda")
    y = torch.full_like(x, float("nan"))
    _lib.check(lib.vtm_attention_lora(x.data_ptr(), w_qkv.data_ptr(), w_o.data_ptr(), pc._ptr(b_o), _ref(dq), _ref(do),
                                      B, L, Cc, H, scale, flags, pc._ptr(len_dev), y.data_ptr(), ws.data_ptr(),
                                      ws_bytes, _stream()), "vtm_attention_lora")
    torch.cuda.synchronize()
    return y, ws


def _self_problem(B, L, d, H, R, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    Cc = d * H
    x, w, _ = pc._exact_inputs(B * L, 3 * Cc, Cc, g, bias=False)
    D, U = _tail(R, Cc, 3 * Cc, g)
    proj = _exact_lora(x, w, None, D, U).view(B * L, 3, Cc).permute(1, 0, 2)
    return x.view(B, L, Cc), w, D, U, proj


SELF_CASES = [(2, 33, 40, 3, 8), (3, 1, 64, 2, 56), (1, 65, 72, 4, 64), (2, 64, 128, 2, 72), (3, 31, 8, 5, 200),
              (2, 3, 80, 1, 8)]


@pytest.mark.parametrize("B,L,d,H,R", SELF_CASES)
def test_head_split_self_lora_exact(B, L, d, H, R):
    x, w, D, U, proj = _self_problem(B, L, d, H, R, seed=B * 1000 + L * 10 + d + R)
    Cc = d * H
    DP = 64 if d <= 64 else 128
    wo = torch.eye(Cc, dtype=torch.float16, device="cuda")
    _, ws = _attn_lora(x, w, wo, None, (D, U), None, H)
    pc._check_head_major(ws.view(torch.float16), 0, proj, B, H, L, d, DP, f"self lora B={B} L={L} d={d} R={R}")
    # the device length projects every row of the capacity: the same head-major buffers
    n = torch.tensor([max(1, L - 2)], dtype=torch.int32, device="cuda")
    _, ws2 = _attn_lora(x, w, wo, None, (D, U), None, H, len_dev=n)
    pc._check_head_major(ws2.view(torch.float16), 0, proj, B, H, L, d, DP, f"self lora dev B={B} L={L} d={d} R={R}")


@pytest.mark.parametrize("B,L,d,H,R", SELF_CASES)
def test_head_split_shared_lora_exact(B, L, d, H, R):
    """VTM_ATTN_SHARED_QK: q and k of sample 0 (with the tail rows of sample 0), v of every sample (U rows [2C, 3C))."""
    x, w, D, U, proj = _self_problem(B, L, d, H, R, seed=B * 1000 + L * 10 + d + R + 1)
    Cc = d * H
    DP = 64 if d <= 64 else 128
    wo = torch.eye(Cc, dtype=torch.float16, device="cuda")
    _, ws = _attn_lora(x, w, wo, None, (D, U), None, H, flags=1)
    qkv = ws.view(torch.float16)[:3 * B * H * L * DP].view(3, B, H, L, DP)
    want = pc._round16(proj).view(3, B, L, H, d).transpose(2, 3)
    what = f"shared lora B={B} L={L} d={d} R={R}"
    pc._assert_equal(qkv[:2, :1, ..., :d], want[:2, :1], what + ": q / k of sample 0")
    pc._assert_equal(qkv[2, ..., :d], want[2], what + ": v")
    assert (qkv[:2, 1:].view(torch.int16) == -1).all(), what + ": q / k of other samples written"


@pytest.mark.parametrize("Lq,Lk,d,H,R", [(33, 77, 40, 2, 8), (3, 65, 64, 3, 56), (65, 1, 80, 2, 72), (31, 33, 128, 1, 200)])
def test_head_split_cross_lora_exact(Lq, Lk, d, H, R):
    lib = _lib.load()
    B, Cctx = 2, 768
    g = torch.Generator(device="cuda").manual_seed(Lq + Lk + d + R)
    Cc = d * H
    DP = 64 if d <= 64 else 128
    x, w_q, _ = pc._exact_inputs(B * Lq, Cc, Cc, g, bias=False)
    ctx, w_kv, _ = pc._exact_inputs(B * Lk, 2 * Cc, Cctx, g, bias=False)
    Dq, Uq = _tail(R, Cc, Cc, g)
    Dkv, Ukv = _tail(R + 8, Cctx, 2 * Cc, g)
    dq, dkv = _lib.VtmLora(Dq.data_ptr(), Uq.data_ptr(), R), _lib.VtmLora(Dkv.data_ptr(), Ukv.data_ptr(), R + 8)
    ws_bytes = lib.vtm_cross_attention_lora_workspace_bytes(B, Lq, Lk, Cc, H, R, R + 8, 0)
    ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device="cuda")
    y = torch.full((B, Lq, Cc), float("nan"), dtype=torch.float16, device="cuda")
    wo = torch.eye(Cc, dtype=torch.float16, device="cuda")
    _lib.check(lib.vtm_cross_attention_lora(x.data_ptr(), ctx.data_ptr(), w_q.data_ptr(), w_kv.data_ptr(), wo.data_ptr(),
                                            None, None, C.byref(dq), C.byref(dkv), None, B, Lq, Lk, Cc, Cctx, H, 0.0,
                                            y.data_ptr(), ws.data_ptr(), ws_bytes, _stream()), "vtm_cross_attention_lora")
    torch.cuda.synchronize()
    wsh = ws.view(torch.float16)
    what = f"cross lora Lq={Lq} Lk={Lk} d={d} R={R}"
    pc._check_head_major(wsh, 0, _exact_lora(x, w_q, None, Dq, Uq).unsqueeze(0), B, H, Lq, d, DP, what)
    kv = _exact_lora(ctx, w_kv, None, Dkv, Ukv).view(B * Lk, 2, Cc).permute(1, 0, 2)
    pc._check_head_major(wsh[B * H * Lq * DP:], 1, kv, B, H, Lk, d, DP, what)


def test_output_projection_lora_follows_the_flash_kernel():
    """to_out's T is computed from the attention output o: vtm_attention_lora with lora_o equals o (an identity output
    projection) sent through vtm_linear_lora_f16 with the same LoRA, bit for bit; self (plain, shared, device length)
    and cross (with the residual)."""
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(3)
    B, L, H, d = 3, 200, 4, 40
    Cc = H * d
    x = torch.randn((B, L, Cc), generator=g, device="cuda").half()
    w = (torch.randn((3 * Cc, Cc), generator=g, device="cuda") / Cc ** 0.5).half()
    wo = (torch.randn((Cc, Cc), generator=g, device="cuda") / Cc ** 0.5).half()
    bo = torch.randn((Cc,), generator=g, device="cuda").half()
    eye = torch.eye(Cc, dtype=torch.float16, device="cuda")
    Do = (torch.randn((24, Cc), generator=g, device="cuda") / Cc ** 0.5).half()
    Uo = (torch.randn((Cc, 24), generator=g, device="cuda") * 0.2).half()
    n = torch.tensor([171], dtype=torch.int32, device="cuda")
    for flags, len_dev in ((0, None), (1, None), (0, n), (1, n)):
        o, _ = _attn_lora(x, w, eye, None, None, None, H, flags=flags, len_dev=len_dev, scale=d ** -0.5)
        y, _ = _attn_lora(x, w, wo, bo, None, (Do, Uo), H, flags=flags, len_dev=len_dev, scale=d ** -0.5)
        rows = L if len_dev is None else 171
        want, _ = _linear_lora(o[:, :rows].reshape(-1, Cc).contiguous(), wo, bo, Do, Uo, ldd=Cc)
        assert torch.equal(y[:, :rows].reshape(-1, Cc), want), (flags, len_dev is not None)
    # cross-attention with the residual
    Lk, Cctx = 77, 768
    ctx = torch.randn((B, Lk, Cctx), generator=g, device="cuda").half()
    wq = (torch.randn((Cc, Cc), generator=g, device="cuda") / Cc ** 0.5).half()
    wkv = (torch.randn((2 * Cc, Cctx), generator=g, device="cuda") / Cctx ** 0.5).half()
    resid = torch.randn((B, L, Cc), generator=g, device="cuda").half()

    def cross(w_o, b_o, lo, res):
        desc = None if lo is None else _lib.VtmLora(lo[0].data_ptr(), lo[1].data_ptr(), lo[0].shape[0])
        ws_bytes = lib.vtm_cross_attention_lora_workspace_bytes(B, L, Lk, Cc, H, 0, 0, 0 if lo is None else 24)
        ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device="cuda")
        out = torch.full_like(x, float("nan"))
        _lib.check(lib.vtm_cross_attention_lora(x.data_ptr(), ctx.data_ptr(), wq.data_ptr(), wkv.data_ptr(), w_o.data_ptr(),
                                                pc._ptr(b_o), pc._ptr(res), None, None, _ref(desc), B, L, Lk, Cc, Cctx, H,
                                                d ** -0.5, out.data_ptr(), ws.data_ptr(), ws_bytes, _stream()),
                   "vtm_cross_attention_lora")
        torch.cuda.synchronize()
        return out
    o = cross(eye, None, None, None)
    y = cross(wo, bo, (Do, Uo), resid)
    want, _ = _linear_lora(o.view(-1, Cc), wo, bo, Do, Uo, ldd=Cc, resid=resid.view(-1, Cc), ldr=Cc)
    assert torch.equal(y.view(-1, Cc), want)


# ---------------------------------------------------------------------------------------------------------------------
# R = 0 and NULL descriptors: the entry points without LoRA, bit for bit

def test_empty_lora_is_the_plain_entry_point():
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(11)
    M, N, K = 1000, 320, 1280
    a = torch.randn((M, K), generator=g, device="cuda").half()
    w = (torch.randn((N, K), generator=g, device="cuda") / K ** 0.5).half()
    b = torch.randn((N,), generator=g, device="cuda").half()
    resid = torch.randn((M, N), generator=g, device="cuda").half()
    plain, _ = pc._linear(a, w, b, ldd=N)
    plain_r, _ = pc._linear(a, w, b, ldd=N, resid=resid, ldr=N)
    for desc_r in (None, 0):
        assert torch.equal(_linear_lora(a, w, b, None, None, ldd=N, desc_r=desc_r)[0], plain)
        assert torch.equal(_linear_lora(a, w, b, None, None, ldd=N, resid=resid, ldr=N, desc_r=desc_r)[0], plain_r)
    wi, bi = ops.interleave_geglu(torch.cat([w, w.flip(0)]), torch.cat([b, b]))
    assert torch.equal(_geglu_lora(a, wi, bi, None, None, ldd=N)[0], pc._geglu(a, wi, bi)[0])
    # attention: NULL descriptors and R = 0 descriptors against vtm_attention_ex / _dev / vtm_cross_attention
    B, L, H, d = 2, 300, 8, 40
    Cc = H * d
    x = torch.randn((B, L, Cc), generator=g, device="cuda").half()
    wqkv = (torch.randn((3 * Cc, Cc), generator=g, device="cuda") / Cc ** 0.5).half()
    wo = (torch.randn((Cc, Cc), generator=g, device="cuda") / Cc ** 0.5).half()
    n = torch.tensor([257], dtype=torch.int32, device="cuda")
    zero = _lib.VtmLora(None, None, 0)
    for flags in (0, 1):
        want = ops.attention(x, wqkv, wo, b, H, d ** -0.5, shared_qk=bool(flags))
        want_dev = ops.attention(x, wqkv, wo, b, H, d ** -0.5, shared_qk=bool(flags), seq_len=n)
        for len_dev, ref in ((None, want), (n, want_dev)):
            for descs in ((None, None), (zero, zero)):
                ws_bytes = lib.vtm_attention_lora_workspace_bytes(B, L, Cc, H, 0, 0)
                ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
                y = torch.empty_like(x)
                _lib.check(lib.vtm_attention_lora(x.data_ptr(), wqkv.data_ptr(), wo.data_ptr(), b.data_ptr(),
                                                  _ref(descs[0]), _ref(descs[1]), B, L, Cc, H, d ** -0.5, flags,
                                                  pc._ptr(len_dev), y.data_ptr(), ws.data_ptr(), ws_bytes, _stream()),
                           "vtm_attention_lora")
                rows = L if len_dev is None else 257
                assert torch.equal(y[:, :rows], ref[:, :rows]), (flags, len_dev is not None, descs[0] is None)
    ctx = torch.randn((B, 77, 768), generator=g, device="cuda").half()
    wq = (torch.randn((Cc, Cc), generator=g, device="cuda") / Cc ** 0.5).half()
    wkv = (torch.randn((2 * Cc, 768), generator=g, device="cuda") / 768 ** 0.5).half()
    want = ops.cross_attention(x, ctx, wq, wkv, wo, b, H, d ** -0.5, resid=x)
    for desc in (None, zero):
        ws_bytes = lib.vtm_cross_attention_lora_workspace_bytes(B, L, 77, Cc, H, 0, 0, 0)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
        y = torch.empty_like(x)
        _lib.check(lib.vtm_cross_attention_lora(x.data_ptr(), ctx.data_ptr(), wq.data_ptr(), wkv.data_ptr(),
                                                wo.data_ptr(), b.data_ptr(), x.data_ptr(), _ref(desc), _ref(desc),
                                                _ref(desc), B, L, 77, Cc, 768, H, d ** -0.5, y.data_ptr(), ws.data_ptr(),
                                                ws_bytes, _stream()), "vtm_cross_attention_lora")
        assert torch.equal(y, want)


# ---------------------------------------------------------------------------------------------------------------------
# modules: LoRA-adapted attn1 / attn2 / ff against float64 module math and the fp16 module forward

FORMS = [("diffusers", None), ("peft", None), ("peft", torch.float32)]


def _lora_block(form, adapter_dtype, dim, heads=8, rank=32, seed=0):
    from vidtome_b200.skeleton import BasicTransformerBlock, add_lora
    torch.manual_seed(seed)
    blk = BasicTransformerBlock(dim, heads, 768, hot_path_only=False).cuda().half()
    return add_lora(blk, rank, form, dtype=adapter_dtype, seed=seed + 1)


def _close(got, want16, ref64, what, tol16=3e-3):
    s = ref64.abs().max().item()
    e64 = (got.double() - ref64).abs().max().item()
    e16 = (got.double() - want16.double()).abs().max().item()
    assert e64 <= 2e-3 * s, f"{what}: {e64:.3e} from float64 (scale {s:.3e})"
    assert e16 <= tol16 * s, f"{what}: {e16:.3e} from the fp16 module forward (scale {s:.3e})"


@pytest.mark.parametrize("dim", [320, 640])
@pytest.mark.parametrize("form,adapter_dtype", FORMS)
def test_lora_modules_match_module_math(form, adapter_dtype, dim):
    """SD1.5's ds1 and ds2 widths: head_dim 40 and 80."""
    from vidtome_b200 import attention, feedforward, patch
    blk = _lora_block(form, adapter_dtype, dim)
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn((2, 1000, dim), generator=g, device="cuda").half()
    ctx = torch.randn((2, 77, 768), generator=g, device="cuda").half()
    what = f"{form} {adapter_dtype} C={dim}"
    assert patch._plain_attention_module(blk.attn1)
    with torch.no_grad():
        blk64 = copy.deepcopy(blk).double()
        got = attention.self_attention(blk.attn1, x)
        _close(got, blk.attn1(x), blk64.attn1(x.double()), what + " attn1")
        assert attention.cross_attention_eligible(blk.attn2, ctx)
        got = attention.cross_attention_residual(blk.attn2, x, ctx, x)
        _close(got, blk.attn2(x, encoder_hidden_states=ctx) + x,
               blk64.attn2(x.double(), encoder_hidden_states=ctx.double()) + x.double(), what + " attn2")
        parts = feedforward.geglu_parts(blk.ff)
        assert parts is not None
        ln = (blk.norm3.weight, blk.norm3.bias, blk.norm3.eps)
        got = feedforward.feed_forward_residual(blk.ff, parts, ln, x)
        _close(got, blk.ff(blk.norm3(x)) + x, blk64.ff(blk64.norm3(x.double())) + x.double(), what + " ff")


# ---------------------------------------------------------------------------------------------------------------------
# a patched SD1.5 skeleton with LoRA on every projection, at C2's ds1 and ds2 shapes

def _skeleton_divergence(form, monkeypatch, calls):
    """Relative L2 difference of a patched SD1.5 skeleton (ds1 and ds2 blocks, full blocks) at C2 between the library and
    the modules' own forward, with LoRA on every projection (form) or without LoRA (form None).  The library's path runs
    first, with `calls` recording the wrappers' forwards."""
    import vidtome_b200
    from vidtome_b200 import attention, patch, skeleton
    net = skeleton.make_skeleton("sd15", hot_path_only=False, max_downsample=2, device="cuda")
    if form is not None:
        skeleton.add_lora(net, 32, form)
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, batch_size=2)
    g = torch.Generator(device="cuda").manual_seed(4)
    lat = torch.randn((2 * 16, 4, 64, 64), generator=g, device="cuda").half()       # 16 frames, 512 x 512, CFG
    cond = torch.randn((2 * 16, 77, 768), generator=g, device="cuda").half()
    ops.STATS.reset()
    with torch.no_grad():
        torch.manual_seed(0)
        out = net(lat, 0, encoder_hidden_states=cond).sample
    torch.cuda.synchronize()
    lib_calls, launches = len(calls), ops.STATS.launches
    with monkeypatch.context() as mp:
        mp.setattr(attention, "ENABLED", False)
        mp.setattr(patch, "FUSE_CROSS_ATTENTION", False)
        mp.setattr(patch, "FUSE_FEED_FORWARD", False)
        with torch.no_grad():
            torch.manual_seed(0)
            ref = net(lat, 0, encoder_hidden_states=cond).sample
    assert torch.isfinite(out).all() and torch.isfinite(ref).all()
    rel = ((out.float() - ref.float()).norm() / ref.float().norm()).item()
    return rel, lib_calls, len(calls) - lib_calls, launches, len(net.blocks)


@pytest.mark.parametrize("form", ["diffusers", "peft"])
def test_patched_skeleton_runs_lora_in_the_library(form, monkeypatch):
    """The library path runs (no wrapper forward is called, the LoRA T launches are counted), and the output is as close
    to the modules' own forward as the library's output without LoRA is to its own.  Neither is bit-identical: the
    library's projections and attention round differently from the modules', and a merging level whose similarity
    ties then fall the other way picks another dst token, which changes a few outputs by more than a rounding."""
    from vidtome_b200 import skeleton
    calls = []
    cls = skeleton.PeftLoraLinear if form == "peft" else skeleton.LoRACompatibleLinear
    orig = cls.forward
    monkeypatch.setattr(cls, "forward", lambda self, *a, **k: (calls.append(1), orig(self, *a, **k))[1])
    rel, lib_calls, off_calls, launches, blocks = _skeleton_divergence(form, monkeypatch, calls)
    assert lib_calls == 0, f"{lib_calls} LoRA wrapper forwards ran: a projection left the library"
    assert off_calls > 0, "the wrappers' own forwards did not run with the library switched off"
    # per block at least: KD (3 + 2 LoRA T launches), XA (4 + 3), LayerNorm + FF (1 + 2 + 2)
    assert launches >= blocks * (5 + 7 + 5), launches
    rel_plain, *_ = _skeleton_divergence(None, monkeypatch, [])
    print(f"relative L2 difference library vs modules: {rel:.3e} with LoRA ({form}), {rel_plain:.3e} without")
    assert rel <= 1.5 * rel_plain + 2e-3, f"with LoRA {rel:.3e}, without {rel_plain:.3e}"


# ---------------------------------------------------------------------------------------------------------------------
# the step driver: CUDA graphs with LoRA are bit-identical to eager stepping

def _drive(graph: bool, pnp: bool, steps: int = 6, frames: int = 8, size: int = 16):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import add_lora, make_skeleton, pnp_attention_modules
    torch.manual_seed(77)
    net = make_skeleton("sd15", hot_path_only=False, max_downsample=2, device="cuda")
    add_lora(net, 16, "peft")
    batch = 3 if pnp else 2
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, batch_size=batch, align_batch=pnp)
    g = torch.Generator(device="cuda").manual_seed(5)
    cond = torch.randn((batch, 77, 768), generator=g, device="cuda").half()
    kw = dict(cuda_graph=graph, graph_warmup=1 if pnp else 2)
    if pnp:
        sources = {}

        def source(t):
            if t not in sources:
                gs = torch.Generator(device="cuda").manual_seed(int(t))
                sources[t] = torch.randn((frames, 4, size, size), generator=gs, device="cuda").half()
            return sources[t]
        kw.update(randomize_chunks=True, chunk_graphs=graph, source_latents=source, pnp_attn_t=0.5,
                  pnp_modules=pnp_attention_modules(net), chunk_ord="mix-4")
    den = ChunkedDenoiser(net, n_timesteps=steps if pnp else 50, chunk_size=4 if pnp else frames, cond=cond, **kw)
    x = torch.randn((frames, 4, size, size), generator=g, device="cuda", dtype=torch.float16)
    torch.manual_seed(2024)
    np.random.seed(2024)
    xs = []
    for i in range(steps):
        x = den.step(x, i)
        xs.append(x.clone())
    torch.cuda.synchronize()
    return xs, den


@pytest.mark.parametrize("pnp", [False, True])
def test_driver_graphs_with_lora_are_bit_identical_to_eager(pnp):
    eager, _ = _drive(False, pnp)
    graph, den = _drive(True, pnp)
    if pnp:
        assert den._chunk_graphs, "no chunk graph was captured"
    else:
        assert den._graph is not None, "the graph was never captured"
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(a).all(), i
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"
