"""The Transformer2DModel entry and exit kernels (transformer_io.cu, NchwEpi in linear.cu) against float64, and the
wrapper through patch / driver.  Needs an H100.

Every kernel call goes through the C-ABI with its output between sentinel guard elements and its interior filled with
NaN (an element left unwritten shows as NaN, a store past an edge changes the sentinel); workspaces are filled with
0xFF bytes."""
import pytest
import torch
import torch.nn.functional as F

from vidtome_b200 import _lib, ops

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24           # unit roundoff of fp32
SENT16 = 0x5A5A
GUARD = 64
HWS = (1, 2, 7, 8, 9, 63, 64, 144, 256, 576, 1024, 4096, 9216)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


def _ulp16(x):
    _, e = torch.frexp(x.abs().clamp(min=2.0 ** -14))
    return torch.ldexp(torch.ones_like(x), e - 11)


def _round16(x):
    u = _ulp16(x)
    return torch.round(x / u) * u


def _ordered(h):
    b = h.view(torch.int16).int()
    return torch.where(b < 0, -(b & 0x7FFF), b)


def _guarded16(numel):
    buf = torch.full((numel + 2 * GUARD,), SENT16, dtype=torch.int16, device="cuda").view(torch.float16)
    buf[GUARD:GUARD + numel] = float("nan")
    return buf


# --------------------------------------------------------------------------------------------------- 1. statistics
def _stats(x, groups, eps=1e-6):
    lib = _lib.load()
    n, C, HW = x.shape
    runs = n * groups
    buf = torch.full((2 * runs + 2 * GUARD,), float("nan"), dtype=torch.float32, device="cuda")
    buf[:GUARD] = 12345.0
    buf[GUARD + 2 * runs:] = 12345.0
    ws_bytes = lib.vtm_group_norm_stats_workspace_bytes(n, C, HW, groups)
    ws = torch.full((max(ws_bytes, 1),), 0xFF, dtype=torch.uint8, device="cuda")
    _lib.check(lib.vtm_group_norm_stats_f16(x.data_ptr(), n, C, HW, groups, eps, buf[GUARD:].data_ptr(),
                                            ws.data_ptr() if ws_bytes else None, ws_bytes, _stream()), "stats")
    torch.cuda.synchronize()
    assert (buf[:GUARD] == 12345.0).all() and (buf[GUARD + 2 * runs:] == 12345.0).all()
    return buf[GUARD:GUARD + 2 * runs].view(n, groups, 2), ws_bytes


def _stats_steps(R, runs):
    """Length of the longest chain of pairwise updates behind one result (transformer_io.cu, "Grid")."""
    if R <= 2048:
        return -(-R // (8 * 32)) + 2 + 5
    S = 1
    if runs < 512 and R > 8192:
        S = min(-(-R // 8192), -(-512 // runs))
    piece = R if S == 1 else (-(-R // S) + 7) // 8 * 8
    return -(-piece // (8 * 256)) + 2 + 5 + 8 + S


def _check_stats(x, groups, eps=1e-6, what="", got=None):
    """Every pairwise update rounds a handful of fp32 operations: after `steps` of them the mean is off by at most
    steps * 4 u max|x|, and M2 (a sum of squared deviations, never a difference of large sums) by steps * 8 u relative
    plus what the mean's error moves it by, 4 max|x - mean| e_mean.  `got`: statistics the caller computed (else they
    are computed here)."""
    n, C, HW = x.shape
    ws_bytes = None
    if got is None:
        got, ws_bytes = _stats(x, groups, eps)
    x64 = x.double().view(n, groups, -1)
    R = x64.shape[-1]
    mean = x64.mean(-1)
    var = x64.var(-1, unbiased=False)
    rstd = 1.0 / torch.sqrt(var + eps)
    steps = _stats_steps(R, n * groups)
    xmax = x64.abs().amax(-1)
    dev = (x64 - mean[..., None]).abs().amax(-1)
    e_mean = steps * 4 * U32 * xmax + U32 * mean.abs()
    assert ((got[..., 0].double() - mean).abs() <= e_mean).all(), f"{what}: mean"
    e_var = steps * 8 * U32 * var + 4 * dev * e_mean + e_mean ** 2
    # d rstd = -rstd^3 / 2 d var, plus the division's and square root's own roundings
    e_rstd = 0.5 * rstd ** 3 * e_var * 1.01 + 4 * U32 * rstd
    assert ((got[..., 1].double() - rstd).abs() <= e_rstd).all(), f"{what}: rstd"
    return got, ws_bytes


def test_stats_every_group_width_and_spatial_size():
    g = torch.Generator(device="cuda").manual_seed(1)
    split_seen = small_seen = False
    for cpg in range(1, 41):
        for HW in HWS:
            n = 1 + (cpg + HW) % 3
            x = (torch.randn((n, 32 * cpg, HW), generator=g, device="cuda") * 1.5 + 0.3).half()
            if (cpg + HW) % 5 == 0:                      # a run that starts off a 16-byte boundary
                x = torch.cat([x.new_zeros(3), x.flatten()])[3:].view(n, 32 * cpg, HW)
            _, ws = _check_stats(x, 32, what=f"cpg={cpg} HW={HW} n={n}")
            split_seen |= ws > 0
            small_seen |= cpg * HW <= 2048
    assert split_seen and small_seen


@pytest.mark.parametrize("n,C,HW", [(40, 320, 4096), (600, 64, 1), (20, 1280, 64), (1, 320, 9216), (3, 1280, 1024)])
def test_stats_more_runs_than_ctas_and_split_runs(n, C, HW):
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn((n, C, HW), generator=g, device="cuda").half()
    _check_stats(x, 32, what=f"n={n} C={C} HW={HW}")


@pytest.mark.parametrize("C,HW", [(320, 4096), (64, 9), (1280, 256), (320, 9216)])
def test_stats_large_mean_does_not_cancel(C, HW):
    """Mean 1000 with the smallest spread fp16 has there (its spacing at 1000 is 1/2): E[x^2] - E[x]^2 in fp32 would be
    off by u * 1e6 = 0.06 against a variance of 0.5."""
    g = torch.Generator(device="cuda").manual_seed(3)
    x = (1000 + (torch.randint(-2, 3, (2, C, HW), generator=g, device="cuda").double() * 0.5)).half()
    assert 0.3 < x.double().var().item() < 0.7
    got, _ = _check_stats(x, 32, what="cancellation")
    x64 = x.double().view(2, 32, -1)
    rstd = 1.0 / torch.sqrt(x64.var(-1, unbiased=False) + 1e-6)
    assert ((got[..., 1].double() - rstd).abs() <= 1e-4 * rstd).all()


def test_stats_constant_group_and_extreme_entries():
    x = torch.randn((2, 64, 144), device="cuda").half()
    x[0, 0:2] = 3.5                                      # group 0 of sample 0 is constant: var = 0
    x[1, 10, 5] = 65504.0
    x[1, 11, 7] = -65504.0
    x[1, 20, :] = 65504.0
    got, _ = _check_stats(x, 32, eps=1e-6, what="extremes")
    assert got[0, 0, 0].item() == 3.5
    assert abs(got[0, 0, 1].item() - 1e-6 ** -0.5) <= 4 * U32 * 1e3
    assert torch.isfinite(got).all()


# ------------------------------------------------------------------------------------- 2. normalise + transpose
def _tokens(x, stats, gamma, beta, groups):
    lib = _lib.load()
    n, C, HW = x.shape
    buf = _guarded16(n * HW * C + 8)
    off = (-(buf.data_ptr() // 2 + GUARD)) % 8           # 16-byte aligned output inside the guards
    y = buf[GUARD + off:GUARD + off + n * HW * C]
    _lib.check(lib.vtm_group_norm_tokens_f16(x.data_ptr(), stats.data_ptr(), _ptr(gamma), _ptr(beta), n, C, HW, groups,
                                             y.data_ptr(), _stream()), "tokens")
    torch.cuda.synchronize()
    bits = buf.view(torch.int16)
    assert (bits[:GUARD] == SENT16).all() and (bits[GUARD + off + n * HW * C + 8:] == SENT16).all()
    assert (bits[GUARD:GUARD + off] == 0x7E00).all()
    return y.view(n, HW, C)


TOKEN_SHAPES = [(2, 320, 4096), (3, 64, 1), (2, 96, 7), (1, 72, 9), (2, 640, 63), (2, 136, 200), (1, 1280, 144),
                (2, 328, 65), (1, 32, 1024), (2, 8, 130)]


@pytest.mark.parametrize("n,C,HW", TOKEN_SHAPES)
@pytest.mark.parametrize("offset", [0, 1])
def test_tokens_against_float64_and_torch(n, C, HW, offset):
    g = torch.Generator(device="cuda").manual_seed(n * 1000 + C + HW)
    groups = 32 if C % 32 == 0 else 8 if C % 8 == 0 else 1
    flat = (torch.randn((n * C * HW + 8,), generator=g, device="cuda") * 2 + 0.5).half()
    x = flat[offset:offset + n * C * HW].view(n, C, HW)  # offset 1: channel rows off the 16-byte grid
    gamma = (1 + 0.2 * torch.randn((C,), generator=g, device="cuda")).half()
    beta = (0.2 * torch.randn((C,), generator=g, device="cuda")).half()
    stats, _ = _stats(x, groups)
    stats = stats.contiguous()
    y = _tokens(x, stats, gamma, beta, groups)
    assert torch.isfinite(y).all()
    cpg = C // groups
    mean = stats[..., 0].double().repeat_interleave(cpg, 1)[:, :, None]
    rstd = stats[..., 1].double().repeat_interleave(cpg, 1)[:, :, None]
    t = (x.double() - mean) * rstd
    want = (t * gamma.double()[None, :, None] + beta.double()[None, :, None]).transpose(1, 2)
    # fp32 steps: the subtraction and the product each round once (relative u), the fma once more; then one fp16 rounding
    bound = (2 * U32 * (t.abs() * gamma.double().abs()[None, :, None]).transpose(1, 2) + U32 * want.abs()) * 1.01 \
        + 0.5 * _ulp16(want)
    err = (y.double() - want).abs()
    assert (err <= bound).all(), (err - bound).max().item()
    off = (_ordered(y) - _ordered(_round16(want).half())).abs()
    assert off.max().item() <= 1
    # results one fp16 ulp from the correctly rounded value arise only where the fp32 error crosses a rounding boundary
    assert (off != 0).float().mean().item() <= 2e-3
    # torch's fp16 group_norm is itself further from float64 than this kernel (the check above): it forms a x + b with
    # a = rstd gamma and b = beta - a mean, and its result is off by fp16 roundings at the size of those terms rather
    # than of their sum.  So "one fp16 ulp from torch" holds for most elements, not all: at least 90 % agree to one ulp
    # of the result, and every element to four fp16 ulps at the size of |a x| + |a mean| + |beta| (plus one of the
    # result).  These two figures are what torch 2.11 on an H100 shows, not a derivation from its source.
    ref = F.group_norm(x.view(n, C, HW, 1), groups, gamma, beta, 1e-6).permute(0, 2, 3, 1).reshape(n, HW, C)
    a = (rstd * gamma.double()[None, :, None]).abs()
    scale = (a * x.double().abs() + a * mean.abs() + beta.double().abs()[None, :, None]).transpose(1, 2)
    diff = (y.double() - ref.double()).abs()
    over = diff - 4 * _ulp16(scale) - _ulp16(want)
    assert (over <= 0).all(), over.max().item()
    if C // groups * HW >= 64:
        assert (diff <= _ulp16(want)).float().mean().item() >= 0.9


# ----------------------------------------------------------------------------------- 3. projection storing NCHW
def _nchw_linear(a, w, b, resid, n, HW):
    lib = _lib.load()
    N, K = w.shape
    buf = _guarded16(n * N * HW + 8)
    off = (-(buf.data_ptr() // 2 + GUARD)) % 8
    d = buf[GUARD + off:GUARD + off + n * N * HW]
    _lib.check(lib.vtm_linear_nchw_residual_f16(a.data_ptr(), w.data_ptr(), _ptr(b), _ptr(resid), n, HW, N, K,
                                                d.data_ptr(), _stream()), "nchw linear")
    torch.cuda.synchronize()
    bits = buf.view(torch.int16)
    assert (bits[:GUARD] == SENT16).all() and (bits[GUARD + off + n * N * HW + 8:] == SENT16).all()
    assert (bits[GUARD:GUARD + off] == 0x7E00).all()
    return d.view(n, N, HW)


def _grid(shape, step, lim, g):
    k = int(round(lim / step))
    return (torch.randint(-k, k + 1, shape, generator=g, device="cuda").double() * step).half()


def _exact_weights(N, K, g, kind):
    if kind == "perm":                                   # signed permutation rows: every output is +-one input
        w = torch.zeros((N, K), device="cuda", dtype=torch.float16)
        cols = torch.randint(0, K, (N,), generator=g, device="cuda")
        sign = torch.randint(0, 2, (N,), generator=g, device="cuda") * 2 - 1
        w[torch.arange(N, device="cuda"), cols] = sign.half()
        return w
    return _grid((N, K), 1.0, 2, g)                      # small integers


NCHW_SHAPES = [(300, 1, 64, 64), (5, 64, 320, 320), (3, 144, 136, 72), (2, 200, 328, 200), (40, 576, 128, 64),
               (7, 63, 72, 136), (1, 4096, 640, 320)]


@pytest.mark.parametrize("n,HW,N,K", NCHW_SHAPES)
@pytest.mark.parametrize("kind", ["perm", "int"])
@pytest.mark.parametrize("bias,resid", [(True, True), (False, True), (True, False), (False, False)])
def test_nchw_projection_bit_exact_on_exact_inputs(n, HW, N, K, kind, bias, resid):
    g = torch.Generator(device="cuda").manual_seed(n + HW + N + K)
    M = n * HW
    a = _grid((M, K), 1 / 8, 4, g)
    w = _exact_weights(N, K, g, kind)
    b = _grid((N,), 2.0 ** -7, 8, g) if bias else None
    r = (torch.randn((n, N, HW), generator=g, device="cuda") * 4).half() if resid else None
    assert (a.double().abs() @ w.double().abs().t()).max().item() + 8 < 2.0 ** 16      # exact in fp32 in any order
    d = _nchw_linear(a, w, b, r, n, HW)
    prod = a.double() @ w.double().t()
    if bias:
        prod = prod + b.double()
    want = _round16(prod).view(n, HW, N).transpose(1, 2)
    if resid:
        want = _round16(want + r.double())
    assert torch.equal(d.double(), want), (d.double() - want).abs().max().item()


@pytest.mark.parametrize("n,HW,N,K", [(5, 64, 320, 320), (3, 144, 136, 72), (300, 1, 64, 64), (2, 4096, 320, 320),
                                      (2, 9, 1280, 1280)])
def test_nchw_projection_equals_row_major_projection_transposed(n, HW, N, K):
    g = torch.Generator(device="cuda").manual_seed(11)
    M = n * HW
    a = torch.randn((M, K), generator=g, device="cuda").half()
    w = (torch.randn((N, K), generator=g, device="cuda") * K ** -0.5).half()
    b = torch.randn((N,), generator=g, device="cuda").half()
    r = torch.randn((n, N, HW), generator=g, device="cuda").half()
    d = _nchw_linear(a, w, b, r, n, HW)
    r_rows = r.transpose(1, 2).reshape(M, N).contiguous()
    rows = ops.linear_residual(a, w, b, r_rows)
    assert torch.equal(d.view(torch.int16), rows.view(n, HW, N).transpose(1, 2).contiguous().view(torch.int16))
    d0 = _nchw_linear(a, w, None, None, n, HW)
    rows0 = ops.linear(a, w)
    assert torch.equal(d0.view(torch.int16), rows0.view(n, HW, N).transpose(1, 2).contiguous().view(torch.int16))


# -------------------------------------------------------------------------------------- 4. the wrapper, patched
def _wrapper(name, form, dim, heads):
    from vidtome_b200.skeleton import BasicTransformerBlock, ModelMixin, Transformer2DModel
    torch.manual_seed(5)
    cad = 1024 if name == "sd21" else 768

    class Net(ModelMixin):
        def __init__(self):
            super().__init__()
            self.attn = Transformer2DModel(dim, BasicTransformerBlock(dim, heads, cad, hot_path_only=False),
                                           use_linear_projection=form == "linear")

        def forward(self, x, t=None, encoder_hidden_states=None):
            return self.attn(x, encoder_hidden_states=encoder_hidden_states, return_dict=False)[0]

    return Net().cuda().half().eval(), cad


@pytest.mark.parametrize("name,form,dim,heads,hw", [("sd15", "conv", 320, 8, (32, 32)), ("sd15", "conv", 1280, 8, (8, 8)),
                                                    ("sd21", "linear", 320, 5, (24, 24)),
                                                    ("sd21", "linear", 640, 10, (12, 12))])
def test_wrapper_library_path_against_fp32_and_switch(name, form, dim, heads, hw):
    import copy
    import vidtome_b200
    from vidtome_b200 import patch
    from vidtome_b200.skeleton import Transformer2DModel
    net, cad = _wrapper(name, form, dim, heads)
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn((8, dim, *hw), generator=g, device="cuda").half()
    ctx = torch.randn((8, 77, cad), generator=g, device="cuda").half()
    with torch.no_grad():
        ref = copy.deepcopy(net).float()(x.float(), 0, ctx.float())
        vidtome_b200.apply_patch(net, local_merge_ratio=0.0, batch_size=2)      # ratio 0: nothing merged, same function
        assert type(net.attn).__name__ == "ToMeTransformer2D"
        Transformer2DModel.torch_calls = 0
        got = net(x, 0, ctx)
        assert Transformer2DModel.torch_calls == 0
        e_lib = (got.float() - ref).abs().max().item()
        patch.FUSE_TRANSFORMER_IO = False
        try:
            off = net(x, 0, ctx)
            assert Transformer2DModel.torch_calls == 1
        finally:
            patch.FUSE_TRANSFORMER_IO = True
        # the patched block inside rounds every intermediate to fp16 and sets the error level of either path: the
        # library wrapper is within 2e-3 max|ref| of the fp32 evaluation, or no further from it than 1.25 x the torch
        # wrapper around the same patched block (test_wrapper_alone holds the new kernels alone to 2e-3)
        e_off = (off.float() - ref).abs().max().item()
        assert e_lib <= max(2e-3 * ref.abs().max().item(), 1.25 * e_off), (e_lib, e_off)
        # the unpatched wrapper around the same patched block
        net.attn.__class__ = net.attn._parent
        assert torch.equal(off, net(x, 0, ctx))
    vidtome_b200.remove_patch(net)


class _PassThrough(torch.nn.Module):
    def forward(self, hidden_states, **kwargs):
        return hidden_states


@pytest.mark.parametrize("form,dim,hw", [("conv", 320, (64, 64)), ("conv", 1280, (8, 8)), ("linear", 320, (96, 96)),
                                         ("linear", 1280, (12, 12)), ("conv", 640, (5, 7))])
def test_wrapper_alone_against_fp32(form, dim, hw):
    """GroupNorm -> proj_in -> proj_out + residual with nothing in between: the new kernels alone."""
    import copy
    from vidtome_b200 import transformer2d
    from vidtome_b200.skeleton import Transformer2DModel
    torch.manual_seed(6)
    m = Transformer2DModel(dim, _PassThrough(), use_linear_projection=form == "linear").cuda().half().eval()
    x = torch.randn((4, dim, *hw), device="cuda").half()
    with torch.no_grad():
        ref = copy.deepcopy(m).float()(x.float()).sample
        assert transformer2d.ineligibility(m, x) is None
        Transformer2DModel.torch_calls = 0
        got = transformer2d.library_forward(m, x).sample
        assert Transformer2DModel.torch_calls == 0 and got.shape == x.shape and got.is_contiguous()
    assert (got.float() - ref).abs().max().item() <= 2e-3 * ref.abs().max().item()


# -------------------------------------------------------------------------------------------------- 5. the driver
def _drive(mode, steps=4, frames=8, size=16, control=False, pnp=False):
    import numpy as np
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import (Transformer2DModel, make_controlnet, make_skeleton, pnp_attention_modules,
                                       pnp_conv_module)
    torch.manual_seed(77)
    bs = 3 if pnp else 2
    net = make_skeleton("sd15", device="cuda", hot_path_only=False, transformer_io="conv", pnp_conv=pnp)
    merge_global = mode in ("capture_global", "eager_global", "chunk_graphs", "eager_random")
    kw_patch = dict(local_merge_ratio=0.9, merge_global=merge_global, global_merge_ratio=0.8, global_rand=0.5,
                    batch_size=bs, align_batch=pnp)
    vidtome_b200.apply_patch(net, **kw_patch)
    g = torch.Generator(device="cuda").manual_seed(5)
    cond = torch.randn((bs, 77, 768), generator=g, device="cuda").half()
    graph = not mode.startswith("eager")
    kw = dict(cuda_graph=graph, graph_warmup=1)
    if mode in ("chunk_graphs", "eager_random"):
        kw.update(randomize_chunks=True, chunk_graphs=graph)
    if mode in ("capture_global", "eager_global"):
        kw.update(capture_global=graph)
    if control:
        cn = make_controlnet("sd15", hot_path_only=False, device="cuda", transformer_io="conv")
        class DiffusionPipeline:                   # matched by name
            pass

        class StableDiffusionControlNetPipeline(DiffusionPipeline):
            pass
        pipe = StableDiffusionControlNetPipeline()
        pipe.unet, pipe.controlnet = net, cn
        vidtome_b200.apply_patch(pipe, include_control=True, **kw_patch)
        assert type(cn.wrappers[0]).__name__ == "ToMeTransformer2D"
        kw.update(controlnet=cn, control_images=torch.randn((frames, 3, size * 8, size * 8), generator=g,
                                                            device="cuda").half())
    if pnp:
        sources = {}

        def source(t):
            if t not in sources:
                gs = torch.Generator(device="cuda").manual_seed(int(t))
                sources[t] = torch.randn((frames, 4, size, size), generator=gs, device="cuda").half()
            return sources[t]
        kw.update(source_latents=source, pnp_attn_t=0.5, pnp_modules=pnp_attention_modules(net), pnp_f_t=0.75,
                  pnp_conv_modules=[pnp_conv_module(net)])
    den = ChunkedDenoiser(net, n_timesteps=steps, chunk_size=4, merge_global=merge_global, chunk_ord="mix-4", cond=cond,
                          **kw)
    x = torch.randn((frames, 4, size, size), generator=g, device="cuda", dtype=torch.float16)
    torch.manual_seed(2024)
    np.random.seed(2024)
    Transformer2DModel.torch_calls = 0
    xs = []
    for i in range(steps):
        x = den.step(x, i)
        xs.append(x.clone())
    torch.cuda.synchronize()
    assert Transformer2DModel.torch_calls == 0
    return xs


@pytest.mark.parametrize("mode,eager_mode", [("step_graph", "eager_plain"), ("capture_global", "eager_global"),
                                             ("chunk_graphs", "eager_random")])
def test_driver_graph_modes_bit_identical_to_eager(mode, eager_mode):
    eager = _drive(eager_mode)
    graph = _drive(mode)
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(b).all(), i
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"


@pytest.mark.parametrize("what", ["pnp", "control"])
def test_driver_pnp_and_controlnet_bit_identical_to_eager(what):
    kw = dict(pnp=what == "pnp", control=what == "control")
    eager = _drive("eager_plain", **kw)
    graph = _drive("step_graph", **kw)
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(b).all(), i
        assert torch.equal(a, b), f"step {i}"


def test_inverter_graph_bit_identical_to_eager():
    import vidtome_b200
    from vidtome_b200.driver import ChunkedInverter
    from vidtome_b200.skeleton import Transformer2DModel, make_skeleton
    net = make_skeleton("sd15", device="cuda", hot_path_only=False, transformer_io="conv")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, batch_size=2)
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn((8, 4, 16, 16), generator=g, device="cuda").half()
    cond = torch.randn((8, 77, 768), generator=g, device="cuda").half()
    kw = dict(n_timesteps=10, batch_size=4, cond=cond)
    Transformer2DModel.torch_calls = 0
    eager = ChunkedInverter(net, **kw)
    eager.invert(x)
    graph = ChunkedInverter(net, cuda_graph=True, graph_warmup=2, **kw)
    graph.invert(x)
    assert Transformer2DModel.torch_calls == 0
    assert torch.isfinite(graph.trajectory).all()
    assert torch.equal(eager.trajectory, graph.trajectory)
