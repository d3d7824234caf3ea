"""Small invocations of every kernel family, for `compute-sanitizer --tool memcheck python tools/sanitize_small.py`."""
import os
import sys
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vidtome_b200 import ops, patch  # noqa: E402

g = torch.Generator(device="cuda").manual_seed(0)
# projections with ragged tiles (staged row stores), with and without bias
for (M, N, K) in [(333, 320, 320), (1000, 960, 320), (130, 1920, 640)]:
    a = torch.randn((M, K), generator=g, device="cuda").half()
    w = torch.randn((N, K), generator=g, device="cuda").half()
    b = torch.randn((N,), generator=g, device="cuda").half()
    y = ops.linear(a, w, b)
    assert torch.isfinite(y).all()
# attention: ragged query and key tails, head_dim 40 / 80 / 64 (three and two consumer warpgroups)
for (B, L, C, H) in [(1, 333, 320, 8), (2, 2561, 640, 8), (3, 1500, 320, 8), (1, 700, 320, 5)]:
    x = torch.randn((B, L, C), generator=g, device="cuda").half()
    ws = [(torch.randn((C, C), generator=g, device="cuda") / C ** 0.5).half() for _ in range(4)]
    y = ops.attention(x, torch.cat(ws[:3], 0).contiguous(), ws[3], torch.zeros(C, device="cuda").half(), H, (C // H) ** -0.5)
    assert torch.isfinite(y).all()
if os.environ.get("VTM_SANITIZE_ONLY") == "attention":
    torch.cuda.synchronize()
    print("sanitize_small (attention only): ok")
    sys.exit(0)
# the merge plan (K0, KA with the filtered epilogue, sort, maps, KC, KE)
info = {"size": (16, 16), "args": dict(max_downsample=2, batch_size=2, align_batch=False, merge_global=False,
                                        global_merge_ratio=0.8, local_merge_ratio=0.9, global_rand=0.5, target_stride=4)}
x = torch.randn((2 * 8, 256, 320), generator=g, device="cuda").half()
mod = SimpleNamespace(generator=torch.Generator(device="cuda").manual_seed(1), global_tokens=None)
plan = patch.build_merge_plan(mod, x, info)
out = plan.unmerge_add(plan.merged_tokens, x)
assert torch.isfinite(out).all()
# ---- r02 additions
# fused LayerNorm in K0 / KC (fp32 rows, gamma / beta in shared memory), ragged channel counts
for C in (320, 640, 1280, 136):
    xx = torch.randn((2, 4 * 40, C), generator=g, device="cuda").half()
    ln = (torch.ones(C, device="cuda").half(), torch.zeros(C, device="cuda").half(), 1e-5)
    from vidtome_b200._lib import VtmSplit
    a_, b_ = ops.normalize_split(xx, None, VtmSplit.local(160, 0, 4, 4, 1), ln=ln)
    y_ = ops.layer_norm(xx.view(-1, C), ln)
    assert torch.isfinite(a_).all() and torch.isfinite(y_).all()
# merge modes (exact reduction with 64-bit atomics)
from vidtome_b200 import merge
xm = torch.randn((2, 4 * 48, 128), generator=g, device="cuda").half()
m_, u_, _ = merge.bipartite_soft_matching_randframe(xm, 4, 0.9, 0, torch.Generator(device="cuda").manual_seed(2))
for mode in ("mean", "sum", "amax", "amin"):
    assert torch.isfinite(m_(xm, mode=mode)).all()
# feed-forward GEMMs: GEGLU epilogue, residual epilogue with 160-wide tiles (N = 320), ragged M
for (M, K, inner) in [(333, 320, 1280), (1000, 640, 2560)]:
    a = torch.randn((M, K), generator=g, device="cuda").half()
    w = (torch.randn((2 * inner, K), generator=g, device="cuda") / K ** 0.5).half()
    bb = torch.randn((2 * inner,), generator=g, device="cuda").half()
    wi, bi = ops.interleave_geglu(w, bb)
    uu = ops.linear_geglu(a, wi, bi)
    w2 = (torch.randn((K, inner), generator=g, device="cuda") / inner ** 0.5).half()
    out = ops.linear_residual(uu, w2, torch.zeros(K, device="cuda").half(), a)
    assert torch.isfinite(out).all()
# cross-attention (Lq != Lk, one ragged key tile) and PnP's shared q / k
xq = torch.randn((3, 333, 320), generator=g, device="cuda").half()
ctx = torch.randn((3, 77, 768), generator=g, device="cuda").half()
wq = (torch.randn((320, 320), generator=g, device="cuda") / 18).half()
wkv = (torch.randn((640, 768), generator=g, device="cuda") / 28).half()
y = ops.cross_attention(xq, ctx, wq, wkv, wq, torch.zeros(320, device="cuda").half(), 8, 40 ** -0.5, resid=xq)
assert torch.isfinite(y).all()
y = ops.attention(xq, torch.cat([wq, wq, wq], 0).contiguous(), wq, None, 8, 40 ** -0.5, shared_qk=True)
assert torch.isfinite(y).all()
# KS: the sampling step's guidance combine and DDIM update, vector path and element path (n % 8 != 0), in place
coef = ops.ddim_table([(0.5, 0.9, 0.95, 0.3)] * 4).cuda()
step = torch.full((1,), 2, dtype=torch.int32, device="cuda")
for n, samples in [(4 * 64 * 64, 2), (3 * 4 * 15 * 15, 3)]:
    xs = torch.randn((n + 1,), generator=g, device="cuda").half()
    es = torch.randn((samples * n,), generator=g, device="cuda").half()
    for x_ in (xs[:n], xs[1:]):
        out = torch.empty_like(x_)
        ops.cfg_ddim_update(x_, es, samples, 7.5, coef, step, out)
        ops.cfg_ddim_update(x_, es, samples, 7.5, coef, step, x_)
        assert torch.isfinite(out).all()
torch.cuda.synchronize()
print("sanitize_small: ok")
