"""Characterization of the library dispatch without a GPU: which route each stage of a patched transformer block takes,
and which C entry point each attention / projection op of ops.py drives with which arguments.

The library calls are replaced by recorders (the eligibility tests read shapes, types and flags, never the device), and
every recorded sequence is compared with tests/golden/stage_dispatch_traces.json.  Run this file as a script to
rewrite that file from the current code.

Blocks: every stage's eligibility checks, merge-plan requests, library calls and module forwards, in call order, for a
matrix of contexts (merging, not merging, _unmerged_blocks(), a served block), FUSE_UNMERGED_ATTENTION, PnP marks, norms,
masks and cross_attention_kwargs, and stock or customised attn1 / attn2 / ff.

Ops: the C entry points are recorded as the `*_impl` call they make in csrc/attention.cu and csrc/linear.cu (every entry
point of a family is a thin wrapper over one implementation), with the arguments that select the path: NULL pointers,
flags, the PnP period, LoRA ranks, workspace sizes; and the launch count and the `_Timed` figures of each op."""
import inspect
import itertools
import json
import pathlib

import pytest
import torch

from vidtome_b200 import _lib, attention, feedforward, ops, patch, pnp
from vidtome_b200.skeleton import Attention, BasicTransformerBlock, GEGLUFeedForward

GOLDEN = pathlib.Path(__file__).parent / "golden" / "stage_dispatch_traces.json"
SIZE = 16                     # latent 16 x 16: 256 tokens per frame at downsample 1, 16 at downsample 4


# ------------------------------------------------------------------------------------------------ blocks
class AdaNorm(torch.nn.Module):
    def __init__(self, trace, name):
        super().__init__()
        self.trace, self.name = trace, name

    def forward(self, x, timestep):
        self.trace.append(f"{self.name}(ada)")
        return x


class AdaNormZero(torch.nn.Module):
    def __init__(self, trace):
        super().__init__()
        self.trace = trace

    def forward(self, x, timestep, class_labels, hidden_dtype=None):
        self.trace.append("norm1(ada_zero)")
        z = torch.zeros(x.shape[0], x.shape[-1], dtype=x.dtype)
        return x, z + 1, z, z, z + 1


class FakePlan:
    def __init__(self, trace, x, seq_len):
        self.trace, self.merged_tokens = trace, x
        self.seq_len = torch.ones(1, dtype=torch.int32) if seq_len else None

    def unmerge_add(self, y, h):
        self.trace.append(f"unmerge_add(B={y.shape[0]})")
        return h + 1


class BlockRecorder:
    def __init__(self, monkeypatch, seq_len=False):
        self.trace = []
        t = self.trace
        self.seq_len = seq_len
        monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
        block_merges, plain, fusable = patch.block_merges, patch._plain_attention_module, patch._fusable_layer_norm
        xa_eligible, geglu_parts = attention.cross_attention_eligible, feedforward.geglu_parts

        def rec_block_merges(x, info):
            r = block_merges(x, info)
            t.append(f"block_merges={r}")
            return r

        def rec_plain(attn):
            r = plain(attn)
            t.append(f"plain={r}")
            return r

        def rec_fusable(norm, x):
            r = fusable(norm, x)
            t.append(f"fusable_ln={r is not None}")
            return r

        def rec_xa_eligible(attn, ctx):
            r = xa_eligible(attn, ctx)
            t.append(f"xa_eligible={r}")
            return r

        def rec_geglu_parts(ff):
            r = geglu_parts(ff)
            t.append(f"geglu_parts={r is not None}")
            return r

        def plan(module, x, info, ln=None):
            t.append(f"build_merge_plan(ln={ln is not None})")
            return FakePlan(t, x, self.seq_len) if patch.block_merges(x, info) else None

        def lib(module, name):
            sig = inspect.signature(getattr(module, name))

            def fn(*args, **kwargs):
                bound = sig.bind(*args, **kwargs)
                bound.apply_defaults()
                t.append(f"{name}({', '.join(f'{k}={_brief(v)}' for k, v in bound.arguments.items())})")
                return torch.zeros_like(args[1]) if name == "self_attention" else args[-1] + 1
            return fn

        def layer_norm(x, ln):
            t.append("ops.layer_norm")
            return x

        def module_attention(attn, x, encoder_hidden_states=None, attention_mask=None, **kw):
            t.append(f"Attention.forward(B={x.shape[0]}, ctx={encoder_hidden_states is not None}, "
                     f"mask={attention_mask is not None}, kw={sorted(kw)})")
            return torch.zeros_like(x)

        def module_ff(ff, x):
            t.append(f"ff.forward(B={x.shape[0]})")
            return torch.zeros_like(x)

        monkeypatch.setattr(patch, "block_merges", rec_block_merges)
        monkeypatch.setattr(patch, "_plain_attention_module", rec_plain)
        monkeypatch.setattr(patch, "_fusable_layer_norm", rec_fusable)
        monkeypatch.setattr(patch, "build_merge_plan", plan)
        monkeypatch.setattr(attention, "cross_attention_eligible", rec_xa_eligible)
        monkeypatch.setattr(feedforward, "geglu_parts", rec_geglu_parts)
        monkeypatch.setattr(ops, "layer_norm", layer_norm)
        for module, name in ((attention, "self_attention"), (attention, "self_attention_residual"),
                             (attention, "cross_attention_residual"), (feedforward, "feed_forward_residual")):
            monkeypatch.setattr(module, name, lib(module, name))
        monkeypatch.setattr(Attention, "forward", module_attention)
        monkeypatch.setattr(GEGLUFeedForward, "forward", module_ff)


def _brief(v):
    if isinstance(v, torch.Tensor):
        return f"tensor{list(v.shape)}"
    if isinstance(v, torch.nn.Module):
        return type(v).__name__
    if isinstance(v, tuple):
        return f"({', '.join(_brief(x) for x in v)})"
    return repr(v)


CONTEXTS = ("merging", "not_merging", "unmerged_blocks", "served")
VARIANTS = ("stock", "ada", "ada_zero", "attention_mask", "encoder_attention_mask", "cross_attention_kwargs",
            "custom_attn1", "custom_attn2", "custom_ff", "norm1_not_fusable", "only_cross", "no_ctx_batch",
            "plan_seq_len")
PNP = {"injecting_one_item": 3, "injecting_two_items": 6, "injecting_does_not_fit": 4, "idle": 6}   # batch

CASES = ([f"{c}-{'fuse' if f else 'nofuse'}-{v}" for c, f, v in itertools.product(CONTEXTS, (False, True), VARIANTS)]
         + [f"{c}-{'fuse' if f else 'nofuse'}-pnp_{p}"
            for c, f, p in itertools.product(CONTEXTS[:3], (False, True), PNP)])


def _run_block(case, monkeypatch):
    context, fuse, variant = case.split("-")
    rec = BlockRecorder(monkeypatch, seq_len=variant == "plan_seq_len")
    t = rec.trace
    monkeypatch.setattr(patch, "FUSE_UNMERGED_ATTENTION", fuse == "fuse")
    monkeypatch.setattr(patch, "FUSE_CONTROLNET_BLOCKS", True)
    torch.manual_seed(0)
    blk = BasicTransformerBlock(320, 8, cross_attention_dim=768, hot_path_only=False).half()
    B = 6
    if context == "served":
        blk.__class__ = patch.make_unmerged_block(blk.__class__)
    else:
        blk.__class__ = patch.make_diffusers_tome_block(blk.__class__)
        blk._tome_info = {"size": (SIZE, SIZE), "hooks": [], "args": dict(
            max_downsample=2, generator=None, seed=123, batch_size=3, align_batch=True, merge_global=False,
            global_merge_ratio=0.8, local_merge_ratio=0.9, global_rand=0.5, target_stride=4)}
        blk.generator = torch.Generator().manual_seed(5)
    for name in ("norm1", "norm2", "norm3"):
        getattr(blk, name).register_forward_pre_hook(lambda m, a, name=name: t.append(f"{name}.forward"))
    tokens = SIZE * SIZE if context == "merging" else SIZE * SIZE // 16
    x = torch.randn(B, tokens, 320).half()
    kwargs = dict(encoder_hidden_states=torch.randn(B, 8, 768).half())
    if variant == "ada":
        blk.use_ada_layer_norm = True
        blk.norm1, blk.norm2 = AdaNorm(t, "norm1"), AdaNorm(t, "norm2")
        kwargs["timestep"] = 1
    elif variant == "ada_zero":
        blk.use_ada_layer_norm_zero = True
        blk.norm1 = AdaNormZero(t)
        kwargs["timestep"] = 1
    elif variant == "attention_mask":
        kwargs["attention_mask"] = torch.zeros(B, 1, tokens).half()
    elif variant == "encoder_attention_mask":
        kwargs["encoder_attention_mask"] = torch.zeros(B, 1, 8).half()
    elif variant == "cross_attention_kwargs":
        kwargs["cross_attention_kwargs"] = {"scale": 1.0}
    elif variant == "custom_attn1":
        blk.attn1.register_forward_hook(lambda *a: t.append("attn1 hook"))
    elif variant == "custom_attn2":
        blk.attn2.register_forward_hook(lambda *a: t.append("attn2 hook"))
    elif variant == "custom_ff":
        blk.ff.register_forward_hook(lambda *a: t.append("ff hook"))
    elif variant == "norm1_not_fusable":
        blk.norm1 = torch.nn.LayerNorm(320, elementwise_affine=False).half()
        blk.norm1.register_forward_pre_hook(lambda m, a: t.append("norm1.forward"))
    elif variant == "only_cross":
        blk.only_cross_attention = True
    elif variant == "no_ctx_batch":
        kwargs["encoder_hidden_states"] = torch.randn(2, 8, 768).half()
    elif variant.startswith("pnp_"):
        pnp.register_attention_control(None, [981, 961], 3, modules=[blk.attn1])
        pnp.register_time(None, 500 if variant == "pnp_idle" else 981, modules=[blk.attn1])

        def pnp_forward(x, *a, **k):
            t.append(f"pnp forward(B={x.shape[0]})")
            return torch.zeros_like(x)
        pnp_forward._vtm_pnp_forward = True
        blk.attn1.forward = pnp_forward
        B = PNP[variant[4:]]
        x = torch.randn(B, tokens, 320).half()
        kwargs["encoder_hidden_states"] = torch.randn(B, 8, 768).half()
    state = None if context == "served" else blk.generator.get_state().clone()
    try:
        if context == "unmerged_blocks":
            with patch._unmerged_blocks():
                y = blk(x, **kwargs)
        else:
            y = blk(x, **kwargs)
        t.append(f"-> {list(y.shape)}")
    except Exception as e:                                   # the error is part of the route
        t.append(f"raise {type(e).__name__}: {str(e)[:60]}")
    if state is not None:
        t.append(f"generator untouched={torch.equal(blk.generator.get_state(), state)}")
    return t


# ------------------------------------------------------------------------------------------------ ops
class FakeLib:
    """The C entry points of the attention and projection families, each recorded as the implementation call it makes;
    the workspace-size queries answered by the real library."""

    def __init__(self, real, names, trace, timed):
        self.real, self.names, self.trace, self.timed = real, names, trace, timed

    def __getattr__(self, name):
        if name.endswith("_workspace_bytes"):
            return getattr(self.real, name)
        return lambda *args: self._record(name, args)

    def _p(self, v):
        if v is None:
            return None
        if isinstance(v, int):
            return self.names.get(v, "allocated")
        raise TypeError(v)

    @staticmethod
    def _lora(ref):
        return None if ref is None else f"R={ref._obj.R}"

    def _record(self, name, a):
        p, lo = self._p, self._lora
        if name in ("vtm_attention_ex", "vtm_attention_dev", "vtm_attention_lora", "vtm_attention_residual",
                    "vtm_attention_residual_ex"):
            if name == "vtm_attention_ex":
                x, wqkv, wo, bo, B, L, Cc, heads, scale, flags, y, ws, wsb, s = a
                lq = lop = ln = resid = None
                items = 1
            elif name == "vtm_attention_dev":
                x, wqkv, wo, bo, B, L, Cc, heads, scale, flags, ln, y, ws, wsb, s = a
                lq = lop = resid = None
                items = 1
            elif name == "vtm_attention_lora":
                x, wqkv, wo, bo, lq, lop, B, L, Cc, heads, scale, flags, ln, y, ws, wsb, s = a
                resid, items = None, 1
            elif name == "vtm_attention_residual":
                x, wqkv, wo, bo, resid, lq, lop, B, L, Cc, heads, scale, y, ws, wsb, s = a
                flags, ln, items = 0, None, 1
            else:
                x, wqkv, wo, bo, resid, lq, lop, B, L, Cc, heads, scale, flags, items, y, ws, wsb, s = a
                ln = None
            if name in ("vtm_attention_dev", "vtm_attention_residual", "vtm_attention_residual_ex"):
                assert (ln if name == "vtm_attention_dev" else resid) is not None      # their own NULL check
            rec = dict(impl="attention_impl", x=p(x), w_qkv=p(wqkv), w_o=p(wo), b_o=p(bo), B=B, L=L, C=Cc,
                       heads=heads, scale=scale, flags=flags, len=p(ln), y=p(y), ws=p(ws), ws_bytes=wsb,
                       lora_qkv=lo(lq), lora_o=lo(lop), resid=p(resid), qk_items=items if flags & 1 else "unused")
        elif name in ("vtm_cross_attention", "vtm_cross_attention_lora"):
            if name == "vtm_cross_attention":
                x, ctx, wq, wkv, wo, bo, resid, B, Lq, Lk, Cc, Cctx, heads, scale, y, ws, wsb, s = a
                lq = lkv = lop = None
            else:
                x, ctx, wq, wkv, wo, bo, resid, lq, lkv, lop, B, Lq, Lk, Cc, Cctx, heads, scale, y, ws, wsb, s = a
            rec = dict(impl="cross_attention_impl", x=p(x), ctx=p(ctx), w_q=p(wq), w_kv=p(wkv), w_o=p(wo), b_o=p(bo),
                       resid=p(resid), lora_q=lo(lq), lora_kv=lo(lkv), lora_o=lo(lop), B=B, Lq=Lq, Lk=Lk, C=Cc,
                       Cctx=Cctx, heads=heads, scale=scale, y=p(y), ws=p(ws), ws_bytes=wsb)
        elif name in ("vtm_linear_residual_f16", "vtm_linear_lora_f16"):
            if name == "vtm_linear_residual_f16":
                aa, w, bias, resid, ldr, M, N, K, d, ldd, s = a
                lr, ws, wsb = None, None, 0
                assert resid is not None                                                 # its own NULL check
            else:
                aa, w, bias, resid, ldr, lr, M, N, K, d, ldd, ws, wsb, s = a
            R = 0 if lr is None else lr._obj.R
            rec = dict(impl="linear_impl", a=p(aa), w=p(w), bias=p(bias), resid=p(resid), ldr=ldr, M=M, N=N, K=K,
                       d=p(d), ldd=ldd, lora=lo(lr) if R else None, ws=p(ws), ws_bytes=wsb)
        elif name in ("vtm_linear_geglu_f16", "vtm_linear_geglu_lora_f16"):
            if name == "vtm_linear_geglu_f16":
                aa, w, bias, M, N, K, d, ldd, s = a
                lr, ws, wsb = None, None, 0
            else:
                aa, w, bias, lr, M, N, K, d, ldd, ws, wsb, s = a
            R = 0 if lr is None else lr._obj.R
            rec = dict(impl="geglu_impl", a=p(aa), w_il=p(w), bias_il=p(bias), M=M, N=N, K=K, d=p(d), ldd=ldd,
                       lora=lo(lr) if R else None, ws=p(ws), ws_bytes=wsb)
        else:
            raise AssertionError(f"unexpected entry point {name}")
        assert s == STREAM
        rec["inside_timed"] = bool(self.timed)
        self.trace.append(rec)
        return 0


STREAM = 0x5EED


def _t(*shape):
    return torch.zeros(*shape, dtype=torch.float16)


def _lora(R, K, N):
    return _t(R, K), _t(N, R)


def _op_case(name):
    B, L, Cc, heads, Lk, Cctx = 6, 64, 320, 8, 77, 768
    x, resid, w_qkv, w_o, b_o = _t(B, L, Cc), _t(B, L, Cc), _t(3 * Cc, Cc), _t(Cc, Cc), _t(Cc)
    ctx, w_q, w_kv = _t(B, Lk, Cctx), _t(Cc, Cc), _t(2 * Cc, Cctx)
    a2, w2, b2, r2 = _t(B * L, 1280), _t(Cc, 1280), _t(Cc), _t(B * L, Cc)
    w_il, b_il = _t(2560, Cc), _t(2560)
    seq_len = torch.ones(1, dtype=torch.int32)
    tensors = dict(x=x, resid=resid, w_qkv=w_qkv, w_o=w_o, b_o=b_o, ctx=ctx, w_q=w_q, w_kv=w_kv, a2=a2, w2=w2, b2=b2,
                   r2=r2, w_il=w_il, b_il=b_il, seq_len=seq_len)
    op, variant = name.split(":")
    lq, lq1, lo_, lkv = _lora(8, Cc, 3 * Cc), _lora(8, Cc, Cc), _lora(16, Cc, Cc), _lora(8, Cctx, 2 * Cc)
    if op == "attention":
        kw = dict(shared_qk="shared" in variant, seq_len=seq_len if "seq_len" in variant else None,
                  lora_qkv=lq if "lora_qkv" in variant else None, lora_o=lo_ if "lora_o" in variant else None)
        call = lambda: ops.attention(x, w_qkv, w_o, b_o, heads, 0.125, **kw)
    elif op == "attention_residual":
        items = {"plain": None, "shared1": 1, "shared3": 3, "lora": None, "lora_shared3": 3, "lora_o": None}[variant]
        kw = dict(shared_items=items, lora_qkv=lq if variant.startswith("lora") and variant != "lora_o" else None,
                  lora_o=lo_ if variant.startswith("lora") else None)
        call = lambda: ops.attention_residual(x, w_qkv, w_o, b_o, heads, 0.125, resid, **kw)
    elif op == "cross_attention":
        parts = variant.split("_")
        kw = dict(resid=None if variant == "no_resid" else resid, lora_q=lq1 if "q" in parts else None,
                  lora_kv=lkv if "kv" in parts else None, lora_o=lo_ if "o" in parts else None)
        call = lambda: ops.cross_attention(x, ctx, w_q, w_kv, w_o, None if variant == "no_bias" else b_o, heads, 0.125,
                                           **kw)
    elif op == "linear_residual":
        lora = _lora(8, 1280, Cc) if variant == "lora" else None
        call = lambda: ops.linear_residual(a2, w2, None if variant == "no_bias" else b2, r2, lora=lora)
    else:
        lora = _lora(16, Cc, 2560) if variant == "lora" else None
        call = lambda: ops.linear_geglu(r2, w_il, None if variant == "no_bias" else b_il, lora=lora)
    return tensors, call


OP_CASES = (["attention:" + v for v in ("plain", "shared", "seq_len", "seq_len_shared", "lora_qkv", "lora_o",
                                         "lora_qkv_lora_o", "lora_qkv_seq_len_shared")]
            + ["attention_residual:" + v for v in ("plain", "shared1", "shared3", "lora", "lora_shared3", "lora_o")]
            + ["cross_attention:" + v for v in ("plain", "no_resid", "no_bias", "lora_q", "lora_kv", "lora_o",
                                               "lora_q_kv_o")]
            + ["linear_residual:" + v for v in ("plain", "no_bias", "lora")]
            + ["linear_geglu:" + v for v in ("plain", "no_bias", "lora")])


def _run_op(case, monkeypatch):
    real = _lib.load()
    trace, timed = [], []
    tensors, call = _op_case(case)
    names = {t.data_ptr(): n for n, t in tensors.items()}

    class Timed:
        def __init__(self, name, flops, nbytes):
            trace.append(dict(timed=name, flops=flops, bytes=nbytes))

        def __enter__(self):
            timed.append(True)
            return self

        def __exit__(self, *exc):
            timed.pop()
            return False

    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setattr(_lib, "load", lambda: FakeLib(real, names, trace, timed))
    monkeypatch.setattr(ops, "_stream", lambda: STREAM)
    monkeypatch.setattr(ops, "_Timed", Timed)
    ops.STATS.reset()
    call()
    trace.append(dict(launches=ops.STATS.launches))
    return trace


# ------------------------------------------------------------------------------------------------ tests
def _golden():
    return json.loads(GOLDEN.read_text())


@pytest.mark.parametrize("case", CASES)
def test_block_stage_routes(case, monkeypatch):
    assert _run_block(case, monkeypatch) == _golden()["blocks"][case]


@pytest.mark.parametrize("case", OP_CASES)
def test_op_entry_points(case, monkeypatch):
    assert json.loads(json.dumps(_run_op(case, monkeypatch))) == _golden()["ops"][case]


def test_golden_covers_exactly_the_cases():
    g = _golden()
    assert sorted(g["blocks"]) == sorted(CASES) and sorted(g["ops"]) == sorted(OP_CASES)


if __name__ == "__main__":
    mp = pytest.MonkeyPatch()
    out = {"blocks": {}, "ops": {}}
    for c in CASES:
        with mp.context() as m:
            out["blocks"][c] = _run_block(c, m)
    for c in OP_CASES:
        with mp.context() as m:
            out["ops"][c] = _run_op(c, m)
    GOLDEN.write_text(json.dumps(out, indent=1) + "\n")
