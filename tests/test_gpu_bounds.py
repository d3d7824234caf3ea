"""Memory behaviour of every compute entry point of the C-ABI: no store past an output or workspace, no write to an
input, every promised element written, every element the header leaves alone left alone, and results that do not
depend on where the buffers sit or on what the workspace held before.  Needs an H100 (sm_90a).

The harness.  Every buffer a call receives is carved out of a larger allocation of its own, with a lead and a trail
guard of at least 4 KB and at least one tile of the buffer's rows (128 rows of GEMM and attention outputs, a whole row of
row kernels), at the weakest alignment the header allows (16 bytes past a 256-byte boundary unless the header allows
less).  Guards of buffers the call may write hold a sentinel byte; guards of read-only inputs hold values that are safe
to read but change the result if read: NaN for fp16 / fp32 data, the index of an extra NaN "poison" row for index maps,
a key that would win for keys, a neutral value for device scalars.  Nothing here ever hands a launch an out-of-range
pointer or size.  Per registered case:
  1. guards: every guard byte is unchanged after the call;
  2. inputs: every read-only buffer (and its guards) is byte-identical after the call;
  3. coverage: outputs are prefilled with 0xA5 bytes here and with 0xFF bytes in the plain call of 4, so an element the
     call does not write differs between the two; elements the header leaves alone must still hold 0xA5, elements it
     calls unspecified may change (inside the buffer only);
  4. placement and workspace independence: the output equals, bit for bit, the same call on plain torch tensors with a
     zeroed workspace, and a second call in place, whose workspace still holds the first call's leftovers;
  5. workspace size: the workspace is exactly `*_workspace_bytes` long; the highest byte any call changed is printed
     (run with -s); with ws_bytes - 1 the call returns VTM_E_WS, and a few argument errors return their code, each
     leaving every byte of every buffer as it was;
  6. float64: where a core test has an exact-input design, the guarded output is also held to its float64 reference.

`REGISTRY` maps every compute entry point to its cases; tests/test_bounds_cpu.py checks that it names them all, and runs
the harness against fake kernels written in torch ops that must each trip the check meant for them."""
import ctypes

import numpy as np
import pytest
import torch

from vidtome_b200 import _lib
from vidtome_b200._lib import VtmLora, VtmSplit

pytestmark = pytest.mark.gpu

GUARD_MIN = 4096
SENTINEL = 0x5A                 # guard bytes of every buffer the call may write
PREFILL = 0xA5                  # outputs and workspaces before the guarded calls
PLAIN_FILL = 0xFF               # outputs before the plain call (fp16 / fp32 NaN)
VTM_E_NULL, VTM_E_SHAPE, VTM_E_WS, VTM_E_UNSUPPORTED = -1, -2, -4, -6


class BoundsFailure(AssertionError):
    """A harness check failed; `check` names which one (guard, input, coverage, kept, workspace, placement, value,
    error)."""

    def __init__(self, check, msg):
        super().__init__(f"[{check}] {msg}")
        self.check = check


# ---------------------------------------------------------------------------------------------------------------------
# buffers

class Buf:
    """One buffer of a call.  kind: "in" (read-only), "out" (written), "inout" (read and written in place) or "ws"
    (workspace).  `data` gives the contents of "in" / "inout" buffers; "out" / "ws" buffers give numel (and dtype).
    `poison` is the value an input's guards hold (default all-ones bytes: NaN for floats, the largest key for keys);
    `guard` the guard size in bytes (at least GUARD_MIN); `align` the buffer's offset from a 256-byte boundary.
    `kept` / `unspec`: boolean masks over the elements of an "out" / "ws" buffer that the call must leave alone / may
    leave in any state.  `same_phase`: the plain call of check 4 places the buffer at the same offset from a 16-byte
    boundary (for a call whose header lets its roundings depend on that offset)."""

    def __init__(self, kind, data=None, *, numel=None, dtype=torch.float16, align=16, guard=0, poison=None, kept=None,
                 unspec=None, same_phase=False):
        assert kind in ("in", "out", "inout", "ws")
        self.kind, self.data, self.align, self.poison, self.kept, self.unspec = kind, data, align, poison, kept, unspec
        self.same_phase = same_phase
        if data is not None:
            self.data = data.contiguous()
            numel, dtype = self.data.numel(), self.data.dtype
        if kind == "ws":
            dtype = torch.uint8
        self.numel, self.dtype = int(numel), dtype
        self.esize = torch.empty((), dtype=dtype).element_size()
        self.nbytes = self.numel * self.esize
        g = max(GUARD_MIN, int(guard))
        self.guard = -(-g // 256) * 256
        if kind == "in" and dtype == torch.int32:
            assert poison is not None, "an int32 input needs an in-range poison value for its guards"

    def writable(self):
        return self.kind != "in"

    def _poison_bytes(self, device):
        if self.poison is None:
            return torch.full((self.esize,), 0xFF, dtype=torch.uint8, device=device)
        return torch.tensor([self.poison], dtype=self.dtype).view(torch.uint8).to(device)

    def _mask(self, m, device):
        return None if m is None else m.reshape(-1).to(device).repeat_interleave(self.esize)

    def promised(self, device):
        """Byte mask of the elements the call must write (and the comparisons of check 4 cover)."""
        p = torch.ones(self.nbytes, dtype=torch.bool, device=device)
        for m in (self.kept, self.unspec):
            if m is not None:
                p &= ~self._mask(m, device)
        return p


class Bufs:
    """The buffers of one call, carved out of guarded allocations (guarded=True) or plain torch tensors of the exact
    size that torch's allocator hands out (guarded=False, as every other test allocates them)."""

    def __init__(self, specs, device, guarded):
        self.specs, self.device, self.guarded = specs, device, guarded
        self.raw, self.start = {}, {}
        for name, s in specs.items():
            if guarded:
                raw = torch.empty(s.nbytes + 2 * s.guard + 256, dtype=torch.uint8, device=device)
                start = s.guard + (s.align - (raw.data_ptr() + s.guard)) % 256
                if s.writable():
                    raw.fill_(SENTINEL)
                else:
                    pat = s._poison_bytes(device)
                    raw.copy_(pat[(torch.arange(raw.numel(), device=device) - start) % s.esize])
            else:
                raw = torch.zeros(s.nbytes + 512, dtype=torch.uint8, device=device)
                start = s.align % 16 if s.same_phase else 0
            self.raw[name], self.start[name] = raw, start
            self.reset(name, guarded)

    def reset(self, name, guarded=True):
        """Restores a buffer's initial contents (the prefill of an output or workspace)."""
        s, v = self.specs[name], self.bytes(name)
        if s.kind in ("in", "inout"):
            v.copy_(s.data.to(self.device).view(torch.uint8).reshape(-1))
        elif s.kind == "out":
            v.fill_(PREFILL if guarded else PLAIN_FILL)
        else:
            v.fill_(PREFILL if guarded else 0)

    def bytes(self, name):
        s = self.specs[name]
        return self.raw[name][self.start[name]:self.start[name] + s.nbytes]

    def t(self, name):
        """The buffer as a flat tensor of its dtype."""
        return self.bytes(name).view(self.specs[name].dtype)

    def __getitem__(self, name):
        return self.bytes(name).data_ptr()

    def guards(self, name):
        r, a, s = self.raw[name], self.start[name], self.specs[name]
        return torch.cat([r[:a], r[a + s.nbytes:]])


# ---------------------------------------------------------------------------------------------------------------------
# cases and the checks

class Case:
    """One registered call.  `fn`: the C-ABI entry point's name, or a callable (the harness self-test).  `args(b)`
    returns its argument list for the buffers b (pointers b[name]).  `ws`: the workspace buffer's name, `ws_arg` the
    index of ws_bytes in the argument list.  `errors`: (expected code, {arg index: value}) calls that must fail and
    write nothing.  `check(b)`: value checks on the guarded outputs (float64 references, contract details)."""

    def __init__(self, fn, bufs, args, ws=None, ws_arg=None, errors=(), check=None):
        self.fn, self.bufs, self.args, self.ws, self.ws_arg = fn, bufs, args, ws, ws_arg
        self.errors, self.check = list(errors), check


def _sync(device):
    if torch.device(device).type == "cuda":
        torch.cuda.synchronize()


def _stream():
    return torch.cuda.current_stream().cuda_stream if torch.cuda.is_available() else None


def _call(case, b, over=None):
    args = list(case.args(b))
    for i, v in (over or {}).items():
        args[i] = v
    fn = getattr(_lib.load(), case.fn) if isinstance(case.fn, str) else case.fn
    rc = fn(*args)
    _sync(b.device)
    return rc


def _first(mask):
    return torch.nonzero(mask)[:1].flatten().tolist()


def _check_guards_and_inputs(case, b, before, what):
    for name, s in case.bufs.items():
        if s.writable():
            a, r = b.start[name], b.raw[name]
            bad = torch.cat([r[:a] != before[name][:a], r[a + s.nbytes:] != before[name][a + s.nbytes:]])
            if bad.any():
                i = int(_first(bad)[0])
                where = f"{a - i} bytes before" if i < a else f"{i - a + 1} bytes past the end"
                raise BoundsFailure("guard", f"{what}: {int(bad.sum())} guard bytes of `{name}` changed, first "
                                             f"{where}")
        elif not torch.equal(b.raw[name], before[name]):
            i = int(_first(b.raw[name] != before[name])[0]) - b.start[name]
            raise BoundsFailure("input", f"{what}: read-only `{name}` changed at byte {i} (of {s.nbytes})")


def _check_kept(case, b, before, what):
    for name, s in case.bufs.items():
        if s.kept is not None:
            m = s._mask(s.kept, b.device)
            a = b.start[name]
            bad = (b.bytes(name) != before[name][a:a + s.nbytes]) & m
            if bad.any():
                raise BoundsFailure("kept", f"{what}: `{name}` changed at element {_first(bad)[0] // s.esize}, "
                                            f"which the call must leave alone")


def _compare(check, case, name, got, want, what, device):
    s = case.bufs[name]
    p = s.promised(device)
    bad = (got != want) & p
    if not bad.any():
        return
    e = int(_first(bad)[0]) // s.esize
    ge, we = got[e * s.esize:(e + 1) * s.esize], want[e * s.esize:(e + 1) * s.esize]
    if check == "placement" and bool((ge == PREFILL).all()) and bool((we == PLAIN_FILL).all()):
        check = "coverage"
    raise BoundsFailure(check, f"{what}: `{name}` differs in {int(bad.sum())} bytes, first at element {e} of "
                               f"{s.numel}: {ge.tolist()} vs {we.tolist()}")


def _high_water(b, name):
    """Highest workspace byte that differs from its guarded prefill (-1: none)."""
    nz = torch.nonzero(b.bytes(name) != PREFILL)
    return int(nz[-1]) if nz.numel() else -1


def run_case(case, what, device="cuda"):
    """All checks of one case; raises BoundsFailure.  Returns the workspace high-water mark (or None)."""
    b = Bufs(case.bufs, device, guarded=True)
    before = {n: r.clone() for n, r in b.raw.items()}
    rc = _call(case, b)
    if rc != 0:
        raise BoundsFailure("call", f"{what}: returned {rc}")
    _check_guards_and_inputs(case, b, before, what)
    _check_kept(case, b, before, what)
    written = [n for n, s in case.bufs.items() if s.kind in ("out", "inout")]
    first = {n: b.bytes(n).clone() for n in written}
    hw = _high_water(b, case.ws) if case.ws else None
    if case.check is not None:
        case.check(b)

    # in place again, the workspace keeping the first call's leftovers
    for n in written:
        b.reset(n)
    rc = _call(case, b)
    if rc != 0:
        raise BoundsFailure("call", f"{what}: second call returned {rc}")
    _check_guards_and_inputs(case, b, before, what + " (second call)")
    _check_kept(case, b, before, what + " (second call)")
    for n in written:
        _compare("workspace", case, n, b.bytes(n), first[n], what + " (second call against the first)", device)
    if case.ws:
        hw = max(hw, _high_water(b, case.ws))

    # plain tensors, zeroed workspace
    p = Bufs(case.bufs, device, guarded=False)
    rc = _call(case, p)
    if rc != 0:
        raise BoundsFailure("call", f"{what}: plain call returned {rc}")
    for n in written:
        _compare("placement", case, n, first[n], p.bytes(n), what + " (guarded against plain tensors)", device)
    if case.ws:
        nz = torch.nonzero(p.bytes(case.ws))
        hw = max(hw, int(nz[-1]) if nz.numel() else -1)
    del p

    # error paths write nothing
    fails = list(case.errors)
    if case.ws:
        fails.append((VTM_E_WS, {case.ws_arg: case.bufs[case.ws].nbytes - 1}))
    for want, over in fails:
        for n, r in b.raw.items():
            r.copy_(before[n])
        rc = _call(case, b, over)
        if rc != want:
            raise BoundsFailure("error", f"{what}: with {over} returned {rc}, want {want}")
        for n, r in b.raw.items():
            if not torch.equal(r, before[n]):
                raise BoundsFailure("error", f"{what}: the failing call with {over} (code {rc}) changed `{n}`")
    return hw


# ---------------------------------------------------------------------------------------------------------------------
# inputs

def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(shape, g, scale=1.0):
    return (torch.randn(shape, generator=g, device="cuda") * scale).half()


def _tile_guard(rows, row_bytes):
    return max(GUARD_MIN, rows * row_bytes)


def _out(numel, row_bytes, rows=128, **kw):
    return Buf("out", numel=numel, guard=_tile_guard(rows, row_bytes), **kw)


def _ws(nbytes, **kw):
    """A workspace with guards as large as itself (within 64 MB): a size function that forgets a term of the layout
    makes the call store up to that term past the end."""
    return Buf("ws", numel=nbytes, guard=min(max(nbytes, GUARD_MIN), 1 << 26), **kw)


def _cols_kept(M, N, ld):
    return (torch.arange(ld) >= N).repeat(M)


def _lora_struct(b, down, up, R):
    return VtmLora(b[down], b[up], R) if R else None


def _ref(p):
    return None if p is None else ctypes.byref(p)


# ---- GEMMs --------------------------------------------------------------------------------------------------------

def _linear_cases():
    import test_gpu_projection_core as pc
    out = {}
    shapes = [(1, 200, 72, 224), (127, 200, 72, 208), (129, 136, 200, 144), (4099, 264, 136, 272)]
    cases = []
    for M, N, K, ldd in shapes:
        def make(M=M, N=N, K=K, ldd=ldd):
            g = _gen(M + N)
            a, w, bias = pc._exact_inputs(M, N, K, g)
            bufs = {"a": Buf("in", a), "w": Buf("in", w), "bias": Buf("in", bias),
                    "d": _out(M * ldd, ldd * 2, kept=_cols_kept(M, N, ldd))}
            want = pc._round16(pc._exact_product(a, w, bias))

            def check(b):
                pc._assert_equal(b.t("d").view(M, ldd)[:, :N], want, f"linear M={M} N={N} K={K}")
            return Case("vtm_linear_f16", bufs,
                        lambda b: [b["a"], b["w"], b["bias"], M, N, K, b["d"], ldd, _stream()],
                        errors=[(VTM_E_NULL, {0: None}), (VTM_E_SHAPE, {5: K + 4}), (VTM_E_SHAPE, {7: N - 8})],
                        check=check)
        cases.append((f"M={M} N={N} K={K} ldd={ldd}", make))
    out["vtm_linear_f16"] = cases

    cases = []
    for M, N, K, ldd, ldr in [(1, 200, 72, 208, 216), (129, 200, 200, 216, 264), (4099, 136, 72, 144, 152)]:
        def make(M=M, N=N, K=K, ldd=ldd, ldr=ldr):
            g = _gen(M + K)
            a, w, bias = pc._exact_inputs(M, N, K, g)
            resid = torch.full((M, ldr), float("nan"), dtype=torch.float16, device="cuda")
            resid[:, :N] = _randn((M, N), g, 64)
            bufs = {"a": Buf("in", a), "w": Buf("in", w), "bias": Buf("in", bias), "r": Buf("in", resid),
                    "d": _out(M * ldd, ldd * 2, kept=_cols_kept(M, N, ldd))}
            want = pc._round16(pc._round16(pc._exact_product(a, w, bias)) + resid[:, :N].double())

            def check(b):
                pc._assert_equal(b.t("d").view(M, ldd)[:, :N], want, f"linear_residual M={M} N={N}")
            return Case("vtm_linear_residual_f16", bufs,
                        lambda b: [b["a"], b["w"], b["bias"], b["r"], ldr, M, N, K, b["d"], ldd, _stream()],
                        errors=[(VTM_E_NULL, {3: None}), (VTM_E_SHAPE, {4: N - 8})], check=check)
        cases.append((f"M={M} N={N} K={K} ldd={ldd} ldr={ldr}", make))
    out["vtm_linear_residual_f16"] = cases

    cases = []
    for M, inner, K, ldd in [(1, 96, 72, 136), (129, 160, 200, 160), (4099, 32, 24, 72)]:
        def make(M=M, inner=inner, K=K, ldd=ldd):
            from vidtome_b200 import ops
            g = _gen(M + inner)
            a, w, bias = pc._exact_inputs(M, 2 * inner, K, g)
            wi, bi = ops.interleave_geglu(w, bias)
            bufs = {"a": Buf("in", a), "w": Buf("in", wi), "bias": Buf("in", bi),
                    "d": _out(M * ldd, ldd * 2, kept=_cols_kept(M, inner, ldd))}
            return Case("vtm_linear_geglu_f16", bufs,
                        lambda b: [b["a"], b["w"], b["bias"], M, 2 * inner, K, b["d"], ldd, _stream()],
                        errors=[(VTM_E_NULL, {1: None}), (VTM_E_SHAPE, {4: 2 * inner + 32})])
        cases.append((f"M={M} inner={inner} K={K} ldd={ldd}", make))
    out["vtm_linear_geglu_f16"] = cases

    cases = []
    for M, N, K, R, resid in [(1, 200, 72, 8, False), (129, 200, 136, 200, True), (4099, 136, 72, 200, False),
                              (127, 264, 200, 8, True)]:
        def make(M=M, N=N, K=K, R=R, resid=resid):
            g = _gen(M + R)
            a = _randn((M, K), g)
            w, bias = _randn((N, K), g, K ** -0.5), _randn((N,), g)
            down, up = _randn((R, K), g, 0.1), _randn((N, R), g, 0.1)
            ldd, ldr = N + 16, N + 8
            bufs = {"a": Buf("in", a), "w": Buf("in", w), "bias": Buf("in", bias), "down": Buf("in", down),
                    "up": Buf("in", up), "d": _out(M * ldd, ldd * 2, kept=_cols_kept(M, N, ldd)),
                    "ws": _ws(_lib.load().vtm_linear_lora_workspace_bytes(M, R))}
            if resid:
                r = torch.full((M, ldr), float("nan"), dtype=torch.float16, device="cuda")
                r[:, :N] = _randn((M, N), g)
                bufs["r"] = Buf("in", r)

            def args(b):
                lo = VtmLora(b["down"], b["up"], R)
                return [b["a"], b["w"], b["bias"], b["r"] if resid else None, ldr if resid else 0, ctypes.byref(lo), M,
                        N, K, b["d"], ldd, b["ws"], bufs["ws"].nbytes, _stream()]
            return Case("vtm_linear_lora_f16", bufs, args, ws="ws", ws_arg=12,
                        errors=[(VTM_E_NULL, {11: None}), (VTM_E_SHAPE, {8: K + 4})])
        cases.append((f"M={M} N={N} K={K} R={R} resid={resid}", make))
    out["vtm_linear_lora_f16"] = cases

    cases = []
    for M, inner, K, R in [(1, 96, 72, 8), (129, 160, 136, 200), (4099, 32, 72, 200)]:
        def make(M=M, inner=inner, K=K, R=R):
            from vidtome_b200 import ops
            g = _gen(M + inner + R)
            a = _randn((M, K), g)
            w, bias = _randn((2 * inner, K), g, K ** -0.5), _randn((2 * inner,), g)
            wi, bi = ops.interleave_geglu(w, bias)
            down, up = _randn((R, K), g, 0.1), _randn((2 * inner, R), g, 0.1)
            ui, _ = ops.interleave_geglu(up, None)
            ldd = inner + 8
            bufs = {"a": Buf("in", a), "w": Buf("in", wi), "bias": Buf("in", bi), "down": Buf("in", down),
                    "up": Buf("in", ui), "d": _out(M * ldd, ldd * 2, kept=_cols_kept(M, inner, ldd)),
                    "ws": _ws(_lib.load().vtm_linear_lora_workspace_bytes(M, R))}

            def args(b):
                lo = VtmLora(b["down"], b["up"], R)
                return [b["a"], b["w"], b["bias"], ctypes.byref(lo), M, 2 * inner, K, b["d"], ldd, b["ws"],
                        bufs["ws"].nbytes, _stream()]
            return Case("vtm_linear_geglu_lora_f16", bufs, args, ws="ws", ws_arg=10,
                        errors=[(VTM_E_NULL, {9: None}), (VTM_E_SHAPE, {5: 2 * inner + 32})])
        cases.append((f"M={M} inner={inner} K={K} R={R}", make))
    out["vtm_linear_geglu_lora_f16"] = cases

    cases = []
    # (n, HW, N, K, form): form "out" = separate d and resid, "inplace" = d == resid, "off16" = d and resid 2 bytes
    # past a 16-byte boundary with HW % 8 == 0 (the scalar store path chosen by alignment alone)
    for n, HW, N, K, form in [(3, 64, 200, 72, "out"), (2, 9, 136, 72, "out"), (3, 64, 200, 72, "inplace"),
                              (2, 64, 136, 136, "off16"), (1, 4096 + 3, 72, 72, "out"), (2, 1024, 320, 320, "inplace")]:
        def make(n=n, HW=HW, N=N, K=K, form=form):
            g = _gen(n * HW + N)
            a = _randn((n * HW, K), g)
            w, bias = _randn((N, K), g, K ** -0.5), _randn((N,), g)
            resid = _randn((n, N, HW), g)
            al = 2 if form == "off16" else 16
            bufs = {"a": Buf("in", a), "w": Buf("in", w), "bias": Buf("in", bias)}
            if form == "inplace":
                bufs["d"] = Buf("inout", resid, guard=_tile_guard(128, N * 2))
                rname = "d"
            else:
                bufs["r"] = Buf("in", resid, align=al)
                bufs["d"] = _out(n * N * HW, N * 2, align=al)
                rname = "r"
            return Case("vtm_linear_nchw_residual_f16", bufs,
                        lambda b: [b["a"], b["w"], b["bias"], b[rname], n, HW, N, K, b["d"], _stream()],
                        errors=[(VTM_E_NULL, {8: None}), (VTM_E_SHAPE, {6: N + 4})])
        cases.append((f"n={n} HW={HW} N={N} K={K} {form}", make))
    out["vtm_linear_nchw_residual_f16"] = cases
    return out


# ---- attention ----------------------------------------------------------------------------------------------------

def _dp(d):
    return 64 if d <= 64 else 128 if d <= 128 else 192


def _self_inputs(name, B, L, d, H, seed, w_o_eye=True):
    """x, W_qkv and scale from the signed-permutation designs of test_gpu_attention_core (exact q, k, v), W_o = I."""
    import test_gpu_attention_core as core
    g = _gen(seed)
    C = d * H
    x, w, scale = core._self_design(name, B, L, C, H, g)
    wo = torch.eye(C, dtype=torch.float16, device="cuda") if w_o_eye else _randn((C, C), g, C ** -0.5)
    return x, w, wo, scale, g


def _attn_f64(x, w, H, scale, flags, what, rows=None):
    """check(b) holding y (W_o = I, no bias) to the float64 bound of test_gpu_attention_core."""
    import test_gpu_attention_core as core
    import test_gpu_attention_wide as wide
    B, L, C = x.shape
    n = L if rows is None else rows
    q, k, v = wide._self_qkv(x[:, :n], w, H)
    O, bound = core._reference(q, k, v, scale, qk_shared=bool(flags & 1))

    def check(b):
        y = b.t("y").view(B, L, C)[:, :n]
        try:
            core._assert_within(y, O, bound, what)
        except pytest.fail.Exception as e:
            raise BoundsFailure("value", str(e)) from None
    return check


# (B, L, d, H): every head_dim class of the flash kernel at the lengths where its tiles end
SELF_SHAPES = [(2, 65, 8, 3), (2, 1, 40, 2), (1, 193, 80, 2), (2, 1000, 128, 2), (1, 4096, 160, 2), (1, 4096, 40, 8)]


def _attention_cases():
    lib = _lib.load
    out = {}

    def self_case(entry, B, L, d, H, flags=0, name="random", length=None, lora=None, resid=False, f64=True, items=1):
        x, w, wo, scale, g = _self_inputs(name, B, L, d, H, seed=B * L + d + flags)
        C = d * H
        if length is not None and length < L:
            x[:, length:] = _randn((B, L - length, C), g, 1000.0).clamp(-1000, 1000)
        Rq, Ro = lora or (0, 0)
        ws_bytes = lib().vtm_attention_lora_workspace_bytes(B, L, C, H, Rq, Ro)
        DP = _dp(d)
        ws_kept = None
        if flags & 1 and B > items:                     # q and k of samples items..B-1 are left as they were
            slab = B * H * L * DP
            ws_kept = torch.zeros(ws_bytes, dtype=torch.bool)
            per = H * L * DP * 2
            for j in range(2):
                ws_kept[(j * slab * 2) + per * items:(j * slab * 2) + slab * 2] = True
        unspec = None
        if length is not None:
            unspec = (torch.arange(L) >= length).repeat_interleave(C).repeat(B)
        bufs = {"x": Buf("in", x), "w": Buf("in", w), "wo": Buf("in", wo),
                "y": _out(B * L * C, C * 2, unspec=unspec), "ws": _ws(ws_bytes, kept=ws_kept)}
        if resid:
            bufs["r"] = Buf("in", torch.zeros_like(x) if f64 else _randn(x.shape, g))
        if length is not None:
            bufs["len"] = Buf("in", torch.tensor([length], dtype=torch.int32, device="cuda"), align=4, poison=length)
        if lora:
            for k, (R, N) in (("q", (Rq, 3 * C)), ("o", (Ro, C))):
                bufs["d" + k], bufs["u" + k] = Buf("in", _randn((R, C), g, 0.05)), Buf("in", _randn((N, R), g, 0.05))
        what = f"{entry} {name} B={B} L={L} d={d} H={H} flags={flags} items={items} len={length} lora={lora}"
        check = _attn_f64(x, w, H, scale, flags, what, rows=length) if f64 and not lora else None

        def los(b):
            return (VtmLora(b["dq"], b["uq"], Rq), VtmLora(b["do"], b["uo"], Ro)) if lora else (None, None)
        if entry == "vtm_attention":
            args = lambda b: [b["x"], b["w"], b["wo"], None, B, L, C, H, scale, b["y"], b["ws"], ws_bytes, _stream()]
            wsa, errs = 11, [(VTM_E_NULL, {9: None}), (VTM_E_SHAPE, {7: 7})]
        elif entry == "vtm_attention_ex":
            args = lambda b: [b["x"], b["w"], b["wo"], None, B, L, C, H, scale, flags, b["y"], b["ws"], ws_bytes,
                              _stream()]
            wsa, errs = 12, [(VTM_E_UNSUPPORTED, {9: 2}), (VTM_E_SHAPE, {5: 0})]
        elif entry == "vtm_attention_dev":
            args = lambda b: [b["x"], b["w"], b["wo"], None, B, L, C, H, scale, flags, b["len"], b["y"], b["ws"],
                              ws_bytes, _stream()]
            wsa, errs = 13, [(VTM_E_NULL, {10: None}), (VTM_E_UNSUPPORTED, {9: 4})]
        elif entry == "vtm_attention_lora":
            def args(b):
                lq, lo = los(b)
                return [b["x"], b["w"], b["wo"], None, _ref(lq), _ref(lo), B, L, C, H, scale, flags,
                        b["len"] if length is not None else None, b["y"], b["ws"], ws_bytes, _stream()]
            wsa, errs = 15, [(VTM_E_NULL, {14: None}), (VTM_E_SHAPE, {8: C + 4})]
        elif entry == "vtm_attention_residual_ex":
            def args(b):
                lq, lo = los(b)
                return [b["x"], b["w"], b["wo"], None, b["r"], _ref(lq), _ref(lo), B, L, C, H, scale, flags, items,
                        b["y"], b["ws"], ws_bytes, _stream()]
            wsa, errs = 16, [(VTM_E_NULL, {4: None}), (VTM_E_SHAPE, {12: 1, 13: B + 1})]
        else:
            def args(b):
                lq, lo = los(b)
                return [b["x"], b["w"], b["wo"], None, b["r"], _ref(lq), _ref(lo), B, L, C, H, scale, b["y"], b["ws"],
                        ws_bytes, _stream()]
            wsa, errs = 14, [(VTM_E_NULL, {4: None}), (VTM_E_SHAPE, {10: 0})]
        return Case(entry, bufs, args, ws="ws", ws_arg=wsa, errors=errs, check=check)

    def reg(entry, label, **kw):
        out.setdefault(entry, []).append((label, lambda: self_case(entry, **kw)))

    for B, L, d, H in SELF_SHAPES:
        reg("vtm_attention_ex", f"B={B} L={L} d={d} H={H}", B=B, L=L, d=d, H=H)
    reg("vtm_attention", "B=2 L=193 d=64 H=2", B=2, L=193, d=64, H=2)
    reg("vtm_attention", "B=1 L=4096 d=40 H=8 negative", B=1, L=4096, d=40, H=8, name="negative")
    for B, L, d in [(3, 65, 40), (4, 193, 128), (3, 1000, 160), (4, 1, 80)]:  # grouped CTAs, last group clamped
        reg("vtm_attention_ex", f"shared B={B} L={L} d={d}", B=B, L=L, d=d, H=2, flags=1)
    for B, L, d, H, n in [(2, 193, 40, 2, 1), (2, 193, 128, 2, 192), (2, 193, 80, 3, 193), (1, 1000, 160, 2, 999),
                          (3, 65, 40, 2, 64)]:
        reg("vtm_attention_dev", f"B={B} cap={L} len={n} d={d}", B=B, L=L, d=d, H=H, length=n,
            flags=1 if B == 3 else 0)
    for B, L, d, H, lo, n in [(2, 65, 40, 2, (8, 200), None), (1, 193, 80, 2, (200, 8), None),
                              (2, 193, 160, 2, (16, 40), 100), (3, 65, 40, 2, (8, 200), None)]:
        reg("vtm_attention_lora", f"B={B} L={L} d={d} R_qkv={lo[0]} R_o={lo[1]} len={n}", B=B, L=L, d=d, H=H,
            lora=lo, length=n, flags=1 if B == 3 else 0, f64=False)
    for B, L, d, H, lo in [(2, 193, 160, 2, None), (1, 1000, 160, 8, None), (2, 65, 40, 2, None),
                           (2, 65, 80, 2, (200, 8))]:
        reg("vtm_attention_residual", f"B={B} L={L} d={d} H={H} lora={lo}", B=B, L=L, d=d, H=H, resid=True, lora=lo,
            f64=lo is None)
    # flags 0, then the map shared from one item and from 3 of 6 (which _attn_f64 does not model), and LoRA
    for B, L, d, H, flags, items, lo in [(2, 193, 160, 2, 0, 1, None), (2, 65, 40, 2, 0, 1, None),
                                         (3, 65, 40, 2, 1, 1, None), (6, 65, 80, 2, 1, 3, None),
                                         (6, 193, 40, 2, 1, 3, (8, 16))]:
        reg("vtm_attention_residual_ex", f"B={B} L={L} d={d} H={H} flags={flags} items={items} lora={lo}", B=B, L=L,
            d=d, H=H, flags=flags, items=items, resid=True, lora=lo, f64=lo is None and items == 1)

    def cross_case(entry, B, Lq, Lk, d, H, lora=None, probe=False):
        import test_gpu_attention_core as core
        g = _gen(B * Lq + Lk + d)
        C = d * H
        if probe:                       # W_q = I, W_k = [I | 0], W_v = [0 | I]: the flash kernel on exactly Q, K, V
            Q, K, V, scale = core._probe_design("random", B, Lq, Lk, C, H, g)
            x, ctx, Cctx = Q, torch.cat([K, V], -1).contiguous(), 2 * C
            wq, wkv, wo = (torch.eye(n, dtype=torch.float16, device="cuda") for n in (C, 2 * C, C))
            O, bound = core._reference(core._heads(Q, H), core._heads(K, H), core._heads(V, H), scale)
        else:
            Cctx = 768
            x, ctx = _randn((B, Lq, C), g), _randn((B, Lk, Cctx), g)
            wq, wkv, wo = _randn((C, C), g, C ** -0.5), _randn((2 * C, Cctx), g, Cctx ** -0.5), _randn((C, C), g, 0.1)
            scale = d ** -0.5
        Rq, Rkv, Ro = lora or (0, 0, 0)
        ws_bytes = lib().vtm_cross_attention_lora_workspace_bytes(B, Lq, Lk, C, H, Rq, Rkv, Ro)
        bufs = {"x": Buf("in", x), "ctx": Buf("in", ctx), "wq": Buf("in", wq), "wkv": Buf("in", wkv),
                "wo": Buf("in", wo), "y": _out(B * Lq * C, C * 2), "ws": _ws(ws_bytes)}
        if not probe:
            bufs["bo"], bufs["r"] = Buf("in", _randn((C,), g)), Buf("in", _randn((B, Lq, C), g))
        if lora:
            for k, (R, K, N) in (("q", (Rq, C, C)), ("kv", (Rkv, Cctx, 2 * C)), ("o", (Ro, C, C))):
                bufs["d" + k], bufs["u" + k] = Buf("in", _randn((R, K), g, 0.05)), Buf("in", _randn((N, R), g, 0.05))
        what = f"{entry} B={B} Lq={Lq} Lk={Lk} d={d} H={H} lora={lora}"
        check = None
        if probe:
            def check(b):
                try:
                    core._assert_within(b.t("y").view(B, Lq, C), O, bound, what)
                except pytest.fail.Exception as e:
                    raise BoundsFailure("value", str(e)) from None

        def head(b):
            return [b["x"], b["ctx"], b["wq"], b["wkv"], b["wo"], None if probe else b["bo"], None if probe else b["r"]]
        if entry == "vtm_cross_attention":
            args = lambda b: head(b) + [B, Lq, Lk, C, Cctx, H, scale, b["y"], b["ws"], ws_bytes, _stream()]
            wsa = 16
        else:
            def args(b):
                ls = [VtmLora(b["d" + k], b["u" + k], R) for k, R in (("q", Rq), ("kv", Rkv), ("o", Ro))]
                return head(b) + [ctypes.byref(v) for v in ls] + [B, Lq, Lk, C, Cctx, H, scale, b["y"], b["ws"],
                                                                  ws_bytes, _stream()]
            wsa = 19
        return Case(entry, bufs, args, ws="ws", ws_arg=wsa,
                    errors=[(VTM_E_NULL, {1: None}), (VTM_E_SHAPE, {wsa - 5: Cctx + 4})], check=check)

    for B, Lq, Lk, d, H, probe in [(2, 193, 77, 40, 8, False), (3, 65, 1, 80, 2, True), (2, 1000, 7, 160, 2, True),
                                   (1, 4096, 77, 40, 8, False), (2, 1, 77, 128, 2, True)]:
        out.setdefault("vtm_cross_attention", []).append(
            (f"B={B} Lq={Lq} Lk={Lk} d={d} H={H}",
             lambda B=B, Lq=Lq, Lk=Lk, d=d, H=H, probe=probe: cross_case("vtm_cross_attention", B, Lq, Lk, d, H,
                                                                          probe=probe)))
    for B, Lq, Lk, d, H, lo in [(2, 193, 77, 40, 8, (8, 16, 200)), (2, 65, 7, 160, 2, (200, 8, 8)),
                                (1, 129, 1, 80, 4, (8, 200, 16))]:
        out.setdefault("vtm_cross_attention_lora", []).append(
            (f"B={B} Lq={Lq} Lk={Lk} d={d} R={lo}",
             lambda B=B, Lq=Lq, Lk=Lk, d=d, H=H, lo=lo: cross_case("vtm_cross_attention_lora", B, Lq, Lk, d, H,
                                                                    lora=lo)))
    return out


# ---- row kernels --------------------------------------------------------------------------------------------------

ROW_WIDTHS = (8, 136, 320, 1280, 2048)


def _table(B, N0, C, g, gap=1):
    """x [B, N0 + gap, C]: rows [N0, N0 + gap) of every sample hold NaN; row N0 is the poison row of index maps."""
    x = _randn((B, N0 + gap, C), g)
    x[:, N0:] = float("nan")
    return x


def _ln_bufs(C, g, bias=True):
    import test_gpu_rows_core as rc
    w, b, eps = rc._ln_params(C, g, bias)
    bufs = {"lw": Buf("in", w)}
    if b is not None:
        bufs["lb"] = Buf("in", b)
    return bufs, (w, b, eps)


def _rows_cases():
    import test_gpu_rows_core as rc
    out = {}

    def k0(entry, C, B, N, src_len, shared_map, ln):
        g = _gen(C + N + B)
        x = _table(B, N, C, g, gap=3)                  # batch stride N + 3 rows, the gap NaN
        bs = (N + 3) * C
        Bm = 1 if shared_map else B
        rowmap = torch.stack([torch.randperm(N, generator=g, device="cuda") for _ in range(Bm)]).int()
        Ns, Nd = src_len, N - src_len
        bufs = {"x": Buf("in", x), "map": Buf("in", rowmap, poison=N), "a": _out(B * Ns * C, C * 2, rows=1),
                "b": _out(B * Nd * C, C * 2, rows=1)}
        lnp = None
        if ln:
            lb, lnp = _ln_bufs(C, g)
            bufs.update(lb)
        sp = VtmSplit.prefix(N, src_len)

        def args(b):
            a = [b["x"], bs, b["map"], 0 if shared_map else N, ctypes.byref(sp), B, C]
            if entry == "vtm_normalize_split_ln":
                a += [b["lw"] if ln else None, b["lb"] if ln else None, lnp[2] if ln else 0.0]
            return a + [b["a"], b["b"], _stream()]
        bad = 8 if entry == "vtm_normalize_split" else 11
        return Case(entry, bufs, args, errors=[(VTM_E_NULL, {bad: None}), (VTM_E_SHAPE, {6: C + 4})])

    for i, C in enumerate(ROW_WIDTHS):
        B, N = 1 + i % 3, (129, 257, 65, 33, 20)[i]
        out.setdefault("vtm_normalize_split", []).append(
            (f"C={C} B={B} N={N}", lambda C=C, B=B, N=N, i=i: k0("vtm_normalize_split", C, B, N, N // 2, i % 2, False)))
        for ln in (True, False):
            out.setdefault("vtm_normalize_split_ln", []).append(
                (f"C={C} B={B} N={N} ln={ln}",
                 lambda C=C, B=B, N=N, ln=ln, i=i: k0("vtm_normalize_split_ln", C, B, N, N - 1, i % 2 == 0, ln)))

    def kc(entry, C, B, L, N0, shared, ln=False, n_peers=0, length=None):
        g = _gen(C + L + N0 + n_peers)
        x = _table(B, N0, C, g)
        xbs = (N0 + 1) * C
        Bm = 1 if shared else B
        mp = torch.randint(0, N0, (Bm, L), generator=g, device="cuda").int()
        ybs = (L + 2) * C                                   # two rows between samples that stay as they were
        kept = ((torch.arange(L + 2) >= L).repeat_interleave(C)).repeat(B)
        bufs = {"x": Buf("in", x), "map": Buf("in", mp, poison=N0),
                "y": _out(B * (L + 2) * C, C * 2, rows=1, kept=kept)}
        lnp = None
        if ln:
            lb, lnp = _ln_bufs(C, g, bias=C % 16 == 0)
            bufs.update(lb)
        for j in range(n_peers):
            bufs[f"p{j}"] = _out(B * (L + 2) * C, C * 2, rows=1, kept=kept)
        if length is not None:
            bufs["len"] = Buf("in", torch.tensor([length], dtype=torch.int32, device="cuda"), align=4, poison=length)
        mbs = 0 if shared else L
        what = f"{entry} C={C} B={B} L={L}"

        def lnargs(b):
            return [b["lw"] if ln else None, b["lb"] if ln and "lb" in bufs else None, lnp[2] if ln else 0.0]
        if entry == "vtm_gather_rows":
            args = lambda b: [b["x"], xbs, b["map"], mbs, B, L, C, b["y"], ybs, _stream()]
            errs = [(VTM_E_NULL, {7: None}), (VTM_E_SHAPE, {6: C + 4})]
        elif entry == "vtm_gather_rows_ln":
            args = lambda b: [b["x"], xbs, b["map"], mbs, B, L, C] + lnargs(b) + [b["y"], ybs, _stream()]
            errs = [(VTM_E_NULL, {0: None}), (VTM_E_SHAPE, {6: C + 4})]
        elif entry == "vtm_gather_rows_dev":
            args = lambda b: [b["x"], xbs, b["map"], mbs, B, L, C, b["len"], b["y"], ybs, _stream()]
            errs = [(VTM_E_NULL, {7: None}), (VTM_E_SHAPE, {6: C + 4})]
        else:
            def args(b):
                arr = (ctypes.c_void_p * max(1, n_peers))(*[b[f"p{j}"] for j in range(n_peers)])
                return [b["x"], xbs, b["map"], mbs, B, L, C] + lnargs(b) + [b["y"], ybs, arr, n_peers, _stream()]
            errs = [(VTM_E_NULL, {10: None}), (VTM_E_SHAPE, {13: 9})]

        def check(b):
            y = b.t("y").view(B, L + 2, C)[:, :L]
            n = L if length is None else length
            if length is not None and not (y[:, length:].view(torch.int16) == 0).all():
                raise BoundsFailure("value", f"{what}: rows [len, L_cap) are not zero")
            for j in range(n_peers):
                if not torch.equal(b.t(f"p{j}").view(B, L + 2, C)[:, :L].view(torch.int16), y.view(torch.int16)):
                    raise BoundsFailure("value", f"{what}: peer {j} differs from y")
            if ln:
                try:
                    rc._check_ln(y[:, :n], rc._gather(x, mp[:, :n]), lnp, what)
                except (AssertionError, pytest.fail.Exception) as e:
                    raise BoundsFailure("value", str(e)) from None
        return Case(entry, bufs, args, errors=errs, check=check)

    for i, C in enumerate(ROW_WIDTHS):
        B, L, N0 = 1 + i % 3, (129, 65, 257, 33, 17)[i], (300, 70, 400, 40, 30)[i]
        out.setdefault("vtm_gather_rows", []).append(
            (f"C={C} B={B} L={L}", lambda C=C, B=B, L=L, N0=N0, i=i: kc("vtm_gather_rows", C, B, L, N0, i % 2)))
        out.setdefault("vtm_gather_rows_ln", []).append(
            (f"C={C} B={B} L={L}", lambda C=C, B=B, L=L, N0=N0, i=i: kc("vtm_gather_rows_ln", C, B, L, N0, i % 2,
                                                                        ln=True)))
        out.setdefault("vtm_gather_rows_dev", []).append(
            (f"C={C} B={B} cap={L} len={L // 2 + 1}",
             lambda C=C, B=B, L=L, N0=N0, i=i: kc("vtm_gather_rows_dev", C, B, L, N0, i % 2, length=L // 2 + 1)))
    for C, ln in ((320, True), (1280, False), (8, True)):
        out.setdefault("vtm_gather_rows_peers", []).append(
            (f"C={C} ln={ln} two peers", lambda C=C, ln=ln: kc("vtm_gather_rows_peers", C, 2, 65, 100, False, ln=ln,
                                                               n_peers=2)))

    def ke(C, B, N, L, shared, resid):
        g = _gen(C + N + resid)
        y = _table(B, L, C, g)
        ybs = (L + 1) * C
        mp = torch.randint(0, L, (1 if shared else B, N), generator=g, device="cuda").int()
        bufs = {"y": Buf("in", y), "map": Buf("in", mp, poison=L), "out": _out(B * N * C, C * 2, rows=1)}
        if resid:
            bufs["r"] = Buf("in", _randn((B, N, C), g))
        return Case("vtm_unmerge_add", bufs,
                    lambda b: [b["y"], ybs, b["map"], 0 if shared else N, b["r"] if resid else None, B, N, C, b["out"],
                               _stream()],
                    errors=[(VTM_E_NULL, {8: None}), (VTM_E_SHAPE, {7: C + 4})])

    for i, C in enumerate(ROW_WIDTHS):
        for resid in (True, False):
            B, N, L = 1 + i % 3, (257, 129, 65, 33, 20)[i], (100, 70, 40, 20, 9)[i]
            out.setdefault("vtm_unmerge_add", []).append(
                (f"C={C} B={B} N={N} resid={resid}", lambda C=C, B=B, N=N, L=L, i=i, resid=resid: ke(C, B, N, L, i % 2,
                                                                                                     resid)))

    def kr(C, B, Bp, N, src_len, r, mode):
        import test_gpu_match_core as mc
        rng = np.random.default_rng(C + N + mode)
        Ns, Nd = src_len, N - src_len
        keys, edge, _, _, _ = mc._match_data(rng, B, Bp, Ns, Nd)
        g = _gen(C + N)
        x = _randn((B, N, C), g, 4.0)
        M = Ns - r + Nd
        ws_bytes = _lib.load().vtm_merge_reduce_workspace_bytes(B, Nd, C)
        bufs = {"x": Buf("in", x), "keys": Buf("in", mc._dev(keys.view(np.int64))),
                "edge": Buf("in", mc._dev(edge), poison=0), "y": _out(B * M * C, C * 2, rows=1), "ws": _ws(ws_bytes)}
        sp = VtmSplit.prefix(N, src_len)
        return Case("vtm_merge_reduce", bufs,
                    lambda b: [b["x"], N * C, ctypes.byref(sp), r, Bp, b["keys"], b["edge"], B, C, mode, b["y"],
                               b["ws"], ws_bytes, _stream()],
                    ws="ws", ws_arg=12, errors=[(VTM_E_UNSUPPORTED, {9: 5}), (VTM_E_NULL, {10: None})])

    for i, C in enumerate(ROW_WIDTHS):
        for mode in (1, 2, 3, 4):
            B, Bp = 2, 1 if (i + mode) % 2 else 2
            N, sl = (129, 65, 257, 33, 40)[i], (70, 30, 129, 16, 21)[i]
            r = (sl, sl // 2, 1, sl - 1)[mode - 1]
            out.setdefault("vtm_merge_reduce", []).append(
                (f"C={C} mode={mode} Bp={Bp} N={N} r={r}",
                 lambda C=C, B=B, Bp=Bp, N=N, sl=sl, r=r, mode=mode: kr(C, B, Bp, N, sl, r, mode)))
    return out


# ---- matching -----------------------------------------------------------------------------------------------------

MATCH_COUNTS = (1, 127, 129, 255, 257)


def _unit(shape, g):
    x = torch.randn(shape, generator=g, device="cuda", dtype=torch.float64)
    return (x / x.norm(dim=-1, keepdim=True)).half()


def _match_cases():
    import test_gpu_match_core as mc
    from test_match_core_cpu import sort_fused
    out = {}

    def ka(entry, B, Ns, Nd, C, align, cap=None):
        g = _gen(B + Ns + Nd + C)
        Bp = 1 if align else B
        ns_cap, nd_cap = (Ns, Nd) if cap is None else cap
        a, bb = _unit((B, ns_cap, C), g), _unit((B, nd_cap, C), g)
        bufs = {"a": Buf("in", a), "b": Buf("in", bb), "keys": _out(Bp * ns_cap, 8, dtype=torch.int64)}
        if entry == "vtm_sim_argmax_dev":
            bufs["cnt"] = Buf("in", torch.tensor([Ns, Nd, 0, Ns + Nd], dtype=torch.int32, device="cuda"), align=4,
                              poison=0)
            args = lambda b: [b["a"], b["b"], B, ns_cap, nd_cap, C, align, b["cnt"], b["keys"], _stream()]
            errs = [(VTM_E_NULL, {7: None}), (VTM_E_SHAPE, {5: C + 4})]
        else:
            args = lambda b: [b["a"], b["b"], B, Ns, Nd, C, align, b["keys"], _stream()]
            errs = [(VTM_E_NULL, {7: None}), (VTM_E_SHAPE, {5: C + 4})]

        def check(b):
            k = b.t("keys").view(Bp, ns_cap)
            if (k[:, Ns:] != 0).any():
                raise BoundsFailure("value", f"{entry}: keys of rows >= Ns are not 0")
        return Case(entry, bufs, args, errors=errs, check=check)

    for i, Ns in enumerate(MATCH_COUNTS):
        for j, Nd in enumerate(MATCH_COUNTS[i % 2::2]):
            align = (i + j) % 2
            B, C = 1 + (i + j) % 3, (64, 320, 136, 640, 8)[(i + j) % 5]
            for entry in ("vtm_sim_argmax", "vtm_sim_argmax_simt"):
                out.setdefault(entry, []).append(
                    (f"B={B} Ns={Ns} Nd={Nd} C={C} align={align}",
                     lambda entry=entry, B=B, Ns=Ns, Nd=Nd, C=C, align=align: ka(entry, B, Ns, Nd, C, align)))
    for Ns, Nd, cap, align in [(1, 257, (129, 257), 0), (127, 129, (255, 255), 1), (257, 1, (257, 127), 0),
                               (129, 255, (257, 257), 1)]:
        out.setdefault("vtm_sim_argmax_dev", []).append(
            (f"Ns={Ns} Nd={Nd} cap={cap} align={align}",
             lambda Ns=Ns, Nd=Nd, cap=cap, align=align: ka("vtm_sim_argmax_dev", 2, Ns, Nd, 320, align, cap)))

    def kb1(entry, Bp, Ns, n=None):
        rng = np.random.default_rng(Bp + Ns)
        keys = mc._sort_keys(rng, Bp, Ns)
        if n is not None:
            keys[:, n:] = np.uint64(0xFFFF) << np.uint64(32)
        ws_bytes = _lib.load().vtm_topr_workspace_bytes(Bp, Ns)
        kept = None if n is None else (torch.arange(Ns) >= n).repeat(Bp)
        bufs = {"keys": Buf("in", mc._dev(keys.view(np.int64))), "edge": _out(Bp * Ns, 4, kept=kept, dtype=torch.int32),
                "rank": _out(Bp * Ns, 4, kept=kept, dtype=torch.int32), "ws": _ws(ws_bytes)}
        what = f"{entry} Bp={Bp} Ns={Ns} n={n}"
        if n is None:
            args = lambda b: [b["keys"], Bp, Ns, b["edge"], b["rank"], b["ws"], ws_bytes, _stream()]
            wsa = 6
        else:
            bufs["cnt"] = Buf("in", torch.tensor([n, 1, 0, n + 1], dtype=torch.int32, device="cuda"), align=4, poison=0)
            args = lambda b: [b["keys"], Bp, Ns, b["cnt"], b["edge"], b["rank"], b["ws"], ws_bytes, _stream()]
            wsa = 7

        def check(b):
            edge = b.t("edge").view(Bp, Ns).cpu().numpy()
            rank = b.t("rank").view(Bp, Ns).cpu().numpy()
            mc._check_sort(keys, edge, rank, Ns if n is None else n, what)
            if n is None:       # the path that ran, from the workspace's grid-barrier word
                ws = b.bytes("ws").cpu().numpy()
                tiles = -(-Ns // 1024)
                off = 2 * (-(-4 * Bp * 256 * tiles // 256) * 256)
                word = int(ws[off:off + 4].view(np.uint32)[0])
                fused = word == 3 * tiles * Bp
                assert fused or word == int(np.frombuffer(bytes([PREFILL] * 4), np.uint32)[0]), f"{what}: {word:#x}"
                assert fused == sort_fused(Bp, Ns), f"{what}: ran the {'fused' if fused else 'fallback'} sort"
        return Case(entry, bufs, args, ws="ws", ws_arg=wsa,
                    errors=[(VTM_E_NULL, {0: None}), (VTM_E_SHAPE, {2: 0})], check=check)

    for Bp, Ns in [(1, 1), (2, 1023), (3, 1024), (1, 1025), (4, 2047), (1, 264 * 1024), (1, 265 * 1024 + 1),
                   (3, 89 * 1024)]:
        out.setdefault("vtm_topr_sort", []).append(
            (f"Bp={Bp} Ns={Ns} {'fused' if sort_fused(Bp, Ns) else 'six launches'}",
             lambda Bp=Bp, Ns=Ns: kb1("vtm_topr_sort", Bp, Ns)))
    for Bp, Ns, n in [(1, 1025, 1), (2, 3000, 2047), (3, 1024, 1023)]:
        out.setdefault("vtm_topr_sort_dev", []).append(
            (f"Bp={Bp} cap={Ns} n={n}", lambda Bp=Bp, Ns=Ns, n=n: kb1("vtm_topr_sort_dev", Bp, Ns, n)))

    def kb2(B, Bp, N, src_len, r, chained):
        rng = np.random.default_rng(N + r + chained)
        Ns, Nd = src_len, N - src_len
        keys, edge, rank, _, _ = mc._match_data(rng, B, Bp, Ns, Nd)
        N0 = N + 7 if chained else N
        M = Ns - r + Nd
        bufs = {"keys": Buf("in", mc._dev(keys.view(np.int64))), "edge": Buf("in", mc._dev(edge), poison=0),
                "rank": Buf("in", mc._dev(rank), poison=0), "mu": _out(Bp * M, 4, dtype=torch.int32),
                "pi": _out(Bp * N0, 4, dtype=torch.int32)}
        if chained:
            bufs["mu_in"] = Buf("in", mc._dev(rng.integers(0, N0, (Bp, N)).astype(np.int32)), poison=0)
            bufs["pi_in"] = Buf("in", mc._dev(rng.integers(0, N, (Bp, N0)).astype(np.int32)), poison=0)
        sp = VtmSplit.prefix(N, src_len)
        return Case("vtm_compose_maps", bufs,
                    lambda b: [ctypes.byref(sp), r, Ns, Nd, Bp, b["keys"], b["edge"], b["rank"],
                               b["mu_in"] if chained else None, b["pi_in"] if chained else None, 0, N0, b["mu"],
                               b["pi"], _stream()],
                    errors=[(VTM_E_NULL, {12: None}), (VTM_E_SHAPE, {1: Ns + 1})])

    for B, Bp, N, sl, r, ch in [(2, 2, 258, 129, 64, False), (3, 1, 256, 127, 127, True), (1, 1, 2, 1, 1, False),
                                (2, 1, 512, 255, 0, True), (2, 2, 514, 257, 200, False)]:
        out.setdefault("vtm_compose_maps", []).append(
            (f"B={B} Bp={Bp} N={N} Ns={sl} r={r} chained={ch}",
             lambda B=B, Bp=Bp, N=N, sl=sl, r=r, ch=ch: kb2(B, Bp, N, sl, r, ch)))

    def mode2(L, gcap, lg, high):
        coin = torch.tensor([0.75 if high else 0.25], dtype=torch.float32, device="cuda")
        glen = torch.tensor([lg], dtype=torch.int32, device="cuda")
        return coin, glen

    def kb2_dev(L, gcap, lg, high, pi_in):
        rng = np.random.default_rng(L + gcap + lg + high)
        B, Bp = 2, 1 + (L % 2)
        coin, glen = mode2(L, gcap, lg, high)
        Ns, Nd = (L, lg) if high else (lg, L)
        r = Ns // 2
        keys, edge, rank, _, _ = mc._match_data(rng, B, Bp, Ns, Nd)
        cap = max(L, gcap)
        K, E, R = np.zeros((Bp, cap), np.uint64), np.zeros((Bp, cap), np.int32), np.zeros((Bp, cap), np.int32)
        K[:, :Ns], E[:, :Ns], R[:, :Ns] = keys, edge, rank
        N = L + gcap
        M = Ns - r + Nd
        N0 = N + 5 if pi_in else N
        bufs = {"coin": Buf("in", coin, align=4), "glen": Buf("in", glen, align=4, poison=lg),
                "cnt": Buf("in", torch.tensor([Ns, Nd, r, M], dtype=torch.int32, device="cuda"), align=4, poison=0),
                "keys": Buf("in", mc._dev(K.view(np.int64))), "edge": Buf("in", mc._dev(E), poison=0),
                "rank": Buf("in", mc._dev(R), poison=0),
                "mu": _out(Bp * N, 4, dtype=torch.int32, unspec=(torch.arange(N) >= M).repeat(Bp)),
                "pi": _out(Bp * N0, 4, dtype=torch.int32,
                           kept=None if pi_in else (torch.arange(N0) >= L + lg).repeat(Bp))}
        if pi_in:
            bufs["pi_in"] = Buf("in", mc._dev(rng.integers(0, L + lg, (Bp, N0)).astype(np.int32)), poison=0)

        def args(b):
            sp = VtmSplit.prefix_coin_dev(L, b.t("glen"), gcap, b.t("coin"), 0.5)
            return [ctypes.byref(sp), b["cnt"], Bp, b["keys"], b["edge"], b["rank"], b["pi_in"] if pi_in else None,
                    N0, b["mu"], b["pi"], _stream()]
        return Case("vtm_compose_maps_dev", bufs, args, errors=[(VTM_E_NULL, {1: None}), (VTM_E_NULL, {9: None})])

    for L, gcap, lg, high, pi_in in [(30, 40, 25, True, False), (40, 30, 30, False, False), (17, 64, 1, True, True),
                                     (129, 257, 255, False, True)]:
        out.setdefault("vtm_compose_maps_dev", []).append(
            (f"L={L} glob_cap={gcap} glob_len={lg} coin_high={high} pi_in={pi_in}",
             lambda L=L, gcap=gcap, lg=lg, high=high, pi_in=pi_in: kb2_dev(L, gcap, lg, high, pi_in)))

    def decode(B, Bp, Ns, Nd, r, optional):
        rng = np.random.default_rng(Ns + Nd + r)
        keys, edge, _, _, _ = mc._match_data(rng, B, Bp, Ns, Nd)
        bufs = {"keys": Buf("in", mc._dev(keys.view(np.int64))), "edge": Buf("in", mc._dev(edge), poison=0),
                "unm": _out(Bp * (Ns - r), 8, dtype=torch.int64), "src": _out(Bp * r, 8, dtype=torch.int64),
                "dst": _out(Bp * r, 8, dtype=torch.int64)}
        if optional:
            bufs["nmax"] = _out(Bp * Ns, 2, dtype=torch.int16)
            bufs["nidx"] = _out(Bp * Ns, 8, dtype=torch.int64)
        for k in ("unm", "src", "dst"):
            if bufs[k].numel == 0:
                del bufs[k]
        p = lambda b, k: b[k] if k in bufs else None
        return Case("vtm_decode_match", bufs,
                    lambda b: [b["keys"], b["edge"], Bp, Ns, Nd, r, p(b, "unm"), p(b, "src"), p(b, "dst"),
                               p(b, "nmax"), p(b, "nidx"), _stream()],
                    errors=[(VTM_E_NULL, {0: None}), (VTM_E_SHAPE, {5: Ns + 1})])

    for B, Bp, Ns, Nd, r, opt in [(1, 1, 1, 1, 0, True), (2, 2, 127, 129, 64, True), (3, 1, 257, 255, 128, False),
                                  (2, 1, 129, 1, 129, True), (2, 2, 255, 257, 1, False)]:
        out.setdefault("vtm_decode_match", []).append(
            (f"B={B} Bp={Bp} Ns={Ns} Nd={Nd} r={r} optional={opt}",
             lambda B=B, Bp=Bp, Ns=Ns, Nd=Nd, r=r, opt=opt: decode(B, Bp, Ns, Nd, r, opt)))

    def counts(L, gcap, lg, high, ratio):
        coin, glen = mode2(L, gcap, lg, high)
        Ns, Nd = (L, lg) if high else (lg, L)
        rr = min(Ns, int(Ns * ratio))
        bufs = {"coin": Buf("in", coin, align=4), "glen": Buf("in", glen, align=4, poison=lg),
                "cnt": _out(4, 16, dtype=torch.int32)}

        def args(b):
            sp = VtmSplit.prefix_coin_dev(L, b.t("glen"), gcap, b.t("coin"), 0.5)
            return [ctypes.byref(sp), ratio, b["cnt"], _stream()]

        def check(b):
            assert b.t("cnt").tolist() == [Ns, Nd, rr, Ns - rr + Nd]
        return Case("vtm_split_counts_dev", bufs, args, errors=[(VTM_E_NULL, {2: None})], check=check)

    for L, gcap, lg, high, ratio in [(30, 40, 25, True, 0.9), (257, 129, 127, False, 0.5), (1, 1, 1, True, 1.0)]:
        out.setdefault("vtm_split_counts_dev", []).append(
            (f"L={L} glob_cap={gcap} glob_len={lg} coin_high={high} ratio={ratio}",
             lambda L=L, gcap=gcap, lg=lg, high=high, ratio=ratio: counts(L, gcap, lg, high, ratio)))
    return out


# ---- KT, KI, KG1, KG2 ---------------------------------------------------------------------------------------------

def _misc_cases():
    out = {}

    def kt(n, num_inputs, E, inject, aligns):
        g = _gen(n + E + inject)
        B = n * num_inputs
        h = _randn((n if inject else B, E), g, 3.0)
        s = _randn((B, E), g, 3.0)
        ah, as_, ao = aligns
        bufs = {"h": Buf("in", h, align=ah), "s": Buf("in", s, align=as_),
                "out": _out(B * E, E * 2, rows=1, align=ao)}
        return Case("vtm_resnet_tail_f16", bufs,
                    lambda b: [b["h"], b["s"], b["out"], n, num_inputs, E, 2.0 ** -0.5, inject, _stream()],
                    errors=[(VTM_E_UNSUPPORTED, {4: 4}), (VTM_E_UNSUPPORTED, {6: 0.0}), (VTM_E_NULL, {2: None})])

    for n, ni, E, inj, al in [(2, 3, 1001, 0, (16, 16, 16)), (2, 3, 1001, 1, (18, 18, 18)), (1, 2, 9, 0, (2, 2, 2)),
                              (3, 2, 4096 + 7, 1, (16, 18, 20)), (4, 3, 64, 0, (2, 16, 2)), (1, 1, 1, 0, (2, 2, 2))]:
        out.setdefault("vtm_resnet_tail_f16", []).append(
            (f"n={n} num_inputs={ni} E={E} inject={inj} align={al}",
             lambda n=n, ni=ni, E=E, inj=inj, al=al: kt(n, ni, E, inj, al)))

    def ki(n, n_steps, step, aligns, with_slots):
        g = _gen(n + step)
        x, eps = _randn((n,), g), _randn((n,), g)
        coef = torch.stack([torch.rand(n_steps, generator=g, device="cuda") + 0.1 for _ in range(4)], 1).float()
        slots = torch.full((n_steps,), -1, dtype=torch.int32, device="cuda")
        slots[::3] = torch.arange(0, n_steps, 3, device="cuda").int() // 3
        n_slots = int(slots.max()) + 1
        ax, ae, at = aligns
        in_range = 0 <= step < n_steps
        bufs = {"x": Buf("inout", x, align=ax, guard=GUARD_MIN,
                         kept=None if in_range else torch.ones(n, dtype=torch.bool)),
                "eps": Buf("in", eps, align=ae), "coef": Buf("in", coef),
                "step": Buf("in", torch.tensor([step], dtype=torch.int32, device="cuda"), align=4, poison=0)}
        if with_slots:
            s = int(slots[step]) if in_range else -1
            kept = torch.ones((n_slots, n), dtype=torch.bool)
            if s >= 0:
                kept[s] = False
            bufs["slot"] = Buf("in", slots, align=4, poison=-1)
            bufs["traj"] = _out(n_slots * n, n * 2, rows=1, align=at, kept=kept)
        return Case("vtm_ddim_update_f16", bufs,
                    lambda b: [b["x"], b["eps"], n, b["coef"], b["slot"] if with_slots else None, b["step"], n_steps,
                               b["traj"] if with_slots else None, n_slots if with_slots else 0, _stream()],
                    errors=[(VTM_E_NULL, {3: None}), (VTM_E_SHAPE, {2: 0})] +
                           ([(VTM_E_NULL, {7: None}), (VTM_E_SHAPE, {8: 0})] if with_slots else []))

    for n, steps, step, al, sl in [(4096 + 5, 10, 0, (16, 16, 16), True), (1001, 10, 3, (2, 4, 6), True),
                                   (1, 10, 9, (2, 2, 2), True), (777, 10, 10, (16, 18, 16), True),
                                   (777, 10, -1, (2, 2, 2), True), (4096, 10, 4, (18, 18, 18), False)]:
        out.setdefault("vtm_ddim_update_f16", []).append(
            (f"n={n} step={step} of {steps} align={al} slots={sl}",
             lambda n=n, steps=steps, step=step, al=al, sl=sl: ki(n, steps, step, al, sl)))

    def kg1(n, C, HW, groups, ax):
        import test_gpu_transformer_io as tio
        g = _gen(n + C + HW)
        x = (torch.randn((n, C, HW), generator=g, device="cuda") * 1.5 + 0.3).half()
        ws_bytes = _lib.load().vtm_group_norm_stats_workspace_bytes(n, C, HW, groups)
        # the sums start at x's first 16-byte boundary: their rounding depends on x's offset from one (the header)
        bufs = {"x": Buf("in", x, align=ax, same_phase=True),
                "stats": _out(n * groups * 2, 8, dtype=torch.float32, align=8)}
        if ws_bytes:
            bufs["ws"] = _ws(ws_bytes)

        def check(b):
            got = b.t("stats").view(n, groups, 2)
            tio._check_stats(x, groups, 1e-6, f"KG1 n={n} C={C} HW={HW}", got=got)
        return Case("vtm_group_norm_stats_f16", bufs,
                    lambda b: [b["x"], n, C, HW, groups, 1e-6, b["stats"], b["ws"] if ws_bytes else None, ws_bytes,
                               _stream()],
                    ws="ws" if ws_bytes else None, ws_arg=8,
                    errors=[(VTM_E_NULL, {6: None}), (VTM_E_SHAPE, {4: 7})], check=check)

    for n, C, HW, ax in [(1, 320, 9216, 2), (2, 64, 9, 2), (3, 1280, 64, 16), (1, 640, 4096 + 1, 18), (40, 320, 64, 2)]:
        out.setdefault("vtm_group_norm_stats_f16", []).append(
            (f"n={n} C={C} HW={HW} x_align={ax}", lambda n=n, C=C, HW=HW, ax=ax: kg1(n, C, HW, 32, ax)))

    def kg2(n, C, HW, groups, ax, affine):
        g = _gen(n + C + HW + affine)
        x = _randn((n, C, HW), g, 2.0)
        stats = torch.stack([torch.randn((n, groups), generator=g, device="cuda"),
                             torch.rand((n, groups), generator=g, device="cuda") + 0.5], -1).float()
        bufs = {"x": Buf("in", x, align=ax), "stats": Buf("in", stats, align=8),
                "y": _out(n * HW * C, C * 2, rows=1)}
        if affine:
            bufs["gm"], bufs["bt"] = Buf("in", _randn((C,), g)), Buf("in", _randn((C,), g))
        return Case("vtm_group_norm_tokens_f16", bufs,
                    lambda b: [b["x"], b["stats"], b["gm"] if affine else None, b["bt"] if affine else None, n, C, HW,
                               groups, b["y"], _stream()],
                    errors=[(VTM_E_NULL, {8: None}), (VTM_E_SHAPE, {7: 7})])

    for n, C, HW, ax, aff in [(2, 320, 64, 16, True), (1, 320, 63, 2, True), (3, 64, 9, 2, False),
                              (2, 1280, 256, 18, True), (1, 640, 4096 + 8, 16, False)]:
        out.setdefault("vtm_group_norm_tokens_f16", []).append(
            (f"n={n} C={C} HW={HW} x_align={ax} affine={aff}",
             lambda n=n, C=C, HW=HW, ax=ax, aff=aff: kg2(n, C, HW, 32, ax, aff)))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# registry

def _registry():
    reg = {}
    for part in (_linear_cases, _attention_cases, _rows_cases, _match_cases, _misc_cases):
        for entry, cases in part().items():
            reg.setdefault(entry, []).extend(cases)
    return reg


# entry point -> [(label, case factory)]; building it imports the core test modules (torch only), and a factory makes
# CUDA tensors only when it runs
REGISTRY = _registry()


def _ids():
    return [(e, label) for e, cases in REGISTRY.items() for label, _ in cases]


@pytest.mark.parametrize("entry,label", _ids(), ids=[f"{e}[{l}]" for e, l in _ids()])
def test_bounds(entry, label):
    make = dict(REGISTRY[entry])[label]
    case = make()
    assert case.fn == entry
    what = f"{entry} [{label}]"
    hw = run_case(case, what)
    if hw is None:
        print(f"bounds {what}: ok (no workspace)")
    else:
        ws_bytes = case.bufs[case.ws].nbytes
        print(f"bounds {what}: ok; workspace {ws_bytes} B, highest byte written {hw} "
              f"({ws_bytes - 1 - hw} B never written at the end)")
