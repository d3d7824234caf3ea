"""The bounds harness of test_gpu_bounds.py without a GPU: its registry names every compute entry point of the C-ABI,
every prototype of include/vidtome_b200.h matches its ctypes binding argument by argument, and the harness catches
fake kernels (torch ops on CPU tensors) that store past an output, write an input, read an input's guard, leave an
output element unwritten or depend on the workspace's previous contents."""
import ctypes as C
import os
import re

import pytest
import torch

import test_gpu_bounds as tb
from vidtome_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST_ONLY = {"vtm_version", "vtm_error_string", "vtm_split_counts", "vtm_merge_count", "vtm_key_score_half_bits",
             "vtm_key_arg"}


def _compute_entries():
    return {n for n in _lib.SIGNATURES if n not in HOST_ONLY and not n.endswith("_workspace_bytes")}


def test_registry_covers_every_compute_entry_point():
    assert set(tb.REGISTRY) == _compute_entries()
    assert all(tb.REGISTRY[e] for e in tb.REGISTRY), "an entry point without cases"


# ---------------------------------------------------------------------------------------------------------------------
# header prototypes against the ctypes bindings

def _prototypes():
    src = open(os.path.join(ROOT, "include", "vidtome_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    src = re.sub(r"#[^\n]*", " ", src)
    out = {}
    for m in re.finditer(r"([A-Za-z_][\w\s\*]*?)\b(vtm_\w+)\s*\(([^;{]*?)\)\s*;", src):
        ret, name, params = m.group(1), m.group(2), m.group(3)
        ps = [] if params.strip() in ("", "void") else [re.sub(r"\b\w+\s*$", "", p).strip() for p in params.split(",")]
        out[name] = (" ".join(ret.split()), ps)
    return out


_INTS = {"int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "size_t": C.c_size_t, "uint16_t": C.c_uint16,
         "uint32_t": C.c_uint32, "uint64_t": C.c_uint64, "float": C.c_float, "double": C.c_double}


def _kind(ctype):
    """A C type string -> ("ptr", pointee or None) / ("val", ctypes type)."""
    t = " ".join(ctype.replace("const", " ").split())
    if t.endswith("*"):
        base = t.rstrip("* ").strip()
        return ("ptr", "char" if base == "char" else base)
    return ("val", _INTS[t])


def _ctypes_kind(ct):
    if ct in (C.c_void_p, C.c_char_p) or (isinstance(ct, type) and issubclass(ct, C._Pointer)):
        return "ptr"
    return "val"


def _size_sign(ct):
    return C.sizeof(ct), ct in (C.c_float, C.c_double), ct(-1).value < 0 if ct not in (C.c_float, C.c_double) else True


def test_header_prototypes_match_the_bindings():
    protos = _prototypes()
    assert set(protos) == set(_lib.SIGNATURES), "header and bindings name different functions"
    for name, (ret, params) in protos.items():
        res, args = _lib.SIGNATURES[name]
        assert len(params) == len(args), f"{name}: {len(params)} parameters in the header, {len(args)} bound"
        for i, (p, a) in enumerate([(ret, res)] + list(zip(params, args))):
            where = f"{name}: {'return value' if i == 0 else f'argument {i - 1} ({p})'}"
            kind, t = _kind(p)
            assert kind == _ctypes_kind(a), f"{where}: pointer-ness differs ({a})"
            if kind == "val":
                assert _size_sign(t) == _size_sign(a), f"{where}: bound as {a.__name__}"
            elif t == "vtm_split_t":
                assert a is _lib._SPL, f"{where}: not a vtm_split_t pointer"
            elif t == "vtm_lora_t":
                assert a is _lib._LORA, f"{where}: not a vtm_lora_t pointer"


def test_struct_layouts_match_the_header():
    assert C.sizeof(_lib.VtmSplitDev) == 72 and C.sizeof(_lib.VtmSplit) == 56
    assert _lib.VtmSplit.coin_threshold.offset == 48 and _lib.VtmSplitDev.glob_cap.offset == 64
    assert C.sizeof(_lib.VtmLora) == 24 and _lib.VtmLora.R.offset == 16


# ---------------------------------------------------------------------------------------------------------------------
# the harness against fake kernels

N = 40


def _fake_case(fn, ws=False):
    x = torch.arange(N, dtype=torch.float16)
    bufs = {"x": tb.Buf("in", x), "y": tb.Buf("out", numel=N)}
    if not ws:
        return tb.Case(fn, bufs, lambda b: [b])
    bufs["ws"] = tb.Buf("ws", numel=4 * N)
    return tb.Case(lambda b, ws_bytes: tb.VTM_E_WS if ws_bytes < 4 * N else fn(b), bufs, lambda b: [b, 4 * N],
                   ws="ws", ws_arg=1)


def _raw_past(b, name, k):
    """The k-th element past the end of buffer `name` (inside its trailing guard), as a 2-byte tensor."""
    s = b.start[name] + b.specs[name].nbytes + 2 * k
    return b.raw[name][s:s + 2].view(torch.float16)


def _good(b):
    b.t("y").copy_(b.t("x") * 2)
    return 0


def _store_past(b):
    _good(b)
    _raw_past(b, "y", 0).copy_(b.t("y")[-1:])
    return 0


def _write_input(b):
    _good(b)
    b.t("x")[3] += 1
    return 0


def _read_guard(b):
    _good(b)
    b.t("y")[-1] = b.t("x")[-1] + _raw_past(b, "x", 0)[0]
    return 0


def _skip_last(b):
    b.t("y")[:-1] = b.t("x")[:-1] * 2
    return 0


def _accumulate(b):
    acc = b.t("ws")[:N]
    acc += b.t("x").to(torch.uint8)
    b.t("y").copy_(acc.half())
    return 0


def test_harness_passes_a_correct_fake():
    tb.run_case(_fake_case(_good), "good", device="cpu")
    tb.run_case(_fake_case(lambda b: (_good(b), b.t("ws").zero_())[0], ws=True), "good with workspace", device="cpu")


@pytest.mark.parametrize("fake,check,ws", [(_store_past, "guard", False), (_write_input, "input", False),
                                           (_read_guard, "placement", False), (_skip_last, "coverage", False),
                                           (_accumulate, "workspace", True)])
def test_harness_catches(fake, check, ws):
    with pytest.raises(tb.BoundsFailure) as e:
        tb.run_case(_fake_case(fake, ws), fake.__name__, device="cpu")
    assert e.value.check == check, str(e.value)


def test_harness_catches_a_store_into_kept_elements():
    case = _fake_case(_good)
    case.bufs["y"].kept = torch.arange(N) >= N - 1           # the call may not write the last element
    with pytest.raises(tb.BoundsFailure) as e:
        tb.run_case(case, "kept", device="cpu")
    assert e.value.check == "kept"


def test_harness_checks_error_paths():
    def refuses_but_writes(b):
        b.t("y")[0] = 1
        return tb.VTM_E_SHAPE
    case = _fake_case(lambda b, *_: _good(b))
    case.args = lambda b: [b, 0]
    case.fn = lambda b, flag: refuses_but_writes(b) if flag else _good(b)
    case.errors = [(tb.VTM_E_SHAPE, {1: 1})]
    with pytest.raises(tb.BoundsFailure) as e:
        tb.run_case(case, "error path", device="cpu")
    assert e.value.check == "error"


def test_input_guards_hold_the_poison():
    x = torch.arange(8, dtype=torch.int32)
    b = tb.Bufs({"m": tb.Buf("in", x, poison=8, align=4), "h": tb.Buf("in", torch.ones(5, dtype=torch.float16),
                                                                        align=2)}, "cpu", guarded=True)
    assert b["m"] % 256 == 4 and b["h"] % 256 == 2
    assert torch.equal(b.t("m"), x) and (b.guards("m").view(torch.int32) == 8).all()
    assert torch.isnan(b.guards("h").view(torch.float16)).all()
    assert b.guards("m").numel() >= 2 * tb.GUARD_MIN
