"""Token / RNG helpers with the reference's names and semantics (vidtome/utils.py:4-60)."""
from __future__ import annotations

import numpy as np
import torch


def isinstance_str(x: object, cls_name: str) -> bool:
    """True if any class *named* cls_name is in x's MRO (vidtome/utils.py:4-16).  The patch API matches
    diffusers classes by name so that it never has to import diffusers."""
    return any(c.__name__ == cls_name for c in x.__class__.__mro__)


def init_generator(device: torch.device, fallback: torch.Generator = None) -> torch.Generator:
    """Fork the current default RNG state of `device` into a new generator (vidtome/utils.py:18-30)."""
    if device.type == "cpu":
        return torch.Generator(device="cpu").set_state(torch.get_rng_state())
    if device.type == "cuda":
        return torch.Generator(device=device).set_state(torch.cuda.get_rng_state())
    if fallback is None:
        return init_generator(torch.device("cpu"))
    return fallback


def join_frame(x: torch.Tensor, fsize: int) -> torch.Tensor:
    """"(B F) N C -> B (F N) C" (vidtome/utils.py:32-35).  A view for contiguous input."""
    bf, n, c = x.shape
    return x.reshape(bf // fsize, fsize * n, c)


def split_frame(x: torch.Tensor, fsize: int) -> torch.Tensor:
    """"B (F N) C -> (B F) N C" (vidtome/utils.py:37-40)."""
    b, fn, c = x.shape
    return x.reshape(b * fsize, fn // fsize, c)


def func_warper(funcs):
    """Compose a list of ops left to right, passing keyword arguments through (vidtome/utils.py:42-48)."""
    def fn(x, **kwarg):
        for func in funcs:
            x = func(x, **kwarg)
        return x
    return fn


def join_warper(fsize):
    def fn(x):
        return join_frame(x, fsize)
    return fn


def split_warper(fsize):
    def fn(x):
        return split_frame(x, fsize)
    return fn


_rng_streams = {}


def draw_scalar(generator: torch.Generator, fn):
    """Evaluate `fn()` (a one-element torch.randint / torch.rand call on `generator`) and return its
    Python value.  The reference does this on the current stream, so reading the value back waits for all
    queued compute (merge.py:56-64 boolean-mask indexing, patch.py:62 `if torch.rand(...) > ...`).  The draw
    depends only on the generator state, never on data, so it is issued on a small side stream instead:
    the read-back then synchronises that stream only and the main stream keeps running.  Draw order and
    values are unchanged (Philox offsets are advanced on the host at call time)."""
    if generator.device.type != "cuda":
        return fn().item()
    dev = generator.device
    st = _rng_streams.get(dev)
    if st is None:
        st = _rng_streams[dev] = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(st):
        return fn().item()


def draw_randf(generator: torch.Generator, stride: int, frames: int):
    """The `torch.randint(0, stride, [1])` of vidtome/merge.py:56-57 (which frame of every `stride` is dst).
    Eagerly: the Python int (read back through the side stream of draw_scalar).  While the current stream is being
    captured into a CUDA graph nothing can be read back, so the draw stays on the device as a 1-element int32
    tensor that the kernels dereference (vtm_split_t.randf_dev); each replay then draws a fresh value from the
    generator, which must be registered with the graph.  That needs src / dst counts that do not depend on the
    draw, i.e. frames % stride == 0."""
    def fn():
        return torch.randint(0, stride, torch.Size([1]), generator=generator, device=generator.device)
    if generator.device.type == "cuda" and torch.cuda.is_current_stream_capturing():
        if frames % stride != 0:
            raise RuntimeError(f"CUDA-graph capture needs a frame count divisible by the target stride "
                               f"(got {frames} frames, stride {stride}): token counts would depend on the draw")
        return fn().to(torch.int32)
    return int(draw_scalar(generator, fn))


def draw_coin(generator: torch.Generator, on_device: bool = None):
    """The global stage's `torch.rand(1)` of vidtome/patch.py:62 (which token set is src).  By default (on_device=None)
    the Python float, read back through the side stream of draw_scalar, except while the current stream is being
    captured into a CUDA graph: then the 1-element fp32 CUDA tensor itself, which the kernels dereference
    (vtm_split_t.coin_dev; the generator must be registered with the graph).  on_device=True asks for the tensor
    eagerly too.  Both forms are one draw that advances the generator by the same offset."""
    def fn():
        return torch.rand(1, generator=generator, device=generator.device)
    if on_device is None:
        on_device = generator.device.type == "cuda" and torch.cuda.is_current_stream_capturing()
    if on_device:
        if generator.device.type != "cuda":
            raise RuntimeError("draw_coin: a device-resident coin needs a CUDA generator")
        return fn()
    return float(draw_scalar(generator, fn))


def coin_above(coin: float, global_rand: float) -> bool:
    """`torch.rand(1) > global_rand` of vidtome/patch.py:62 for a coin read back as a Python float: torch compares an
    fp32 tensor with a Python scalar in fp32, so global_rand is rounded to the nearest float first.  A draw equal to
    fp32(global_rand) is then never greater, even where that float lies above global_rand (0.3, 0.6, 0.8, ...)."""
    return bool(np.float32(coin) > np.float32(global_rand))

