"""Which attention modules the library takes, as a function of `attention.MAX_HEAD_DIM` (CPU only: the eligibility
tests read shapes, types and flags, never the device)."""
import pytest
import torch

from vidtome_b200 import attention, patch
from vidtome_b200.skeleton import Attention


@pytest.fixture
def limit():
    saved = attention.MAX_HEAD_DIM
    yield
    attention.MAX_HEAD_DIM = saved


def _self(d, heads=8):
    return Attention(d * heads, heads, d)


WIDE = (136, 144, 152, 160)


def test_default_limit_is_128():
    assert attention.MAX_HEAD_DIM == 128
    assert attention.max_head_dim() == 128


def test_wide_heads_not_eligible_at_default(limit):
    for d in WIDE + (168,):
        assert not patch._plain_attention_module(_self(d)), d
    for d in (40, 80, 128):
        assert patch._plain_attention_module(_self(d)), d


def test_wide_heads_eligible_at_160(limit):
    attention.MAX_HEAD_DIM = 160
    for d in WIDE + (40, 80, 128):
        assert patch._plain_attention_module(_self(d)), d
    assert not patch._plain_attention_module(_self(168))
    assert not patch._plain_attention_module(_self(176))


def test_intermediate_limit(limit):
    attention.MAX_HEAD_DIM = 144
    assert patch._plain_attention_module(_self(144))
    assert not patch._plain_attention_module(_self(152))


def _cross(d, heads=8, cctx=768):
    return Attention(d * heads, heads, d, cross_attention_dim=cctx).half()


def test_cross_attention_limit(limit, monkeypatch):
    # cross_attention_eligible requires CUDA weights; pretend they are, since only the head_dim rule is under test
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    ctx = torch.zeros((2, 77, 768), dtype=torch.float16)
    for d in WIDE:
        assert not attention.cross_attention_eligible(_cross(d), ctx), d
    assert attention.cross_attention_eligible(_cross(128), ctx)
    attention.MAX_HEAD_DIM = 160
    for d in WIDE:
        assert attention.cross_attention_eligible(_cross(d), ctx), d
    assert not attention.cross_attention_eligible(_cross(168), ctx)


@pytest.mark.parametrize("bad", (168, 256, 132, 100, 0, -8, 8.0, "160", None, True))
def test_bad_limits_raise(limit, bad):
    attention.MAX_HEAD_DIM = bad
    with pytest.raises(ValueError, match="MAX_HEAD_DIM"):
        patch._plain_attention_module(_self(40))
    with pytest.raises(ValueError, match="MAX_HEAD_DIM"):
        attention.max_head_dim()
