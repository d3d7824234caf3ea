"""K0 (normalise + split) and KC (merge gather) outputs, byte for byte, against digests recorded with the previous build
of the row kernels (K0's slow division branch still a loop, which kept each row in local memory as well as registers).

The inputs are seeded CUDA tensors at the level shapes of the SD1.5 headline step (ds1: 65 536 level-0 rows of 320
channels per sample, ds2: 16 384 of 640; level 2 reads the level-0 table through a row map).  They run with and without
the fused LayerNorm, with a row map per sample and one shared map (align_batch), plus the device-count (mode 2) split of
the global stage.  Row scales span fp16's range, so rows whose norm is zero, sub-normal or past fp16's range take the
slow division branch.

    python tests/test_gpu_rows_identity.py     # prints the digests of the library it loads
"""
from __future__ import annotations

import hashlib
import json
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

B, F, STRIDE, RANDF = 2, 16, 4, 1
# (name, level-0 rows per sample, C, level-2 rows per sample, level-2 carried tokens, merged length)
BLOCKS = [("ds1", 65536, 320, 21300, 4916, 10241), ("ds2", 16384, 640, 5325, 1229, 2561)]

EXPECTED = {
    "K0 ds1 L1 noln": "96569543de7bbf4ec41b87d4",
    "K0 ds1 L2 noln": "292eceb150ffe1f459f4b5b4",
    "K0 ds1 L2 noln align": "b8d6a27dcf34d95f2f9cd588",
    "K0 ds1 L1 ln": "a6724f84c432d161a6dd1864",
    "K0 ds1 L2 ln": "00b69b10ec6f6011a4777f4b",
    "K0 ds1 L2 ln align": "e5be355253f11cf1a5f217af",
    "KC ds1 ln": "bcf289cd9daeab2119a0d7bd",
    "KC ds1 noln": "644284c24688ed58a24e9f63",
    "KC ds1 ln align": "d758a4f04db15b0a4ae8ab69",
    "K0 ds1 DC coin 0.75": "868f58b7c97072ad0a6bcf33",
    "K0 ds1 DC coin 0.25": "f1bd87acb93522b419a4b0cf",
    "K0 ds2 L1 noln": "ebbc6f333f0db830d0808b8f",
    "K0 ds2 L2 noln": "4d8346db1c2aae19164eb719",
    "K0 ds2 L2 noln align": "fa478061062be4ad146d6959",
    "K0 ds2 L1 ln": "50a7f68aa15ecd6cd78442c2",
    "K0 ds2 L2 ln": "b77f2cd143bd1f117f41af73",
    "K0 ds2 L2 ln align": "efd483d70082911f16be83fe",
    "KC ds2 ln": "de4748334fa0588e7da9735a",
    "KC ds2 noln": "5801756ab702062580e85888",
    "KC ds2 ln align": "56c9c7472fc5c5628cb280ea",
    "K0 ds2 DC coin 0.75": "d2c6239da03e7638a1386fa5",
    "K0 ds2 DC coin 0.25": "7e8866a79da38462f60ac5a1",
}


def _digest(*ts):
    h = hashlib.sha256()
    for t in ts:
        h.update(t.contiguous().view(-1).view(torch.uint8).cpu().numpy().tobytes())
    return h.hexdigest()[:24]


def _rows(g, n, C):
    """[B, n, C] fp16 with per-row scales from 2^-30 to 2^13 (sub-normal and overflowing norms among them)."""
    x = torch.randn((B, n, C), generator=g, device="cuda")
    e = torch.randint(-30, 14, (B, n, 1), generator=g, device="cuda").float()
    return (x * torch.exp2(e)).half()


def _ln(g, C):
    w = (1 + 0.25 * torch.randn(C, generator=g, device="cuda")).half()
    b = (0.25 * torch.randn(C, generator=g, device="cuda")).half()
    return (w, b, 1e-5)


def digests():
    from vidtome_b200 import ops
    from vidtome_b200._lib import VtmSplit
    out = {}
    g = torch.Generator(device="cuda").manual_seed(20261018)
    for name, N0, C, L2, unm2, M in BLOCKS:
        T = N0 // F
        x = _rows(g, N0, C)
        ln = _ln(g, C)
        mp = torch.stack([torch.randperm(N0, generator=g, device="cuda")[:L2] for _ in range(B)]).int()
        for use_ln in (False, True):
            lnv = ln if use_ln else None
            tag = "ln" if use_ln else "noln"
            sp1 = VtmSplit.local(N0, 0, F, STRIDE, RANDF)
            sp2 = VtmSplit.local(L2, unm2, (L2 - unm2) // T, STRIDE, RANDF)
            out[f"K0 {name} L1 {tag}"] = _digest(*ops.normalize_split(x, None, sp1, lnv))
            out[f"K0 {name} L2 {tag}"] = _digest(*ops.normalize_split(x, mp, sp2, lnv))
            out[f"K0 {name} L2 {tag} align"] = _digest(*ops.normalize_split(x, mp[:1].contiguous(), sp2, lnv))
        mu = torch.stack([torch.randperm(N0, generator=g, device="cuda")[:M] for _ in range(B)]).int()
        out[f"KC {name} ln"] = _digest(ops.gather_rows(x, mu, ln=ln))
        out[f"KC {name} noln"] = _digest(ops.gather_rows(x, mu))
        out[f"KC {name} ln align"] = _digest(ops.gather_rows(x, mu[:1].contiguous(), ln=ln))
        # the global stage's device-count split: [local (M rows) | global (glen of gcap rows)], coin picks the src half
        gcap, glen = M // 2 + 7, M // 2 - 5
        t = _rows(g, M + gcap, C)
        for coin_v in (0.75, 0.25):
            coin = torch.tensor([coin_v], device="cuda")
            sp = VtmSplit.prefix_coin_dev(M, torch.tensor([glen], device="cuda", dtype=torch.int32), gcap, coin, 0.5)
            a, b = ops.normalize_split(t, None, sp)
            ns, nd = (M, glen) if coin_v > 0.5 else (glen, M)
            out[f"K0 {name} DC coin {coin_v}"] = _digest(a[:, :ns], b[:, :nd])
    return out


@pytest.mark.gpu
def test_row_kernel_outputs_match_recorded_digests():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    got = digests()
    assert set(got) == set(EXPECTED)
    diff = {k: (got[k], EXPECTED[k]) for k in got if got[k] != EXPECTED[k]}
    assert not diff, diff


if __name__ == "__main__":
    print(json.dumps(digests(), indent=1))
