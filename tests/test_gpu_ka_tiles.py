"""KA (similarity + arg-max) at the shapes its tiling makes special: 256-wide dst tiles with every kind of ragged
last tile, more work items than CTAs (the src block resident in shared memory is reloaded), and channel counts whose
src block does not fit next to the dst ring (streamed src chunks).  Bit exact against the numpy oracle on
exact-arithmetic tokens.  Needs an H100 (sm_90a)."""
import numpy as np
import pytest
import torch

import vidtome_oracle as O

pytestmark = pytest.mark.gpu


def _exact_tokens(rng, shape, nnz=64, val=0.125):
    """Rows with exactly `nnz` entries of +-val: every score is an exact multiple of val^2 in any summation order."""
    B, N, C = shape
    x = np.zeros(shape, dtype=np.float16)
    for b in range(B):
        for i in range(N):
            cols = rng.choice(C, size=nnz, replace=False)
            x[b, i, cols] = rng.choice([-val, val], size=nnz)
    return x


@pytest.mark.parametrize("B,Ns,Nd,C,align", [
    (2, 300, 868, 320, False),     # Nd % 256 = 100: last dst tile at most half full
    (2, 300, 712, 320, True),      # Nd % 256 = 200: last dst tile more than half full
    (1, 257, 200, 320, False),     # Nd < 256: one partial dst tile
    (2, 10240, 868, 320, False),   # 160 work items for at most 132 CTAs: src blocks are reloaded
    (2, 10240, 712, 320, True),
    (2, 300, 712, 640, False),     # C = 640: src chunks streamed through the ring
    (2, 300, 868, 640, True),
    (2, 260, 868, 1280, False),    # C = 1280: streamed
    (1, 129, 300, 1280, True),
])
def test_sim_argmax_tiles_bit_exact_on_exact_inputs(B, Ns, Nd, C, align):
    from vidtome_b200 import ops
    rng = np.random.default_rng(B * 100003 + Ns * 31 + Nd + C)
    nnz = min(64, C // 2)
    a = _exact_tokens(rng, (B, Ns, C), nnz=nnz)
    b = _exact_tokens(rng, (B, Nd, C), nnz=nnz)
    s = O.scores_matmul(a, b)
    if align:
        s = np.concatenate([s[i] for i in range(s.shape[0])], axis=-1)[None]
    idx = s.argmax(-1)
    mx = np.take_along_axis(s, idx[..., None], -1)[..., 0]
    keys = ops.sim_argmax(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda(), align)
    score, arg = ops.keys_to_score_arg(keys)
    np.testing.assert_array_equal(score.cpu().numpy().view(np.uint16), mx.view(np.uint16))
    np.testing.assert_array_equal(arg.cpu().numpy(), idx)
