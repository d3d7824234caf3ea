"""Chunk-per-GPU sharding and the global-token exchange (SURVEY.md §8e).

One process per GPU, `torch.distributed` for the plumbing (NCCL over NVLink on the GPU box, gloo in the CPU
tests).  Two cases:

* `merge_global=False` — frame chunks of one denoising step are independent (generate.py:216-219): each rank
  takes its chunks (`shard_chunks`), weights are replicated, NOTHING crosses GPUs in the data path.  Every rank must
  hold the same generator state so that the per-block random target frames agree (`seed_all_ranks`).

* `merge_global=True` — in the reference the global token set is a sequential recurrence over chunks
  (patch.py:59-82; chunk k's block l sees what chunk k-1's block l left in `module.global_tokens`).  Sharded one
  chunk per GPU, the exchange is ONE all-gather of the local merged tokens per merged block
  (`exchange_global_tokens`): rank k then matches against the local tokens of rank (k-1) mod G.  This is the
  north-star variant, a semantic variant of the recurrence (it reproduces one step of it with "previous chunk's
  local tokens" in place of the running set); parity is defined against the reference's own `_2s` matcher fed
  the same global tokens (the attribute is public, patch.py:60).

DDIM inversion and reconstruction (driver.ChunkedInverter(shard=True)) shard the frame batches (`shard_batches`):
nothing crosses GPUs during the steps, and one all-gather at the end (`gather_batches`) gives every rank all frames.
Generation of K edits (driver.ChunkedDenoiser(cond=[K, S, 77, D], shard=True), K > 1) shards the edits the same way
(`shard_edits`, `gather_edits`): every rank makes the draws of the whole job, so each edit is what the unsharded run
computes for it, with the reference's own global-token recurrence.  `check_ranks_agree` verifies up front that the ranks
would draw alike.
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist


def initialized() -> bool:
    return dist.is_available() and dist.is_initialized()


def world() -> int:
    return dist.get_world_size() if initialized() else 1


def rank() -> int:
    return dist.get_rank() if initialized() else 0


def shard_chunks(chunks: Sequence, rank_: Optional[int] = None, world_: Optional[int] = None) -> List:
    """Round-robin assignment of a step's chunk list to ranks (chunk i -> rank i % world).

    Contract for the collective exchange modes (`patch.GLOBAL_EXCHANGE` = "allgather" / "p2p"): every merged block
    forward issues one collective (or one symmetric-memory barrier), so EVERY rank must run the same number of UNet
    forwards per step — `len(chunks)` must be a multiple of the world size.  `check_step_lockstep` verifies that
    (and whether the chunks are equally long, which the fused p2p exchange additionally needs) once per step; the
    driver calls it before the first forward of the step."""
    r = rank() if rank_ is None else rank_
    w = world() if world_ is None else world_
    return [c for i, c in enumerate(chunks) if i % w == r]


def shard_batches(flen: int, batch_size: int, rank_: Optional[int] = None,
                  world_: Optional[int] = None) -> List[Tuple[int, int]]:
    """The frame ranges [lo, hi) of the inversion batches this rank runs: the batches of `batch_size` frames of the
    unsharded run (the last one may be ragged, invert.py:124-129), batch k -> rank k % world.  Batch shapes do not
    change, so every frame is computed exactly as without sharding.  A rank may get no batch (world > batch count)."""
    r = rank() if rank_ is None else rank_
    w = world() if world_ is None else world_
    return [(lo, min(lo + batch_size, flen)) for k, lo in enumerate(range(0, flen, batch_size)) if k % w == r]


def gather_batches(local: torch.Tensor, flen: int, batch_size: int, frame_dim: int = 0, group=None) -> torch.Tensor:
    """Assemble every rank's `local` frames (its shard_batches, concatenated in order along `frame_dim`) into the
    full [.., flen, ..] tensor, in frame order, on every rank: one all-gather of equal-size slabs, each padded to
    ceil(n_batches / world) batches, then each rank's batches put back at their frame ranges.  Without sharding
    (world 1) `local` is returned as it is."""
    w = world()
    if w == 1:
        return local
    n_batches = -(-flen // batch_size)
    slab = -(-n_batches // w) * batch_size
    shape = list(local.shape)
    shape[frame_dim] = slab
    padded = local.new_zeros(shape)
    padded.narrow(frame_dim, 0, local.shape[frame_dim]).copy_(local)
    out = torch.empty((w * shape[0],) + tuple(shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, padded, group=group)                 # rank-major concatenation
    out = out.view([w] + shape)
    shape[frame_dim] = flen
    full = local.new_empty(shape)
    for r in range(w):
        for j, (lo, hi) in enumerate(shard_batches(flen, batch_size, r, w)):
            full.narrow(frame_dim, lo, hi - lo).copy_(out[r].narrow(frame_dim, j * batch_size, hi - lo))
    return full


def shard_edits(K: int, rank_: Optional[int] = None, world_: Optional[int] = None) -> List[int]:
    """The edits of a K-edit generation this rank runs: k with k % world == rank (the batches of one edit each of
    shard_batches)."""
    return [lo for lo, _ in shard_batches(K, 1, rank_, world_)]


def gather_edits(local: torch.Tensor, K: int, group=None) -> torch.Tensor:
    """Every rank's edits `local` [K_r, flen, ...] (its shard_edits, in order) as the full [K, flen, ...] in edit
    order, on every rank: one all-gather of slabs padded to ceil(K / world) edits (gather_batches with batches of one
    edit).  Without sharding (world 1) `local` is returned as it is."""
    return gather_batches(local, K, 1, 0, group)


def check_ranks_agree(entry: Dict[str, Any], group=None) -> None:
    """Collective check before a job whose ranks must make the same draws: all-gathers every rank's `entry` (the same
    keys on every rank) and raises ValueError on ALL ranks, naming the keys, when any value differs between ranks, so
    that no rank is left waiting in a later collective."""
    w = world()
    if w == 1:
        return
    everyone = [None] * w
    dist.all_gather_object(everyone, entry, group=group)
    differ = [k for k in everyone[0] if any(e.get(k) != everyone[0][k] for e in everyone)]
    if differ:
        raise ValueError("vidtome_b200.dist: the ranks disagree on " + ", ".join(differ) + ": " +
                         "; ".join(f"rank {r}: " + ", ".join(f"{k}={e.get(k)!r}" for k in differ)
                                   for r, e in enumerate(everyone)))


def check_step_lockstep(local_chunk_lens: Sequence[int], group=None) -> bool:
    """Collective sanity check, once per denoising step, before any block-level exchange: all-gathers every
    rank's list of chunk lengths (frames).  Raises on ALL ranks (so nobody is left waiting in a collective) when
    the ranks would run different numbers of UNet forwards — e.g. the reference's random first-chunk length
    (generate.py:176-178) changed the chunk count so that it no longer divides by the world size.  Returns True
    when all chunks of all ranks have the same length (token counts then agree at every block: the fused
    peer-to-peer exchange is usable), False when they are ragged (only the padded all-gather is)."""
    w = world()
    lens = [int(v) for v in local_chunk_lens]
    if w == 1:
        return len(set(lens)) <= 1
    everyone = [None] * w
    dist.all_gather_object(everyone, lens, group=group)
    counts = [len(v) for v in everyone]
    if len(set(counts)) != 1:
        raise RuntimeError(
            f"vidtome_b200.dist: ranks would run different numbers of chunks this step ({counts}); the global-token "
            "exchange issues one collective per merged block and needs lock-step ranks. Use a chunk count that is a "
            "multiple of the world size (pad with a repeated chunk) or patch.GLOBAL_EXCHANGE = 'recurrence'.")
    return len({n for v in everyone for n in v}) <= 1


def seed_all_ranks(seed: int) -> None:
    """Same default-RNG state on every rank: the per-block generators are forked from it at first forward
    (patch.py:219-226), so all ranks then draw identical random target frames."""
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)


def all_gather_tokens(local: torch.Tensor, group=None) -> List[torch.Tensor]:
    """All-gather of `[B, L_k, C]` token sets whose length L_k may differ per rank (ragged first chunk,
    generate.py:176-178).  One small all-gather of the lengths, one padded all-gather of the tokens."""
    w = world()
    if w == 1:
        return [local]
    B, L, C = local.shape
    lens = torch.tensor([L], device=local.device, dtype=torch.int64)
    all_lens = [torch.zeros_like(lens) for _ in range(w)]
    dist.all_gather(all_lens, lens, group=group)
    all_lens = [int(t.item()) for t in all_lens]
    Lmax = max(all_lens)
    padded = local if L == Lmax else torch.cat([local, local.new_zeros((B, Lmax - L, C))], dim=1)
    out = torch.empty((w * B, Lmax, C), dtype=local.dtype, device=local.device)   # rank-major concatenation
    dist.all_gather_into_tensor(out, padded.contiguous(), group=group)
    out = out.view(w, B, Lmax, C)
    return [out[k, :, : all_lens[k]] for k in range(w)]


def exchange_global_tokens(local_tokens: torch.Tensor, group=None) -> Optional[torch.Tensor]:
    """The single collective of the global-merge path: all-gather the local merged tokens of this block and
    return the set this rank matches against — the tokens of rank (k-1) mod G (None when running alone)."""
    w = world()
    if w == 1:
        return None
    gathered = all_gather_tokens(local_tokens, group=group)
    return gathered[(rank() - 1) % w].contiguous()


# ------------------------------------------------------------------ exchange fused into the producing kernel
class PeerExchange:
    """Global-token exchange without a collective pass: every rank owns a symmetric buffer `[2, world, B, L, C]`
    (torch symmetric memory: peer-mapped over NVLink), and the KC kernel that creates a rank's merged tokens stores
    each row into slot `rank` of EVERY rank's buffer (vtm_gather_rows_peers).  One barrier later all slots are
    readable locally.  Two buffers alternate so that a rank may already write block l+1 while a peer still reads
    block l (a rank can only reach its second-next write after passing the barrier in between, which every peer
    enters after its reads of the older buffer are enqueued).

    Same token length L on every rank is part of the contract (fixed chunking); it is verified once per shape."""

    _cache = {}

    def __init__(self, B: int, L: int, C: int, device: torch.device, group=None):
        import torch.distributed._symmetric_memory as symm
        self.group = group if group is not None else dist.group.WORLD
        self.w, self.r = dist.get_world_size(self.group), dist.get_rank(self.group)
        if self.w - 1 > 8:
            raise RuntimeError("PeerExchange: at most 9 ranks (8 peer destinations per store)")
        lens = [None] * self.w
        dist.all_gather_object(lens, (B, L, C), group=self.group)
        if any(t != (B, L, C) for t in lens):
            raise RuntimeError(f"PeerExchange needs identical token shapes on every rank, got {lens}")
        self.shape = (B, L, C)
        self.buf = symm.empty((2, self.w, B, L, C), dtype=torch.float16, device=device)
        self.hdl = symm.rendezvous(self.buf, self.group)
        self.phase = 0
        self.slot_elems = B * L * C

    @classmethod
    def get(cls, B: int, L: int, C: int, device: torch.device, group=None) -> "PeerExchange":
        key = (B, L, C, device.index, id(group))
        ex = cls._cache.get(key)
        if ex is None:
            ex = cls._cache[key] = cls(B, L, C, device, group)
        return ex

    def produce(self, table: torch.Tensor, mu: torch.Tensor, ln=None, everyone: bool = False):
        """Run KC for this rank's tokens into slot `rank` of the consumer's buffer — rank k+1, the only rank that matches
        against them (DESIGN §8) — or, with `everyone`, of every rank's buffer (the all-gather semantics: 7x the NVLink
        bytes on 8 GPUs for data nobody reads).  Returns (local tokens, tokens of rank-1)."""
        from . import ops
        ph = self.phase
        self.phase ^= 1
        mine = self.buf[ph, self.r]
        off = ((ph * self.w + self.r) * self.slot_elems) * 2                  # bytes from a buffer's base
        targets = [p for p in range(self.w) if p != self.r] if everyone else [(self.r + 1) % self.w]
        peers = [int(self.hdl.buffer_ptrs[p]) + off for p in targets if p != self.r]
        ops.gather_rows_peers(table, mu, mine, peers, ln=ln)
        self.hdl.barrier(channel=ph)            # all ranks' stores of this block have landed
        return mine, self.buf[ph, (self.r - 1) % self.w]


def exchange_fused(table: torch.Tensor, mu: torch.Tensor, ln=None, group=None, everyone: bool = False):
    """KC + exchange in one kernel (`patch.GLOBAL_EXCHANGE = "p2p"` / `"p2p_all"`): (local merged tokens, tokens of rank k-1)."""
    B, L, C = table.shape[0], mu.shape[1], table.shape[2]
    ex = PeerExchange.get(B, L, C, table.device, group)
    return ex.produce(table, mu, ln=ln, everyone=everyone)

