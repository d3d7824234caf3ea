"""Chunks of a captured step on concurrent lanes (driver.LANES): the latents stay bit-identical to eager stepping in
every single-graph mode, and the captured graph really is concurrent (its CUDA debug dump, parsed: the same kernels as
the one-stream capture on a strictly shorter longest path, and with local merging no edge between lanes)."""
import re
from collections import defaultdict, deque

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _equal(eager, graph):
    for i, (a, b) in enumerate(zip(eager, graph)):
        assert torch.isfinite(b).all(), i
        assert torch.equal(a, b), f"step {i}: max |diff| = {(a.float() - b.float()).abs().max().item()}"


def _steps(den, x, steps):
    torch.manual_seed(2024)              # the device RNG the blocks fork from, and get_chunks' permutations
    np.random.seed(2024)
    xs = []
    for i in range(steps):
        x = den.step(x, i)
        xs.append(x.clone())
    torch.cuda.synchronize()
    return xs


def _latents(frames, size, seed=5):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn((frames, 4, size, size), generator=g, device="cuda", dtype=torch.float16)


# --------------------------------------------------------------------------- 1. global merging, capture_global
def _global(graph, steps, chunk_ord, frames, size=16, name="tiny"):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton
    torch.manual_seed(77)
    net = make_skeleton(name, device="cuda")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=True, global_merge_ratio=0.8, batch_size=2)
    den = ChunkedDenoiser(net, n_timesteps=50, chunk_size=4, merge_global=True, chunk_ord=chunk_ord,
                          cuda_graph=graph, capture_global=graph, graph_warmup=2)
    return _steps(den, _latents(frames, size), steps), den


@pytest.mark.parametrize("slots", [4, 8])
@pytest.mark.parametrize("chunk_ord", ["seq", "rand", "mix-4"])
def test_capture_global_on_lanes_is_bit_identical_to_eager(slots, chunk_ord):
    from vidtome_b200 import driver
    eager, _ = _global(False, 7, chunk_ord, 4 * slots)
    graph, den = _global(True, 7, chunk_ord, 4 * slots)
    assert den._graph is not None and den._lane_count == driver.LANES
    assert len(den._lanes[torch.device("cuda", torch.cuda.current_device())]) == min(driver.LANES, slots)
    _equal(eager, graph)
    assert not torch.equal(graph[3], graph[4])


def test_capture_global_on_lanes_full_size():
    """BASELINE config 3's shape: the SD1.5 skeleton at 512x512 (latent 64), 32 frames in chunks of 4, global 0.8."""
    eager, _ = _global(False, 4, "mix-4", 32, size=64, name="sd15")
    graph, den = _global(True, 4, "mix-4", 32, size=64, name="sd15")
    assert den._graph is not None and den._lane_count > 1
    _equal(eager, graph)


# --------------------------------------------------------------------------- 2. PnP, both injection boundaries
PNP_STEPS = 8          # pnp_attn_t 0.25, pnp_f_t 0.75: steps 0-1 both injections, 2-5 conv only, 6-7 neither


def _pnp(graph, frames):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton, pnp_attention_modules, pnp_conv_module
    torch.manual_seed(77)
    net = make_skeleton("sd15", device="cuda", pnp_conv=True)
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=True, global_merge_ratio=0.8, global_rand=0.5,
                             batch_size=3, align_batch=True)
    g = torch.Generator(device="cuda").manual_seed(5)
    cond = torch.randn((3, 77, 768), generator=g, device="cuda").half()
    sources = {}

    def source(t):
        if t not in sources:
            gs = torch.Generator(device="cuda").manual_seed(int(t))
            sources[t] = torch.randn((frames, 4, 16, 16), generator=gs, device="cuda").half()
        return sources[t]
    den = ChunkedDenoiser(net, n_timesteps=PNP_STEPS, chunk_size=4, merge_global=True, chunk_ord="mix-4", cond=cond,
                          source_latents=source, pnp_attn_t=0.25, pnp_modules=pnp_attention_modules(net),
                          pnp_f_t=0.75, pnp_conv_modules=[pnp_conv_module(net)], cuda_graph=graph,
                          capture_global=graph, graph_warmup=1)
    keys = []
    x = _latents(frames, 16, seed=6)
    torch.manual_seed(2024)
    np.random.seed(2024)
    xs = []
    for i in range(PNP_STEPS):
        x = den.step(x, i)
        xs.append(x.clone())
        keys.append(den._graph.key if graph and den._graph is not None else None)
    torch.cuda.synchronize()
    return xs, keys, den


@pytest.mark.parametrize("slots", [4, 8])
def test_pnp_capture_global_on_lanes_across_both_injection_boundaries(slots):
    eager, _, _ = _pnp(False, 4 * slots)
    graph, keys, den = _pnp(True, 4 * slots)
    assert den._lane_count > 1
    assert [k[1:] for k in keys[1:]] == [(True, True)] + [(False, True)] * 4 + [(False, False)] * 2, keys
    _equal(eager, graph)


# --------------------------------------------------------------------------- 3. ControlNet patched with include_control
def test_patched_controlnet_capture_global_on_lanes():
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_controlnet, make_skeleton

    class DiffusionPipeline:
        pass

    class StableDiffusionControlNetPipeline(DiffusionPipeline):
        def __init__(self):
            self.unet = make_skeleton("sd15", device="cuda")
            self.controlnet = make_controlnet("sd15", device="cuda")

    def run(graph):
        torch.manual_seed(77)
        pipe = StableDiffusionControlNetPipeline()
        vidtome_b200.apply_patch(pipe, local_merge_ratio=0.9, merge_global=True, global_merge_ratio=0.8,
                                 global_rand=0.5, batch_size=2, include_control=True)
        g = torch.Generator(device="cuda").manual_seed(5)
        cond = torch.randn((2, 77, 768), generator=g, device="cuda").half()
        ctrl = torch.rand((16, 3, 128, 128), generator=g, device="cuda").half()
        den = ChunkedDenoiser(pipe.unet, n_timesteps=50, chunk_size=4, merge_global=True, chunk_ord="mix-4",
                              cond=cond, controlnet=pipe.controlnet, control_images=ctrl, cuda_graph=graph,
                              capture_global=graph, graph_warmup=2)
        xs = _steps(den, _latents(16, 16), 7)
        if graph:
            edges = den._lane_edges(den._lane_streams(torch.device("cuda", torch.cuda.current_device()), 4))
            blocks = [m for m in pipe.controlnet.modules() if type(m).__name__ == "ToMeBlock"]
            assert blocks and all(id(m) in edges.events for m in blocks)
        return xs, den
    eager, _ = run(False)
    graph, den = run(True)
    assert den._lane_count > 1
    _equal(eager, graph)


# --------------------------------------------------------------------------- 4. SD2-depth
def test_depth_capture_global_on_lanes():
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton

    def run(graph):
        torch.manual_seed(77)
        net = make_skeleton("sd21", device="cuda", hot_path_only=False, transformer_io="linear", depth=True)
        vidtome_b200.apply_patch(net, local_merge_ratio=0.9, merge_global=True, global_merge_ratio=0.9,
                                 global_rand=0.5, batch_size=2)
        g = torch.Generator(device="cuda").manual_seed(5)
        cond = torch.randn((2, 77, 1024), generator=g, device="cuda").half()
        gd = torch.Generator(device="cuda").manual_seed(9)
        depth = torch.rand((16, 1, 16, 16), generator=gd, device="cuda") * 2 - 1
        den = ChunkedDenoiser(net, n_timesteps=8, chunk_size=4, merge_global=True, chunk_ord="mix-4", cond=cond,
                              depth=depth, cuda_graph=graph, capture_global=graph, graph_warmup=1)
        return _steps(den, _latents(16, 16), 6), den
    eager, _ = run(False)
    graph, den = run(True)
    assert den._lane_count > 1
    _equal(eager, graph)


# --------------------------------------------------------------------------- 5. local merging, cuda_graph=True
def _local(graph, frames, chunk, steps=6):
    import vidtome_b200
    from vidtome_b200.driver import ChunkedDenoiser
    from vidtome_b200.skeleton import make_skeleton
    torch.manual_seed(77)
    net = make_skeleton("tiny", device="cuda")
    vidtome_b200.apply_patch(net, local_merge_ratio=0.9, batch_size=2)
    den = ChunkedDenoiser(net, n_timesteps=50, chunk_size=chunk, cuda_graph=graph, graph_warmup=2)
    return _steps(den, _latents(frames, 16), steps), den


@pytest.mark.parametrize("chunks", [4, 8])
def test_local_merging_on_lanes_is_bit_identical_to_eager(chunks):
    eager, _ = _local(False, 4 * chunks, 4)
    graph, den = _local(True, 4 * chunks, 4)
    assert den._graph is not None and den._lane_count > 1
    _equal(eager, graph)


def test_one_chunk_captures_on_the_capture_stream():
    graph, den = _local(True, 16, 16, steps=3)
    assert den._graph is not None
    assert den._lanes[torch.device("cuda", torch.cuda.current_device())] == []


# --------------------------------------------------------------------------- 6. the structure of the graph
class Dot:
    """Nodes and edges of a cudaGraphDebugDotPrint dump; a node is a kernel if its label says KERNEL."""

    def __init__(self, text: str):
        self.text = text
        self.succ, self.pred = defaultdict(set), defaultdict(set)
        for a, b in re.findall(r'"([^"]+)"\s*->\s*"([^"]+)"', text):
            self.succ[a].add(b)
            self.pred[b].add(a)
        defs = [(m.start(), m.group(1)) for m in re.finditer(r'^\s*"([^"]+)"\s*\[', text, re.M)]
        self.nodes, self.kernels = set(), set()
        for (pos, name), nxt in zip(defs, defs[1:] + [(len(text), None)]):
            self.nodes.add(name)
            if "KERNEL" in text[pos:nxt[0]]:
                self.kernels.add(name)
        self.nodes |= set(self.succ) | set(self.pred)
        assert self.kernels, "no kernel node in the dump: " + text[:1500]

    def longest_path(self) -> int:
        """Most kernel nodes on one dependency path."""
        indeg = {n: len(self.pred[n]) for n in self.nodes}
        best = {n: 0 for n in self.nodes}
        q = deque(n for n in self.nodes if indeg[n] == 0)
        seen = 0
        while q:
            n = q.popleft()
            seen += 1
            best[n] += n in self.kernels
            for s in self.succ[n]:
                best[s] = max(best[s], best[n])
                indeg[s] -= 1
                if indeg[s] == 0:
                    q.append(s)
        assert seen == len(self.nodes), "the dump has a cycle"
        return max(best.values())

    def _reach(self, start, nbrs):
        out, q = set(), deque([start])
        while q:
            n = q.popleft()
            for m in nbrs[n]:
                if m not in out:
                    out.add(m)
                    q.append(m)
        return out

    def lane_groups(self):
        """Weakly connected groups of nodes once the fork side (ancestors of every sink) and the join side
        (descendants of every root) are set aside: kernel counts per group."""
        roots = [n for n in self.nodes if not self.pred[n]]
        sinks = [n for n in self.nodes if not self.succ[n]]
        shared = set()
        if len(sinks) > 1:
            anc = [self._reach(s, self.pred) for s in sinks]
            shared |= set.intersection(*anc)
        if len(roots) > 1:
            desc = [self._reach(r, self.succ) for r in roots]
            shared |= set.intersection(*desc)
        left, groups = self.nodes - shared, []
        while left:
            seed = left.pop()
            group, q = {seed}, deque([seed])
            while q:
                n = q.popleft()
                for m in (self.succ[n] | self.pred[n]) - shared:
                    if m not in group:
                        group.add(m)
                        q.append(m)
            left -= group
            groups.append(len(group & self.kernels))
        return sorted(groups)


def _dump(monkeypatch, tmp_path, lanes, make, tag):
    """Capture with `lanes` lanes (the driver's LANES, monkeypatched) and parse the graph's debug dump."""
    from vidtome_b200 import driver
    real = torch.cuda.CUDAGraph

    def debug_graph():
        g = real(keep_graph=True)                   # keeps the cudaGraph_t to dump; replay() instantiates it
        g.enable_debug_mode()
        return g
    with monkeypatch.context() as mp:
        mp.setattr(driver, "LANES", lanes)
        mp.setattr(torch.cuda, "CUDAGraph", debug_graph)
        _, den = make()
    assert den._graph is not None and den._lane_count == lanes
    path = str(tmp_path / f"{tag}_{lanes}.dot")
    den._graph.graph.debug_dump(path)
    with open(path) as f:
        return Dot(f.read())


def test_global_capture_is_concurrent(monkeypatch, tmp_path):
    from vidtome_b200 import driver
    make = lambda: _global(True, 3, "mix-4", 32)                      # noqa: E731
    one = _dump(monkeypatch, tmp_path, 1, make, "global")
    many = _dump(monkeypatch, tmp_path, driver.LANES, make, "global")
    assert len(one.kernels) == len(many.kernels)
    assert many.longest_path() < one.longest_path(), (many.longest_path(), one.longest_path())
    assert one.longest_path() == len(one.kernels)                      # one stream: a chain


@pytest.mark.parametrize("chunks", [4, 8])
def test_local_capture_has_no_edge_between_lanes(monkeypatch, tmp_path, chunks):
    from vidtome_b200 import driver
    make = lambda: _local(True, 4 * chunks, 4, steps=3)              # noqa: E731
    one = _dump(monkeypatch, tmp_path, 1, make, f"local{chunks}")
    many = _dump(monkeypatch, tmp_path, driver.LANES, make, f"local{chunks}")
    assert len(one.kernels) == len(many.kernels)
    assert many.longest_path() < one.longest_path()
    n = min(driver.LANES, chunks)
    per_chunk = len(one.kernels) // chunks
    want = sorted(per_chunk * len(range(k, chunks, n)) for k in range(n))
    assert many.lane_groups() == want, (many.lane_groups(), want)
