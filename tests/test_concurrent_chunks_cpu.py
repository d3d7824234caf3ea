"""The lane capture of a chunked step without a GPU: which lane each chunk runs on (driver.run_on_lanes), and the
recurrence edge between chunks (patch.LaneEdges), with stand-in streams and events."""
import contextlib
from types import SimpleNamespace

import pytest
import torch

from vidtome_b200 import driver, patch


class Log(list):
    pass


class Stream:
    def __init__(self, name, log):
        self.name, self.log = name, log

    def wait_stream(self, other):
        self.log.append(("wait_stream", self.name, other.name))

    def wait_event(self, ev):
        self.log.append(("wait_event", self.name, ev.name))


class Event:
    def __init__(self, log, name):
        self.log, self.name = log, name

    def record(self, stream):
        self.log.append(("record", stream.name, self.name))


class Tokens:
    def __init__(self, name, log):
        self.name, self.log = name, log

    def record_stream(self, stream):
        self.log.append(("record_stream", stream.name, self.name))


@pytest.fixture
def lanes(monkeypatch):
    """Stand-in streams: `current` tracks torch.cuda.stream(...) as the CUDA context manager would."""
    log = Log()
    main = Stream("main", log)
    state = {"current": main}

    @contextlib.contextmanager
    def use(stream):
        prev, state["current"] = state["current"], stream
        try:
            yield
        finally:
            state["current"] = prev
    monkeypatch.setattr(torch.cuda, "stream", use)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: state["current"])
    return log, main, state


@pytest.mark.parametrize("n,k", [(4, 2), (4, 3), (8, 3), (8, 4), (3, 4)])
def test_chunk_k_runs_on_lane_k_mod_lanes_between_fork_and_join(lanes, n, k):
    log, main, state = lanes
    streams = [Stream(f"lane{i}", log) for i in range(k)]
    seen = []
    driver.run_on_lanes(n, streams, lambda c: seen.append((c, state["current"].name)))
    assert seen == [(c, f"lane{c % k}") for c in range(n)]
    assert state["current"] is main
    forks = [("wait_stream", s.name, "main") for s in streams]
    joins = [("wait_stream", "main", s.name) for s in streams]
    assert log == forks + joins                      # every fork before the first chunk, every join after the last


def test_one_lane_or_none_runs_on_the_current_stream(lanes):
    log, main, state = lanes
    for streams in ([], [Stream("lane0", log)]):
        seen = []
        driver.run_on_lanes(3, streams, lambda c: seen.append(state["current"].name))
        assert seen == ["main"] * 3
    assert log == []                                 # no fork, no join: the graph of one stream


def test_lanes_are_joined_and_edges_removed_when_a_chunk_raises(lanes):
    log, main, state = lanes
    streams = [Stream(f"lane{i}", log) for i in range(2)]
    edges = patch.LaneEdges([], event=lambda: None, current_stream=lambda: state["current"])

    def body(c):
        assert patch.active_lane_edges() is edges
        if c == 1:
            raise ValueError("boom")
    with pytest.raises(ValueError, match="boom"):
        driver.run_on_lanes(3, streams, body, edges)
    assert log[-2:] == [("wait_stream", "main", "lane0"), ("wait_stream", "main", "lane1")]
    assert patch.active_lane_edges() is None and state["current"] is main


def test_edges_are_inactive_outside_a_lane_capture():
    assert patch.active_lane_edges() is None
    edges = patch.LaneEdges([], event=lambda: None, current_stream=lambda: None)
    with patch.lane_edges(edges):
        assert patch.active_lane_edges() is edges
        with pytest.raises(RuntimeError, match="already"):
            with patch.lane_edges(patch.LaneEdges([], event=lambda: None, current_stream=lambda: None)):
                pass
    assert patch.active_lane_edges() is None
    with patch.lane_edges(None):
        assert patch.active_lane_edges() is None


def test_one_event_per_merged_block():
    log = Log()
    made = []

    def event():
        made.append(Event(log, f"ev{len(made)}"))
        return made[-1]
    blocks = [SimpleNamespace(name=f"b{i}") for i in range(5)]
    edges = patch.LaneEdges(blocks + blocks[:2], event=event, current_stream=lambda: None)
    assert len(made) == 5 and len(edges.events) == 5
    assert {id(b) for b in blocks} == set(edges.events)
    with pytest.raises(RuntimeError, match="recurrence event"):
        edges.record(SimpleNamespace())
    with pytest.raises(RuntimeError, match="recurrence event"):
        edges.wait(SimpleNamespace(), Tokens("t", log))


def test_read_waits_for_the_previous_store_and_holds_the_tokens_for_its_stream():
    """Three chunks on lanes a, b, c through two blocks, in the order the global stage issues the calls: block l of
    chunk k waits on the event chunk k-1 recorded for block l, marks the tokens it reads as used by its own stream, and
    records after its store.  The first chunk has no predecessor: it only records."""
    log = Log()
    cur = {"s": None}
    blocks = [SimpleNamespace(name="b0"), SimpleNamespace(name="b1")]
    evs = iter(["ev_b0", "ev_b1"])
    edges = patch.LaneEdges(blocks, event=lambda: Event(log, next(evs)), current_stream=lambda: cur["s"])
    for k, lane in enumerate("abc"):
        cur["s"] = Stream(lane, log)
        for b in blocks:
            if k:                                    # patch.py:60: global tokens exist from the previous chunk
                edges.wait(b, Tokens(f"g_{b.name}_{k - 1}", log))
            edges.record(b)                          # after global_tokens <- u(merged) (or the first chunk's copy)
    assert log == [
        ("record", "a", "ev_b0"), ("record", "a", "ev_b1"),
        ("wait_event", "b", "ev_b0"), ("record_stream", "b", "g_b0_0"), ("record", "b", "ev_b0"),
        ("wait_event", "b", "ev_b1"), ("record_stream", "b", "g_b1_0"), ("record", "b", "ev_b1"),
        ("wait_event", "c", "ev_b0"), ("record_stream", "c", "g_b0_1"), ("record", "c", "ev_b0"),
        ("wait_event", "c", "ev_b1"), ("record_stream", "c", "g_b1_1"), ("record", "c", "ev_b1")]


def test_a_read_before_any_store_does_not_wait():
    log = Log()
    b = SimpleNamespace()
    edges = patch.LaneEdges([b], event=lambda: Event(log, "ev"), current_stream=lambda: Stream("a", log))
    edges.wait(b, Tokens("g", log))
    assert log == [("record_stream", "a", "g")]


def test_lanes_are_a_small_fixed_count():
    assert isinstance(driver.LANES, int) and 2 <= driver.LANES <= 4


def _bare_driver(**kw):
    den = driver.ChunkedDenoiser.__new__(driver.ChunkedDenoiser)
    den.shard, den._eager_steps, den._lane_count, den._lanes = False, 2, 3, {}
    den.__dict__.update(kw)
    return den


def test_lane_count_follows_the_chunks_and_stays_one_without_a_warm_up_or_with_sharding(monkeypatch):
    made = []
    monkeypatch.setattr(torch.cuda, "Stream", lambda device: made.append(device) or object())
    den = _bare_driver()
    assert len(den._lane_streams("dev", 8)) == 3 and len(made) == 3
    assert len(den._lane_streams("dev", 2)) == 2 and len(made) == 3        # made once per driver and device
    assert den._lane_streams("dev", 1) == []
    assert _bare_driver(shard=True)._lane_streams("dev", 8) == []
    assert _bare_driver(_eager_steps=0)._lane_streams("dev", 8) == []
    assert _bare_driver(_lane_count=1)._lane_streams("dev", 8) == []
    assert len(made) == 3


def test_lanes_are_dropped_when_single_launch_sorts_could_not_all_be_resident(monkeypatch):
    from vidtome_b200 import ops
    monkeypatch.setattr(ops, "sort_co_resident", lambda device: 264)
    den = _bare_driver()
    three = [object()] * 3
    assert den._lanes_fit(three, [88, 12, 300], None)       # 300 CTAs: the multi-launch sort, no barrier
    assert not den._lanes_fit(three, [89], None)
    assert den._lanes_fit([], [264], None)
    assert den._lanes_fit(three, [], None)
    assert ops.sort_ctas(3, 12288) == 36 and ops.sort_ctas(1, 1) == 1
