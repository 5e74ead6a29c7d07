"""CPU tests of the engines' cache and capture plumbing: `BoundedCache`'s bound, eviction order and seen-shape
`touch`, and `capture_graphs`' keep-alive registry (CUDA's stream and graph calls replaced by recording fakes)."""
import contextlib
import gc

import pytest
import torch

from simple_tip_b200 import engine as E


def test_bounded_cache_keeps_its_capacity_and_drops_the_oldest_first():
    cache = E.BoundedCache(3)
    made = []

    def make(k):
        made.append(k)
        return k * 10

    for k in (1, 2, 3):
        assert cache.get_or_make(k, lambda: make(k)) == k * 10
    assert cache.get_or_make(1, lambda: make(-1)) == 10 and made == [1, 2, 3]      # a hit makes nothing
    assert cache.get_or_make(4, lambda: make(4)) == 40
    assert list(cache) == [2, 3, 4]                                                   # a hit does not refresh 1
    cache.get_or_make(5, lambda: make(5))
    assert list(cache) == [3, 4, 5] and len(cache) == cache.capacity
    assert isinstance(cache, dict) and dict(cache.items()) == {3: 30, 4: 40, 5: 50}
    cache.clear()
    assert cache.get_or_make(3, lambda: make(3)) == 30 and made == [1, 2, 3, 4, 5, 3]


def test_bounded_cache_touch_reports_first_and_later_sightings():
    seen = E.BoundedCache(2)
    assert [seen.touch(k) for k in ("a", "a", "b", "a", "c")] == [False, True, False, True, False]
    assert list(seen) == ["b", "c"]                      # "a" was the oldest key when "c" arrived
    assert seen.touch("a") is False and list(seen) == ["c", "a"]


class _FakeGraph:
    def __init__(self):
        self.replays = 0

    def replay(self):
        self.replays += 1


def _fake_cuda(monkeypatch, log):
    """torch.cuda's stream and graph entry points as recorders, so the helper's control flow runs without a GPU."""
    class Stream:
        def __init__(self, device=None):
            pass

        def wait_stream(self, other):
            pass

    @contextlib.contextmanager
    def graph(g, capture_error_mode=None):
        assert capture_error_mode == "thread_local" and not gc.isenabled()
        log.append("capture-begin")
        yield
        log.append("capture-end")

    monkeypatch.setattr(torch.cuda, "Stream", Stream)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda: Stream())
    monkeypatch.setattr(torch.cuda, "synchronize", lambda: log.append("sync"))
    monkeypatch.setattr(torch.cuda, "CUDAGraph", _FakeGraph)
    monkeypatch.setattr(torch.cuda, "graph", graph)


def test_keep_for_capture_collects_only_inside_a_capture(monkeypatch):
    log = []
    _fake_cuda(monkeypatch, log)
    a, b, c, d = (torch.zeros(1) for _ in range(4))

    def seg(name, *tensors):
        def fn():
            log.append(name)
            E.keep_for_capture(*tensors, None)
        return fn

    E.keep_for_capture(a)                                # outside any capture: a no-op
    exch = seg("exch", c)
    segments = [(seg("a", a), True), (exch, False), (seg("b", b, d), True)]
    steps, graphs, keep = E.capture_graphs(segments, torch.device("cpu"))
    # every segment once eagerly, then the capturable ones captured and the others run eagerly again
    assert log == ["a", "exch", "b", "sync", "capture-begin", "a", "capture-end", "exch",
                   "capture-begin", "b", "capture-end"]
    assert [id(t) for t in keep] == [id(a), id(b), id(d)]        # the warm-up and the eager segment add nothing
    assert len(graphs) == 2 and steps[1] is exch
    steps[0]()
    steps[2]()
    assert [g.replays for g in graphs] == [1, 1]
    E.keep_for_capture(c)                                # the capture is over: nothing more is collected
    assert len(keep) == 3 and gc.isenabled()


def test_capture_graphs_leaves_no_registry_behind_after_a_failed_capture(monkeypatch):
    _fake_cuda(monkeypatch, [])
    calls = []

    def body():
        calls.append(1)
        if len(calls) == 2:
            raise RuntimeError("capture failed")

    with pytest.raises(RuntimeError, match="capture failed"):
        E.capture_graphs([(body, True)], torch.device("cpu"))
    assert E._capture_keep is None and gc.isenabled()
