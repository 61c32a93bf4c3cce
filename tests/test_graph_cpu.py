"""GraphRunner's control flow (eager -> capture -> replay; a refused capture degrades to eager) with torch.cuda mocked out."""
import torch

from parakeet_b200 import graph as G


def test_graph_runner_state_machine(monkeypatch):
    class FakeGraph:
        replays = 0

        def replay(self):
            FakeGraph.replays += 1

    class Ctx:
        def __init__(self, fail):
            self.fail = fail

        def __enter__(self):
            if self.fail:
                raise RuntimeError("capture refused")

        def __exit__(self, *a):
            return False

    fail = {"v": False}
    monkeypatch.setattr(torch.cuda, "synchronize", lambda: None)
    monkeypatch.setattr(torch.cuda, "CUDAGraph", FakeGraph)
    monkeypatch.setattr(torch.cuda, "graph", lambda g: Ctx(fail["v"]))
    r = G.GraphRunner()
    r.enabled = True
    calls = []
    fn = lambda x: (calls.append(1), x * 2)[1]
    x = torch.ones(3)
    a = r.run("k", fn, [x])                       # first sight of the key: eager
    r.run("k", fn, [x])                           # second: capture (fn runs once more under the fake capture) + replay
    r.run("k", fn, [x + 1])                       # third: replay only
    assert len(calls) == 2 and FakeGraph.replays == 2 and torch.equal(a, x * 2) and r.replays == 2
    fail["v"] = True
    for _ in range(3):
        out = r.run("j", fn, [x])
    assert "j" in r._disabled and torch.equal(out, x * 2) and FakeGraph.replays == 2   # refused capture: eager from then on
    r.clear()
    assert not r._graphs and not r._disabled and not r._seen
    r.enabled = False
    assert torch.equal(r.run("k", fn, [x]), x * 2) and not r._seen                     # PK_CUDA_GRAPHS=0: always eager
    off = G.GraphRunner(enabled=False)
    for _ in range(3):
        assert torch.equal(off.run("k", fn, [x]), x * 2)
    assert not off._seen and not off._graphs and off.replays == 0 and FakeGraph.replays == 2


def test_training_steps_graph_switch(monkeypatch):
    """One switch for every training step: use_graphs when given, else PK_TRAIN_GRAPH; PK_CUDA_GRAPHS=0 wins over both."""
    from parakeet_b200.training.flat import StepGraphs, step_graphs
    monkeypatch.delenv("PK_CUDA_GRAPHS", raising=False)
    monkeypatch.delenv("PK_TRAIN_GRAPH", raising=False)
    for make in (step_graphs, StepGraphs):
        assert make(4).enabled and not make(4, use_graphs=False).enabled and make(4).max_graphs == 4
    monkeypatch.setenv("PK_TRAIN_GRAPH", "0")
    for make in (step_graphs, StepGraphs):
        assert not make(4).enabled and make(4, use_graphs=True).enabled
    assert G.GraphRunner().enabled                                                      # the inference graphs do not follow it
    monkeypatch.setenv("PK_CUDA_GRAPHS", "0")
    monkeypatch.setenv("PK_TRAIN_GRAPH", "1")
    for make in (step_graphs, StepGraphs):
        assert not make(4).enabled and not make(4, use_graphs=True).enabled


def test_step_graphs_file_planes_and_graph_under_one_key(monkeypatch):
    """training/flat.py StepGraphs: running a key makes its zero planes current, and evicting the planes of a key drops the graph
    of the same key (its kernels hold the planes' addresses).  With a bound of 2 after A, A, B, B, C, A's planes and A's graph are
    both gone; a replay makes its key the most recent.  GE2E used to file its planes under (B, T) and its graph under (B, T, n_mels),
    so the eviction never found the graph."""
    from parakeet_b200.training.flat import StepGraphs

    class FakeGraph:
        def replay(self):
            pass

    class Ctx:
        def __enter__(self):
            pass

        def __exit__(self, *a):
            return False

    monkeypatch.setattr(torch.cuda, "synchronize", lambda: None)
    monkeypatch.setattr(torch.cuda, "CUDAGraph", FakeGraph)
    monkeypatch.setattr(torch.cuda, "graph", lambda g: Ctx())
    sg = StepGraphs(2, use_graphs=True)
    sg.enabled = True
    planes = {}

    def fn(x):                         # a step body: takes operand planes of the current key
        planes.setdefault(sg.planes._cur, sg.planes.get("xt", (4, 64), "cpu"))
        return x * 2

    A, B, C = (20, 50, 40), (20, 31, 40), (20, 12, 40)        # GE2E's key: the specs' shape
    x = torch.ones(3)
    for k in (A, A, B, B, C):                                  # eager, capture; eager, capture; eager
        sg.run(k, fn, [x])
    assert A not in sg.planes._geoms and A not in sg._graphs and A not in sg._seen
    assert B in sg._graphs and list(sg.planes._geoms) == [B, C]
    assert sg.planes.get("xt", (4, 64), "cpu") is planes[C]
    sg.run(C, fn, [x])                                         # capture C
    sg.run(B, fn, [x])                                         # replay B: the most recent now
    replays = sg.replays
    sg.run(A, fn, [x])                                         # A again: C goes, with its graph; B stays captured
    assert list(sg.planes._geoms) == [B, A] and C not in sg._graphs and B in sg._graphs
    sg.run(B, fn, [x])
    assert sg.replays == replays + 1 and sg.planes.get("xt", (4, 64), "cpu") is planes[B]
    assert torch.equal(sg.run(C, fn, [x], graph=False), x * 2) and C not in sg._seen      # eager: planes only, no graph
    assert list(sg.planes._geoms) == [B, C] and A not in sg._graphs


def test_zero_planes_lru_is_tied_to_the_graphs():
    """training/wgrad.py ZeroPlanes: persistent zero-initialised operand planes are filed per batch geometry, bounded (LRU), and
    evicting a geometry tells the owner to drop the CUDA graph captured for it (its buffer addresses are baked into the graph)."""
    import torch
    from parakeet_b200.graph import GraphRunner
    from parakeet_b200.training.wgrad import ZeroPlanes
    runner = GraphRunner(max_graphs=8)
    dropped = []

    def on_evict(key):
        dropped.append(key)
        runner.drop(key)

    zp = ZeroPlanes(max_geoms=2, on_evict=on_evict)
    zp.begin("a")
    pa = zp.get(("xt", 2, 10), (4, 64), "cpu")
    assert pa.hi.shape == (4, 64) and not pa.hi.any() and not pa.lo.any()
    assert zp.get(("xt", 2, 10), (4, 64), "cpu") is pa                    # same key, same geometry: the same buffer
    assert zp.get(("dyt", 2, 10), (4, 64), "cpu") is not pa               # the role keeps live operands apart
    pa.hi.fill_(1)                                                         # "valid region" written by a transpose
    zp.begin("b")
    assert zp.get(("xt", 2, 10), (4, 64), "cpu") is not pa                # other geometry: its own planes (its own padding)
    zp.touch("a")                                                          # a graph replay of "a" keeps it recent
    runner._seen.add("b")
    zp.begin("c")                                                          # bound 2: "b" (least recently used) goes, with its graph
    assert dropped == ["b"] and "b" not in runner._seen and len(zp) == 2
    zp.begin("a")
    assert zp.get(("xt", 2, 10), (4, 64), "cpu") is pa                    # "a" survived
    zp.begin("b")                                                          # back again: fresh zeros
    assert dropped == ["b", "c"] and not zp.get(("xt", 2, 10), (4, 64), "cpu").hi.any()
