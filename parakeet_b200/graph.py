"""CUDA-graph replay for the launch-bound inference paths (FastSpeech2: ~120 launches of 10-100 us; WaveFlow: 5 040
launches per call).  The reference has no counterpart (Paddle dygraph launches op by op); SURVEY 8(d) asks for CUDA
events around the captured graph.

`GraphRunner.run(key, fn, inputs)` runs `fn(*inputs)` eagerly the first time a key is seen (that call is also the
warm-up that packs weights and sets kernel attributes), captures it into a CUDA graph the second time, and replays the
graph afterwards: inputs are copied into the graph's static input tensors, outputs are the graph's static output tensors
(valid until the next replay of the same key - callers clone what they hand out).  `fn` must not synchronise with the
host.  `enabled=False`, or PK_CUDA_GRAPHS=0 for every runner, runs everything eagerly.
"""
import os

import torch


def _tensors(obj):
    if isinstance(obj, torch.Tensor):
        return [obj]
    if isinstance(obj, (tuple, list)):
        return [t for o in obj for t in _tensors(o)]
    return []


class GraphRunner:
    def __init__(self, max_graphs=32, enabled=True):
        self.enabled = enabled and os.environ.get("PK_CUDA_GRAPHS", "1") != "0"
        self.max_graphs = max_graphs
        self._seen = set()
        self._disabled = set()
        self._graphs = {}
        self.replays = 0

    def run(self, key, fn, inputs):
        if not self.enabled or key in self._disabled:
            return fn(*inputs)
        ent = self._graphs.get(key)
        if ent is None:
            if key not in self._seen:
                self._seen.add(key)
                return fn(*inputs)
            if len(self._graphs) >= self.max_graphs:      # LRU: drop the least recently replayed graph (and its memory pool)
                self._graphs.pop(next(iter(self._graphs)))
            static_in = [t.clone() for t in inputs]
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            try:
                with torch.cuda.graph(graph):
                    out = fn(*static_in)
            except Exception:                      # capture refused (another thread touched CUDA, unsupported call, ...):
                torch.cuda.synchronize()           # never let the graph layer break the call - run this key eagerly from now on
                self._disabled.add(key)
                return fn(*inputs)
            ent = (graph, static_in, out)
            self._graphs[key] = ent
        self._graphs[key] = self._graphs.pop(key)       # most recently used last
        graph, static_in, out = ent
        for s, t in zip(static_in, inputs):
            s.copy_(t)
        graph.replay()
        self.replays += 1
        return out

    def drop(self, key):
        """Forget one key: its graph (and the memory pool it pins) is released; the key runs eagerly, then is captured again."""
        self._graphs.pop(key, None)
        self._seen.discard(key)
        self._disabled.discard(key)

    def clear(self):
        self._graphs.clear()
        self._seen.clear()
        self._disabled.clear()
