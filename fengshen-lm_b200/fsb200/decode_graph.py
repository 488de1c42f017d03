"""The decode step of `generate` (GPT-2, mT5, LLaMA) as one CUDA-graph replay per generated token.

A decode step issues about a dozen `fsb_*` calls per layer for a few microseconds of device work each, so an eager step is
bound by the Python / ctypes launch path. `DecodeGraphs` is the step function `generation.run` drives. A model's `generate`
supplies its prefill, its caches and a `body(tok, index, a, b) -> fp32 logits` that decodes the token ids in the static
buffer `tok` from cache `a` into cache `b`, keeping every position on the device: `kv_len` and the position counters advance
inside the body and the new keys / values land at slot kv_len - 1 (ops.kv_append). Without beam search `b` is `a`. Beam
search needs a second cache, the twin: a reordering step gathers the rows named by the static buffer `index` from the live
cache into the twin (ops.kv_reorder), which then holds the live cache. The body gets the static buffers as arguments: a
body that read them from this object would close a reference cycle that keeps the caches alive after `generate` returns,
until the garbage collector runs. Such a body issues identical launches at every step, so

  * the first decode step runs it eagerly (it also warms workspaces and lazily set kernel attributes up);
  * the first later step with a given key captures it and replays the capture (a capture runs nothing);
  * every later step with that key replays the graph.

The key is (live cache, reorder): beam search alternates the twins A -> B and B -> A. Before a replay the engine's
`param_hook` is run for every bucket (pending parameter all-gathers are joined outside the graph, never captured); after
it, a clone of the static logits is returned, since the caller may keep the tensor (scores) across steps.

`FSB_GENERATE_GRAPH=0` runs the same body eagerly at every step (the reference the graphs are checked against). So does a
process with a per-call profiler set (lib.call_profiler, ops.set_profiler): those record CUDA events around every call.
The graphs, and the static buffers the body reads, live for one `generate` call."""
import os

import torch

from . import lib as L
from . import ops


class DecodeGraphs:
    def __init__(self, model, rows, caches, body, prefill=None):
        """rows: sequences decoded together. caches: [cache], or [cache, twin] for beam search. prefill: the step without
        tokens (the prompt), or None to decode the token ids already in `tok`."""
        dev = model.flat.params.device
        self.model, self.caches, self.body, self.prefill = model, caches, body, prefill
        self.tok = torch.zeros(rows, dtype=torch.int64, device=dev)
        self.index = torch.zeros(rows, dtype=torch.int64, device=dev)
        self.live = 0            # the cache holding the current keys / values
        self.enabled = os.environ.get("FSB_GENERATE_GRAPH", "1") != "0"
        self.warm = False
        self.graphs = {}         # key -> (CUDAGraph, static logits, (kernel launches, fsb_* calls) per replay, workspaces)

    def __call__(self, tokens, reorder):
        """generation.run's step."""
        if tokens is None and self.prefill is not None:
            return self.prefill()
        if tokens is not None:
            self.tok.copy_(tokens)
        key = (self.live, reorder is not None)
        if reorder is not None:
            self.index.copy_(reorder)
            self.live = 1 - self.live
        if not self.enabled or L.call_profiler is not None or ops._profiler is not None:
            return self._body(key)
        if not self.warm:
            self.warm = True
            return self._body(key)
        if key not in self.graphs:
            self._capture(key)
        graph, out, (kernels, calls), _ = self.graphs[key]
        for bucket in self.model.flat.bucket_index:
            self.model._need(bucket)
        graph.replay()
        L.kernel_launches += kernels
        L.launch_count += calls
        return out.clone()

    def _body(self, key):
        src, reorder = key
        a = self.caches[src]
        return self.body(self.tok, self.index, a, self.caches[1 - src] if reorder else a)

    def _capture(self, key):
        m = self.model
        hook = m.__dict__.get("param_hook")
        k0, c0 = L.kernel_launches, L.launch_count
        graph = torch.cuda.CUDAGraph()
        m.param_hook = None      # joined before each replay instead
        try:
            with torch.cuda.graph(graph):
                out = self._body(key)
        finally:
            m.param_hook = hook
        per_replay = (L.kernel_launches - k0, L.launch_count - c0)
        L.kernel_launches, L.launch_count = k0, c0          # the capture launched nothing
        # the graph bakes in the scratch buffers' addresses: keep them alive even if a later call grows a workspace
        self.graphs[key] = (graph, out, per_replay, list(ops._ws_cache.values()))
