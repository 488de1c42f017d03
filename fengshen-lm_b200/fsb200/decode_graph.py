"""One CUDA-graph replay per generated token: the decode step of `generate` (GPT-2, mT5, LLaMA) captured once and replayed.

A decode step issues about a dozen `fsb_*` calls per layer for a few microseconds of device work each, so an eager step is
bound by the Python / ctypes launch path. The models write their step as a `body(key) -> fp32 logits` that reads its inputs
(token ids, beam index) from static buffers and keeps every position on the device: `kv_len` and the position counters
advance inside the body, the new keys / values land at slot kv_len - 1 (ops.kv_append) and beam search gathers the caches
from one static twin into the other (ops.kv_reorder). Such a body issues identical launches at every step, so

  * the first call runs it eagerly (it also warms workspaces and lazily set kernel attributes up);
  * the first later call with a given key captures it and replays the capture (a capture runs nothing);
  * every later call with that key replays the graph.

`key` names a body variant with its own graph: beam search alternates the twin caches A -> B and B -> A. Before a replay the
engine's `param_hook` is run for every bucket (pending parameter all-gathers are joined outside the graph, never captured);
after it, a clone of the static logits is returned, since the caller may keep the tensor (scores) across steps.

`FSB_GENERATE_GRAPH=0` runs the same body eagerly at every step (the reference the graphs are checked against). So does a
process with a per-call profiler set (lib.call_profiler, ops.set_profiler): those record CUDA events around every call.
The graphs, and the static buffers the body closes over, live for one `generate` call."""
import os

import torch

from . import lib as L
from . import ops


class DecodeGraphs:
    def __init__(self, model, body):
        self.model, self.body = model, body
        self.enabled = os.environ.get("FSB_GENERATE_GRAPH", "1") != "0"
        self.warm = False
        self.graphs = {}        # key -> (CUDAGraph, static logits, (kernel launches, fsb_* calls) per replay, workspaces)

    def __call__(self, key=0):
        if not self.enabled or L.call_profiler is not None or ops._profiler is not None:
            return self.body(key)
        if not self.warm:
            self.warm = True
            return self.body(key)
        if key not in self.graphs:
            self._capture(key)
        graph, out, (kernels, calls), _ = self.graphs[key]
        for bucket in self.model.flat.bucket_index:
            self.model._need(bucket)
        graph.replay()
        L.kernel_launches += kernels
        L.launch_count += calls
        return out.clone()

    def _capture(self, key):
        m = self.model
        hook = m.__dict__.get("param_hook")
        k0, c0 = L.kernel_launches, L.launch_count
        graph = torch.cuda.CUDAGraph()
        m.param_hook = None      # joined before each replay instead
        try:
            with torch.cuda.graph(graph):
                out = self.body(key)
        finally:
            m.param_hook = hook
        per_replay = (L.kernel_launches - k0, L.launch_count - c0)
        L.kernel_launches, L.launch_count = k0, c0          # the capture launched nothing
        # the graph bakes in the scratch buffers' addresses: keep them alive even if a later call grows a workspace
        self.graphs[key] = (graph, out, per_replay, list(ops._ws_cache.values()))
