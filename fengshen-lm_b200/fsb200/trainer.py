"""Public step API: what a user (or the Lightning-compatible shim in compat/) calls once per optimizer step.

`PretrainStep.step(host_batches)` performs, for each micro-batch: the host->device copy of the token tensors from pinned
memory, forward + backward through the fsb200 model, the engine's bucketed reduce-scatter / fp32 accumulation; then the
sharded AdamW update + parameter all-gather, the LR schedule, and returns the mean loss as a Python float (one
device->host read per step, the `self.log('train/loss', ...)` of the reference's training_step,
examples/ziya_llama/finetune_ziya_llama.py:133-148).
"""
import torch

from .engine import ZeroEngine


class PretrainStep:
    def __init__(self, model, lr_fn, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.1, grad_clip=0.0, ga_steps=1,
                 process_group=None, stage=2, comm_sms=0, cuda_graph=False):
        self.model = model
        self.engine = ZeroEngine(model, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, grad_clip=grad_clip,
                                 ga_steps=ga_steps, process_group=process_group, stage=stage, comm_sms=comm_sms)
        self.lr_fn = lr_fn
        self.global_step = 0
        self.device = model.flat.params.device
        self._loss_acc = torch.zeros((), dtype=torch.float32, device=self.device)
        # CUDA-graph mode (single GPU): the whole optimizer step — every micro-batch's forward + backward, the fp32 gradient
        # accumulation, clipping, AdamW — is captured ONCE and replayed; per-step values (token batches, lr, Adam bias
        # corrections) live in static device buffers that are refreshed before each replay. What a tracing compiler would do
        # for a launch-bound step (BERT-base at batch 8 is ~600 launches for ~1 ms of GPU work), done with the stream API.
        self.cuda_graph = bool(cuda_graph)
        self._graph, self._static, self._graph_recompute = None, None, None
        if self.cuda_graph:
            if self.engine.world > 1:
                raise RuntimeError("PretrainStep(cuda_graph=True) is single-GPU: the engine's side-stream collectives of step t "
                                   "are joined by the forward of step t + 1, outside a one-step capture")
            self.engine.enable_device_hyper()

    def _capture(self, device_batches):
        self._static = [{k: v.clone() for k, v in b.items()} for b in device_batches]
        eng = self.engine
        saved = (eng.step_count, eng.micro)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):       # warm-up on a side stream (allocator pools, lazy kernel attributes), as torch documents
            eng.set_device_hyper(0.0, step=1)
            self._eager_body(self._static, lr=0.0, dry=True)
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        from . import lib as L
        k0, c0 = L.kernel_launches, L.launch_count
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._eager_body(self._static, lr=0.0, dry=True)
        self.launches_per_step = (L.kernel_launches - k0, L.launch_count - c0)   # kernels a replay launches on our behalf
        eng.step_count, eng.micro = saved
        self._graph = g

    def _eager_body(self, batches, lr, dry=False):
        eng = self.engine
        self._loss_acc.zero_()
        for b in batches:
            out = self.model(**b)
            out.loss.backward()
            eng.backward_done()
            self._loss_acc += out.loss.detach()
        eng.step(lr=lr)
        if dry:                    # lr = 0 and weight decay scaled by lr: parameters are unchanged, but m / v were touched
            eng.step_count -= 1

    def step_device(self, device_batches):
        """One optimizer step from batches already resident on the device. Returns the loss as a 0-d device tensor."""
        eng = self.engine
        if self.cuda_graph:
            # the graph holds the launches of the activation-recompute mode set at capture (model.gradient_checkpointing)
            recompute = bool(getattr(self.model, "is_gradient_checkpointing", False))
            if self._graph is not None and recompute != self._graph_recompute:
                raise RuntimeError(f"PretrainStep(cuda_graph=True) captured its step with gradient checkpointing "
                                   f"{'on' if self._graph_recompute else 'off'}; the model now has it "
                                   f"{'on' if recompute else 'off'}, and a replay would run the captured mode. Set the mode "
                                   "before the first step, or build a new PretrainStep")
            if self._graph is None:
                self._graph_recompute = recompute
                state = [eng.master, eng.exp_avg, eng.exp_avg_sq, self.model.flat.params]
                counter = getattr(self.model, "dropout_counter", None)
                if counter is not None:    # the dropout stream counter advances on the device in every training forward
                    state.append(counter)
                snap = [t.clone() for t in state]
                self._capture(device_batches)
                for dst, src in zip(state, snap):
                    dst.copy_(src)     # the warm-up + capture passes must leave no trace in the optimizer or dropout state
            for dst, src in zip(self._static, device_batches):
                for k, v in src.items():
                    dst[k].copy_(v, non_blocking=True)
            eng.set_device_hyper(self.lr_fn(self.global_step))
            self._graph.replay()
            from . import lib as L
            L.kernel_launches += self.launches_per_step[0]
            L.launch_count += self.launches_per_step[1]
            eng.step_count += 1
            self.global_step += 1
            return self._loss_acc / len(device_batches)
        self._loss_acc.zero_()
        for b in device_batches:
            out = self.model(**b)
            out.loss.backward()
            eng.backward_done()
            self._loss_acc += out.loss.detach()
        if eng.hyper is not None:      # device-side scalars are in use (graph mode switched off for a while): keep them current
            eng.set_device_hyper(self.lr_fn(self.global_step))
        eng.step(lr=self.lr_fn(self.global_step))
        self.global_step += 1
        return self._loss_acc / len(device_batches)

    def step(self, host_batches):
        """One optimizer step from pinned host batches (dicts of CPU tensors). Returns the loss as a float."""
        dev = [{k: v.to(self.device, non_blocking=True) for k, v in b.items()} for b in host_batches]
        return float(self.step_device(dev).item())
