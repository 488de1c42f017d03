"""ZeRO-1/2 step engine: what the reference delegates to DeepSpeed through
`fengshen/strategies/megatron_deepspeed.py:302-320` (`deepspeed.initialize`) and `models/model_utils.py:62-72`
(`FusedAdam(adam_w_mode=True)`), re-designed for one NVSwitch domain (SURVEY.md §8a A13/A15, §8e, Appendix D).

  stage 2   : the model reports each bucket (one transformer layer) as soon as its gradients are final; the engine
              reduce-scatters that bucket's bf16 gradients on a side stream (NCCL over NVLink), overlapping the rest of
              backward, and accumulates the reduced shard into an fp32 shard buffer when GA > 1. The per-layer buckets
              share TWO rotating gradient slots (`FlatBuffers.compact_grads`): a full-size gradient buffer never exists
              ("gradients are partitioned as they are produced"). Slot reuse is fenced with CUDA events: backward may
              overwrite a slot only after the reduce-scatter that read it has finished.
  stage 1   : full-size bf16 gradients are kept and accumulated by the wgrad epilogues across the micro-batches; each
              bucket is reduce-scattered ONCE per optimizer step, during the last micro-batch's backward (1/GA of the
              stage-2 traffic, +2 B/param of memory): DeepSpeed's "reduce at the gradient-accumulation boundary".
  step      : (clipping only) local sum-of-squares of the owned shard -> scalar all-reduce -> clip coefficient on the
              device -> fused AdamW on the fp32 {master, m, v} shard writing the bf16 parameters of the owned slice in
              place -> per-bucket in-place all-gather ON THE SIDE STREAM, in forward order. The next forward waits per
              bucket (`model.param_hook`), so the parameter all-gather overlaps the following forward pass instead of
              sitting exposed at the end of the step. Without clipping, each bucket's AdamW waits only for that bucket's
              reduce-scatter, so the tail collective overlaps the update of the other buckets.
The 1/(world*GA) average is folded into dlogits upstream, so the wire op is a plain SUM.
Sharding is per bucket (fsb200/flat.py): rank r owns slice r of every bucket. With world_size == 1 the same code runs
with the collectives compiled out of the data path (config 2, single GPU).

`kernels` is the object providing accumulate / sumsq / clip_coef / adamw_flat (default: fsb200.ops, i.e. the CUDA
library; it raises if the library or a GPU is missing). CPU unit tests of the sharding logic inject a test double.
"""
import torch
import torch.distributed as dist


class ZeroEngine:
    def __init__(self, model, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.1, grad_clip=0.0, ga_steps=1,
                 process_group=None, stage=2, kernels=None, overlap_comm=True, comm_sms=None, comm_backend="torch", tp_group=None):
        fmt = getattr(model, "weight_format", "bf16")   # "int8" / "int4": a load_in_8bit / load_in_4bit model
        if fmt != "bf16":
            raise NotImplementedError(f"fsb200 ZeroEngine: an {fmt} (load_in_{fmt[3:]}bit=True) model only runs inference; "
                                      "training it is not implemented")
        self.model = model
        self.flat = model.flat
        self.lr, self.betas, self.eps, self.weight_decay = lr, betas, eps, weight_decay
        self.grad_clip, self.ga_steps, self.stage = float(grad_clip), int(ga_steps), int(stage)
        if stage not in (1, 2):
            raise ValueError("ZeroEngine supports ZeRO stage 1 and 2 (optimizer-state / gradient sharding)")
        self.pg = process_group
        self.distributed = dist.is_available() and dist.is_initialized() and dist.get_world_size(process_group) > 1
        self.world = dist.get_world_size(process_group) if self.distributed else 1
        self.rank = dist.get_rank(process_group) if self.distributed else 0
        if self.world != self.flat.world_size:
            raise ValueError(f"model was laid out for world_size={self.flat.world_size}, process group has {self.world}")
        if kernels is None:
            from . import ops as kernels  # CUDA library; no fallback
        self.k = kernels
        dev = self.flat.params.device
        self.device = dev
        n = self.flat.shard_numel
        nb = len(self.flat.buckets)
        self.master = torch.empty(n, dtype=torch.float32, device=dev)
        for i in range(nb):
            self._seg(self.master, i).copy_(self.flat.bucket_slice(i, self.rank).float())
        self.exp_avg = torch.zeros(n, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros(n, dtype=torch.float32, device=dev)
        # stage 2 accumulates reduced shards in fp32 across micro-batches; stage 1 accumulates full bf16 gradients in place
        self.acc32 = torch.zeros(n, dtype=torch.float32, device=dev) if (self.ga_steps > 1 and self.stage == 2) else None
        self.recv16 = torch.zeros(n, dtype=torch.bfloat16, device=dev) if self.world > 1 else None
        # tensor parallelism: `process_group` is the DATA-parallel group; the gradient norm also sums over `tp_group`, with
        # the buckets every tensor-parallel rank holds identically (model.tp_replicated_buckets: norms) counted once
        self.tp_group = tp_group
        self.tp = dist.get_world_size(tp_group) if tp_group is not None else 1
        rep_names = set(getattr(model, "tp_replicated_buckets", ())) if self.tp > 1 else set()
        self.tp_replicated = [b[0] in rep_names for b in self.flat.buckets]
        self.sumsq_rep = torch.zeros((), dtype=torch.float32, device=dev)
        self.sumsq = torch.zeros((), dtype=torch.float32, device=dev)
        self.coef = torch.ones((), dtype=torch.float32, device=dev)
        self.grad_norm = torch.zeros((), dtype=torch.float32, device=dev)
        # per-step scalars of AdamW in device memory (CUDA-graph mode: see set_device_hyper / trainer.PretrainStep)
        self.hyper = None
        self.use_streams = dev.type == "cuda" and overlap_comm and self.world > 1
        self.comm_stream = torch.cuda.Stream(device=dev) if self.use_streams else None
        # ZeRO-2: per-layer gradients live in rotating slots whenever they are consumed bucket by bucket (reduced or
        # accumulated into the fp32 shard); with world == 1 and GA == 1 AdamW reads the full gradients at the step.
        self.grad_bytes_released = 0
        if self.stage == 2 and (self.world > 1 or self.acc32 is not None):
            self.grad_bytes_released = self.flat.compact_grads(slots=2)
        self.rs_event = [None] * nb      # per bucket: reduce-scatter (+ fp32 accumulation) finished on the side stream
        self.ag_event = [None] * nb      # per bucket: parameter all-gather finished on the side stream
        self._last_rot_event = {}        # rotating family -> event of the most recently issued reduce-scatter
        self.micro = 0
        self.step_count = 0
        self.comm_bytes = 0
        # Data-path collectives: torch.distributed's NCCL communicator (default), or the library's own fsb_comm_* entry
        # points (comm_backend="fsb": the C-ABI a non-PyTorch host binds; torch.distributed then only carries the
        # 128-byte NCCL id at start-up).
        self.fsb_comm = None
        # DIAGNOSTIC ONLY (results are wrong): FSB_ENGINE_SKIP_COLLECTIVES=1 keeps every stream / event / kernel of the step but
        # drops the NCCL calls — step time with minus step time without is the EXPOSED communication (bench.py `comm_probe`)
        import os
        self.skip_collectives = os.environ.get("FSB_ENGINE_SKIP_COLLECTIVES", "0") == "1"
        if comm_backend not in ("torch", "fsb"):
            raise ValueError(f"comm_backend {comm_backend!r}: expected 'torch' or 'fsb'")
        if comm_backend == "fsb" and self.world > 1:
            if dev.type != "cuda":
                raise RuntimeError("comm_backend='fsb' needs CUDA devices (NCCL)")
            from . import comm as _comm
            self.fsb_comm = _comm.Communicator(self.world, self.rank, process_group, dev)
        # buckets in the order the forward pass first touches them (no-decay parameters — norms, biases — are read by
        # every layer, so that bucket is gathered first)
        order = list(range(nb))
        nd = [i for i in order if not self.flat.buckets[i][3]]
        self.fwd_order = nd + [i for i in order if i not in nd]
        model.grad_hook = self._on_bucket
        model.param_hook = self._need_params
        model.backward_begin_hook = self._backward_begin
        model.loss_scale = 1.0 / (self.ga_steps * self.world)
        model.accumulate_grads = False
        # NCCL's kernels need SMs of their own while they overlap the persistent GEMMs (one CTA per SM, a full register
        # file each): leave them `comm_sms` SMs instead of letting a GEMM CTA queue behind a collective.
        # (off by default: measure with bench.py --comm-sms N before turning it on for a config)
        self.comm_sms = int(comm_sms or 0) if self.use_streams else 0
        if hasattr(self.k, "set_reserved_sms") and dev.type == "cuda":
            self.k.set_reserved_sms(self.comm_sms)

    # rank-local segment of bucket i inside a shard-sized buffer
    def _seg(self, buf, i):
        off = self.flat.shard_offsets[i]
        per = self.flat.buckets[i][2] // self.world
        return buf[off:off + per]

    # ---- forward side ------------------------------------------------------------------------------------------
    def _need_params(self, name):
        """The forward pass is about to read bucket `name`: wait for its parameter all-gather (issued by step())."""
        i = self.flat.bucket_index.get(name)
        if i is None:
            return
        ev = self.ag_event[i]
        if ev is not None:
            torch.cuda.current_stream(self.device).wait_event(ev)
            self.ag_event[i] = None

    def wait_params(self):
        """Join every outstanding parameter all-gather (checkpointing, evaluation, reading flat.params from the host)."""
        for i, ev in enumerate(self.ag_event):
            if ev is not None:
                torch.cuda.current_stream(self.device).wait_event(ev)
                self.ag_event[i] = None

    # ---- backward side -----------------------------------------------------------------------------------------
    def _backward_begin(self):
        """A micro-batch's backward is about to overwrite gradient buckets: every collective that still reads the
        previous micro-batch's gradients must have finished (they had a whole forward pass to do so)."""
        if self.use_streams:
            torch.cuda.current_stream(self.device).wait_stream(self.comm_stream)

    def _reduce_now(self):
        return self.stage == 2 or self.micro == self.ga_steps - 1

    def _on_bucket(self, name):
        i = self.flat.bucket_index[name]
        first = self.micro == 0
        if not self._reduce_now():
            return                      # stage 1: gradients keep accumulating in the full-size bf16 buffer
        if self.world > 1:
            full = self.flat.bucket_view(i, grad=True)
            out = self._seg(self.recv16, i)
            if self.use_streams:
                cur = torch.cuda.current_stream(self.device)
                self.comm_stream.wait_stream(cur)
                with torch.cuda.stream(self.comm_stream):
                    self._reduce_scatter(out, full)
                    if self.acc32 is not None:
                        self.k.accumulate(self._seg(self.acc32, i), out, 1.0, overwrite=first)
                    ev = torch.cuda.Event()
                    ev.record(self.comm_stream)
                self.rs_event[i] = ev
                rot = self.flat.rot_group[i]
                if rot is not None:
                    # the NEXT layer of this family writes the other slot, last read by the previously issued
                    # reduce-scatter of the family: backward may proceed into it only once that one is done
                    prev = self._last_rot_event.get(rot[0])
                    if prev is not None:
                        cur.wait_event(prev)
                    self._last_rot_event[rot[0]] = ev
            else:
                self._reduce_scatter(out, full)
                if self.acc32 is not None:
                    self.k.accumulate(self._seg(self.acc32, i), out, 1.0, overwrite=first)
            self.comm_bytes += full.numel() * 2 * (self.world - 1) // self.world
        elif self.acc32 is not None:
            self.k.accumulate(self._seg(self.acc32, i), self.flat.bucket_view(i, grad=True), 1.0, overwrite=first)

    def _reduce_scatter(self, out, full):
        if self.skip_collectives:
            return
        if self.fsb_comm is not None:
            self.fsb_comm.reduce_scatter(out, full)
        else:
            dist.reduce_scatter_tensor(out, full, op=dist.ReduceOp.SUM, group=self.pg)

    def _all_gather(self, full, mine):
        if self.skip_collectives:
            return
        if self.fsb_comm is not None:
            self.fsb_comm.all_gather(full, mine)
        else:
            dist.all_gather_into_tensor(full, mine, group=self.pg)

    def backward_done(self):
        """Call once after each micro-batch's loss.backward()."""
        self.micro += 1
        self._last_rot_event.clear()
        if self.stage == 1:
            self.model.accumulate_grads = 0 < self.micro < self.ga_steps

    def _grad_seg(self, i):
        if self.acc32 is not None:
            return self._seg(self.acc32, i)
        if self.world > 1:
            return self._seg(self.recv16, i)
        return self.flat.bucket_view(i, grad=True)

    def _wait_rs(self, i):
        ev = self.rs_event[i]
        if ev is not None:
            torch.cuda.current_stream(self.device).wait_event(ev)
            self.rs_event[i] = None

    # ---- optimizer step ----------------------------------------------------------------------------------------
    def enable_device_hyper(self):
        """Keep {lr, 1 - beta1^t, sqrt(1 - beta2^t)} in a device tensor that AdamW reads: every step then issues byte-identical
        launches, so the whole step can be captured in a CUDA graph. Call set_device_hyper(lr) before each (replayed) step."""
        self.hyper = torch.zeros(3, dtype=torch.float32, device=self.device)

    def set_device_hyper(self, lr, step=None):
        step = (self.step_count + 1) if step is None else step
        # a fresh PAGEABLE host tensor per call: cudaMemcpyAsync stages pageable memory before it returns, so the host may run
        # many steps ahead of the device without a later step's scalars overtaking an earlier step's copy
        # the C side receives beta1 / beta2 as C floats and forms the corrections in double from THOSE values: do the same, so
        # that a replayed step is bit-identical to the eager one
        b1, b2 = (float(torch.tensor(x, dtype=torch.float32)) for x in self.betas)
        host = torch.tensor([float(lr), 1.0 - b1 ** step, (1.0 - b2 ** step) ** 0.5], dtype=torch.float32)
        self.hyper.copy_(host, non_blocking=True)

    def step(self, lr=None, weight_decay=None):
        if self.micro != self.ga_steps:
            raise RuntimeError(f"ZeroEngine.step() after {self.micro} micro-batches, expected {self.ga_steps}")
        lr = self.lr if lr is None else lr
        wd = self.weight_decay if weight_decay is None else weight_decay
        nb = len(self.flat.buckets)
        coef = None
        if self.grad_clip > 0.0:
            if self.use_streams:
                torch.cuda.current_stream(self.device).wait_stream(self.comm_stream)
                self.rs_event = [None] * nb
            first, first_rep = True, True
            for i in range(nb):
                if self.tp_replicated[i]:
                    self.k.sumsq(self._grad_seg(i), self.sumsq_rep, accumulate=not first_rep)
                    first_rep = False
                else:
                    self.k.sumsq(self._grad_seg(i), self.sumsq, accumulate=not first)
                    first = False
            if self.tp > 1:
                if not first_rep:
                    self.sumsq.add_(self.sumsq_rep, alpha=1.0 / self.tp)
                dist.all_reduce(self.sumsq, op=dist.ReduceOp.SUM, group=self.tp_group)
            if self.world > 1 and not self.skip_collectives:
                if self.fsb_comm is not None:
                    self.fsb_comm.all_reduce(self.sumsq)
                else:
                    dist.all_reduce(self.sumsq, op=dist.ReduceOp.SUM, group=self.pg)
            self.k.clip_coef(self.sumsq, self.grad_clip, self.coef, self.grad_norm)
            coef = self.coef
        self.step_count += 1
        cur = torch.cuda.current_stream(self.device) if self.use_streams else None
        for i in self.fwd_order:
            decay_on = self.flat.buckets[i][3]
            if self.use_streams:
                self._wait_rs(i)
            self.k.adamw_flat(self._seg(self.master, i), self._seg(self.exp_avg, i), self._seg(self.exp_avg_sq, i),
                              self._grad_seg(i), self.flat.bucket_slice(i, self.rank), lr, self.betas[0], self.betas[1],
                              self.eps, wd if decay_on else 0.0, self.step_count, coef,
                              **({"hyper": self.hyper} if self.hyper is not None else {}))
            if self.world > 1:
                if self.use_streams:
                    self.comm_stream.wait_stream(cur)
                    with torch.cuda.stream(self.comm_stream):
                        self._all_gather(self.flat.bucket_view(i), self.flat.bucket_slice(i, self.rank))
                        ev = torch.cuda.Event()
                        ev.record(self.comm_stream)
                    self.ag_event[i] = ev
                else:
                    self._all_gather(self.flat.bucket_view(i), self.flat.bucket_slice(i, self.rank))
                self.comm_bytes += self.flat.buckets[i][2] * 2 * (self.world - 1) // self.world
        self.micro = 0
        self.model.accumulate_grads = False

    def memory_report(self):
        """Bytes this engine + the model's flat buffers hold per rank (DESIGN.md §1 memory budget)."""
        f = self.flat
        return {"params": f.params.numel() * 2, "grads": f.grads.numel() * f.grads.element_size(),
                "grads_released_by_zero2": self.grad_bytes_released,
                "optimizer_state": 3 * self.master.numel() * 4,
                "acc32": 0 if self.acc32 is None else self.acc32.numel() * 4,
                "recv16": 0 if self.recv16 is None else self.recv16.numel() * 2}

    # ---- checkpoint (rank-local optimizer shard, the analogue of DeepSpeed's zero_pp_rank_*_optim_states.pt) ----
    def state_dict(self):
        self.wait_params()
        return {"format": "fsb200-zero-shard-v1", "master": self.master, "exp_avg": self.exp_avg,
                "exp_avg_sq": self.exp_avg_sq, "step": self.step_count, "world": self.world, "rank": self.rank}

    def load_state_dict(self, sd):
        if not isinstance(sd, dict) or "master" not in sd or "world" not in sd:
            raise ValueError("not an fsb200 optimizer shard (expected keys master / exp_avg / exp_avg_sq / step / world / "
                             "rank); DeepSpeed's own zero_pp_rank_* files are not readable by this engine")
        if sd["world"] != self.world or sd["rank"] != self.rank:
            raise ValueError("optimizer shard was saved for a different (world, rank)")
        self.master.copy_(sd["master"]); self.exp_avg.copy_(sd["exp_avg"]); self.exp_avg_sq.copy_(sd["exp_avg_sq"])
        self.step_count = int(sd["step"])
