"""Data-parallel training engine for the ivb200 modules: one process per GPU, NCCL over NVLink.

What it replaces in the reference: DDP / DeepSpeed ZeRO-1 gradient reduction + AdamW
(InternVideo2/single_modality/run_pretraining.py:368-382, utils.py:814-908, optim_factory.py:56-190)
for the one data-parallel path this repo accelerates.  Design (H100-first):

  * all parameters live in ONE flat bf16 buffer (16-byte aligned slices, what the TMA descriptors and
    vector loads want), all gradients in one flat bf16 buffer that `param.grad` aliases, fp32 master
    weights + Adam moments in three flat fp32 buffers: 16 B/param -> 17 GB for the 1B model, 95 GB
    for 6B, which exceeds one H100's 80 GB: 6B needs zero1=True over several GPUs;
  * gradient all-reduce is bucketed over contiguous slices of the flat gradient and launched as soon as
    a bucket is complete, so NCCL (NVLS/ring over NVSwitch) overlaps the remaining backward GEMMs.
    Stream ordering is explicit: every "gradient written" signal records an event on the stream it was
    issued from; the collective is enqueued from the engine's own communication stream after that stream
    has waited on EVERY such event of the bucket (autograd runs AccumulateGrad nodes on the stream their
    node was created on, which is not necessarily the stream the Block kernels run on);
  * the 1/world_size and the global-norm clip coefficient are folded into the AdamW kernel's gradient
    scale (no extra pass over the gradients);
  * the step is a single fused AdamW kernel per weight-decay group over the flat buffers;
  * `zero1=True` shards the fp32 optimizer state (master weights + both moments) over the ranks —
    DeepSpeed ZeRO stage 1, the reference's bf16 recipe (utils.py:863-870): every rank steps its own
    contiguous 1/world slice of the flat buffer and the updated bf16 parameters are all-gathered in
    place; 4 + 12/world bytes per parameter instead of 16.

Host logic (bucketing, ordering, scaling, sharding, checkpoint round trip) is exercised on CPU with gloo in
tests/test_dist_cpu.py; the kernels themselves need the GPU.
"""
from __future__ import annotations

import contextlib
import os
from dataclasses import dataclass, field

import torch
import torch.distributed as dist

ALIGN = 8  # elements (16 bytes of bf16)


@dataclass
class Bucket:
    start: int
    end: int
    pending: int = 0
    total: int = 0
    handle: object = None
    launched: bool = False
    events: dict = field(default_factory=dict)   # stream id -> (stream, event) of the writers seen this step


def plan_layout(named_shapes, no_decay_names=()):
    """Flat-buffer layout: decay group first, then no-decay (1-D tensors, biases, skip list —
    optim_factory.py:56-98).  Returns (entries, n_decay_elems, total_elems); entries are
    (name, offset, numel, decay) with offsets aligned to ALIGN elements."""
    decay, nodecay = [], []
    for name, shape in named_shapes:
        numel = 1
        for s in shape:
            numel *= s
        nd = len(shape) == 1 or name.endswith(".bias") or name.endswith("_bias") or name in no_decay_names \
            or name.split(".")[-1] in no_decay_names
        (nodecay if nd else decay).append((name, numel))
    entries, off = [], 0
    n_decay = 0
    for group, flag in ((decay, True), (nodecay, False)):
        for name, numel in group:
            entries.append((name, off, numel, flag))
            off += (numel + ALIGN - 1) // ALIGN * ALIGN
        if flag:
            n_decay = off
    return entries, n_decay, off


def plan_buckets(entries, total, bucket_elems, first_elems=None, split_at=None):
    """Contiguous buckets over the flat gradient, each made of WHOLE entries (cut at the first entry boundary
    at or past the bucket's target size).  A bucket is all-reduced as soon as every entry in it has its gradient, so an
    entry must never straddle two buckets: backward produces gradients in reverse layout order, and the
    tail of an earlier-layer tensor inside a later bucket would be reduced before it is written.
    `first_elems`: target of the FIRST bucket in layout order, doubling per bucket up to `bucket_elems`.  The first
    layers' gradients are produced last, so their all-reduce cannot hide behind backward: a small final bucket
    shortens the exposed tail (2 GPUs, cfg-2: 119.2 -> 118.7 ms with 128 MB instead of 256 MB buckets).
    `split_at`: an offset at which a bucket boundary is forced — the start of the no-decay section.  That section
    (position tables, biases, norm weights of EVERY layer) is only complete at the very end of backward; sharing a
    bucket with it would hold the last blocks' weight gradients (ready first) back until then."""
    ordered = sorted(entries, key=lambda e: e[1])
    buckets, owner = [], {}
    start, count = 0, 0
    for i, (name, off, numel, _) in enumerate(ordered):
        owner[name] = len(buckets)
        count += 1
        nxt = ordered[i + 1][1] if i + 1 < len(ordered) else total
        target = bucket_elems if not first_elems else min(bucket_elems, first_elems << len(buckets))
        if nxt - start >= target or i + 1 == len(ordered) or (split_at is not None and nxt == split_at and nxt > start):
            buckets.append(Bucket(start, nxt, total=count))
            start, count = nxt, 0
    if not buckets:
        buckets.append(Bucket(0, total))
    return buckets, owner


def plan_shards(total, world):
    """ZeRO-1 partition of the flat buffers: `world` equal contiguous slices of ALIGN-multiple length.
    Returns (shard_len, padded_total)."""
    per = (total + world - 1) // world
    per = (per + ALIGN - 1) // ALIGN * ALIGN
    return per, per * world


class PretrainEngine:
    """Flat-buffer AdamW + overlapped gradient all-reduce around an ivb200 model (bf16 params)."""

    def __init__(self, model, lr=1.5e-4, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.05, clip_grad=3.0,
                 process_group=None, bucket_mb=256, overlap=True, direct_grads=True,
                 broadcast_init=True, zero1=False, check_finite=False, first_bucket_mb=32, allreduce="auto"):
        self.model = model
        self.lr, self.betas, self.eps, self.wd = lr, betas, eps, weight_decay
        self.clip_grad = clip_grad
        self.pg = process_group
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(process_group) if dist.is_initialized() else 0
        self.step_count = 0
        self.dyn = None
        self.check_finite = check_finite
        self.skipped = None            # device flag: 1.0 when the last step was skipped (non-finite gradient)
        named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
        skip = model.no_weight_decay() if hasattr(model, "no_weight_decay") else set()
        entries, self.n_decay, total = plan_layout([(n, tuple(p.shape)) for n, p in named], skip)
        self.entries, self.total = entries, total
        self.zero1 = bool(zero1) and self.world > 1
        self.shard_len, padded = plan_shards(total, self.world) if self.zero1 else (total, total)
        self.padded = padded
        self.shard_lo = self.rank * self.shard_len if self.zero1 else 0
        self.shard_hi = min(self.shard_lo + self.shard_len, padded)
        p0 = named[0][1]
        dev, dt = p0.device, p0.dtype
        self.flat_param = torch.zeros(padded, device=dev, dtype=dt)
        # gradient all-reduce: "nvls" = libivb200's in-switch kernel over a symmetric (multicast-mapped) gradient buffer,
        # "nccl" = ncclAllReduce, "auto" = nvls where the platform offers it (CUDA, 2..16 ranks, NVLink multicast)
        allreduce = os.environ.get("IVB_ALLREDUCE", allreduce)
        if allreduce not in ("auto", "nvls", "nccl"):
            raise ValueError(f"allreduce must be auto / nvls / nccl, not {allreduce!r}")
        self.nvls = None
        self.allreduce_note = ""
        if self.world > 1 and dev.type == "cuda" and not self.zero1 and allreduce != "nccl":
            from .nvls import NvlsBuffer, NvlsUnavailable
            try:
                self.nvls = NvlsBuffer(padded, dt, dev, process_group)
            except NvlsUnavailable as e:
                if allreduce == "nvls":
                    raise
                self.allreduce_note = f"nvls unavailable ({e}); using nccl"
        elif allreduce == "nvls":
            raise RuntimeError("ivb200 engine: allreduce='nvls' needs CUDA, world_size > 1 and zero1=False")
        self.allreduce = "nvls" if self.nvls is not None else ("nccl" if self.world > 1 else "none")
        self.flat_grad = self.nvls.tensor if self.nvls is not None else torch.zeros(padded, device=dev, dtype=dt)
        self._inflight = False           # reductions launched and not yet joined by reduce_gradients()
        self.comm_profile = False        # eager steps only: CUDA events around every bucket's all-reduce
        self._comm_events, self._exposed_events = [], []
        nstate = self.shard_hi - self.shard_lo
        self.master = torch.zeros(nstate, device=dev, dtype=torch.float32)
        self.exp_avg = torch.zeros(nstate, device=dev, dtype=torch.float32)
        self.exp_avg_sq = torch.zeros(nstate, device=dev, dtype=torch.float32)
        pmap = dict(named)
        self._params = [pmap[name] for name, *_ in entries]
        with torch.no_grad():
            for name, off, numel, _ in entries:
                p = pmap[name]
                self.flat_param[off:off + numel].copy_(p.data.reshape(-1))
                p.data = self.flat_param[off:off + numel].view(p.shape)
                p.grad = self.flat_grad[off:off + numel].view(p.shape)
                # gradient sink: ops.BlockFn writes this parameter's gradient straight into flat_grad
                p._ivb_sink, p._ivb_off, p._ivb_bucket = self, off, None
        if self.world > 1 and broadcast_init:
            # DDP semantics (run_pretraining.py:378): every replica starts from rank 0's parameters
            dist.broadcast(self.flat_param, src=dist.get_global_rank(process_group, 0) if process_group is not None else 0,
                           group=process_group)
        self.sync_master_from_params()
        self.buckets, self.owner = plan_buckets(entries, total, int(bucket_mb * 1024 * 1024 // 2),
                                                int(first_bucket_mb * 1024 * 1024 // 2) if first_bucket_mb else None,
                                                split_at=self.n_decay)
        self.overlap = overlap and self.world > 1
        self.accumulating = False
        self._legacy_stream_order = False
        self._hooks = []
        self.direct = direct_grads
        self.comm_stream = None
        for name, p in named:
            p._ivb_bucket = self.owner[name]
        if self.overlap:
            for name, p in named:
                b = self.owner[name]
                self._hooks.append(p.register_post_accumulate_grad_hook(self._make_hook(b)))
        self._reset_buckets()

    # ---- gradient sink protocol (ops.BlockFn)
    def direct_enabled(self):
        return self.direct

    def grad_written(self, p):
        """A kernel accumulating p's gradient into flat_grad has been enqueued on the current stream
        (what the post-accumulate-grad hook signals for autograd-accumulated parameters)."""
        if self.overlap:
            # autograd still runs the parameter's AccumulateGrad node with an undefined gradient when the
            # Function returns None for it, and torch >= 2.x fires the post-accumulate hook for that too:
            # remember that this parameter has signalled so the hook's echo is dropped (round 1 counted
            # both, handed buckets to NCCL half-written and let the replicas drift apart)
            self._sunk.add(id(p))
            self._bucket_ready(p._ivb_bucket)

    # ---- gradient reduction
    def _reset_buckets(self):
        for b in self.buckets:
            b.pending, b.handle, b.launched = b.total, None, False
            b.events = {}
        self._sunk = set()

    def _is_cuda(self):
        return self.flat_grad.is_cuda

    def _bucket_ready(self, bi):
        """One entry of bucket `bi` has its gradient enqueued on the CURRENT stream."""
        b = self.buckets[bi]
        if self.accumulating:
            return                       # micro-batch accumulation: every bucket is reduced in reduce_gradients()
        if b.launched or b.pending <= 0:
            raise RuntimeError(
                f"ivb200 engine: gradient arrived for bucket {bi} after it was handed to NCCL "
                "(a parameter produced more than one gradient between zero_grad() and step()); "
                "wrap extra backward passes in `with engine.accumulate():`")
        if self._is_cuda():
            s = torch.cuda.current_stream()
            rec = b.events.get(s.cuda_stream)
            if rec is None:
                rec = b.events[s.cuda_stream] = (s, torch.cuda.Event())
            rec[1].record(s)             # re-recording keeps only the latest point of that stream: covers all earlier work
        b.pending -= 1
        if b.pending == 0:
            self._launch(b)

    def _launch(self, b):
        """All-reduce bucket `b` on the communication stream, ordered after every stream that wrote into it."""
        view = self.flat_grad[b.start:b.end]
        b.launched = True
        self._inflight = True
        if not self._is_cuda() or self._legacy_stream_order:
            # (debug switch for tools/dp_check.py: round-1 behaviour — order NCCL after the CURRENT stream only)
            b.handle = dist.all_reduce(view, group=self.pg, async_op=True)
            return
        if self.comm_stream is None:
            # high priority: the few CTAs of a reduction take SMs as soon as any become free instead of queueing behind
            # the next persistent GEMM grid
            self.comm_stream = torch.cuda.Stream(priority=-1)
        cs = self.comm_stream
        cur = torch.cuda.current_stream()
        if not b.events:                              # launched from reduce_gradients(): order after the caller
            cs.wait_stream(cur)
        for _, ev in b.events.values():
            cs.wait_event(ev)
        with torch.cuda.stream(cs):
            if self.comm_profile:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(cs)
            if self.nvls is not None:
                # the first layers' buckets (layout order) are produced last: nothing is left to hide behind, use more CTAs
                self.nvls.all_reduce_(b.start, b.end, wide=(b.start == 0 or b.start == self.n_decay))
                b.handle = None
            else:
                b.handle = dist.all_reduce(view, group=self.pg, async_op=True)
            if self.comm_profile:
                if b.handle is not None:
                    b.handle.wait()        # NCCL runs on its own stream: pull its completion onto `cs` for the end event
                e1.record(cs)
                self._comm_events.append((e0, e1, (b.end - b.start) * self.flat_grad.element_size()))

    def _make_hook(self, bi):
        def hook(p):
            if not self.overlap:          # switched off after construction: reduce_gradients() does everything
                return
            if id(p) in self._sunk:       # echo of a gradient the sink already signalled (see grad_written)
                self._sunk.discard(id(p))
                return
            self._bucket_ready(bi)
        return hook

    @contextlib.contextmanager
    def accumulate(self):
        """Gradient accumulation over several backward passes (DDP.no_sync): nothing is reduced until
        reduce_gradients()/step()."""
        prev, self.accumulating = self.accumulating, True
        try:
            yield self
        finally:
            self.accumulating = prev

    def _drain(self):
        """Wait for reductions that were launched but never joined (a step abandoned between backward and
        reduce_gradients(), e.g. after an exception): they would otherwise land in the buffer after it is cleared."""
        for b in self.buckets:
            if b.handle is not None:
                b.handle.wait()
        if self.comm_stream is not None and self._is_cuda():
            torch.cuda.current_stream().wait_stream(self.comm_stream)
        self._inflight = False

    def zero_grad(self):
        if self._inflight:
            self._drain()
        self.flat_grad.zero_()
        self._reset_buckets()

    def check_aliases(self):
        """Every parameter's .grad must still alias the flat gradient buffer (model.zero_grad(set_to_none=True)
        or an optimizer that replaces .grad breaks the sink silently — use engine.zero_grad())."""
        base = self.flat_grad.data_ptr()
        esz = self.flat_grad.element_size()
        for (name, off, numel, _), p in zip(self.entries, self._params):
            if p.grad is None or p.grad.data_ptr() != base + off * esz:
                raise RuntimeError(f"ivb200 engine: {name}.grad no longer aliases the flat gradient buffer; "
                                   "only engine.zero_grad() may reset gradients")

    def reduce_gradients(self):
        if self.world == 1:
            return
        if self.overlap:
            for b in self.buckets:
                if not b.launched:        # params that received no gradient this step / accumulation mode
                    b.events = {}
                    self._launch(b)
            for b in self.buckets:
                if b.handle is not None:
                    b.handle.wait()
            if self.comm_stream is not None:
                cur = torch.cuda.current_stream()
                if self.comm_profile:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(cur)
                cur.wait_stream(self.comm_stream)
                if self.comm_profile:
                    e1.record(cur)
                    self._exposed_events.append((e0, e1))
            self._inflight = False
        elif self.nvls is not None:
            self.nvls.all_reduce_(0, self.total)
        else:
            dist.all_reduce(self.flat_grad[:self.total], group=self.pg)

    def comm_report(self, steps=1):
        """(eager steps run with comm_profile=True) per-step all-reduce time on the communication stream and the part
        of it the compute stream had to wait for after backward; clears the record."""
        torch.cuda.synchronize()
        busy = sum(a.elapsed_time(b) for a, b, _ in self._comm_events)
        nbytes = sum(n for _, _, n in self._comm_events)
        exposed = sum(a.elapsed_time(b) for a, b in self._exposed_events)
        nb = len(self._comm_events)
        self._comm_events, self._exposed_events = [], []
        steps = max(steps, 1)
        return {"allreduce": self.allreduce, "buckets_per_step": nb // steps, "bytes_per_step": nbytes // steps,
                "comm_stream_ms_per_step": round(busy / steps, 3), "exposed_ms_per_step": round(exposed / steps, 3),
                "bus_GBps": round(nbytes / max(busy, 1e-9) / 1e6, 1)}

    # ---- optimizer
    def set_lr(self, lr):
        """Schedule hook (engine_for_pretraining.py:56-61 pokes param_group['lr'] every step)."""
        self.lr = lr
        if self.dyn is not None:
            self.dyn[0:1].fill_(lr)

    def sync_master_from_params(self):
        """fp32 master weights := current bf16 parameters (call after model.load_state_dict())."""
        with torch.no_grad():
            self.master.copy_(self.flat_param[self.shard_lo:self.shard_hi].float())

    def state_dict(self):
        """Optimizer state for checkpoint/resume (the reference resumes it through the DeepSpeed checkpoint,
        utils.py:814-908).  With zero1 each rank holds (and saves) its own shard, like DeepSpeed's per-rank
        `*_optim_states.pt`."""
        return {"master": self.master.clone(), "exp_avg": self.exp_avg.clone(), "exp_avg_sq": self.exp_avg_sq.clone(),
                "step": self.step_count, "lr": self.lr, "shard": (self.shard_lo, self.shard_hi), "total": self.total,
                "layout": [(n, o, k) for n, o, k, _ in self.entries]}

    def load_state_dict(self, sd):
        if sd["total"] != self.total or tuple(sd["shard"]) != (self.shard_lo, self.shard_hi) or \
                [tuple(x) for x in sd["layout"]] != [(n, o, k) for n, o, k, _ in self.entries]:
            raise RuntimeError("ivb200 engine: optimizer state does not match this model's flat layout / sharding")
        with torch.no_grad():
            self.master.copy_(sd["master"]); self.exp_avg.copy_(sd["exp_avg"]); self.exp_avg_sq.copy_(sd["exp_avg_sq"])
            self.flat_param[self.shard_lo:self.shard_hi].copy_(self.master.to(self.flat_param.dtype))
            if self.zero1:
                self._gather_params()
        self.step_count = int(sd["step"])
        self.lr = float(sd["lr"])
        if self.dyn is not None:
            self.dyn[0:1].fill_(self.lr); self.dyn[1:2].fill_(float(self.step_count))

    def _gather_params(self):
        shard = self.flat_param[self.shard_lo:self.shard_hi]
        dist.all_gather_into_tensor(self.flat_param, shard, group=self.pg)

    def grad_norm(self):
        """Global L2 norm of the (already summed) gradient, scaled to the mean over ranks — device scalar."""
        return torch.linalg.vector_norm(self.flat_grad, dtype=torch.float32) * (1.0 / self.world)

    def step(self):
        """Reduce gradients, clip (global norm), AdamW.  lr and the step counter live in a device
        float[2] (`self.dyn`), so the whole step can sit inside one captured CUDA graph.
        With check_finite the step is skipped on every rank when the reduced gradient has a NaN/Inf
        (the reference aborts on a non-finite loss after an all-reduce vote: engine_for_pretraining.py:151-161;
        the gradient norm is already global here, so no extra collective and no host sync is needed)."""
        from . import lowlevel as ll
        if self.step_count == 0:
            self.check_aliases()          # model.zero_grad(set_to_none=True) before the first step would unhook the sink
        self.reduce_gradients()
        self.step_count += 1
        if self.dyn is None:
            self.dyn = torch.tensor([self.lr, float(self.step_count - 1)], device=self.flat_grad.device, dtype=torch.float32)
        self.dyn[1:2].add_(1.0)
        inv_world = 1.0 / self.world
        coef = None
        if (self.clip_grad and self.clip_grad > 0) or self.check_finite:
            gn = self.grad_norm()
            clip = self.clip_grad if (self.clip_grad and self.clip_grad > 0) else float("inf")
            coef = torch.clamp(clip / (gn + 1e-6), max=1.0).reshape(1)
            if self.check_finite:
                # a NaN/Inf norm makes coef NaN/0: the AdamW kernel leaves all state untouched for such a scale
                self.skipped = (~torch.isfinite(gn)).float().reshape(1)
                self.dyn[1:2].sub_(self.skipped)             # a skipped step does not advance bias correction
            coef = coef.contiguous()
        b1, b2 = self.betas
        lo_s, hi_s = self.shard_lo, min(self.shard_hi, self.total)
        for lo, hi, wd in ((0, self.n_decay, self.wd), (self.n_decay, self.total, 0.0)):
            lo, hi = max(lo, lo_s), min(hi, hi_s)
            if hi > lo:
                a, b = lo - lo_s, hi - lo_s
                ll.adamw_step(self.master[a:b], self.exp_avg[a:b], self.exp_avg_sq[a:b],
                              self.flat_grad[lo:hi], self.flat_param[lo:hi], self.lr, b1, b2, self.eps, wd,
                              self.step_count, grad_scale=inv_world, grad_scale_dev=coef, dyn_lr_step=self.dyn)
        if self.zero1:
            self._gather_params()

    def replica_divergence(self):
        """max |param - rank 0's param| over ranks (device scalar, 0 when replicas are bit-identical)."""
        if self.world == 1:
            return torch.zeros((), device=self.flat_param.device)
        worst = torch.zeros((), device=self.flat_param.device, dtype=torch.float32)
        step = 1 << 27
        for lo in range(0, self.total, step):
            mine = self.flat_param[lo:min(lo + step, self.total)]
            ref = mine.clone()
            dist.broadcast(ref, src=dist.get_global_rank(self.pg, 0) if self.pg is not None else 0, group=self.pg)
            worst = torch.maximum(worst, (mine.float() - ref.float()).abs().max())
        dist.all_reduce(worst, op=dist.ReduceOp.MAX, group=self.pg)
        return worst


class GraphedStep:
    """Capture `fn(*static_inputs) -> loss` (forward + backward + engine.step) into ONE CUDA graph.

    The training step issues ~5 000 kernel launches; replaying them from a graph removes the Python /
    ctypes / autograd issue cost from the critical path (the GPU finishes the small row kernels faster
    than the host can enqueue them).  Inputs are copied into static device buffers before each replay;
    TMA tensor maps are encoded at capture time and stay valid because the graph's private memory pool
    pins every activation address."""

    def __init__(self, fn, static_inputs, warmup=3):
        self.static_inputs = list(static_inputs)
        self.fn = fn
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                loss = fn(*self.static_inputs)
                del loss                  # drop the autograd graph: stale AccumulateGrad nodes keep their old stream
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            loss = fn(*self.static_inputs)
            self.static_loss = loss.detach().float().reshape(1).clone()
            del loss

    def __call__(self, *inputs):
        for dst, src in zip(self.static_inputs, inputs):
            if src is not dst:
                dst.copy_(src, non_blocking=True)
        self.graph.replay()
        return self.static_loss
