"""world_size-2 gloo tests (CPU) of the host-side distributed logic: flat-buffer layout/bucketing,
hook-driven bucketed gradient all-reduce, and the packed embedding all-gather (rank order, bit-exact idx,
local-rows-only gradient — AllGather semantics of multi_modality/models/utils.py:193-212)."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from internvideo_b200 import engine as eng


def test_layout_and_buckets():
    shapes = [("a.weight", (10, 7)), ("a.bias", (10,)), ("pos_embed", (1, 5, 8)), ("b.weight", (33, 3)), ("g.gamma", (9,))]
    entries, n_decay, total = eng.plan_layout(shapes, {"pos_embed"})
    by = {e[0]: e for e in entries}
    assert by["a.weight"][3] and by["b.weight"][3]
    assert not by["a.bias"][3] and not by["pos_embed"][3] and not by["g.gamma"][3]
    for name, off, numel, decay in entries:
        assert off % eng.ALIGN == 0
        assert (off < n_decay) == decay
    offs = sorted((e[1], e[1] + e[2]) for e in entries)
    assert all(a[1] <= b[0] for a, b in zip(offs, offs[1:])) and offs[-1][1] <= total
    buckets, owner = eng.plan_buckets(entries, total, 64)
    assert sum(b.total for b in buckets) == len(entries)
    assert buckets[0].start == 0 and buckets[-1].end == total
    for name, off, numel, _ in entries:
        assert buckets[owner[name]].start <= off < buckets[owner[name]].end
        # an entry never straddles two buckets: a bucket is reduced when ITS entries are complete, and backward
        # writes the tail of an earlier-layer tensor after the later layers that share the bucket
        assert off + numel <= buckets[owner[name]].end, name
    assert all(a.end == b.start for a, b in zip(buckets, buckets[1:]))
    # geometric schedule + forced boundary at the decay / no-decay border (the no-decay section completes last)
    bk3, own3 = eng.plan_buckets(entries, total, 10 ** 9, first_elems=16, split_at=n_decay)
    assert any(b.end == n_decay for b in bk3) and sum(b.total for b in bk3) == len(entries)
    assert all(a.end == b.start for a, b in zip(bk3, bk3[1:])) and bk3[-1].end == total
    for name, off, numel, decay in entries:
        assert (bk3[own3[name]].end <= n_decay) == decay, name
    # a tensor larger than the bucket size gets a bucket of its own instead of being split
    big, _, tot2 = eng.plan_layout([("w0", (100, 10)), ("w1", (7, 3)), ("b0", (5,))])
    bk, own = eng.plan_buckets(big, tot2, 64)
    assert bk[own["w0"]].end - bk[own["w0"]].start >= 1000


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.manual_seed(rank)           # replicas start DIFFERENT: the engine broadcasts rank 0's parameters (DDP semantics)
    model = nn.Sequential(nn.Linear(16, 24), nn.Linear(24, 8)).to(torch.bfloat16)
    e = eng.PretrainEngine(model, clip_grad=0.0, bucket_mb=0.0002, overlap=True)
    assert len(e.buckets) > 1
    torch.manual_seed(0)
    ref0 = nn.Sequential(nn.Linear(16, 24), nn.Linear(24, 8)).to(torch.bfloat16)
    for p_, r_ in zip(model.parameters(), ref0.parameters()):
        assert torch.equal(p_.data, r_.data)
    assert torch.equal(e.master, e.flat_param.float())
    # parameters now alias the flat buffer
    assert model[0].weight.data_ptr() >= e.flat_param.data_ptr()
    e.zero_grad()
    x = torch.full((4, 16), float(rank + 1), dtype=torch.bfloat16)
    model(x).float().sum().backward()
    e.reduce_gradients()
    q.put(("grad", rank, e.flat_grad.float().numpy().copy()))
    # ---- same step, but layer 0 uses the gradient-sink protocol (what ops.BlockFn does on the GPU): its backward
    # accumulates straight into the flat gradient, calls engine.grad_written(p) and returns None for the parameter,
    # while layer 1 still goes through autograd's post-accumulate hooks.  Buckets must complete all the same.
    class SinkLinear(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, w, b):
            ctx.save_for_backward(x, w)
            ctx.params = (w, b)
            return x @ w.t() + b

        @staticmethod
        def backward(ctx, dy):
            x, w = ctx.saved_tensors
            pw, pb = ctx.params
            sink = pw._ivb_sink
            pw.grad.add_((dy.float().t() @ x.float()).to(pw.grad.dtype)); sink.grad_written(pw)
            pb.grad.add_(dy.float().sum(0).to(pb.grad.dtype)); sink.grad_written(pb)
            return dy @ w, None, None

    e.zero_grad()
    h = SinkLinear.apply(x, model[0].weight, model[0].bias)
    model[1](h).float().sum().backward()
    assert any(b.handle is not None for b in e.buckets)      # buckets fired during backward, not only at the end
    e.reduce_gradients()
    q.put(("grad_sink", rank, e.flat_grad.float().numpy().copy()))
    # ---- three sink layers whose weights share ONE bucket, rank-specific inputs.  autograd fires the
    # post-accumulate hook even for the `None` gradients the sink returns; counting those echoes as arrivals
    # (round-1 bug) hands the bucket to the collective before the first layer's gradient is written.
    torch.manual_seed(5)
    chain = nn.Sequential(nn.Linear(8, 8), nn.Linear(8, 8), nn.Linear(8, 8)).to(torch.bfloat16)
    e3 = eng.PretrainEngine(chain, clip_grad=0.0, bucket_mb=1.0, overlap=True)
    assert len(e3.buckets) == 2 and e3.buckets[0].total == 3      # the three weights share a bucket; the biases (no-decay) have their own
    xr = (torch.arange(16, dtype=torch.float32).reshape(2, 8) * 0.125 + rank).to(torch.bfloat16)

    def chain_fwd():
        h3 = xr
        for lyr in chain:
            h3 = SinkLinear.apply(h3, lyr.weight, lyr.bias)
        return h3.float().sum()
    e3.zero_grad()
    chain_fwd().backward()
    assert all(b.launched for b in e3.buckets) and not e3._sunk   # launched by the LAST arrival, every echo dropped
    e3.reduce_gradients()
    q.put(("chain", rank, e3.flat_grad.float().numpy().copy()))
    # local (unreduced) gradient of this rank for the parent's exact check
    e3.overlap = False
    e3.zero_grad(); chain_fwd().backward()
    q.put(("chain_local", rank, e3.flat_grad.float().numpy().copy()))
    e3.overlap = True
    # a second backward between zero_grad() and step() must raise, not silently land in a reduced bucket ...
    e3.zero_grad(); chain_fwd().backward()
    try:
        chain_fwd().backward()
        raised = False
    except RuntimeError as ex:
        raised = "after it was handed to NCCL" in str(ex)
    # ... unless it is declared as accumulation: then nothing is reduced until reduce_gradients()
    e3.zero_grad()
    with e3.accumulate():
        chain_fwd().backward(); chain_fwd().backward()
        assert not any(b.launched for b in e3.buckets)
    e3.reduce_gradients()
    q.put(("accum", rank, raised, e3.flat_grad.float().numpy().copy()))
    # ---- ZeRO-1: sharded optimizer state, in-place parameter all-gather, checkpoint round trip.  The AdamW
    # kernel is CUDA-only; the host logic is exercised with a torch stand-in of the same signature.
    from internvideo_b200 import lowlevel as ll_

    def adamw_torch(master, m, v, grad, param, lr, b1, b2, eps, wd, step, grad_scale=1.0, grad_scale_dev=None, dyn_lr_step=None):
        g = grad.float() * grad_scale * (float(grad_scale_dev) if grad_scale_dev is not None else 1.0)
        t = float(dyn_lr_step[1]); lr_ = float(dyn_lr_step[0])
        master.mul_(1 - lr_ * wd); m.mul_(b1).add_(g, alpha=1 - b1); v.mul_(b2).addcmul_(g, g, value=1 - b2)
        master.sub_(lr_ * (m / (1 - b1 ** t)) / ((v / (1 - b2 ** t)).sqrt() + eps))
        param.copy_(master.to(param.dtype))
    ll_.adamw_step = adamw_torch
    outs = {}
    for z1 in (False, True):
        torch.manual_seed(9)
        mz = nn.Sequential(nn.Linear(16, 24), nn.Linear(24, 8)).to(torch.bfloat16)
        ez = eng.PretrainEngine(mz, clip_grad=1.0, bucket_mb=0.0002, overlap=True, zero1=z1, lr=1e-2)
        if z1:
            assert ez.master.numel() == ez.shard_len < ez.total and ez.flat_param.numel() == ez.padded
        for it in range(3):
            ez.zero_grad()
            mz(torch.full((4, 16), float(rank + 1 + it), dtype=torch.bfloat16)).float().pow(2).sum().backward()
            ez.step()
            if z1 and it == 1:
                saved = ez.state_dict()
                params_then = ez.flat_param.clone()
        outs[z1] = ez.flat_param[:ez.total].float().clone()
    # resume: reload the step-2 optimizer state into the live engine, redo step 3 -> same parameters
    ez.load_state_dict(saved)
    assert torch.equal(ez.flat_param, params_then) and ez.step_count == 2
    ez.zero_grad()
    mz(torch.full((4, 16), float(rank + 3), dtype=torch.bfloat16)).float().pow(2).sum().backward()
    ez.step()
    q.put(("zero1", rank, outs[False].numpy().copy(), outs[True].numpy().copy(), ez.flat_param[:ez.total].float().numpy().copy()))
    # ---- packed embedding gather
    from internvideo_b200 import contrastive as c
    g = torch.Generator().manual_seed(10 + rank)
    v = torch.randn(4, 8, generator=g, requires_grad=True); t = torch.randn(4, 8, generator=g, requires_grad=True)
    idx = torch.tensor([2 ** 40 + rank, 7, 123456789012 + rank, rank], dtype=torch.int64)
    v_all, t_all, idx_all, r, bl = c.gather_embeddings(v, t, idx)
    (v_all.sum() * (rank + 1) + t_all.sum()).backward()
    q.put(("gather", rank, v_all.detach().numpy().copy(), idx_all.numpy().copy(), v.grad.numpy().copy(), r, bl))
    dist.barrier()
    dist.destroy_process_group()


def _free_port():
    """A port nobody listens on right now (a fixed one can still be in TIME_WAIT from the previous run of the suite)."""
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_two_rank_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in ps]
    res = [q.get(timeout=180) for _ in range(14)]
    [p.join(timeout=60) for p in ps]
    T = torch.from_numpy
    grads = {r[1]: T(r[2]) for r in res if r[0] == "grad"}
    gath = {r[1]: (r[0], r[1], T(r[2]), T(r[3]), T(r[4]), r[5], r[6]) for r in res if r[0] == "gather"}
    # all-reduce(sum): both ranks hold the same reduced gradient, equal to the sum of the two local ones
    assert torch.equal(grads[0], grads[1])
    torch.manual_seed(0)
    ref = nn.Sequential(nn.Linear(16, 24), nn.Linear(24, 8)).to(torch.bfloat16)
    tot = None
    for rank in range(2):
        ref.zero_grad()
        ref(torch.full((4, 16), float(rank + 1), dtype=torch.bfloat16)).float().sum().backward()
        gl = [p.grad.float().reshape(-1) for p in ref.parameters()]
        tot = gl if tot is None else [a + b for a, b in zip(tot, gl)]
    # layout: weights (decay) first, then biases
    names = [n for n, _ in ref.named_parameters()]
    order = [i for i, n in enumerate(names) if n.endswith("weight")] + [i for i, n in enumerate(names) if n.endswith("bias")]
    flat_ref = torch.cat([tot[i] for i in order])
    nz = grads[0][grads[0] != 0]
    assert torch.allclose(nz, flat_ref[flat_ref != 0], rtol=2e-2)
    # gradient-sink protocol mixed with autograd hooks: identical reduced gradient
    gs = {r[1]: T(r[2]) for r in res if r[0] == "grad_sink"}
    assert torch.equal(gs[0], gs[1])
    assert torch.allclose(gs[0], grads[0], rtol=2e-2, atol=1e-3)
    # sink-only chain in one bucket: reduced gradient == sum of the two local gradients, bit for bit, on both ranks
    ch = {r[1]: T(r[2]) for r in res if r[0] == "chain"}
    loc = {r[1]: T(r[2]) for r in res if r[0] == "chain_local"}
    assert torch.equal(ch[0], ch[1])
    assert torch.equal(ch[0], (loc[0].bfloat16() + loc[1].bfloat16()).float())
    acc = {r[1]: (r[2], T(r[3])) for r in res if r[0] == "accum"}
    assert acc[0][0] and acc[1][0]                                   # un-declared second backward raised
    assert torch.equal(acc[0][1], acc[1][1])
    assert torch.allclose(acc[0][1], 2 * ch[0], rtol=2e-2, atol=1e-3)  # two micro-batches accumulated, then reduced
    # ZeRO-1 == unsharded AdamW, identical on both ranks, and resumable from its state_dict
    z = {r[1]: (T(r[2]), T(r[3]), T(r[4])) for r in res if r[0] == "zero1"}
    assert torch.equal(z[0][0], z[1][0]) and torch.equal(z[0][1], z[1][1])
    assert torch.equal(z[0][0], z[0][1])
    assert torch.equal(z[0][2], z[0][1]) and torch.equal(z[1][2], z[0][1])
    # gather: rank order, bit-exact int64 idx, local-slice backward
    v0, v1 = gath[0][2], gath[1][2]
    assert torch.equal(v0, v1) and v0.shape == (8, 8)
    assert torch.equal(gath[0][3], gath[1][3])
    assert gath[0][3].tolist() == [2 ** 40, 7, 123456789012, 0, 2 ** 40 + 1, 7, 123456789013, 1]
    assert torch.equal(gath[0][4], torch.ones(4, 8)) and torch.equal(gath[1][4], 2 * torch.ones(4, 8))
    assert (gath[0][5], gath[0][6]) == (0, 4) and (gath[1][5], gath[1][6]) == (1, 4)


def test_gradient_sink_planning_cpu():
    """ops.BlockFn's gradient sink (host logic only): the O(D) gradients of a block are planned at their
    parameters' relative offsets inside the engine's flat gradient, so ONE add lands them; the engine's
    grad_written() does the bucket bookkeeping autograd's post-accumulate hook does for other parameters."""
    from internvideo_b200 import ops

    class Blk(torch.nn.Module):
        def __init__(self, D=16, Hd=32):
            super().__init__()
            P = lambda *s: torch.nn.Parameter(torch.zeros(*s, dtype=torch.bfloat16))
            self.n1w, self.qkvw, self.qnw, self.knw = P(D), P(3 * D, D), P(D), P(D)
            self.projw, self.projb, self.g1, self.n2w = P(D, D), P(D), P(D), P(D)
            self.fc1w, self.fc1b, self.fc2w, self.fc2b, self.g2 = P(Hd, D), P(Hd), P(D, Hd), P(D), P(D)

    D, Hd = 16, 32
    m = Blk(D, Hd)
    e = eng.PretrainEngine(m, clip_grad=0.0, bucket_mb=0.0002, overlap=False)
    params = (m.n1w, m.qkvw, None, m.qnw, m.knw, m.projw, m.projb, m.g1, m.n2w, m.fc1w, m.fc1b, m.fc2w, m.fc2b, m.g2)
    sink = ops._common_sink(params)
    assert sink is e
    small = (("g2", m.g2, D), ("fc2b", m.fc2b, D), ("n2w", m.n2w, D), ("g1", m.g1, D), ("projb", m.projb, D),
             ("qnw", m.qnw, D), ("knw", m.knw, D), ("n1w", m.n1w, D), ("fc1b", m.fc1b, Hd), ("qkvb", None, 3 * D))
    seg, vec, span, base = ops._plan_small(small, sink, torch.device("cpu"))
    assert span is not None and vec.dtype == torch.float32
    # every present parameter's segment sits at its flat-buffer offset relative to `base`
    for j, (name, p, sz) in enumerate(small):
        if p is None:
            assert seg[name].numel() == sz          # scratch past the span (kernels still need the buffer)
            continue
        seg[name].fill_(float(j + 1))               # small integers: exact in bf16
    e.flat_grad[base:base + span].add_(vec[:span])
    for j, (name, p, sz) in enumerate(small):
        if p is not None:
            assert torch.all(p.grad.float() == float(j + 1)), name
    # weights were not touched by the fused add
    assert float(m.qkvw.grad.float().abs().sum()) == 0.0
    # a parameter without a sink (or with direct_grads=False) disables the direct path
    e2 = eng.PretrainEngine(Blk(D, Hd), clip_grad=0.0, direct_grads=False)
    assert ops._common_sink(tuple(e2.model.parameters())) is None
    stray = torch.nn.Parameter(torch.zeros(D, dtype=torch.bfloat16))
    assert ops._common_sink(params + (stray,)) is None
    # without a sink the scratch is simply packed
    seg2, vec2, span2, _ = ops._plan_small(small, None, torch.device("cpu"))
    assert span2 is None and vec2.numel() == 8 * D + Hd + 3 * D
