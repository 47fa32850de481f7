"""The step around forward/backward: gradient exchange, clipping, optimiser and EMA (SURVEY §8e, §8f row 1).

Reference call sites (e2_tts_pytorch/trainer.py of the original project): DDP gradient all-reduce :155-162/:270, `clip_grad_norm_` :272-273,
`Adopt(model.parameters(), lr=...)` :183 + `optimizer.step()` :275, `EMA(model, include_online_model=False)` :170-174 + `.update()`
:279. Here they are three launches over flat fp32 buffers:

    GradSync()      b200_flat_gather  every p.grad (x 1/world) -> ONE contiguous buffer, then ONE ncclAllReduce (no bucket hooks)
    .accumulate()   b200_flat_accumulate  buffer += p.grad x 1/(steps*world) per micro-batch (grad_accumulation_steps, :142/:160/:250)
    FusedAdoptEMA   b200_sumsq        global gradient norm^2 of that buffer
                    b200_adopt_step   clip + Adopt + EMA in one pass

Parameters remain the model's ordinary fp32 nn.Parameters (state_dict compatible); gradient / m / v / EMA storage is flat and owned
here. `Adopt` and `EMA` are third-party packages that are not vendored with the original project: their update rules are restated in
oracle/optim_oracle.py (test infrastructure) and this module is checked against that restatement.
"""
from __future__ import annotations

import numpy as np
import torch

from . import lib

F32 = torch.float32
CHUNK = 16384   # elements per chunk-table entry (one CTA each); parameter offsets are padded to 4 elements (16-byte vector path)
_CHUNK_DT = np.dtype([('ptr', '<u8'), ('off', '<i8'), ('n', '<i4'), ('pidx', '<i4')])
assert _CHUNK_DT.itemsize == 24


def _stream():
    return torch.cuda.current_stream().cuda_stream


class FlatLayout:
    """Offsets of a parameter list inside flat fp32 buffers + chunk tables (include/b200_e2tts.h: b200_chunk)."""

    def __init__(self, params):
        self.params = [p for p in params]
        assert self.params, 'no parameters'
        self.device = self.params[0].device
        for p in self.params:
            assert p.dtype == F32 and p.is_contiguous() and p.device == self.device, 'flat layout needs contiguous fp32 parameters on one device'
        self.numels = [p.numel() for p in self.params]
        self.offsets, o = [], 0
        for n in self.numels:
            self.offsets.append(o)
            o += (n + 3) // 4 * 4
        self.total = o
        # per-chunk (parameter index, element start, length) — pointer-independent part of every table
        pidx, start, length = [], [], []
        for i, n in enumerate(self.numels):
            s = np.arange(0, max(n, 1), CHUNK, dtype=np.int64)[: (n + CHUNK - 1) // CHUNK]
            pidx.append(np.full(s.shape, i, dtype=np.int64))
            start.append(s)
            length.append(np.minimum(CHUNK, n - s))
        self._pidx, self._start, self._len = np.concatenate(pidx), np.concatenate(start), np.concatenate(length)
        self._off = np.asarray(self.offsets, dtype=np.int64)[self._pidx] + self._start
        self.n_chunks = int(self._pidx.shape[0])
        self._cache = {}
        self.param_table = self.table([p.data for p in self.params])

    def table(self, tensors):
        """Device chunk table whose `ptr`s point into `tensors` (same shapes as the parameters; None -> NULL). Cached per pointer set."""
        ptrs = tuple(0 if t is None else t.data_ptr() for t in tensors)
        hit = self._cache.get(ptrs)
        if hit is not None:
            return hit
        for t, n in zip(tensors, self.numels):
            assert t is None or (t.dtype == F32 and t.is_contiguous() and t.numel() == n), 'gradient layout differs from its parameter'
        base = np.asarray(ptrs, dtype=np.uint64)[self._pidx]
        arr = np.empty(self.n_chunks, dtype=_CHUNK_DT)
        arr['ptr'] = np.where(base != 0, base + (self._start * 4).astype(np.uint64), 0)
        arr['off'], arr['n'], arr['pidx'] = self._off, self._len, self._pidx
        dev = torch.from_numpy(arr.view(np.uint8).copy()).to(self.device)
        if len(self._cache) > 8:
            self._cache.clear()
        self._cache[ptrs] = dev
        return dev

    def views(self, flat):
        return [flat[o:o + n].view_as(p) for o, n, p in zip(self.offsets, self.numels, self.params)]


def broadcast_module(module, src=0, process_group=None):
    """Make every rank start from rank `src`'s parameters AND buffers — what DistributedDataParallel does when it wraps a module
    (trainer.py:155-162 via accelerate). Needed because part of the reference's initialisation is rank dependent: the
    hyper-connections pick their initial stream with python's `randrange` (SURVEY A.5) and RandomFourierEmbed draws its
    frequencies with torch.randn (e2_tts.py:358), so replicas seeded only through torch.manual_seed are NOT identical."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(process_group) == 1:
        return
    with torch.no_grad():
        for t in list(module.parameters()) + list(module.buffers()):
            dist.broadcast(t.data, src=src, group=process_group)


class GradSync:
    """Data-parallel gradient exchange for one replica per GPU (SURVEY §8e): after `loss.backward()` every parameter gradient is
    gathered (x 1/world, one launch) into ONE flat buffer which is all-reduced (SUM) with a single NCCL call; `p.grad` then becomes a
    view of that buffer. Equivalent to DDP's bucketed mean all-reduce (trainer.py:155-162, :270) including parameters that received no
    gradient on this rank (zeros, `find_unused_parameters=True`), without per-bucket copies, autograd hooks, or NCCL kernels competing
    with the persistent compute kernels for SMs during backward. world_size 1 (or `process_group=None` with torch.distributed
    uninitialised) only flattens — useful for the fused optimiser."""

    def __init__(self, params, process_group=None):
        import torch.distributed as dist
        self.layout = FlatLayout(params)
        self.group = process_group
        self.world = dist.get_world_size(process_group) if dist.is_available() and dist.is_initialized() else 1
        # [gradients (layout.total) | used flags (one per parameter)] in ONE buffer: a single all-reduce moves both
        n_par = len(self.layout.params)
        self._buf = torch.zeros(self.layout.total + (n_par + 3) // 4 * 4, device=self.layout.device, dtype=F32)
        self.flat = self._buf[:self.layout.total]
        self.used = self._buf[self.layout.total:self.layout.total + n_par]
        self.grad_views = self.layout.views(self.flat)

    def gather(self, table=None):
        """Enqueue the gather of the CURRENT p.grad tensors. Under stream capture pass a preallocated `table` (new_table()): the
        launch is recorded against it and the caller fills it with fill_table() once the capture has ended (building a table is a
        host-to-device copy, which a capturing stream cannot take; the kernel only reads it when the graph is replayed).
        Returns the gradient tensors the table (will) point at."""
        lay = self.layout
        grads = [p.grad for p in lay.params]
        for g, v in zip(grads, self.grad_views):
            if g is not None and g.data_ptr() == v.data_ptr():
                raise RuntimeError('GradSync.gather: p.grad already is the flat view (gather twice without a backward in between?)')
        lib.call('b200_flat_gather', table if table is not None else lay.table(grads), lay.n_chunks, self.flat, 1.0 / self.world, self.used, _stream())
        return grads

    def accumulate(self, table=None, scale=1.0):
        """The accumulating twin of gather(): flat += scale * p.grad (one fmaf per element), `used` ORed with this micro-step's
        presence flags; a parameter without a gradient keeps its slot. scale = 1 / (steps * world) for accelerate's `loss / steps`
        plus DDP's average. Clear the buffer with zero() at the start of each accumulation window. Same `table` rule as gather()."""
        lay = self.layout
        grads = [p.grad for p in lay.params]
        for g, v in zip(grads, self.grad_views):
            if g is not None and g.data_ptr() == v.data_ptr():
                raise RuntimeError('GradSync.accumulate: p.grad is the flat view itself (attach() ran without a backward in between?)')
        lib.call('b200_flat_accumulate', table if table is not None else lay.table(grads), lay.n_chunks, self.flat, float(scale), self.used,
                 _stream())
        return grads

    def zero(self):
        """Clear the gradients and the `used` flags (one memset over the shared buffer)."""
        self._buf.zero_()

    def new_table(self):
        return torch.zeros(self.layout.n_chunks * _CHUNK_DT.itemsize, device=self.layout.device, dtype=torch.uint8)

    def fill_table(self, table, grads):
        table.copy_(self.layout.table(grads))

    def all_reduce(self):
        if self.world > 1:
            import torch.distributed as dist
            dist.all_reduce(self._buf, op=dist.ReduceOp.SUM, group=self.group)

    def attach(self):
        """p.grad = view of the reduced buffer (zeros for a parameter no rank used; FusedAdoptEMA skips those through `used`)"""
        for p, v in zip(self.layout.params, self.grad_views):
            p.grad = v

    def __call__(self):
        self.gather()
        self.all_reduce()
        self.attach()
        return self.flat


class FusedAdoptEMA:
    """`Adopt` (adam-atan2-pytorch, trainer.py:183,275) + `clip_grad_norm_` (:272-273) + `EMA.update` (ema-pytorch, :170-174,:279)
    as ONE kernel pass per step over flat state. `step(flat_grads)` takes the flat gradient buffer of a GradSync built over the
    same parameter list (or gathers p.grad itself). EMA follows ema-pytorch's defaults: copy until `update_after_step`, then every
    `update_every` steps  ema += (1 - decay) (w - ema),  decay = clamp(1 - (1 + epoch/inv_gamma)^-power, min_value, beta)."""

    def __init__(self, params, lr=1e-4, betas=(0.9, 0.99), eps=1e-6, weight_decay=0., decoupled_wd=True, max_grad_norm=0.,
                 ema=False, ema_beta=0.9999, ema_update_after_step=100, ema_update_every=10, ema_inv_gamma=1.0, ema_power=2. / 3.,
                 ema_min_value=0.0, grad_sync: GradSync | None = None):
        self.sync = grad_sync if grad_sync is not None else GradSync(params)
        self.layout = self.sync.layout
        dev, n = self.layout.device, self.layout.total
        self.lr, self.init_lr, self.betas, self.eps = lr, lr, betas, eps
        self.weight_decay, self.decoupled_wd, self.max_grad_norm = weight_decay, decoupled_wd, max_grad_norm
        self.m = torch.zeros(n, device=dev, dtype=F32)
        self.v = torch.zeros(n, device=dev, dtype=F32)
        self.steps = 0
        self.chunk_state = torch.zeros(self.layout.n_chunks, device=dev, dtype=torch.int32)   # 0 = this piece has no Adopt state yet
        self.norm_sq = torch.zeros(1, device=dev, dtype=F32)
        self.ema = torch.zeros(n, device=dev, dtype=F32) if ema else None
        self.ema_cfg = dict(beta=ema_beta, update_after_step=ema_update_after_step, update_every=ema_update_every, inv_gamma=ema_inv_gamma,
                            power=ema_power, min_value=ema_min_value)
        self.ema_step, self.ema_initted = 0, False

    # ---- ema-pytorch's schedule (EMA.update / get_current_decay)
    def _ema_action(self):
        """-> (mode, weight) for THIS optimiser step: 0 none, 1 lerp with weight 1 - decay, 2 copy"""
        if self.ema is None:
            return 0, 0.0
        c = self.ema_cfg
        step = self.ema_step
        self.ema_step += 1
        if step % c['update_every'] != 0:
            return 0, 0.0
        if step <= c['update_after_step'] or not self.ema_initted:
            self.ema_initted = self.ema_initted or step > c['update_after_step']
            return 2, 0.0
        epoch = max(step - c['update_after_step'], 0)   # ema-pytorch evaluates the decay after incrementing its step counter
        decay = 0.0 if epoch <= 0 else min(max(1.0 - (1.0 + epoch / c['inv_gamma']) ** -c['power'], c['min_value']), c['beta'])
        return 1, 1.0 - decay

    @torch.no_grad()
    def step(self, flat_grads=None):
        """One optimiser step. `flat_grads` = GradSync.flat (already reduced); None -> gather the current p.grad first."""
        if flat_grads is None:
            flat_grads = self.sync()
        lay = self.layout
        clip = self.max_grad_norm > 0
        if clip:
            lib.call('b200_sumsq', flat_grads, lay.total, self.norm_sq, _stream())
        wd = self.weight_decay / self.init_lr if (self.decoupled_wd and self.weight_decay > 0) else self.weight_decay
        mode, weight = self._ema_action()
        a = lib.make_args('b200_adopt_args', chunks_dev=lay.param_table, n_chunks=lay.n_chunks, grad_flat=flat_grads, m_flat=self.m, v_flat=self.v,
                          ema_flat=self.ema, gradnorm_sq=self.norm_sq if clip else None, max_grad_norm=float(self.max_grad_norm), lr=float(self.lr),
                          beta1=float(self.betas[0]), beta2=float(self.betas[1]), eps=float(self.eps), weight_decay=float(wd), chunk_state=self.chunk_state,
                          ema_mode=int(mode), ema_weight=float(weight), used=self.sync.used if flat_grads is self.sync.flat else None,
                          one_minus_beta1=float(1.0 - self.betas[0]), one_minus_beta2=float(1.0 - self.betas[1]))
        lib.call('b200_adopt_step', a, _stream())
        self.steps += 1

    def grad_norm(self):
        """total gradient norm seen by the last clipped step (device tensor; what clip_grad_norm_ returns)"""
        return self.norm_sq.sqrt()

    def zero_grad(self, set_to_none=True):
        for p in self.layout.params:
            if set_to_none:
                p.grad = None
            elif p.grad is not None:
                p.grad.zero_()

    def ema_parameters(self):
        """views of the EMA weights shaped like the parameters (ema-pytorch: ema_model.parameters())"""
        return self.layout.views(self.ema)

    @torch.no_grad()
    def copy_ema_to(self, module_params):
        """write the EMA weights into another module's parameters (same order/shapes), e.g. a deepcopy used for sampling or as
        the `velocity_consistency_model` (trainer.py:259-268)"""
        other = FlatLayout(list(module_params))
        assert other.numels == self.layout.numels
        lib.call('b200_flat_scatter', other.param_table, other.n_chunks, self.ema, _stream())

    def state_dict(self):
        return dict(steps=self.steps, chunk_state=self.chunk_state, m=self.m, v=self.v, ema=self.ema, ema_step=self.ema_step, ema_initted=self.ema_initted, lr=self.lr)

    def load_state_dict(self, sd):
        self.steps, self.ema_step, self.ema_initted, self.lr = sd['steps'], sd['ema_step'], sd['ema_initted'], sd['lr']
        self.chunk_state.copy_(sd['chunk_state'])
        self.m.copy_(sd['m'])
        self.v.copy_(sd['v'])
        if self.ema is not None and sd.get('ema') is not None:
            self.ema.copy_(sd['ema'])
