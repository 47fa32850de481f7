"""One CUDA graph per training step: forward + backward of an E2TTS model captured once, replayed every step — on one GPU or as one
replica of a data-parallel job (one process per GPU).

The reference's training step (trainer.py:263-270: `loss, cond, pred = self.model(mel_spec, text=text_inputs, lens=mel_lengths)` then
`self.accelerator.backward(loss)`, gradients all-reduced by DDP) is ~800 kernel launches and ~180 autograd nodes here; on a slow host
the Python / driver side of that costs more than the GPU work. Capturing the step removes the host from the critical path. Per step:
  * the new batch is copied into the static input tensors (`mel`, optional `text` / `lens`) — shapes are fixed at capture time;
  * torch's graph-safe CUDA generator advances on every replay (noise x0, flow times, span masks);
  * dropout seeds are kernel ARGUMENTS and therefore frozen in the graph, so every seeded kernel also adds one DEVICE word
    (`seed_dev` in the args structs, include/b200_e2tts.h "dropout seeds") that the graph's first node (`b200_seed_advance`)
    steps in stream order — no host write, so replays may be enqueued back to back without racing on a pinned seed word;
  * with more than one rank (torch.distributed initialised, or `process_group=` given) the graph ends with ONE gather of all
    parameter gradients into a flat fp32 buffer (x 1/world) and the replay is followed by ONE ncclAllReduce of that buffer
    (optim.GradSync): the data-parallel exchange of SURVEY §8e without DDP's bucket hooks, which cannot be captured cheaply and
    whose NCCL kernels would compete with the persistent compute kernels for SMs all through backward;
  * with a velocity-consistency teacher (the EMA model, e2_tts.py:1556-1589) the teacher's no-grad pass at t + delta is captured
    ahead of the student's forward, through E2TTS.forward itself; its weights are packed from its parameters on every replay.
Gradients are left in `param.grad` exactly as after `loss.backward()` (+ DDP's averaging when world > 1); run the optimiser after
the call (optim.FusedAdoptEMA takes `step.grad_sync.flat` directly). Do not keep an output of an earlier EAGER forward of the same
model alive while constructing this object: its autograd graph pins the parameters' AccumulateGrad nodes to the default (legacy)
stream, which cannot take part in a capture. `cond_drop_prob` must be 0 or 1 while captured (the text-drop coin is a Python-side
branch: it would be frozen either way).
"""
from __future__ import annotations

import random
import time

import torch

from . import lib
from .optim import GradSync, broadcast_module

MAX_BATCH = 64   # b200_small_linear's row limit (csrc/small.cu): the per-item conditioning GEMMs take at most 64 items


class _Loss:
    def __init__(self, loss):
        self.loss = loss


def _refuse_ddp_wrapper(model, who):
    if hasattr(model, 'module') and not hasattr(model, 'transformer'):
        raise ValueError(f'{who}: pass the bare E2TTS module, not a DistributedDataParallel wrapper '
                         '(gradients are averaged by one flat all-reduce after the replay)')


def _world(process_group):
    import torch.distributed as dist
    return dist.get_world_size(process_group) if dist.is_available() and dist.is_initialized() else 1


def _new_seed_word(model, dev):
    """the device seed word: every dropout seed of the step is `host seed + *seed_dev` (frozen host part, stepping device part)"""
    seed_dev = torch.randint(0, 2 ** 62, (1,), dtype=torch.int64).to(dev)
    model.transformer._seed_dev = seed_dev
    return seed_dev


def _geometry(model):
    """what a teacher must share with its student beyond the state_dict shapes: the stem layout and the attention geometry"""
    t = model.transformer
    return dict(concat_cond=model.concat_cond, num_channels=model.num_channels, heads=t.heads, dim_head=t.dim_head,
                text_heads=t.text_heads, text_dim_head=t.text_dim_head, softclamp=t.softclamp, num_residual_streams=t.num_streams)


class VelocityTeacher:
    """The velocity-consistency teacher of a graphed step (e2_tts.py:1556-1589; the reference trainer passes its EMA model,
    trainer.py:259-268): every refusal that must come before a launch, and the per-call check that the graph may still read it.

    The graph runs E2TTS.forward(velocity_consistency_model=teacher) as the eager step does, so its teacher pass packs the teacher's
    weights from the parameters' storage on every replay: an in-place update between replays (FusedAdoptEMA.copy_ema_to, ema-pytorch's
    EMA.update) is picked up, a parameter with new storage is refused. A teacher in training mode gets a device seed word of its own,
    stepped on every replay like the student's; its mode at construction is the one captured."""

    def __init__(self, model, teacher, delta, frames, who):
        from .modules import E2TTS
        self.who = who
        if not isinstance(model, E2TTS):
            raise ValueError(f'{who}: velocity_consistency_model is given for a {type(model).__name__}; only an E2TTS has the '
                             'velocity-consistency term')
        if not float(model.velocity_consistency_weight) > 0.0:
            raise ValueError(f'{who}: velocity_consistency_model is given but velocity_consistency_weight is '
                             f'{model.velocity_consistency_weight}, so the teacher would never be used')
        if not isinstance(teacher, E2TTS):
            raise ValueError(f'{who}: velocity_consistency_model must be an E2TTS (the EMA copy of the model), got {type(teacher).__name__}')
        if teacher is model:
            raise ValueError(f'{who}: velocity_consistency_model is the model itself; pass a separate copy (the EMA model)')
        mine, theirs = model.state_dict(), teacher.state_dict()
        if list(mine) != list(theirs) or any(mine[k].shape != theirs[k].shape for k in mine):
            diff = sorted(set(mine) ^ set(theirs)) or [k for k in mine if mine[k].shape != theirs[k].shape]
            raise ValueError(f'{who}: velocity_consistency_model is not of the model\'s architecture (state_dict differs at {diff[0]!r})')
        g_m, g_t = _geometry(model), _geometry(teacher)
        for k in g_m:
            if g_m[k] != g_t[k]:
                raise ValueError(f'{who}: velocity_consistency_model is not of the model\'s architecture ({k} {g_t[k]} != {g_m[k]})')
        dev_m, dev_t = next(model.parameters()).device, next(teacher.parameters()).device
        if dev_m != dev_t:
            raise ValueError(f'{who}: velocity_consistency_model lives on {dev_t}, the model on {dev_m}')
        if frames > teacher.transformer.max_seq_len:
            raise ValueError(f'{who}: {frames} frames exceed the velocity_consistency_model\'s max_seq_len ({teacher.transformer.max_seq_len})')
        self.model, self.delta = teacher, float(delta)
        self.seed_dev = None
        self._ptrs, self._training, self._keep = None, None, None

    def add_seed_word(self):
        """a device seed word for a teacher in training mode (none in eval mode: it draws no dropout seed)"""
        if self.model.training:
            self.seed_dev = _new_seed_word(self.model, next(self.model.parameters()).device)

    def seal(self):
        """after capture: the storage and mode the graph was recorded against. The teacher's derived state (weight pack, rotary
        tables) is held here too: the graph reads those buffers, and a `.to()` on the teacher would otherwise free them."""
        self._ptrs = tuple(p.data_ptr() for p in self.model.parameters())
        self._training = self.model.training
        from .modules import _PackOwner
        self._keep = [dict(m._derived) for m in self.model.modules() if isinstance(m, _PackOwner)]

    def check(self):
        if tuple(p.data_ptr() for p in self.model.parameters()) != self._ptrs:
            raise ValueError(f'{self.who}: a velocity_consistency_model parameter has new storage since capture (the graph reads the '
                             'old one); update the teacher in place (copy_ema_to, EMA.update) or build a new step')
        if self.model.training != self._training:
            raise ValueError(f'{self.who}: the velocity_consistency_model was captured in {"training" if self._training else "eval"} '
                             'mode; switch it back or build a new step')


def velocity_flag(teacher, velocity, who):
    """the velocity switch of one call: default on when the step has a teacher; raises before any launch"""
    v = (teacher is not None) if velocity is None else bool(velocity)
    if v and teacher is None:
        raise ValueError(f'{who}: velocity=True on a step built without velocity_consistency_model')
    if v:
        teacher.check()
    return v


def _train_pass(model, seed_dev, mel, text, lens, teacher=None):
    """one forward + backward as captured: the seed words step first, then the model's own training objective (with the
    velocity-consistency term of `teacher`, a VelocityTeacher, when given)"""
    stream = torch.cuda.current_stream().cuda_stream
    lib.call('b200_seed_advance', seed_dev, stream)
    if teacher is None:
        out = model(mel, text=text, lens=lens)
    else:
        if teacher.seed_dev is not None:
            lib.call('b200_seed_advance', teacher.seed_dev, stream)
        out = model(mel, text=text, lens=lens, velocity_consistency_model=teacher.model, velocity_consistency_delta=teacher.delta)
    if torch.is_tensor(out):       # DurationPredictor.forward returns the scalar loss itself (e2_tts.py:1113)
        out = _Loss(out)
    out.loss.backward()
    return out


def _clear_grads(model):
    for p in model.parameters():
        p.grad = None


class GraphedTrainStep:
    def __init__(self, model, mel, *, text=None, lens=None, warmup=3, process_group=None, flat_grads=None,
                 velocity_consistency_model=None, velocity_consistency_delta=1e-5):
        """model: an E2TTS or a DurationPredictor (NOT wrapped in DistributedDataParallel — the exchange is done here). flat_grads: True forces the flat
        gradient buffer even on one rank (for the fused optimiser); default = only when world_size > 1.
        velocity_consistency_model: the teacher of the velocity-consistency term (an E2TTS of the model's architecture, e.g. its EMA copy;
        the model needs velocity_consistency_weight > 0). Then two graphs are captured into one pool, with and without the teacher
        pass, and each call picks one with `velocity=` (default: with)."""
        _refuse_ddp_wrapper(model, 'GraphedTrainStep')
        self.teacher = None
        if velocity_consistency_model is not None:
            self.teacher = VelocityTeacher(model, velocity_consistency_model, velocity_consistency_delta, int(mel.shape[1]), 'GraphedTrainStep')
        if model.training and 0.0 < float(getattr(model, 'cond_drop_prob', 0.0)) < 1.0:
            raise ValueError('GraphedTrainStep: cond_drop_prob must be 0 or 1 (the text-drop branch is decided on the host)')
        if not mel.is_cuda:
            raise ValueError('GraphedTrainStep: inputs must live on the GPU')
        self.model = model
        dev = mel.device
        self.mel = mel.clone()
        self.text = text.clone() if torch.is_tensor(text) else (model.tokenizer(text).to(dev) if isinstance(text, list) else None)
        self.lens = lens.clone() if torch.is_tensor(lens) else None
        world = _world(process_group)
        if world > 1:
            broadcast_module(model, 0, process_group)    # replicas must start identical (DDP does this when it wraps the module)
            if self.teacher is not None:
                broadcast_module(self.teacher.model, 0, process_group)
        use_flat = (world > 1) if flat_grads is None else bool(flat_grads) or world > 1
        self.grad_sync = GradSync(list(model.parameters()), process_group) if use_flat else None
        self._seed_dev = _new_seed_word(model, dev)
        modes = (True, False) if self.teacher is not None else (False,)   # the teacher's graph first: it is the larger
        if self.teacher is not None:
            self.teacher.add_seed_word()
        cur = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):          # warm-up off the capture stream: lazy initialisation, allocator pools, packed weights
            for v in modes:
                for _ in range(max(1, warmup)):
                    self._eager(v)
                    self._clear_grads()
            if self.grad_sync is not None and world > 1:
                self.grad_sync.all_reduce()    # NCCL communicator / channel setup outside the timed path
        cur.wait_stream(side)
        torch.cuda.synchronize(dev)
        torch.cuda.empty_cache()   # the warm-up's side-stream blocks would sit beside the graph's private pool (a full set of activations each)
        pool = torch.cuda.graph_pool_handle() if len(modes) > 1 else None
        self.graphs, self.outs, self.launches, self._tables, self._grad_sets = {}, {}, {}, {}, {}
        for v in modes:
            self._clear_grads()      # each graph writes gradient tensors of its own (a backward into existing ones would add)
            graph = torch.cuda.CUDAGraph()
            table = self.grad_sync.new_table() if self.grad_sync is not None else None
            n0 = lib.launch_count()
            with torch.cuda.graph(graph, pool=pool):
                out = self._eager(v)
                if self.grad_sync is not None:
                    static_grads = self.grad_sync.gather(table)   # recorded against the (still empty) chunk table
            if self.grad_sync is not None:
                self.grad_sync.fill_table(table, static_grads)    # the graph's static gradient tensors, known only now
                self._tables[v] = table
            self.launches[v] = lib.launch_count() - n0   # kernel nodes of ours in the graph (they all run on every replay)
            # the gradient tensors the graph writes into: re-attached after every replay in case the training loop dropped them
            # (optimizer.zero_grad(set_to_none=True)); each replay OVERWRITES them, exactly like backward() into empty .grad fields
            self._grad_sets[v] = [(p, p.grad) for p in self.model.parameters() if p.grad is not None]
            self.graphs[v], self.outs[v] = graph, out
        if self.teacher is not None:
            self.teacher.seal()
        self.graph, self.out, self.launches_per_step = self.graphs[modes[0]], self.outs[modes[0]], self.launches[modes[0]]
        self._grads = self._grad_sets[modes[0]]
        if self.grad_sync is not None:
            self._table = self._tables[modes[0]]
            self.grad_sync.attach()
        else:
            self._attach(self._grads)

    def _eager(self, velocity=False):
        return _train_pass(self.model, self._seed_dev, self.mel, self.text, self.lens, self.teacher if velocity else None)

    def _clear_grads(self):
        _clear_grads(self.model)

    @staticmethod
    def _attach(grads):
        for p, g in grads:
            if p.grad is not g:
                p.grad = g

    def __call__(self, mel=None, *, text=None, lens=None, velocity=None):
        """Run one step on a new batch of the captured shapes; returns the (device) loss tensor of that step (this rank's).
        velocity: replay the graph with the velocity-consistency term (default: when the step has a teacher). `self.out` is then
        that graph's output, with `out.loss_breakdown` (flow, velocity_consistency)."""
        v = velocity_flag(self.teacher, velocity, 'GraphedTrainStep')
        if mel is not None:
            self.mel.copy_(mel, non_blocking=True)
        if text is not None:
            self.text.copy_(text, non_blocking=True)
        if lens is not None:
            self.lens.copy_(lens, non_blocking=True)
        self.graph, self.out, self._grads = self.graphs[v], self.outs[v], self._grad_sets[v]
        self.graph.replay()
        if self.grad_sync is not None:
            self.grad_sync.all_reduce()
            self.grad_sync.attach()
        else:
            self._attach(self._grads)
        return self.out.loss


# ----------------------------------------------------------------------------------------------------------------------
# ragged batches: one graph per (length bucket, text mode), all in one memory pool, with gradient accumulation


class BucketPlan:
    """The host side of BucketedTrainStep, no GPU needed: which bucket a batch of `n` frames goes to, how its text ids are padded,
    and every refusal that must come before a launch."""

    def __init__(self, buckets, batch_size, max_seq_len, interpolated_text=False, who='BucketedTrainStep'):
        self.who = who
        b = sorted({int(x) for x in buckets})
        if not b or b[0] < 1:
            raise ValueError(f'{who}: buckets must be positive frame counts, got {tuple(buckets)}')
        if b[-1] > max_seq_len:
            raise ValueError(f'{who}: bucket {b[-1]} exceeds the transformer\'s max_seq_len ({max_seq_len})')
        if not 1 <= int(batch_size) <= MAX_BATCH:
            raise ValueError(f'{who}: batch_size {batch_size} is outside 1..{MAX_BATCH} (b200_small_linear takes at most '
                             f'{MAX_BATCH} items per launch)')
        self.buckets, self.batch_size, self.interpolated_text = tuple(b), int(batch_size), bool(interpolated_text)

    def bucket(self, n):
        """the smallest bucket >= n"""
        for nb in self.buckets:
            if n <= nb:
                return nb
        raise ValueError(f'{self.who}: a batch of {n} frames exceeds the largest bucket ({self.buckets[-1]})')

    def check(self, batch, n, text_width=None):
        """-> the bucket of a [batch, n, channels] mel with text ids `text_width` columns wide (None: no text); raises ValueError"""
        if batch != self.batch_size:
            raise ValueError(f'{self.who}: batch of {batch} items, the graphs were captured for batch_size={self.batch_size}')
        nb = self.bucket(n)
        if self.interpolated_text and text_width is not None and text_width > nb:
            raise ValueError(f'{self.who}: {text_width} text ids do not fit bucket {nb}: with interpolated_text the text is '
                             'spread over the frames, so it cannot be cut')
        return nb

    @staticmethod
    def pad_text(ids, nb, out=None):
        """(b, nt) ids with -1 padding -> (b, nb): padded with -1 or cut to nb columns — CharacterEmbed cuts and pads to the
        sequence length itself (e2_tts.py:407-412), so its rows are unchanged"""
        if out is None:
            out = torch.empty(ids.shape[0], nb, dtype=torch.int64, device=ids.device)
        w = min(ids.shape[1], nb)
        out[:, :w].copy_(ids[:, :w], non_blocking=True)
        out[:, w:].fill_(-1)
        return out


def text_modes(model):
    """the text-drop decisions a call can reach, as (drop,) flags: E2TTS in training mode draws the reference's coin
    `random() < cond_drop_prob` (e2_tts.py:1261), so 0 < p < 1 reaches both, p <= 0 only the text and p >= 1 only the dropped one;
    an E2TTS in eval mode or a DurationPredictor always uses the text"""
    p = float(getattr(model, 'cond_drop_prob', 0.0))
    if not (hasattr(model, 'cond_drop_prob') and model.training):
        return (False,)
    if p <= 0.0:
        return (False,)
    if p >= 1.0:
        return (True,)
    return (False, True)


def draw_text_drop(model, has_text):
    """the text-drop decision of one call: exactly one python `random.random()` for an E2TTS in training mode (as
    transformer_with_pred_head draws it, whether or not text is given); no text at all means the dropped graph"""
    drop = hasattr(model, 'cond_drop_prob') and model.training and random.random() < model.cond_drop_prob
    return bool(drop) or not has_text


class _KeepPythonRandom:
    """restores python's `random` state on exit: warm-ups and captures run the model's own coin, which must not shift the user's"""

    def __enter__(self):
        self.state = random.getstate()

    def __exit__(self, *a):
        random.setstate(self.state)


class BucketedTrainStep:
    """CUDA-graphed training steps on ragged batches with gradient accumulation (trainer.py:61-82 pads each batch to its longest clip,
    :142/:160/:250 accumulate `grad_accumulation_steps` micro-batches). GraphedTrainStep is the fixed-shape, k = 1 special case.

        steps = BucketedTrainStep(model, batch_size=16, buckets=(256, 512, 768, 1024, 1408), grad_accumulation_steps=4)
        for batch in loader:
            loss = steps(batch['mel'], text=batch['text'], lens=batch['lens'])
            if steps.sync_gradients:
                opt.step(steps.grad_sync.flat)

    * A batch of n frames replays the graph of the smallest bucket N_b >= n: mel is zero-padded to N_b, `lens` defaults to n (the
      reference's full(seq_len)) and is kept as given otherwise, text ids are padded with -1 / cut to N_b columns. Frames at or past
      `lens` are masked keys, zeroed ahead of both convolutions and outside the loss span, so the padding changes no loss or gradient;
      only the noise the CUDA generator draws differs (it is drawn at the padded shape).
    * The text-drop coin is drawn per call on the host (one `random.random()`, as the reference) and picks the text or the
      text-dropped graph of the bucket; only the modes cond_drop_prob can reach are captured.
    * Every graph ends with b200_flat_accumulate (x 1 / (k * world)) into one GradSync buffer: the first call of a window clears it,
      the k-th does ONE all-reduce, attaches p.grad as views of it and sets `sync_gradients`. Between windows p.grad holds the
      previous window's views; feed the optimiser only when `sync_gradients` is set.
    * All graphs share one memory pool (captured largest bucket first) and one dropout seed word. Nothing a caller reads lives in
      the pool: the loss is copied into a buffer of its own and the gradients are consumed by the in-graph accumulate.
    * With `velocity_consistency_model=` (the EMA teacher, VelocityTeacher) every (bucket, text mode) also gets a graph with the
      teacher pass, in the same pool; `velocity=` picks one per call (the trainer's `ema_model.initted`), and the velocity part of
      the loss is copied out to `velocity_loss`.
    FusedAdoptEMA runs one EMA update per optimiser step (ema-pytorch's EMA.update runs per micro-batch in trainer.py:279)."""

    def __init__(self, model, batch_size, buckets, *, grad_accumulation_steps=1, process_group=None, warmup=3,
                 velocity_consistency_model=None, velocity_consistency_delta=1e-5):
        _refuse_ddp_wrapper(model, 'BucketedTrainStep')
        self.teacher = None
        if velocity_consistency_model is not None:
            self.teacher = VelocityTeacher(model, velocity_consistency_model, velocity_consistency_delta, max(int(x) for x in buckets),
                                           'BucketedTrainStep')
        elif float(getattr(model, 'velocity_consistency_weight', 0.0)) > 0.0:
            raise ValueError('BucketedTrainStep: velocity consistency needs its teacher (the reference trainer feeds it the EMA model '
                             'each step, trainer.py:259-268); pass velocity_consistency_model=')
        k = int(grad_accumulation_steps)
        if k < 1:
            raise ValueError(f'BucketedTrainStep: grad_accumulation_steps must be >= 1, got {grad_accumulation_steps}')
        from .modules import InterpolatedCharacterEmbed
        self.plan = BucketPlan(buckets, batch_size, model.transformer.max_seq_len,
                               isinstance(getattr(model, 'embed_text', None), InterpolatedCharacterEmbed))
        dev = next(model.parameters()).device
        if dev.type != 'cuda':
            raise ValueError('BucketedTrainStep: the model must live on the GPU')
        self.model, self.grad_accumulation_steps = model, k
        self.modes = text_modes(model)
        vmodes = (True, False) if self.teacher is not None else (False,)   # with the teacher first: the larger graph
        world = _world(process_group)
        if world > 1:
            broadcast_module(model, 0, process_group)    # replicas must start identical (DDP does this when it wraps the module)
            if self.teacher is not None:
                broadcast_module(self.teacher.model, 0, process_group)
        self.grad_sync = GradSync(list(model.parameters()), process_group)
        self._scale = 1.0 / (k * world)
        self._seed_dev = _new_seed_word(model, dev)
        if self.teacher is not None:
            self.teacher.add_seed_word()
        self._e2tts = hasattr(model, 'cond_drop_prob')
        B, C = self.plan.batch_size, model.num_channels
        order = sorted(self.plan.buckets, reverse=True)   # largest first: it sizes the zero pool and the caches before the small ones
        # static inputs and loss outputs, all outside the graph pool
        self._mel = {nb: torch.zeros(B, nb, C, device=dev) for nb in order}
        self._lens = {nb: torch.full((B,), nb, device=dev, dtype=torch.int64) for nb in order}
        self._text = {}
        for nb in order:
            t = torch.full((B, nb), -1, device=dev, dtype=torch.int64)
            t[:, :max(1, nb // 4)] = ord('a')
            self._text[nb] = t
        # per velocity mode: graphs, loss buffers and chunk tables keyed (bucket, text mode). The plain graphs keep the names they
        # have without a teacher; the velocity graphs also copy out their velocity part.
        self._loss = {(nb, d): torch.zeros((), device=dev) for nb in order for d in self.modes}
        self.graphs, self._tables = {}, {}
        self.velocity_graphs, self._vel_tables = {}, {}
        self._vel_loss = {(nb, d): torch.zeros((), device=dev) for nb in order for d in self.modes} if self.teacher is not None else {}
        self._vel_part = {(nb, d): torch.zeros((), device=dev) for nb in order for d in self.modes} if self.teacher is not None else {}
        self._zero = torch.zeros((), device=dev)
        self.launches = {}
        cdp = getattr(model, 'cond_drop_prob', None)
        t0 = time.perf_counter()
        with _KeepPythonRandom():
            try:
                cur = torch.cuda.current_stream(dev)
                side = torch.cuda.Stream(dev)
                side.wait_stream(cur)
                with torch.cuda.stream(side):   # warm-up off the capture stream: lazy initialisation, caches, packed weights, rotary tables
                    for nb in order:
                        for drop in self.modes:
                            for v in vmodes:
                                for _ in range(max(1, warmup)):
                                    self._pass(nb, drop, v)
                                    _clear_grads(model)
                    if world > 1:
                        self.grad_sync.all_reduce()    # NCCL communicator / channel setup outside the timed path
                cur.wait_stream(side)
                torch.cuda.synchronize(dev)
                torch.cuda.empty_cache()
                self.pool = torch.cuda.graph_pool_handle()
                n0 = lib.launch_count()
                for nb in order:
                    for drop in self.modes:
                        for v in vmodes:
                            _clear_grads(model)      # no graph's backward may add into another graph's gradient tensors
                            table = self.grad_sync.new_table()
                            g = torch.cuda.CUDAGraph()
                            n1 = lib.launch_count()
                            with torch.cuda.graph(g, pool=self.pool):
                                out = self._pass(nb, drop, v)
                                (self._vel_loss if v else self._loss)[nb, drop].copy_(out.loss.reshape(()))
                                if v:
                                    self._vel_part[nb, drop].copy_(out.loss_breakdown.velocity_consistency.reshape(()))
                                grads = self.grad_sync.accumulate(table, self._scale)   # recorded against the (still empty) table
                            self.grad_sync.fill_table(table, grads)
                            self.launches[nb, drop, v] = lib.launch_count() - n1
                            del out, grads
                            _clear_grads(model)
                            if v:
                                self.velocity_graphs[nb, drop], self._vel_tables[nb, drop] = g, table
                            else:
                                self.graphs[nb, drop], self._tables[nb, drop] = g, table
                self.launches_per_step = (lib.launch_count() - n0) // (len(self.graphs) + len(self.velocity_graphs))
            finally:
                if cdp is not None:
                    model.cond_drop_prob = cdp
        if self.teacher is not None:
            self.teacher.seal()
        torch.cuda.synchronize(dev)
        self.capture_seconds = time.perf_counter() - t0   # warm-ups + captures
        self.grad_sync.zero()
        self._micro = 0
        self.sync_gradients = False
        self.velocity_loss = self._zero

    def _pass(self, nb, drop, velocity=False):
        if self._e2tts:    # pin the coin inside the capture; python's random state is restored by the caller
            self.model.cond_drop_prob = 1.0 if drop else 0.0
        text = None if (drop and self._e2tts) else self._text[nb]
        return _train_pass(self.model, self._seed_dev, self._mel[nb], text, self._lens[nb], self.teacher if velocity else None)

    def __call__(self, mel, *, text=None, lens=None, velocity=None):
        """One micro-step on a [batch_size, n, channels] mel (n <= the largest bucket), text ids [batch_size, nt] or a list of
        strings, optional lens [batch_size]. Returns this micro-batch's (unscaled) loss on the device. velocity: replay the graph
        with the velocity-consistency term (default: when the step has a teacher); its velocity part is then in
        `self.velocity_loss` (0 otherwise)."""
        v = velocity_flag(self.teacher, velocity, 'BucketedTrainStep')
        if isinstance(text, list):
            from .modules import list_str_to_tensor
            text = (self.model.tokenizer(text) if self._e2tts else list_str_to_tensor(text)).to(mel.device)
        B, n = int(mel.shape[0]), int(mel.shape[1])
        nb = self.plan.check(B, n, None if text is None else int(text.shape[1]))
        if text is None and True not in self.modes:
            raise ValueError('BucketedTrainStep: text=None needs the text-dropped graph, which is only captured for an E2TTS in '
                             'training mode with cond_drop_prob > 0')
        drop = draw_text_drop(self.model, text is not None)
        if self._micro == 0:
            self.grad_sync.zero()
        m = self._mel[nb]
        m[:, :n].copy_(mel, non_blocking=True)
        if n < nb:
            m[:, n:].zero_()
        if lens is None:
            self._lens[nb].fill_(n)
        else:
            self._lens[nb].copy_(lens, non_blocking=True)
        if text is not None and not drop:
            self.plan.pad_text(text, nb, out=self._text[nb])
        (self.velocity_graphs if v else self.graphs)[nb, drop].replay()
        self._micro += 1
        self.sync_gradients = self._micro == self.grad_accumulation_steps
        if self.sync_gradients:
            self._micro = 0
            self.grad_sync.all_reduce()
            self.grad_sync.attach()
        self.velocity_loss = self._vel_part[nb, drop].clone() if v else self._zero
        return (self._vel_loss if v else self._loss)[nb, drop].clone()
