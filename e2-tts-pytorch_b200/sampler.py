"""GraphedSampler: E2TTS.sample() with its whole fixed-grid ODE solve as one CUDA graph per (duration bucket, text present / absent).

Eager sample() drives every function evaluation from Python: at the 32-step midpoint default, 62 evaluations of two transformer passes
each (the conditional and the text-dropped prediction of classifier-free guidance), several hundred launches per pass. On a small
model and a short clip the GPU finishes each kernel before the host has issued the next, so the host sets the latency. Here
  * the host does, eagerly, exactly what sample() does ahead of its ODE loop (mel of a raw wave, tokens, lens, the duration or the
    DurationPredictor, the clamp, the y0 draw in sample()'s order and shape), then pads cond, y0 and the masks to the smallest bucket
    that holds the longest duration and replays that bucket's graph; padded frames are masked keys, so valid frames do not depend on
    the padding. The output is sliced back and finished as sample() finishes it (the prompt frames, the Vocos decode);
  * with cfg_strength > 0 and no cfg_null_model, each evaluation is ONE pass over 2B items (E2TTS.cfg_pred_batched): the text
    items and their text-dropped copies. With a cfg_null_model (a different model) or cfg_strength = 0 the evaluation is
    cfg_transformer_with_pred_head's, two passes or one;
  * the graph starts by packing the weights from the live parameters (one launch), so a replay always uses the current weights:
    a load_state_dict or an optimiser step between calls needs nothing. If a parameter or buffer gets new storage (`.to()`,
    reassignment), the next call captures the graphs again;
  * all graphs share one memory pool, captured largest bucket first.
Only the fixed-grid methods (midpoint, euler, rk4) can be graphed: the adaptive ones decide every step on the host.
"""
from __future__ import annotations

import contextlib
import time

import torch

from . import modules, ode, ops
from .graphed import MAX_BATCH, BucketPlan

FIXED_GRID_METHODS = ('midpoint', 'euler', 'rk4')


def stage_times(method, steps):
    """the evaluation times of the fixed-grid solve on linspace(0, 1, steps), in the order the solve evaluates them (fp32 host
    floats, computed as sample() computes them)"""
    if method == 'rk4':
        return [float(t) for t in ode.rk4_times(steps)]
    ts = torch.linspace(0, 1, steps)
    out = []
    for i in range(steps - 1):
        out.append(float(ts[i]))
        if method == 'midpoint':
            out.append(float(ts[i] + 0.5 * float(ts[i + 1] - ts[i])))
    return out


def solve(fn, y, method, steps, tt):
    """sample()'s fixed-grid solve with the stage times `tt` (stage_times(method, steps) on the device): no host work between steps"""
    if method == 'rk4':
        return ode.rk4(fn, y, steps, tt=tt)
    ts = torch.linspace(0, 1, steps)
    j = 0
    for i in range(steps - 1):
        dt = float(ts[i + 1] - ts[i])
        if method == 'euler':
            y = ops.axpy(y, fn(tt[j], y), dt)
            j += 1
        else:
            half = 0.5 * dt
            ymid = ops.axpy(y, fn(tt[j], y), half)
            y = ops.axpy(y, fn(tt[j + 1], ymid), dt)
            j += 2
    return y


def bucket_buffers(B, nb, C, rows, device):
    """the static inputs of bucket nb: y0 and the step conditioning fp32 [B, nb, C], the duration mask bool [rows, nb] (rows = 2B for
    the batched guidance pass: the mask of the B items, twice), text ids [B, nb] (-1 padding)"""
    text = torch.full((B, nb), -1, device=device, dtype=torch.int64)
    text[:, :max(1, nb // 4)] = ord('a')
    return dict(y0=torch.zeros(B, nb, C, device=device), cond=torch.zeros(B, nb, C, device=device),
                mask=torch.ones(rows, nb, device=device, dtype=torch.bool), text=text)


def stage_inputs(plan, rows, y0, step_cond, duration, text, buffers=None):
    """Pad one call's inputs to its bucket: y0 and step_cond [B, md, C] with zero frames, the duration mask (lens_to_mask(duration)
    to nb frames: the padding is masked keys), text ids [B, nt] by BucketPlan.pad_text (None: no text). Writes into `buffers`
    ({bucket: bucket_buffers(...)}; new ones when None). -> (nb, that bucket's buffers)"""
    from .modules import lens_to_mask
    B, md, C = y0.shape
    nb = plan.check(B, md, None if text is None else int(text.shape[1]))
    buf = buffers[nb] if buffers is not None else bucket_buffers(B, nb, C, rows, y0.device)
    for static, src in ((buf['y0'], y0), (buf['cond'], step_cond)):
        static[:, :md].copy_(src)
        static[:, md:].zero_()
    mask = lens_to_mask(duration, nb)
    for r in range(0, rows, B):
        buf['mask'][r:r + B].copy_(mask)
    if text is not None:
        plan.pad_text(text, nb, out=buf['text'])
    return nb, buf


class GraphedSampler:
    """E2TTS.sample() as CUDA-graph replays for batches of `batch_size` items whose longest duration fits one of `buckets` (frames).

        sampler = GraphedSampler(model, batch_size=1, buckets=(512, 1024, 2048), steps=32, cfg_strength=1.)
        mel = sampler(cond, text=['hello world'], return_raw_output=True)

    The call takes the arguments of E2TTS.sample (steps, cfg_strength and cfg_null_model are fixed at construction) and returns
    what it returns. With the same seed it integrates from the same y0 as sample(). The graphs are captured in the constructor:
    `warmup` function evaluations per graph run eagerly first. `capture_seconds` is the time the warm-ups and captures took."""

    def __init__(self, model, batch_size, buckets, *, steps=32, cfg_strength=1., cfg_null_model=None, warmup=1):
        from .modules import InterpolatedCharacterEmbed, _parse_odeint_kwargs
        method = _parse_odeint_kwargs(model.odeint_kwargs)['method']
        if method not in FIXED_GRID_METHODS:
            raise ValueError(f"GraphedSampler: odeint_kwargs method {method!r} is adaptive: it decides every step on the host, so its "
                             f"solve cannot be one graph; use E2TTS.sample() for it (graphed: {', '.join(FIXED_GRID_METHODS)})")
        if int(steps) < 2:
            raise ValueError(f'GraphedSampler: steps must be >= 2 (got {steps!r}): the grid linspace(0, 1, steps) needs an interval')
        B = int(batch_size)
        self.batched = cfg_strength >= 1e-5 and cfg_null_model is None
        rows = 2 * B if self.batched else B
        if B < 1 or rows > MAX_BATCH:
            limit = f'2 * batch_size <= {MAX_BATCH}: the batched guidance pass runs 2 * batch_size items' if self.batched else \
                f'batch_size <= {MAX_BATCH}'
            raise ValueError(f'GraphedSampler: batch_size {batch_size} is outside what the kernels take ({limit}; b200_small_linear '
                             f'takes at most {MAX_BATCH} items per launch)')
        self.plan = BucketPlan(buckets, B, model.transformer.max_seq_len, isinstance(model.embed_text, InterpolatedCharacterEmbed),
                               who='GraphedSampler')
        for name, m in (('model', model), ('cfg_null_model', cfg_null_model)):
            if m is not None and next(m.parameters()).device.type != 'cuda':
                raise ValueError(f'GraphedSampler: {name} must live on the GPU')
        if cfg_null_model is not None and self.plan.buckets[-1] > cfg_null_model.transformer.max_seq_len:
            raise ValueError(f'GraphedSampler: bucket {self.plan.buckets[-1]} exceeds the cfg_null_model\'s max_seq_len '
                             f'({cfg_null_model.transformer.max_seq_len})')
        self.model, self.null_model = model, cfg_null_model
        self.method, self.steps, self.cfg_strength, self.warmup = method, int(steps), float(cfg_strength), max(1, int(warmup))
        self.device = next(model.parameters()).device
        self._rows = rows
        self._capture()

    # ------------------------------------------------------------------ capture
    def _models(self):
        return [m for m in (self.model, self.null_model) if m is not None]

    def _fingerprint(self):
        """what the graphs have baked in: each model's pack object and the storage of every parameter and buffer"""
        out = []
        for m in self._models():
            pack = m._derived.get('pack')
            out.append(id(pack[0]) if pack is not None else None)
            out += [t.data_ptr() for t in m.parameters()] + [t.data_ptr() for t in m.buffers()]
        return tuple(out)

    def _fn(self, t, x, cond, mask, text):
        if self.batched:
            return self.model.cfg_pred_batched(x, cond, t, mask, text, self.cfg_strength)
        return self.model.cfg_transformer_with_pred_head(x, cond, times=t, text=text, mask=mask, cfg_strength=self.cfg_strength,
                                                         cfg_null_model=self.null_model)

    def _solve(self, nb, has_text):
        """the captured body: pack each model's weights once, then the whole solve on the bucket's static inputs"""
        buf = self._bufs[nb]
        text = buf['text'] if has_text else None
        with contextlib.ExitStack() as stack:
            for m in self._models():
                stack.enter_context(m._pack()[0].freeze())
            return solve(lambda t, x: self._fn(t, x, buf['cond'], buf['mask'], text), buf['y0'], self.method, self.steps, self._tt)

    def _capture(self):
        # The text sub-blocks run on the current stream inside these graphs, not on the side stream of modules.TWO_STREAM: a capture
        # cannot reuse a block that was used on another stream until the capture ends, so the text stream's tensors of every layer of
        # every function evaluation would stay allocated (hundreds of GB over a 62-evaluation solve at d1024 / B8 / 2048 frames).
        two_stream, modules.TWO_STREAM = modules.TWO_STREAM, False
        try:
            self._capture_graphs()
        finally:
            modules.TWO_STREAM = two_stream

    def _capture_graphs(self):
        model, dev, B, C = self.model, self.device, self.plan.batch_size, self.model.num_channels
        self.graphs, self._out = {}, {}
        t0 = time.perf_counter()
        with torch.no_grad(), torch.cuda.device(dev):
            for m in self._models():
                m.eval()
            order = sorted(self.plan.buckets, reverse=True)   # largest first: it sizes the pool the smaller ones reuse
            # static inputs, outside the graph pool
            self._tt = torch.tensor(stage_times(self.method, self.steps), dtype=torch.float32, device=dev)
            self._bufs = {nb: bucket_buffers(B, nb, C, self._rows, dev) for nb in order}
            cur = torch.cuda.current_stream(dev)
            side = torch.cuda.Stream(dev)
            side.wait_stream(cur)
            with torch.cuda.stream(side):   # off the capture stream: packs' pointer tables, rotary tables, lazy initialisation
                for nb in order:
                    for has_text in (True, False):
                        buf = self._bufs[nb]
                        for _ in range(self.warmup):
                            self._fn(self._tt[0], buf['y0'], buf['cond'], buf['mask'], buf['text'] if has_text else None)
            cur.wait_stream(side)
            torch.cuda.synchronize(dev)
            torch.cuda.empty_cache()
            self.pool = torch.cuda.graph_pool_handle()
            for nb in order:
                for has_text in (True, False):
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g, pool=self.pool):
                        self._out[nb, has_text] = self._solve(nb, has_text)
                    self.graphs[nb, has_text] = g
            torch.cuda.synchronize(dev)
        self.capture_seconds = time.perf_counter() - t0
        self._captured = self._fingerprint()

    # ------------------------------------------------------------------ call
    @torch.no_grad()
    def __call__(self, cond, *, text=None, lens=None, duration=None, max_duration=4096, vocoder=None, return_raw_output=None):
        from .modules import _rng
        model = self.model
        with torch.cuda.device(self.device):
            model.eval()
            model._check_decoder(vocoder, return_raw_output)
            if self._fingerprint() != self._captured:
                self._capture()
            cond, cond_mask, text, duration = model._sample_inputs(cond, text, lens, duration, max_duration)
            md = cond.shape[1]
            self.plan.check(cond.shape[0], md, None if text is None else int(text.shape[1]))   # before the y0 draw
            step_cond = torch.where(cond_mask, cond, torch.zeros_like(cond))
            y0 = _rng.draw('y0', lambda: torch.randn_like(cond))
            nb, _ = stage_inputs(self.plan, self._rows, y0, step_cond, duration, text, self._bufs)
            self.graphs[nb, text is not None].replay()
            y = self._out[nb, text is not None][:, :md]
            return model._sample_output(torch.where(cond_mask, cond, y), duration, vocoder, return_raw_output)
