"""Element-wise float64 bounds for the optimiser-step kernels of csrc/optim.cu: b200_flat_gather, b200_sumsq, b200_adopt_step and
b200_flat_scatter, and FusedAdoptEMA / GradSync around them.

Method of tests/kernel_checks.py: each entry point is called through the C ABI (lib.call / lib.make_args) over
chunk tables built by optim.FlatLayout, with NaN-prefilled outputs and a sentinel in the flat buffers' padding slots (parameter
offsets are rounded up to 4 elements; no kernel may write those slots). References are computed in float64 (torch's float64 ops,
on the device for the 64 M-element layouts) from the exact fp32 inputs of the same call. Every bound is E (bit for bit) or F:

  standard model fl(a op b) = (a op b)(1 + d), |d| <= u = 2^-24, per fp32 rounding; a result with n roundings whose inputs carry
  the propagated error p is within p + gamma_n (|v| + p) (`_rnd`); a sum of terms that each pass through at most d roundings is
  within gamma_d sum|terms| (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., (3.4)-(3.5)); sqrtf and / are
  correctly rounded (the library is built without fast-math); an expression the compiler may contract into an FMA is given the
  roundings of its uncontracted form (2 for a*b + c), which bounds the fused form too.

b200_sumsq (per call, n terms, grid G, restated from the host code below): each thread sums 4 products per float4 (or 1 per
  scalar) over its grid-stride loop, then a warp butterfly (5), the 8 warp sums in order (8), and the last block adds the G block
  partials: ceil(G / 256) per thread, 5, 8. So every x_i^2 passes through at most d = t + 13 + ceil(G / 256) + 13 roundings,
  t = 4 * (float4 iterations) + 2 (aligned x) or (scalar iterations) + 1 (misaligned x), and
  |got - sum x^2| <= gamma_d sum x^2 + n 2^-149 (underflowed products) + gamma64_n sum x^2 (the float64 reference's own sum).

b200_adopt_step (one element; scalars as the reference applies them: lerp weights c_k = fp32(1 - beta_k) formed in double,
  decay factor F = fp32(1 - lr wd) with wd = weight_decay / init_lr, EMA weight fp32(1 - decay), clip = min(1, mn / (sqrt(ns) + 1e-6))):
  clip   the kernel's sqrtf, the fp32 1e-6 and its add, the division: relative gamma_4 of q = mn / (sqrt(ns) + 1e-6) (plus the
         relative error h of sqrt(ns) when ns itself is the kernel's sumsq: h = r / (1 + sqrt(1 - r)) for a relative error r of ns);
         the clamp at 1 only shrinks it. Clipping off, or q(1 - r) > 1: the coefficient is exactly 1 and g is exact.
  g      = fl(g0 clip)                                     1 rounding (none at an exact coefficient of 1)
  F      kernel fl(1 - fl32(lr) fl32(wd)): |F_k - (1 - lr wd)| <= gamma_2 lr wd + gamma_2 (1 + 2 lr wd); w1 = fl(w0 F_k): 1 rounding
  D      max(sqrtf(v0), fp32(eps)): within max(u sqrt(v0), |fp32(eps) - eps|) of max(sqrt(v0), eps) (max is 1-Lipschitz)
  u      = fl(g / D)                                       quotient of perturbed values, 1 rounding
  m      = m0 + c1 fl(u - m0)                              1 + 2 roundings
  w      = w1 - fl32(lr) m                                 2 roundings, and |fl32(lr) - lr|
  v      = v0 + c2 fl(fl(g g) - v0)                        1 + 1 + 2 roundings
  EMA    mode 1: e0 + ew fl(w - e0) from the kernel's own written w: 1 + 2 roundings; mode 2: bit-equal to that w.
  The complement error of 1.f - beta formed in fp32 (16 u relative for beta 0.99, 2784 u for 0.9999) exceeds the v bound where
  v0 << g^2 (v_new ~ c2 g^2 with ~6 u of rounding), which is why those elements exist.
Re-anchoring: the FusedAdoptEMA schedule starts each step's reference from the kernel's own fp32 w, m, v and EMA of the previous
step, so the bounds do not compound.
"""
import bisect
import copy
import io
import math
import re

import numpy as np
import pytest
import torch

from oracle import optim_oracle as OO
from kernel_checks import F32, F64, U, Rv, _rnd, check_e, dev, gamma, mul, pkg, sms, stream

pytestmark = pytest.mark.gpu

I32 = torch.int32
CHUNK = 16384                         # optim.CHUNK: elements per chunk-table entry
SUMSQ_MAX_GRID = 4096                 # optim.cu kSumsqMaxGrid
SENTINEL = -1234.5                    # padding slots
EDGE_SHAPES = [(1,), (3,), (4,), (5,), (16383,), (16384,), (16385,), (3 * CHUNK + 5,), (129, 515)]
EDGE_W_SHIFT = [0, 1, 0, 2, 3, 0, 1, 3, 2]     # storage offset (elements) of each parameter in its buffer: 1, 2, 3 -> misaligned w
EDGE_G_SHIFT = [1, 0, 3, 0, 2, 1, 0, 0, 3]     # the same for the gradients (flat_gather's scalar path)
TEXT = re.compile(r'(text|^transformer\.(layers|hyper_conns)\.\d+\.1\.)')   # parameters without a gradient when the text is dropped


def gamma64(n):
    return n * 2.0 ** -53 / (1 - n * 2.0 ** -53)


def f32(x):
    """the fp32 value of a python float, as a python float"""
    return float(np.float32(x))


_CFG2 = {}


def cfg2_shapes():
    """(names, shapes) of E2TTS(dim=512, depth=8, heads=8)'s parameters, built on the CPU"""
    if not _CFG2:
        import e2_tts_pytorch_b200 as pkg
        m = pkg.E2TTS(transformer=dict(dim=512, depth=8, heads=8), use_vocos=False)
        _CFG2['v'] = ([n for n, _ in m.named_parameters()], [tuple(p.shape) for p in m.parameters()])
    return _CFG2['v']


def edge_params(shifts=EDGE_W_SHIFT):
    """the edge shapes, each at storage offset `shift` inside its own buffer"""
    out = []
    for s, k in zip(EDGE_SHAPES, shifts):
        n = math.prod(s)
        out.append(torch.zeros(n + 4, device=dev(), dtype=F32)[k:k + n].view(s))
    return out


def packed_params(shapes, start):
    """the shapes back to back in one buffer from element `start`: every tensor after an odd-sized one is misaligned"""
    numels = [math.prod(s) for s in shapes]
    buf = torch.zeros(start + sum(numels), device=dev(), dtype=F32)
    out, o = [], start
    for s, n in zip(shapes, numels):
        out.append(buf[o:o + n].view(s))
        o += n
    return out


def layout_params(which):
    """-> (names, params) for the edge or the cfg2 layout"""
    if which == 'edge':
        return [f'edge{i}{tuple(s)}' for i, s in enumerate(EDGE_SHAPES)], edge_params()
    names, shapes = cfg2_shapes()
    return names, packed_params(shapes, 0)


def grad_tensors(which, shapes):
    if which == 'edge':
        return edge_params(EDGE_G_SHIFT)
    return packed_params(shapes, 1)


class Slots:
    """restated chunk table of a FlatLayout: per flat slot, its chunk (-1 for padding) and parameter"""

    def __init__(self, lay, names):
        self.lay, self.names = lay, names
        chunk, pid, off, lens = [], [], [], []
        for i, (o, n) in enumerate(zip(lay.offsets, lay.numels)):
            for s in range(0, n, CHUNK):
                chunk.append(len(chunk))
                pid.append(i)
                off.append(o + s)
                lens.append(min(CHUNK, n - s))
        assert len(chunk) == lay.n_chunks
        self.chunk_pid = torch.tensor(pid, device=dev())
        lens = torch.tensor(lens, device=dev())
        cid = torch.repeat_interleave(torch.arange(lay.n_chunks, device=dev()), lens)
        first = torch.repeat_interleave(torch.tensor(off, device=dev()) - (torch.cumsum(lens, 0) - lens), lens)
        self.chunk_of = torch.full((lay.total,), -1, dtype=torch.int64, device=dev())
        self.chunk_of[first + torch.arange(cid.numel(), device=dev())] = cid
        self.pad = self.chunk_of < 0
        self.valid = ~self.pad
        self.pid = torch.where(self.valid, self.chunk_pid[self.chunk_of.clamp(min=0)], -1)
        assert int(self.valid.sum()) == sum(lay.numels)

    def where(self, i):
        lay = self.lay
        k = bisect.bisect_right(lay.offsets, i) - 1
        e = i - lay.offsets[k]
        if e >= lay.numels[k]:
            return f'padding slot {e} of {self.names[k]}'
        idx = tuple(int(j) for j in np.unravel_index(e, tuple(lay.params[k].shape))) if lay.params[k].dim() else ()
        return f'{self.names[k]} element {idx}'

    def flat(self, tensors, fill=float('nan')):
        out = torch.full((self.lay.total,), fill, device=dev(), dtype=F32)
        for o, n, t in zip(self.lay.offsets, self.lay.numels, tensors):
            if t is not None:
                out[o:o + n] = t.reshape(-1)
        return out

    def scatter(self, flat, tensors):
        for o, n, t in zip(self.lay.offsets, self.lay.numels, tensors):
            t.copy_(flat[o:o + n].view_as(t))


def fcheck_f(name, sl, got, ref, bound, mask):
    """|got - ref| <= bound on the slots of `mask`; NaN never passes; names the parameter and element of the first failure"""
    bad = ~((got.double() - ref).abs() <= bound) & mask
    if bool(bad.any()):
        idx = bad.nonzero()[:, 0]
        i = int(idx[0])
        raise AssertionError(f'{name}: |got - ref| exceeds the bound at {sl.where(i)}: got {got[i].item():.9g}, ref {ref[i].item():.9g}, '
                             f'bound {bound[i].item():.3g}; {idx.numel()} of {int(mask.sum())} elements')


def fcheck_e(name, sl, got, want, mask):
    """bit for bit on the slots of `mask` (int32 views: +0 and -0 differ, NaN payloads count)"""
    bad = (got.contiguous().view(I32) != want.contiguous().view(I32)) & mask
    if bool(bad.any()):
        idx = bad.nonzero()[:, 0]
        i = int(idx[0])
        raise AssertionError(f'{name}: {idx.numel()} of {int(mask.sum())} elements differ, first at {sl.where(i)}: '
                             f'got {got[i].item()!r}, want {want[i].item()!r}')


# ------------------------------------------------------------------------------------------------------------- running bounds
def sub(a, b, n=1):
    return _rnd(a.v - b.v, a.e + b.e, n)


def div(a, b):
    """b.v > b.e >= 0: |a'/b' - a/b| <= (e_a + |a/b| e_b) / (b - e_b)"""
    v = a.v / b.v
    return _rnd(v, (a.e + v.abs() * b.e) / (b.v - b.e))


def axpy(x, a, y):
    """y + a x with an exact scalar a, as the kernel's fma (or mul + add): 2 roundings"""
    return _rnd(y.v + a * x.v, a * x.e + y.e, 2)


def clip_rv(ns, max_norm, ns_rel=0.0):
    """clip coefficient min(1, mn / (sqrt(ns) + 1e-6)) in float64 and the bound on the kernel's fp32 one (module docstring)"""
    q = max_norm / (math.sqrt(ns) + 1e-6)
    h = ns_rel / (1 + math.sqrt(1 - ns_rel))
    r = h + gamma(4) * (1 + h)
    c = min(1.0, q)
    e = max(abs(min(1.0, q * (1 + r)) - c), abs(min(1.0, q * (1 - r)) - c))
    return c, e


# ------------------------------------------------------------------------------------------------------------------- gather
def _special_grads(tensors, gen):
    """N(0, 1) gradients with +-0, subnormals, +-inf, NaN and +-FLT_MAX at fixed elements"""
    special = torch.tensor([0.0, -0.0, 1e-40, -1e-40, 2.0 ** -149, -(2.0 ** -149), float('inf'), float('-inf'), float('nan'),
                            3.4028234663852886e38, -3.4028234663852886e38, 2.0 ** -126], dtype=F32)
    for i, t in enumerate(tensors):
        t.view(-1).copy_(torch.randn(t.numel(), generator=gen).to(dev()))
        k = min(t.numel(), special.numel())
        pos = (torch.arange(k) * 7 + i) % t.numel()
        t.view(-1)[pos.to(dev())] = special[(torch.arange(k) + i) % special.numel()].to(dev())


def _check_gather(name, sl, flat, used, grads, scale):
    live = torch.zeros(sl.lay.total, dtype=torch.bool, device=dev())
    want = torch.zeros(sl.lay.total, device=dev(), dtype=F32)
    for o, n, g in zip(sl.lay.offsets, sl.lay.numels, grads):
        if g is not None:
            want[o:o + n] = (g.reshape(-1).double() * f32(scale)).float()   # exact product, rounded once: fl(g * fp32(scale))
            live[o:o + n] = True
    nan = torch.isnan(want)
    fcheck_e(f'{name} flat (finite slots, scale {scale:.6g})', sl, flat, want, sl.valid & ~nan)
    assert bool(torch.isnan(flat[nan]).all()), f'{name}: a NaN gradient element did not give a NaN slot'
    fcheck_e(f'{name} flat padding', sl, flat, torch.full_like(flat, SENTINEL), sl.pad)
    check_e(f'{name} used', used, torch.tensor([0.0 if g is None else 1.0 for g in grads], device=dev()))


def _prefill(sl, buf):
    buf.fill_(float('nan'))
    buf[:sl.lay.total][sl.pad] = SENTINEL


@pytest.mark.parametrize('which', ['edge', 'cfg2'])
def test_flat_gather(pkg, which):
    names, params = layout_params(which)
    lay = pkg.optim.FlatLayout(params)
    sl = Slots(lay, names)
    grads = grad_tensors(which, [tuple(p.shape) for p in params])
    _special_grads(grads, torch.Generator().manual_seed(0))
    none = {2, 7} if which == 'edge' else {i for i, n in enumerate(names) if TEXT.search(n)}
    grads = [None if i in none else g for i, g in enumerate(grads)]
    if which == 'edge':
        assert any(g is not None and g.data_ptr() % 16 for g in grads) and any(g is not None and g.data_ptr() % 16 == 0 for g in grads)
    flat = torch.empty(lay.total, device=dev(), dtype=F32)
    used = torch.empty(len(params), device=dev(), dtype=F32)
    for scale in (1.0, 1.0 / 3.0):
        _prefill(sl, flat)
        used.fill_(float('nan'))
        pkg.lib.call('b200_flat_gather', lay.table(grads), lay.n_chunks, flat, f32(scale), used, stream())
        _check_gather(which, sl, flat, used, grads, scale)


def test_flat_gather_under_graph_capture(pkg):
    """GraphedTrainStep's path: the gather is recorded against new_table() inside torch.cuda.graph, the table is filled after the
    capture, the graph replays; then the gradients change in place and it replays again"""
    names, params = layout_params('edge')
    params = [torch.nn.Parameter(p, requires_grad=False) for p in params]
    sync = pkg.optim.GradSync(params)
    sl = Slots(sync.layout, names)
    grads = edge_params(EDGE_G_SHIFT)
    _special_grads(grads, torch.Generator().manual_seed(1))
    for i, (p, g) in enumerate(zip(params, grads)):
        p.grad = None if i == 4 else g
    table = sync.new_table()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = sync.gather(table)
    sync.fill_table(table, static)
    assert static[4] is None
    for seed in (2, 3):
        _prefill(sl, sync._buf)
        graph.replay()
        torch.cuda.synchronize()
        _check_gather('captured gather', sl, sync.flat, sync.used, static, 1.0)
        _special_grads([g for g in static if g is not None], torch.Generator().manual_seed(seed))   # in place, same storage


# ------------------------------------------------------------------------------------------------------------------- sumsq
def sumsq_grid(n):
    """b200_sumsq's launch: (grid, whether the 8-per-SM cap applies)"""
    blocks = (n // 4 + 255) // 256
    cap = min(sms() * 8, SUMSQ_MAX_GRID)
    return max(1, min(blocks, cap)), blocks > cap


def sumsq_rel_bound(n, aligned):
    """relative bound gamma_d of the module docstring (without the underflow and float64 terms)"""
    grid, _ = sumsq_grid(n)
    if aligned:
        t = 4 * -(-(n // 4) // (grid * 256)) + 2
    else:
        t = -(-n // (grid * 256)) + 1
    return gamma(t + 13 + -(-grid // 256) + 13)


def sumsq_bound(n, aligned, ref):
    return sumsq_rel_bound(n, aligned) * ref + n * 2.0 ** -149 + gamma64(n) * ref


def _spread(n, gen_seed, out):
    """|x| spread over 2^-60 .. 2^30, random signs, written into `out` in slices"""
    g = torch.Generator(device=dev()).manual_seed(gen_seed)
    step = 1 << 26
    for a in range(0, n, step):
        b = min(n, a + step)
        e = torch.rand(b - a, generator=g, device=dev(), dtype=F64) * 90 - 60
        s = torch.where(torch.rand(b - a, generator=g, device=dev()) < 0.5, -1.0, 1.0).double()
        out[a:b] = (s * torch.exp2(e)).float()


def _sumsq64(x):
    step, acc = 1 << 26, 0.0
    for a in range(0, x.numel(), step):
        acc += float(x[a:a + step].double().square().sum())
    return acc


def _run_sumsq(pkg, n, seed):
    buf = torch.empty(n + 4, device=dev(), dtype=F32)
    assert buf.data_ptr() % 16 == 0
    out = torch.empty(1, device=dev(), dtype=F32)
    for shift in (0, 1):
        x = buf[shift:shift + n]
        _spread(n, seed, x)
        ref = _sumsq64(x)
        out.fill_(float('nan'))
        pkg.lib.call('b200_sumsq', x, n, out, stream())
        got = float(out)
        bound = sumsq_bound(n, shift == 0, ref)
        assert abs(got - ref) <= bound, (f'sumsq n={n} x {"aligned" if shift == 0 else "at buf[1:]"} grid {sumsq_grid(n)[0]}: '
                                         f'got {got!r}, ref {ref!r}, bound {bound:.3g}')
        again = out.clone()
        pkg.lib.call('b200_sumsq', x, n, out, stream())
        check_e(f'sumsq n={n} shift {shift} repeated call', out, again)       # block partials are added in a fixed order


def _cap_blocks():
    return min(sms() * 8, SUMSQ_MAX_GRID)


@pytest.mark.parametrize('which', ['1', '3', '4', '5', 'below_cap', 'wraps', 'cfg2'])
def test_sumsq(pkg, which):
    cap = _cap_blocks()
    if which == 'below_cap':
        n = (cap - 1) * 1024 + 3
        assert sumsq_grid(n) == (cap - 1, False)
    elif which == 'wraps':
        n = 5 * cap * 1024 + 7
        grid, capped = sumsq_grid(n)
        assert capped and grid == cap and (n // 4) > 3 * grid * 256 and n > 3 * grid * 256    # both loops wrap at least 3 times
    elif which == 'cfg2':
        lay = pkg.optim.FlatLayout(layout_params('cfg2')[1])
        n = lay.total
        assert n == 64_238_164 and lay.n_chunks == 4_393 and sumsq_grid(n)[1]
    else:
        n = int(which)
        assert sumsq_grid(n) == (1, False)
    _run_sumsq(pkg, n, 10 + len(which))


def test_sumsq_cfg3_total(pkg):
    """cfg3 / cfg5 (d1024 depth24 h16): 723,598,052 parameters, 723,598,916 padded slots (2.9 GB of fp32)"""
    n = 723_598_916
    assert sumsq_grid(n)[1]
    _run_sumsq(pkg, n, 99)


# --------------------------------------------------------------------------------------------------------------- adopt_step
BETAS = [(0.9, 0.99), (0.9, 0.9999)]
CASES = [   # (ema_mode, user weight_decay, clip)
    (0, 0.0, 'off'), (1, 0.0, 'below'), (2, 0.0, 'above'), (1, 1e-5, 'zero'),
    (2, 1e-5, 'off'), (0, 1e-5, 'below'), (1, 1e-5, 'above'), (0, 0.0, 'zero'), (2, 0.0, 'inf'),
]
NORM_SQ = {'below': 6.25, 'above': 0.25, 'zero': 0.0, 'inf': float('inf')}   # exact fp32 values of *gradnorm_sq
LR, INIT_LR, EPS, MAX_NORM = 1e-3, 1e-3, 1e-6, 1.0
EMA_W = f32(1.0 - 0.99)


class AdoptCall:
    """one b200_adopt_step: the inputs (flat, fp32), the call, and the element-wise checks against float64 Adopt"""

    def __init__(self, pkg, sl, params, betas, weight_decay, ema_mode, gradnorm_sq, max_norm, used, chunk_state, lr=LR, ema_weight=EMA_W):
        self.pkg, self.sl, self.params, self.betas = pkg, sl, params, betas
        self.wd = weight_decay / INIT_LR if weight_decay > 0 else 0.0     # FusedAdoptEMA's decoupled weight decay
        self.lr, self.ema_mode, self.ema_weight, self.max_norm = lr, ema_mode, ema_weight, max_norm
        self.gradnorm_sq, self.used, self.chunk_state = gradnorm_sq, used, chunk_state

    def run(self, g, m, v, e):
        lay = self.sl.lay
        self.g0, self.w0, self.m0, self.v0 = g.clone(), self.sl.flat(self.params), m.clone(), v.clone()
        self.e0 = e.clone()
        self.cs0 = self.chunk_state.clone()
        a = self.pkg.lib.make_args(
            'b200_adopt_args', chunks_dev=lay.param_table, n_chunks=lay.n_chunks, grad_flat=g, m_flat=m, v_flat=v, ema_flat=e if self.ema_mode else None,
            gradnorm_sq=self.gradnorm_sq, max_grad_norm=f32(self.max_norm), lr=f32(self.lr), beta1=f32(self.betas[0]),
            beta2=f32(self.betas[1]), eps=f32(EPS), weight_decay=f32(self.wd), chunk_state=self.chunk_state, ema_mode=self.ema_mode,
            ema_weight=f32(self.ema_weight), used=self.used, one_minus_beta1=f32(1.0 - self.betas[0]), one_minus_beta2=f32(1.0 - self.betas[1]))
        self.pkg.lib.call('b200_adopt_step', a, stream())

    def check(self, m, v, e, clip, tag):
        """clip: None (off) or (c, e_c)"""
        sl = self.sl
        first_c = self.cs0 == 0
        live_p = torch.ones(len(sl.lay.params), dtype=torch.bool, device=dev()) if self.used is None else self.used > 0
        live_c = live_p[sl.chunk_pid]
        cs_want = torch.where(live_c & first_c, 1, self.cs0).to(I32)
        check_e(f'{tag} chunk_state', self.chunk_state, cs_want)
        ci = sl.chunk_of.clamp(min=0)
        live, first = sl.valid & live_c[ci], sl.valid & first_c[ci]
        stale, fresh, cont = sl.valid & ~live, live & first, live & ~first
        w = sl.flat(self.params)
        exact_one = clip is None or (clip[0] == 1.0 and clip[1] == 0.0)
        decay = self.wd > 0

        # bit-exact parts
        for name, got, want in (('w', w, self.w0), ('m', m, self.m0), ('v', v, self.v0)):
            fcheck_e(f'{tag} {name} of parameters without a gradient', sl, got, want, stale)
        fcheck_e(f'{tag} m on a first step', sl, m, torch.zeros_like(m), fresh)
        for name, got, want in (('m', m, self.m0), ('v', v, self.v0)):
            fcheck_e(f'{tag} {name} padding', sl, got, want, sl.pad)
        if exact_one:
            fcheck_e(f'{tag} v on a first step', sl, v, (self.g0.double() ** 2).float(), fresh)
            if not decay:
                fcheck_e(f'{tag} w on a first step', sl, w, self.w0, fresh)

        # float64 Adopt
        g0, w0, m0, v0 = (Rv(t.double()) for t in (self.g0, self.w0, self.m0, self.v0))
        if exact_one:
            g = g0
        else:
            g = mul(g0, Rv(torch.tensor(clip[0], dtype=F64, device=dev()), clip[1]))
        if decay:
            x = self.lr * self.wd
            f_ref = f32(1.0 - x)
            ef = abs(f_ref - (1.0 - x)) + gamma(2) * x + gamma(2) * (1 + 2 * x)
            w1 = mul(w0, Rv(torch.tensor(f_ref, dtype=F64, device=dev()), ef))
        else:
            w1 = w0
        if decay:
            fcheck_f(f'{tag} w (first step, decay)', sl, w, w1.v, w1.e, fresh)
        else:
            fcheck_e(f'{tag} w on a first step without decay', sl, w, self.w0, fresh)
        vg = mul(g, g)
        if not exact_one:
            fcheck_f(f'{tag} v (first step)', sl, v, vg.v, vg.e, fresh)
        c1, c2 = f32(1.0 - self.betas[0]), f32(1.0 - self.betas[1])
        sq = v0.v.clamp(min=0).sqrt()
        dd = Rv(torch.maximum(sq, torch.full_like(sq, EPS)), torch.maximum(U * sq, torch.full_like(sq, abs(f32(EPS) - EPS))))
        uu = div(g, dd)
        mr = axpy(sub(uu, m0), c1, m0)
        lr = Rv(torch.tensor(self.lr, dtype=F64, device=dev()), abs(f32(self.lr) - self.lr))
        wr = _rnd(w1.v - lr.v * mr.v, w1.e + lr.mag() * mr.e + lr.e * mr.v.abs(), 2)
        vr = axpy(sub(vg, v0), c2, v0)
        fcheck_f(f'{tag} m (beta1 {self.betas[0]})', sl, m, mr.v, mr.e, cont)
        fcheck_f(f'{tag} w', sl, w, wr.v, wr.e, cont)
        fcheck_f(f'{tag} v (beta2 {self.betas[1]})', sl, v, vr.v, vr.e, cont)

        # EMA, from the w the kernel wrote
        if self.ema_mode == 0:
            fcheck_e(f'{tag} EMA buffer in mode 0', sl, e, self.e0, sl.valid | sl.pad)
            return
        fcheck_e(f'{tag} EMA padding', sl, e, self.e0, sl.pad)
        if self.ema_mode == 2:
            fcheck_e(f'{tag} EMA copy', sl, e, w, sl.valid)
        else:
            er = axpy(sub(Rv(w.double()), Rv(self.e0.double())), f32(self.ema_weight), Rv(self.e0.double()))
            fcheck_f(f'{tag} EMA lerp', sl, e, er.v, er.e, sl.valid)


def _adopt_inputs(sl, params, gen_seed, zero_grad, first_c):
    """flat g, m, v, EMA with the populations of the module docstring; padding slots hold SENTINEL"""
    n = sl.lay.total
    gen = torch.Generator(device=dev()).manual_seed(gen_seed)
    k = torch.arange(n, device=dev())
    g = torch.randn(n, generator=gen, device=dev()) * 0.5
    w = torch.randn(n, generator=gen, device=dev())
    m = torch.randn(n, generator=gen, device=dev()) * 0.3
    v = (torch.randn(n, generator=gen, device=dev()) * 0.5).square() * (0.5 + torch.rand(n, generator=gen, device=dev()) * 1.5)
    e = torch.randn(n, generator=gen, device=dev())
    v = torch.where(k % 7 == 3, 0.0, v)                                  # eps side of the max, g != 0
    small = k % 7 == 5                                                    # v << g^2 with m = 0
    v = torch.where(small, (g * 2.0 ** -12).square(), v)
    m = torch.where(small, 0.0, m)
    if zero_grad:
        g = torch.zeros_like(g)
    first = sl.valid & first_c[sl.chunk_of.clamp(min=0)]
    m = torch.where(first, float('nan'), m)                               # a first step must not read m or v
    v = torch.where(first, float('nan'), v)
    for t in (g, m, v, e, w):
        t[sl.pad] = SENTINEL
    sl.scatter(w, params)
    return g, m, v, e


_LAYOUTS = {}


def adopt_layout(pkg, which):
    if which not in _LAYOUTS:
        names, params = layout_params(which)
        lay = pkg.optim.FlatLayout(params)
        _LAYOUTS.clear()
        _LAYOUTS[which] = (Slots(lay, names), params)
    return _LAYOUTS[which]


@pytest.mark.parametrize('which', ['edge', 'cfg2'])
@pytest.mark.parametrize('betas', BETAS, ids=['b0.99', 'b0.9999'])
@pytest.mark.parametrize('case', CASES, ids=[f'ema{c[0]}-wd{c[1]:g}-{c[2]}' for c in CASES])
def test_adopt_step(pkg, which, betas, case):
    ema_mode, weight_decay, clip_kind = case
    sl, params = adopt_layout(pkg, which)
    lay = sl.lay
    gen = torch.Generator(device=dev()).manual_seed(2 * CASES.index(case) + BETAS.index(betas))
    first_c = torch.rand(lay.n_chunks, generator=gen, device=dev()) < 0.4
    chunk_state = torch.where(first_c, 0, 1).to(I32)
    used = torch.tensor([0.0 if i % 4 == 1 else 1.0 for i in range(len(params))], device=dev())
    assert any(p.data_ptr() % 16 for p in params) and any(p.data_ptr() % 16 == 0 for p in params)   # both paths of the kernel
    g, m, v, e = _adopt_inputs(sl, params, 100 + 2 * CASES.index(case) + BETAS.index(betas), clip_kind == 'zero', first_c)
    if clip_kind == 'off':
        ns, clip = None, None
    else:
        ns = torch.tensor([NORM_SQ[clip_kind]], device=dev(), dtype=F32)
        clip = clip_rv(NORM_SQ[clip_kind], MAX_NORM)
        if clip_kind == 'above' or clip_kind == 'zero':
            assert clip == (1.0, 0.0)
        if clip_kind == 'below':
            assert clip[0] < 0.5
    call = AdoptCall(pkg, sl, params, betas, weight_decay, ema_mode, ns, MAX_NORM if ns is not None else 0.0, used, chunk_state)
    call.run(g, m, v, e)
    call.check(m, v, e, clip, f'{which} betas {betas} ema_mode {ema_mode} wd {weight_decay} clip {clip_kind}')


def test_adopt_step_nan_gradient_norm_spreads(pkg):
    """clip_grad_norm_ clamps a NaN total norm to NaN, so every clipped gradient and every live parameter becomes NaN; parameters
    without a gradient keep w, m and v"""
    sl, params = adopt_layout(pkg, 'edge')
    lay = sl.lay
    cs = torch.ones(lay.n_chunks, dtype=I32, device=dev())
    used = torch.tensor([0.0 if i == 3 else 1.0 for i in range(len(params))], device=dev())
    g, m, v, e = _adopt_inputs(sl, params, 5, False, cs == 0)
    ns = torch.tensor([float('nan')], device=dev(), dtype=F32)
    call = AdoptCall(pkg, sl, params, BETAS[0], 0.0, 1, ns, MAX_NORM, used, cs)
    call.run(g, m, v, e)
    live = sl.valid & (sl.pid != 3)
    w = sl.flat(params)
    for name, t in (('w', w), ('m', m), ('v', v), ('EMA', e)):
        bad = live & ~torch.isnan(t)
        if bool(bad.any()):
            i = int(bad.nonzero()[0, 0])
            raise AssertionError(f'NaN gradient norm: {name} at {sl.where(i)} is {t[i].item()!r}, want NaN ({int(bad.sum())} elements)')
    stale = sl.valid & (sl.pid == 3)
    for name, got, want in (('w', w, call.w0), ('m', m, call.m0), ('v', v, call.v0)):
        fcheck_e(f'NaN gradient norm: {name} of the parameter without a gradient', sl, got, want, stale)


# ------------------------------------------------------------------------------------------------- FusedAdoptEMA over a schedule
class RecordingEMA(OO.EMA):
    """the restated ema-pytorch schedule over one dummy weight, recording what each update does"""

    def __init__(self, **kw):
        super().__init__([torch.zeros(1, dtype=F64)], **kw)
        self.events = []

    def _copy(self):
        self.events.append('copy')
        super()._copy()

    def get_current_decay(self):
        d = super().get_current_decay()
        self.events.append(('lerp', d))
        return d

    def decide(self):
        """-> (mode, weight) of the next update: a copy followed by a lerp between equal weights is a copy"""
        self.events = []
        self.update()
        if not self.events:
            return 0, 0.0
        if self.events[0] == 'copy':
            return 2, 0.0
        return 1, 1.0 - self.events[0][1]


def _ema_recorder(opt):
    rec = []
    orig = opt._ema_action

    def wrapped():
        r = orig()
        rec.append(r)
        return r

    opt._ema_action = wrapped
    return rec


def test_fused_adopt_ema_schedule_cfg2(pkg):
    names, params = layout_params('cfg2')
    text = [bool(TEXT.search(n)) for n in names]
    grads = grad_tensors('cfg2', [tuple(p.shape) for p in params])
    kw = dict(lr=1e-3, betas=(0.9, 0.99), eps=EPS, weight_decay=1e-5, max_grad_norm=MAX_NORM, ema=True, ema_update_after_step=4,
              ema_update_every=3)
    opt = pkg.optim.FusedAdoptEMA(params, **kw)
    sl = Slots(opt.layout, names)
    gen = torch.Generator(device=dev()).manual_seed(21)
    wflat = torch.randn(opt.layout.total, generator=gen, device=dev())
    sl.scatter(wflat, params)
    remas = RecordingEMA(update_after_step=4, update_every=3)
    rec = _ema_recorder(opt)
    clipped = set()
    seen_modes = set()
    for step in range(25):
        if step == 12:
            opt.lr = 3e-4
        scale = 3e-4 if step % 4 in (1, 2) else 1e-5          # |g| ~ 8000 scale: clipped on some steps only
        gflat = torch.randn(opt.layout.total, generator=gen, device=dev()) * scale
        sl.scatter(gflat, grads)
        absent = step in (0, 1, 2, 7)
        for p, gr, t in zip(params, grads, text):
            p.grad = None if (absent and t) else gr
        gref = sl.flat([None if (absent and t) else gr for gr, t in zip(grads, text)], fill=0.0)
        m0, v0, e0 = opt.m.clone(), opt.v.clone(), opt.ema.clone()
        call = AdoptCall(pkg, sl, params, kw['betas'], kw['weight_decay'], 0, None, MAX_NORM, opt.sync.used, opt.chunk_state, lr=opt.lr)
        call.g0, call.w0, call.m0, call.v0, call.e0, call.cs0 = gref, sl.flat(params), m0, v0, e0, opt.chunk_state.clone()
        opt.step()
        tag = f'schedule step {step}'
        fcheck_e(f'{tag}: gathered gradients', sl, opt.sync.flat, gref, sl.valid)
        ns = _sumsq64(gref)
        nsb = sumsq_bound(opt.layout.total, True, ns)
        got = float(opt.norm_sq)
        assert abs(got - ns) <= nsb, f'{tag}: norm^2 got {got!r}, ref {ns!r}, bound {nsb:.3g}'
        rel = nsb / ns
        gn, gref_n = float(opt.grad_norm()), math.sqrt(ns)
        gb = (rel / (1 + math.sqrt(1 - rel)) + U) * gref_n
        assert abs(gn - gref_n) <= gb, f'{tag}: grad_norm() got {gn!r}, ref {gref_n!r}, bound {gb:.3g}'
        clip = clip_rv(ns, MAX_NORM, rel)
        if clip[0] < 1:
            clipped.add(step)
        mode, weight = remas.decide()
        assert rec[-1] == (mode, weight), f'{tag}: EMA action {rec[-1]} != restated {(mode, weight)}'
        seen_modes.add(mode)
        call.ema_mode, call.ema_weight = mode, weight
        call.check(opt.m, opt.v, opt.ema, clip, tag)
    assert 0 < len(clipped) < 25 and seen_modes == {0, 1, 2}

    # copy_ema_to into a deep copy of a module whose parameters sit at misaligned storage offsets
    mod = torch.nn.ParameterList([torch.nn.Parameter(p.detach().clone(), requires_grad=False) for p in params])
    twin = copy.deepcopy(mod)
    for p, q in zip(twin.parameters(), packed_params([tuple(p.shape) for p in params], 3)):
        q.fill_(float('nan'))
        p.data = q
    assert sum(int(p.data_ptr() % 16 != 0) for p in twin.parameters()) > len(params) // 2
    opt.copy_ema_to(twin.parameters())
    for i, (p, e) in enumerate(zip(twin.parameters(), opt.ema_parameters())):
        check_e(f'copy_ema_to {names[i]}', p.detach(), e)


# ------------------------------------------------------------------------------------------------------------------- resume
@pytest.mark.parametrize('split', [2, 8], ids=['copy_phase', 'after_copy_phase'])
def test_resume_is_bit_identical(pkg, split):
    """state_dict() through torch.save / torch.load into a new optimiser over a deep copy: 5 more identical steps agree bit for bit"""
    names, params = layout_params('edge')
    mod = torch.nn.ParameterList([torch.nn.Parameter(p, requires_grad=False) for p in params])
    gen = torch.Generator(device=dev()).manual_seed(31)
    for p in mod.parameters():
        p.data.copy_(torch.randn(p.shape, generator=gen, device=dev()))
    kw = dict(lr=1e-3, weight_decay=1e-5, max_grad_norm=MAX_NORM, ema=True, ema_update_after_step=4, ema_update_every=3)
    opt = pkg.optim.FusedAdoptEMA(list(mod.parameters()), **kw)
    grads = [[torch.randn(p.shape, generator=gen, device=dev()) * (0.3 if s % 2 else 3e-3) for p in params] for s in range(split + 5)]

    def step(o, module, s):
        for i, (p, g) in enumerate(zip(module.parameters(), grads[s])):
            p.grad = None if (i == 2 and s in (0, 1, 2, 7)) else g.clone()
        o.step()

    for s in range(split):
        step(opt, mod, s)
    blob = io.BytesIO()
    torch.save(opt.state_dict(), blob)
    blob.seek(0)
    twin = copy.deepcopy(mod)
    opt2 = pkg.optim.FusedAdoptEMA(list(twin.parameters()), **kw)
    opt2.load_state_dict(torch.load(blob))
    for s in range(split, split + 5):
        step(opt, mod, s)
        step(opt2, twin, s)
        tag = f'resumed after {split} steps, step {s}'
        for i, (a, b) in enumerate(zip(mod.parameters(), twin.parameters())):
            check_e(f'{tag}: w of {names[i]}', b.detach(), a.detach())
        for name in ('m', 'v', 'ema', 'chunk_state'):
            check_e(f'{tag}: {name}', getattr(opt2, name), getattr(opt, name))
        check_e(f'{tag}: grad_norm()', opt2.grad_norm(), opt.grad_norm())
