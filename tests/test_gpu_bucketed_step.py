"""GPU: graphed training steps on ragged batches (e2_tts_pytorch_b200.BucketedTrainStep) and the kernel under their gradient
accumulation (b200_flat_accumulate).

  * the kernel over FlatLayout chunk tables — sizes around the 16 Ki chunk at storage offsets 1 / 2 / 3, and the cfg2 parameter
    shapes — three accumulations with different scales and NULL pointers, bit for bit against the float32 fmaf sequence restated in
    exact arithmetic; NULL slots and padding sentinels untouched, `used` the OR of the presence flags;
  * one micro-step per bucket with the randomness pinned (as model_checks.graphed_matches_eager does) against the eager step at the
    padded shape and at the unpadded shape with the same noise cropped: padding changes neither the loss nor a gradient;
  * k = 3 micro-batches from three buckets in both text modes against eager `(loss / 3).backward()` accumulated by autograd (the
    randomness pinned by re-seeding torch's CUDA generator, whose graph-safe state gives a replay the eager draws); every micro-step
    dropping the text leaves the text stream unused and FusedAdoptEMA leaves it bit for bit;
  * one shared memory pool: replays A, B, A give A's results twice, and take less memory than one GraphedTrainStep per bucket;
  * two ranks (skipped on one GPU): k = 2 equals one rank on the concatenated micro-batches, with one all-reduce per optimiser step.
"""
import math
import os
import random
import re
import socket
import traceback

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2
from kernel_checks import dev, pkg, stream  # noqa: F401  (pkg is a fixture)
from oracle import e2tts_oracle as O

pytestmark = pytest.mark.gpu

F32 = torch.float32
I32 = torch.int32
CHUNK = 16384
SENTINEL = -1234.5
EDGE_SHAPES = [(1,), (3,), (4,), (5,), (16383,), (16384,), (16385,), (3 * CHUNK + 5,), (129, 515)]
EDGE_SHIFT = [0, 1, 0, 2, 3, 0, 1, 3, 2]        # storage offsets of the gradients: 1, 2, 3 take the scalar path
TEXT = re.compile(r'(text|^transformer\.(layers|hyper_conns)\.\d+\.1\.)')   # parameters without a gradient when the text is dropped


# ------------------------------------------------------------------------------------------------------------------ kernel
def fma_f32(s, g, a):
    """fp32 fmaf(s, g, a) element-wise, restated exactly: s * g is exact in float64; the sum is split into hi + lo (TwoSum) and
    rounded to odd before the one rounding to fp32, so no double rounding (53 >= 24 + 2 bits)"""
    p = s.double() * g.double()
    a = a.double()
    hi = p + a
    bb = hi - p
    lo = (p - (hi - bb)) + (a - bb)
    even = (hi.view(torch.int64) & 1) == 0
    toward = torch.where(lo > 0, torch.full_like(hi, math.inf), torch.full_like(hi, -math.inf))
    hi = torch.where((lo != 0) & even, torch.nextafter(hi, toward), hi)
    return hi.float()


def _edge_tensors(shifts):
    out = []
    for s, k in zip(EDGE_SHAPES, shifts):
        n = math.prod(s)
        out.append(torch.zeros(n + 4, device=dev(), dtype=F32)[k:k + n].view(s))
    return out


def _cfg2_tensors(start):
    m = pkg_module().E2TTS(transformer=dict(dim=512, depth=8, heads=8), use_vocos=False)
    names = [n for n, _ in m.named_parameters()]
    shapes = [tuple(p.shape) for p in m.parameters()]
    numels = [math.prod(s) for s in shapes]
    buf = torch.zeros(start + sum(numels), device=dev(), dtype=F32)
    out, o = [], start
    for s, n in zip(shapes, numels):
        out.append(buf[o:o + n].view(s))
        o += n
    return names, out


def pkg_module():
    import e2_tts_pytorch_b200
    return e2_tts_pytorch_b200


@pytest.mark.parametrize('which', ['edge', 'cfg2'])
def test_flat_accumulate_is_the_fmaf_sequence(pkg, which):
    if which == 'edge':
        params = _edge_tensors([0] * len(EDGE_SHAPES))
        names = [f'edge{i}' for i in range(len(params))]
        nulls = [{2, 3, 7}, {0, 3, 7}, {3, 5, 7}]      # 3 and 7 never have a gradient; 7's flag starts set and must stay set
        pre_used = {7}
    else:
        names, params = _cfg2_tensors(0)
        text = {i for i, n in enumerate(names) if TEXT.search(n)}
        assert len(text) > 20
        nulls = [text, set(), text | {0}]
        pre_used = set()
    lay = pkg.optim.FlatLayout(params)
    gen = torch.Generator().manual_seed(3)
    flat = torch.full((lay.total,), SENTINEL, device=dev(), dtype=F32)
    valid = torch.zeros(lay.total, dtype=torch.bool, device=dev())
    for o, n in zip(lay.offsets, lay.numels):
        flat[o:o + n] = torch.randn(n, generator=gen).to(dev())
        valid[o:o + n] = True
    assert int((~valid).sum()) > 0
    used = torch.tensor([1.0 if i in pre_used else 0.0 for i in range(len(params))], device=dev())
    want, want_used = flat.clone(), used.clone()
    for step, (scale, none) in enumerate(zip((1.0 / 3.0, 0.25, 1.7), nulls)):
        scale = float(torch.tensor(scale, dtype=F32))
        grads = _edge_tensors(EDGE_SHIFT) if which == 'edge' else _cfg2_tensors(1 + step)[1]
        for g in grads:
            g.view(-1).copy_(torch.randn(g.numel(), generator=gen).to(dev()))
        if which == 'edge':
            grads[4].view(-1)[:3] = -grads[4].view(-1)[:3]      # sign changes inside a misaligned chunk
            assert any(g.data_ptr() % 16 for g in grads) and any(g.data_ptr() % 16 == 0 for g in grads)
        grads = [None if i in none else g for i, g in enumerate(grads)]
        pkg.lib.call('b200_flat_accumulate', lay.table(grads), lay.n_chunks, flat, scale, used, stream())
        s = torch.tensor(scale, dtype=F32, device=dev())
        for i, (o, n, g) in enumerate(zip(lay.offsets, lay.numels, grads)):
            if g is not None:
                want[o:o + n] = fma_f32(s, g.reshape(-1), want[o:o + n])
                want_used[i] = 1.0
        torch.cuda.synchronize()
        bad = (flat.view(I32) != want.view(I32))
        assert not bool(bad.any()), f'{which} step {step}: {int(bad.sum())} slots differ from the fmaf sequence (padding: {int((bad & ~valid).sum())})'
        assert torch.equal(used, want_used), (which, step)
    assert bool((flat[~valid] == SENTINEL).all())
    if which == 'edge':
        assert used.tolist() == [1.0, 1.0, 1.0, 0.0, 1.0, 1.0, 1.0, 1.0, 1.0]


# ------------------------------------------------------------------------------------------------------------- whole steps
def _model(pkg, cls='E2TTS', seed=0, tkw=None, **e2kw):
    torch.manual_seed(seed)
    random.seed(seed)
    t = dict(dim=128, depth=2, heads=2, dropout=0., max_seq_len=256, **(tkw or {}))
    m = pkg.E2TTS(transformer=t, use_vocos=False, **e2kw) if cls == 'E2TTS' else pkg.DurationPredictor(transformer=t)
    m.load_state_dict(O.randomize_zero_init({k: v.clone() for k, v in m.state_dict().items()}, seed=seed + 1))
    return m.to(dev()).train()


def _grads(model):
    return {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}


def _clear(model):
    for p in model.parameters():
        p.grad = None


def _loss(out):
    return out if torch.is_tensor(out) else out.loss


def _close(tag, got_loss, got, want_loss, want):
    """model_checks.graphed_matches_eager's bounds: loss within 1e-3 |loss| + 1e-5, the same parameters with a gradient, each within
    rel-L2 2e-3"""
    assert abs(got_loss - want_loss) <= 1e-3 * abs(want_loss) + 1e-5, (tag, got_loss, want_loss)
    assert set(got) == set(want), (tag, sorted(set(got) ^ set(want))[:5])
    for n in want:
        e = rel_l2(got[n].float().cpu(), want[n].float().cpu())
        assert e < 2e-3 or float(want[n].norm()) == 0, (tag, n, e)


def _grads_close(tag, got, want, rel=1e-2):
    """accumulated gradients against autograd's sum of `(loss / k).backward()`: the same parameters with a gradient, the whole gradient
    (all parameters in one vector) within rel-L2 `rel`, and every parameter not negligible next to the largest (>= 1e-3 of its norm)
    pointing the same way, cosine >= 0.98. Looser than _close because the eager side runs its bf16 backward on a loss scaled by 1 / k
    and the graphs scale the fp32 gradient afterwards: the bf16 roundings differ (0.6 % on the whole gradient, 0.8 % on
    abs_pos_emb, whose rows are sums over few items and keep that rounding nearly unaveraged)"""
    assert set(got) == set(want), (tag, sorted(set(got) ^ set(want))[:5])
    names = sorted(want)
    g_all = torch.cat([got[n].double().flatten().cpu() for n in names])
    w_all = torch.cat([want[n].double().flatten().cpu() for n in names])
    e_all = rel_l2(g_all, w_all)
    top = max(float(want[n].norm()) for n in names)
    worst_c, worst_n = 2.0, ''
    for n in names:
        g, w = got[n].double().flatten().cpu(), want[n].double().flatten().cpu()
        if float(w.norm()) < 1e-3 * top:
            continue
        c = float((g @ w) / (g.norm() * w.norm() + 1e-30))
        if c < worst_c:
            worst_c, worst_n = c, n
    print(f'{tag}: whole-gradient rel-L2 {e_all:.3g}, lowest cosine {worst_c:.5f} ({worst_n})')
    assert e_all < rel, (tag, e_all)
    assert worst_c >= 0.98, (tag, worst_n, worst_c)


def _flat_grads(step, model):
    used = step.grad_sync.used.tolist()
    return {n: v.detach().clone() for (n, _), v, u in zip(model.named_parameters(), step.grad_sync.grad_views, used) if u > 0}


CASES = {
    'text': dict(cls='E2TTS', drop=False),
    'dropped': dict(cls='E2TTS', drop=True),
    'duration': dict(cls='DurationPredictor', drop=False),
    'plain_residual': dict(cls='E2TTS', drop=False, tkw=dict(num_residual_streams=1)),
    'interpolated_text': dict(cls='E2TTS', drop=False, interpolated_text=True),
}


@pytest.mark.parametrize('case', list(CASES))
def test_one_micro_step_matches_eager_padded_and_unpadded(pkg, case):
    c = dict(CASES[case])
    cls, drop = c.pop('cls'), c.pop('drop')
    model = _model(pkg, cls, seed=11, **c)
    # n = 152: (n + 32 registers) * B * 4 streams is a multiple of 64 at both lengths, so the padded and the unpadded step take the
    # same hyper-connection backward schedule (ops.hc_can_fuse); a different schedule rounds differently, beyond these bounds
    B, n, nb = 2, 152, 192
    g = torch.Generator().manual_seed(5)
    mel = torch.randn(B, n, 100, generator=g).to(dev())
    lens = torch.tensor([n, n - 23], device=dev())
    text = pkg.list_str_to_tensor(['Hello there', 'Goodbye']).to(dev())
    if cls == 'E2TTS':
        model.cond_drop_prob = 1.0 if drop else 0.0
        span = torch.zeros(B, nb, dtype=torch.bool)
        span[0, 30:120] = True
        span[1, 5:100] = True
        rnd = dict(x0=torch.randn(B, nb, 100, generator=g).to(dev()), times=torch.rand(B, generator=g).to(dev()), span_mask=span.to(dev()),
                   drop_text_cond=drop)
        crop = dict(rnd, x0=rnd['x0'][:, :n].contiguous(), span_mask=rnd['span_mask'][:, :n].contiguous())
    else:
        rnd = dict(duration_rand_frac=torch.tensor([0.4, 0.8], device=dev()))
        crop = rnd
    mel_p = F.pad(mel, (0, 0, 0, nb - n))
    with pkg.inject_randomness(**rnd):             # (a) eager at the padded shape
        out = model(mel_p, text=text, lens=lens)
        _loss(out).backward()
    want_pad_loss, want_pad = float(_loss(out).detach()), _grads(model)
    del out
    _clear(model)
    with pkg.inject_randomness(**crop):            # (b) eager at the unpadded shape, the same noise cropped
        out = model(mel, text=text, lens=lens)
        _loss(out).backward()
    want_loss, want = float(_loss(out).detach()), _grads(model)
    del out
    _clear(model)
    _close(f'{case}: padded vs unpadded eager', want_pad_loss, want_pad, want_loss, want)
    with pkg.inject_randomness(**rnd):
        step = pkg.BucketedTrainStep(model, B, (nb,), grad_accumulation_steps=1)
    assert step.sync_gradients is False and set(step.graphs) == {(nb, drop)}
    got_loss = float(step(mel, text=text, lens=lens))
    torch.cuda.synchronize()
    assert step.sync_gradients
    got = _flat_grads(step, model)
    print(f'{case}: loss {got_loss:.6f} (eager padded {want_pad_loss:.6f}, unpadded {want_loss:.6f}), {step.launches_per_step} launches, '
          f'capture {step.capture_seconds:.2f} s')
    _close(f'{case}: graphed vs padded eager', got_loss, got, want_pad_loss, want_pad)
    _close(f'{case}: graphed vs unpadded eager', got_loss, got, want_loss, want)
    assert all(p.grad is v for p, v in zip(model.parameters(), step.grad_sync.grad_views))
    del rnd, crop


def _seed_for(pattern, p):
    """a python seed whose first draws against cond_drop_prob p give `pattern` (True = drop the text)"""
    for s in range(10000):
        r = random.Random(s)
        if [r.random() < p for _ in pattern] == list(pattern):
            return s
    raise AssertionError('no seed')


def test_accumulation_over_three_buckets_matches_eager(pkg):
    model = _model(pkg, seed=21, cond_drop_prob=0.5)
    B, k = 2, 3
    sizes, buckets = (80, 150, 230), (96, 160, 256)
    g = torch.Generator().manual_seed(9)
    mels = [torch.randn(B, n, 100, generator=g).to(dev()) for n in sizes]
    lens = [torch.tensor([n, n - 11], device=dev()) for n in sizes]
    texts = [pkg.list_str_to_tensor(['Hello there', 'Goodbye']).to(dev()),
             pkg.list_str_to_tensor(['a', 'bcd']).to(dev()),
             pkg.list_str_to_tensor(['the third one', 'x' * 40]).to(dev())]
    pattern = (False, True, False)
    # eager reference: (loss / k).backward() accumulated by autograd, each micro-batch at its bucket's padded shape with the CUDA
    # generator re-seeded, so it draws what the replay draws
    for i in range(k):
        torch.cuda.manual_seed(100 + i)
        nb = buckets[i]
        with pkg.inject_randomness(drop_text_cond=pattern[i]):
            out = model(F.pad(mels[i], (0, 0, 0, nb - sizes[i])), text=texts[i], lens=lens[i])
        (out.loss / k).backward()
        del out
    want = _grads(model)
    _clear(model)
    with pkg.inject_randomness(drop_text_cond=True):     # the text stream: what gets no gradient when the text is dropped
        out = model(mels[0], text=texts[0], lens=lens[0])
    out.loss.backward()
    del out
    text_names = {n for n, p in model.named_parameters() if p.grad is None}
    _clear(model)
    assert len(text_names) > 10 and text_names <= set(want)

    random.seed(1234)
    before = random.getstate()
    step = pkg.BucketedTrainStep(model, B, buckets, grad_accumulation_steps=k)
    assert random.getstate() == before, 'construction moved python random state'
    assert set(step.graphs) == {(nb, d) for nb in buckets for d in (False, True)}
    random.seed(_seed_for(pattern, 0.5))
    losses = []
    for i in range(k):
        torch.cuda.manual_seed(100 + i)
        losses.append(step(mels[i], text=texts[i], lens=lens[i]))
        assert step.sync_gradients == (i == k - 1)
    torch.cuda.synchronize()
    _grads_close('k = 3 over three buckets', _flat_grads(step, model), want)
    assert all(float(x) == float(x) and float(x) > 0 for x in losses)

    # every micro-step drops the text: the text stream is unused, and the optimiser leaves it alone
    model.cond_drop_prob = 1.0
    step = pkg.BucketedTrainStep(model, B, buckets, grad_accumulation_steps=k)
    assert set(step.graphs) == {(nb, True) for nb in buckets}
    for i in range(k):
        step(mels[i], text=texts[i], lens=lens[i])
    torch.cuda.synchronize()
    used = dict(zip([n for n, _ in model.named_parameters()], step.grad_sync.used.tolist()))
    assert all(used[n] == 0.0 for n in text_names) and sum(used.values()) > 0
    assert all((used[n] == 0.0) == (n in text_names) for n in used)
    opt = pkg.FusedAdoptEMA(list(model.parameters()), lr=1e-3, grad_sync=step.grad_sync)
    before = {n: p.detach().clone() for n, p in model.named_parameters()}
    opt.step(step.grad_sync.flat)
    opt.step(step.grad_sync.flat)    # past Adopt's first (initialising) step
    torch.cuda.synchronize()
    changed = {n for n, p in model.named_parameters() if not torch.equal(p.detach().view(I32), before[n].view(I32))}
    assert changed and not (changed & text_names), sorted(changed & text_names)[:5]


def test_shared_pool_replays_do_not_interfere(pkg):
    model = _model(pkg, seed=31, cond_drop_prob=0.0)
    B = 2
    g = torch.Generator().manual_seed(4)
    mel_a, mel_b = torch.randn(B, 90, 100, generator=g).to(dev()), torch.randn(B, 240, 100, generator=g).to(dev())
    text = pkg.list_str_to_tensor(['Hello there', 'Goodbye']).to(dev())
    step = pkg.BucketedTrainStep(model, B, (96, 256))
    torch.cuda.manual_seed(7)
    loss_a1 = float(step(mel_a, text=text))
    grads_a1 = step.grad_sync.flat.clone()
    buf_a = step._loss[96, False]
    torch.cuda.manual_seed(8)
    loss_b = float(step(mel_b, text=text))
    torch.cuda.synchronize()
    assert float(buf_a) == loss_a1, 'replaying B changed the loss buffer of A'
    torch.cuda.manual_seed(7)
    loss_a2 = float(step(mel_a, text=text))
    grads_a2 = step.grad_sync.flat.clone()
    torch.cuda.synchronize()
    print(f'pool: loss A {loss_a1:.6f} / {loss_a2:.6f}, B {loss_b:.6f}')
    assert abs(loss_a2 - loss_a1) <= 1e-5 * abs(loss_a1), (loss_a1, loss_a2)
    assert rel_l2(grads_a2, grads_a1) < 1e-4
    assert loss_b != loss_a1


def test_one_pool_takes_less_memory_than_one_graph_per_bucket(pkg):
    model = _model(pkg, seed=41, cond_drop_prob=0.0)
    B, buckets = 4, (128, 192, 256)
    text = pkg.list_str_to_tensor(['Hello there', 'Goodbye', 'a', 'bc']).to(dev())
    for nb in buckets:           # the caches both sides share (packed weights, rotary tables) exist before either is measured
        out = model(torch.randn(B, nb, 100, device=dev()), text=text)
        out.loss.backward()
        del out
        _clear(model)
    torch.cuda.synchronize()

    def reserved():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        return torch.cuda.memory_reserved()

    r0 = reserved()
    step = pkg.BucketedTrainStep(model, B, buckets)
    shared = reserved() - r0
    del step
    _clear(model)
    r0 = reserved()
    separate = [pkg.GraphedTrainStep(model, torch.randn(B, nb, 100, device=dev()), text=text) for nb in buckets]
    apart = reserved() - r0
    print(f'graph memory for buckets {buckets}: one shared pool {shared / 2**20:.1f} MiB, one GraphedTrainStep per bucket '
          f'{apart / 2**20:.1f} MiB')
    del separate
    assert shared < apart


# ------------------------------------------------------------------------------------------------------------------ two ranks
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, errs):
    try:
        os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
        import torch.distributed as dist
        import e2_tts_pytorch_b200 as pkg
        torch.cuda.set_device(rank)
        d = torch.device('cuda', rank)
        dist.init_process_group('nccl', device_id=d)
        model = _model(pkg, seed=51, cond_drop_prob=0.0)
        pkg.broadcast_module(model)
        B, N, k = 2, 96, 2
        g = torch.Generator().manual_seed(5)
        mels = [torch.randn(2 * B, N, 100, generator=g).to(d) for _ in range(k)]      # micro-step j: items 2r, 2r+1 on rank r
        x0 = torch.randn(2 * B, N, 100, generator=g).to(d)
        times = torch.rand(2 * B, generator=g).to(d)
        span = torch.zeros(2 * B, N, dtype=torch.bool)
        for b in range(2 * B):
            span[b, 10 + 3 * b: 60 + 3 * b] = True     # the same span length on every item: mean of rank means == global mean
        span = span.to(d)
        text = pkg.list_str_to_tensor(['Hello', 'Goodbye', 'Good morning', 'Hi']).to(d)
        mine = slice(B * rank, B * rank + B)
        # one rank on the concatenated micro-batches: (loss / k).backward() accumulated over the k micro-steps
        for j in range(k):
            with pkg.inject_randomness(x0=x0, times=times, span_mask=span, drop_text_cond=False):
                out = model(mels[j], text=text)
            (out.loss / k).backward()
            del out
        want = _grads(model)
        _clear(model)
        with pkg.inject_randomness(x0=x0[mine].contiguous(), times=times[mine].contiguous(), span_mask=span[mine].contiguous(),
                                   drop_text_cond=False):
            step = pkg.BucketedTrainStep(model, B, (N,), grad_accumulation_steps=k)
        assert step.grad_sync.world == world
        calls = []
        real = dist.all_reduce

        def counted(*a, **kw):
            calls.append(1)
            return real(*a, **kw)

        dist.all_reduce = counted
        try:
            for window in range(2):
                n_before = len(calls)
                for j in range(k):
                    step(mels[j][mine].contiguous(), text=text[mine].contiguous())
                assert step.sync_gradients and len(calls) - n_before == 1, (window, len(calls) - n_before)
        finally:
            dist.all_reduce = real
        torch.cuda.synchronize()
        _grads_close('two ranks', {n: p.grad for n, p in model.named_parameters() if n in want}, want)
        dist.barrier()
        dist.destroy_process_group()
    except Exception:  # noqa: BLE001
        errs.put((rank, traceback.format_exc()))
        raise


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_ranks_accumulate_then_one_all_reduce():
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    errs = ctx.SimpleQueue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, errs)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
    msgs = []
    while not errs.empty():
        msgs.append(errs.get())
    for p in procs:
        if p.is_alive():
            p.kill()
            msgs.append((-1, 'worker timed out'))
    assert not msgs and all(p.exitcode == 0 for p in procs), '\n'.join(f'rank {r}:\n{m}' for r, m in msgs)
