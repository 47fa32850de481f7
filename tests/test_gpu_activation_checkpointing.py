"""Transformer(checkpoint_activations=True) on the GPU: each layer's audio sub-blocks and each text block run as one ops.Segment, which
keeps only its inputs and runs the sub-blocks again in the backward.

Checked against the plain step of the same model, weights and draws: loss and prediction bit for bit; every gradient that two plain
runs reproduce bit for bit is reproduced bit for bit, the others (fp32 atomics) stay within the graphed-step bound rel-L2 2e-3; and
every gradient holds the oracle bounds of model_checks.whole_model. The recompute draws the forward's dropout seeds (tests/
dropout_ref.py's recorder); memory held for the backward per layer is what the boundary tensors take; the peak of a cfg2 step
drops; the step launches the plain step's kernels plus one more forward of the segments; graphed and bucketed replays equal the
eager checkpointed step; eval forwards and sample() ignore the switch."""
import random
import re

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2
from dropout_ref import SeedRecorder
from kernel_checks import dev, pkg  # noqa: F401  (pytest fixture)
from model_checks import cos, graphed_matches_eager, step_inputs
from oracle import e2tts_oracle as O

pytestmark = pytest.mark.gpu

SMALL = dict(dim=128, depth=4, heads=2)
CASES = {   # transformer kwargs, E2TTS kwargs, lens (B = len(lens)), frames, dropout p, text dropped
    'default': dict(tkw=SMALL, lens=[96, 61]),
    'residual1': dict(tkw=dict(SMALL, num_residual_streams=1), lens=[96, 70]),
    'duration': dict(cls='DurationPredictor', tkw=SMALL, lens=[72, 50, 31], N=72),
    'text_dropped': dict(tkw=SMALL, lens=[96, 61], drop=True),
    'dropout0.1': dict(tkw=SMALL, lens=[96, 61], p=0.1),
    'headdim128': dict(tkw=dict(dim=256, depth=2, heads=2, dim_head=128), lens=[96, 53]),
    'fourier_input': dict(tkw=dict(SMALL, attn_fourier_embed_input=True), lens=[96, 80]),
    'interpolated_text': dict(tkw=SMALL, e2kw=dict(interpolated_text=True), lens=[96, 61]),
    'concat_cond': dict(tkw=SMALL, e2kw=dict(concat_cond=True), lens=[96, 61]),
    'ff_kwargs': dict(tkw=dict(SMALL, ff_kwargs=dict(swish=True, glu_mult_bias=True, no_bias=True)), lens=[96, 61]),
    'attn_kwargs': dict(tkw=dict(SMALL, attn_kwargs=dict(gate_value_heads=True)), lens=[96, 61]),
    'text_depth1_registers0': dict(tkw=dict(SMALL, text_depth=1, num_registers=0), lens=[96, 61]),
}
TEXT = ['Hello', 'Goodbye', 'x']
# the weights of the wgmma GEMMs: their gradients come out of split-K GEMMs with a fixed reduction order
GEMM_WEIGHT = re.compile(r'\.(to_q|to_k|to_v|to_out|proj|2|text_to_audio|audio_to_text|linear|to_v_head_gate|0)\.weight$')


@pytest.fixture(params=['two_stream', 'serial'])
def schedule(request, pkg, monkeypatch):
    if request.param == 'serial':
        monkeypatch.setattr(pkg.modules, 'TWO_STREAM', False)
    return request.param


def build(pkg, c, seed=31):
    torch.manual_seed(seed)
    random.seed(seed)
    t = dict(dropout=c.get('p', 0.), max_seq_len=max(256, c.get('N', 96)), **c['tkw'])
    cls = c.get('cls', 'E2TTS')
    model = pkg.E2TTS(transformer=t, use_vocos=False, **c.get('e2kw', {})) if cls == 'E2TTS' else pkg.DurationPredictor(transformer=t)
    sd = O.randomize_zero_init({k: v.clone() for k, v in model.state_dict().items()}, seed=seed + 1, dyn_scale=0.05)
    model.load_state_dict(sd)
    return model.to(dev()).train(), sd


def inputs(c, seed=37):
    g = torch.Generator().manual_seed(seed)
    lens = c['lens']
    B, N = len(lens), c.get('N', 96)
    span = torch.zeros(B, N, dtype=torch.bool)
    for b, n in enumerate(lens):
        span[b, n // 8: n - n // 10] = True
    return dict(mel=torch.randn(B, N, 100, generator=g), x0=torch.randn(B, N, 100, generator=g), times=torch.rand(B, generator=g),
                span=span, lens=torch.tensor(lens), rand_frac=torch.tensor([0.9, 0.6, 0.3][:B]), text=(TEXT * B)[:B])


def step(pkg, model, c, x, ckpt, backward=True):
    """one eager training step with the switch set to `ckpt`, the dropout host seed pinned -> dict(loss, pred, grads, launches
    (forward, whole step))"""
    model.transformer.checkpoint_activations = ckpt
    for p in model.parameters():
        p.grad = None
    torch.manual_seed(1234)   # the host seed of the step's dropout masks (Transformer._forward_from_h)
    if c.get('cls', 'E2TTS') == 'E2TTS':
        rnd = pkg.inject_randomness(x0=x['x0'].to(dev()), times=x['times'].to(dev()), span_mask=x['span'].to(dev()),
                                    drop_text_cond=c.get('drop', False))
    else:
        rnd = pkg.inject_randomness(duration_rand_frac=x['rand_frac'].to(dev()))
    torch.cuda.synchronize()
    n0 = pkg.lib.launch_count()
    with rnd:
        out = model(x['mel'].to(dev()), text=x['text'], lens=x['lens'].to(dev()))
    n_fwd = pkg.lib.launch_count() - n0
    loss = out if torch.is_tensor(out) else out.loss
    if backward:
        loss.backward()
    torch.cuda.synchronize()
    pred = None if torch.is_tensor(out) else out.pred_flow.detach().clone()
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
    return dict(loss=loss.detach().clone(), pred=pred, grads=grads, launches=(n_fwd, pkg.lib.launch_count() - n0))


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8))


def oracle_grads(c, sd, x):
    """(loss, prediction or None, {name: gradient}) of the fp32 oracle on the case (dropout off)"""
    osd = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    tkw = dict(c['tkw'])
    text = O.list_str_to_tensor(x['text'])
    if c.get('cls', 'E2TTS') == 'E2TTS':
        ref = O.e2tts_forward(osd, O.TransformerCfg(**tkw), x['mel'], text, x0=x['x0'], times=x['times'], span_mask=x['span'],
                              lens=x['lens'], drop_text_cond=c.get('drop', False))
        loss, pred = ref['loss'], ref['pred'].detach()
    else:
        loss, pred = O.duration_forward(osd, O.TransformerCfg(cond_on_time=False, **tkw), x['mel'], text, lens=x['lens'],
                                        rand_frac=x['rand_frac']), None
    loss.backward()
    return float(loss), pred, {k: v.grad for k, v in osd.items() if v.is_floating_point()}


@pytest.mark.parametrize('case', list(CASES))
def test_step_matches_plain_step(pkg, case, schedule):
    c = CASES[case]
    model, sd = build(pkg, c)
    x = inputs(c)
    plain1, plain2 = step(pkg, model, c, x, False), step(pkg, model, c, x, False)
    got = step(pkg, model, c, x, True)
    # 1. forward bits: the prediction. The loss's reduction adds fp32 partial sums atomically: two plain runs timed alike add them
    #    in the same order, the checkpointed step (timed differently) may not, so the loss is held to 1e-6 of itself (a few ulp)
    if got['pred'] is not None:
        assert same_bits(got['pred'], plain1['pred'])
    assert abs(float(got['loss']) - float(plain1['loss'])) <= 1e-6 * abs(float(plain1['loss']))
    # 2. gradients: bit for bit wherever the plain step reproduces itself, with one exception: the small accumulators the backward
    #    kernels add into with fp32 atomics (hyper-connection scalars and static_beta, convolution weights and biases, the embedding
    #    table) reproduce between two plain runs only because those run with the same timing; the checkpointed step's
    #    recompute changes the timing and so the order of the atomic adds, which moves them by a few ulp (rel-L2 < 1e-5). The GEMM
    #    weight gradients (split-K with a fixed order) must always come out bit for bit. Every gradient is also within
    #    model_checks.graphed_matches_eager's rel-L2 2e-3 of the plain one, and within the oracle bounds below
    assert set(got['grads']) == set(plain1['grads']) == set(plain2['grads'])
    moving, broke = [], []
    for n, want in plain1['grads'].items():
        e = rel_l2(got['grads'][n].double().cpu(), want.double().cpu())
        assert e < 2e-3 or float(want.norm()) == 0, (n, e)
        if not same_bits(want, plain2['grads'][n]):
            moving.append(n)
        elif not same_bits(got['grads'][n], want):
            broke.append((n, f'{e:.2g}', tuple(want.shape)))
    print(f'{case}/{schedule}: {len(plain1["grads"])} gradients, {len(moving)} not reproducible by the plain step itself; '
          f'atomic-order differences {len(broke)}: {broke}')
    for n, e, shape in broke:
        assert float(e) < 1e-5 and not (GEMM_WEIGHT.search(n) and len(shape) == 2), (n, e, shape)
    if c.get('p', 0.) > 0:
        return   # the dropout masks: test_recompute_draws_the_forward_masks; the plain dropout step is held to the oracle elsewhere
    # the oracle bounds of model_checks.whole_model on every gradient of the checkpointed step
    rloss, rpred, rgrads = oracle_grads(c, sd, x)
    assert abs(float(got['loss']) - rloss) <= 1e-2 * abs(rloss), (float(got['loss']), rloss)
    if rpred is not None:
        assert rel_l2(got['pred'].float().cpu(), rpred) < 3e-2
    total = float(torch.cat([g.flatten() for g in rgrads.values() if g is not None]).norm())
    for n, p in model.named_parameters():
        gr = rgrads[n]
        if gr is None:
            assert n not in got['grads'] or float(got['grads'][n].abs().max()) == 0.0, f'{n} should be unused'
            continue
        assert n in got['grads'], n
        if float(gr.norm()) < 1e-4 * total:
            continue
        c_ = cos(got['grads'][n].cpu(), gr)
        if c_ < 0.99:   # the case is ill-conditioned for this gradient on the bf16 path: the plain step misses the bound too, alike
            assert cos(plain1['grads'][n].cpu(), gr) < 0.99 and rel_l2(got['grads'][n].double().cpu(), plain1['grads'][n].double().cpu()) < 1e-5, (n, c_)
            print(f'{case}: {n} cosine {c_:.4f} against the oracle, as the plain step')


@pytest.mark.parametrize('case', ['dropout0.1', 'default'])
def test_recompute_draws_the_forward_masks(pkg, case, schedule):
    """every attention and feed-forward call runs twice, and the second run (the recompute) takes the seed, the device-word flag and
    the probability of the first: the kernels hash the same masks"""
    c = dict(CASES[case], p=0.1)
    model, _ = build(pkg, c)
    model.transformer.checkpoint_activations = True
    model.transformer._seed_dev = torch.tensor([987654321], dtype=torch.int64, device=dev())   # a device word, as the graphed steps set
    word = model.transformer._seed_dev.clone()
    x = inputs(c)
    with SeedRecorder(pkg, model) as rec:
        torch.manual_seed(1234)
        with pkg.inject_randomness(x0=x['x0'].to(dev()), times=x['times'].to(dev()), span_mask=x['span'].to(dev()), drop_text_cond=False):
            out = model(x['mel'].to(dev()), text=x['text'], lens=x['lens'].to(dev()))
        n_fwd = len(rec.log)
        out.loss.backward()
        torch.cuda.synchronize()
    fwd = rec.calls(last=n_fwd) if n_fwd else {}
    again = dict(rec.log[n_fwd:])
    assert n_fwd > 0 and len(rec.log) == 2 * n_fwd and set(again) == set(fwd)
    for name in fwd:
        assert again[name] == fwd[name], (name, fwd[name], again[name])
        assert again[name].device_word and again[name].p == 0.1
    assert torch.equal(model.transformer._seed_dev, word)   # nothing but the graphed steps' seed advance moves the word
    model.transformer._seed_dev = None


def _layer_bytes(model, B, N):
    tr = model.transformer
    return B * (N + tr.num_registers) * tr.num_streams * 2   # bytes per stream width unit of one bf16 [B * N', S, width] tensor


def _held(pkg, depth, ckpt, B=4, N=1024):
    """memory_allocated after a cfg2-width training forward minus before it"""
    c = dict(tkw=dict(dim=512, depth=depth, heads=8), lens=[N] * B, N=N)
    model, _ = build(pkg, c, seed=5)
    model.transformer.checkpoint_activations = ckpt
    x = inputs(c)
    step(pkg, model, c, x, ckpt)            # packs, rotary tables, zero-pool slab sized
    for p in model.parameters():
        p.grad = None
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    with pkg.inject_randomness(x0=x['x0'].to(dev()), times=x['times'].to(dev()), span_mask=x['span'].to(dev()), drop_text_cond=False):
        out = model(x['mel'].to(dev()), text=x['text'], lens=x['lens'].to(dev()))
    torch.cuda.synchronize()
    held = torch.cuda.memory_allocated() - m0
    del out
    unit = _layer_bytes(model, B, N)
    del model
    torch.cuda.empty_cache()
    return held, unit


def test_memory_held_for_the_backward(pkg):
    """Per layer, the checkpointed forward holds its boundary tensors and nothing else. The stream tensors of layer i that stay alive
    until the backward: the text block's output and the cross-conditioning's two outputs (held by the cross-conditioning's backward
    and the next segments), the audio segment's input and output; in the second half also the skip projection's output. The
    issue-level boundary B N' S (d + dt) 2 is printed next to it."""
    d, dt = 512, 256
    rows = {}
    for ckpt in (False, True):
        (h4, unit), (h8, _) = _held(pkg, 4, ckpt), _held(pkg, 8, ckpt)
        rows[ckpt] = (h8 - h4) / 4
    boundary = unit * (d + dt)
    held_shapes = unit * (2 * (d + dt) + (d + 2 * (d + dt))) / 2     # first-half and second-half layers alternate in the added four
    print(f'held per layer: plain {rows[False] / 2**20:.1f} MiB, checkpointed {rows[True] / 2**20:.1f} MiB; one boundary (d + dt) '
          f'{boundary / 2**20:.1f} MiB ({rows[True] / boundary:.2f}x), the boundary tensors kept {held_shapes / 2**20:.1f} MiB '
          f'({rows[True] / held_shapes:.2f}x); plain / checkpointed {rows[False] / rows[True]:.1f}x')
    assert rows[True] <= 1.25 * held_shapes
    assert rows[False] > 3 * rows[True]


def test_peak_memory_of_a_cfg2_step(pkg):
    B, N = 16, 1024
    c = dict(tkw=dict(dim=512, depth=8, heads=8), lens=[N] * B, N=N)
    model, _ = build(pkg, c, seed=6)
    x = inputs(c)
    peaks = {}
    for ckpt in (False, True, False, True):
        step(pkg, model, c, x, ckpt)
        for p in model.parameters():
            p.grad = None
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        step(pkg, model, c, x, ckpt)
        peaks[ckpt] = torch.cuda.max_memory_allocated() - base
    print(f'cfg2 B{B} x {N} step peak above the resident state: plain {peaks[False] / 2**30:.2f} GiB, checkpointed '
          f'{peaks[True] / 2**30:.2f} GiB')
    assert peaks[True] < peaks[False]


@pytest.mark.parametrize('case', ['default', 'residual1', 'duration', 'headdim128'])
def test_launches_one_more_forward_of_the_segments(pkg, case, schedule, monkeypatch):
    c = CASES[case]
    model, _ = build(pkg, c)
    x = inputs(c)
    step(pkg, model, c, x, False)   # first-use work (rotary tables, the pack's table upload) out of the count
    plain = step(pkg, model, c, x, False)
    seg = [0, 0]
    fwd = pkg.ops.Segment.forward

    def counted(ctx, run, *inputs):
        n0 = pkg.lib.launch_count()
        out = fwd(ctx, run, *inputs)
        seg[0] += pkg.lib.launch_count() - n0
        seg[1] += 1
        return out
    monkeypatch.setattr(pkg.ops.Segment, 'forward', staticmethod(counted))
    got = step(pkg, model, c, x, True)
    tr = model.transformer
    assert seg[1] == tr.depth + tr.text_depth, seg   # one segment per audio layer and one per text block
    assert got['launches'][0] == plain['launches'][0]                    # the forward launches what the plain forward launches
    assert got['launches'][1] == plain['launches'][1] + seg[0], (got['launches'], plain['launches'], seg)
    print(f'{case}/{schedule}: plain step {plain["launches"][1]} launches, checkpointed {got["launches"][1]} '
          f'(+{seg[0]} in {seg[1]} segments)')


def test_graphed_step_matches_eager(pkg, schedule):
    c = CASES['default']
    model, _ = build(pkg, c)
    model.transformer.checkpoint_activations = True
    mel, text, rnd = step_inputs(pkg)
    graphed_matches_eager(pkg, model, mel, text, rnd)


def _grads(model):
    return {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}


def _close(tag, got_loss, got, want_loss, want, rel=2e-3):
    assert abs(got_loss - want_loss) <= 1e-3 * abs(want_loss) + 1e-5, (tag, got_loss, want_loss)
    assert set(got) == set(want), (tag, sorted(set(got) ^ set(want))[:5])
    for n in want:
        e = rel_l2(got[n].float().cpu(), want[n].float().cpu())
        assert e < rel or float(want[n].norm()) == 0, (tag, n, e)


def test_bucketed_steps_match_eager(pkg):
    """one micro-step per bucket against the eager checkpointed step at the bucket's shape, then k = 2 accumulation against eager
    (loss / 2).backward() (model_checks.graphed_matches_eager's bounds; the accumulation at the looser whole-gradient bound of the
    bucketed-step tests, since eager runs its bf16 backward on a loss scaled by 1 / k)"""
    c = CASES['default']
    model, _ = build(pkg, c)
    model.transformer.checkpoint_activations = True
    model.cond_drop_prob = 0.0
    B, sizes, buckets = 2, (80, 150), (96, 160)
    g = torch.Generator().manual_seed(9)
    mels = [torch.randn(B, n, 100, generator=g).to(dev()) for n in sizes]
    lens = [torch.tensor([n, n - 11], device=dev()) for n in sizes]
    text = pkg.list_str_to_tensor(['Hello there', 'Goodbye']).to(dev())
    want = []
    for i, nb in enumerate(buckets):
        torch.cuda.manual_seed(100 + i)
        out = model(F.pad(mels[i], (0, 0, 0, nb - sizes[i])), text=text, lens=lens[i])
        out.loss.backward()
        want.append((float(out.loss), _grads(model)))
        del out
        for p in model.parameters():
            p.grad = None
    for i in range(2):
        torch.cuda.manual_seed(100 + i)
        out = model(F.pad(mels[i], (0, 0, 0, buckets[i] - sizes[i])), text=text, lens=lens[i])
        (out.loss / 2).backward()
        del out
    want_acc = _grads(model)
    for p in model.parameters():
        p.grad = None

    step = pkg.BucketedTrainStep(model, B, buckets, grad_accumulation_steps=1)
    for i in range(2):
        torch.cuda.manual_seed(100 + i)
        loss = float(step(mels[i], text=text, lens=lens[i]))
        torch.cuda.synchronize()
        got = {n: v.detach().clone() for (n, _), v, u in zip(model.named_parameters(), step.grad_sync.grad_views,
                                                              step.grad_sync.used.tolist()) if u > 0}
        _close(f'bucket {buckets[i]}', loss, got, *want[i])
    del step
    step = pkg.BucketedTrainStep(model, B, buckets, grad_accumulation_steps=2)
    for i in range(2):
        torch.cuda.manual_seed(100 + i)
        step(mels[i], text=text, lens=lens[i])
    torch.cuda.synchronize()
    assert step.sync_gradients
    got = {n: v.detach().clone() for (n, _), v, u in zip(model.named_parameters(), step.grad_sync.grad_views,
                                                          step.grad_sync.used.tolist()) if u > 0}
    assert set(got) == set(want_acc)
    names = sorted(want_acc)
    e = rel_l2(torch.cat([got[n].double().flatten().cpu() for n in names]), torch.cat([want_acc[n].double().flatten().cpu() for n in names]))
    print(f'k = 2 accumulation: whole-gradient rel-L2 {e:.3g}')
    assert e < 1e-2


@pytest.mark.parametrize('case', ['default', 'residual1'])
def test_eval_and_sample_ignore_the_switch(pkg, case):
    c = CASES[case]
    model, _ = build(pkg, c)
    x = inputs(c)
    model.eval()
    runs = []
    for ckpt in (False, False, True):   # the first run takes the first-use work (rotary tables, the pack's table upload)
        model.transformer.checkpoint_activations = ckpt
        n0 = pkg.lib.launch_count()
        with pkg.inject_randomness(x0=x['x0'].to(dev()), times=x['times'].to(dev()), span_mask=x['span'].to(dev()), drop_text_cond=False):
            out = model(x['mel'].to(dev()), text=x['text'], lens=x['lens'].to(dev()))   # eval forward, grad mode on
        n1 = pkg.lib.launch_count()
        torch.manual_seed(3)
        y0 = torch.randn(2, 64, 100, device=dev())
        with pkg.inject_randomness(y0=y0):
            s = model.sample(x['mel'][:, :24].to(dev()), text=x['text'], duration=64, steps=4, return_raw_output=True)
        torch.cuda.synchronize()
        runs.append((out.pred_flow.detach().clone(), out.loss.detach().clone(), s.clone(), n1 - n0, pkg.lib.launch_count() - n1))
    (p0, l0, s0, nf0, ns0), (p1, l1, s1, nf1, ns1) = runs[1:]
    assert same_bits(p0, p1) and same_bits(s0, s1)
    assert abs(float(l0) - float(l1)) <= 1e-6 * abs(float(l0))   # the loss's atomic reduction (see test_step_matches_plain_step)
    assert (nf0, ns0) == (nf1, ns1)
