"""Whole-model checks shared by the test modules: the GPU model against the fp32 oracle (oracle/e2tts_oracle.py) computed on the host,
the small seeded models of the sampling / duration / graphed-step tests and those checks, and the oracle against the original's stored
outputs, gradient samples and parameter shapes (tests/golden/reference/)."""
import random

import torch

from conftest import rel_l2
from dropout_ref import with_dropout
from kernel_checks import dev
from oracle import e2tts_oracle as O
from oracle import reference_cases as RC


def cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def check(name, got, want, tol):
    e = rel_l2(got.float().cpu(), want.float().cpu())
    assert e < tol, f'{name}: rel-L2 {e:.4g} >= {tol}'


def whole_model(pkg, tkw, B, N, lens, seed, tol_pred=3e-2, e2tts_kw=None, drop_text_cond=False, dyn_scale=0.05, grads=True):
    torch.manual_seed(seed)
    random.seed(seed)   # the hyper-connections draw their initial stream with python's randrange: the same case on every run
    model = pkg.E2TTS(transformer=dict(dropout=0., max_seq_len=N, **tkw), use_vocos=False, **(e2tts_kw or {}))
    # dyn_scale 0.05 (5x the reference's init of the hyper-connections' dynamic scales): with the 0.5 of the 2-layer fixtures a depth-8
    # stack amplifies bf16 rounding of the residual streams ~10x — the fp32 oracle with its OWN stage outputs rounded to bf16
    # (O.STAGE_ROUND) then moves its prediction by 12.6 %, exactly what the kernels showed. The probe below
    # keeps this test honest: the case must be well conditioned for a bf16 path before the kernels are held to 3e-2.
    sd = O.randomize_zero_init({k: v.clone() for k, v in model.state_dict().items()}, seed=seed + 1, dyn_scale=dyn_scale)
    model.load_state_dict(sd)
    model.to(dev()).train()
    mel = torch.randn(B, N, 100)
    text = ['Hello', 'Goodbye', 'Good day'][:B]
    x0, times = torch.randn(B, N, 100), torch.rand(B)
    lens_t = torch.tensor(lens)
    span = torch.zeros(B, N, dtype=torch.bool)
    for b in range(B):
        span[b, lens[b] // 8: lens[b] - lens[b] // 10] = True
    with pkg.inject_randomness(x0=x0.to(dev()), times=times.to(dev()), span_mask=span.to(dev()), drop_text_cond=drop_text_cond):
        out = model(mel.to(dev()), text=text, lens=lens_t.to(dev()))
    out.loss.backward()
    torch.cuda.synchronize()
    # oracle on the host (fp32, all cores)
    osd = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    kw = dict(x0=x0, times=times, span_mask=span, lens=lens_t, drop_text_cond=drop_text_cond)
    ref = O.e2tts_forward(osd, O.TransformerCfg(**tkw), mel, O.list_str_to_tensor(text), **kw)
    ref['loss'].backward()
    O.STAGE_ROUND = O.bf16_ste
    try:
        with torch.no_grad():
            probe = O.e2tts_forward(sd, O.TransformerCfg(**tkw), mel, O.list_str_to_tensor(text), **kw)
    finally:
        O.STAGE_ROUND = None
    e_probe = rel_l2(probe['pred'], ref['pred'].detach())
    assert e_probe < 1.5e-2, f'test case is ill-conditioned for bf16 activations (oracle vs bf16-stage oracle: {e_probe:.3g})'
    loss, rloss = float(out.loss), float(ref['loss'])
    assert abs(loss - rloss) <= 1e-2 * abs(rloss), (loss, rloss)
    check('pred', out.pred_flow, ref['pred'].detach(), tol_pred)
    print(f'pred rel-L2 {rel_l2(out.pred_flow.float().cpu(), ref["pred"].detach()):.4g} (bf16-stage oracle probe {e_probe:.4g})')
    if not grads:   # a case whose gradients are ill-conditioned for any bf16 path: loss and prediction only
        return dict(probe=e_probe, worst_cos=None)
    total = float(torch.cat([v.grad.flatten() for v in osd.values() if v.grad is not None]).norm())
    worst = (1.0, None)
    for k, p in model.named_parameters():
        gr = osd[k].grad
        if gr is None:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, f'{k} should be unused'
            continue
        assert p.grad is not None, k
        if float(gr.norm()) < 1e-4 * total:     # negligible next to the whole gradient: direction is rounding noise in any bf16 path
            continue
        cs_ = cos(p.grad.cpu(), gr)
        worst = min(worst, (cs_, k))
        assert cs_ >= 0.99, (k, cs_)
    print(f'whole model {tkw}: loss {loss:.5f} (oracle {rloss:.5f}), worst grad cosine {worst}')
    return dict(probe=e_probe, worst_cos=worst)


def small_model(pkg, seed, cls='E2TTS', **transformer_kw):
    """an E2TTS (or DurationPredictor) with these Transformer kwargs on the GPU, every zero-initialised tensor randomised:
    (model, its state dict)"""
    torch.manual_seed(seed)
    random.seed(seed)
    t = dict(dropout=0., max_seq_len=256, **transformer_kw)
    model = pkg.E2TTS(transformer=t, use_vocos=False) if cls == 'E2TTS' else pkg.DurationPredictor(transformer=t)
    sd = O.randomize_zero_init({k: v.clone() for k, v in model.state_dict().items()}, seed=seed + 1)
    model.load_state_dict(sd)
    return model.to(dev()), sd


def sample_vs_oracle(pkg, seed, tkw, cond=(2, 24), text=('Hello', 'Goodbye'), duration=64, lens=None, steps=32, cfg_strength=1.0):
    """E2TTS.sample of small_model(pkg, seed, **tkw) against the oracle's fixed-grid ODE on the same weights: cond (batch, frames) and
    then y0 drawn under seed + 1, y0 as long as the longest duration (an int, or a tensor of one per batch element, as `lens`). Same
    shape, rel-L2 < 5e-2. Returns the GPU sample."""
    model, sd = small_model(pkg, seed, **tkw)
    torch.manual_seed(seed + 1)
    cond = torch.randn(*cond, 100)
    y0 = torch.randn(cond.shape[0], int(torch.as_tensor(duration).max()), 100)
    on_dev = lambda t: t.to(dev()) if torch.is_tensor(t) else t   # noqa: E731
    with pkg.inject_randomness(y0=y0.to(dev())):
        out = model.sample(cond.to(dev()), text=list(text), lens=on_dev(lens), duration=on_dev(duration), steps=steps,
                           cfg_strength=cfg_strength, return_raw_output=True)
    want = O.e2tts_sample(sd, O.TransformerCfg(**tkw), cond, O.list_str_to_tensor(list(text)), duration=duration, lens=lens, y0=y0,
                          steps=steps, cfg_strength=cfg_strength)
    assert out.shape == want.shape
    e = rel_l2(out.cpu(), want)
    print(f'{steps}-step sample {tkw}: rel-L2 {e:.4g}')
    assert e < 5e-2
    return out


def duration_vs_oracle(pkg, seed, tkw):
    """DurationPredictor small_model(pkg, seed, **tkw) in training mode on three ragged items drawn after it, with the prefix fractions
    pinned, against the oracle: loss within 1e-2; a parameter the oracle leaves without a gradient gets none (or an all-zero one); every
    other gradient present, with cosine >= 0.99 wherever it is not negligible next to the whole gradient"""
    model, sd = small_model(pkg, seed, 'DurationPredictor', **tkw)
    model.train()
    mel = torch.randn(3, 72, 100)
    lens = torch.tensor([72, 50, 31])
    text = ['abc', 'hello world', 'x']
    rand_frac = torch.tensor([0.3, 0.6, 0.9])
    with pkg.inject_randomness(duration_rand_frac=rand_frac.to(dev())):
        loss = model(mel.to(dev()), text=text, lens=lens.to(dev()))
    loss.backward()
    osd = grad_sd(sd)
    ref = O.duration_forward(osd, O.TransformerCfg(cond_on_time=False, **tkw), mel, O.list_str_to_tensor(text), lens=lens,
                             rand_frac=rand_frac)
    ref.backward()
    print(f'duration predictor {tkw}: loss {float(loss):.6f} (oracle {float(ref):.6f})')
    assert abs(float(loss) - float(ref)) <= 1e-2 * abs(float(ref))
    total = float(torch.cat([v.grad.flatten() for v in osd.values() if v.grad is not None]).norm())
    for k, p in model.named_parameters():
        gr = osd[k].grad
        if gr is None:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, f'{k} should be unused'
            continue
        assert p.grad is not None, k
        if float(gr.norm()) < 1e-4 * total:
            continue
        assert cos(p.grad.cpu(), gr) >= 0.99, k


def step_inputs(pkg, B=2, N=96, span=(20, 70)):
    """(mel, text ids, inject_randomness kwargs) of one training step on the GPU: mel, x0 and times drawn in that order from torch's
    global generator, frames span[0]:span[1] of every item masked, the text kept"""
    mel = torch.randn(B, N, 100, device=dev())
    text = pkg.list_str_to_tensor(['Hello', 'Goodbye']).to(dev())
    x0, times = torch.randn(B, N, 100, device=dev()), torch.rand(B, device=dev())
    span_mask = torch.zeros(B, N, dtype=torch.bool, device=dev())
    span_mask[:, span[0]:span[1]] = True
    return mel, text, dict(x0=x0, times=times, span_mask=span_mask, drop_text_cond=False)


def graphed_matches_eager(pkg, model, mel, text, rnd):
    """One eager step of `model` (training mode, text never dropped) with the randomness `rnd` pinned, then a GraphedTrainStep on the
    same inputs: loss within 1e-3 |loss| + 1e-5, the same parameters with a gradient, each within rel-L2 2e-3 of the eager one (fp32
    atomics reorder between runs). Returns (the step, its loss)."""
    model.train()
    model.cond_drop_prob = 0.0
    with pkg.inject_randomness(**rnd):
        out = model(mel, text=text)
        out.loss.backward()
        want_loss = float(out.loss)
        want = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
        for p in model.parameters():
            p.grad = None
        del out   # an alive eager graph keeps its AccumulateGrad nodes (bound to the default stream) and would drag stream 0 into the capture
        step = pkg.GraphedTrainStep(model, mel, text=text)
        got_loss = float(step())
    torch.cuda.synchronize()
    assert abs(got_loss - want_loss) <= 1e-3 * abs(want_loss) + 1e-5, (got_loss, want_loss)
    got = {n: p.grad for n, p in model.named_parameters() if p.grad is not None}
    assert set(got) == set(want)
    for n in want:
        assert rel_l2(got[n].float().cpu(), want[n].float().cpu()) < 2e-3 or float(want[n].norm()) == 0, n
    return step, got_loss


def grad_sd(sd):
    return {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}


def check_grads(sd, rec, rel=2e-4, floor=1e-7):
    """Elementwise on the stored sample: |got - want| <= rel * max|want| + floor (the tolerance of a full comparison), plus max|g| and
    the norm. A parameter the original left without a gradient must get none (or an all-zero one) from the oracle."""
    for k, r in rec.items():
        got = sd[k].grad
        if r is None:
            assert got is None or float(got.abs().max()) == 0.0, k
            continue
        assert got is not None, k
        g = got.detach().double().flatten()
        if r['values'].numel() == 0:    # an empty parameter (Transformer(num_registers=0).registers)
            assert g.numel() == 0, k
            continue
        tol = rel * r['max'] + floor
        assert float((g[RC.sample_index(g.numel())] - r['values'].double()).abs().max()) <= tol, k
        assert abs(float(g.abs().max()) - r['max']) <= tol, k
        assert abs(float(g.norm()) - r['norm']) <= 5 * rel * r['norm'] + floor, k


def oracle_case(c, rec, sd=None, hook=None):
    """The oracle on a stored case of the original: `c` holds cls, seed, tkw (the Transformer kwargs) and, where they are not the
    defaults, kw (the E2TTS kwargs), lens and drop (drop_text_cond); `rec` is its record (tests/golden/reference/). Weights `sd` (default:
    the case's seeded weights, taking gradients), inputs rebuilt from the seed, the original's draws injected, O.DROPOUT = hook; the
    loss is backpropagated when it takes a gradient. Returns (sd, loss, prediction or None for a DurationPredictor)."""
    cls = c.get('cls', 'E2TTS')
    if sd is None:
        sd = grad_sd(RC.state_dict(cls, c['seed'], c['tkw'], **c.get('kw', {})))
    mel = RC.randn((c['mel'][0], c['mel'][1], 100), c['seed'] + 1000)
    lens = torch.tensor(c['lens']) if c.get('lens') else None
    text = O.list_str_to_tensor(c['text'])
    if cls == 'E2TTS':
        o = with_dropout(hook, O.e2tts_forward, sd, O.TransformerCfg(**c['tkw']), mel, text, lens=lens, drop_text_cond=c.get('drop', False),
                         x0=RC.randn(mel.shape, c['seed'] + 2000), times=rec['times'], span_mask=rec['span_mask'])
        loss, pred = o['loss'], o['pred']
    else:
        torch.manual_seed(c['seed'])
        rand_frac = mel.new_zeros(mel.shape[0]).uniform_(0, 1)   # the draw of e2_tts.py:1082 under the same seed
        loss = with_dropout(hook, O.duration_forward, sd, O.TransformerCfg(cond_on_time=False, **c['tkw']), mel, text, lens=lens,
                            rand_frac=rand_frac)
        pred = None
    if loss.requires_grad:
        loss.backward()
    return sd, loss, pred


def check_case(c, rec, sd, loss, pred):
    """oracle_case's results against the record: prediction sample rel-L2 < 1e-4 and its norm within 1e-4, loss within 1e-5, gradient
    samples within check_grads at the case's grad_tol (default: the 2-layer E2TTS fixtures' bound, a DurationPredictor's looser one)"""
    if pred is not None:
        assert RC.compact_rel_l2(pred, rec['pred']) < 1e-4
        assert abs(float(pred.detach().double().norm()) - rec['pred']['norm']) <= 1e-4 * rec['pred']['norm']
    assert abs(float(loss.detach()) - rec['loss']) <= 1e-5 * abs(rec['loss'])
    check_grads(sd, rec['grads'], *c.get('grad_tol', (2e-4, 1e-7) if c.get('cls', 'E2TTS') == 'E2TTS' else (5e-4, 1e-6)))


def state_dict_vs_reference(c, rec):
    """keys and shapes of the package's model of stored case `c` (cls, tkw) equal the original's (`rec['shapes']`), so its checkpoints
    load; returns them"""
    import e2_tts_pytorch_b200 as pkg
    t = dict(dropout=0., max_seq_len=128, **c['tkw'])
    m = pkg.E2TTS(transformer=t, use_vocos=False) if c['cls'] == 'E2TTS' else pkg.DurationPredictor(transformer=t)
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == rec['shapes']
    return got


def sample_vs_reference(s, rec, lens=None):
    """the oracle's E2TTS.sample on stored sample case `s` (seed, tkw, cond (batch, frames), text, duration, steps, cfg_strength) with the
    prompt lengths `lens`, from the y0 the original drew (generator 3000 + seed), against its record: same shape, rel-L2 < 1e-4"""
    cond = RC.randn((s['cond'][0], s['cond'][1], 100), s['seed'] + 1000)
    with torch.no_grad():
        got = O.e2tts_sample(RC.state_dict('E2TTS', s['seed'], s['tkw']), O.TransformerCfg(**s['tkw']), cond,
                             O.list_str_to_tensor(s['text']), duration=torch.tensor(s['duration']), lens=lens,
                             y0=RC.randn(rec['shape'], 3000 + s['seed']), steps=s['steps'], cfg_strength=s['cfg_strength'])
    assert tuple(got.shape) == rec['shape']
    assert RC.compact_rel_l2(got, rec['out']) < 1e-4
