"""Whole-model checks shared by the test modules: the GPU model against the fp32 oracle (oracle/e2tts_oracle.py) computed on the host,
the small seeded models of the sampling / duration / graphed-step tests, and the oracle's gradients against the original's stored
samples (tests/golden/reference/)."""
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
