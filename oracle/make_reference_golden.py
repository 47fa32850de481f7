"""Run the ORIGINAL e2-tts-pytorch code (its own e2_tts.py, loaded unmodified by oracle/load_reference.py) on the reference-pinned
cases and store what it computed under tests/golden/reference/ (one file per test, each well under 1 MB). TEST INFRASTRUCTURE: needs
a checkout of the original project (E2TTS_REFERENCE_FILE points at its e2_tts.py).

    E2TTS_REFERENCE_FILE=<original>/e2_tts_pytorch/e2_tts.py python oracle/make_reference_golden.py [family ...]

A family is one case table (FAMILIES); each writes only its own files, and with no family named every one runs. Only outputs are
stored: weights, inputs and injected noise are rebuilt from seeds (oracle/reference_cases.py). While the original runs, its
`FeedForward` name is bound to tests/ff_variants.py's XTFeedForward, the restatement of x-transformers' FeedForward / GLU for the
`ff_kwargs` the restated leaf does not take (without keywords it has the leaf's parameters and draws). The dropout family builds its
models with dropout P_REF and replaces every nn.Dropout by the hashed mask of tests/dropout_ref.py (its qualified name, the input
shape and the case seed), so the tests can give the oracle the same masks without the original code; its records list the modules
that dropped.
"""
import argparse
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from attn_variants import ATTN_KWARGS_CASES  # noqa: E402
from dropout_ref import DROPOUT_CASES, P_REF, HashedDropout  # noqa: E402
from ff_variants import FF_KWARGS_CASES, XTFeedForward  # noqa: E402
from geometry_variants import GEOMETRY_CASES, GEOMETRY_SAMPLE  # noqa: E402
from headdim_variants import HEADDIM_CASES, HEADDIM_SAMPLE  # noqa: E402
from oracle import reference_cases as RC  # noqa: E402
from oracle.load_reference import TorchRecorder, load_reference, run_reference_forward  # noqa: E402
from residual_variants import RESIDUAL1_CASES, RESIDUAL1_SAMPLE  # noqa: E402


def save(name, obj):
    os.makedirs(RC.GOLDEN, exist_ok=True)
    path = os.path.join(RC.GOLDEN, name + '.pt')
    torch.save(obj, path)
    print(f'{name}.pt {os.path.getsize(path) // 1024} KiB')


def grads_of(model):
    return {k: (p.grad.clone() if p.grad is not None else None) for k, p in model.named_parameters()}


def hash_dropouts(model, seed, p, log):
    """every nn.Dropout of `model` -> HashedDropout of its qualified name; returns how many were replaced"""
    found = [(n, m) for n, m in model.named_modules() if isinstance(m, torch.nn.Dropout)]
    for name, m in found:
        assert m.p == p, (name, m.p)
        parent, _, leaf = name.rpartition('.')
        model.get_submodule(parent)._modules[leaf] = HashedDropout(name, seed, p, log)
    return len(found)


def record_forward(ref, c, keys, dropout=0.):
    """The original's forward + backward on case `c` (cls, seed, tkw and, where they are not the defaults, kw, lens, drop): the record
    fields `keys` that the model class computes. With `dropout` every nn.Dropout draws the hashed masks of the case's seed."""
    cls, kw = c.get('cls', 'E2TTS'), c.get('kw', {})
    transformer = dict(dropout=dropout, max_seq_len=128, **c['tkw'])
    if cls == 'E2TTS':
        model = ref.E2TTS(transformer=transformer, use_vocos=False, **kw)
    else:
        model = ref.DurationPredictor(transformer=transformer)
    model.load_state_dict(RC.state_dict(cls, c['seed'], c['tkw'], **kw))
    dropped = []
    if dropout:
        assert hash_dropouts(model, c['seed'], dropout, dropped) > 0
    mel = RC.randn((c['mel'][0], c['mel'][1], 100), c['seed'] + 1000)
    lens = torch.tensor(c['lens']) if c['lens'] else None
    torch.manual_seed(c['seed'])
    if cls == 'E2TTS':
        ref.torch = RC.noise(torch, c['seed'] + 2000)   # x0 = the first draw of that generator
        try:
            out, rec = run_reference_forward(ref, model, mel, c['text'], lens=lens, drop_text_cond=c.get('drop', False))
        finally:
            ref.torch = torch
        loss = out.loss
        r = dict(pred=RC.compact(out.pred_flow), times=rec['times'], span_mask=rec['span_mask'])
    else:
        loss = model(mel, text=c['text'], lens=lens)
        r = {}
    loss.backward()
    r.update(loss=float(loss.detach()), grads=RC.grad_record(grads_of(model)), dropped=dropped,
             shapes={k: tuple(v.shape) for k, v in model.state_dict().items()})
    return {k: r[k] for k in keys if k in r}


def record_sample(ref, s):
    """The original's E2TTS.sample on case `s` (seed, tkw, cond (batch, frames), text, duration, steps, cfg_strength and, for a ragged
    prompt, lens); y0 = the first draw of generator 3000 + seed"""
    model = ref.E2TTS(transformer=dict(dropout=0., max_seq_len=128, **s['tkw']), use_vocos=False)
    model.load_state_dict(RC.state_dict('E2TTS', s['seed'], s['tkw']))
    model.eval()
    cond = RC.randn((s['cond'][0], s['cond'][1], 100), s['seed'] + 1000)
    lens = torch.tensor(s['lens']) if 'lens' in s else None
    ref.torch = RC.noise(torch, 3000 + s['seed'])
    try:
        with torch.no_grad():
            want = model.sample(cond, text=s['text'], lens=lens, duration=torch.tensor(s['duration']), steps=s['steps'],
                                cfg_strength=s['cfg_strength'], return_raw_output=True)
    finally:
        ref.torch = torch
    return dict(shape=tuple(want.shape), out=RC.compact(want))


def record_base(ref):
    """the records of oracle/reference_cases.py besides its forward cases"""
    torch.manual_seed(9)
    wave = torch.randn(1, 256 * 10 + 17)
    save('melspec', dict(wave=wave, mel=ref.MelSpec()(wave)))

    kw = dict(transformer=dict(dim=128, depth=2, heads=2, attn_fourier_embed_input=True), use_vocos=False, interpolated_text=True, concat_cond=True)
    save('variant_state_dict', dict(kw=kw, shapes={k: tuple(v.shape) for k, v in ref.E2TTS(**kw).state_dict().items()}))

    model = ref.E2TTS(transformer=dict(dropout=0., max_seq_len=128, **RC.KW), use_vocos=False)
    model.load_state_dict(RC.state_dict('E2TTS', 31))
    model.eval()
    cond = RC.randn((2, 20, 100), 1031)
    text = ['Hello', 'Goodbye then']
    samples = []
    for steps, cfg_strength, duration in RC.SAMPLE_CASES:
        dur = torch.tensor(duration) if isinstance(duration, list) else duration
        ref.torch = RC.noise(torch, 3000 + steps)   # y0 = the first draw of that generator
        try:
            with torch.no_grad():
                want = model.sample(cond, text=text, duration=dur, steps=steps, cfg_strength=cfg_strength, return_raw_output=True)
        finally:
            ref.torch = torch
        samples.append(dict(steps=steps, cfg_strength=cfg_strength, duration=duration, shape=tuple(want.shape), out=RC.compact(want)))
    save('sample', dict(cond=cond, text=text, cases=samples))

    dp = ref.DurationPredictor(transformer=dict(dropout=0., max_seq_len=128, **RC.KW))
    dp.load_state_dict(RC.state_dict('DurationPredictor', 41))
    mel = RC.randn((3, 72, 100), 1041)
    lens = torch.tensor([72, 50, 31])
    torch.manual_seed(5)
    loss = dp(mel, text=['abc', 'hello world', 'x'], lens=lens)
    loss.backward()
    save('duration', dict(loss=float(loss.detach()), grads=RC.grad_record(grads_of(dp))))

    g = torch.Generator().manual_seed(0)
    masks = []
    for case in range(200):
        b = int(torch.randint(1, 9, (1,), generator=g))
        n = int(torch.randint(8, 300, (1,), generator=g))
        lens = torch.randint(1, n + 1, (b,), generator=g)
        if case % 3 == 0:
            lens[int(torch.randint(0, b, (1,), generator=g))] = n
        frac = torch.rand(b, generator=g) * 0.3 + 0.7
        torch.manual_seed(1000 + case)
        want = ref.mask_from_frac_lengths(lens, frac, max_length=n)
        masks.append(dict(span=torch.from_numpy(np.packbits(want.numpy(), axis=-1)), shape=tuple(want.shape),
                          lens_n=torch.from_numpy(np.packbits(ref.lens_to_mask(lens, length=n).numpy(), axis=-1)),
                          lens_auto=ref.lens_to_mask(lens).shape))
    save('mask_helpers', dict(cases=masks, ids=ref.list_str_to_tensor(['Hello', 'Goodbye', 'héllo wörld'])))

    s = RC.VELOCITY_SEED
    random.seed(s)
    model = ref.E2TTS(transformer=dict(dropout=0., max_seq_len=128, **RC.KW), use_vocos=False, velocity_consistency_weight=0.7)
    model.load_state_dict(RC.state_dict('E2TTS', s, velocity_consistency_weight=0.7))
    ema = ref.E2TTS(transformer=dict(dropout=0., max_seq_len=128, **RC.KW), use_vocos=False)
    ema.load_state_dict(RC.state_dict('E2TTS', s + 1))
    ema.eval()
    mel = RC.randn((2, 64, 100), 1000 + s)
    lens = torch.tensor([64, 50])
    rec = TorchRecorder(RC.noise(torch, 2000 + s))
    span = {}
    orig = ref.mask_from_frac_lengths

    def mffl(*a, **k):
        span['mask'] = orig(*a, **k)
        return span['mask'].clone()

    model.cond_drop_prob = -1.0
    torch.manual_seed(s)
    ref.torch, ref.mask_from_frac_lengths = rec, mffl
    try:
        out = model(mel, text=['abc', 'some text'], lens=lens, velocity_consistency_model=ema, velocity_consistency_delta=1e-3)
    finally:
        ref.torch, ref.mask_from_frac_lengths = torch, orig
    out.loss.backward()
    gr = grads_of(model)
    total = float(torch.cat([v.flatten() for v in gr.values() if v is not None]).norm())
    save('velocity_consistency', dict(times=rec.log['rand'][0], span_mask=span['mask'] & ref.lens_to_mask(lens, length=64),
                                      loss=float(out.loss.detach()), flow=float(out.loss_breakdown.flow),
                                      velocity=float(out.loss_breakdown.velocity_consistency), grads=RC.grad_record(gr), total=total))


VARIANT_KEYS = ('loss', 'pred', 'times', 'span_mask', 'grads', 'shapes')
# family -> record name prefix, forward + backward cases, record fields in stored order, the sample case, the model's dropout and the
# family's other records
FAMILIES = {
    'base': dict(prefix='forward_', cases=RC.FORWARD_CASES, keys=('loss', 'pred', 'grads', 'times', 'span_mask'), more=record_base),
    'attn_kwargs': dict(prefix='attn_kwargs_', cases=ATTN_KWARGS_CASES, keys=VARIANT_KEYS),
    'ff_kwargs': dict(prefix='ff_kwargs_', cases=FF_KWARGS_CASES, keys=VARIANT_KEYS),
    'residual': dict(prefix='residual1_', cases=RESIDUAL1_CASES, keys=VARIANT_KEYS, sample=RESIDUAL1_SAMPLE),
    'headdim': dict(prefix='headdim_', cases=HEADDIM_CASES, keys=VARIANT_KEYS, sample=HEADDIM_SAMPLE),
    'geometry': dict(prefix='geometry_', cases=GEOMETRY_CASES, keys=VARIANT_KEYS, sample=GEOMETRY_SAMPLE),
    'dropout': dict(prefix='dropout_', cases=DROPOUT_CASES, keys=('loss', 'pred', 'times', 'span_mask', 'grads', 'dropped'),
                    dropout=P_REF),
}


def main():
    parser = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    parser.add_argument('families', nargs='*', choices=list(FAMILIES), help='default: every family')
    families = parser.parse_args().families or FAMILIES
    ref = load_reference()
    ref.FeedForward = XTFeedForward   # e2_tts.py:646, :692 build FeedForward(dim=..., glu=True, mult=..., dropout=..., **ff_kwargs)
    for family in families:
        f = FAMILIES[family]
        for name, c in f['cases'].items():
            save(f['prefix'] + name, record_forward(ref, c, f['keys'], f.get('dropout', 0.)))
        if 'sample' in f:
            save(f['prefix'] + 'sample', record_sample(ref, f['sample']))
        if 'more' in f:
            f['more'](ref)


if __name__ == '__main__':
    main()
