"""Run the ORIGINAL e2-tts-pytorch code (its own e2_tts.py, loaded unmodified by oracle/load_reference.py) on the cases of
oracle/reference_cases.py and store what it computed under tests/golden/reference/ (one file per test, each well under 1 MB).
TEST INFRASTRUCTURE: needs a checkout of the original project (E2TTS_REFERENCE_FILE points at its e2_tts.py).

    E2TTS_REFERENCE_FILE=<original>/e2_tts_pytorch/e2_tts.py python oracle/make_reference_golden.py
"""
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import reference_cases as RC  # noqa: E402
from oracle.load_reference import TorchRecorder, load_reference, run_reference_forward  # noqa: E402


def save(name, obj):
    os.makedirs(RC.GOLDEN, exist_ok=True)
    path = os.path.join(RC.GOLDEN, name + '.pt')
    torch.save(obj, path)
    print(f'{name}.pt {os.path.getsize(path) // 1024} KiB')


def grads_of(model):
    return {k: (p.grad.clone() if p.grad is not None else None) for k, p in model.named_parameters()}


def main():
    ref = load_reference()
    for name, c in RC.FORWARD_CASES.items():
        model = ref.E2TTS(transformer=dict(dropout=0., max_seq_len=128, **c['tkw']), use_vocos=False, **c['kw'])
        model.load_state_dict(RC.state_dict('E2TTS', c['seed'], c['tkw'], **c['kw']))
        mel = RC.randn((c['mel'][0], c['mel'][1], 100), c['seed'] + 1000)
        lens = torch.tensor(c['lens']) if c['lens'] else None
        torch.manual_seed(c['seed'])
        ref.torch = RC.noise(torch, c['seed'] + 2000)   # x0 = the first draw of that generator
        try:
            out, rec = run_reference_forward(ref, model, mel, c['text'], lens=lens, drop_text_cond=c['drop'])
        finally:
            ref.torch = torch
        out.loss.backward()
        save('forward_' + name, dict(loss=float(out.loss.detach()), pred=RC.compact(out.pred_flow), grads=RC.grad_record(grads_of(model)),
                                     times=rec['times'], span_mask=rec['span_mask']))

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


if __name__ == '__main__':
    main()
