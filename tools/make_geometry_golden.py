"""Run the ORIGINAL e2-tts-pytorch code (its own e2_tts.py, loaded unmodified by oracle/load_reference.py) with the model-shape knobs
of tests/geometry_variants.py (depth 12, text_depth < depth, dim_text != dim // 2, ff_mult / text_ff_mult != 4, num_registers 0 / 8 /
16, abs_pos_emb=False, kernel_size 1 / 5 / 7) and store what it computed as tests/golden/reference/geometry_<case>.pt, in the record
format of tools/make_residual_golden.py (outputs only: weights, inputs and injected noise are rebuilt from seeds). Writes only those
files. Needs a checkout of the original project:

    E2TTS_REFERENCE_FILE=<original>/e2_tts_pytorch/e2_tts.py python tools/make_geometry_golden.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from geometry_variants import GEOMETRY_CASES, GEOMETRY_SAMPLE  # noqa: E402
from oracle import reference_cases as RC  # noqa: E402
from oracle.load_reference import load_reference, run_reference_forward  # noqa: E402


def save(name, obj):
    path = os.path.join(RC.GOLDEN, f'geometry_{name}.pt')
    torch.save(obj, path)
    print(f'{os.path.basename(path)} {os.path.getsize(path) // 1024} KiB')


def main():
    ref = load_reference()
    os.makedirs(RC.GOLDEN, exist_ok=True)
    for name, c in GEOMETRY_CASES.items():
        tkw = c['tkw']
        mel = RC.randn((c['mel'][0], c['mel'][1], 100), c['seed'] + 1000)
        lens = torch.tensor(c['lens'])
        if c['cls'] == 'E2TTS':
            model = ref.E2TTS(transformer=dict(dropout=0., max_seq_len=128, **tkw), use_vocos=False)
            model.load_state_dict(RC.state_dict('E2TTS', c['seed'], tkw))
            torch.manual_seed(c['seed'])
            ref.torch = RC.noise(torch, c['seed'] + 2000)   # x0 = the first draw of that generator
            try:
                out, rec = run_reference_forward(ref, model, mel, c['text'], lens=lens, drop_text_cond=c['drop'])
            finally:
                ref.torch = torch
            out.loss.backward()
            obj = dict(loss=float(out.loss.detach()), pred=RC.compact(out.pred_flow), times=rec['times'], span_mask=rec['span_mask'])
        else:
            model = ref.DurationPredictor(transformer=dict(dropout=0., max_seq_len=128, **tkw))
            model.load_state_dict(RC.state_dict('DurationPredictor', c['seed'], tkw))
            torch.manual_seed(c['seed'])
            loss = model(mel, text=c['text'], lens=lens)
            loss.backward()
            obj = dict(loss=float(loss.detach()))
        obj['grads'] = RC.grad_record({k: (p.grad.clone() if p.grad is not None else None) for k, p in model.named_parameters()})
        obj['shapes'] = {k: tuple(v.shape) for k, v in model.state_dict().items()}
        save(name, obj)

    s = GEOMETRY_SAMPLE
    model = ref.E2TTS(transformer=dict(dropout=0., max_seq_len=128, **s['tkw']), use_vocos=False)
    model.load_state_dict(RC.state_dict('E2TTS', s['seed'], s['tkw']))
    model.eval()
    cond = RC.randn((s['cond'][0], s['cond'][1], 100), s['seed'] + 1000)
    ref.torch = RC.noise(torch, 3000 + s['seed'])   # y0 = the first draw of that generator
    try:
        with torch.no_grad():
            want = model.sample(cond, text=s['text'], lens=torch.tensor(s['lens']), duration=torch.tensor(s['duration']), steps=s['steps'],
                                cfg_strength=s['cfg_strength'], return_raw_output=True)
    finally:
        ref.torch = torch
    save('sample', dict(shape=tuple(want.shape), out=RC.compact(want)))


if __name__ == '__main__':
    main()
