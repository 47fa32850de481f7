"""Run the ORIGINAL e2-tts-pytorch code (its own e2_tts.py, loaded unmodified by oracle/load_reference.py) on the ff_kwargs cases of
tests/ff_variants.py and store what it computed as tests/golden/reference/ff_kwargs_<case>.pt, in the record format of
oracle/make_reference_golden.py. The restated x-transformers leaf's FeedForward takes no keywords, so while the original runs its
`FeedForward` name is bound to tests/ff_variants.py's XTFeedForward, the restatement of x-transformers' FeedForward / GLU for these
keywords. Writes only those files. Needs a checkout of the original project:

    E2TTS_REFERENCE_FILE=<original>/e2_tts_pytorch/e2_tts.py python tools/make_ff_kwargs_golden.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from ff_variants import FF_KWARGS_CASES, XTFeedForward  # noqa: E402
from oracle import reference_cases as RC  # noqa: E402
from oracle.load_reference import load_reference, run_reference_forward  # noqa: E402


def main():
    ref = load_reference()
    ref.FeedForward = XTFeedForward   # e2_tts.py:646, :692 build FeedForward(dim=..., glu=True, mult=..., dropout=..., **ff_kwargs)
    os.makedirs(RC.GOLDEN, exist_ok=True)
    for name, c in FF_KWARGS_CASES.items():
        tkw = dict(c['tkw'], ff_kwargs=c['ff_kwargs'])
        mel = RC.randn((c['mel'][0], c['mel'][1], 100), c['seed'] + 1000)
        lens = torch.tensor(c['lens'])
        if c['cls'] == 'E2TTS':
            model = ref.E2TTS(transformer=dict(dropout=0., max_seq_len=128, **tkw), use_vocos=False)
            model.load_state_dict(RC.state_dict(c['cls'], c['seed'], tkw))
            torch.manual_seed(c['seed'])
            ref.torch = RC.noise(torch, c['seed'] + 2000)   # x0 = the first draw of that generator
            try:
                out, rec = run_reference_forward(ref, model, mel, c['text'], lens=lens, drop_text_cond=False)
            finally:
                ref.torch = torch
            out.loss.backward()
            obj = dict(loss=float(out.loss.detach()), pred=RC.compact(out.pred_flow), times=rec['times'], span_mask=rec['span_mask'])
        else:
            model = ref.DurationPredictor(transformer=dict(dropout=0., max_seq_len=128, **tkw))
            model.load_state_dict(RC.state_dict(c['cls'], c['seed'], tkw))
            torch.manual_seed(c['seed'])
            loss = model(mel, text=c['text'], lens=lens)
            loss.backward()
            obj = dict(loss=float(loss.detach()))
        obj['grads'] = RC.grad_record({k: (p.grad.clone() if p.grad is not None else None) for k, p in model.named_parameters()})
        obj['shapes'] = {k: tuple(v.shape) for k, v in model.state_dict().items()}
        path = os.path.join(RC.GOLDEN, f'ff_kwargs_{name}.pt')
        torch.save(obj, path)
        print(f'{os.path.basename(path)} {os.path.getsize(path) // 1024} KiB')


if __name__ == '__main__':
    main()
