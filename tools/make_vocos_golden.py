"""Run the ORIGINAL e2-tts-pytorch code (its own e2_tts.py, loaded unmodified by oracle/load_reference.py) with use_vocos=True on the
cases of VOCOS_CASES and store what it computed as tests/golden/reference/vocos_<case>.pt. The vocos package is not installed, so while
the original runs its `Vocos` name is bound to tests/vocos_ref.py's RefVocos, the fp32 restatement of the published Vocos, loading a
seeded random checkpoint written to a temporary directory (nothing large is stored: the tests rebuild the same weights from the
seeds). Records the sampled mel, y0, each item's audio and the model's state_dict keys and shapes. Needs a checkout of the original:

    E2TTS_REFERENCE_FILE=<original>/e2_tts_pytorch/e2_tts.py python tools/make_vocos_golden.py
"""
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import vocos_ref as V  # noqa: E402
from vocos_ref import VOCOS_CASES, full_state_dict  # noqa: E402
from oracle import reference_cases as RC  # noqa: E402
from oracle.load_reference import load_reference  # noqa: E402

def main():
    ref = load_reference()
    ref.Vocos = V.RefVocos
    os.makedirs(RC.GOLDEN, exist_ok=True)
    for name, c in VOCOS_CASES.items():
        with tempfile.TemporaryDirectory() as d:
            V.write_checkpoint(d, c['g'], c['vseed'], opened=c['opened'])
            model = ref.E2TTS(transformer=dict(dropout=0., max_seq_len=128, **RC.KW), use_vocos=True, pretrained_vocos_path=d)
        model.load_state_dict(full_state_dict(c))
        model.eval()
        cond = RC.randn((c['cond'][0], c['cond'][1], 100), c['seed'] + 1000)
        kw = dict(text=c['text'], lens=torch.tensor(c['lens']), duration=torch.tensor(c['duration']), steps=c['steps'])
        with torch.no_grad():
            ref.torch = RC.noise(torch, 3000 + c['seed'])   # y0 = the first draw of that generator
            try:
                mel = model.sample(cond, return_raw_output=True, **kw)
            finally:
                ref.torch = torch
            ref.torch = RC.noise(torch, 3000 + c['seed'])
            try:
                audio = model.sample(cond, **kw)
            finally:
                ref.torch = torch
        y0 = RC.randn(tuple(mel.shape), 3000 + c['seed'])
        obj = dict(shape=tuple(mel.shape), mel=RC.compact(mel), y0=RC.compact(y0), audio=[RC.compact(a) for a in audio],
                   audio_lens=[int(a.numel()) for a in audio], shapes={k: tuple(v.shape) for k, v in model.state_dict().items()})
        path = os.path.join(RC.GOLDEN, f'vocos_{name}.pt')
        torch.save(obj, path)
        print(f'{os.path.basename(path)} {os.path.getsize(path) // 1024} KiB')


if __name__ == '__main__':
    main()
