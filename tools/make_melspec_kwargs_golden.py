"""Run the ORIGINAL e2-tts-pytorch MelSpec (its own e2_tts.py, loaded unmodified by oracle/load_reference.py, on the installed
torchaudio) on the mel_spec_kwargs cases of tests/mel_kwargs_ref.py and store what it computed as
tests/golden/reference/melspec_kwargs_<case>.pt: the log-mel and the state_dict shapes. The waves are regenerated from the seeds.
Writes only those files. Needs a checkout of the original project:

    E2TTS_REFERENCE_FILE=<original>/e2_tts_pytorch/e2_tts.py python tools/make_melspec_kwargs_golden.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from mel_kwargs_ref import MEL_KWARGS_CASES, case_wave  # noqa: E402
from oracle import reference_cases as RC  # noqa: E402
from oracle.load_reference import load_reference  # noqa: E402


def main():
    ref = load_reference()
    import torchaudio
    os.makedirs(RC.GOLDEN, exist_ok=True)
    for name, c in MEL_KWARGS_CASES.items():
        ms = ref.MelSpec(**c['kw'])
        mel = ms(case_wave(c))
        obj = dict(kw=c['kw'], mel=mel.detach().clone(), shapes={k: tuple(v.shape) for k, v in ms.state_dict().items()},
                   torchaudio=torchaudio.__version__)
        path = os.path.join(RC.GOLDEN, f'melspec_kwargs_{name}.pt')
        torch.save(obj, path)
        print(f'{os.path.basename(path)} {os.path.getsize(path) // 1024} KiB, mel {tuple(mel.shape)}')


if __name__ == '__main__':
    main()
