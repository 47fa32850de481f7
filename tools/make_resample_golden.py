"""Run the ORIGINAL e2-tts-pytorch dataset path — HFDataset.__getitem__ (torchaudio.transforms.Resample to the target rate, then its
MelSpec) and collate_fn, from its own trainer.py, unmodified — on the resampling cases of tests/resample_ref.py, and store what it
computed as tests/golden/reference/resample_<case>.pt: mel_lengths, the mel's shape, a seeded sample of its elements and
the last TAIL frames of every item in full (the frames the resampled length reaches through the reflect padding). The waves
are regenerated from the seeds and handed to the dataset as in-memory rows {'audio': {'array', 'sampling_rate'}, 'transcript'}.

trainer.py imports a few packages the dataset path does not use (matplotlib, accelerate, adam_atan2_pytorch, ema_pytorch); they
are replaced by empty stand-ins, and `e2_tts_pytorch.e2_tts` resolves to the reference module oracle/load_reference.py loads.
Writes only those files. Needs a checkout of the original project:

    E2TTS_REFERENCE_FILE=<original>/e2_tts_pytorch/e2_tts.py python tools/make_resample_golden.py
"""
import importlib.util
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from oracle import reference_cases as RC  # noqa: E402
from oracle.load_reference import REF_FILE, load_reference  # noqa: E402
from resample_ref import MEL_SAMPLE, RESAMPLE_CASES, TAIL, case_waves  # noqa: E402


def _stand_in(name, **attrs):
    mod = types.ModuleType(name)
    mod.__dict__.update(attrs)
    sys.modules[name] = mod
    return mod


def load_trainer():
    ref = load_reference()
    pkg = _stand_in('e2_tts_pytorch', __path__=[])
    pkg.e2_tts = ref
    sys.modules['e2_tts_pytorch.e2_tts'] = ref
    mpl = _stand_in('matplotlib', use=lambda *a, **k: None)
    mpl.pylab = _stand_in('matplotlib.pylab')
    acc = _stand_in('accelerate', Accelerator=object)
    acc.utils = _stand_in('accelerate.utils', DistributedDataParallelKwargs=object)
    _stand_in('adam_atan2_pytorch', __path__=[])
    _stand_in('adam_atan2_pytorch.adopt', Adopt=object)
    _stand_in('ema_pytorch', EMA=object)
    path = os.path.join(os.path.dirname(REF_FILE), 'trainer.py')
    spec = importlib.util.spec_from_file_location('_e2tts_reference_trainer', path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    trainer = load_trainer()
    trainer.logger.remove()      # the dataset logs every item's shape
    import torchaudio
    os.makedirs(RC.GOLDEN, exist_ok=True)
    for name, c in RESAMPLE_CASES.items():
        waves, rates, target = case_waves(name)
        rows = [{'audio': {'array': w.numpy(), 'sampling_rate': r}, 'transcript': f'item {i}'} for i, (w, r) in enumerate(zip(waves, rates))]
        ds = trainer.HFDataset(rows, target_sample_rate=target)
        batch = trainer.collate_fn([ds[i] for i in range(len(ds))])
        mel = batch['mel']
        obj = dict(target=target, items=c['items'], mel_lengths=batch['mel_lengths'].clone(), mel_shape=tuple(mel.shape),
                   mel_values=mel.flatten()[RC.sample_index(mel.numel(), MEL_SAMPLE)].clone(),
                   mel_tail=torch.stack([mel[b, :, n - TAIL:n] for b, n in enumerate(batch['mel_lengths'].tolist())]).clone(),
                   torchaudio=torchaudio.__version__)
        path = os.path.join(RC.GOLDEN, f'resample_{name}.pt')
        torch.save(obj, path)
        print(f'{os.path.basename(path)} {os.path.getsize(path) // 1024} KiB, mel {tuple(mel.shape)}, lengths {batch["mel_lengths"].tolist()}')


if __name__ == '__main__':
    main()
