"""Run the ORIGINAL e2-tts-pytorch code (its own e2_tts.py, loaded unmodified by oracle/load_reference.py) with the HL-Gauss
classification head of DurationPredictor (hl_gauss_loss=dict(...), use_regression=False) and store what it computed under
tests/golden/reference/:
  hl_gauss_<case>.pt   per case of tests/hl_gauss_variants.py HL_GAUSS_CASES: the training loss, a gradient sample per parameter and
                       the state_dict shapes (the record format of oracle/make_reference_golden.py's forward cases)
  hl_gauss_predict.pt  each case's predictions (return_loss=False) on the same inputs
  hl_gauss_sample.pt   E2TTS.sample without `duration` driven by such a predictor (HL_GAUSS_SAMPLE): the predictions it made and the
                       sample; y0 = the first draw of generator 3000 + seed
hl-gauss-pytorch is not installed and the restated leaf of oracle/ref_leaves/ takes the regression mode only, so while the original
runs its `HLGaussLayer` name is bound to tests/hl_gauss_ref.py's restatement of both modes. Only outputs are stored: weights, inputs
and injected noise are rebuilt from seeds (oracle/reference_cases.py). Needs a checkout of the original:

    E2TTS_REFERENCE_FILE=<original>/e2_tts_pytorch/e2_tts.py python tools/make_hl_gauss_golden.py
"""
import copy
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from hl_gauss_ref import HLGaussLayer  # noqa: E402
from hl_gauss_variants import HL_GAUSS_CASES, HL_GAUSS_SAMPLE  # noqa: E402
from oracle import reference_cases as RC  # noqa: E402
from oracle.load_reference import load_reference  # noqa: E402


def save(name, obj):
    os.makedirs(RC.GOLDEN, exist_ok=True)
    path = os.path.join(RC.GOLDEN, name + '.pt')
    torch.save(obj, path)
    print(f'{name}.pt {os.path.getsize(path) // 1024} KiB')


def duration_predictor(ref, c):
    model = ref.DurationPredictor(transformer=dict(dropout=0., max_seq_len=128, **c['tkw']), **copy.deepcopy(c['kw']))
    model.load_state_dict(RC.state_dict(c['cls'], c['seed'], c['tkw'], **c['kw']))
    return model, RC.randn((c['mel'][0], c['mel'][1], 100), c['seed'] + 1000), torch.tensor(c['lens'])


def record_case(ref, c):
    """training loss (prefix fractions drawn under torch.manual_seed(seed), as e2_tts.py:1082 draws them), gradients, shapes"""
    model, mel, lens = duration_predictor(ref, c)
    torch.manual_seed(c['seed'])
    loss = model(mel, text=c['text'], lens=lens)
    loss.backward()
    grads = {k: (p.grad.clone() if p.grad is not None else None) for k, p in model.named_parameters()}
    return dict(loss=float(loss.detach()), grads=RC.grad_record(grads), shapes={k: tuple(v.shape) for k, v in model.state_dict().items()})


def record_predictions(ref):
    preds = {}
    for name, c in HL_GAUSS_CASES.items():
        model, mel, lens = duration_predictor(ref, c)
        model.eval()
        with torch.no_grad():
            preds[name] = model(mel, text=c['text'], lens=lens, return_loss=False)
    return preds


def record_sample(ref):
    s = HL_GAUSS_SAMPLE
    model = ref.E2TTS(transformer=dict(dropout=0., max_seq_len=128, **s['tkw']), duration_predictor=copy.deepcopy(s['duration_predictor']),
                      use_vocos=False)
    model.load_state_dict(RC.state_dict('E2TTS', s['seed'], s['tkw'], duration_predictor=copy.deepcopy(s['duration_predictor'])))
    model.eval()
    seen = []
    dp_forward = model.duration_predictor.forward
    model.duration_predictor.forward = lambda *a, **k: seen.append(dp_forward(*a, **k)) or seen[-1]
    cond = RC.randn((s['cond'][0], s['cond'][1], 100), s['seed'] + 1000)
    ref.torch = RC.noise(torch, 3000 + s['seed'])
    try:
        with torch.no_grad():
            want = model.sample(cond, text=s['text'], steps=s['steps'], cfg_strength=s['cfg_strength'], return_raw_output=True)
    finally:
        ref.torch = torch
    assert len(seen) == 1
    return dict(pred=seen[0], shape=tuple(want.shape), out=RC.compact(want))


def main():
    ref = load_reference()
    ref.HLGaussLayer = HLGaussLayer   # e2_tts.py:1035 builds HLGaussLayer(dim, hl_gauss_loss=..., use_regression=..., regress_activation=...)
    for name, c in HL_GAUSS_CASES.items():
        save('hl_gauss_' + name, record_case(ref, c))
    save('hl_gauss_predict', record_predictions(ref))
    save('hl_gauss_sample', record_sample(ref))


if __name__ == '__main__':
    main()
