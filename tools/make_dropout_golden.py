"""Run the ORIGINAL e2-tts-pytorch code (its own e2_tts.py, loaded unmodified by oracle/load_reference.py) with dropout on, on the cases
of tests/dropout_ref.py, and store what it computed as tests/golden/reference/dropout_<case>.pt, in the record format of
oracle/make_reference_golden.py. The models are built with dropout = P_REF; before the forward every nn.Dropout module is replaced by
one that multiplies by the hashed mask of tests/dropout_ref.py (its qualified name, the input shape and the case seed), so the test can
give the oracle the same masks without the original code. The record also lists the modules that dropped. Writes only those files.
Needs a checkout of the original project:

    E2TTS_REFERENCE_FILE=<original>/e2_tts_pytorch/e2_tts.py python tools/make_dropout_golden.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from dropout_ref import DROPOUT_CASES, P_REF, HashedDropout  # noqa: E402
from oracle import reference_cases as RC  # noqa: E402
from oracle.load_reference import load_reference, run_reference_forward  # noqa: E402


def hash_dropouts(model, seed, log):
    """every nn.Dropout of `model` -> HashedDropout of its qualified name; returns how many were replaced"""
    found = [(n, m) for n, m in model.named_modules() if isinstance(m, torch.nn.Dropout)]
    for name, m in found:
        assert m.p == P_REF, (name, m.p)
        parent, _, leaf = name.rpartition('.')
        model.get_submodule(parent)._modules[leaf] = HashedDropout(name, seed, P_REF, log)
    return len(found)


def main():
    ref = load_reference()
    os.makedirs(RC.GOLDEN, exist_ok=True)
    for name, c in DROPOUT_CASES.items():
        tkw = c['tkw']
        mel = RC.randn((c['mel'][0], c['mel'][1], 100), c['seed'] + 1000)
        lens = torch.tensor(c['lens'])
        log = []
        if c['cls'] == 'E2TTS':
            model = ref.E2TTS(transformer=dict(dropout=P_REF, max_seq_len=128, **tkw), use_vocos=False)
            model.load_state_dict(RC.state_dict('E2TTS', c['seed'], tkw))
            assert hash_dropouts(model, c['seed'], log) > 0
            model.train()
            torch.manual_seed(c['seed'])
            ref.torch = RC.noise(torch, c['seed'] + 2000)   # x0 = the first draw of that generator
            try:
                out, rec = run_reference_forward(ref, model, mel, c['text'], lens=lens, drop_text_cond=c['drop'])
            finally:
                ref.torch = torch
            out.loss.backward()
            obj = dict(loss=float(out.loss.detach()), pred=RC.compact(out.pred_flow), times=rec['times'], span_mask=rec['span_mask'])
        else:
            model = ref.DurationPredictor(transformer=dict(dropout=P_REF, max_seq_len=128, **tkw))
            model.load_state_dict(RC.state_dict('DurationPredictor', c['seed'], tkw))
            assert hash_dropouts(model, c['seed'], log) > 0
            model.train()
            torch.manual_seed(c['seed'])
            loss = model(mel, text=c['text'], lens=lens)
            loss.backward()
            obj = dict(loss=float(loss.detach()))
        obj['grads'] = RC.grad_record({k: (p.grad.clone() if p.grad is not None else None) for k, p in model.named_parameters()})
        obj['dropped'] = log
        path = os.path.join(RC.GOLDEN, f'dropout_{name}.pt')
        torch.save(obj, path)
        print(f'{os.path.basename(path)} {os.path.getsize(path) // 1024} KiB, {len(log)} dropout calls')


if __name__ == '__main__':
    main()
