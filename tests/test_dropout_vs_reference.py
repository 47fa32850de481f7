"""CPU: the oracle's dropout hook (O.DROPOUT) against the original e2_tts.py trained with dropout on. tools/make_dropout_golden.py ran
the original with dropout = 0.25, every nn.Dropout replaced by a seeded mask of its qualified name (tests/dropout_ref.py), on an E2TTS
of depth 2 with ragged lengths, with the text dropped, with num_residual_streams=1, with 2 x 128 audio heads and 1 x 64 text heads,
and on a DurationPredictor (tests/golden/reference/dropout_*.pt). The oracle, given the same masks through the hook, must match its
loss, prediction and gradient samples within the bounds of tests/test_oracle_vs_reference.py and drop at exactly the same modules;
without the hook it must not match (negative control).

Where inside Attention and FeedForward the reference drops (the softmax probabilities before `attn @ v`, the GEGLU hidden before the
output Linear) comes from the restated x-transformers leaf (oracle/ref_leaves/x_transformers/x_transformers.py:53, :113), which is
parity-unpinned (oracle/ref_leaves/README.md): these fixtures pin the oracle to the reference's composition around those two modules,
not the placement inside them."""
import pytest
import torch

from dropout_ref import DROPOUT_CASES, P_REF, HashedHook, with_dropout
from headdim_variants import cfg, headdim_oracle
from model_checks import check_grads, grad_sd
from oracle import e2tts_oracle as O
from oracle import reference_cases as RC


def _oracle(c, g, hook):
    """loss (with grads in the returned state dict) and prediction of the oracle on case `c` with O.DROPOUT = hook"""
    sd = grad_sd(RC.state_dict(c['cls'], c['seed'], c['tkw']))
    mel = RC.randn((c['mel'][0], c['mel'][1], 100), c['seed'] + 1000)
    lens = torch.tensor(c['lens'])
    text = O.list_str_to_tensor(c['text'])
    pred = None
    with headdim_oracle(c['tkw']):
        if c['cls'] == 'E2TTS':
            x0 = RC.randn(mel.shape, c['seed'] + 2000)
            o = with_dropout(hook, O.e2tts_forward, sd, cfg(c['tkw']), mel, text, lens=lens, x0=x0, times=g['times'],
                             span_mask=g['span_mask'], drop_text_cond=c['drop'])
            loss, pred = o['loss'], o['pred']
        else:
            torch.manual_seed(c['seed'])
            rand_frac = mel.new_zeros(mel.shape[0]).uniform_(0, 1)   # the draw of e2_tts.py:1082 under the same seed
            loss = with_dropout(hook, O.duration_forward, sd, cfg(c['tkw'], cond_on_time=False), mel, text, lens=lens,
                                rand_frac=rand_frac)
    loss.backward()
    return sd, loss, pred


def _check(c, g, sd, loss, pred):
    if pred is not None:
        assert RC.compact_rel_l2(pred, g['pred']) < 1e-4
        assert abs(float(pred.detach().double().norm()) - g['pred']['norm']) <= 1e-4 * g['pred']['norm']
    assert abs(float(loss.detach()) - g['loss']) <= 1e-5 * abs(g['loss'])
    if c['cls'] == 'E2TTS':
        check_grads(sd, g['grads'])
    else:
        check_grads(sd, g['grads'], rel=5e-4, floor=1e-6)


@pytest.mark.parametrize('name', list(DROPOUT_CASES))
def test_oracle_dropout_vs_reference(name):
    c = DROPOUT_CASES[name]
    g = RC.load('dropout_' + name)
    hook = HashedHook(c['seed'], P_REF)
    sd, loss, pred = _oracle(c, g, hook)
    # one drop per attention and feed-forward the reference ran, at the same qualified names
    assert sorted(hook.names) == sorted(g['dropped']) and len(set(hook.names)) == len(hook.names)
    tkw = c['tkw']
    n_blocks = tkw['depth'] + (0 if c['drop'] else tkw['depth'])
    assert len(hook.names) == 2 * n_blocks
    _check(c, g, sd, loss, pred)
    # negative control: the same comparison without the hook fails
    with pytest.raises(AssertionError):
        _check(c, g, *_oracle(c, g, None))
