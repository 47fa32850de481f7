"""CPU: the oracle's dropout hook (O.DROPOUT) against the original e2_tts.py trained with dropout on. oracle/make_reference_golden.py ran
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

from dropout_ref import DROPOUT_CASES, P_REF, HashedHook
from model_checks import check_case, oracle_case
from oracle import reference_cases as RC


@pytest.mark.parametrize('name', list(DROPOUT_CASES))
def test_oracle_dropout_vs_reference(name):
    c = DROPOUT_CASES[name]
    g = RC.load('dropout_' + name)
    hook = HashedHook(c['seed'], P_REF)
    sd, loss, pred = oracle_case(c, g, hook=hook)
    # one drop per attention and feed-forward the reference ran, at the same qualified names
    assert sorted(hook.names) == sorted(g['dropped']) and len(set(hook.names)) == len(hook.names)
    tkw = c['tkw']
    n_blocks = tkw['depth'] + (0 if c['drop'] else tkw['depth'])
    assert len(hook.names) == 2 * n_blocks
    check_case(c, g, sd, loss, pred)
    # negative control: the same comparison without the hook fails
    with pytest.raises(AssertionError):
        check_case(c, g, *oracle_case(c, g))
