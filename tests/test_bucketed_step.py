"""CPU: the host side of BucketedTrainStep (graphed training steps on ragged batches) — bucket choice, text padding, the text-drop
coin, and every refusal, each raised before any kernel launch — and the C-ABI declaration of b200_flat_accumulate."""
import ctypes
import os
import random
import subprocess

import pytest
import torch

from conftest import ROOT


@pytest.fixture(scope='module')
def pkg():
    so = os.path.join(ROOT, 'e2-tts-pytorch_b200', 'libb200e2tts.so')
    if not os.path.isfile(so):
        subprocess.run(['make', '-C', os.path.join(ROOT, 'e2-tts-pytorch_b200', 'csrc'), '-j8', 'all'], check=True)
    import e2_tts_pytorch_b200 as pkg
    return pkg


def _model(pkg, **kw):
    torch.manual_seed(0)
    return pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2, max_seq_len=512), use_vocos=False, **kw)


def test_header_declares_flat_accumulate(pkg):
    restype, argt = pkg.lib.FUNCTIONS['b200_flat_accumulate']
    assert restype is ctypes.c_int
    assert argt == [ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p]
    assert pkg.lib.FUNCTIONS['b200_flat_gather'] == pkg.lib.FUNCTIONS['b200_flat_accumulate']   # the same signature as its twin
    assert hasattr(pkg.lib.load(), 'b200_flat_accumulate')


def test_bucket_choice(pkg):
    from e2_tts_pytorch_b200.graphed import BucketPlan
    plan = BucketPlan((512, 256, 768), 4, 1024)
    assert plan.buckets == (256, 512, 768)
    assert [plan.bucket(n) for n in (1, 255, 256, 257, 512, 513, 768)] == [256, 256, 256, 512, 512, 768, 768]
    assert plan.check(4, 300) == 512 and plan.check(4, 300, text_width=900) == 512   # CharacterEmbed: the text is cut
    with pytest.raises(ValueError, match='largest bucket'):
        plan.bucket(769)
    with pytest.raises(ValueError, match='batch_size=4'):
        plan.check(5, 100)
    interp = BucketPlan((256, 512), 4, 1024, interpolated_text=True)
    assert interp.check(4, 300, text_width=512) == 512
    with pytest.raises(ValueError, match='interpolated_text'):
        interp.check(4, 300, text_width=513)


def test_plan_refusals(pkg):
    from e2_tts_pytorch_b200.graphed import BucketPlan
    with pytest.raises(ValueError, match='max_seq_len'):
        BucketPlan((256, 1025), 4, 1024)
    with pytest.raises(ValueError, match='64'):
        BucketPlan((256,), 65, 1024)
    with pytest.raises(ValueError, match='positive'):
        BucketPlan((), 4, 1024)


def test_text_padding_and_cutting_equal_character_embed(pkg):
    from e2_tts_pytorch_b200.graphed import BucketPlan
    embed = _model(pkg).embed_text
    ids = pkg.list_str_to_tensor(['a short one', 'x', 'a much longer line of text than the others']).long()
    for nb in (4, 11, 40, 64):
        padded = BucketPlan.pad_text(ids, nb)
        assert padded.shape == (3, nb)
        assert torch.equal(embed.ids(padded, nb), embed.ids(ids, nb)), nb
        w = min(nb, ids.shape[1])
        assert torch.equal(padded[:, :w], ids[:, :w]) and bool((padded[:, w:] == -1).all())


def test_constructor_refusals_before_any_launch(pkg):
    n0 = pkg.lib.launch_count()
    m = _model(pkg)
    with pytest.raises(ValueError, match='max_seq_len'):
        pkg.BucketedTrainStep(m, 4, (256, 1024))
    with pytest.raises(ValueError, match='64'):
        pkg.BucketedTrainStep(m, 65, (256,))
    with pytest.raises(ValueError, match='grad_accumulation_steps'):
        pkg.BucketedTrainStep(m, 4, (256,), grad_accumulation_steps=0)
    with pytest.raises(ValueError, match='velocity consistency'):
        pkg.BucketedTrainStep(_model(pkg, velocity_consistency_weight=0.1), 4, (256,))
    with pytest.raises(ValueError, match='GPU'):      # every argument is fine: only the device is missing
        pkg.BucketedTrainStep(m, 4, (256,))
    assert pkg.lib.launch_count() == n0


def test_text_modes_follow_cond_drop_prob(pkg):
    from e2_tts_pytorch_b200.graphed import text_modes
    m = _model(pkg).train()
    for p, want in ((0.0, (False,)), (0.25, (False, True)), (1.0, (True,))):
        m.cond_drop_prob = p
        assert text_modes(m) == want, p
    m.eval()
    assert text_modes(m) == (False,)
    d = pkg.DurationPredictor(transformer=dict(dim=128, depth=2, heads=2)).train()
    assert text_modes(d) == (False,)


def test_text_drop_coin_is_one_python_draw_per_call(pkg):
    from e2_tts_pytorch_b200.graphed import draw_text_drop
    m = _model(pkg).train()
    m.cond_drop_prob = 0.25
    random.seed(1234)
    got = [draw_text_drop(m, True) for _ in range(200)]
    random.seed(1234)
    want = [random.random() < 0.25 for _ in range(200)]   # transformer_with_pred_head's coin, e2_tts.py:1261
    assert got == want and 20 < sum(got) < 80
    random.seed(7)
    assert draw_text_drop(m, False) is True                # no text: the dropped graph, and the coin is still drawn
    after_one = random.getstate()
    random.seed(7)
    random.random()
    assert random.getstate() == after_one
    for p in (0.0, 1.0):                                   # one draw whatever the probability
        m.cond_drop_prob = p
        random.seed(7)
        assert draw_text_drop(m, True) is (p == 1.0)
        assert random.getstate() == after_one
    m.eval()
    d = pkg.DurationPredictor(transformer=dict(dim=128, depth=2, heads=2)).train()   # its constructor draws from `random` itself
    random.seed(7)
    before = random.getstate()
    assert draw_text_drop(m, True) is False and random.getstate() == before   # eval mode draws nothing (`self.training and ...`)
    assert draw_text_drop(d, True) is False and random.getstate() == before


def test_python_random_state_is_restored_after_construction_work(pkg):
    from e2_tts_pytorch_b200.graphed import _KeepPythonRandom
    random.seed(99)
    before = random.getstate()
    with pytest.raises(RuntimeError):
        with _KeepPythonRandom():
            [random.random() for _ in range(5)]
            raise RuntimeError('a capture failed')
    assert random.getstate() == before
