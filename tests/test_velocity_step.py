"""CPU: the host side of graphed training steps with a velocity-consistency teacher (GraphedTrainStep / BucketedTrainStep with
`velocity_consistency_model=`): every refusal, in the constructors and per call, raised before any kernel launch."""
import os
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


def _model(pkg, weight=0.1, tkw=None, **kw):
    torch.manual_seed(0)
    t = {**dict(dim=128, depth=2, heads=2, max_seq_len=512), **(tkw or {})}
    return pkg.E2TTS(transformer=t, use_vocos=False, velocity_consistency_weight=weight, **kw)


def _both(pkg, model, teacher, frames=256, **kw):
    """the constructors of both steps with this teacher; each must raise the same ValueError"""
    mel = torch.zeros(2, frames, 100)
    yield lambda: pkg.GraphedTrainStep(model, mel, velocity_consistency_model=teacher, **kw)
    yield lambda: pkg.BucketedTrainStep(model, 2, (128, frames), velocity_consistency_model=teacher, **kw)


TEACHER_REFUSALS = {
    'duration_predictor': (lambda pkg: (pkg.DurationPredictor(transformer=dict(dim=128, depth=2, heads=2)), _model(pkg)), 'only an E2TTS'),
    'zero_weight': (lambda pkg: (_model(pkg, weight=0.0), _model(pkg)), 'velocity_consistency_weight is 0'),
    'not_e2tts': (lambda pkg: (_model(pkg), _model(pkg).transformer), 'must be an E2TTS'),
    'itself': (lambda pkg: (lambda m: (m, m))(_model(pkg)), 'the model itself'),
    'depth': (lambda pkg: (_model(pkg), _model(pkg, tkw=dict(depth=4))), 'state_dict differs'),
    'concat_cond': (lambda pkg: (_model(pkg), _model(pkg, concat_cond=True)), 'state_dict differs'),
    'num_channels': (lambda pkg: (_model(pkg), _model(pkg, num_channels=80)), 'state_dict differs'),
    'softclamp': (lambda pkg: (_model(pkg), _model(pkg, tkw=dict(attn_kwargs=dict(gate_value_heads=True, softclamp_logits=False)))),
                  'softclamp'),
    'device': (lambda pkg: (_model(pkg), _model(pkg).to('meta')), 'lives on meta'),
}


@pytest.mark.parametrize('case', list(TEACHER_REFUSALS))
def test_teacher_refused_before_any_launch(pkg, case):
    make, match = TEACHER_REFUSALS[case]
    model, teacher = make(pkg)
    n0 = pkg.lib.launch_count()
    for ctor in _both(pkg, model, teacher):
        with pytest.raises(ValueError, match=match):
            ctor()
    assert pkg.lib.launch_count() == n0


def test_frames_above_the_teachers_max_seq_len_refused(pkg):
    # without the absolute position table the two max_seq_len give the same state_dict: only the length check can catch it
    model = _model(pkg, tkw=dict(abs_pos_emb=False))
    teacher = _model(pkg, tkw=dict(abs_pos_emb=False, max_seq_len=256))
    n0 = pkg.lib.launch_count()
    for ctor in _both(pkg, model, teacher, frames=300):
        with pytest.raises(ValueError, match=r"300 frames exceed the velocity_consistency_model's max_seq_len \(256\)"):
            ctor()
    model.cond_drop_prob = 0.0      # GraphedTrainStep captures one text mode
    for ctor in _both(pkg, model, teacher, frames=256):      # at the teacher's limit only the device is missing
        with pytest.raises(ValueError, match='GPU'):
            ctor()
    assert pkg.lib.launch_count() == n0


def test_weight_without_teacher_still_refused_by_the_bucketed_step(pkg):
    n0 = pkg.lib.launch_count()
    with pytest.raises(ValueError, match='velocity consistency'):
        pkg.BucketedTrainStep(_model(pkg), 4, (256,))
    assert pkg.lib.launch_count() == n0


def test_per_call_refusals(pkg):
    from e2_tts_pytorch_b200.graphed import VelocityTeacher, velocity_flag
    n0 = pkg.lib.launch_count()
    assert velocity_flag(None, None, 'X') is False and velocity_flag(None, False, 'X') is False
    with pytest.raises(ValueError, match='velocity=True on a step built without velocity_consistency_model'):
        velocity_flag(None, True, 'X')
    model, teacher = _model(pkg), _model(pkg).eval()
    vt = VelocityTeacher(model, teacher, 1e-5, 256, 'X')
    vt.add_seed_word()
    assert vt.seed_dev is None and teacher.transformer._seed_dev is None     # eval mode: no dropout seed, no seed word
    vt.seal()
    assert velocity_flag(vt, None, 'X') is True and velocity_flag(vt, False, 'X') is False
    teacher.train()
    with pytest.raises(ValueError, match='captured in eval mode'):
        velocity_flag(vt, None, 'X')
    teacher.eval()
    with torch.no_grad():
        teacher.to_pred.weight.mul_(0.5)           # in place, as copy_ema_to and EMA.update write: fine
    assert velocity_flag(vt, True, 'X') is True
    teacher.to_pred.weight.data = teacher.to_pred.weight.data.clone()     # new storage: the graph would read the old one
    with pytest.raises(ValueError, match='new storage since capture'):
        velocity_flag(vt, True, 'X')
    assert velocity_flag(vt, False, 'X') is False   # the graph without the teacher does not read it
    assert pkg.lib.launch_count() == n0


def test_teacher_in_training_mode_gets_its_own_seed_word(pkg):
    from e2_tts_pytorch_b200.graphed import VelocityTeacher
    model, teacher = _model(pkg).train(), _model(pkg).train()
    vt = VelocityTeacher(model, teacher, 1e-5, 256, 'X')
    vt.add_seed_word()
    assert vt.seed_dev is teacher.transformer._seed_dev and vt.seed_dev is not None
    assert model.transformer._seed_dev is None
