"""CPU: the host side of GraphedSampler (E2TTS.sample as CUDA-graph replays per duration bucket) — every constructor refusal, each
raised before any kernel launch, the stage times of the fixed-grid solve, and the bucket choice and padding of y0, the conditioning,
the duration mask and the text ids for ragged prompts and durations."""
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


def _model(pkg, **kw):
    torch.manual_seed(0)
    return pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2, max_seq_len=512), use_vocos=False, **kw)


@pytest.mark.parametrize('kw, args, match', [
    (dict(odeint_kwargs=dict(method='dopri5')), {}, r"method 'dopri5'.*sample\(\)"),
    (dict(odeint_kwargs=dict(method='adaptive_heun', atol=1e-3)), {}, r"method 'adaptive_heun'.*sample\(\)"),
    ({}, dict(batch_size=33), r'batch_size 33.*2 \* batch_size <= 64'),
    ({}, dict(batch_size=0), 'batch_size 0'),
    ({}, dict(batch_size=64, cfg_strength=0.), 'model must live on the GPU'),     # one pass per evaluation: 64 items fit
    ({}, dict(batch_size=65, cfg_strength=0.), r'batch_size 65.*batch_size <= 64'),
    ({}, dict(buckets=(256, 513)), r"bucket 513 exceeds the transformer's max_seq_len \(512\)"),
    ({}, dict(buckets=()), 'buckets must be positive'),
    ({}, dict(steps=1), 'steps must be >= 2'),
    ({}, {}, 'model must live on the GPU'),
])
def test_refusals_before_any_launch(pkg, kw, args, match):
    model = _model(pkg, **kw)
    n0 = pkg.lib.launch_count()
    a = {**dict(batch_size=2, buckets=(256, 512)), **args}
    with pytest.raises(ValueError, match=match):
        pkg.GraphedSampler(model, a.pop('batch_size'), a.pop('buckets'), **a)
    assert pkg.lib.launch_count() == n0


def test_null_model_keeps_batch_limit_and_device_check(pkg):
    """with a cfg_null_model the two predictions come from two models, so each pass runs batch_size items"""
    model, null = _model(pkg), _model(pkg)
    n0 = pkg.lib.launch_count()
    with pytest.raises(ValueError, match='model must live on the GPU'):
        pkg.GraphedSampler(model, 64, (256,), cfg_null_model=null)
    assert pkg.lib.launch_count() == n0


def test_unsupported_method_name(pkg):
    model = _model(pkg)
    model.odeint_kwargs = dict(method='dopri8')
    with pytest.raises(NotImplementedError, match='dopri8'):
        pkg.GraphedSampler(model, 1, (256,))


@pytest.mark.parametrize('method, per_step', [('midpoint', 2), ('euler', 1), ('rk4', 4)])
def test_stage_times(pkg, method, per_step):
    from e2_tts_pytorch_b200.sampler import stage_times
    steps = 9
    tt = stage_times(method, steps)
    assert len(tt) == per_step * (steps - 1)
    ts = torch.linspace(0, 1, steps)
    assert tt[::per_step] == [float(t) for t in ts[:-1]]      # every step evaluates at its start first
    if method == 'midpoint':   # sample()'s t0 + 0.5 dt on an fp32 tensor
        assert tt[1::2] == [float(ts[i] + 0.5 * float(ts[i + 1] - ts[i])) for i in range(steps - 1)]
    if method == 'rk4':
        assert tt[3::4] == [float(t) for t in ts[1:]]
    assert tt == sorted(tt)


def _staged(pkg, model, buckets, cond, text, lens, duration, rows_per_item=2):
    from e2_tts_pytorch_b200.graphed import BucketPlan
    from e2_tts_pytorch_b200.modules import InterpolatedCharacterEmbed
    from e2_tts_pytorch_b200.sampler import stage_inputs
    cond, cond_mask, text, duration = model._sample_inputs(cond, text, lens, duration, 4096)
    B = cond.shape[0]
    plan = BucketPlan(buckets, B, 1024, isinstance(model.embed_text, InterpolatedCharacterEmbed), who='GraphedSampler')
    step_cond = torch.where(cond_mask, cond, torch.zeros_like(cond))
    y0 = torch.randn_like(cond)
    nb, buf = stage_inputs(plan, rows_per_item * B, y0, step_cond, duration, text)
    return nb, buf, dict(cond=cond, cond_mask=cond_mask, text=text, duration=duration, y0=y0, step_cond=step_cond)


@pytest.mark.parametrize('interpolated', [False, True])
def test_bucket_padding_ragged(pkg, interpolated):
    model = _model(pkg, interpolated_text=interpolated)
    torch.manual_seed(1)
    cond = torch.randn(3, 40, 100)
    text = ['a' * 50, 'hi', 'hello there']        # item 0's text is wider than its 40-frame prompt: lens grows to 50
    lens = torch.tensor([40, 12, 30])
    duration = torch.tensor([120, 5, 300])                             # item 1 is raised to its lens + 1
    nb, buf, got = _staged(pkg, model, (128, 256, 384, 512), cond, text, lens, duration)
    assert nb == 384 and got['cond'].shape[1] == 300                   # md = 300 -> the smallest bucket >= 300
    assert got['cond_mask'][:, :, 0].sum(1).tolist() == [50, 12, 30]  # lens = max(text lens, lens)
    assert got['duration'].tolist() == [120, 13, 300]                 # max(lens + 1, duration)
    for k in ('y0', 'cond'):
        assert buf[k].shape == (3, 384, 100)
        src = got['y0'] if k == 'y0' else got['step_cond']
        assert torch.equal(buf[k][:, :300], src) and not buf[k][:, 300:].any()
    assert not buf['cond'][1, 12:].any()                              # the step conditioning stops at the prompt
    mask = buf['mask']
    assert mask.shape == (6, 384) and torch.equal(mask[:3], mask[3:])  # both halves of the batched guidance pass
    assert mask[:3].sum(1).tolist() == [120, 13, 300]
    ids = got['text']
    assert buf['text'].shape == (3, 384)
    assert torch.equal(buf['text'][:, :ids.shape[1]], ids) and (buf['text'][:, ids.shape[1]:] == -1).all()


def test_bucket_padding_cuts_wide_text_and_refuses_it_when_interpolated(pkg):
    cond, lens, duration = torch.randn(1, 10, 100), torch.tensor([10]), torch.tensor([60])
    wide = torch.full((1, 200), -1, dtype=torch.long)
    wide[0, :5] = ord('x')                                            # 5 characters in 200 columns of -1 padding
    nb, buf, got = _staged(pkg, _model(pkg), (64, 128), cond, wide, lens, duration, rows_per_item=1)
    assert nb == 64 and buf['mask'].shape == (1, 64)
    assert torch.equal(buf['text'], wide[:, :64])                     # CharacterEmbed cuts to the frames itself
    with pytest.raises(ValueError, match='GraphedSampler: 200 text ids do not fit bucket 64'):
        _staged(pkg, _model(pkg, interpolated_text=True), (64, 128), cond, wide, lens, duration)


def test_duration_beyond_the_largest_bucket(pkg):
    with pytest.raises(ValueError, match=r'GraphedSampler: a batch of 300 frames exceeds the largest bucket \(256\)'):
        _staged(pkg, _model(pkg), (128, 256), torch.randn(1, 20, 100), ['hi'], None, torch.tensor([300]))
