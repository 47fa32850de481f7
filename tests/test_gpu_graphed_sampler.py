"""GPU: GraphedSampler (e2-tts-pytorch_b200/sampler.py) and the batched guidance pass it runs (E2TTS.cfg_pred_batched).

The batched pass — the conditional and the text-dropped prediction as one transformer pass over 2B items — against
cfg_transformer_with_pred_head's two passes on the same inputs, on every geometry whose text stream differs; its text-dropped half
against a drop_text_cond pass. The sampler against the oracle's fixed-grid ODE (the bound of sample_vs_oracle) and against eager
sample() with the same seed, for midpoint / euler / rk4, several guidance strengths, ragged prompts and durations, no text, a
cfg_null_model and a DurationPredictor; and the properties of the replays: repeatable bits, buckets that do not leak into each
other, one memory pool, and weights that follow load_state_dict."""
import gc
import random

import pytest
import torch

import ode_ref
from conftest import rel_l2
from kernel_checks import dev, pkg  # noqa: F401
from model_checks import small_model
from oracle import e2tts_oracle as O

pytestmark = pytest.mark.gpu

SMALL = dict(dim=128, depth=2, heads=2)


def model_of(pkg, seed, e2tts_kw=None, max_seq_len=256, **tkw):
    """small_model with E2TTS keyword arguments too: (model on the GPU, its state dict)"""
    torch.manual_seed(seed)
    random.seed(seed)
    model = pkg.E2TTS(transformer=dict(dropout=0., max_seq_len=max_seq_len, **tkw), use_vocos=False, **(e2tts_kw or {}))
    sd = O.randomize_zero_init({k: v.clone() for k, v in model.state_dict().items()}, seed=seed + 1)
    model.load_state_dict(sd)
    return model.to(dev()).eval(), sd


# ---------------------------------------------------------------------------------------------------- the batched guidance pass
GEOMETRIES = {
    'default': (SMALL, {}),
    'concat_cond': (SMALL, dict(concat_cond=True)),
    'interpolated_text': (SMALL, dict(interpolated_text=True)),
    'plain_residual': (dict(SMALL, num_residual_streams=1), {}),
    'text_depth_2_of_4': (dict(dim=128, depth=4, heads=2, text_depth=2), {}),
    'dim_head_128': (dict(dim=256, depth=2, heads=2, dim_head=128, text_dim_head=128), {}),
}


# The hyper-connections fuse each depth connection into the next width connection when a stream's rows allow it (ops.hc_can_fuse:
# T * S a multiple of 64), and that changes where the residual streams round to bf16. At 80 frames (112 rows per item with the 32
# registers) B and 2B items decide alike, so the batched pass runs the kernels of the two passes on the same rows: the same bits. At
# 72 frames only the 2B-item audio stream fuses, so the two differ by bf16 rounding.
CASES = [(name, 80) for name in GEOMETRIES] + [('default', 72)]


@pytest.mark.parametrize('name, N', CASES, ids=[f'{n}-N{N}' for n, N in CASES])
def test_batched_pass_matches_two_passes(pkg, name, N):
    tkw, ekw = GEOMETRIES[name]
    model, _ = model_of(pkg, 11, ekw, **tkw)
    B = 3
    torch.manual_seed(12)
    x, cond = torch.randn(B, N, 100, device=dev()), torch.randn(B, N, 100, device=dev())
    cond[:, 30:] = 0.
    duration = torch.tensor([N, 40, 61], device=dev())
    mask = pkg.lens_to_mask(duration, N)
    text = pkg.list_str_to_tensor(['Hello', 'Goodbye then', 'x']).to(dev())
    t = torch.tensor(0.37, device=dev())
    with torch.no_grad():
        w = model._pack()[0]
        with w.freeze():
            pred, null = model._pred_pair(x, cond, t, torch.cat([mask, mask]), text)
            want_pred = model.transformer_with_pred_head(x, cond, times=t, mask=mask, text=text, drop_text_cond=False)
            want_null = model.transformer_with_pred_head(x, cond, times=t, mask=mask, text=text, drop_text_cond=True)
            got = model.cfg_pred_batched(x, cond, t, torch.cat([mask, mask]), text, 2.0)
            want = model.cfg_transformer_with_pred_head(x, cond, times=t, mask=mask, text=text, cfg_strength=2.0)
    torch.cuda.synchronize()
    for b in range(B):
        m = mask[b]
        e_p = rel_l2(pred[b][m].cpu(), want_pred[b][m].cpu())
        e_n = rel_l2(null[b][m].cpu(), want_null[b][m].cpu())
        e_c = rel_l2(got[b][m].cpu(), want[b][m].cpu())
        print(f'{name} item {b}: conditional {e_p:.3g}, text-dropped {e_n:.3g} (bitwise {torch.equal(null[b], want_null[b])}), '
              f'guided {e_c:.3g}')
        assert e_p < 3e-2 and e_c < 3e-2 and e_n < 3e-2   # the bound of the whole-model checks against the oracle
    same_fusion = pkg.ops.hc_can_fuse(B * (N + 32), 4) == pkg.ops.hc_can_fuse(2 * B * (N + 32), 4)
    if same_fusion or tkw.get('num_residual_streams') == 1:
        assert torch.equal(null, want_null)        # the text-dropped half is a pass without text over the same items
        assert torch.equal(pred, want_pred)        # and the text half the conditional pass
    # the text stream reaches only the first half: with all rows there, the prediction moves; the text-dropped half has no text path
    assert rel_l2(pred.cpu(), null.cpu()) > 1e-3


def test_batched_pass_without_text_is_one_pass(pkg):
    model, _ = model_of(pkg, 13, **SMALL)
    x, cond = torch.randn(2, 48, 100, device=dev()), torch.zeros(2, 48, 100, device=dev())
    mask = torch.ones(2, 48, dtype=torch.bool, device=dev())
    t = torch.tensor(0.5, device=dev())
    with torch.no_grad():
        n0 = pkg.lib.launch_count()
        got = model.cfg_pred_batched(x, cond, t, torch.cat([mask, mask]), None, 1.0)
        n_batched = pkg.lib.launch_count() - n0
        n0 = pkg.lib.launch_count()
        want = model.cfg_transformer_with_pred_head(x, cond, times=t, mask=mask, text=None, cfg_strength=1.0)
        n_eager = pkg.lib.launch_count() - n0
    assert torch.equal(got, want)     # both eager passes see the same inputs: one pass combined with itself gives their bits
    assert n_batched < n_eager


# ---------------------------------------------------------------------------------------------------- the sampler
def eager_and_graphed(pkg, model, sampler_kw, call_kw, y0, steps, cfg_strength, cfg_null_model=None, buckets=(64, 128)):
    sampler = pkg.GraphedSampler(model, y0.shape[0], buckets, steps=steps, cfg_strength=cfg_strength, cfg_null_model=cfg_null_model,
                                 **sampler_kw)
    with pkg.inject_randomness(y0=y0.to(dev())):
        got = sampler(**call_kw, return_raw_output=True)
        want = model.sample(**call_kw, steps=steps, cfg_strength=cfg_strength, cfg_null_model=cfg_null_model, return_raw_output=True)
    torch.cuda.synchronize()
    assert got.shape == want.shape
    e = rel_l2(got.cpu(), want.cpu())
    print(f'graphed vs eager sample(): rel-L2 {e:.3g}')
    assert e < 2e-2
    return sampler, got


SAMPLE_CASES = {
    'midpoint_cfg1': dict(method='midpoint', cfg=1.0),
    'euler_cfg2.5': dict(method='euler', cfg=2.5),
    'rk4_cfg0': dict(method='rk4', cfg=0.0),
    'rk4_cfg1': dict(method='rk4', cfg=1.0),
    'midpoint_ragged_cfg2.5': dict(method='midpoint', cfg=2.5, lens=[20, 9], duration=[70, 41]),
    'midpoint_no_text': dict(method='midpoint', cfg=1.0, text=None),
    'euler_null_model': dict(method='euler', cfg=1.5, null=True),
}


@pytest.mark.parametrize('name', list(SAMPLE_CASES))
def test_sampler_vs_oracle(pkg, name):
    c = SAMPLE_CASES[name]
    model, sd = small_model(pkg, 60, **SMALL)
    model.odeint_kwargs = dict(method=c['method'])
    null, null_sd = small_model(pkg, 80, **SMALL) if c.get('null') else (None, None)
    torch.manual_seed(61)
    cond = torch.randn(2, 24, 100)
    text = c.get('text', ['Hello', 'Goodbye'])
    lens = torch.tensor(c['lens']) if 'lens' in c else None
    duration = torch.tensor(c['duration']) if 'duration' in c else 64
    y0 = torch.randn(2, int(torch.as_tensor(duration).max()), 100)
    steps = 5
    call_kw = dict(cond=cond.to(dev()), text=text, lens=lens.to(dev()) if lens is not None else None,
                   duration=duration.to(dev()) if torch.is_tensor(duration) else duration)
    _, got = eager_and_graphed(pkg, model, {}, call_kw, y0, steps, c['cfg'], null)
    want = ode_ref.e2tts_sample(sd, O.TransformerCfg(**SMALL), cond, O.list_str_to_tensor(text) if text else None, duration=duration,
                                y0=y0, steps=steps, cfg_strength=c['cfg'], lens=lens, odeint_kwargs=dict(method=c['method']),
                                null_sd=null_sd)
    assert got.shape == want.shape
    e = rel_l2(got.cpu(), want)
    print(f'{name}: graphed sampler vs oracle rel-L2 {e:.4g}')
    assert e < 5e-2


def test_sampler_with_duration_predictor(pkg):
    torch.manual_seed(90)
    random.seed(90)
    model = pkg.E2TTS(transformer=dict(dropout=0., max_seq_len=256, **SMALL), use_vocos=False,
                      duration_predictor=dict(transformer=dict(dropout=0., max_seq_len=256, **SMALL))).to(dev()).eval()
    cond = torch.randn(2, 30, 100, device=dev())
    y0 = torch.randn(2, 256, 100)
    with torch.no_grad():
        cond_, _, _, duration = model._sample_inputs(cond, ['Hello', 'Good day to you'], None, None, 4096)
    md = int(duration.max())
    print(f'predicted durations {duration.tolist()}')
    eager_and_graphed(pkg, model, {}, dict(cond=cond, text=['Hello', 'Good day to you']), y0[:, :md], 4, 1.0, buckets=(64, 256))


def test_replays_repeat_and_buckets_do_not_leak(pkg):
    model, _ = small_model(pkg, 60, **SMALL)
    sampler = pkg.GraphedSampler(model, 2, (64, 128), steps=4)
    torch.manual_seed(5)
    cond, text = torch.randn(2, 24, 100, device=dev()), ['Hello', 'Goodbye']
    y_small, y_large = torch.randn(2, 50, 100, device=dev()), torch.randn(2, 120, 100, device=dev())
    outs = []
    for y0, d in ((y_small, 50), (y_small, 50), (y_large, 120), (y_small, 50)):
        with pkg.inject_randomness(y0=y0):
            outs.append(sampler(cond, text=text, duration=d, return_raw_output=True))
    torch.cuda.synchronize()
    assert outs[0].shape == (2, 50, 100) and outs[2].shape == (2, 120, 100)
    assert torch.equal(outs[0], outs[1])     # the same seed twice: the same bits
    assert torch.equal(outs[0], outs[3])     # after a call in the larger bucket: the same bits as before it
    torch.manual_seed(7)
    a = sampler(cond, text=text, duration=50, return_raw_output=True)
    torch.manual_seed(7)
    b = sampler(cond, text=text, duration=50, return_raw_output=True)
    assert torch.equal(a, b)                 # y0 from torch's generator: the same seed, the same output


POOL_SLACK = 0.25   # the smaller buckets' static inputs and kept outputs, and allocator rounding: at most 25 % of the largest bucket alone


def test_buckets_share_one_pool(pkg):
    model, _ = model_of(pkg, 21, max_seq_len=1024, dim=256, depth=2, heads=4)

    def reserved_by(buckets):
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        r0 = torch.cuda.memory_reserved()
        s = pkg.GraphedSampler(model, 4, buckets, steps=3)
        torch.cuda.synchronize()
        r = torch.cuda.memory_reserved() - r0
        del s
        return r

    reserved_by((1024,))                     # the model's own lazily built state (weight pack, rotary tables) comes first
    alone = reserved_by((1024,))
    shared = reserved_by((256, 512, 1024))
    print(f'reserved: largest bucket alone {alone / 2**20:.1f} MiB, three buckets {shared / 2**20:.1f} MiB')
    assert shared <= alone * (1 + POOL_SLACK) + 8 * 2 ** 20


def test_load_state_dict_reaches_the_replays(pkg):
    model, _ = small_model(pkg, 60, **SMALL)
    _, new_sd = small_model(pkg, 61, **SMALL)
    sampler = pkg.GraphedSampler(model, 2, (64,), steps=4)
    torch.manual_seed(5)
    cond, text, y0 = torch.randn(2, 24, 100, device=dev()), ['Hello', 'Goodbye'], torch.randn(2, 64, 100, device=dev())
    with pkg.inject_randomness(y0=y0):
        before = sampler(cond, text=text, duration=64, return_raw_output=True)
        model.load_state_dict(new_sd)
        got = sampler(cond, text=text, duration=64, return_raw_output=True)
        want = model.sample(cond, text=text, duration=64, steps=4, return_raw_output=True)
    e, moved = rel_l2(got.cpu(), want.cpu()), rel_l2(before.cpu(), want.cpu())
    print(f'after load_state_dict: rel-L2 {e:.3g} to eager sample() (the old weights: {moved:.3g})')
    assert e < 2e-2 and moved > 10 * e
    model.to(torch.float32)                  # a .to() drops the weight pack: the next call captures again
    again = sampler(cond, text=text, duration=64, return_raw_output=True)
    assert again.shape == got.shape
