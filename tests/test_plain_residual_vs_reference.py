"""CPU: Transformer(num_residual_streams=1), the plain residual backbone (e2_tts.py:547, :607 with disable=True). The oracle with
one stream against what the original e2_tts.py computed with that setting (tests/golden/reference/residual1_*.pt,
oracle/make_reference_golden.py), the package's parameter layout against the original's, the stream counts that still raise, and the
C-ABI validation of the branch-norm and residual-convolution fields."""
import pytest

from model_checks import check_case, oracle_case, sample_vs_reference, state_dict_vs_reference
from oracle import reference_cases as RC
from residual_variants import RESIDUAL1_CASES, RESIDUAL1_SAMPLE

import e2_tts_pytorch_b200 as pkg


@pytest.mark.parametrize('name', list(RESIDUAL1_CASES))
def test_oracle_vs_reference(name):
    """loss, prediction and gradient samples within the bounds of tests/test_oracle_vs_reference.py"""
    c, g = RESIDUAL1_CASES[name], RC.load('residual1_' + name)
    sd, loss, pred = oracle_case(c, g)
    assert not any('.hyper_conns.' in k for k in sd)
    check_case(c, g, sd, loss, pred)
    if c.get('drop'):   # the text stream is skipped: its parameters get no gradient
        assert g['grads']['transformer.layers.0.1.2.to_q.weight'] is None


def test_sample_vs_reference():
    sample_vs_reference(RESIDUAL1_SAMPLE, RC.load('residual1_sample'))


@pytest.mark.parametrize('name', list(RESIDUAL1_CASES))
def test_state_dict_matches_reference(name):
    """keys and shapes of the original's model: no hyper_conns entries, so its checkpoints load"""
    state_dict_vs_reference(RESIDUAL1_CASES[name], RC.load('residual1_' + name))


def test_plain_residual_makes_no_randrange_draw():
    """the reference's disabled hyper-connections draw nothing from python's random (the 4-stream ones draw one index each)"""
    import random
    random.seed(7)
    before = random.getstate()
    t = pkg.Transformer(dim=128, depth=2, heads=2, num_residual_streams=1)
    assert random.getstate() == before
    assert all(isinstance(h, pkg.modules.Residual) for layer in t.hyper_conns for part in layer if part is not None
               for h in part if h is not None)
    assert sum(p.numel() for p in t.hyper_conns.parameters()) == 0


@pytest.mark.parametrize('streams', [2, 3, 8])
def test_other_stream_counts_raise(streams):
    with pytest.raises(NotImplementedError, match='supported values are 1 .* and 4'):
        pkg.Transformer(dim=128, depth=2, heads=2, num_residual_streams=streams)
    with pytest.raises(NotImplementedError, match='num_residual_streams'):
        pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2, num_residual_streams=streams), use_vocos=False)


def _call_fails(name, struct, match, **kw):
    a = pkg.lib.make_args(struct, **kw)
    with pytest.raises(RuntimeError, match=match):
        pkg.lib.call(name, a, None)


def test_cabi_branch_norm_and_residual_conv_validation_without_gpu():
    """the trailing branch-norm / residual fields are checked before the device is touched (placeholder pointers, never read)"""
    fn = 'b200_final_norm_args'
    base = dict(xres=256, y=256, dy=256, d_xres=256, B=2, N=40, D=128)
    for name in ('b200_final_norm_fwd', 'b200_final_norm_bwd'):
        # all-zero new fields: today's refusals (g required, D bound)
        _call_fails(name, fn, 'null pointer', **base, S=1, g_g=256)
        _call_fails(name, fn, 'multiple of 8', **dict(base, D=2048), S=1, g=256, g_g=256)
        # gains / d_res without the branch-norm mode
        _call_fails(name, fn, 'rows_per_batch > 0', **base, S=1, g=256, g_g=256, gains=256, d_gains=256)
        _call_fails(name, fn, 'rows_per_batch must be >= 0', **base, S=1, g=256, g_g=256, rows_per_batch=-1)
        # branch-norm mode: one stream, no registers, whole batches, a gain
        _call_fails(name, fn, 'S == 1 and R == 0', **base, S=4, g=256, g_g=256, rows_per_batch=40)
        _call_fails(name, fn, 'S == 1 and R == 0', **base, S=1, R=32, g=256, g_g=256, rows_per_batch=40)
        _call_fails(name, fn, 'multiple of rows_per_batch', **base, S=1, g=256, g_g=256, rows_per_batch=33)
        _call_fails(name, fn, 'needs gains or g', **base, S=1, g_g=256, d_gains=256, rows_per_batch=40)
        _call_fails(name, fn, 'multiple of 8', **dict(base, D=1032), S=1, g=256, g_g=256, rows_per_batch=40)
    _call_fails('b200_final_norm_bwd', fn, 'gains need d_gains', **base, S=1, gains=256, rows_per_batch=40)
    _call_fails('b200_final_norm_bwd', fn, 'gains need d_gains', **base, S=1, g=256, rows_per_batch=40)
    _call_fails('b200_final_norm_bwd', fn, 'rows_per_batch > 0', **base, S=1, g=256, g_g=256, d_res=256)
    # residual convolution
    cv = dict(x=256, weight=256, bias=256, B=1, Np=64, D=64, ksize=31)
    _call_fails('b200_dwconv_fwd', 'b200_dwconv_args', 'must not alias x', **cv, y=256, residual=1)
    _call_fails('b200_dwconv_fwd', 'b200_dwconv_args', 'residual must be 0 or 1', **cv, y=512, residual=2)
    _call_fails('b200_dwconv_bwd', 'b200_dwconv_args', 'residual must be 0 or 1', **cv, dy=256, dx=256, dweight=256, dbias=256, pre=256,
                residual=-1)
    _call_fails('b200_dwconv_bwd', 'b200_dwconv_args', 'pre-activation', **cv, dy=256, dx=256, dweight=256, dbias=256, residual=1)
    # the gate backward of a residual epilogue needs the residual
    with pytest.raises(RuntimeError, match='null resid'):
        pkg.lib.call('b200_rowgate_resid_bwd', 256, 256, None, 256, None, 256, 256, None, 1, 64, 64, None)
