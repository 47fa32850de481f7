"""CPU: the x-transformers `ff_kwargs` of Transformer (e2_tts.py:552) — SwiGLU, ReLU^2 GLU, the GLU multiplicative bias and the output
Linear without bias. The oracle with the same ff_kwargs against what the original e2_tts.py computed on those settings
(tests/golden/reference/ff_kwargs_*.pt, oracle/make_reference_golden.py), a negative control per switch family (ff_kwargs, attn_kwargs,
text geometry), the package's parameter layout against the original's, the parsing of the keywords (precedence, explicit defaults,
refusals), and the C-ABI validation of the GLU activation fields."""
import pytest
import torch

from attn_variants import ATTN_KWARGS_CASES
from ff_variants import FF_KWARGS_CASES, XTFeedForward
from headdim_variants import HEADDIM_CASES
from model_checks import check_case, oracle_case, state_dict_vs_reference
from oracle import reference_cases as RC
from oracle.ref_leaves.x_transformers.x_transformers import FeedForward as LeafFeedForward

import e2_tts_pytorch_b200 as pkg

GLU_GELU, GLU_SILU, GLU_RELU2 = pkg.ops.GLU_GELU, pkg.ops.GLU_SILU, pkg.ops.GLU_RELU2


@pytest.mark.parametrize('name', list(FF_KWARGS_CASES))
def test_oracle_vs_reference(name):
    """loss, prediction and gradient samples (mult_bias included) within the bounds of tests/test_oracle_vs_reference.py"""
    c, g = FF_KWARGS_CASES[name], RC.load('ff_kwargs_' + name)
    check_case(c, g, *oracle_case(c, g))
    if c['tkw']['ff_kwargs'].get('glu_mult_bias'):
        assert any(k.endswith('.ff.0.mult_bias') and v is not None for k, v in g['grads'].items())


# one stored case per switch family, by record name, with its whole Transformer kwargs, and the least the oracle without the switch
# misses its prediction by (rel-L2; the cases pass at 1e-4)
SEES = {
    'ff_kwargs_swish': (FF_KWARGS_CASES['swish'], 1e-2),
    'attn_kwargs_clamp30': (ATTN_KWARGS_CASES['clamp30'], 1e-2),
    # text geometry 1 x 128, as wide as the audio's 2 x 64, so the default text geometry runs on the same weights; the text stream
    # reaches the prediction through the cross-conditions only, and 2 x 64 moves it by 8.7e-3
    'headdim_mixed_a64_t128': (HEADDIM_CASES['mixed_a64_t128'], 5e-3),
}


def test_oracle_sees_the_variant():
    """the stored outputs tell the variants apart, one switch family at a time: the oracle configured with the defaults of everything
    but the audio geometry, on the case's own weights plus the default model's for what the case lacks (clamp30's head gates: its clamp
    value alone moves the prediction by ~3e-6), misses the case's prediction, so a test that built the model with a switch and the
    oracle without it fails"""
    for record, (c, bound) in SEES.items():
        g = RC.load(record)
        default = {k: v for k, v in c['tkw'].items() if k in ('dim', 'depth', 'heads', 'dim_head')}
        sd = RC.state_dict(c['cls'], c['seed'], c['tkw'])
        for k, v in RC.state_dict(c['cls'], c['seed'], default).items():
            sd.setdefault(k, v)
        _, _, pred = oracle_case(dict(c, tkw=default), g, sd=sd)
        e = RC.compact_rel_l2(pred, g['pred'])
        print(f'{record}: the default config misses by {e:.3g}')
        assert e > bound, record


@pytest.mark.parametrize('name', list(FF_KWARGS_CASES))
def test_state_dict_matches_reference(name):
    """keys and shapes of the original's model with the same ff_kwargs (ff.0.mult_bias present, ff.2.bias absent where asked)"""
    c = FF_KWARGS_CASES[name]
    got = state_dict_vs_reference(c, RC.load('ff_kwargs_' + name))
    kw = c['tkw']['ff_kwargs']
    n_ff = sum(k.endswith('.ff.0.proj.weight') for k in got)
    assert n_ff == 2 * c['tkw']['depth']   # audio and text feed-forward of every layer
    assert sum(k.endswith('.ff.0.mult_bias') for k in got) == (n_ff if kw.get('glu_mult_bias') else 0)
    assert sum(k.endswith('.ff.2.bias') for k in got) == (0 if kw.get('no_bias') else n_ff)
    assert sum(k.endswith('.ff.0.proj.bias') for k in got) == n_ff   # x-transformers' GLU keeps its bias under no_bias


def test_restated_feedforward_default_matches_leaf():
    """XTFeedForward without keywords has the leaf's parameters and draws the same random numbers, so every existing golden holds"""
    torch.manual_seed(3)
    a = LeafFeedForward(dim=64, glu=True, mult=4, dropout=0.)
    torch.manual_seed(3)
    b = XTFeedForward(dim=64, glu=True, mult=4, dropout=0.)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    assert all(torch.equal(sa[k], sb[k]) for k in sa)
    assert torch.equal(torch.rand(4), (torch.manual_seed(3), LeafFeedForward(dim=64, glu=True), torch.rand(4))[2])


@pytest.mark.parametrize('ff_kwargs,act,mult,bias', [
    (dict(), GLU_GELU, False, True),
    (dict(swish=True), GLU_SILU, False, True),
    (dict(relu_squared=True), GLU_RELU2, False, True),
    (dict(relu_squared=True, swish=True), GLU_RELU2, False, True),   # x-transformers checks relu_squared before swish
    (dict(swish=False, relu_squared=False), GLU_GELU, False, True),
    (dict(glu_mult_bias=True, no_bias=True), GLU_GELU, True, False),
    (dict(swish=True, post_act_ln=False, solu=False, custom_activation=None, sublayer_dropout=0., dim_out=None), GLU_SILU, False, True),
])
def test_ff_kwargs_parse(ff_kwargs, act, mult, bias):
    """a missing key takes x-transformers' default; the text feed-forward takes the same kwargs"""
    t = pkg.Transformer(dim=128, depth=2, heads=2, ff_kwargs=ff_kwargs)
    for ff in (t.layers[0][0][7], t.layers[1][1][4]):
        assert ff.act == act
        assert (ff.ff[0].mult_bias is not None) == mult
        assert (ff.ff[2].bias is not None) == bias
        assert ff.ff[0].proj.bias is not None
        if mult:
            assert torch.equal(ff.ff[0].mult_bias.detach(), torch.ones(ff.ff[2].weight.shape[1]))


def test_zero_init_output():
    t = pkg.Transformer(dim=128, depth=2, heads=2, ff_kwargs=dict(zero_init_output=True))
    t_nb = pkg.Transformer(dim=128, depth=2, heads=2, ff_kwargs=dict(zero_init_output=True, no_bias=True))
    for ff in (t.layers[0][0][7], t.layers[1][1][4], t_nb.layers[0][0][7]):
        assert not ff.ff[2].weight.detach().any()
        assert ff.ff[2].bias is None or not ff.ff[2].bias.detach().any()
        assert ff.ff[0].proj.weight.detach().any()


def test_duration_predictor_inherits_ff_kwargs():
    m = pkg.DurationPredictor(transformer=dict(dim=128, depth=2, heads=2, ff_kwargs=dict(relu_squared=True, no_bias=True)))
    ff = m.transformer.layers[0][0][7]
    assert ff.act == GLU_RELU2 and ff.ff[2].bias is None


def test_unsupported_ff_kwargs_raise():
    for key, value in (('post_act_ln', True), ('solu', True), ('custom_activation', torch.nn.ReLU()), ('sublayer_dropout', 0.1),
                       ('dim_out', 64), ('laser', True)):
        with pytest.raises(NotImplementedError, match=f"ff_kwargs\\['{key}'\\].*e2_tts.py:552"):
            pkg.Transformer(dim=128, depth=2, heads=2, ff_kwargs={key: value, 'swish': True})
    for key in ('dim', 'mult', 'glu', 'dropout'):   # the reference passes these itself: its call raises TypeError as well
        with pytest.raises(TypeError, match=key):
            pkg.Transformer(dim=128, depth=2, heads=2, ff_kwargs={key: 1})
    with pytest.raises(NotImplementedError, match='post_act_ln'):
        pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2, ff_kwargs=dict(post_act_ln=True)), use_vocos=False)


def test_cabi_glu_validation_without_gpu():
    """the GLU activation code, glu_mult and b200_glu_bwd's arguments are checked before the device is touched (placeholder pointers,
    never read)"""
    base = dict(A=256, lda=64, B=256, ldb=64, M=128, N=256, K=64, D=256, ldd=128)
    for code in (-1, 4, 7):
        a = pkg.lib.make_args('b200_gemm_args', **base, geglu=code)
        with pytest.raises(RuntimeError, match='activation code'):
            pkg.lib.call('b200_gemm', a, None)
    a = pkg.lib.make_args('b200_gemm_args', **base, glu_mult=256)
    with pytest.raises(RuntimeError, match='glu_mult'):
        pkg.lib.call('b200_gemm', a, None)
    ptrs = dict(dh=256, ug=256, dug=256)
    for missing in ptrs:
        a = pkg.lib.make_args('b200_glu_bwd_args', **{k: v for k, v in ptrs.items() if k != missing}, T=8, inner=64, act=1)
        with pytest.raises(RuntimeError, match='null pointer'):
            pkg.lib.call('b200_glu_bwd', a, None)
    for act in (0, 4, -1):
        a = pkg.lib.make_args('b200_glu_bwd_args', **ptrs, T=8, inner=64, act=act)
        with pytest.raises(RuntimeError, match='activation code'):
            pkg.lib.call('b200_glu_bwd', a, None)
    a = pkg.lib.make_args('b200_glu_bwd_args', **ptrs, T=8, inner=96, act=2)
    with pytest.raises(RuntimeError, match='multiple of 64'):
        pkg.lib.call('b200_glu_bwd', a, None)
    a = pkg.lib.make_args('b200_glu_bwd_args', **ptrs, d_mult=256, T=8, inner=64, act=3)
    with pytest.raises(RuntimeError, match='d_mult needs mult'):
        pkg.lib.call('b200_glu_bwd', a, None)
