"""CPU: DurationPredictor(hl_gauss_loss=dict(...), use_regression=False), the HL-Gauss classification head (e2_tts.py:966-967,
1035-1040, 1107, 1111; hl-gauss-pytorch, SURVEY A.6). The oracle configured with the same hl_gauss_loss against what the original
e2_tts.py computed (tests/golden/reference/hl_gauss_*.pt, tools/make_hl_gauss_golden.py): losses and gradient samples, predictions,
and E2TTS.sample driven by the predicted durations. The restatements of tests/hl_gauss_ref.py against the oracle's and the leaf's
regression head, a negative control, the parameter layout against the original's, the parsing of the keywords and their refusals,
and the C-ABI validation of b200_hl_gauss_fwd / _bwd."""
import copy

import pytest
import torch

import hl_gauss_ref as H
from hl_gauss_variants import HL_GAUSS_CASES, HL_GAUSS_SAMPLE
from model_checks import check_grads, grad_sd
from oracle import e2tts_oracle as O
from oracle import reference_cases as RC

import e2_tts_pytorch_b200 as pkg


def oracle_loss(c, sd, hl_gauss):
    """the oracle's training-mode loss on case `c` (inputs rebuilt from its seed, the prefix fractions the original drew)"""
    mel = RC.randn((c['mel'][0], c['mel'][1], 100), c['seed'] + 1000)
    torch.manual_seed(c['seed'])
    rand_frac = mel.new_zeros(mel.shape[0]).uniform_(0, 1)   # the draw of e2_tts.py:1082 under the same seed
    text = O.list_str_to_tensor(c['text']) if c['text'] else None
    return H.duration_forward(sd, O.TransformerCfg(cond_on_time=False, **c['tkw']), mel, text, lens=torch.tensor(c['lens']),
                              rand_frac=rand_frac, hl_gauss=hl_gauss)


def oracle_predict(c, sd, hl_gauss):
    mel = RC.randn((c['mel'][0], c['mel'][1], 100), c['seed'] + 1000)
    text = O.list_str_to_tensor(c['text']) if c['text'] else None
    with torch.no_grad():
        return H.duration_forward(sd, O.TransformerCfg(cond_on_time=False, **c['tkw']), mel, text, lens=torch.tensor(c['lens']),
                                  return_loss=False, hl_gauss=hl_gauss)


def case_sd(c):
    return RC.state_dict(c['cls'], c['seed'], c['tkw'], **c['kw'])


@pytest.mark.parametrize('name', list(HL_GAUSS_CASES))
def test_oracle_vs_reference(name):
    """loss within 1e-5 and the gradient samples within the DurationPredictor bound of tests/test_oracle_vs_reference.py"""
    c, rec = HL_GAUSS_CASES[name], RC.load('hl_gauss_' + name)
    sd = grad_sd(case_sd(c))
    loss = oracle_loss(c, sd, c['kw']['hl_gauss_loss'])
    loss.backward()
    assert abs(float(loss.detach()) - rec['loss']) <= 1e-5 * abs(rec['loss'])
    check_grads(sd, rec['grads'], 5e-4, 1e-6)
    assert rec['grads']['hl_gauss_layer.to_pred.0.weight'] is not None


def test_predictions_vs_reference():
    """return_loss=False: sum softmax * centres per item, within 1e-5 relative"""
    rec = RC.load('hl_gauss_predict')
    for name, c in HL_GAUSS_CASES.items():
        got = oracle_predict(c, case_sd(c), c['kw']['hl_gauss_loss'])
        assert torch.allclose(got, rec[name], rtol=1e-5, atol=0), name


def test_clamp_and_support_edges():
    """the cases reach the regimes they are named for: targets beyond max_value (clamped, or 2 sigma out unclamped)"""
    hl = HL_GAUSS_CASES['clamp_beyond_max']['kw']['hl_gauss_loss']
    assert max(HL_GAUSS_CASES['clamp_beyond_max']['lens']) > hl['max_value']
    p = H.hl_gauss_probs(torch.tensor([72., 40.]), hl)
    assert torch.equal(p[0], p[1])   # clamped onto max_value
    hl = HL_GAUSS_CASES['beyond_unclamped']['kw']['hl_gauss_loss']
    p = H.hl_gauss_probs(torch.tensor([72.]), hl)
    assert abs(float(p.sum()) - 1) < 1e-5 and float(p[0, -1]) == float(p.max())


def test_nan_far_outside_the_support():
    """the reference's z is 0 for a target >= 8 sigma outside an unclamped support: the loss is NaN, as the original's"""
    hl = dict(min_value=0., max_value=10., num_bins=10, sigma=1.)
    assert torch.isnan(H.hl_gauss_probs(torch.tensor([18.5]), hl)).all()
    assert not torch.isnan(H.hl_gauss_probs(torch.tensor([18.5]), dict(hl, clamp_to_range=True))).any()


def test_sample_durations_vs_reference():
    """E2TTS.sample without `duration`: the HL-Gauss duration predictor's predictions and, from their .long(), the sample"""
    s, rec = HL_GAUSS_SAMPLE, RC.load('hl_gauss_sample')
    dp = s['duration_predictor']
    sd = RC.state_dict('E2TTS', s['seed'], s['tkw'], duration_predictor=copy.deepcopy(dp))
    dsd = {k[len('duration_predictor.'):]: v for k, v in sd.items() if k.startswith('duration_predictor.')}
    cond = RC.randn((s['cond'][0], s['cond'][1], 100), s['seed'] + 1000)
    text = O.list_str_to_tensor(s['text'])
    lens = torch.maximum((text != -1).sum(-1), torch.full((cond.shape[0],), cond.shape[1]))   # e2_tts.py:1372-1373
    dtkw = {k: v for k, v in dp['transformer'].items() if k not in ('dropout', 'max_seq_len')}
    with torch.no_grad():
        pred = H.duration_forward(dsd, O.TransformerCfg(cond_on_time=False, **dtkw), cond, text, lens=lens, return_loss=False,
                                  hl_gauss=dp['hl_gauss_loss'])
        assert torch.allclose(pred, rec['pred'], rtol=1e-5, atol=0)
        assert torch.equal(pred.long(), rec['pred'].long())
        got = O.e2tts_sample(sd, O.TransformerCfg(**s['tkw']), cond, text, duration=pred.long(), y0=RC.randn(rec['shape'], 3000 + s['seed']),
                             steps=s['steps'], cfg_strength=s['cfg_strength'])
    assert tuple(got.shape) == rec['shape']
    assert RC.compact_rel_l2(got, rec['out']) < 1e-4


@pytest.mark.parametrize('name', list(HL_GAUSS_CASES))
def test_state_dict_matches_reference(name):
    """keys and shapes of the original's model: hl_gauss_layer.to_pred.0.weight [num_bins, dim] and its bias, no loss buffers"""
    c, rec = HL_GAUSS_CASES[name], RC.load('hl_gauss_' + name)
    m = pkg.DurationPredictor(transformer=dict(dropout=0., max_seq_len=128, **c['tkw']), **c['kw'])
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == rec['shapes']
    assert got['hl_gauss_layer.to_pred.0.weight'] == (c['kw']['hl_gauss_loss']['num_bins'], c['tkw']['dim'])


def test_sample_model_state_dict():
    s = HL_GAUSS_SAMPLE
    m = pkg.E2TTS(transformer=dict(dropout=0., max_seq_len=128, **s['tkw']), duration_predictor=copy.deepcopy(s['duration_predictor']),
                  use_vocos=False)
    assert m.state_dict()['duration_predictor.hl_gauss_layer.to_pred.0.weight'].shape == (48, 128)
    assert not m.duration_predictor.hl_gauss_layer.use_regression


def test_regression_oracle_misses_the_classification_record():
    """negative control: the regression head (Softplus + MSE) on the same seed's regression weights misses every record's loss, and
    the classification oracle with 1.5 x sigma misses it by more than ten times the 1e-5 the cases pass at (near-uniform logits of
    seeded weights: sigma moves the loss by 8e-4 relative or more)"""
    for name, c in HL_GAUSS_CASES.items():
        rec = RC.load('hl_gauss_' + name)
        with torch.no_grad():
            reg = oracle_loss(c, RC.state_dict(c['cls'], c['seed'], c['tkw']), None)
            hl = c['kw']['hl_gauss_loss']
            sigma = hl.get('sigma') or (hl['max_value'] - hl['min_value']) / hl['num_bins'] * 2.
            wrong = oracle_loss(c, case_sd(c), dict(hl, sigma=1.5 * sigma))
        assert abs(float(reg) - rec['loss']) > 1e-2 * abs(rec['loss']), name
        assert abs(float(wrong) - rec['loss']) > 1e-4 * abs(rec['loss']), name


def test_restatements_keep_the_regression_head():
    """hl_gauss_ref.duration_forward without hl_gauss is the oracle's DurationPredictor bit for bit (loss, prediction, gradients), and
    its HLGaussLayer in regression mode has the restated leaf's parameters and draws, so the original runs as before with it bound"""
    from oracle.ref_leaves.hl_gauss_pytorch import HLGaussLayer as LeafLayer
    c = HL_GAUSS_CASES['explicit_sigma']
    mel = RC.randn((3, 72, 100), 7)
    text, lens, frac = O.list_str_to_tensor(c['text']), torch.tensor(c['lens']), torch.tensor([0.3, 0.6, 0.9])
    cfg = O.TransformerCfg(cond_on_time=False, **c['tkw'])
    sd_a, sd_b = grad_sd(RC.state_dict(c['cls'], c['seed'], c['tkw'])), grad_sd(RC.state_dict(c['cls'], c['seed'], c['tkw']))
    a = O.duration_forward(sd_a, cfg, mel, text, lens=lens, rand_frac=frac)
    b = H.duration_forward(sd_b, cfg, mel, text, lens=lens, rand_frac=frac)
    assert torch.equal(a, b)
    a.backward()
    b.backward()
    assert all((sd_a[k].grad is None and sd_b[k].grad is None) or torch.equal(sd_a[k].grad, sd_b[k].grad) for k in sd_a)
    with torch.no_grad():
        assert torch.equal(O.duration_forward(sd_a, cfg, mel, text, lens=lens, return_loss=False),
                           H.duration_forward(sd_b, cfg, mel, text, lens=lens, return_loss=False))
    torch.manual_seed(3)
    leaf = LeafLayer(64, use_regression=True, regress_activation=torch.nn.Softplus())
    torch.manual_seed(3)
    mine = H.HLGaussLayer(64, use_regression=True, regress_activation=torch.nn.Softplus())
    sa, sb = leaf.state_dict(), mine.state_dict()
    assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)
    assert torch.equal(torch.rand(4), (torch.manual_seed(3), LeafLayer(64, use_regression=True), torch.rand(4))[2])
    x, t = torch.randn(5, 64), torch.rand(5) * 10
    assert torch.equal(leaf(x, t), mine(x, t)) and torch.equal(leaf(x), mine(x))


def test_restated_loss_is_the_oracle_head():
    """hl_gauss_ref.HLGaussLoss (run inside the original) and the functional oracle head give the same loss and prediction"""
    hl = dict(min_value=0., max_value=40., num_bins=16, clamp_to_range=True)
    logits, target = torch.randn(4, 16), torch.tensor([3., 39.5, 55., 0.])
    loss = H.HLGaussLoss(**hl)
    assert torch.equal(loss(logits, target), torch.nn.functional.cross_entropy(logits, H.hl_gauss_probs(target, hl)))
    assert torch.equal(loss(logits), (logits.softmax(-1) * H.hl_gauss_centres(hl)).sum(-1))


def test_oracle_reads_the_head_from_state_dict_and_config():
    c = HL_GAUSS_CASES['explicit_sigma']
    sd = case_sd(c)
    with pytest.raises(KeyError):
        oracle_predict(c, sd, dict(c['kw']['hl_gauss_loss'], num_bins=33))   # the config's bins against the weight's rows
    del sd['hl_gauss_layer.to_pred.0.bias']
    with pytest.raises(KeyError):
        oracle_predict(c, sd, c['kw']['hl_gauss_loss'])


# ---------------------------------------------------------------------------------------------------------------------- parsing
TKW = dict(dim=128, depth=2, heads=2)


def test_hl_gauss_keywords_parse():
    hl = pkg.DurationPredictor(transformer=TKW, hl_gauss_loss=dict(min_value=0., max_value=100., num_bins=50),
                               use_regression=False).hl_gauss_layer
    assert not hl.use_regression and hl.spec.sigma == 4.0 and not hl.spec.clamp_to_range   # the default ratio 2 x bin size 2
    spec = pkg.ops.HLGaussSpec(min_value=-1, max_value=3, num_bins=8, sigma_to_bin_ratio=0.75, clamp_to_range=True)
    assert (spec.min_value, spec.max_value, spec.num_bins, spec.sigma, spec.clamp_to_range) == (-1., 3., 8, 0.375, True)
    assert pkg.ops.HLGaussSpec(0, 1, pkg.ops.HL_GAUSS_MAX_BINS, sigma=0.1).num_bins == 4096
    # hl_gauss_loss with use_regression=True: the regression head, unchanged
    m = pkg.DurationPredictor(transformer=TKW, hl_gauss_loss=dict(min_value=0., max_value=100., num_bins=50))
    plain = pkg.DurationPredictor(transformer=TKW)
    assert m.hl_gauss_layer.use_regression and isinstance(m.hl_gauss_layer.to_pred[1], torch.nn.Softplus)
    assert {k: v.shape for k, v in m.state_dict().items()} == {k: v.shape for k, v in plain.state_dict().items()}
    assert plain.hl_gauss_layer.use_regression and plain.hl_gauss_layer.spec is None


@pytest.mark.parametrize('hl,exc,match', [
    (dict(min_value=0., max_value=10., num_bins=1), ValueError, 'num_bins'),
    (dict(min_value=10., max_value=10., num_bins=8), ValueError, 'min_value'),
    (dict(min_value=11., max_value=10., num_bins=8), ValueError, 'min_value'),
    (dict(min_value=0., max_value=10., num_bins=8, sigma=0.), ValueError, 'sigma'),
    (dict(min_value=0., max_value=10., num_bins=8, sigma_to_bin_ratio=-1.), ValueError, 'sigma'),
    (dict(min_value=0., max_value=10., num_bins=8, temperature=2.), TypeError, 'temperature'),
    (dict(min_value=0., max_value=10.), TypeError, 'num_bins'),
])
def test_bad_hl_gauss_loss_raises(hl, exc, match):
    """refused in both modes, as the reference's HLGaussLoss(**hl_gauss_loss) is built in both"""
    for use_regression in (False, True):
        with pytest.raises(exc, match=match):
            pkg.DurationPredictor(transformer=TKW, hl_gauss_loss=hl, use_regression=use_regression)


def test_classification_without_loss_and_bin_cap_raise():
    with pytest.raises(ValueError, match='hl_gauss_loss'):
        pkg.DurationPredictor(transformer=TKW, use_regression=False)
    with pytest.raises(NotImplementedError, match='4096'):
        pkg.DurationPredictor(transformer=TKW, hl_gauss_loss=dict(min_value=0., max_value=1., num_bins=4097), use_regression=False)
    with pytest.raises(NotImplementedError, match='4096'):
        pkg.E2TTS(transformer=TKW, duration_predictor=dict(transformer=TKW, hl_gauss_loss=dict(min_value=0., max_value=1., num_bins=5000),
                                                           use_regression=False), use_vocos=False)
    # the regression head ignores num_bins: a large one is no reason to refuse it
    assert pkg.DurationPredictor(transformer=TKW, hl_gauss_loss=dict(min_value=0., max_value=1., num_bins=5000)).hl_gauss_layer.use_regression


# ---------------------------------------------------------------------------------------------------------------------- C ABI
def test_cabi_hl_gauss_validation_without_gpu():
    """b200_hl_gauss_fwd / _bwd refuse bad shapes, ranges and missing pointers before the device is touched (placeholder pointers,
    never read)"""
    ok = dict(logits=256, target=256, ce=256, loss=256, diff=256, ws_count=256, B=4, num_bins=32, min_value=0., max_value=10., sigma=1.)
    for bad, match in ((dict(B=0), 'batch'), (dict(B=65), 'batch'), (dict(num_bins=1), 'num_bins'), (dict(num_bins=4097), 'num_bins'),
                       (dict(min_value=10.), 'min_value'), (dict(max_value=float('inf')), 'min_value'), (dict(min_value=float('nan')), 'min_value'),
                       (dict(sigma=0.), 'sigma'), (dict(sigma=float('nan')), 'sigma'), (dict(clamp_to_range=2), 'clamp_to_range'),
                       (dict(logits=None), 'logits'), (dict(ws_count=None), 'ws_count'), (dict(diff=None), 'training'),
                       (dict(target=None), 'pred')):
        a = pkg.lib.make_args('b200_hl_gauss_args', **dict(ok, **bad))
        with pytest.raises(RuntimeError, match=match):
            pkg.lib.call('b200_hl_gauss_fwd', a, None)
    bwd = dict(diff=256, dloss=256, dlogits=256, B=4, num_bins=32, min_value=0., max_value=10., sigma=1.)
    for missing in ('diff', 'dloss', 'dlogits'):
        a = pkg.lib.make_args('b200_hl_gauss_args', **dict(bwd, **{missing: None}))
        with pytest.raises(RuntimeError, match='null pointer'):
            pkg.lib.call('b200_hl_gauss_bwd', a, None)
    a = pkg.lib.make_args('b200_hl_gauss_args', **dict(bwd, num_bins=5000))
    with pytest.raises(RuntimeError, match='num_bins'):
        pkg.lib.call('b200_hl_gauss_bwd', a, None)
