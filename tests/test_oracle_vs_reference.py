"""CPU: pins oracle/e2tts_oracle.py against what the original e2-tts-pytorch code (its own e2_tts.py, unmodified) computed on the
cases of oracle/reference_cases.py. The original's outputs are stored under tests/golden/reference/ (oracle/make_reference_golden.py);
weights, inputs and injected noise are rebuilt from seeds here. Gradients are compared on a fixed sample of each parameter's elements
plus its max |g| and norm."""
import numpy as np
import pytest
import torch

from oracle import e2tts_oracle as O
from model_checks import check_case, check_grads, grad_sd, oracle_case
from oracle import reference_cases as RC


def _forward_case(name):
    c, g = RC.FORWARD_CASES[name], RC.load('forward_' + name)
    sd, loss, pred = oracle_case(c, g)
    check_case(c, g, sd, loss, pred)
    return sd


@pytest.mark.parametrize('depth,lens', [(2, None), (4, [80, 51])])
def test_forward_backward_vs_reference(depth, lens):
    _forward_case('depth2' if depth == 2 else 'depth4_lens')


def test_melspec_vs_torchaudio():
    g = RC.load('melspec')
    assert (g['mel'] - O.melspec(g['wave'])).abs().max() < 1e-3


def test_text_dropped_branch_vs_reference():
    """cond_drop (e2_tts.py:1530-1534, :1263-1264): the text stream is skipped, its parameters receive no gradient."""
    _forward_case('text_dropped')


def test_variant_state_dicts_match_reference():
    """The non-default switches that are built (attn_fourier_embed_input, interpolated_text, concat_cond) keep the original's parameter
    names and shapes, so its checkpoints of those variants load."""
    import e2_tts_pytorch_b200 as pkg
    g = RC.load('variant_state_dict')
    b = pkg.E2TTS(**g['kw']).state_dict()
    a = g['shapes']
    assert set(a) == set(b), (sorted(set(a) - set(b))[:5], sorted(set(b) - set(a))[:5])
    for k in a:
        assert tuple(b[k].shape) == a[k], k


def test_concat_cond_vs_reference():
    """E2TTS(concat_cond=True) (e2_tts.py:1134, :1200-1201, :1263-1267): one Linear(2C -> dim) on cat(cond, x) instead of two summed
    projections."""
    sd = _forward_case('concat_cond')
    assert 'cond_proj_in.weight' not in sd and sd['proj_in.weight'].shape == (128, 200)


def test_interpolated_text_vs_reference():
    """E2TTS(interpolated_text=True) (e2_tts.py:1135, :1233; InterpolatedCharacterEmbed :414-482, interpolate_1d :237-244): ragged text
    lengths, ragged audio lengths, loss / prediction / every gradient incl. the embedding table and both abs_pos_mlp linears."""
    sd = _forward_case('interpolated_text')
    assert float(sd['embed_text.abs_pos_mlp.1.weight'].grad.abs().max()) > 0 and float(sd['embed_text.embed.weight'].grad.abs().max()) > 0


def test_attn_fourier_embed_input_vs_reference():
    """Transformer(attn_fourier_embed_input=True) (e2_tts.py:545-546, LinearFourierEmbed :368-386 applied at :909): loss, prediction and
    every gradient incl. `layers.{i}.0.4.linear.weight`."""
    sd = _forward_case('attn_fourier_embed_input')
    assert float(sd['transformer.layers.1.0.4.linear.weight'].grad.abs().max()) > 0


@pytest.mark.parametrize('steps,cfg_strength,duration', RC.SAMPLE_CASES)
def test_sample_vs_reference(steps, cfg_strength, duration):
    """E2TTS.sample (:1332-1466): midpoint grid, CFG with the APG orthogonal projection (:1303-1330, :113-124), the
    cond mask / duration logic (:1376-1405) — same y0 injected into the oracle."""
    g = RC.load('sample')
    c = next(c for c in g['cases'] if c['steps'] == steps)
    dur = torch.tensor(duration) if isinstance(duration, list) else duration
    with torch.no_grad():
        got = O.e2tts_sample(RC.state_dict('E2TTS', 31), O.TransformerCfg(**RC.KW), g['cond'], O.list_str_to_tensor(g['text']), duration=dur,
                             y0=RC.randn(c['shape'], 3000 + steps), steps=steps, cfg_strength=cfg_strength)
    assert tuple(got.shape) == c['shape']
    assert RC.compact_rel_l2(got, c['out']) < 1e-4


def test_duration_predictor_vs_reference():
    """DurationPredictor.forward (:1042-1113): random prefix mask, masked mean pool, softplus head, L1-on-frames loss."""
    g = RC.load('duration')
    sd = grad_sd(RC.state_dict('DurationPredictor', 41))
    mel = RC.randn((3, 72, 100), 1041)
    torch.manual_seed(5)
    rand_frac = mel.new_zeros(3).uniform_(0, 1)   # the draw of e2_tts.py:1082 under the same seed
    got = O.duration_forward(sd, O.TransformerCfg(cond_on_time=False, **RC.KW), mel, O.list_str_to_tensor(['abc', 'hello world', 'x']),
                             lens=torch.tensor([72, 50, 31]), rand_frac=rand_frac)
    assert abs(float(got) - g['loss']) <= 1e-4 * abs(g['loss'])
    got.backward()
    check_grads(sd, g['grads'], rel=5e-4, floor=1e-6)


def test_mask_helpers_bit_exact_vs_reference():
    """The product's host-side mask helpers (e2-tts-pytorch_b200/modules.py: lens_to_mask, mask_from_frac_lengths — SURVEY §8 row a14)
    against the original's (e2_tts.py:173-210), bit for bit on 200 seeded ragged cases (same torch RNG state -> same rand_like draw)."""
    import e2_tts_pytorch_b200 as pkg
    ref = RC.load('mask_helpers')
    g = torch.Generator().manual_seed(0)
    for case in range(200):
        b = int(torch.randint(1, 9, (1,), generator=g))
        n = int(torch.randint(8, 300, (1,), generator=g))
        lens = torch.randint(1, n + 1, (b,), generator=g)
        if case % 3 == 0:
            lens[int(torch.randint(0, b, (1,), generator=g))] = n
        frac = torch.rand(b, generator=g) * 0.3 + 0.7          # frac_lengths_mask = (0.7, 1.0), e2_tts.py:1133
        r = ref['cases'][case]
        torch.manual_seed(1000 + case)
        got = pkg.mask_from_frac_lengths(lens, frac, n)
        want = torch.from_numpy(np.unpackbits(r['span'].numpy(), axis=-1)[:, :n].astype(bool))
        assert got.dtype == torch.bool and tuple(got.shape) == r['shape'] and torch.equal(got, want), case
        want_n = torch.from_numpy(np.unpackbits(r['lens_n'].numpy(), axis=-1)[:, :n].astype(bool))
        assert torch.equal(pkg.lens_to_mask(lens, length=n), want_n), case
        auto = pkg.lens_to_mask(lens)
        assert auto.shape == r['lens_auto'] and torch.equal(auto, want_n[:, :auto.shape[1]]), case
    assert torch.equal(pkg.list_str_to_tensor(['Hello', 'Goodbye', 'héllo wörld']), ref['ids'])


def test_velocity_consistency_loss_vs_reference():
    """E2TTS.forward with a velocity_consistency_model (e2_tts.py:1556-1576, trainer hook trainer.py:259-268): total loss, breakdown and
    gradients of the online model against the oracle's restatement."""
    g = RC.load('velocity_consistency')
    s = RC.VELOCITY_SEED
    sd = grad_sd(RC.state_dict('E2TTS', s, velocity_consistency_weight=0.7))
    mel = RC.randn((2, 64, 100), 1000 + s)
    o = O.e2tts_forward(sd, O.TransformerCfg(**RC.KW), mel, O.list_str_to_tensor(['abc', 'some text']), lens=torch.tensor([64, 50]),
                        x0=RC.randn(mel.shape, 2000 + s), times=g['times'], span_mask=g['span_mask'], velocity_sd=RC.state_dict('E2TTS', s + 1),
                        velocity_consistency_weight=0.7, velocity_consistency_delta=1e-3)
    o['loss'].backward()
    assert abs(float(o['loss']) - g['loss']) <= 1e-5 * abs(g['loss'])
    assert abs(float(o['flow_loss']) - g['flow']) <= 1e-5 * abs(g['flow'])
    assert abs(float(o['velocity_loss']) - g['velocity']) <= 1e-5 * abs(g['velocity'])
    assert g['velocity'] > 0
    for k, r in g['grads'].items():
        if r is None:
            continue
        # fp32 summation order differs between the two autograd graphs (and with the host's thread count), and the velocity term's
        # finite difference divides by delta = 1e-3, amplifying fp32 rounding ~1000x: agreement relative to the parameter's own
        # gradient with an absolute floor of 1e-4 of the total gradient norm (as for the full-gradient comparison)
        got = sd[k].grad.detach().double().flatten()
        diff = (got[RC.sample_index(got.numel())] - r['values'].double()).norm()
        assert diff <= 6e-3 * r['norm'] + 1e-4 * g['total'], k
        assert abs(float(got.norm()) - r['norm']) <= 6e-3 * r['norm'] + 1e-4 * g['total'], k
