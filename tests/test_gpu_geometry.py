"""GPU: the model-shape knobs of Transformer (e2_tts.py:518-552) from the kernels up to the whole model.

Kernels: b200_hc_width_fwd / _bwd (unfused and fused depth -> width) and b200_hc_depth_fwd / _bwd at the model widths D = 192, 384,
640, 768 and 896. Their D / 8 16-byte chunks do not fill the 32 * VPT lane slots of the width kernels (VPT chunks per lane), so lanes
of the last pass stay idle — the widths tested elsewhere (128, 256, 512, 1024) fill every lane. Each case asserts, from the host rules
of hyper.cu restated in tests/hyper_conv_ref.py, the <VPT, prefetching> instantiation it runs, that lanes are idle, and whether the
persistent loop of the forward wraps. The bounds are those of tests/test_gpu_attention_hyper_kernels.py (check_hc_case). The final
norm, branch norm, depthwise convolution, GLU and gain-projection kernels are held at these geometries by their own modules' cases.

Whole models against the oracle within the bounds of tests/model_checks.py (loss 1e-2, prediction 3e-2, gradient cosine 0.99, after
the bf16 conditioning probe): depth 24 (loss and prediction) and depth 12 at d1024, d768 at N = 1024, every case of
tests/geometry_variants.py, num_registers=0 on both sides of the fused hyper-connection rule; then the serial and two-stream
schedules and GraphedTrainStep with text_depth < depth."""
import pytest
import torch

from conftest import rel_l2
from geometry_variants import GEOMETRY_CASES, GEOMETRY_SAMPLE
from hyper_conv_ref import S, check_hc_case, hc_fwd_launch
from kernel_checks import dev, pkg, sms  # noqa: F401
from model_checks import duration_vs_oracle, graphed_matches_eager, sample_vs_oracle, small_model, step_inputs, whole_model

pytestmark = pytest.mark.gpu


# ================================================================================================================ hyper-connections
# (name, T, D, rows_per_batch, norm mode, fused, d_beta given, zero tokens, isolation slice in batch elements,
#  expected (VPT, prefetching) of the width kernels)
HC_GEOMETRY_CASES = [
    ('d192-t99-m2', 99, 192, 33, 2, False, True, (), None, (1, True)),
    ('d192-t4224-fused-wrap', 4224, 192, 1056, 2, True, True, (), (1, 3), (1, True)),
    ('d384-t7-m0', 7, 384, 7, 0, False, True, (), None, (2, True)),
    ('d384-t4224-m1-fused-wrap', 4224, 384, 1056, 1, True, True, ((11, (0, 3)),), None, (2, True)),
    ('d640-t99-m2', 99, 640, 33, 2, False, True, ((5, (2,)),), None, (4, False)),
    ('d640-t64-fused-m0', 64, 640, 32, 0, True, True, (), None, (4, False)),
    ('d768-t99-m1', 99, 768, 33, 1, False, False, (), None, (4, False)),
    ('d768-t16896-fused-wrap', 16896, 768, 1056, 2, True, True, (), (3, 5), (4, False)),
    ('d896-t16-fused-m1', 16, 896, 16, 1, True, True, (), None, (4, False)),
    ('d896-t9000-m2-wrap', 9000, 896, 1125, 2, False, True, (), (2, 4), (4, False)),
]


@pytest.mark.parametrize('name,T,D,rpb,mode,fused,use_dbeta,zeros,iso,inst', HC_GEOMETRY_CASES, ids=[c[0] for c in HC_GEOMETRY_CASES])
def test_hyper_connection_kernels_idle_lanes(pkg, name, T, D, rpb, mode, fused, use_dbeta, zeros, iso, inst):
    pf, vpt, fwd_warps = hc_fwd_launch(T, D)
    assert (vpt, pf) == inst, f'{name}: runs hc_width_*<{vpt}, {pf}>'
    assert D // 8 < 32 * vpt                                  # the last pass of the lanes leaves some of them idle
    assert fused == pkg.ops.hc_can_fuse(T, S)                 # fused exactly where the model fuses: T S a multiple of 64
    assert ('wrap' in name) == (fwd_warps < T)                # the persistent forward loop makes a second pass
    check_hc_case(pkg, name, T, D, rpb, mode, fused, use_dbeta, zeros, iso)


def test_hyper_geometry_cases_reach_every_idle_instantiation():
    """every width-kernel instantiation with idle lanes: (VPT 1 | 2, prefetching) and (4, not), each unfused and fused"""
    reached = {(c[9], c[5]) for c in HC_GEOMETRY_CASES}
    assert reached == {((v, v < 4), f) for v in (1, 2, 4) for f in (False, True)}


# ================================================================================================================ whole models
def test_e2tts_depth24_d1024_vs_oracle(pkg):
    """the depth-24 d1024 models' geometry (16 heads of 64), B = 2 ragged at N = 224: twelve skip levels, v_first carried through 24
    layers, 96 gain segments of the batched conditioning projection. Loss and prediction only, with the hyper-connections' dynamic
    scales at the reference's init 0.01 (bf16-stage oracle probe 1.19e-2; at 0.05 it reads 1.37e-2). The gradients of 24 layers are
    ill-conditioned for any bf16 path: the fp32 oracle with only its stage outputs rounded to bf16 (straight-through) moves its own
    gradients to cosine 0.981 (layer 6 audio attention dynamic_alpha_fn) and flips the sign of a scalar dynamic_alpha_scale, where the
    kernels reach 0.986. test_e2tts_depth12_d1024_vs_oracle holds the gradients at this width, at the depth where that probe stays
    above 0.99 (0.995 at depth 12, 0.991 at depth 16)."""
    r = whole_model(pkg, dict(dim=1024, depth=24, heads=16), B=2, N=224, lens=[224, 170], seed=110, dyn_scale=0.01, grads=False)
    print(f'depth 24 d1024: probe {r["probe"]:.4g}')


def test_e2tts_depth12_d1024_vs_oracle(pkg):
    """d1024 / 16 heads at depth 12 (six skip levels, 48 gain segments), B = 2 ragged at N = 224: loss, prediction and every gradient"""
    r = whole_model(pkg, dict(dim=1024, depth=12, heads=16), B=2, N=224, lens=[224, 170], seed=110, dyn_scale=0.01)
    print(f'depth 12 d1024: probe {r["probe"]:.4g}, worst gradient cosine {r["worst_cos"]}')


def test_e2tts_d768_n1024_vs_oracle(pkg):
    """d768 (12 heads; text 384): the hyper-connection, norm and convolution kernels at VPT 4 / 2 with idle lanes, GEMM N tails"""
    r = whole_model(pkg, dict(dim=768, depth=4, heads=12), B=2, N=1024, lens=[1024, 700], seed=111)
    print(f'd768 N1024: probe {r["probe"]:.4g}, worst gradient cosine {r["worst_cos"]}')


E2TTS_CASES = [n for n, c in GEOMETRY_CASES.items() if c['cls'] == 'E2TTS']


@pytest.mark.parametrize('name', E2TTS_CASES)
def test_e2tts_geometry_cases_vs_oracle(pkg, name):
    """the reference-pinned cases of tests/geometry_variants.py on the GPU, at their batch, frames and lengths"""
    c = GEOMETRY_CASES[name]
    r = whole_model(pkg, c['tkw'], B=c['mel'][0], N=c['mel'][1], lens=c['lens'], seed=120 + E2TTS_CASES.index(name),
                    drop_text_cond=c['drop'])
    print(f'{name}: probe {r["probe"]:.4g}, worst gradient cosine {r["worst_cos"]}')


@pytest.mark.parametrize('N', [200, 201])
def test_e2tts_no_registers_vs_oracle(pkg, N):
    """num_registers=0: N' = N. B N' = 400 makes T S a multiple of 64 (the fused depth -> width path); 402 does not (unfused)"""
    B = 2
    assert pkg.ops.hc_can_fuse(B * N, S) == (N == 200)
    r = whole_model(pkg, dict(dim=256, depth=4, heads=4, num_registers=0), B=B, N=N, lens=[N, N - 63], seed=130 + N)
    print(f'no registers N{N}: probe {r["probe"]:.4g}, worst gradient cosine {r["worst_cos"]}')


def test_duration_predictor_geometry_vs_oracle(pkg):
    """DurationPredictor with text_depth < depth and dim_text != dim // 2 (the reference-pinned 'duration' case's geometry)"""
    duration_vs_oracle(pkg, 140, GEOMETRY_CASES['duration']['tkw'])


def test_sample_ragged_duration_vs_oracle(pkg):
    """E2TTS.sample with a per-element duration and ragged prompt lengths, at the sample case's geometry (text_depth 2 of 4, 8
    registers, kernel 5)"""
    s = GEOMETRY_SAMPLE
    out = sample_vs_oracle(pkg, 141, s['tkw'], cond=s['cond'], text=s['text'], duration=torch.tensor(s['duration']),
                           lens=torch.tensor(s['lens']), steps=s['steps'], cfg_strength=s['cfg_strength'])
    assert out.shape == (2, max(s['duration']), 100)


TEXT_DEPTH = dict(dim=128, depth=6, heads=2, text_depth=3, dim_text=128, num_registers=16)


def _step(pkg, B, N, seed):
    torch.manual_seed(seed)
    return step_inputs(pkg, B, N, span=(N // 5, N - N // 6))


def test_text_depth_schedules_agree_without_dropout(pkg, monkeypatch):
    """text_depth < depth: the two-stream schedule forks no text block past text_depth. At p = 0 the serial and the two-stream
    schedule give a bit-identical prediction (the gradients are held to the run-to-run scatter, as in
    tests/test_gpu_dropout_step.py)"""
    model, _ = small_model(pkg, 150, **TEXT_DEPTH)
    model.train()
    B, N = 2, 96
    mel, text, rnd = _step(pkg, B, N, 151)
    lens = torch.tensor([96, 70], device=dev())

    def run():
        model.zero_grad(set_to_none=True)
        with pkg.inject_randomness(**rnd):
            out = model(mel, text=text, lens=lens)
        out.loss.backward()
        torch.cuda.synchronize()
        return float(out.loss), out.pred_flow.detach().clone(), {k: p.grad.detach().clone() for k, p in model.named_parameters()
                                                                 if p.grad is not None}

    monkeypatch.setattr(pkg.modules, 'TWO_STREAM', False)
    s1 = run()
    monkeypatch.setattr(pkg.modules, 'TWO_STREAM', True)
    t = run()
    assert torch.equal(s1[1], t[1]), 'the prediction differs between the schedules'
    assert set(s1[2]) == set(t[2])
    assert not any(k.startswith('transformer.layers.3.1.') for k in t[2])     # no text sub-blocks past text_depth
    assert abs(t[0] - s1[0]) <= 1e-6 * abs(s1[0])
    for k in s1[2]:
        assert rel_l2(t[2][k].cpu(), s1[2][k].cpu()) <= 4e-3, k


def test_graphed_step_matches_eager_text_depth(pkg):
    """GraphedTrainStep replays the eager step's gradients with text_depth < depth"""
    model, _ = small_model(pkg, 152, **TEXT_DEPTH)
    graphed_matches_eager(pkg, model, *_step(pkg, 2, 96, 153))
