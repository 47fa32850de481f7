"""CPU: the Transformer(checkpoint_activations) switch — its default, how it reaches the model through the E2TTS and DurationPredictor
transformer dicts, that it adds no state and draws no randomness at construction — and the ops.Segment autograd node on host tensors."""
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


TKW = dict(dim=128, depth=2, heads=2, max_seq_len=512)


def test_switch_defaults_off(pkg):
    assert pkg.Transformer(**TKW).checkpoint_activations is False
    assert pkg.E2TTS(transformer=TKW, use_vocos=False).transformer.checkpoint_activations is False
    assert pkg.DurationPredictor(transformer=TKW).transformer.checkpoint_activations is False


def test_switch_passes_through_the_transformer_dicts(pkg):
    tkw = dict(TKW, checkpoint_activations=True)
    assert pkg.Transformer(**tkw).checkpoint_activations is True
    assert pkg.E2TTS(transformer=tkw, use_vocos=False).transformer.checkpoint_activations is True
    assert pkg.DurationPredictor(transformer=tkw).transformer.checkpoint_activations is True
    m = pkg.E2TTS(transformer=TKW, use_vocos=False)
    m.transformer.checkpoint_activations = True   # a plain attribute, read by every forward
    assert m.transformer.checkpoint_activations


@pytest.mark.parametrize('cls', ['E2TTS', 'DurationPredictor'])
def test_state_dict_unchanged(pkg, cls):
    def build(on):
        tkw = dict(TKW, checkpoint_activations=on)
        return pkg.E2TTS(transformer=tkw, use_vocos=False) if cls == 'E2TTS' else pkg.DurationPredictor(transformer=tkw)
    off, on = build(False).state_dict(), build(True).state_dict()
    assert list(off) == list(on)
    assert all(off[k].shape == on[k].shape and off[k].dtype == on[k].dtype for k in off)


def test_reference_checkpoint_loads_strictly(pkg):
    g = torch.load(os.path.join(ROOT, 'tests', 'golden', 'e2tts_d128_L2.pt'), weights_only=False)
    model = pkg.E2TTS(transformer=dict(dropout=0., max_seq_len=g['max_seq_len'], checkpoint_activations=True, **g['transformer']),
                      use_vocos=False)
    model.load_state_dict(g['state_dict'], strict=True)
    assert model.transformer.checkpoint_activations


def test_construction_draws_no_extra_randomness(pkg):
    def draws(on):
        random.seed(7)
        torch.manual_seed(7)
        pkg.E2TTS(transformer=dict(TKW, checkpoint_activations=on), use_vocos=False)
        return random.random(), torch.rand(4)
    (py_off, t_off), (py_on, t_on) = draws(False), draws(True)
    assert py_off == py_on
    assert torch.equal(t_off, t_on)


# ------------------------------------------------------------------------------------------------ the autograd node, on host tensors
def _run(w):
    def run(x, v, g):
        h = torch.tanh(x * w)
        out = h * g + x
        return (out, h.sum(-1)) if v is None else (out + v,)
    return run


def test_segment_matches_the_plain_graph(pkg):
    ops = pkg.ops
    torch.manual_seed(0)
    x0, g0, v0 = torch.randn(5, 3, 8), torch.randn(8), torch.randn(5, 3, 8)
    w = torch.randn(8, requires_grad=True)
    grads = []
    for seg in (False, True):
        w.grad = None
        x, g, v = (t.clone().requires_grad_() for t in (x0, g0, v0))
        run = _run(w)
        out1, hs = ops.Segment.apply(run, x, None, g) if seg else run(x, None, g)
        (out2,) = ops.Segment.apply(run, out1, v, g) if seg else run(out1, v, g)
        if seg:
            assert out1.grad_fn is not None and type(out1.grad_fn).__name__ == 'SegmentBackward'
        (out2.square().sum() + hs.sum()).backward()
        grads.append((out2.detach(), x.grad, g.grad, v.grad, w.grad.clone()))
    for a, b in zip(*grads):
        torch.testing.assert_close(a, b, rtol=0, atol=0)


def test_segment_output_without_gradient(pkg):
    """an output nobody reads (the last text block's values) gets no gradient: the recompute backpropagates the others only"""
    ops = pkg.ops
    x = torch.randn(4, 2, 8, requires_grad=True)
    g = torch.randn(8, requires_grad=True)
    w = torch.randn(8, requires_grad=True)
    out, _ = ops.Segment.apply(_run(w), x, None, g)
    out.sum().backward()
    want = torch.autograd.grad(_run(w)(x, None, g)[0].sum(), (x, g, w))
    torch.testing.assert_close(x.grad, want[0], rtol=0, atol=0)
    torch.testing.assert_close(g.grad, want[1], rtol=0, atol=0)
    torch.testing.assert_close(w.grad, want[2], rtol=0, atol=0)


def test_segment_inputs_without_gradient(pkg):
    """inputs that take no gradient (the packed weight handles) and None inputs get None back"""
    ops = pkg.ops
    x = torch.randn(4, 2, 8, requires_grad=True)
    packed = torch.randn(8)
    (out,) = ops.Segment.apply(lambda x, v, p: (x * p + v,), x, torch.ones(4, 2, 8), packed)
    assert out.requires_grad
    out.sum().backward()
    torch.testing.assert_close(x.grad, packed.expand(4, 2, 8), rtol=0, atol=0)
