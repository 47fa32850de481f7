"""Cases and oracle of the x-transformers `ff_kwargs` of Transformer (e2_tts.py:552, passed to the audio FeedForward :646 and the text
FeedForward :692): SwiGLU (swish=True), ReLU^2 GLU (relu_squared=True), the GLU multiplicative bias (glu_mult_bias=True) and the output
Linear without bias (no_bias=True). Shared by tests/test_ff_kwargs_vs_reference.py (oracle against the original's stored outputs),
tests/test_gpu_ff_variants.py (kernels against the oracle) and tools/make_ff_kwargs_golden.py.

`XTFeedForward` restates x-transformers' FeedForward / GLU (the >= 1.42 line, SURVEY Appendix A.2) for these keywords; the golden tool
puts it in place of the restated leaf's FeedForward, which takes no keywords, while the original e2_tts.py runs. Built with no keyword it
has the leaf's parameters and draws the same random numbers. `variant_oracle` swaps the oracle's feedforward (oracle/e2tts_oracle.py)
for the same semantics for the duration of a `with` block, keeping the `drop(p + '.ff.1', ...)` hook on the GLU output."""
import contextlib

import torch
import torch.nn.functional as F
from torch import nn

from oracle import e2tts_oracle as O
from oracle import reference_cases as RC
from residual_variants import plain_residual_oracle

KW = dict(dim=128, depth=2, heads=2)

# name -> (ff_kwargs, model class, seed, transformer kwargs besides ff_kwargs, mel shape, lens, text)
FF_KWARGS_CASES = {
    'swish': dict(ff_kwargs=dict(swish=True), cls='E2TTS', seed=81, tkw=KW, mel=(2, 64), lens=[64, 64], text=['abc', 'defgh ij']),
    'relu_squared': dict(ff_kwargs=dict(relu_squared=True), cls='E2TTS', seed=82, tkw=KW, mel=(2, 64), lens=[64, 41],
                         text=['abc', 'xy z']),
    # seed 83 left one hyper-connection scale gradient (max |g| 1.4e-4) 1.5e-7 away from the original's, fp32 summation noise just above
    # the 1e-7 floor of check_grads; this seed's draw keeps every gradient inside it
    'swish_mult_nobias': dict(ff_kwargs=dict(swish=True, glu_mult_bias=True, no_bias=True), cls='E2TTS', seed=86, tkw=KW, mel=(2, 64),
                              lens=[64, 64], text=['hello', 'abc']),
    'gelu_mult_residual1': dict(ff_kwargs=dict(glu_mult_bias=True), cls='E2TTS', seed=84, tkw=dict(KW, num_residual_streams=1),
                                mel=(2, 64), lens=[64, 64], text=['abc', 'a longer text']),
    'duration_relu2_nobias': dict(ff_kwargs=dict(relu_squared=True, no_bias=True), cls='DurationPredictor', seed=85, tkw=KW, mel=(3, 72),
                                  lens=[72, 50, 31], text=['abc', 'hello world', 'x']),
}


def act_of(ff_kwargs):
    """the GLU activation of these kwargs, x-transformers' precedence: relu_squared, then swish, then the exact erf GELU"""
    if ff_kwargs.get('relu_squared'):
        return lambda g: F.relu(g) ** 2
    if ff_kwargs.get('swish'):
        return F.silu
    return F.gelu


def perturb_mult_bias(sd, seed):
    """every GLU mult_bias of `sd` moved away from its all-ones init: O.randomize_zero_init leaves ones alone, and a multiplier of 1
    is invisible"""
    g = torch.Generator().manual_seed(seed + 500)
    for k in sorted(sd):
        if k.endswith('.ff.0.mult_bias'):
            sd[k] = 1.0 + 0.5 * torch.randn(sd[k].shape, generator=g)
    return sd


def state_dict(c):
    """RC.state_dict of the case, its GLU multipliers perturbed"""
    return perturb_mult_bias(RC.state_dict(c['cls'], c['seed'], dict(c['tkw'], ff_kwargs=c['ff_kwargs'])), c['seed'])


@contextlib.contextmanager
def mult_bias_randomized():
    """inside the block O.randomize_zero_init (which the whole-model checks seed their weights with) also perturbs mult_bias"""
    orig = O.randomize_zero_init
    O.randomize_zero_init = lambda sd, seed, **kw: perturb_mult_bias(orig(sd, seed=seed, **kw), seed)
    try:
        yield
    finally:
        O.randomize_zero_init = orig


class _XTGLU(nn.Module):
    def __init__(self, dim_in, dim_out, activation, mult_bias=False):
        super().__init__()
        self.act = activation
        self.proj = nn.Linear(dim_in, dim_out * 2)
        self.mult_bias = nn.Parameter(torch.ones(dim_out)) if mult_bias else 1.

    def forward(self, x):
        x, gate = self.proj(x).chunk(2, dim=-1)
        return x * self.act(gate) * self.mult_bias


class XTFeedForward(nn.Module):
    """x-transformers FeedForward(glu=True) with the keywords above; any other keyword away from its default is not restated"""

    def __init__(self, dim, mult=4, glu=False, dropout=0., swish=False, relu_squared=False, glu_mult_bias=False, no_bias=False,
                 zero_init_output=False):
        super().__init__()
        assert glu
        inner = int(dim * mult)
        act = act_of(dict(swish=swish, relu_squared=relu_squared))
        self.ff = nn.Sequential(_XTGLU(dim, inner, act, glu_mult_bias), nn.Dropout(dropout), nn.Linear(inner, dim, bias=not no_bias))
        if zero_init_output:
            nn.init.zeros_(self.ff[2].weight)
            if self.ff[2].bias is not None:
                nn.init.zeros_(self.ff[2].bias)

    def forward(self, x):
        return self.ff(x)


def feedforward(sd, p, x, act):
    """O.feedforward with the activation `act`, the optional GLU multiplier (p.ff.0.mult_bias) and the optional output bias"""
    h = x @ sd[p + '.ff.0.proj.weight'].t() + sd[p + '.ff.0.proj.bias']
    u, g = h.chunk(2, dim=-1)
    hid = u * act(g)
    if p + '.ff.0.mult_bias' in sd:
        hid = hid * sd[p + '.ff.0.mult_bias']
    y = O.drop(p + '.ff.1', hid) @ sd[p + '.ff.2.weight'].t()
    if p + '.ff.2.bias' in sd:
        y = y + sd[p + '.ff.2.bias']
    return y


@contextlib.contextmanager
def variant_oracle(ff_kwargs):
    """O.e2tts_forward / O.duration_forward / O.e2tts_sample run the feed-forward of `ff_kwargs` inside the block"""
    act = act_of(ff_kwargs)
    orig = O.feedforward
    O.feedforward = lambda sd, p, x: feedforward(sd, p, x, act)
    try:
        yield
    finally:
        O.feedforward = orig


@contextlib.contextmanager
def case_oracle(c):
    """variant_oracle of the case, on the plain residual backbone when the case has one stream"""
    with contextlib.ExitStack() as stack:
        stack.enter_context(variant_oracle(c['ff_kwargs']))
        if c['tkw'].get('num_residual_streams', 4) == 1:
            stack.enter_context(plain_residual_oracle())
        yield


def cfg(c, **kw):
    return O.TransformerCfg(**c['tkw'], **kw)
