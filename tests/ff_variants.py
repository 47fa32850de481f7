"""Cases of the x-transformers `ff_kwargs` of Transformer (e2_tts.py:552, passed to the audio FeedForward :646 and the text
FeedForward :692): SwiGLU (swish=True), ReLU^2 GLU (relu_squared=True), the GLU multiplicative bias (glu_mult_bias=True) and the output
Linear without bias (no_bias=True). Shared by tests/test_ff_kwargs_vs_reference.py (oracle against the original's stored outputs),
tests/test_gpu_ff_variants.py (kernels against the oracle) and oracle/make_reference_golden.py. The oracle takes the same ff_kwargs as
configuration (oracle/e2tts_oracle.py TransformerCfg).

`XTFeedForward` restates x-transformers' FeedForward / GLU (the >= 1.42 line, SURVEY Appendix A.2) for these keywords;
oracle/make_reference_golden.py puts it in place of the restated leaf's FeedForward, which takes no keywords, while the original
e2_tts.py runs. Built with no keyword it has the leaf's parameters and draws the same random numbers."""
import torch
from torch import nn

from oracle import e2tts_oracle as O

KW = dict(dim=128, depth=2, heads=2)

# name -> (model class, seed, transformer kwargs, mel shape, lens, text)
FF_KWARGS_CASES = {
    'swish': dict(cls='E2TTS', seed=81, tkw=dict(KW, ff_kwargs=dict(swish=True)), mel=(2, 64), lens=[64, 64], text=['abc', 'defgh ij']),
    'relu_squared': dict(cls='E2TTS', seed=82, tkw=dict(KW, ff_kwargs=dict(relu_squared=True)), mel=(2, 64), lens=[64, 41],
                         text=['abc', 'xy z']),
    # seed 83 left one hyper-connection scale gradient (max |g| 1.4e-4) 1.5e-7 away from the original's, fp32 summation noise just above
    # the 1e-7 floor of check_grads; this seed's draw keeps every gradient inside it
    'swish_mult_nobias': dict(cls='E2TTS', seed=86, tkw=dict(KW, ff_kwargs=dict(swish=True, glu_mult_bias=True, no_bias=True)),
                              mel=(2, 64), lens=[64, 64], text=['hello', 'abc']),
    'gelu_mult_residual1': dict(cls='E2TTS', seed=84, tkw=dict(KW, num_residual_streams=1, ff_kwargs=dict(glu_mult_bias=True)),
                                mel=(2, 64), lens=[64, 64], text=['abc', 'a longer text']),
    'duration_relu2_nobias': dict(cls='DurationPredictor', seed=85, tkw=dict(KW, ff_kwargs=dict(relu_squared=True, no_bias=True)),
                                  mel=(3, 72), lens=[72, 50, 31], text=['abc', 'hello world', 'x']),
}


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
        act = O.act_of(dict(swish=swish, relu_squared=relu_squared))
        self.ff = nn.Sequential(_XTGLU(dim, inner, act, glu_mult_bias), nn.Dropout(dropout), nn.Linear(inner, dim, bias=not no_bias))
        if zero_init_output:
            nn.init.zeros_(self.ff[2].weight)
            if self.ff[2].bias is not None:
                nn.init.zeros_(self.ff[2].bias)

    def forward(self, x):
        return self.ff(x)
