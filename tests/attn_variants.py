"""Cases of the x-transformers `attn_kwargs` the model builds besides the reference's default (gate_value_heads=True,
softclamp_logits=True): no head gate, no logit soft-clamp, another clamp value. Shared by tests/test_attn_kwargs_vs_reference.py
(oracle against the original's stored outputs), tests/test_gpu_attention_variants.py (kernels against the oracle) and
oracle/make_reference_golden.py. The oracle takes the same attn_kwargs as configuration (oracle/e2tts_oracle.py TransformerCfg)."""

KW = dict(dim=128, depth=2, heads=2)

# name -> (model class, seed, transformer kwargs, mel shape, lens, text)
ATTN_KWARGS_CASES = {
    'plain': dict(cls='E2TTS', seed=51, tkw=dict(KW, attn_kwargs=dict()), mel=(2, 64), lens=[64, 45], text=['abc', 'defgh ij']),
    'gate_only': dict(cls='E2TTS', seed=52, tkw=dict(KW, attn_kwargs=dict(gate_value_heads=True)), mel=(2, 64), lens=[64, 37],
                      text=['abc', 'xy z']),
    'clamp30': dict(cls='E2TTS', seed=53, tkw=dict(KW, attn_kwargs=dict(softclamp_logits=True, logit_softclamp_value=30.)), mel=(2, 64),
                    lens=[64, 50], text=['hello', 'abc']),
    'duration_plain': dict(cls='DurationPredictor', seed=54, tkw=dict(KW, attn_kwargs=dict()), mel=(3, 72), lens=[72, 50, 31],
                           text=['abc', 'hello world', 'x']),
}
