"""Cases of the reference's attention geometry knobs besides the defaults (e2_tts.py:527-531, defaults :569-570): 128-wide heads
(dim_head, text_dim_head) and a text stream with its own head count (text_heads), stored from the original e2_tts.py by
oracle/make_reference_golden.py. Shared by tests/test_headdim_vs_reference.py (oracle against the original's stored outputs) and the
GPU tests of the same geometry.

The oracle takes the same kwargs as configuration (oracle/e2tts_oracle.py TransformerCfg: text_heads, text_dim_head and the text
stream's own RotaryEmbedding(text_dim_head), :600, :798, :875)."""

# forward + backward cases of the original: class, seed, transformer kwargs, (batch, frames), lens, text, drop_text_cond
HEADDIM_CASES = {
    'h1_d128': dict(cls='E2TTS', seed=81, tkw=dict(dim=128, depth=2, heads=1, dim_head=128), mel=(2, 64), lens=[64, 64],
                    text=['abc', 'a longer text than the first'], drop=False),
    'd256_depth4_lens': dict(cls='E2TTS', seed=82, tkw=dict(dim=256, depth=4, heads=2, dim_head=128, text_heads=1), mel=(2, 80),
                             lens=[80, 51], text=['abc', 'a longer text than the first'], drop=False),
    'mixed_a64_t128': dict(cls='E2TTS', seed=83, tkw=dict(dim=128, depth=2, heads=2, dim_head=64, text_heads=1, text_dim_head=128),
                           mel=(2, 64), lens=[64, 45], text=['abc', 'defgh ij'], drop=False),
    'text_heads1_d64': dict(cls='E2TTS', seed=84, tkw=dict(dim=128, depth=2, heads=2, text_heads=1), mel=(2, 64), lens=[64, 37],
                            text=['hello', 'xy z'], drop=False),
    'text_dropped': dict(cls='E2TTS', seed=85, tkw=dict(dim=128, depth=2, heads=1, dim_head=128), mel=(3, 64), lens=[64, 40, 17],
                         text=['one', 'two words', ''], drop=True),
    'plain_unclamped_d128': dict(cls='E2TTS', seed=86, tkw=dict(dim=128, depth=2, heads=1, dim_head=128, num_residual_streams=1,
                                                                attn_kwargs=dict()),
                                 mel=(2, 64), lens=[64, 50], text=['abc', 'hello']),
    'duration': dict(cls='DurationPredictor', seed=87, tkw=dict(dim=128, depth=2, heads=1, dim_head=128, text_heads=2, text_dim_head=64),
                     mel=(3, 72), lens=[72, 50, 31], text=['abc', 'hello world', 'x']),
}
for _c in HEADDIM_CASES.values():
    _c.setdefault('drop', False)
# E2TTS.sample: weights seed, transformer kwargs, cond (batch, frames), text, duration, steps, cfg_strength; y0 = first draw of
# generator 3000 + seed
HEADDIM_SAMPLE = dict(seed=88, tkw=dict(dim=128, depth=2, heads=1, dim_head=128, text_heads=2, text_dim_head=64), cond=(2, 20),
                      text=['Hello', 'Goodbye then'], duration=[40, 33], steps=4, cfg_strength=1.0)
