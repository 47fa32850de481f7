"""Cases of Transformer(num_residual_streams=1), the plain residual backbone (e2_tts.py:547, :607 with disable=True), stored from the
original e2_tts.py by oracle/make_reference_golden.py. The oracle of oracle/e2tts_oracle.py runs that backbone when its config has one
stream: with one stream the reference's hyper-connection modules are `Residual` (oracle/ref_leaves/hyper_connections.py), the width
connection hands the stream itself to the branch and keeps it as the residual, the depth connection is `branch_out + residual`, and
expand / reduce are identities."""

KW1 = dict(dim=128, depth=2, heads=2, num_residual_streams=1)

# forward + backward cases of the original: class, seed, transformer kwargs, (batch, frames), lens, text, drop_text_cond
RESIDUAL1_CASES = {
    'depth2': dict(cls='E2TTS', seed=62, tkw=KW1, mel=(2, 80), lens=[80, 80], text=['abc', 'a longer text than the first'], drop=False),
    'depth4_lens': dict(cls='E2TTS', seed=64, tkw=dict(KW1, depth=4), mel=(2, 80), lens=[80, 51], text=['abc', 'a longer text than the first'],
                        drop=False),
    'text_dropped': dict(cls='E2TTS', seed=66, tkw=dict(KW1, heads=4), mel=(3, 64), lens=[64, 40, 17], text=['one', 'two words', ''],
                         drop=True),
    'duration': dict(cls='DurationPredictor', seed=68, tkw=KW1, mel=(3, 72), lens=[72, 50, 31], text=['abc', 'hello world', 'x']),
}
# E2TTS.sample: weights seed, transformer kwargs, cond (batch, frames), text, duration, steps, cfg_strength; y0 = first draw of
# generator 3000 + seed
RESIDUAL1_SAMPLE = dict(seed=70, tkw=KW1, cond=(2, 20), text=['Hello', 'Goodbye then'], duration=[40, 33], steps=4, cfg_strength=1.0)
