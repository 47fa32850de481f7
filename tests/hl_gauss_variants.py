"""Cases of DurationPredictor(hl_gauss_loss=dict(...), use_regression=False) (e2_tts.py:966-967, 1035-1040, 1107, 1111): the HL-Gauss
classification head of hl-gauss-pytorch (SURVEY A.6). Shared by tests/test_hl_gauss_vs_reference.py (oracle against the original's
stored outputs), tests/test_gpu_hl_gauss.py (kernels and models against the oracle) and tools/make_hl_gauss_golden.py."""
KW = dict(dim=128, depth=2, heads=2)

# name -> DurationPredictor case: seed, transformer kwargs, DurationPredictor kwargs,
# mel (batch, frames), lens, text
HL_GAUSS_CASES = {
    'explicit_sigma': dict(cls='DurationPredictor', seed=91, tkw=KW, kw=dict(hl_gauss_loss=dict(min_value=0., max_value=128., num_bins=32,
                                                                                                 sigma=3.), use_regression=False),
                           mel=(3, 72), lens=[72, 50, 31], text=['abc', 'hello world', 'x']),
    # sigma from the default sigma_to_bin_ratio, no text
    'default_sigma_no_text': dict(cls='DurationPredictor', seed=92, tkw=KW, kw=dict(hl_gauss_loss=dict(min_value=0., max_value=100.,
                                                                                                        num_bins=50), use_regression=False),
                                  mel=(3, 72), lens=[72, 50, 31], text=None),
    # two targets beyond max_value, clamped onto it
    'clamp_beyond_max': dict(cls='DurationPredictor', seed=93, tkw=KW, kw=dict(hl_gauss_loss=dict(min_value=0., max_value=40., num_bins=16,
                                                                                                   clamp_to_range=True), use_regression=False),
                             mel=(3, 72), lens=[72, 50, 31], text=['abc', 'hello world', 'x']),
    # a target 2 sigma beyond max_value, unclamped: the histogram is the Gaussian's tail inside the support, renormalised
    'beyond_unclamped': dict(cls='DurationPredictor', seed=94, tkw=KW, kw=dict(hl_gauss_loss=dict(min_value=0., max_value=64., num_bins=64,
                                                                                                   sigma=4.), use_regression=False),
                             mel=(3, 72), lens=[72, 60, 17], text=['abc', 'hello world', 'x']),
}

# E2TTS.sample with an HL-Gauss duration predictor and no `duration`: seed, transformer kwargs, the duration predictor's kwargs, cond
# (batch, frames), text, steps, cfg_strength
HL_GAUSS_SAMPLE = dict(seed=95, tkw=KW, duration_predictor=dict(transformer=dict(dropout=0., max_seq_len=128, **KW),
                                                                hl_gauss_loss=dict(min_value=0., max_value=96., num_bins=48),
                                                                use_regression=False),
                       cond=(2, 24), text=['Hello', 'Goodbye then'], steps=4, cfg_strength=1.0)
