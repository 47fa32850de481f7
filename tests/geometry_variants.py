"""Cases of the reference's model-shape knobs besides the defaults (Transformer, e2_tts.py:518-552): depth past 8 (six skip levels),
text_depth < depth, dim_text != dim // 2, ff_mult / text_ff_mult != 4 (one of them non-integer), num_registers != 32 (0 included),
abs_pos_emb=False and kernel_size != 31, stored from the original e2_tts.py by oracle/make_reference_golden.py. Shared by
tests/test_geometry_vs_reference.py (oracle against the original's stored outputs) and tests/test_gpu_geometry.py.

Every knob is a field of the oracle's TransformerCfg, so TransformerCfg(**tkw) is the whole oracle configuration of a case. `knobs`
names the knobs a case's negative control reverts, one at a time, to the reference's default (test_geometry_vs_reference.py): the
oracle must then miss the stored outputs."""
from oracle import reference_cases as RC

# the reference's defaults of the knobs (e2_tts.py:524-541); dim_text, text_ff_mult and text_depth follow dim, ff_mult and depth
DEFAULTS = dict(depth=8, text_depth=None, dim_text=None, ff_mult=4, text_ff_mult=None, num_registers=32, abs_pos_emb=True, kernel_size=31)

# forward + backward cases of the original: class, seed, transformer kwargs, (batch, frames), lens, text, drop_text_cond, knobs;
# grad_tol = (rel, floor) of model_checks.check_grads where it is not the default of the 2-layer E2TTS fixtures
GEOMETRY_CASES = {
    # 12 layers chain twice the fp32 roundings of the depth-4 fixtures: the scalar dynamic_alpha_scale of layer 4's text conv
    # hyper-connection (a sum over every token and stream) differs from the original's by 5.5e-4 of its value, so this case takes the
    # DurationPredictor fixtures' bound
    'depth12_text5': dict(cls='E2TTS', seed=101, tkw=dict(dim=128, depth=12, heads=2, text_depth=5), mel=(2, 64), lens=[64, 41],
                          text=['abc', 'a longer text than the first'], knobs=('depth', 'text_depth'), grad_tol=(5e-4, 1e-6)),
    'd192_ff2_text2p5': dict(cls='E2TTS', seed=102, tkw=dict(dim=192, depth=2, heads=3, dim_text=128, ff_mult=2, text_ff_mult=2.5),
                             mel=(2, 64), lens=[64, 50], text=['hello', 'xy z'], knobs=('ff_mult', 'text_ff_mult')),
    'registers0_k7': dict(cls='E2TTS', seed=103, tkw=dict(dim=128, depth=2, heads=2, num_registers=0, kernel_size=7), mel=(2, 64),
                          lens=[64, 37], text=['abc', 'defgh ij'], knobs=('num_registers', 'kernel_size')),
    'registers16_noabs_k1': dict(cls='E2TTS', seed=104, tkw=dict(dim=128, depth=2, heads=2, num_registers=16, abs_pos_emb=False,
                                                                kernel_size=1),
                                 mel=(3, 64), lens=[64, 45, 30], text=['one', 'two words', 'x'],
                                 knobs=('num_registers', 'abs_pos_emb', 'kernel_size')),
    # text dropped: text_depth changes the parameters only, so its control is num_registers'
    'text_depth1_dropped': dict(cls='E2TTS', seed=105, tkw=dict(dim=128, depth=4, heads=2, text_depth=1, num_registers=8), mel=(3, 64),
                                lens=[64, 40, 17], text=['one', 'two words', ''], drop=True, knobs=('num_registers',)),
    'duration': dict(cls='DurationPredictor', seed=106, tkw=dict(dim=128, depth=4, heads=2, text_depth=2, dim_text=128), mel=(3, 72),
                     lens=[72, 50, 31], text=['abc', 'hello world', 'x'], knobs=('text_depth', 'dim_text')),
}
for _c in GEOMETRY_CASES.values():
    _c.setdefault('drop', False)
    _c.setdefault('grad_tol', (2e-4, 1e-7) if _c['cls'] == 'E2TTS' else (5e-4, 1e-6))
# E2TTS.sample with a per-element duration and a ragged prompt: weights seed, transformer kwargs, cond (batch, frames), prompt lens,
# text, duration, steps, cfg_strength; y0 = first draw of generator 3000 + seed
GEOMETRY_SAMPLE = dict(seed=107, tkw=dict(dim=128, depth=4, heads=2, text_depth=2, num_registers=8, kernel_size=5), cond=(2, 20),
                       lens=[20, 13], text=['Hello', 'Goodbye then'], duration=[40, 33], steps=4, cfg_strength=1.0)


def reverted(c, knob):
    """(transformer kwargs, state dict) of case `c` with `knob` back at the reference's default: the case's own weights, plus the seeded
    weights of the default model for every parameter the case lacks or holds in another shape (the default's 32 registers, its
    31-tap convolutions, abs_pos_emb, the text sub-blocks past text_depth, ...)"""
    tkw = {**c['tkw'], knob: DEFAULTS[knob]}
    tkw = {k: v for k, v in tkw.items() if v is not None}
    sd = RC.state_dict(c['cls'], c['seed'], c['tkw'])
    for k, v in RC.state_dict(c['cls'], c['seed'], tkw).items():
        if k not in sd or sd[k].shape != v.shape:
            sd[k] = v
    return tkw, sd
