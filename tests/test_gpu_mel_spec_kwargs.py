"""GPU: the mel-spectrogram kernels with the reference's `mel_spec_kwargs` (csrc/small.cu melspec_kernel, radix-2, and
melspec_mixed_kernel, Stockham radix-4/2/3/5), and the raw-wave paths of the modules that use them.

Kernels: b200_melspec_ex is called through the C ABI with NaN-filled outputs and every element is held to the float64 restatement
of tests/mel_kwargs_ref.py (`mel64`) within the bound its docstring derives (radix-2 stages as in
test_gpu_conv_melspec_kernels' mel_ref, radix-3/4/5 Stockham stages with their own per-stage growth, |.| * scale, the power, the
band-limited filter sum, the log). Modules: MelSpec against the original's golden files, MelSpec.collate on a ragged batch without
centring, and E2TTS forward / backward, sample() and DurationPredictor from raw 16 kHz waves (n_fft 400, 80 mels) against the oracle
fed the mel the kernel computed.
"""
import math

import pytest
import torch

from kernel_checks import F32, check_e, check_f, dev, gen, nans, pkg, stream  # noqa: F401 (pkg: the fixture)
from mel_kwargs_ref import LOG_FLOOR, MEL_KWARGS_CASES, case_wave, mel64, mel_of_module, norm_scale, radices
from model_checks import cos, rel_l2
from oracle import e2tts_oracle as O
from oracle import reference_cases as RC

pytestmark = pytest.mark.gpu


def mel_launch_ex(pkg, wave, window, fb, n_fft, hop, center, power, scale, lens=None, out_bnd=False):
    """b200_melspec_ex with a NaN-filled output; returns [B, n_mels, frames] whatever the layout"""
    B, nw = wave.shape
    n_mels = fb.shape[1]
    frames = pkg.ops.melspec_frames(nw, n_fft, hop, center)
    out = nans((B, frames, n_mels) if out_bnd else (B, n_mels, frames), F32)
    bands = torch.empty(2 * n_mels, device=dev(), dtype=torch.int32)
    a = pkg.lib.make_args('b200_melspec_args', wave=wave, window=window, fb=fb, out=out, B=B, nw=nw, n_fft=n_fft, hop=hop, n_mels=n_mels,
                          ws_bands=bands, wave_lens=lens, out_bnd=int(out_bnd), win_length=window.shape[0], center=int(center),
                          power=float(power), norm_scale=float(scale))
    pkg.lib.call('b200_melspec_ex', a, stream())
    return out.transpose(1, 2) if out_bnd else out


def mel_inputs(pkg, n_fft, win, n_mels, sr, norm, B, nw, seed):
    """a wave of B items at 0.3 rms whose first third is 1e-6 quieter and first ninth 1e-12 quieter (log-mel below the 1e-5 clamp,
    for powers below 1 too), the periodic Hann window of win taps and the (HTK or Slaney) filterbank"""
    g = gen(seed)
    wave = torch.randn(B, nw, generator=g) * 0.3
    wave[:, :nw // 3] *= 1e-6
    wave[:, :nw // 9] *= 1e-6
    return wave, torch.hann_window(win, periodic=True), pkg.modules.mel_filterbank(n_fft // 2 + 1, n_mels, sr, norm=norm)


# name, n_fft, hop, n_mels, win_length, center, power, normalize, norm, sample rate, nw, B, out_bnd
MEL_EX_CASES = [
    ('win800-even-offset', 1024, 256, 100, 800, True, 1, False, None, 24000, 256 * 12, 2, False),
    ('win801-odd-offset', 1024, 256, 100, 801, True, 1, False, None, 24000, 256 * 12 - 1, 2, True),
    ('valid-one-frame', 1024, 256, 100, 1024, False, 1, False, None, 24000, 1024, 2, False),
    ('valid-k-hop-minus-1', 1024, 256, 100, 1024, False, 1, False, None, 24000, 1024 + 6 * 256 - 1, 2, True),
    ('power0.5', 1024, 256, 100, 1024, True, 0.5, False, None, 24000, 256 * 40, 2, False),
    ('power1.5', 1024, 256, 100, 1024, True, 1.5, False, None, 24000, 256 * 10, 1, True),
    ('power2', 1024, 256, 100, 1024, True, 2, False, None, 24000, 256 * 10, 2, False),
    ('normalize-window', 1024, 256, 100, 1024, True, 1, True, None, 24000, 256 * 10, 2, False),
    ('normalize-frame-length', 1024, 256, 100, 1024, True, 1, 'frame_length', None, 24000, 256 * 10, 1, True),
    ('slaney', 1024, 256, 100, 1024, True, 1, False, 'slaney', 24000, 256 * 10, 2, False),
    ('nfft64-win33-empty', 64, 1, 100, 33, True, 2, True, 'slaney', 24000, 200, 1, True),
    ('nfft4096-valid-win4000', 4096, 512, 100, 4000, False, 1, False, None, 24000, 4096 + 512 * 3 - 1, 1, False),
    ('nfft96-radix3-empty', 96, 7, 100, 96, True, 1, False, None, 24000, 300, 2, False),
    ('nfft375-odd', 375, 100, 40, 300, True, 1.5, False, None, 8000, 2000, 2, True),
    ('nfft400-16k', 400, 160, 80, 400, True, 1, False, None, 16000, 16000 // 2 + 17, 2, False),
    ('nfft400-16k-valid', 400, 160, 80, 399, False, 2, 'frame_length', 'slaney', 16000, 400 + 160 * 7 - 1, 2, True),
    ('nfft1200-win960-valid', 1200, 300, 100, 960, False, 1, False, None, 24000, 1200 + 300 * 8, 2, False),
    ('nfft2187-radix3x7', 2187, 300, 90, 2187, True, 1, False, None, 22050, 4000, 1, True),
    ('nfft3840', 3840, 480, 128, 3840, True, 1, False, None, 48000, 3840 * 3, 1, False),
    ('nfft4000-valid', 4000, 500, 100, 3999, False, 0.5, True, None, 24000, 4000, 2, True),
    ('nfft4050-largest', 4050, 256, 100, 4050, True, 2, False, 'slaney', 24000, 4050 * 2 + 3, 1, False),
    ('all-960', 960, 240, 64, 777, False, 1.5, True, 'slaney', 16000, 960 + 240 * 10, 2, True),
]


def check_ex(pkg, case, lens=None):
    name, n_fft, hop, n_mels, win, center, power, normalize, norm, sr, nw, B, out_bnd = case
    wave, window, fb = mel_inputs(pkg, n_fft, win, n_mels, sr, norm, B, nw, seed=sum(map(ord, name)))
    scale = norm_scale(window, normalize, n_fft)
    got = mel_launch_ex(pkg, wave.to(dev()), window.to(dev()), fb.to(dev()), n_fft, hop, center, power, scale, out_bnd=out_bnd)
    torch.cuda.synchronize()
    ref, bound = mel64(wave, window, fb, n_fft, hop, center=center, power=power, scale=scale, bound=True)
    check_f(f'{name} log-mel', got, ref, bound)
    return got.cpu(), ref, fb


@pytest.mark.parametrize('case', MEL_EX_CASES, ids=[c[0] for c in MEL_EX_CASES])
def test_melspec_ex_kernel(pkg, case):
    got, ref, fb = check_ex(pkg, case)
    name, n_fft, hop, n_mels, win, center, power, normalize, norm, sr, nw, B, out_bnd = case
    assert got.shape == (B, n_mels, pkg.ops.melspec_frames(nw, n_fft, hop, center))
    floor = torch.log(torch.tensor([LOG_FLOOR], device=dev(), dtype=F32)).cpu()
    empty = (fb == 0).all(0)
    if bool(empty.any()):
        v = got[:, empty]
        check_e('empty filters', v, floor.expand_as(v))
    if name.startswith('power'):
        assert bool((ref <= math.log(LOG_FLOOR)).any()), 'the quiet part of the wave reaches below the log floor'


def test_melspec_ex_cases_reach_every_edge():
    """every switch alone and together; radix-3 and radix-5 stages, many stages, n_fft near 4096 on both FFTs; odd and even window
    offsets; valid framing with one frame and with nw = n_fft + k hop - 1; powers 0.5, 1.5 and 2; empty filters; both layouts"""
    sw = lambda c: (c[4] != c[1], not c[5], c[6] != 1, c[7] is not False, c[8] is not None)
    assert all(any(sw(c)[i] and sum(sw(c)) == 1 for c in MEL_EX_CASES) for i in range(5))
    assert any(all(sw(c)) for c in MEL_EX_CASES)
    rad = [radices(c[1]) for c in MEL_EX_CASES]
    assert any(3 in r for r in rad) and any(5 in r for r in rad) and any(len(r) >= 6 and set(r) != {2} for r in rad)
    assert any(c[1] in (3840, 4000) for c in MEL_EX_CASES) and any(c[1] == 4096 for c in MEL_EX_CASES)
    offs = {(c[1] - c[4]) // 2 % 2 for c in MEL_EX_CASES if c[4] < c[1]}
    assert offs == {0, 1}
    valid = [c for c in MEL_EX_CASES if not c[5]]
    assert any(c[10] == c[1] for c in valid) and any((c[10] - c[1]) % c[2] == c[2] - 1 for c in valid)
    assert {0.5, 1.5, 2} <= {c[6] for c in MEL_EX_CASES}
    assert any(bool((pkg_fb(c) == 0).all(0).any()) for c in MEL_EX_CASES)
    assert {c[12] for c in MEL_EX_CASES} == {False, True}


def pkg_fb(c):
    import e2_tts_pytorch_b200 as pkg
    return pkg.modules.mel_filterbank(c[1] // 2 + 1, c[3], c[9], norm=c[8])


def test_melspec_ex_defaults_equal_positional(pkg):
    """b200_melspec_ex at the defaults (win_length = n_fft, center, power 1, scale 1) gives b200_melspec's bits, ragged or not"""
    for n_fft, hop, nw in ((1024, 256, 256 * 20 + 5), (256, 100, 1999), (4096, 256, 256 * 20 - 1), (1200, 300, 5000)):
        wave, window, fb = mel_inputs(pkg, n_fft, n_fft, 100, 24000, None, 3, nw, seed=n_fft)
        wd, wnd, fbd = wave.to(dev()), window.to(dev()), fb.to(dev())
        lens = torch.tensor([nw, nw // 2, n_fft // 2], dtype=torch.int32, device=dev())
        for ld in (None, lens):
            for bnd in (False, True):
                ex = mel_launch_ex(pkg, wd, wnd, fbd, n_fft, hop, True, 1, 1.0, lens=ld, out_bnd=bnd)
                frames = 1 + nw // hop
                out = nans((3, frames, 100) if bnd else (3, 100, frames), F32)
                bands = torch.empty(200, device=dev(), dtype=torch.int32)
                pkg.lib.call('b200_melspec', wd, wnd, fbd, out, 3, nw, n_fft, hop, 100, bands, ld, int(bnd), stream())
                check_e(f'n_fft {n_fft} lens={ld is not None} bnd={bnd}', ex, out.transpose(1, 2) if bnd else out)


def test_melspec_ex_ragged_valid_framing(pkg):
    """wave_lens without centring: items shorter than n_fft give zero frames, others 1 + (len - n_fft) // hop frames bit-identical to
    the item launched alone, then +0; mixed-radix and radix-2 FFTs; both layouts"""
    for n_fft, hop, win in ((1200, 300, 960), (1024, 256, 1000)):
        nw_max = n_fft + hop * 12
        lens = [n_fft - 1, n_fft, n_fft + 3 * hop - 1, 300, nw_max, 99999]
        wave, window, fb = mel_inputs(pkg, n_fft, win, 100, 24000, None, len(lens), nw_max, seed=n_fft + 1)
        for i, n in enumerate(lens):
            wave[i, min(n, nw_max):] = 0
        wd, wnd, fbd = wave.to(dev()), window.to(dev()), fb.to(dev())
        ld = torch.tensor(lens, dtype=torch.int32, device=dev())
        for bnd in (False, True):
            got = mel_launch_ex(pkg, wd, wnd, fbd, n_fft, hop, False, 2, 0.5, lens=ld, out_bnd=bnd).cpu()
            for i, n in enumerate(lens):
                n = min(n, nw_max)
                if n < n_fft:
                    check_e(f'item {i} (len {n})', got[i], torch.zeros_like(got[i]))
                    continue
                alone = mel_launch_ex(pkg, wd[i:i + 1, :n].contiguous(), wnd, fbd, n_fft, hop, False, 2, 0.5, out_bnd=bnd).cpu()
                fi = 1 + (n - n_fft) // hop
                check_e(f'item {i} (len {n})', got[i, :, :fi], alone[0])
                check_e(f'item {i} (len {n}) padding', got[i, :, fi:], torch.zeros_like(got[i, :, fi:]))
                if not bnd:
                    ref, bound = mel64(wave[i:i + 1, :n], window, fb, n_fft, hop, center=False, power=2, scale=0.5, bound=True)
                    check_f(f'item {i} (len {n})', alone, ref, bound)


# ======================================================================================================== modules
@pytest.mark.parametrize('name', list(MEL_KWARGS_CASES))
def test_melspec_module_vs_reference(pkg, name):
    """MelSpec(**kwargs) on the GPU within the kernel bound of the restatement, and within twice it of the original's output"""
    c = MEL_KWARGS_CASES[name]
    ms = pkg.MelSpec(**c['kw'])
    wave = case_wave(c)
    ref, bound = mel_of_module(ms, wave, bound=True)
    got = ms.to(dev())(wave.to(dev())).cpu()
    check_f(f'{name} vs restatement', got, ref, bound)
    check_f(f'{name} vs reference', got, RC.load('melspec_kwargs_' + name)['mel'].double(), 2 * bound)


def test_collate_valid_framing_vs_per_item(pkg):
    """MelSpec(center=False, n_fft=1200).collate of a ragged list, items shorter than n_fft included: mel_lengths, each item's rows
    against its own float64 log-mel, zero rows behind them"""
    ms = pkg.MelSpec(filter_length=1200, hop_length=300, win_length=960, center=False, power=2, normalize=True).to(dev())
    g = gen(31)
    sizes = [700, 1199, 1200, 1200 + 300 * 5 - 1, 24000, 1500]
    waves = [torch.randn(n, generator=g) * 0.3 for n in sizes]
    batch = ms.collate(waves)
    want_len = [0, 0, 1, 5, 1 + (24000 - 1200) // 300, 2]
    assert batch['mel_lengths'].tolist() == want_len
    assert batch['mel'].shape == (len(sizes), 1 + (24000 - 1200) // 300, 100)
    mel = batch['mel'].cpu()
    for i, (w, n) in enumerate(zip(waves, want_len)):
        if n:
            ref, bound = mel_of_module(ms, w[None], bound=True)
            check_f(f'item {i}', mel[i, :n].T, ref[0], bound[0])
        check_e(f'item {i} padding', mel[i, n:], torch.zeros_like(mel[i, n:]))


KW16K = dict(filter_length=400, hop_length=160, win_length=400, n_mel_channels=80, sampling_rate=16000)
TKW = dict(dim=128, depth=2, heads=2)


def _model(pkg, cls, seed):
    torch.manual_seed(seed)
    t = dict(dropout=0., max_seq_len=256, **TKW)
    m = pkg.E2TTS(transformer=t, mel_spec_kwargs=KW16K, use_vocos=False) if cls == 'E2TTS' else pkg.DurationPredictor(transformer=t, mel_spec_kwargs=KW16K)
    sd0 = m.state_dict()
    # dyn_scale 0.05 as model_checks.whole_model: hyper-connection scales at which a bf16 path is well conditioned
    sd = O.randomize_zero_init({k: v.clone() for k, v in sd0.items()}, seed=seed + 1, dyn_scale=0.05)
    sd.update({k: v.clone() for k, v in sd0.items() if k.startswith('mel_spec.')})   # the filterbank's zeros are the filterbank
    m.load_state_dict(sd)
    return m.to(dev()), sd


def _waves(seed, B=2, n=16000 // 2 + 77):
    g = gen(seed)
    return torch.randn(B, n, generator=g) * 0.3


def test_e2tts_forward_backward_from_raw_16k_waves(pkg):
    """E2TTS(mel_spec_kwargs=16 kHz, n_fft 400, 80 mels) on raw waves: the mel it computes within the kernel bound, then loss,
    prediction and gradients against the oracle fed that mel (80 channels through the padded stem and to_pred)"""
    model, sd = _model(pkg, 'E2TTS', 51)
    model.train()
    wave = _waves(52)
    ref_mel, bound = mel_of_module(model.mel_spec, wave, bound=True)
    mel_gpu = model.mel_spec(wave.to(dev()))
    check_f('mel', mel_gpu, ref_mel, bound)
    mel = mel_gpu.transpose(1, 2).cpu().contiguous()            # [B, N, 80]
    B, N, C = mel.shape
    assert C == 80 and N == 1 + wave.shape[1] // 160
    x0, times = torch.randn(B, N, C, generator=gen(53)), torch.rand(B, generator=gen(54))
    span = torch.zeros(B, N, dtype=torch.bool)
    span[:, N // 6:N - N // 7] = True
    text = ['Hello', 'Goodbye']
    with pkg.inject_randomness(x0=x0.to(dev()), times=times.to(dev()), span_mask=span.to(dev()), drop_text_cond=False):
        out = model(wave.to(dev()), text=text)
    out.loss.backward()
    osd = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    ref = O.e2tts_forward(osd, O.TransformerCfg(**TKW), mel, O.list_str_to_tensor(text), x0=x0, times=times, span_mask=span)
    ref['loss'].backward()
    assert out.pred_flow.shape == (B, N, 80)
    assert abs(float(out.loss) - float(ref['loss'])) <= 1e-2 * abs(float(ref['loss']))
    assert rel_l2(out.pred_flow.float().cpu(), ref['pred'].detach()) < 3e-2
    total = float(torch.cat([v.grad.flatten() for v in osd.values() if v.grad is not None]).norm())
    for k, p in model.named_parameters():
        gr = osd[k].grad
        if gr is None or float(gr.norm()) < 1e-4 * total:
            continue
        assert cos(p.grad.cpu(), gr) >= 0.99, k


def test_e2tts_sample_from_raw_wave_cond(pkg):
    """E2TTS.sample(cond=raw 16 kHz wave) against the oracle's sample fed the kernel's mel of that wave"""
    model, sd = _model(pkg, 'E2TTS', 61)
    wave = _waves(62, n=16000 // 4)
    mel = model.mel_spec(wave.to(dev())).transpose(1, 2).cpu().contiguous()
    B, N, C = mel.shape
    duration = torch.tensor([N + 9, N + 4])
    y0 = torch.randn(B, int(duration.max()), C, generator=gen(63))
    with pkg.inject_randomness(y0=y0.to(dev())):
        out = model.sample(wave.to(dev()), text=['Hi there', 'Yo'], duration=duration.to(dev()), steps=4, cfg_strength=1.0,
                           return_raw_output=True)
    want = O.e2tts_sample(sd, O.TransformerCfg(**TKW), mel, O.list_str_to_tensor(['Hi there', 'Yo']), duration=duration, y0=y0, steps=4,
                          cfg_strength=1.0)
    assert out.shape == want.shape == (B, int(duration.max()), 80)
    assert rel_l2(out.cpu(), want) < 5e-2


def test_duration_predictor_from_raw_waves(pkg):
    """DurationPredictor(mel_spec_kwargs=16 kHz) on raw waves against the oracle fed the kernel's mel"""
    model, sd = _model(pkg, 'DurationPredictor', 71)
    model.train()
    wave = _waves(72)
    mel = model.mel_spec(wave.to(dev())).transpose(1, 2).cpu().contiguous()
    rand_frac = torch.tensor([0.4, 0.8])
    with pkg.inject_randomness(duration_rand_frac=rand_frac.to(dev())):
        loss = model(wave.to(dev()), text=['abc', 'hello world'])
    loss.backward()
    osd = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    ref = O.duration_forward(osd, O.TransformerCfg(cond_on_time=False, **TKW), mel, O.list_str_to_tensor(['abc', 'hello world']),
                             rand_frac=rand_frac)
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-2 * abs(float(ref))
    total = float(torch.cat([v.grad.flatten() for v in osd.values() if v.grad is not None]).norm())
    for k, p in model.named_parameters():
        gr = osd[k].grad
        if gr is None or float(gr.norm()) < 1e-4 * total:
            continue
        assert cos(p.grad.cpu(), gr) >= 0.99, k
