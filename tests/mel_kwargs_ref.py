"""The reference's `mel_spec_kwargs` (e2_tts.py:249-260): the cases pinned to the original MelSpec (tools/make_melspec_kwargs_golden.py,
tests/golden/reference/melspec_kwargs_<case>.pt) and a float64 restatement of torchaudio's MelSpectrogram for them, with the
element-wise bound of the CUDA kernels (csrc/small.cu melspec_kernel / melspec_mixed_kernel) against it.

torchaudio semantics (functional.spectrogram, melscale_fbanks): a periodic Hann window of win_length taps, zero-padded to n_fft with
(n_fft - win_length) // 2 zeros on the left (torch.stft); center reflect-pads by n_fft // 2 on both sides, otherwise only whole
frames; X / sqrt(sum window^2) (normalize True / 'window') or X / sqrt(n_fft) ('frame_length'); |X| ** power; HTK mel filterbank,
Slaney-scaled by 2 / (f[i+2] - f[i]) with norm='slaney'; then the reference's log(clamp(mel, 1e-5)).
"""
import math

import torch
import torch.nn.functional as F

from kernel_checks import F64, U, gamma, h64

LOG_FLOOR = 9.99999974737875e-06   # float(np.float32(1e-5)): the kernel's clamp 1e-5f

# name -> MelSpec kwargs, batch, samples, seed. The waves are RC.randn((B, nw), seed) * 0.3 with the first third 1e-3 quieter.
MEL_KWARGS_CASES = {
    'win800': dict(kw=dict(win_length=800), B=2, nw=4000, seed=11),                        # left pad 112
    'win801': dict(kw=dict(win_length=801), B=1, nw=3001, seed=12),                        # odd n_fft - win_length: left pad 111
    'center_false': dict(kw=dict(center=False), B=2, nw=1024 + 256 * 9 + 100, seed=13),
    'power2': dict(kw=dict(power=2), B=2, nw=3500, seed=14),
    'power_half': dict(kw=dict(power=0.5), B=1, nw=3500, seed=15),
    'normalize_window': dict(kw=dict(normalize=True), B=2, nw=3000, seed=16),
    'normalize_frame_length': dict(kw=dict(normalize='frame_length'), B=1, nw=3000, seed=17),
    'slaney': dict(kw=dict(norm='slaney'), B=2, nw=3000, seed=18),
    'sr16k_nfft400': dict(kw=dict(filter_length=400, hop_length=160, win_length=400, n_mel_channels=80, sampling_rate=16000),
                          B=2, nw=16000 // 4 + 37, seed=19),
    'nfft1200_win960_valid': dict(kw=dict(filter_length=1200, hop_length=300, win_length=960, center=False), B=2, nw=1200 + 300 * 8 + 299,
                                  seed=20),
    'all': dict(kw=dict(filter_length=960, hop_length=240, win_length=777, n_mel_channels=64, sampling_rate=16000, normalize=True,
                        power=1.5, norm='slaney', center=False), B=2, nw=960 + 240 * 10, seed=21),
}

TA_NAMES = dict(filter_length='n_fft', hop_length='hop_length', win_length='win_length', n_mel_channels='n_mels',
                sampling_rate='sample_rate', normalize='normalized', power='power', norm='norm', center='center')
DEFAULTS = dict(filter_length=1024, hop_length=256, win_length=1024, n_mel_channels=100, sampling_rate=24000, normalize=False, power=1,
                norm=None, center=True)


def case_wave(c):
    g = torch.Generator().manual_seed(c['seed'])
    wave = torch.randn((c['B'], c['nw']), generator=g) * 0.3
    wave[:, :c['nw'] // 3] *= 1e-3
    return wave


def settings(kw):
    """the MelSpec kwargs with the reference's defaults filled in"""
    s = dict(DEFAULTS, **kw)
    if s['win_length'] is None:
        s['win_length'] = s['filter_length']
    return s


def norm_scale(window, normalize, n_fft):
    """float64 scale of X: 1, 1/sqrt(sum window^2) (True, 'window') or 1/sqrt(n_fft) ('frame_length')"""
    if normalize is False:
        return 1.0
    if normalize == 'frame_length':
        return n_fft ** -0.5
    return float(h64(window).square().sum().rsqrt())


def frame_matrix(wave64, n_fft, hop, center):
    if center:
        pad = n_fft // 2
        wave64 = F.pad(wave64[:, None], (pad, pad), mode='reflect')[:, 0]
    return wave64.unfold(-1, n_fft, hop)                  # [B, frames, n_fft]


def padded_window(window64, n_fft):
    left = (n_fft - window64.shape[0]) // 2
    return F.pad(window64, (left, n_fft - window64.shape[0] - left))


def radices(n):
    """the stages of the kernels' FFT: log2(n) radix-2 stages for a power of two, else the Stockham order 4s, a 2, 3s, 5s"""
    if n & (n - 1) == 0:
        return [2] * int(math.log2(n))
    r = []
    while n % 4 == 0:
        r.append(4)
        n //= 4
    for p in (2, 3, 5):
        while n % p == 0:
            r.append(p)
            n //= p
    assert n == 1
    return r


def mel64(wave, window, fb, n_fft, hop, center=True, power=1.0, scale=1.0, bound=False, kernel_scale=None):
    """float64 log-mel [B, n_mels, frames] of the fp32 wave, window [win_length] and filterbank the kernel received, and, with bound,
    its element-wise bound for the kernels of csrc/small.cu (`kernel_scale`: the fp32 scale the kernel got, default fp32(scale)).

    Frame: x_n = wave_j window_(n - off) inside the window, 0 outside; the fp32 product rounds once (u |x_n|).
    FFT: every stage of radix R turns its inputs by twiddles read from a table and combines R of them with a fixed R-point DFT.
        Twiddles: sincospif (1 ulp per component, |w^ - w| <= 2u) of -2k/n; for a power of two 2k/n is exact, otherwise its fp32
        quotient is off by <= u 2k/n < 2u, which turns the angle by < 2 pi u: mu = 2u, or (2 + 2 pi) u for the mixed-radix FFT.
        A turned input t = fl(w^ x) is within tau |x| of w x, tau = mu + sqrt2 gamma_2 (1 + mu) (complex product, Higham (3.5)).
        Each output component of the R-point DFT is a linear form in the 2R real components of the t_q with coefficients cos, sin of
        modulus <= 1, evaluated through at most 2R + 1 roundings (the fp32 constants count as one): within gamma_(2R+1)
        sum_q |t_q| per component (|cos||Re t| + |sin||Im t| <= |t|), sqrt2 gamma_(2R+1) sum_q |t_q| in modulus. So a stage
        adds eta_R = tau + sqrt2 gamma_(2R+1) (1 + tau) times the l1 norm of the frame samples under its output, and passes the
        errors of its inputs on with factors of modulus <= 1 + mu: element-wise, |Z^ - Z| <= (prod_s (1 + eta_s + mu) (1 + u) - 1)
        sum|x_n| (radix-2 stages: the derivation of test_gpu_conv_melspec_kernels' mel_ref gives the smaller eta = mu +
        gamma_4 (sqrt2 + mu), which is used for them).
    |.| * scale: sqrtf(re^2 + im^2) adds gamma_2 relative and 2^-70 absolute (squares below the normal range); the product with the
        fp32 scale another u plus the scale's own rounding |s^ - s| / s.
    ** power: 1 exact; 2 one fp32 product (m^2 - M^2 <= (2M + e) e, plus u (M + e)^2); otherwise powf, 4 ulp (8u relative, plus
        2^-100 absolute for results in the subnormal range) after |m^p - M^p| <= p (M + e)^(p-1) e (p >= 1), or, for p < 1,
        min(e^p, p (M - e)^(p-1) e) (x^p is subadditive; its slope is largest at the lower end).
    Filter: acc = sum over the filter's band (hi - lo bins) of P_k fb_km: gamma(hi - lo) sum fb (P + e_P) + sum fb e_P.
    log: |log max(a, c) - log max(b, c)| <= |a - b| / max(min(a, b), c), with min(a, b) >= mel - e_mel; logf adds 1 ulp
        (<= 2u of the result). c = 1e-5f, the kernel's clamp."""
    w64 = padded_window(h64(window), n_fft)
    xw = frame_matrix(h64(wave), n_fft, hop, center) * w64
    Z = torch.fft.rfft(xw, dim=-1)
    M = Z.abs() * scale
    P = M if power == 1 else M ** power
    fb64 = h64(fb)
    mel = P @ fb64
    ref = mel.clamp(min=LOG_FLOOR).log()
    if not bound:
        return ref.transpose(1, 2)
    rad = radices(n_fft)
    pow2 = n_fft & (n_fft - 1) == 0
    mu = 2 * U if pow2 else (2 + 2 * math.pi) * U
    growth = 1.0
    for R in rad:
        if pow2:
            eta = mu + gamma(4) * (math.sqrt(2) + mu)
        else:
            tau = mu + math.sqrt(2) * gamma(2) * (1 + mu)
            eta = tau + math.sqrt(2) * gamma(2 * R + 1) * (1 + tau)
        growth *= 1 + eta + (0 if pow2 else mu)
    if pow2:   # mel_ref's form for the radix-2 FFT: (L eta + u) / (1 - L eta - u)
        L = len(rad)
        rel = (L * eta + U) / (1 - L * eta - U)
    else:
        rel = growth * (1 + U) - 1
    e_F = rel * xw.abs().sum(-1, keepdim=True)
    absZ = Z.abs()
    e_abs = e_F + gamma(2) * (absZ + e_F) + 2.0 ** -70
    s32 = float(torch.tensor(scale, dtype=torch.float32)) if kernel_scale is None else kernel_scale
    rs = abs(s32 - scale) / scale
    e_M = scale * e_abs + (rs + U + rs * U) * scale * (absZ + e_abs) if scale != 1.0 or s32 != 1.0 else e_abs
    if power == 1:
        e_P = e_M
    elif power == 2:
        e_P = (2 * M + e_M) * e_M + U * (M + e_M) ** 2
    else:
        if power > 1:
            e_pow = power * (M + e_M) ** (power - 1) * e_M
        else:
            lo = (M - e_M).clamp(min=0)
            slope = torch.where(lo > 0, power * lo.clamp(min=1e-300) ** (power - 1) * e_M, torch.full_like(lo, math.inf))
            e_pow = torch.minimum(e_M ** power, slope)
        e_P = e_pow + 8 * U * (M + e_M) ** power + 2.0 ** -100
    nz = fb64 != 0
    k = torch.arange(fb64.shape[0], dtype=F64)[:, None]
    band = torch.where(nz.any(0), (k * nz).max(0).values - torch.where(nz, k, math.inf).min(0).values + 1, 0.0)
    e_mel = gamma(band) * ((P + e_P) @ fb64.abs()) + e_P @ fb64.abs()
    e_log = e_mel / (mel - e_mel).clamp(min=LOG_FLOOR)
    out_bound = e_log + 2 * U * (ref.abs() + e_log)
    return ref.transpose(1, 2), out_bound.transpose(1, 2)


def mel_of_module(ms, wave, bound=False):
    """mel64 with the buffers and settings of a MelSpec module of this package"""
    st = ms.mel_stft
    return mel64(wave, st.spectrogram.window.cpu(), st.mel_scale.fb.cpu(), ms.n_fft, ms.hop, center=ms.center, power=ms.power,
                 scale=ms.norm_scale, bound=bound)
