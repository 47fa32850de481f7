"""Element-wise float64 bounds for the depthwise convolution and mel-spectrogram kernels (csrc/small.cu).

Method of tests/test_gpu_leaf_kernels.py: b200_dwconv_fwd / b200_dwconv_bwd and b200_melspec are called through the C ABI with
NaN-prefilled outputs (dweight / dbias are the exception: the header says they are ADDED into caller buffers, so they start from
random values here), and every output is compared element by element with a float64 restatement computed on the host from the
exact bf16 / fp32 tensors the kernel received. Every bound is E (bit-identical), F (fp32, derived in the helper's docstring) or
B (one bf16 rounding of an F value, check_b). Figures for functions and instructions (CUDA C++ Programming Guide, appendix
"Mathematical Functions"): __expf 2 + floor(1.173 |x|) ulp, __fdividef 2 ulp, sincospif 1 ulp per component, logf 1 ulp;
sqrtf, + - * correctly rounded. A sum of n terms in any order (FMA chains, shared-memory and global atomics) is within
gamma(n) sum|terms| of the exact sum (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., (3.4)-(3.5)).
Every case asserts which side of each launch threshold it is on, from the launch rules of small.cu restated below.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from hyper_conv_ref import CV_TN, cdiv, corr, dw_mask, dw_ref, model_mask
from kernel_checks import F32, F64, BF16, U, check_b, check_e, check_f, dev, gamma, gen, h64, nans, pkg, stream
from oracle import e2tts_oracle as O

pytestmark = pytest.mark.gpu


# ======================================================================================================== depthwise conv
CV_TC, CV_FWD_TILES, CV_BWD_TILES = 64, 2, 4   # channel tile, tiles per forward / backward block (token tile: CV_TN)


def dw_geometry(Np, D):
    """the launch of b200_dwconv_fwd / _bwd: grid (token blocks, channel tiles, B); a forward block marches CV_FWD_TILES token tiles,
    a backward block CV_BWD_TILES. -> (tiles of the last forward block, of the last backward block, tokens of the last tile,
    channel pairs of the last channel tile)"""
    ntiles = cdiv(Np, CV_TN)
    fwd_blocks, bwd_blocks, ctiles = cdiv(ntiles, CV_FWD_TILES), cdiv(ntiles, CV_BWD_TILES), cdiv(D, CV_TC)
    return (ntiles - CV_FWD_TILES * (fwd_blocks - 1), ntiles - CV_BWD_TILES * (bwd_blocks - 1), Np - CV_TN * (ntiles - 1),
            (D - CV_TC * (ctiles - 1)) // 2)


def dw_launch_fwd(pkg, x, mask, w, b, with_pre=True):
    B, Np, D = x.shape
    y, pre = nans((B, Np, D), BF16), (nans((B, Np, D), BF16) if with_pre else None)
    a = pkg.lib.make_args('b200_dwconv_args', x=x, mask=mask, weight=w, bias=b, y=y, B=B, Np=Np, D=D, ksize=w.shape[1], pre=pre)
    pkg.lib.call('b200_dwconv_fwd', a, stream())
    return y, pre


def dw_launch_bwd(pkg, x, mask, w, b, dy, pre, dw0, db0):
    B, Np, D = x.shape
    dx, dw, db = nans((B, Np, D), BF16), dw0.clone(), db0.clone()
    a = pkg.lib.make_args('b200_dwconv_args', x=x, mask=mask, weight=w, bias=b, dy=dy, dx=dx, dweight=dw, dbias=db, B=B, Np=Np, D=D,
                          ksize=w.shape[1], pre=pre)
    pkg.lib.call('b200_dwconv_bwd', a, stream())
    return dx, dw, db


def check_dwconv(pkg, B, Np, D, ks, masks, seed, scale=1.0, poison=False, chans=None, tag=''):
    """one forward and one backward launch, every output against dw_ref; masks None = the null mask pointer (every token valid).
    chans: the channels compared against float64 (all when None); every element is checked finite and masked rows +0 regardless.
    poison: x, dy and the saved pre hold NaN on masked rows (the kernel selects valid rows, it does not multiply by the mask)."""
    g = gen(seed)
    m = torch.ones(B, Np, dtype=torch.bool) if masks is None else torch.stack([dw_mask(Np, s, g) for s in masks])
    x = (torch.randn(B, Np, D, generator=g) * scale).to(BF16)
    w = torch.randn(D, ks, generator=g) * (1.0 / math.sqrt(ks)) + 0.1 * torch.arange(ks) / ks    # asymmetric taps: a flip shows
    b = torch.randn(D, generator=g) * 0.5
    dy = torch.randn(B, Np, D, generator=g).to(BF16)
    dw0, db0 = torch.randn(D, ks, generator=g), torch.randn(D, generator=g)
    bad = ~m[..., None]
    if poison:
        assert bool(bad.any())
        x, dy = x.masked_fill(bad, float('nan')), dy.masked_fill(bad, float('nan'))
    mask_d = None if masks is None else m.to(torch.uint8).to(dev())
    xd, wd, bd, dyd = x.to(dev()), w.to(dev()), b.to(dev()), dy.to(dev())
    y, pre = dw_launch_fwd(pkg, xd, mask_d, wd, bd)
    pre_in = pre.masked_fill(bad.to(dev()), float('nan')) if poison else pre
    dx, dw, db = dw_launch_bwd(pkg, xd, mask_d, wd, bd, dyd, pre_in, dw0.to(dev()), db0.to(dev()))
    torch.cuda.synchronize()
    for nm, t in (('y', y), ('pre', pre), ('dx', dx), ('dweight', dw), ('dbias', db)):
        assert bool(torch.isfinite(t).all()), f'{tag}{nm}: non-finite elements (never written, or NaN read from a masked row)'
    bad_d = bad.expand(B, Np, D).to(dev())
    for nm, t in (('y', y), ('dx', dx)):       # masked rows are +0 in every channel
        bits = t.view(torch.int16)[bad_d]
        assert bool((bits == 0).all()), f'{tag}{nm}: {int((bits != 0).sum())} masked elements are not +0'
    c = torch.arange(D) if chans is None else chans
    r = dw_ref(h64(x[..., c]), m, h64(w[c]), h64(b[c]), h64(dy[..., c]), h64(pre[..., c]))
    check_b(f'{tag}pre', pre.cpu()[..., c], r['conv'], r['e_pre'])
    mm = m[..., None].expand(B, Np, len(c))
    check_b(f'{tag}y', y.cpu()[..., c][mm], r['y'][mm], r['e_y'][mm])
    check_b(f'{tag}dx', dx.cpu()[..., c][mm], r['dx'][mm], r['e_dx'][mm])
    n = B * cdiv(Np, CV_TN) * CV_TN + 1
    check_f(f'{tag}dweight', dw.cpu()[c], h64(dw0[c]) + r['dW'], gamma(n) * (r['dWabs'] + h64(dw0[c]).abs()) + r['dWcar'])
    check_f(f'{tag}dbias', db.cpu()[c], h64(db0[c]) + r['db'], gamma(n) * (r['dbabs'] + h64(db0[c]).abs()) + r['dbcar'])
    return dict(m=m, x=x, w=w, b=b, dy=dy, y=y, pre=pre, dx=dx, r=r)


# name, B, Np, D, ksize, per-row masks (None: null mask pointer), x scale, poison, channel subset,
# expected (tiles of the last forward block, of the last backward block, tokens of the last tile, pairs of the last channel tile)
DW_CASES = [
    ('np1-null', 2, 1, 72, 31, None, 1.0, False, False, (1, 1, 1, 4)),
    ('np15-holes', 3, 15, 8, 31, ['holes', 'all', 7], 1.0, False, False, (1, 1, 15, 4)),
    ('np40-k7', 2, 40, 264, 7, ['all', 28], 1.0, False, False, (1, 1, 40, 4)),
    ('np64-k3-null', 2, 64, 128, 3, None, 1.0, False, False, (1, 1, 64, 32)),
    ('np65-edges', 3, 65, 72, 31, [63, 64, 65], 1.0, False, False, (2, 2, 1, 4)),
    ('np128-rows', 4, 128, 264, 31, [63, 64, 65, 'none'], 1.0, False, False, (2, 2, 64, 4)),
    ('np192-k1', 2, 192, 512, 1, ['holes', 150], 1.0, False, False, (1, 3, 64, 32)),
    ('np257-k5', 2, 257, 136, 5, ['holes', 256], 1.0, False, False, (1, 1, 1, 4)),
    ('np320-null', 1, 320, 1024, 31, None, 1.0, False, False, (1, 1, 64, 32)),
    ('np449-rows', 4, 449, 72, 31, ['all', 'holes', 'none', 300], 1.0, False, False, (2, 4, 1, 4)),
    ('saturated', 2, 130, 72, 31, ['holes', 100], 40.0, False, False, (1, 3, 2, 4)),
    ('poisoned', 3, 200, 136, 31, ['holes', 150, 'none'], 1.0, True, False, (2, 4, 8, 4)),
    ('cfg2-audio', 16, 1056, 512, 31, 'model', 1.0, False, True, (1, 1, 32, 32)),
    ('cfg2-text', 16, 1056, 256, 31, 'model', 1.0, False, True, (1, 1, 32, 32)),
    ('cfg3', 4, 2080, 1024, 31, 'model', 1.0, False, True, (1, 1, 32, 32)),
    # model widths off the powers of two (3, 6, 12 channel tiles) with the short kernels of Transformer(kernel_size=...)
    ('d192-k7', 2, 300, 192, 7, ['holes', 250], 1.0, False, False, (1, 1, 44, 32)),
    ('d384-k1-model', 2, 1056, 384, 1, 'model', 1.0, False, False, (1, 1, 32, 32)),
    ('d768-k7', 3, 130, 768, 7, [100, 'holes', 'all'], 1.0, False, False, (1, 3, 2, 32)),
    ('d768-k1', 2, 65, 768, 1, [64, 'holes'], 1.0, False, False, (2, 2, 1, 32)),
]


def test_dw_cases_reach_every_edge():
    """the case list covers both forward block ends, every backward block end, partial / exact / one-token last tiles, a last
    channel tile of 4 pairs, Np < 16 (every window overruns both ends), every kernel size class and every mask kind"""
    geo = [dw_geometry(Np, D) for _, _, Np, D, *_ in DW_CASES]
    assert {g[0] for g in geo} == {1, 2} and {g[1] for g in geo} == {1, 2, 3, 4}
    assert {1, 64} <= {g[2] for g in geo} and any(1 < g[2] < 64 for g in geo) and 4 in {g[3] for g in geo}
    assert any(c[2] < 16 for c in DW_CASES) and {1, 3, 5, 7, 31} <= {c[4] for c in DW_CASES}
    specs = [s for c in DW_CASES if isinstance(c[5], list) for s in c[5]]
    assert None in [c[5] for c in DW_CASES] and {'all', 'none', 'holes', 63, 64, 65} <= set(specs)


@pytest.mark.parametrize('name,B,Np,D,ks,masks,scale,poison,subset,geo', DW_CASES, ids=[c[0] for c in DW_CASES])
def test_dwconv_kernels(pkg, name, B, Np, D, ks, masks, scale, poison, subset, geo):
    assert dw_geometry(Np, D) == geo
    seed = sum(map(ord, name))
    if masks == 'model':
        masks = model_mask(B, Np, gen(seed + 1))
    chans = None
    if subset:      # first, a middle and the last channel tile
        mid = (cdiv(D, CV_TC) // 2) * CV_TC
        chans = torch.cat([torch.arange(0, 64), torch.arange(mid, mid + 64), torch.arange(D - 64, D)]).unique()
    out = check_dwconv(pkg, B, Np, D, ks, masks, seed=seed, scale=scale, poison=poison, chans=chans, tag=f'{name} ')
    if name == 'saturated':
        pre = h64(out['pre'])[out['m']]
        assert bool((pre > 88).any()) and bool((pre < -88).any()) and float(pre.abs().max()) >= 100


def test_dwconv_reference_matches_autograd():
    """dw_ref's formulas (the flipped convolution for dx, tap sums for dW) against float64 autograd of O.depthwise_conv"""
    g = gen(3)
    B, Np, D, ks = 2, 50, 16, 7
    x = torch.randn(B, Np, D, generator=g, dtype=F64)
    m = torch.stack([dw_mask(Np, 'holes', g), dw_mask(Np, 40, g)])
    w, b = torch.randn(D, ks, generator=g, dtype=F64), torch.randn(D, generator=g, dtype=F64)
    dy = torch.randn(B, Np, D, generator=g, dtype=F64)
    xr, wr, br = x.clone().requires_grad_(), w[:, None].clone().requires_grad_(), b.clone().requires_grad_()
    yr = O.depthwise_conv({'c.dw_conv1d.0.weight': wr, 'c.dw_conv1d.0.bias': br}, 'c', xr, m.to(F64))
    gx, gw, gb = torch.autograd.grad(yr, [xr, wr, br], dy)
    r = dw_ref(x, m, w, b, dy, corr(x * m[..., None], w) + b)
    for nm, got, want in (('y', r['y'], yr), ('dx', r['dx'] * m[..., None], gx), ('dW', r['dW'], gw[:, 0]), ('db', r['db'], gb)):
        check_f(nm, got, want.detach(), 1e-12 * (1 + want.detach().abs()))


def test_dwconv_bit_exact_properties(pkg):
    """pre = NULL (the no-grad path) gives the same y; each batch element launched alone (B = 1) reproduces its slice of y, pre
    and dx of the batched launch"""
    B, Np, D, ks = 3, 300, 136, 31
    out = check_dwconv(pkg, B, Np, D, ks, ['holes', 200, 'all'], seed=11, tag='batched ')
    m = out['m'].to(torch.uint8).to(dev())
    xd, wd, bd, dyd = out['x'].to(dev()), out['w'].to(dev()), out['b'].to(dev()), out['dy'].to(dev())
    y0, none = dw_launch_fwd(pkg, xd, m, wd, bd, with_pre=False)
    assert none is None
    check_e('y without pre', y0, out['y'])
    for i in range(B):
        yi, pi = dw_launch_fwd(pkg, xd[i:i + 1].contiguous(), m[i:i + 1].contiguous(), wd, bd)
        dxi, _, _ = dw_launch_bwd(pkg, xd[i:i + 1].contiguous(), m[i:i + 1].contiguous(), wd, bd, dyd[i:i + 1].contiguous(), pi,
                                  torch.zeros(D, ks, device=dev()), torch.zeros(D, device=dev()))
        check_e(f'y[{i}] alone', yi[0], out['y'][i])
        check_e(f'pre[{i}] alone', pi[0], out['pre'][i])
        check_e(f'dx[{i}] alone', dxi[0], out['dx'][i])


# ======================================================================================================== MelSpec
def mel_geometry(n_fft, hop, n_mels, nw):
    """melspec_kernel runs one 256-thread block per (frame, batch item): passes per thread of the load / twiddle loop
    (n_fft samples), of each butterfly stage (n_fft/2 pairs) and of the mel loop; frames = 1 + nw/hop; and the frames whose window
    reflects at both ends of the wave (j = f hop + n - n_fft/2 below 0 and at or past nw for some n)"""
    pad = n_fft // 2
    frames = 1 + nw // hop
    both = sum(1 for f in range(frames) if f * hop - pad < 0 and f * hop + pad - 1 >= nw)
    return cdiv(n_fft, 256), cdiv(n_fft // 2, 256), cdiv(n_mels, 256), frames, both


LOG_FLOOR = float(np.float32(1e-5))   # the kernel's clamp 1e-5f


def mel_launch(pkg, wave, window, fb, n_fft, hop, lens=None, out_bnd=False):
    """b200_melspec with a NaN-filled output; returns [B, n_mels, frames] whatever the layout"""
    B, nw = wave.shape
    n_mels, frames = fb.shape[1], 1 + nw // hop
    out = nans((B, frames, n_mels) if out_bnd else (B, n_mels, frames), F32)
    bands = torch.empty(2 * n_mels, device=dev(), dtype=torch.int32)
    pkg.lib.call('b200_melspec', wave, window, fb, out, B, nw, n_fft, hop, n_mels, bands, lens, int(out_bnd), stream())
    return out.transpose(1, 2) if out_bnd else out


def mel_ref(wave, window, fb, n_fft, hop):
    """float64 log-mel of the fp32 wave, window and filterbank the kernel received, and its element-wise bound.

    Frame: reflect padding by n_fft/2, x_n = wave_j window_n; the kernel's fp32 product rounds once (u |x_n|).
    FFT: a radix-2 FFT whose twiddles err by mu (sincospif: 1 ulp per component, so |w^ - w| <= 2u) is, element-wise, within
        ((1 + eta)^L - 1) sum|x_n| <= L eta / (1 - L eta) sum|x_n| of the exact DFT, L = log2(n_fft), eta = mu + gamma_4 (sqrt2 + mu)
        (Higham (24.5)): every butterfly output gains <= eta times the l1 norm of the inputs feeding it, and errors pass the later
        stages with factors of modulus <= 1 + eta. With the product rounding: e_F = (L eta + u) / (1 - L eta - u) sum|x_n|.
    |.|: sqrtf(re^2 + im^2) adds gamma_2 relative (two roundings in the sum of squares, halved by the square root, plus the
        correctly rounded sqrtf) and 2^-70 absolute for squares below the normal range.
    Filter: acc = sum over the filter's band (hi - lo bins) of mag_k fb_km: gamma(hi - lo) sum fb (|Z| + e_mag) + sum fb e_mag.
    log: |log max(a, c) - log max(b, c)| <= |a - b| / max(min(a, b), c), with min(a, b) >= mel - e_mel; logf adds 1 ulp
        (<= 2u of the result). c = 1e-5f, the kernel's clamp."""
    w64 = h64(wave)
    pad = n_fft // 2
    frames = F.pad(w64[:, None], (pad, pad), mode='reflect')[:, 0].unfold(-1, n_fft, hop)   # [B, frames, n_fft]
    xw = frames * h64(window)
    Z = torch.fft.rfft(xw, dim=-1)
    mag = Z.abs()
    L = int(math.log2(n_fft))
    mu = 2 * U
    eta = mu + gamma(4) * (math.sqrt(2) + mu)
    e_F = (L * eta + U) / (1 - L * eta - U) * xw.abs().sum(-1, keepdim=True)
    e_mag = e_F + gamma(2) * (mag + e_F) + 2.0 ** -70
    fb64 = h64(fb)
    nz = fb64 != 0
    k = torch.arange(fb64.shape[0], dtype=F64)[:, None]
    band = torch.where(nz.any(0), (k * nz).max(0).values - torch.where(nz, k, math.inf).min(0).values + 1, 0.0)
    mel = mag @ fb64
    e_mel = gamma(band) * ((mag + e_mag) @ fb64) + e_mag @ fb64
    ref = mel.clamp(min=LOG_FLOOR).log()
    e_log = e_mel / (mel - e_mel).clamp(min=LOG_FLOOR)
    bound = e_log + 2 * U * (ref.abs() + e_log)
    return ref.transpose(1, 2), bound.transpose(1, 2)


def mel_inputs(n_fft, n_mels, B, nw, seed, zero=False):
    """a wave of B items at 0.3 rms whose first third is 1e-6 quieter (so the log-mel also sits below the 1e-5 clamp), the
    periodic Hann window and the HTK filterbank of MelSpec at 24 kHz"""
    g = gen(seed)
    wave = torch.randn(B, nw, generator=g) * 0.3
    wave[:, :nw // 3] *= 1e-6
    if zero:
        wave.zero_()
    window = torch.hann_window(n_fft, periodic=True)
    fb = O.mel_filterbank(n_fft // 2 + 1, n_mels, 24000)
    return wave, window, fb


def check_mel(pkg, n_fft, hop, n_mels, nw, B, out_bnd, seed, zero=False, tag=''):
    wave, window, fb = mel_inputs(n_fft, n_mels, B, nw, seed, zero)
    got = mel_launch(pkg, wave.to(dev()), window.to(dev()), fb.to(dev()), n_fft, hop, out_bnd=out_bnd)
    torch.cuda.synchronize()
    ref, bound = mel_ref(wave, window, fb, n_fft, hop)
    check_f(f'{tag}log-mel', got, ref, bound)
    return got.cpu(), fb


def floor_value():
    """logf(1e-5f) on the device: what the kernel writes where the filter sum is below the clamp"""
    return torch.log(torch.tensor([LOG_FLOOR], device=dev(), dtype=F32)).cpu()


# n_fft, hop, n_mels, nw, B, out_bnd, expected (load passes, butterfly passes, mel passes)
MEL_CASES = [
    (64, 1, 100, 33, 2, False, (1, 1, 1)),          # nw = n_fft/2 + 1, threads >= 64 idle in the load loop, empty filters
    (64, 100, 1, 1000, 2, True, (1, 1, 1)),
    (256, 1, 300, 129, 1, True, (1, 1, 2)),         # nw = n_fft/2 + 1, two mel passes
    (256, 100, 300, 1999, 2, False, (1, 1, 2)),     # nw = 20 hop - 1
    (1024, 256, 100, 513, 2, True, (4, 2, 1)),      # nw = n_fft/2 + 1
    (1024, 256, 100, 256 * 16, 2, False, (4, 2, 1)),
    (1024, 1024, 300, 1024 * 5 - 1, 2, True, (4, 2, 2)),
    (4096, 4096, 100, 4096 * 3, 1, False, (16, 8, 1)),
    (4096, 100, 1, 2049, 1, True, (16, 8, 1)),      # nw = n_fft/2 + 1
    (4096, 1, 100, 2049, 1, False, (16, 8, 1)),
    (4096, 256, 300, 256 * 20 - 1, 2, True, (16, 8, 2)),
]


@pytest.mark.parametrize('n_fft,hop,n_mels,nw,B,out_bnd,geo', MEL_CASES,
                         ids=[f'nfft{c[0]}-hop{c[1]}-mels{c[2]}-nw{c[3]}-{"bnd" if c[5] else "bmn"}' for c in MEL_CASES])
def test_melspec_kernel(pkg, n_fft, hop, n_mels, nw, B, out_bnd, geo):
    load, fly, mels, frames, both = mel_geometry(n_fft, hop, n_mels, nw)
    assert (load, fly, mels) == geo
    if nw == n_fft // 2 + 1 and hop < n_fft // 2 - 1:
        assert both > 0
    got, fb = check_mel(pkg, n_fft, hop, n_mels, nw, B, out_bnd, seed=n_fft + hop + n_mels + nw)
    assert got.shape == (B, n_mels, frames)
    empty = (fb == 0).all(0)
    if bool(empty.any()):
        v = got[:, empty]
        check_e('empty filters', v, floor_value().expand_as(v))


def test_melspec_cases_reach_every_edge():
    """n_fft below 256 and at 4096, hop 1 and hop = n_fft, 1 / 100 / 300 mels, empty filters, nw = n_fft/2 + 1 with frames that
    reflect at both ends, nw = k hop and k hop - 1, both layouts"""
    assert {c[0] for c in MEL_CASES} == {64, 256, 1024, 4096} and {1, 100, 256} <= {c[1] for c in MEL_CASES}
    assert any(c[1] == c[0] for c in MEL_CASES) and {c[2] for c in MEL_CASES} == {1, 100, 300}
    assert any(bool((O.mel_filterbank(c[0] // 2 + 1, c[2], 24000) == 0).all(0).any()) for c in MEL_CASES)
    assert any(c[3] == c[0] // 2 + 1 and mel_geometry(*c[:4])[4] > 0 for c in MEL_CASES)
    assert any(c[3] % c[1] == 0 for c in MEL_CASES) and any(c[3] % c[1] == c[1] - 1 for c in MEL_CASES)
    assert {c[5] for c in MEL_CASES} == {False, True}


def test_melspec_reference_settings(pkg):
    """the float64 restatement agrees with the oracle's torchaudio-pinned O.melspec at the model's settings (to a tenth of the
    kernel's bound), and the kernel is
    within its bound there; an all-zero wave gives logf(1e-5f) everywhere"""
    wave, window, fb = mel_inputs(1024, 100, 2, 256 * 40, seed=5)
    ref, bound = mel_ref(wave, window, fb, 1024, 256)
    want = O.melspec(wave.double())
    check_f('restatement vs O.melspec', ref, want, bound / 10)   # they differ only in the window: float64 there, fp32 here
    got = mel_launch(pkg, wave.to(dev()), window.to(dev()), fb.to(dev()), 1024, 256)
    check_f('log-mel', got, ref, bound)
    got0, _ = check_mel(pkg, 1024, 256, 100, 4096, 2, False, seed=6, zero=True, tag='zero wave ')
    check_e('zero wave', got0, floor_value().expand_as(got0))


def test_melspec_ragged_batch(pkg):
    """wave_lens: items of <= n_fft/2 samples give zero frames, others 1 + len/hop frames bit-identical to the item launched alone
    without wave_lens, then +0; a length past nw_max clamps to it. Both layouts."""
    n_fft, hop, n_mels, nw_max = 1024, 256, 100, 256 * 20
    lens = [300, 512, 513, 256 * 7 - 1, nw_max, 9999]
    wave, window, fb = mel_inputs(n_fft, n_mels, len(lens), nw_max, seed=8)
    for i, n in enumerate(lens):
        wave[i, min(n, nw_max):] = 0        # the collate's zero padding
    wd, wnd, fbd = wave.to(dev()), window.to(dev()), fb.to(dev())
    ld = torch.tensor(lens, dtype=torch.int32, device=dev())
    for bnd in (False, True):
        got = mel_launch(pkg, wd, wnd, fbd, n_fft, hop, lens=ld, out_bnd=bnd).cpu()
        for i, n in enumerate(lens):
            n = min(n, nw_max)
            if n <= n_fft // 2:
                check_e(f'item {i} (len {n}) bnd={bnd}', got[i], torch.zeros_like(got[i]))
                continue
            alone = mel_launch(pkg, wd[i:i + 1, :n].contiguous(), wnd, fbd, n_fft, hop, out_bnd=bnd).cpu()
            fi = 1 + n // hop
            check_e(f'item {i} (len {n}) bnd={bnd}', got[i, :, :fi], alone[0])
            check_e(f'item {i} (len {n}) padding bnd={bnd}', got[i, :, fi:], torch.zeros_like(got[i, :, fi:]))
            if not bnd:
                ref, bound = mel_ref(wave[i:i + 1, :n], window, fb, n_fft, hop)
                check_f(f'item {i} (len {n})', alone, ref, bound)


def test_melspec_collate_short_items(pkg):
    """MelSpec.collate reports 0 frames for an item of <= n_fft/2 samples (its mel rows are +0) and clamps lengths past the
    padded wave, so mel_lengths always match what the kernel wrote"""
    ms = pkg.MelSpec().to(dev())
    g = gen(9)
    waves = [torch.randn(n, generator=g) * 0.3 for n in (400, 512, 513, 256 * 12)]
    batch = ms.collate(waves)
    assert batch['mel_lengths'].tolist() == [0, 0, 3, 13]
    check_e('short items', batch['mel'][:2].cpu(), torch.zeros_like(batch['mel'][:2].cpu()))
    padded = torch.zeros(2, 3000)
    padded[0, :400], padded[1] = waves[0][:400], torch.randn(3000, generator=g)
    b2 = ms.collate(padded.to(dev()), lens=torch.tensor([400, 99999]))
    assert b2['mel_lengths'].tolist() == [0, 1 + 3000 // 256]
