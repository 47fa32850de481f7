"""Vocos decoder kernels (include/b200_e2tts.h: b200_vocos_im2col, b200_vocos_dwconv_ln / b200_vocos_ln, b200_gemm act=1,
b200_vocos_istft) against float64 restatements with element-wise bounds, the whole decode against the fp32 restatement of
tests/vocos_ref.py, and E2TTS.sample() with a loaded Vocos. Outputs start NaN-filled, so an element a kernel never writes fails."""
import copy
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import vocos_ref as V  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0') if torch.cuda.is_available() else None


@pytest.fixture(scope='module')
def pkg():
    import e2_tts_pytorch_b200 as pkg
    return pkg


def nans(*shape, dtype=torch.float32):
    return torch.full(shape, float('nan'), device=DEV, dtype=dtype)


def call(pkg, name, *args):
    pkg.lib.call(name, *args, torch.cuda.current_stream().cuda_stream)


def check(name, got, ref, bound):
    got, ref = got.double().cpu(), ref.double().cpu()
    err = (got - ref).abs()
    ok = torch.isfinite(got) & (err <= bound)
    worst = float((err / bound).nan_to_num(1e30).max())
    print(f'{name}: max err/bound {worst:.3f}, max err {float(err.max()):.3e}')
    assert bool(ok.all()), f'{name}: {int((~ok).sum())} elements out of bound (worst err/bound {worst:.3f})'


def bf(t):
    return t.to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------------------------ im2col


@pytest.mark.parametrize('db', [0, 1])
def test_im2col_bit_exact(pkg, db):
    g = torch.Generator().manual_seed(1)
    B, T, C = 3, 40, 100
    lens = torch.tensor([40, 1, 6], dtype=torch.int32)
    mel = torch.randn(B, T, C, generator=g) * 4
    lda = 704
    out = nans(B * T, lda, dtype=torch.bfloat16)
    call(pkg, 'b200_vocos_im2col', mel.to(DEV), lens.to(DEV), out, B, T, C, lda, db)
    src = torch.pow(10., mel.double() * 0.05).float() if db else mel
    want = torch.zeros(B, T, lda)
    for b in range(B):
        L = int(lens[b])
        for t in range(L):
            for j in range(7):
                s = t + j - 3
                if 0 <= s < L:
                    want[b, t, torch.arange(C) * 7 + j] = src[b, s]
    assert torch.equal(out.cpu().view(B, T, lda).float(), bf(want).float())


# ------------------------------------------------------------------------------------------------------------------ LayerNorm


def ln_ref(x, lens, w, b, eps, cw=None, cb=None):
    """float64: masked depthwise k-7 conv (zero padding at each item's end) + bias, then LayerNorm; padded rows 0"""
    B, T, D = x.shape
    out = torch.zeros(B, T, D, dtype=torch.float64)
    for i in range(B):
        L = int(lens[i])
        h = x[i, :L].double()
        if cw is not None:
            h = F.conv1d(h.t()[None], cw.double().view(D, 1, 7), cb.double(), padding=3, groups=D)[0].t()
        out[i, :L] = F.layer_norm(h, (D,), w.double(), b.double(), eps)
    return out


def run_ln(pkg, x, lens, w, b, eps, cw=None, cb=None):
    B, T, D = x.shape
    y = nans(B * T, D, dtype=torch.bfloat16)
    a = pkg.lib.make_args('b200_vocos_ln_args', x=x, lens=lens, conv_w=cw, conv_b=cb, ln_w=w, ln_b=b, y=y, B=B, T=T, D=D, eps=eps)
    call(pkg, 'b200_vocos_dwconv_ln' if cw is not None else 'b200_vocos_ln', a)
    return y.view(B, T, D)


@pytest.mark.parametrize('D', [64, 384, 512, 768, 1024])
@pytest.mark.parametrize('conv', [True, False])
def test_layernorm(pkg, D, conv):
    g = torch.Generator().manual_seed(D + conv)
    lens = torch.tensor([1, 2, 3, 6, 7, 63, 64, 65, 2048], dtype=torch.int32)
    B, T = len(lens), 2048
    x = bf(torch.randn(B, T, D, generator=g) * 2 + 0.5)
    for i in range(B):          # NaN in every padded row: none may reach a valid row
        x[i, int(lens[i]):] = float('nan')
    w, b = 1 + 0.3 * torch.randn(D, generator=g), 0.2 * torch.randn(D, generator=g)
    cw, cb = (torch.randn(D, 7, generator=g) / math.sqrt(7), 0.1 * torch.randn(D, generator=g)) if conv else (None, None)
    d = lambda t: None if t is None else t.to(DEV).contiguous()  # noqa: E731
    y = run_ln(pkg, x.to(DEV), lens.to(DEV), d(w), d(b), 1e-6, d(cw), d(cb))
    ref = ln_ref(x, lens, w, b, 1e-6, cw, cb)
    check(f'ln D{D} conv{conv}', y.float(), ref, 2 ** -8 * ref.abs() + 1e-4 * (1 + w.abs().double()))
    for i in range(B):
        assert torch.equal(y[i, int(lens[i]):].float().cpu(), torch.zeros(T - int(lens[i]), D))
    # an item alone is bit-identical to the same item in the batch
    i = 5
    L = int(lens[i])
    alone = run_ln(pkg, x[i:i + 1, :L].to(DEV).contiguous(), lens[i:i + 1].to(DEV), d(w), d(b), 1e-6, d(cw), d(cb))
    assert torch.equal(alone[0], y[i, :L])


# ------------------------------------------------------------------------------------------------------------------ GELU epilogue


@pytest.mark.parametrize('force_tile', [0, 1, 2, 3])
@pytest.mark.parametrize('M,N,K', [(200, 1536, 512), (1000, 328, 136), (37, 72, 64), (513, 264, 704)])
def test_gemm_gelu_epilogue(pkg, force_tile, M, N, K):
    g = torch.Generator().manual_seed(M + N + K + force_tile)
    A, W = bf(torch.randn(M, K, generator=g)), bf(torch.randn(N, K, generator=g) / math.sqrt(K))
    bias = 0.5 * torch.randn(N, generator=g)
    out = nans(M, (N + 7) // 8 * 8, dtype=torch.bfloat16)
    pkg.ops.gemm(A.to(DEV), W.to(DEV), M, N, K, bias=bias.to(DEV), out=out, act=pkg.ops.ACT_GELU, force_tile=force_tile)
    z = A.double() @ W.double().t() + bias.double()
    ref = F.gelu(z)
    acc_err = K * 2 ** -23 * (A.double().abs() @ W.double().abs().t())
    check(f'gelu M{M} N{N} K{K} t{force_tile}', out[:, :N].float(), ref, 2 ** -8 * ref.abs() + 1.2 * acc_err + 1e-6)


def test_gemm_act_refusals(pkg):
    A = torch.zeros(128, 64, device=DEV, dtype=torch.bfloat16)
    W = torch.zeros(128, 64, device=DEV, dtype=torch.bfloat16)
    for kw in (dict(geglu=1), dict(split_k=2, out_fp32=True), dict(out_fp32=True), dict(a_mn=True)):
        with pytest.raises(RuntimeError, match='act'):
            pkg.ops.gemm(A, W, 128, 128, 64, act=1, **kw)


# ------------------------------------------------------------------------------------------------------------------ ISTFT


def run_istft(pkg, spec, window, lens, n_fft, hop):
    B = len(lens)
    T = spec.shape[0] // B
    frames, audio = nans(B * T, n_fft), nans(B, T * hop)
    a = pkg.lib.make_args('b200_vocos_istft_args', spec=spec, window=window, lens=lens, frames=frames, audio=audio, B=B, T=T,
                          n_fft=n_fft, hop=hop)
    call(pkg, 'b200_vocos_istft', a)
    return audio


@pytest.mark.parametrize('n_fft,hop', [(1024, 256), (512, 128), (256, 64)])
def test_istft(pkg, n_fft, hop):
    g = torch.Generator().manual_seed(n_fft)
    lens = torch.tensor([1, 2, 3, 4, 5, 257, 2048], dtype=torch.int32)
    B, T, K = len(lens), 2048, n_fft // 2 + 1
    mag = torch.rand(B * T, K, generator=g) * 12 - 6          # across the exp clip at log(100) = 4.6
    ph = (torch.rand(B * T, K, generator=g) * 2 - 1) * 50      # phases to +-50 rad
    spec = torch.cat([mag, ph], 1)
    window = torch.hann_window(n_fft)
    d_spec, d_win, d_lens = spec.to(DEV), window.to(DEV), lens.to(DEV)
    audio = run_istft(pkg, d_spec, d_win, d_lens, n_fft, hop)
    w64 = window.double()
    for b in range(B):
        L = int(lens[b])
        rows = spec[b * T:b * T + L].double()
        X = rows[:, :K].exp().clip(max=1e2) * (torch.cos(rows[:, K:]) + 1j * torch.sin(rows[:, K:]))
        ref = V.istft_same(X.t()[None], w64, n_fft, hop)[0]
        # bound: fp32 FFT of a frame (log2 n stages) and the exp / sincos roundings, relative to sum |X_k| / n per frame, through the
        # window and the envelope division
        size = (L - 1) * hop + n_fft
        s = (X.abs().sum(1) * 2 / n_fft)
        frame_scale = F.fold((s[None, :] * w64.abs()[:, None])[None], output_size=(1, size), kernel_size=(1, n_fft),
                             stride=(1, hop))[0, 0, 0]
        env = F.fold(w64.square()[None, :, None].expand(1, -1, L), output_size=(1, size), kernel_size=(1, n_fft),
                     stride=(1, hop))[0, 0, 0]
        pad = (n_fft - hop) // 2
        bound = (2 * math.log2(n_fft) + 8) * 2 ** -24 * (frame_scale / env)[pad:size - pad] + 2 ** -22 * ref.abs()
        check(f'istft {n_fft}/{hop} T{L}', audio[b, :L * hop], ref, bound)
        assert torch.equal(audio[b, L * hop:].cpu(), torch.zeros(T * hop - L * hop))
    # the sines of bins 0 and n_fft/2 are dropped (irfft): negating those phases changes only their sines. A repeat call is
    # bit-identical, and so is an item alone
    spec2 = spec.clone()
    spec2[:, K] = -spec2[:, K]
    spec2[:, 2 * K - 1] = -spec2[:, 2 * K - 1]
    assert torch.equal(run_istft(pkg, spec2.to(DEV), d_win, d_lens, n_fft, hop), audio)
    assert torch.equal(run_istft(pkg, d_spec, d_win, d_lens, n_fft, hop), audio)
    b = 5
    alone = run_istft(pkg, d_spec[b * T:(b + 1) * T].contiguous(), d_win, d_lens[b:b + 1].contiguous(), n_fft, hop)
    assert torch.equal(alone[0], audio[b])


# ------------------------------------------------------------------------------------------------------------------ whole decode


def _vocos(pkg, tmp_path, g, seed, opened):
    sd = V.write_checkpoint(str(tmp_path / 'vocos'), g, seed, opened=opened)
    return pkg.Vocos.from_pretrained(str(tmp_path / 'vocos')).to(DEV), sd


@pytest.mark.parametrize('opened', [False, True])
def test_decode_vs_fp32_oracle(pkg, tmp_path, opened):
    g = V.MEL_24KHZ
    voc, sd = _vocos(pkg, tmp_path, g, 7, opened)
    gen = torch.Generator().manual_seed(3)
    T = 300
    mel = torch.randn(2, T, 100, generator=gen) * 2 - 4
    got = voc.decode(mel.transpose(1, 2).to(DEV)).cpu()
    ref = V.decode(sd, g, mel.transpose(1, 2))
    probe = V.decode(sd, g, mel.transpose(1, 2), round_bf16=True)
    rl2 = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm())  # noqa: E731
    p, k = rl2(probe, ref), rl2(got, ref)
    print(f'decode vocos-mel-24khz opened={opened}: conditioning probe rel-L2 {p:.3e}, kernels rel-L2 {k:.3e}')
    assert p < 0.2, 'the bf16-rounded restatement is too far from fp32 for a bound derived from it'
    assert k <= 2 * p + 1e-3


def test_decode_follows_parameters_and_lifecycle(pkg, tmp_path):
    voc, sd = _vocos(pkg, tmp_path, V.SMALL, 9, True)
    mel = torch.randn(1, 100, 50, device=DEV)
    a0 = voc.decode(mel)
    assert 'pack' in voc._derived
    with torch.no_grad():
        voc.backbone.convnext[0].pwconv1.weight.mul_(1.5)
    a1 = voc.decode(mel)
    assert not torch.equal(a0, a1)
    cp = copy.deepcopy(voc)
    assert cp._derived == {}
    assert torch.equal(cp.decode(mel), a1)
    voc.to(torch.device('cpu'))
    assert voc._derived == {}


def test_decode_launches_independent_of_batch(pkg, tmp_path):
    voc, _ = _vocos(pkg, tmp_path, V.SMALL, 11, False)
    counts = []
    for B in (1, 4):
        mel = torch.randn(B, 64, 100, device=DEV)
        n0 = pkg.lib.launch_count()
        voc.decode_padded(mel, torch.full((B,), 64, dtype=torch.int32))
        counts.append(pkg.lib.launch_count() - n0)
    assert counts[0] == counts[1] == 3 * V.SMALL['num_layers'] + 8


# ------------------------------------------------------------------------------------------------------------------ E2TTS


def _e2tts(pkg, tmp_path, seed=5):
    V.write_checkpoint(str(tmp_path / 'vocos'), V.SMALL, seed, opened=True)
    torch.manual_seed(seed)
    m = pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2, dropout=0., max_seq_len=256), use_vocos=True,
                  pretrained_vocos_path=str(tmp_path / 'vocos'), cond_drop_prob=0.)
    return m.to(DEV)


def test_sample_decodes_each_item(pkg, tmp_path):
    model = _e2tts(pkg, tmp_path)
    assert model.vocos is not None and not model.vocos.training
    B = 3
    cond = torch.randn(B, 20, 100, device=DEV)
    duration = torch.tensor([40, 23, 31], device=DEV)
    text = ['abc', 'de', 'fghij']
    y0 = torch.randn(B, 40, 100, device=DEV)
    with pkg.inject_randomness(y0=y0):
        raw = model.sample(cond, text=text, duration=duration, steps=3, return_raw_output=True)
    with pkg.inject_randomness(y0=y0):
        audio = model.sample(cond, text=text, duration=duration, steps=3)
    assert isinstance(audio, list) and len(audio) == B
    hop = V.SMALL['hop_length']
    sd = {k: v.cpu() for k, v in model.vocos.state_dict().items()}
    for b in range(B):
        n = int(duration[b])
        assert audio[b].shape == (n * hop,) and audio[b].dtype == torch.float32
        mel = raw[b, :n]
        alone = model.vocos.decode_padded(mel[None], torch.tensor([n]), db_to_amp=True)[0]
        assert torch.equal(alone, audio[b])
        amp = torch.pow(torch.pow(10., 0.1 * mel.cpu()), 0.5).t()[None]
        ref = V.decode(sd, V.SMALL, amp)[0]
        probe = V.decode(sd, V.SMALL, amp, round_bf16=True)[0]
        rl2 = lambda a, r: float((a.cpu().double() - r.double()).norm() / r.double().norm())  # noqa: E731
        p, k = rl2(probe, ref), rl2(audio[b], ref)
        print(f'sample item {b}: conditioning probe rel-L2 {p:.3e}, kernels rel-L2 {k:.3e}')
        assert p < 0.2 and k <= 2 * p + 1e-3


def test_training_unchanged_by_vocos(pkg, tmp_path):
    with_v = _e2tts(pkg, tmp_path)
    torch.manual_seed(5)
    without = pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2, dropout=0., max_seq_len=256), use_vocos=False, cond_drop_prob=0.).to(DEV)
    without.load_state_dict({k: v for k, v in with_v.state_dict().items() if not k.startswith('vocos.')})
    mel = torch.randn(2, 64, 100, device=DEV)
    text = ['abc', 'hello']
    x0, times = torch.randn(2, 64, 100, device=DEV), torch.rand(2, device=DEV)
    span = torch.zeros(2, 64, dtype=torch.bool, device=DEV)
    span[:, 10:50] = True
    losses, grads = [], []
    for m in (with_v, without):
        m.train()
        with pkg.inject_randomness(x0=x0, times=times, span_mask=span, drop_text_cond=False):
            step = pkg.GraphedTrainStep(m, mel, text=text)
            losses.append(float(step()))
        torch.cuda.synchronize()
        grads.append({n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None and not n.startswith('vocos.')})
    # the parameter-gradient reductions use fp32 atomics, so two runs of the same step agree to summation order, not bit for bit
    assert abs(losses[0] - losses[1]) <= 1e-6 * abs(losses[1])
    assert grads[0].keys() == grads[1].keys()
    for n in grads[0]:
        a, b = grads[0][n].double(), grads[1][n].double()
        assert float((a - b).norm()) <= 1e-4 * float(b.norm()) + 1e-30, n
    assert all(p.grad is None or not bool(p.grad.any()) for p in with_v.vocos.parameters())
