"""The feed-forward variants of `ff_kwargs` on the GPU: the GLU epilogue of b200_gemm per activation, b200_glu_bwd, the ops.FeedForward
node, and whole models against the oracle with the same ff_kwargs.

GLU epilogue (NaN-filled outputs, element-wise float64 bounds, the method of tests/test_gpu_gemm_schedule.py): the kernel forms
h = u act(g) [* m] [* keep / (1 - p)] from the bf16 pre-activations it also stores in D2, so the reference starts from D2. Each product
rounds once (u = 2^-24) and the bf16 store once (2^-8); the activation's own fp32 error is bounded per element by `act_err`:
  GELU:  the degree-7 tail polynomial of gelu_erf2, < 5e-7 absolute (gemm.cu);
  SiLU:  x / (1 + 2^(-x log2 e)) with ex2.approx (2^-22 relative) and __fdividef (2 ulp): (8 + 1.5 |x|) u relative, + 1e-35 where the
         exponential overflows and the kernel returns 0;
  ReLU^2: one product, u relative; exactly 0 for x <= 0.
The dropout keep set is the restated hash of kernel_checks.drop_mask, and D2 must equal the GELU run's bit for bit.

b200_glu_bwd: against float64 autograd of h = drop(dh) u act(g) m, with the error model of tests/test_gpu_leaf_kernels.py::test_geglu_bwd
for GELU, kernel_checks.sig_err for the SiLU's sigmoid, and one rounding per product; d_mult and db are T-term fp32 sums (gamma_T)."""
import math
import random

import pytest
import torch

from conftest import rel_l2
from dropout_ref import KernelMasks, SeedRecorder, with_dropout
from kernel_checks import BF16, F32, F64, U, U16, assert_close, check_b, check_e, check_f, dev, drop_mask, gamma, gen, nans, pkg, ref64, sig_err  # noqa: F401
from model_checks import cos, duration_vs_oracle, graphed_matches_eager, sample_vs_oracle, small_model, step_inputs, whole_model
from oracle import e2tts_oracle as O

pytestmark = pytest.mark.gpu

GELU, SILU, RELU2 = 1, 2, 3
ACTS = {GELU: 'gelu', SILU: 'silu', RELU2: 'relu2'}
T2 = 16 * 1056     # cfg2 tokens: B16 x (1024 frames + 32 registers)


def act64(code, g):
    if code == GELU:
        return g * 0.5 * (1 + torch.erf(g / math.sqrt(2)))
    if code == SILU:
        return g * torch.sigmoid(g)
    return torch.relu(g) ** 2


def act_err(code, g):
    """absolute bound on the kernel epilogue's fp32 act(g) at the float64 g (see the module docstring)"""
    if code == GELU:
        return torch.full_like(g, 5e-7)
    if code == SILU:
        return act64(SILU, g).abs() * (8 + 1.5 * g.abs()) * U + 1e-35
    return act64(RELU2, g) * U


def split_packed(t, N):
    """packed [u(64) | g(64)] blocks -> (u, g) in hidden-unit order, float64"""
    M = t.shape[0]
    z = t.to(F64).view(M, N // 128, 2, 64)
    return z[:, :, 0].reshape(M, N // 2), z[:, :, 1].reshape(M, N // 2)


def operands(M, N, K, seed, scale=0.1):
    g = torch.Generator(device=dev()).manual_seed(seed)
    return torch.randn(M, K, device=dev(), generator=g).to(BF16), (torch.randn(N, K, device=dev(), generator=g) * scale).to(BF16)


def glu_gemm(pkg, A, W, act, *, bias=None, mult=None, p=0.0, seed=0, force_tile=0):
    M, K = A.shape
    N = W.shape[0]
    D2, out = nans((M, N), BF16), nans((M, N // 2), BF16)
    pkg.ops.gemm(A, W, M, N, K, out=out, ldd=N // 2, D2=D2, ldd2=N, bias=bias, geglu=act, dropout_p=p, seed=seed, glu_mult=mult,
                 force_tile=force_tile)
    return D2, out


def check_glu(name, act, D2, out, mult, p, seed):
    """out against h restated from D2 (bound of the module docstring); dropped units exactly 0, kept units with a non-zero value not 0"""
    M, N = D2.shape
    H = N // 2
    u, g = split_packed(D2, N)
    thresh16 = int(p * 65536)
    kept = drop_mask(seed, M, H) >= (thresh16 << 16) if p > 0 else torch.ones(M, H, dtype=torch.bool, device=dev())
    scale = 65536.0 / (65536 - thresh16)
    m = mult.to(F64)[None] if mult is not None else torch.ones(1, H, dtype=F64, device=dev())
    full = u * act64(act, g) * m * scale
    want = torch.where(kept, full, torch.zeros_like(full))
    got = out.to(F64)
    assert bool((got[~kept] == 0).all()), f'{name}: a dropped hidden unit is not zero'
    bound = (u.abs() * act_err(act, g) * m.abs() * scale + 5 * U * want.abs()) * (1 + U16) + U16 * want.abs()
    assert_close(name, got, want, bound)
    nz = kept & (want.abs() > 1e-30) & (full.abs() > 2 * bound)
    assert bool((got[nz] != 0).all()), f'{name}: a kept hidden unit is zero'
    return kept


GLU_SHAPES = [
    (T2, 4096, 512),      # cfg2 audio FF-in (d512, inner 2048)
    (T2, 2048, 256),      # cfg2 text FF-in
    (4 * 1056, 8192, 1024),   # a d1024 FF-in
    (1096, 512, 320),     # M tail, K tail
    (1096, 512, 192),
    (100, 256, 200),      # fewer rows than one tile
    (2112, 640, 128),     # a text FF-in of dim_text 128, text_ff_mult 2.5: inner 320, an odd number of 64-wide halves
]


@pytest.mark.parametrize('act', list(ACTS), ids=list(ACTS.values()))
@pytest.mark.parametrize('M,N,K', GLU_SHAPES)
def test_glu_gemm(pkg, M, N, K, act):
    """per activation: with bias, multiplier and dropout 0.1, and with none of them; D2 equals the GELU run's bit for bit"""
    A, W = operands(M, N, K, 80 + K + N)
    g = torch.Generator(device=dev()).manual_seed(81 + act)
    bias = torch.randn(N, device=dev(), generator=g) * 0.3
    mult = 1 + 0.5 * torch.randn(N // 2, device=dev(), generator=g)
    ref, acc = ref64(A, W)
    for with_opts in (True, False):
        kw = dict(bias=bias, mult=mult, p=0.1, seed=1234 + M) if with_opts else dict()
        D2, out = glu_gemm(pkg, A, W, act, **kw)
        z = ref + (bias.to(F64) if with_opts else 0)
        tag = f'{ACTS[act]} {M}x{N}x{K} opts={with_opts}'
        assert_close(f'D2 {tag}', D2.to(F64), z, (acc + U * z.abs()) * (1 + U16) + U16 * z.abs())
        kept = check_glu(f'h {tag}', act, D2, out, kw.get('mult'), kw.get('p', 0.0), kw.get('seed', 0))
        if act != GELU:
            D2g, outg = glu_gemm(pkg, A, W, GELU, **kw)
            check_e(f'D2 = GELU run {tag}', D2, D2g)
            if with_opts:   # the GELU run's dropped units are the same
                assert bool((outg.to(F64)[~kept] == 0).all())


@pytest.mark.parametrize('force_tile', [0, 1, 2, 3])
def test_glu_gemm_every_force_tile(pkg, force_tile, N=768):
    M, K = 1096, 320
    A, W = operands(M, N, K, 90 + force_tile)
    g = torch.Generator(device=dev()).manual_seed(91)
    bias, mult = torch.randn(N, device=dev(), generator=g) * 0.3, 1 + 0.5 * torch.randn(N // 2, device=dev(), generator=g)
    for act in ACTS:
        D2, out = glu_gemm(pkg, A, W, act, bias=bias, mult=mult, p=0.25, seed=77, force_tile=force_tile)
        check_glu(f'{ACTS[act]} N{N} tile {force_tile}', act, D2, out, mult, 0.25, 77)


@pytest.mark.parametrize('force_tile', [0, 1, 2, 3])
def test_glu_gemm_every_force_tile_inner320(pkg, force_tile):
    """inner 320 (N = 640): five [u(64) | g(64)] blocks, so a 256-wide tile row ends on half a tile"""
    test_glu_gemm_every_force_tile(pkg, force_tile, N=640)


def regime_operands(gate_bias):
    """M = 256 rows, 128 hidden units; u = small product + 1, gate = small product + gate_bias (one value per hidden unit)"""
    M, N, K = 256, 256, 64
    A, W = operands(M, N, K, 95, scale=0.01)
    bias = torch.zeros(N, device=dev())
    blk = bias.view(N // 128, 2, 64)
    blk[:, 0] = 1.0
    blk[:, 1] = gate_bias.view(N // 128, 64)
    return A, W, bias


def test_silu_large_gate(pkg):
    """SiLU from -120 to 120: the exponential overflows below -88 (value 0 within 1e-35), silu(x) = x for large x"""
    A, W, bias = regime_operands(torch.linspace(-120, 120, 128, device=dev()))
    D2, out = glu_gemm(pkg, A, W, SILU, bias=bias)
    check_glu('silu large |g|', SILU, D2, out, None, 0.0, 0)
    u, g = split_packed(D2, 256)
    big = g > 30
    check_e('silu(x) = x for large x', out[big], (u * g)[big].to(BF16))


def test_relu2_zero_regimes(pkg):
    """ReLU^2: exactly 0 for g < 0, and for g = 0 (gate weights and bias 0)"""
    A, W, bias = regime_operands(-torch.linspace(1, 8, 128, device=dev()))   # the product term is ~0.08 in size
    D2, out = glu_gemm(pkg, A, W, RELU2, bias=bias)
    _, g = split_packed(D2, 256)
    assert bool((g < 0).all()) and bool((out.to(F64) == 0).all())
    W = W.clone()
    W.view(2, 2, 64, -1)[:, 1] = 0
    bias.view(2, 2, 64)[:, 1] = 0
    D2, out = glu_gemm(pkg, A, W, RELU2, bias=bias)
    _, g = split_packed(D2, 256)
    assert bool((g == 0).all()) and bool((out.to(F64) == 0).all())


# ---------------------------------------------------------------------------------------------------------------------- GLU backward
def glu_bwd(pkg, dh, ug, act, *, mult=None, p=0.0, seed=0, sdev=None, db=True, dmult=True):
    T, inner = dh.shape
    dug = nans(tuple(ug.shape), BF16)
    dbp = torch.zeros(2 * inner, device=dev()) if db else None
    dm = torch.zeros(inner, device=dev()) if (dmult and mult is not None) else None
    a = pkg.lib.make_args('b200_glu_bwd_args', dh=dh, ug=ug, dug=dug, db_packed=dbp, mult=mult, d_mult=dm, T=T, inner=inner, act=act,
                          dropout_p=float(p), seed=int(seed), seed_dev=sdev)
    pkg.lib.call('b200_glu_bwd', a, pkg.ops._stream())
    return dug, dbp, dm


def bwd_refs(act, dh, ug, mult, p, seed):
    """float64 (du, dg, d_mult terms) and their element bounds before the bf16 store; dh already on the host"""
    T, inner = dh.shape
    u, g = split_packed(ug.cpu(), 2 * inner)
    d = dh.to(F64)
    if p > 0:
        th = int(p * 65536)
        keep = (drop_mask(seed, T, inner) >= (th << 16)).cpu()
        d = torch.where(keep, d * (65536.0 / (65536 - th)), torch.zeros_like(d))
    m = mult.cpu().to(F64)[None] if mult is not None else torch.ones(1, inner, dtype=F64)
    uu, gg = u.clone().requires_grad_(), g.clone().requires_grad_()
    a64 = act64(act, gg)
    du, dg = torch.autograd.grad(uu * a64 * m, [uu, gg], d)
    a64 = a64.detach()
    if act == GELU:   # test_gpu_leaf_kernels.test_geglu_bwd's error model
        cdf = 0.5 * (1 + torch.erf(g / math.sqrt(2)))
        pdf = torch.exp(-0.5 * g ** 2) / math.sqrt(2 * math.pi)
        e_cdf, e_pdf = 3.5 * U, pdf * (2 * (2 + 1.173 * 0.5 * g ** 2) + g ** 2 + 2) * U
        e_a = g.abs() * e_cdf + U * a64.abs()
        dact = cdf + g * pdf
        e_da = e_cdf + g.abs() * (e_pdf + U * pdf) + U * dact.abs()
    elif act == SILU:
        s = torch.sigmoid(g)
        e_s = sig_err(g)
        e_a = g.abs() * e_s + U * a64.abs()
        dact = s * (1 + g * (1 - s))
        e_da = e_s + e_a * (1 - s).abs() + a64.abs() * (e_s + U) + 3 * U * (s.abs() + (a64 * (1 - s)).abs())
    else:
        r = torch.relu(g)
        e_a, dact, e_da = U * a64, 2 * r, torch.zeros_like(g)
    dm = (d * m).abs()
    b_du = dm * e_a + 3 * U * du.abs()
    b_dg = (dm * u.abs()) * e_da + 4 * U * dg.abs()
    terms = d * u * a64
    b_terms = (d * u).abs() * e_a + 3 * U * terms.abs()
    return du, dg, b_du, b_dg, terms, b_terms


@pytest.mark.parametrize('act', list(ACTS), ids=list(ACTS.values()))
@pytest.mark.parametrize('T,inner', [(1, 64), (257, 2048), (1056, 512), (33, 320), (1056, 320)])
def test_glu_bwd(pkg, act, T, inner):
    g = gen(inner + T + act)
    nb = inner // 64
    ug = (torch.randn(T, 2 * inner, generator=g) * 2).to(BF16).to(dev())
    dh = torch.randn(T, inner, generator=g).to(BF16).to(dev())
    mult = (1 + 0.5 * torch.randn(inner, generator=g)).to(dev())
    for with_mult, p in ((False, 0.0), (True, 0.0), (True, 0.25)):
        m = mult if with_mult else None
        tag = f'{ACTS[act]} T{T} inner{inner} mult={with_mult} p={p}'
        dug, dbp, dm = glu_bwd(pkg, dh, ug, act, mult=m, p=p, seed=99 + T)
        du, dg, b_du, b_dg, terms, b_terms = bwd_refs(act, dh.cpu(), ug, m, p, 99 + T)
        gu, gg = split_packed(dug.cpu(), 2 * inner)
        check_f(f'du {tag}', gu, du, U16 * du.abs() + (1 + U16) * b_du)
        check_f(f'dg {tag}', gg, dg, U16 * dg.abs() + (1 + U16) * b_dg)
        got = dug.cpu().to(F64)
        check_f(f'db {tag}', dbp.cpu(), got.sum(0), gamma(T) * got.abs().sum(0))
        if with_mult:
            check_f(f'd_mult {tag}', dm.cpu(), terms.sum(0), b_terms.sum(0) + gamma(T) * (terms.abs() + b_terms).sum(0))
        assert nb >= 1


def test_geglu_bwd_is_glu_bwd_gelu(pkg):
    """b200_geglu_bwd equals b200_glu_bwd(act=GELU, mult=NULL) bit for bit: dropout with a device seed word, bias gradient"""
    g = gen(5)
    T, inner = 1056, 1024
    ug = (torch.randn(T, 2 * inner, generator=g) * 2).to(BF16).to(dev())
    dh = torch.randn(T, inner, generator=g).to(BF16).to(dev())
    sdev = torch.tensor([0x2545F4914F6CDD1D], device=dev(), dtype=torch.int64)
    for p in (0.0, 0.1):
        dug, dbp, _ = glu_bwd(pkg, dh, ug, GELU, p=p, seed=17, sdev=sdev)
        dug2, dbp2 = nans((T, 2 * inner), BF16), torch.zeros(2 * inner, device=dev())
        pkg.lib.call('b200_geglu_bwd', dh, ug, dug2, dbp2, T, inner, float(p), 17, sdev, pkg.ops._stream())
        check_e(f'dug p={p}', dug, dug2)
        assert rel_l2(dbp.cpu(), dbp2.cpu()) < 1e-6   # fp32 atomics: order may differ


# ---------------------------------------------------------------------------------------------------------------------- node
def pack_rows(t, nb):
    return t.reshape(2, nb, 64, *t.shape[1:]).transpose(0, 1).reshape(t.shape)


@pytest.mark.parametrize('act,with_mult,with_b2,with_cs,p', [
    (SILU, True, False, True, 0.1), (RELU2, True, False, False, 0.0), (SILU, False, True, False, 0.25), (GELU, True, True, True, 0.1),
    (RELU2, False, True, True, 0.0),
])
def test_feed_forward_node(pkg, monkeypatch, act, with_mult, with_b2, with_cs, p):
    """ops.FeedForward with each option, cut at the kernels: h from the saved ug (epilogue bound), y from h (GEMM bound), dh from dz
    (GEMM bound), dug = b200_glu_bwd re-run on the recorded dh (bit for bit), d_mult (float64 bound), no d_b2 without b2, dx from dug"""
    ops = pkg.ops
    B, Np, Din, inner = 3, 150, 256, 512
    T, nb = B * Np, inner // 64
    g = torch.Generator(device=dev()).manual_seed(300 + act)
    prm = lambda shape, s: (torch.randn(shape, device=dev(), generator=g) * s).requires_grad_()
    w1, b1, w2 = prm((2 * inner, Din), Din ** -0.5), prm((2 * inner,), 0.2), prm((Din, inner), inner ** -0.5)
    b2 = prm((Din,), 0.2) if with_b2 else None
    mult = (1 + 0.5 * torch.randn(inner, device=dev(), generator=g)).requires_grad_() if with_mult else None
    cs = (torch.rand(B, Din, device=dev(), generator=g) + 0.5).requires_grad_() if with_cs else None
    w1p, b1p, w2p = pack_rows(w1.detach(), nb).to(BF16), pack_rows(b1.detach(), nb).contiguous(), w2.detach().to(BF16)
    xn = torch.randn(T, Din, device=dev(), generator=g).to(BF16).requires_grad_()
    calls = []
    gemm = ops.gemm
    monkeypatch.setattr(ops, 'gemm', lambda *a, **k: calls.append((a, gemm(*a, **k))) or calls[-1][1])
    s = 4242 + act
    y = ops.FeedForward.apply(xn, w1, b1, w2, b2, w1p, b1p, w2p, cs, B, Np, p, s, None, None, act, mult)
    ctx = y.grad_fn
    assert ctx.meta[6:] == (act, with_b2)
    _, ug, h, _, _, _, _ = ctx.saved_tensors
    check_glu(f'h act{act}', act, ug, h, mult.detach() if with_mult else None, p, s)
    ref, acc = ref64(h, w2p)
    z = ref + (b2.detach().to(F64) if with_b2 else 0)
    csr = cs.detach().to(F64).repeat_interleave(Np, 0) if with_cs else 1.0
    want = z * csr
    assert_close('y', y.to(F64), want, ((acc + U * z.abs()) * csr + U * want.abs()) * (1 + U16) + U16 * want.abs())
    dy = torch.randn(T, Din, device=dev(), generator=g).to(BF16)
    calls.clear()
    y.backward(dy)
    # backward GEMMs: dh = dz W2, dW2 = dz^T h, dx = dug W1p (its A operand is the node's dug), dW1
    (dz, *_), dh = calls[0]
    dug = calls[2][0][0]
    want = dy.to(F64) * csr
    assert_close('dz', dz.to(F64), want, U16 * want.abs() + U * want.abs())
    ref, acc = ref64(dz, w2p.t())
    assert_close('dh', dh.to(F64), ref, acc * (1 + U16) + U16 * ref.abs())
    dug2, _, _ = glu_bwd(pkg, dh, ug, act, mult=mult.detach() if with_mult else None, p=p, seed=s, db=False, dmult=False)
    check_e('dug = b200_glu_bwd re-run', dug, dug2)
    ref, acc = ref64(dug, w1p.t())
    assert_close('dx', xn.grad.to(F64), ref, acc * (1 + U16) + U16 * ref.abs())
    if with_b2:
        ref = want.sum(0)
        check_f('d_b2', b2.grad, ref, gamma(T + 1) * want.abs().sum(0))
    if with_mult:
        _, _, _, _, terms, b_terms = bwd_refs(act, dh.cpu(), ug, mult.detach(), p, s)
        check_f('d_mult', mult.grad.cpu(), terms.sum(0), b_terms.sum(0) + gamma(T) * (terms.abs() + b_terms).sum(0))


# ---------------------------------------------------------------------------------------------------------------------- whole model
CFG2 = dict(dim=512, depth=8, heads=8)
WHOLE = {'swish': dict(swish=True), 'relu2_mult_nobias': dict(relu_squared=True, glu_mult_bias=True, no_bias=True)}


@pytest.mark.parametrize('setting', list(WHOLE))
def test_e2tts_cfg2_shape_ff_kwargs_vs_oracle(pkg, setting):
    """BASELINE cfg2's model with these ff_kwargs, the criteria of model_checks.whole_model"""
    kw = WHOLE[setting]
    whole_model(pkg, dict(CFG2, ff_kwargs=kw), B=2, N=1024, lens=[1024, 800], seed=40)


def test_e2tts_plain_residual_ff_kwargs_vs_oracle(pkg):
    """the case of test_gpu_plain_residual.test_e2tts_cfg2_shape_plain_residual_vs_oracle (cfg2's model with one residual stream) with
    SwiGLU and the GLU multiplier; the residual add sits in the FF-out GEMM's epilogue"""
    kw = dict(swish=True, glu_mult_bias=True)
    whole_model(pkg, dict(CFG2, num_residual_streams=1, ff_kwargs=kw), B=2, N=1024, lens=[1024, 800], seed=40)


def test_duration_predictor_ff_kwargs_vs_oracle(pkg):
    duration_vs_oracle(pkg, 41, dict(dim=128, depth=2, heads=2, ff_kwargs=dict(relu_squared=True, glu_mult_bias=True, no_bias=True)))


@pytest.mark.parametrize('setting', list(WHOLE))
def test_sample_32_steps_ff_kwargs_vs_oracle(pkg, setting):
    sample_vs_oracle(pkg, 60, dict(dim=128, depth=2, heads=2, ff_kwargs=WHOLE[setting]))


@pytest.mark.parametrize('setting', list(WHOLE))
def test_graphed_step_matches_eager(pkg, setting):
    """GraphedTrainStep replays the eager step's gradients with these ff_kwargs (mult_bias and its gradient included)"""
    model, _ = small_model(pkg, 3, dim=128, depth=2, heads=2, ff_kwargs=WHOLE[setting])
    graphed_matches_eager(pkg, model, *step_inputs(pkg))
    assert any(n.endswith('mult_bias') and p.grad is not None for n, p in model.named_parameters()) == ('glu_mult_bias' in WHOLE[setting])


def test_dropout_step_vs_oracle(pkg):
    """one training step with dropout 0.5 and the kernels' own masks (tests/test_gpu_dropout_step.py's method), SwiGLU with multiplier
    and no output bias: loss, prediction and gradient cosines against the oracle given the recorded masks; the masks of seed + 1 miss"""
    kw = dict(swish=True, glu_mult_bias=True, no_bias=True)
    seed, B, N, p = 211, 2, 96, 0.5
    torch.manual_seed(seed)
    random.seed(seed)
    model = pkg.E2TTS(transformer=dict(dropout=p, max_seq_len=128, dim=128, depth=2, heads=2, ff_kwargs=kw), use_vocos=False)
    sd = O.randomize_zero_init({k: v.clone() for k, v in model.state_dict().items()}, seed=seed + 1, dyn_scale=0.05)
    for k in sd:
        if k.endswith('to_gamma.bias'):
            sd[k].zero_()   # AdaLNZero gates open: the branches, dropout included, weigh more in the prediction
    model.load_state_dict(sd)
    model.to(dev()).train()
    g = torch.Generator().manual_seed(seed + 7)
    mel, x0, times = torch.randn(B, N, 100, generator=g), torch.randn(B, N, 100, generator=g), torch.rand(B, generator=g)
    lens = torch.tensor([96, 70])
    span = torch.zeros(B, N, dtype=torch.bool)
    for b, n in enumerate(lens.tolist()):
        span[b, n // 8: n - n // 10] = True
    text = ['Hello', 'Goodbye']
    with pkg.inject_randomness(x0=x0.to(dev()), times=times.to(dev()), span_mask=span.to(dev()), drop_text_cond=False), \
            SeedRecorder(pkg, model) as rec:
        out = model(mel.to(dev()), text=text, lens=lens.to(dev()))
    out.loss.backward()
    torch.cuda.synchronize()
    calls = rec.calls()
    assert sum(1 for n in calls if n.endswith('.ff.1')) == 4

    def oracle(masks, grad=True):
        osd = {k: (v.detach().clone().to(F64).requires_grad_(grad) if v.is_floating_point() else v) for k, v in sd.items()}
        old = torch.get_default_dtype()
        torch.set_default_dtype(F64)
        try:
            with torch.set_grad_enabled(grad):
                o = with_dropout(masks, O.e2tts_forward, osd, O.TransformerCfg(dim=128, depth=2, heads=2, ff_kwargs=kw), mel.to(F64),
                                 O.list_str_to_tensor(text), x0=x0.to(F64), times=times.to(F64), span_mask=span, lens=lens)
            if grad:
                o['loss'].backward()
        finally:
            torch.set_default_dtype(old)
        return float(o['loss']), o['pred'].detach(), {k: v.grad for k, v in osd.items() if grad and v.is_floating_point()}

    masks = KernelMasks(calls, 0)
    rloss, rpred, rgrads = oracle(masks)
    assert sorted(masks.used) == sorted(calls)
    pred = out.pred_flow.detach().float().cpu()
    assert abs(float(out.loss) - rloss) <= 1e-2 * abs(rloss)
    e_pred = rel_l2(pred, rpred)
    print(f'dropout step: loss {float(out.loss):.6f} (oracle {rloss:.6f}), pred rel-L2 {e_pred:.4g}')
    assert e_pred < 3e-2, e_pred
    total = float(torch.cat([v.flatten() for v in rgrads.values() if v is not None]).norm())
    for k, prm in model.named_parameters():
        gr = rgrads[k]
        if gr is None or float(gr.norm()) < 1e-4 * total:
            continue
        assert cos(prm.grad.cpu(), gr) >= 0.99, k
    _, npred, _ = oracle(KernelMasks(calls, 0, offset=1), grad=False)
    assert rel_l2(pred, npred) >= 3 * 3e-2
