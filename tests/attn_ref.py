"""Float64 reference of the attention kernels (csrc/attn_tc.cu), shared by the attention kernel tests: the key bitmask and dropout
hash, the error model of the logit evaluation, the input recipes, the restatement of the forward and backward as `Rv`
(tests/kernel_checks.py) at any head dim, clamped or unclamped, float64 autograd of the same attention, and the C-ABI launches.

Figures for the instructions (PTX ISA) and the tanh polynomials:
  tanh.approx.f32: 2^-10.987 absolute, the PTX ISA's maximum error for it (its later wording, 2^-11 relative, is smaller for |tanh| <= 1);
  ex2.approx.ftz.f32: 2 ulp relative (PTX ISA, ex2), and results below 2^-126 flush to zero;
  the odd Taylor polynomials of tanh (Abramowitz and Stegun 4.5.64: u - u^3/3 + 2u^5/15 - 17u^7/315 + 62u^9/2835 - 1382u^11/155925 ...)
  alternate in sign with decreasing terms for |u| < pi/2, so truncating after u^5 (u^9) errs by at most the u^7 (u^11) term;
  a Horner evaluation of degree n in x^2 with fp32 coefficients is within gamma_(2n + 6) sum |c_i||x|^(2i+1) (Higham (5.3), plus the
  rounding of x^2, of the last product by x and of each coefficient); the attention forward folds clamp * log2(e) * scale^(2i+1) /
  clamp^(2i+1) into its coefficients with at most 16 fp32 roundings each, hence gamma_(2n + 22) there.
The unclamped forward's online softmax is bounded per score term: its exponent 2^((s - m) scale log2 e) is evaluated from fp32 s with
fp32 roundings of scale log2 e, m scale log2 e and the fma, and is rescaled by one factor 2^((m_old - m_new) scale log2 e) per key tile,
each an ex2.approx (2 ulp) of a rounded argument of magnitude <= 2 max|s| scale log2 e. The kernel's final row maximum differs from the
exact one by at most the score error; that common factor cancels in o and lse.
"""
import math

import torch

from kernel_checks import (BF16, F32, F64, U, Rv, _rnd, dev, dot, exact, gamma, h64, mono, mul, nans, ones_rv, stream,
                           to_bf16)

LOG2E = 1.0 / math.log(2.0)
TANH_APPROX = 2.0 ** -10.987  # tanh.approx.f32
EX2_REL = 2.0 ** -22          # ex2.approx.ftz.f32: 2 ulp
FTZ = 2.0 ** -126
TANH_C = [1.0, -1 / 3, 2 / 15, -17 / 315, 62 / 2835, -1382 / 155925]
TQ, TKV_FWD, TQB = 128, 64, 64


def mask_words(Np):
    return ((Np + 127) // 128) * 4


def host_maskbits(m, Np):
    """the layout of attn_maskbits_kernel: bit n % 32 of word n / 32 set iff key n < Np is kept; words per batch padded to 4 per 128 keys"""
    B = m.shape[0]
    W = mask_words(Np)
    keep = torch.zeros(B, W * 32, dtype=torch.int64)
    keep[:, :Np] = m.to(torch.int64)
    w = (keep.view(B, W, 32) << torch.arange(32, dtype=torch.int64)).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32).flatten()


def _mul32(x, c):
    """(x * c) mod 2^32 for int64 tensors x < 2^32 and a 32-bit constant c, without overflowing int64."""
    return (x * (c & 0xFFFF) + ((x * (c >> 16)) & 0xFFFF) * 65536) & 0xFFFFFFFF


def dropout_keep(seed, B, H, Np, p):
    """The kernels' attention-dropout mask (ptx.cuh: drop_seed_word, drop_words) for element ((b*H + h)*Np + i)*stride + j, as bool
    [B, H, Np, Np]: keep iff the 32-bit word of the element >= thresh16 << 16, thresh16 = int(p * 65536)."""
    stride = (Np + 1) & ~1
    seedmix = (seed & 0xFFFFFFFF) ^ (((seed >> 32) * 0x85EBCA77) & 0xFFFFFFFF)
    row = torch.arange(B * H * Np, dtype=torch.int64).view(B, H, Np, 1)
    idx = row * stride + torch.arange(Np, dtype=torch.int64)
    x = (_mul32((idx >> 1) & 0xFFFFFFFF, 0x9E3779B1) + seedmix) & 0xFFFFFFFF
    x = x ^ (x >> 15)
    word = torch.where((idx & 1) == 1, _mul32(x, 0xC2B2AE35), _mul32(x, 0x85EBCA6B))
    return word >= (int(p * 65536) << 16)


def warp_tile_amax(q, k):
    """max |s| over each forward warp's fragment (16 query rows x 64 keys, the dot product over all dh head dims: the head-dim-128
    forward has the same 128-query / 64-key tiles), over the rows the TMA boxes read: past the end of a head they are the next head's
    rows, past the end of the tensor zeros"""
    B, H, Np, dh = q.shape
    Qf, Kf = h64(q).reshape(-1, dh), h64(k).reshape(-1, dh)
    Qf, Kf = torch.cat([Qf, torch.zeros(1, dh, dtype=F64)]), torch.cat([Kf, torch.zeros(1, dh, dtype=F64)])
    total = B * H * Np
    nq, nk = -(-Np // TQ) * TQ, -(-Np // TKV_FWD) * TKV_FWD
    out_all, out_valid = [], []
    for bh in range(B * H):
        qi = (bh * Np + torch.arange(nq)).clamp(max=total)
        ki = (bh * Np + torch.arange(nk)).clamp(max=total)
        s = (Qf[qi] @ Kf[ki].t()).abs()
        out_all.append(s.view(nq // 16, 16, nk // 64, 64).amax((1, 3)))
        sv = s.clone()
        sv[Np:] = 0
        sv[:, Np:] = 0
        sv = sv.view(nq // 16, 16, nk // 64, 64).amax((1, 3))
        sv[(torch.arange(nq // 16) * 16 >= Np)] = math.inf        # warps without a query row of this head write nothing
        out_valid.append(sv)
    return torch.stack(out_all), torch.stack(out_valid)


def poly_mag(au, n):
    return sum(abs(TANH_C[i]) * au ** (2 * i + 1) for i in range(n))


def logit_eval_err(au, fwd, w=1e-3):
    """bound on |computed tanh(u) - tanh(u)| of the forward (fwd: the folded polynomials in the raw score, degree 5 for a warp tile within
    |u| <= 0.15, degree 9 within 0.5, tanh.approx beyond) or of the backward (degree 9 for |u| <= 0.5, tanh.approx beyond). A path is
    allowed for an element when its own |u| permits it, with a relative window w around each threshold for the fp32 score's error."""
    c = 22 if fwd else 6
    e5 = abs(TANH_C[3]) * au ** 7 + gamma(4 + c) * poly_mag(au, 3)
    e9 = abs(TANH_C[5]) * au ** 11 + gamma(8 + c) * poly_mag(au, 5)
    et = TANH_APPROX + gamma(2) * au
    e = torch.zeros_like(au)
    if fwd:
        e = torch.where(au <= 0.15 * (1 + w), torch.maximum(e, e5), e)
    e = torch.where(au <= 0.5 * (1 + w), torch.maximum(e, e9), e)
    return torch.where(au >= 0.5 * (1 - w), torch.maximum(e, et), e)


def ex2_rv(arg, valid):
    """p = ex2.approx.ftz(arg) for valid elements, exactly 0 elsewhere"""
    v = torch.exp2(arg.v)
    e = v * (torch.exp2(arg.e) * (1 + EX2_REL) - 1) + FTZ
    z = torch.zeros_like(v)
    return Rv(torch.where(valid, v, z), torch.where(valid, e, z))


def assert_regime(regime, q, k, m, clamp, w=1e-3):
    """the case's scores lie where the regime's name says (score scale dh^-1/2); returns max |u| per forward warp tile over the
    head's own rows and keys (inf for warps without a query row of the head), None for the unclamped 'big'"""
    scale = q.shape[-1] ** -0.5
    if regime == 'big':          # unclamped: 2^(scale s log2 e) of some valid score is beyond fp32 without the running maximum
        sv = (h64(q) @ h64(k).transpose(-1, -2)).abs() * scale
        assert clamp is None and float(sv[m[:, None, None, :].expand_as(sv)].max()) > 90
        return None
    soc = scale / clamp
    amax, amax_valid = warp_tile_amax(q, k)
    ua = amax * soc
    uv = (h64(q) @ h64(k).transpose(-1, -2)).abs() * soc
    uv = uv[m[:, None, None, :].expand_as(uv)]
    if regime == 'deg5':
        assert bool((ua <= 0.15 * (1 - w)).all())                  # every warp tile on the degree-5 polynomial
    elif regime == 'deg9':
        assert bool((ua <= 0.5 * (1 - w)).all()) and bool((ua > 0.15 * (1 + w)).any())
    elif regime == 'mixed':
        assert bool((ua > 0.5 * (1 + w)).any()) and 0 < float((uv > 0.5).double().mean()) < 0.5
    elif regime == 'tanh':
        assert float((uv > 0.5 * (1 + w)).double().mean()) > 0.5  # mostly tanh.approx
    elif regime == 'sat':
        assert clamp == 64.0 and float((uv > 4).double().mean()) > 0.9   # tanh(4) = 0.99933: the clamp saturates
    return amax_valid * soc


# ------------------------------------------------------------------------------------------------------------------ inputs
def attn_inputs(B, H, Np, regime, masks, gate, seed, dh=64, device=None):
    """regime: the logit regime assert_regime proves ('big': |scale s| > 90 somewhere, for the unclamped kernels). The clamp argument
    u = s dh^-1/2 / clamp of scores of standard deviation sd^2 dh^1/2 does not depend on dh, so the recipes hold at every head dim.
    masks: one kind per batch element (cycled) — 'edges', 'tail', 'random', 'none', 'empty' (no valid key)."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)
    if regime == 'deg9':
        # s = dh c^2 a_i b_j + noise along one sign vector per head, c^2 dh^1/2 constant: |u| up to just under 0.5 (|s| / 400 at
        # dh = 64), so whole tiles need degree 9
        c = 1.75 * (64 / dh) ** 0.25
        sv = torch.where(rn(B, H, 1, dh) > 0, 1.0, -1.0)
        a = c * (0.5 + 0.5 * torch.rand(B, H, Np, 1, generator=g))
        b = c * (2 * torch.rand(B, H, Np, 1, generator=g) - 1)
        q, k = sv * a + 0.01 * rn(B, H, Np, dh), sv * b
    else:
        sd = {'deg5': 1.0, 'mixed': 1.0, 'tanh': 7.0, 'sat': 60.0, 'big': 6.0}[regime]
        q, k = rn(B, H, Np, dh) * sd, rn(B, H, Np, dh) * sd
        if regime == 'mixed':
            k[:, :, ::7] *= 16                                        # every 7th key far outside the polynomial range
            # and every warp tile with a row of the head beyond the degree-5 range: the first key of each 64-key tile and the last
            # key are |s| ~ 16 |sum q| (std 128), the last query row meets them at s = 64 * 4 * 16
            k[:, :, ::64] = 16.0
            k[:, :, -1] = 16.0
            q[:, :, -1] = 4.0
    v = rn(B, H, Np, dh)
    m = torch.ones(B, Np, dtype=torch.bool)
    for b in range(B):
        kind = masks[b % len(masks)]
        if kind == 'empty':
            m[b] = False
            continue
        if kind == 'edges':                                         # both sides of the 32-bit word, 64-key tile and 128-key tile edges
            for n in (31, 32, 63, 64, 127, 128):
                if n < Np:
                    m[b, n] = False
        elif kind == 'tail':                                        # a padded tail and the key before the last valid one
            n_valid = max(Np - Np // 4 - 1, 2)
            m[b, n_valid:] = False
            m[b, n_valid - 2] = False
        elif kind == 'random':
            m[b] = torch.rand(Np, generator=g) > 0.3
        m[b, 0] = True                                              # (the model's register keys are always valid)
    gt = torch.rand(B * Np, H, generator=g) if gate else None
    dog = rn(B * Np, H * dh)
    to = lambda t: None if t is None else t.to(dev() if device is None else device).contiguous()
    return (to(q.to(BF16)), to(k.to(BF16)), to(v.to(BF16)), to(gt), m, to(m.to(torch.uint8)) if masks != ('none',) else None,
            to(dog.to(BF16)))


def unclamped_inputs(B, H, Np, kind, seed, gate=True):
    """kind: 'big' (|scale s| > 90 somewhere), 'grow' (the row maximum grows from key tile to key tile), 'first_tile' (keys 0..63 of
    every batch element masked), 'all_masked' (batch element 1 has no valid key), 'random'"""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)
    q, k = rn(B, H, Np, 64), rn(B, H, Np, 64)
    m = torch.rand(B, Np, generator=g) > 0.25
    if kind == 'big':
        q, k = q * 6.0, k * 6.0                                       # |s| up to ~ 36 * 64 ^ 0.5 * 4: scale s beyond 90
    elif kind == 'grow':
        d = torch.where(rn(1, H, 1, 64) > 0, 1.0, -1.0)
        q = d * 2.0 + 0.1 * q
        k = d * (torch.arange(Np, dtype=torch.float32) / 16.0)[None, None, :, None] + 0.1 * k   # s grows with the key index
        m[:, -1] = True                                             # (the last key tile holds a valid key)
    elif kind == 'first_tile':
        m[:, :64] = False
        m[:, 64] = True
    elif kind == 'all_masked':
        m[1] = False
    v = rn(B, H, Np, 64)
    gt = torch.rand(B * Np, H, generator=g) if gate else None
    dog = rn(B * Np, H * 64)
    to = lambda t: None if t is None else t.to(dev()).contiguous()
    return to(q.to(BF16)), to(k.to(BF16)), to(v.to(BF16)), to(gt), m, to(m.to(torch.uint8)), to(dog.to(BF16))


def d128_inputs(B, H, Np, kind, gate, masked, seed, dh=128):
    """kind: 'small' (|u| mostly in the polynomial ranges), 'mixed' (every 7th key far outside them), 'big' (unclamped: |scale s| > 90
    somewhere). masked: random key masks, and batch element 1 (if any) without a valid key."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)
    q, k = rn(B, H, Np, dh), rn(B, H, Np, dh)
    if kind == 'mixed':
        k[:, :, ::7] *= 16
    elif kind == 'big':
        q, k = q * 5.0, k * 5.0
    v = rn(B, H, Np, dh)
    m = torch.ones(B, Np, dtype=torch.bool)
    if masked:
        m = torch.rand(B, Np, generator=g) > 0.3
        m[:, 0] = True
        if B > 1:
            m[1] = False
    gt = torch.rand(B * Np, H, generator=g) if gate else None
    dog = rn(B * Np, H * dh)
    to = lambda t: None if t is None else t.to(dev()).contiguous()
    return (to(q.to(BF16)), to(k.to(BF16)), to(v.to(BF16)), to(gt), m, to(m.to(torch.uint8)) if masked else None, to(dog.to(BF16)))


# ------------------------------------------------------------------------------------------------------------------ restatement
def restate(q, k, v, gate, m, clamp, p_drop, seed, dog, o_k, lse_k):
    """forward and backward of attn_tc.cu at head dim dh as Rv on [B, H, Np(query), Np(key)]; clamp None: the unclamped kernels.
    o_k / lse_k: the kernel's saved forward outputs. Rows without a valid key are left to the caller."""
    B, H, Np, dh = q.shape
    scale = dh ** -0.5
    sl2 = scale * LOG2E
    nkv = -(-Np // 64)
    Q, K, V = exact(q), exact(k), exact(v)
    thr = int(p_drop * 65536)
    ks = 65536 / (65536 - thr)
    ksR = Rv(torch.tensor(ks, dtype=F64), U * ks if p_drop > 0 else 0.0)
    valid = m[:, None, None, :].expand(B, H, Np, Np)
    row_ok = valid.any(-1, keepdim=True)
    keep = dropout_keep(seed, B, H, Np, p_drop).to(F64) if p_drop > 0 else torch.ones(B, H, Np, Np, dtype=F64)
    s = dot('bhid,bhjd->bhij', Q, K, dh)
    zero = torch.zeros_like(s.v)
    if clamp is None:
        M = torch.where(valid, s.v, torch.full_like(s.v, -math.inf)).amax(-1, keepdim=True)
        M = torch.where(row_ok, M, torch.zeros_like(M))
        Mabs = torch.where(valid, s.v.abs() + s.e, zero).amax(-1, keepdim=True)
        # exponent error of one term in log2 units: its own score error, the fp32 roundings of scale log2 e, -m scale log2 e and the
        # fma, and the arguments of the rescale factors it goes through (one rounding of m_old - m_new, one of the product, per tile)
        A = sl2 * (s.e + 4 * U * (s.v.abs() + Mabs)) + nkv * sl2 * 3 * U * 2 * Mabs
        r = torch.exp2(A) * (1 + EX2_REL) ** (nkv + 1) - 1
        pv = torch.where(valid, torch.exp2(sl2 * (s.v - M)), zero)
        p = Rv(pv, torch.where(valid, pv * r + FTZ, zero))
        l = dot('bhij,j->bhi', p, ones_rv(Np), Np + 2 * nkv)         # + the rescaling multiplies, one per tile
        nacc = Np + 2 * nkv
    else:
        # y = clamp log2(e) tanh(u), p = 2^y on valid keys
        soc, clog = scale / clamp, clamp * LOG2E
        u = s.v * soc
        y = Rv(clog * torch.tanh(u), LOG2E * scale * s.e + clog * logit_eval_err(u.abs(), True) + gamma(3) * clog * torch.tanh(u).abs())
        p = ex2_rv(y, valid)
        l = dot('bhij,j->bhi', p, ones_rv(Np), Np)
        nacc = Np
    # lse = ln l (+ the row maximum), o = (sum bf16(p keep) v) keep_scale / l
    l1 = Rv(torch.where(row_ok[..., 0], l.v, torch.ones_like(l.v)), l.e)
    lnl = mono(l1, torch.log, 2 * U)                                 # logf: 1 ulp
    if clamp is None:
        lse = Rv(M[..., 0] * scale + lnl.v, lnl.e + U * (M[..., 0].abs() * scale + lnl.v.abs()) * 2)
    else:
        lse = lnl
    pk = to_bf16(Rv(p.v * keep, p.e * keep))
    oacc = dot('bhij,bhjd->bhid', pk, V, nacc)
    inv = mono(l1, lambda t: ks / t, gamma(2))                       # keep_scale (rounded) / l
    o = mul(oacc, inv[..., None])
    G = Rv(h64(gate).view(B, Np, H).permute(0, 2, 1)[..., None]) if gate is not None else Rv(torch.ones(B, H, Np, 1, dtype=F64))
    og = mul(to_bf16(o), G)                                          # gate times the kernel's bf16 o, rounded again to bf16
    # backward: P recomputed from the kernel's lse
    DOG = Rv(h64(dog).view(B, Np, H, dh).permute(0, 2, 1, 3))
    dO = to_bf16(mul(DOG, G))
    ok64 = h64(o_k)
    dgate_own = (DOG.v * ok64).sum(-1)                               # prep: <dog, o> with the kernel's own o
    dgate_e = gamma(dh) * (DOG.v.abs() * ok64.abs()).sum(-1)
    delta = Rv((dO.v * o.v).sum(-1),
               G.v[..., 0].abs() * ((DOG.v.abs() * (ok64 - o.v).abs()).sum(-1) + gamma(dh + 1) * (DOG.v.abs() * ok64.abs()).sum(-1)))
    dP = dot('bhid,bhjd->bhij', dO, V, dh)
    lk = torch.where(row_ok[..., 0], h64(lse_k), torch.zeros_like(lse.v))
    dlse = (lk - torch.where(row_ok[..., 0], lse.v, torch.zeros_like(lse.v))).abs()
    lv = torch.where(row_ok, lse.v[..., None], torch.zeros_like(lse.v[..., None]))
    if clamp is None:
        arg = _rnd(sl2 * s.v - lv * LOG2E, sl2 * s.e + LOG2E * dlse[..., None] + gamma(2) * (sl2 * s.v.abs() + LOG2E * lk.abs()[..., None]))
        dsc = Rv(torch.tensor(scale, dtype=F64))
    else:
        th = Rv(torch.tanh(u), soc * s.e + logit_eval_err(u.abs(), False))
        arg = _rnd(clog * th.v - lv * LOG2E, clog * th.e + gamma(2) * clog * th.v.abs() + LOG2E * dlse[..., None] +
                   gamma(2) * LOG2E * lk.abs()[..., None])                # the fma rounds once
        dsc = _rnd(scale * (1 - th.v ** 2), scale * (2 * th.v.abs() * th.e + th.e ** 2))
    pb = ex2_rv(arg, valid)
    if p_drop > 0:                                                   # fma(keep ? dP : 0, keep_scale, -delta)
        tt = _rnd(keep * ks * dP.v - delta.v[..., None], keep * (ks * dP.e + dP.v.abs() * ksR.e) + delta.e[..., None])
    else:
        tt = _rnd(dP.v - delta.v[..., None], dP.e + delta.e[..., None])
    ds = to_bf16(mul(mul(pb, tt), dsc))
    dk = dot('bhij,bhid->bhjd', ds, Q, Np)
    dq = dot('bhij,bhjd->bhid', ds, K, Np)
    dv = mul(dot('bhij,bhid->bhjd', to_bf16(Rv(pb.v * keep, pb.e * keep)), dO, Np), ksR)
    return dict(o=o, og=og, lse=lse, dO=dO, dgate_own=dgate_own, dgate_e=dgate_e, dq=dq, dk=dk, dv=dv, row_ok=row_ok[..., 0])


def autograd64(q, k, v, gate, m, clamp, p_drop, seed, dog):
    """float64 autograd of the softmax attention the kernels implement (x-transformers Attend as the reference configures it; rows
    with a valid key)"""
    B, H, Np, dh = q.shape
    qr, kr, vr = (h64(t).requires_grad_() for t in (q, k, v))
    sim = torch.einsum('bhid,bhjd->bhij', qr, kr) * dh ** -0.5
    if clamp is not None:
        sim = torch.tanh(sim / clamp) * clamp
    valid = m[:, None, None, :].expand_as(sim)
    row_ok = valid.any(-1, keepdim=True)
    sim = torch.where(row_ok, sim.masked_fill(~valid, -math.inf), torch.zeros_like(sim))   # (no NaN through rows without a valid key)
    lse = torch.logsumexp(sim, -1)
    attn = torch.where(row_ok, torch.softmax(sim, -1), torch.zeros_like(sim))
    if p_drop > 0:
        attn = attn * dropout_keep(seed, B, H, Np, p_drop) * (65536 / (65536 - int(p_drop * 65536)))
    o = attn @ vr
    g = h64(gate).view(B, Np, H).permute(0, 2, 1)[..., None] if gate is not None else 1.0
    dog4 = h64(dog).view(B, Np, H, dh).permute(0, 2, 1, 3)
    dq, dk, dv = torch.autograd.grad(o * g, [qr, kr, vr], dog4)
    return dict(o=o.detach(), lse=lse.detach(), dq=dq, dk=dk, dv=dv)


# ------------------------------------------------------------------------------------------------------------------ launches
def _clamp_fields(clamp):
    return dict(softclamp=0.0, unclamped=1) if clamp is None else dict(softclamp=clamp, unclamped=0)


def attn_fwd(pkg, q, k, v, gate, mask, clamp, p_drop, seed, ws=None, ready=0, seed_dev=None):
    """b200_attn_fwd into NaN-filled outputs at the head dim of q, scale dh^-1/2; clamp None: the unclamped kernels"""
    B, H, Np, dh = q.shape
    o, og, lse = nans(q.shape, BF16), nans((B * Np, H * dh), BF16), nans((B, H, Np), F32)
    if ws is None:
        ws = torch.full((mask_words(Np) * B,), -1, device=dev(), dtype=torch.int32)
    a = pkg.lib.make_args('b200_attn_fwd_args', q=q, k=k, v=v, keymask=mask, gate=gate, o=o, og=og, lse=lse, B=B, H=H, Np=Np, dim_head=dh,
                          scale=dh ** -0.5, dropout_p=p_drop, seed=seed, ws_maskbits=ws, seed_dev=seed_dev, maskbits_ready=ready,
                          **_clamp_fields(clamp))
    pkg.lib.call('b200_attn_fwd', a, stream())
    return dict(o=o, og=og, lse=lse, ws=ws)


def attn_bwd(pkg, q, k, v, o, lse, gate, mask, dog, clamp, p_drop, seed, ws=None, ready=0, seed_dev=None, d_gate=None):
    """b200_attn_bwd into NaN-filled outputs; d_gate: whether to pass a d_gate output (by default only with a gate; without one the
    kernel writes <dog, o> there)"""
    B, H, Np, dh = q.shape
    if d_gate is None:
        d_gate = gate is not None
    r = dict(dq=nans(q.shape, F32), dk=nans(q.shape, BF16), dv=nans(q.shape, BF16), ws_dO=nans(q.shape, BF16), ws_delta=nans((B, H, Np), F32),
             d_gate=nans((B * Np, H), F32) if d_gate else None)
    if ws is None:
        ws = torch.full((mask_words(Np) * B,), -1, device=dev(), dtype=torch.int32)
    a = pkg.lib.make_args('b200_attn_bwd_args', q=q, k=k, v=v, o=o, d_og=dog, keymask=mask, gate=gate, lse=lse, ws_dO=r['ws_dO'],
                          ws_delta=r['ws_delta'], d_gate=r['d_gate'], dq=r['dq'], dk=r['dk'], dv=r['dv'], B=B, H=H, Np=Np, dim_head=dh,
                          scale=dh ** -0.5, dropout_p=p_drop, seed=seed, ws_maskbits=ws, seed_dev=seed_dev, maskbits_ready=ready,
                          **_clamp_fields(clamp))
    pkg.lib.call('b200_attn_bwd', a, stream())
    return r
