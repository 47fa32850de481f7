"""Element-wise float64 bounds for the autograd nodes of ops.py: the layer that wires the proven kernels together.

Each multi-launch torch.autograd.Function runs forward and backward as the model calls it, and every forward output and every
returned gradient is compared element by element with a float64 reference. The kernels themselves are held by
test_gpu_leaf_kernels.py, test_gpu_gemm_schedule.py, test_gpu_attention_hyper_kernels.py and test_gpu_conv_melspec_kernels.py, so
the references cut at them and bounds do not compound: wherever a node hands a value to, or takes one from, one of those kernels,
the reference starts from the node's own value at that point (forward values from the node's ctx; backward values recorded by
wrappers installed on the ops module attributes the node calls: ops.gemm, ops._attn_core_bwd, ops._hc_width_bwd). Each remaining
stage is then bounded on its own:
  GEMM:   the exact inner product of the bf16 / fp32 operands the stage reads, within gamma_K sum_k |a_k b_k| (fp32 accumulation in
          any order, split-K atomics included: Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., (3.5)); each fp32
          epilogue operation (bias, gate, residual) rounds once (u = 2^-24); a bf16 output rounds once more (2^-8, check_bf16).
  colsum: a T-term fp32 sum in any order, gamma_(T-1) sum|x|.
  kernel: an element-wise kernel stage (qkv post-processing, attention forward, GEGLU backward, Fourier features, hyper-connection
          width forward) is re-run on the inputs the reference says the node must pass, with NaN-filled outputs, and must match the
          node bit for bit; these kernels are deterministic (no atomics), and their accuracy is held by the kernel tests.
  layout: slices, views, transposes and gradient slots match bit for bit.
Every compared buffer is checked for NaN (NaN never passes a bound). Shapes: the widths bench.py config 2 builds (read from
bench.CONFIGS and the Transformer defaults), and small odd ones: B = 3 with its own mask and gate row per batch element, Np = 150
(not a multiple of 64), a fully masked batch element, C = 100 in a 104-column operand, T*S-row cross / skip GEMMs with Dt != D.
The last tests hold the per-step zero-filled gradient slab (ops._ZeroPool) that every bias, gate and hyper-connection parameter
gradient is drawn from.
"""
import inspect

import pytest
import torch

import bench
from attn_ref import attn_fwd
from hyper_conv_ref import CV_TN, S, cdiv, dw_ref, hc_fwd, hc_inputs, hc_params
from kernel_checks import U, U16, assert_close, check_bf16, check_e, dev, drop_mask, gamma, h64, nans, pkg, ref64

pytestmark = pytest.mark.gpu

F64, BF16, F32 = torch.float64, torch.bfloat16, torch.float32
U8 = torch.uint8


# ------------------------------------------------------------------------------------------------------------ widths of config 2
def cfg2():
    """config 2 of bench.py with the Transformer defaults it leaves in place (text width, registers, FF multiplier)"""
    from e2_tts_pytorch_b200.modules import Transformer
    c = bench.CONFIGS[2]
    p = inspect.signature(Transformer.__init__).parameters
    d, H, B, N = c['dim'], c['heads'], c['batch'], c['seq']
    R, mult = p['num_registers'].default, p['ff_mult'].default
    return dict(d=d, dt=d // 2, H=H, B=B, N=N, Np=N + R, inner=d * mult, inner_t=(d // 2) * mult)


# ------------------------------------------------------------------------------------------------------------ helpers
def rng(seed):
    return torch.Generator(device=dev()).manual_seed(seed)


def rnd(shape, g, scale=1.0, dtype=BF16, grad=False):
    t = (torch.randn(shape, device=dev(), generator=g) * scale).to(dtype)
    return t.requires_grad_() if grad else t


def param(shape, g, scale, grad=True):
    return rnd(shape, g, scale, F32, grad)


def _2d(t):
    return t.reshape(-1, t.shape[-1]) if t.dim() >= 2 else t.reshape(1, -1)


def cf(name, got, ref, bound):
    """fp32 (F): |got - ref| <= bound element-wise"""
    assert got is not None, f'{name}: no gradient'
    ref = ref.to(F64)
    bound = torch.as_tensor(bound, dtype=F64, device=ref.device).expand_as(ref)
    assert_close(name, _2d(got.detach().reshape(ref.shape)), _2d(ref), _2d(bound))


def cb(name, got, ref, acc):
    """bf16 (B): one rounding of an fp32 value within acc of ref"""
    assert got is not None and got.dtype == BF16, f'{name}: {None if got is None else got.dtype}'
    ref = ref.to(F64)
    acc = torch.as_tensor(acc, dtype=F64, device=ref.device).expand_as(ref)
    check_bf16(name, _2d(got.detach().reshape(ref.shape)), _2d(ref), _2d(acc))


def ce(name, got, want):
    """E: bit for bit"""
    assert got is not None, f'{name}: missing'
    check_e(name, got.detach(), want.detach())


def same(a, b):
    """a and b are the same buffer (or both absent)"""
    if a is None or b is None:
        return a is None and b is None
    return a.data_ptr() == b.data_ptr() and a.shape == b.shape and a.dtype == b.dtype


def colsum_ref(x):
    x = x.to(F64)
    return x.sum(0), gamma(x.shape[0] - 1) * x.abs().sum(0)


def unpack_rows(t, nb):
    """undo the GEGLU interleave of the packed first FF layer: packed row blk*128 + s*64 + j is unpacked row s*inner + blk*64 + j"""
    return t.reshape(nb, 2, 64, *t.shape[1:]).transpose(0, 1).reshape(t.shape)


def pack_rows(t, nb):
    return t.reshape(2, nb, 64, *t.shape[1:]).transpose(0, 1).reshape(t.shape)


def row_mask(B, Np, lens):
    """uint8 [B, Np]: element b keeps its first lens[b] tokens"""
    return (torch.arange(Np, device=dev())[None] < torch.tensor(lens, device=dev())[:, None]).to(U8).contiguous()


def seed_word(v):
    return torch.tensor([v], device=dev(), dtype=torch.int64)


def gate_rows(cs, Np):
    return cs.detach().to(F64).repeat_interleave(Np, 0)


def d_gate_ref(dy, y, cs, B):
    """gradient of the per-batch AdaLNZero gate through y = cs * z: sum over the batch element's rows of dy * y / cs, from the bf16
    y the forward stored (the kernel recovers z as y / cs). Each term is a product and a quotient (two roundings, in either order),
    and Np terms are summed: gamma_(Np + 2) sum|dy y / cs|."""
    Np = y.shape[0] // B
    t = dy.to(F64) * y.to(F64) / gate_rows(cs, Np)
    t = t.reshape(B, Np, -1)
    return t.sum(1), gamma(Np + 2) * t.abs().sum(1)


class Recorder:
    """wraps ops module attributes so that the backward's intermediates can be read: calls[name] = [(args, kwargs, result)]"""

    def __init__(self, monkeypatch, ops, names=('gemm', '_attn_core_bwd', '_hc_width_bwd')):
        self.calls = {n: [] for n in names}
        for n in names:
            f = getattr(ops, n)

            def wrap(*a, _f=f, _n=n, **k):
                r = _f(*a, **k)
                self.calls[_n].append((a, k, r))
                return r
            monkeypatch.setattr(ops, n, wrap)

    def clear(self):
        for v in self.calls.values():
            v.clear()


@pytest.fixture
def rec(pkg, monkeypatch):
    return Recorder(monkeypatch, pkg.ops)


@pytest.fixture
def pool(pkg, monkeypatch):
    """a private zero pool whose slab holds a whole node backward (16 MB), so every accumulator comes from the slab as in training"""
    p = pkg.ops._ZeroPool()
    p.peak = 1 << 22
    monkeypatch.setattr(pkg.ops, 'zero_pool', p)
    return p


def slab_only(pool):
    assert pool.buf is not None and pool.used <= pool.buf.numel(), 'an accumulator took the torch.zeros fallback'


# ============================================================================================================ Attention
def attn_case(pkg, rec, pool, *, B, Np, H, Din, lens, has_mix, extra, p_drop, use_seed_dev, shared_bits, seed):
    """ops.Attention: the fused q/k/v/gate(/mix) GEMM, qkv post-processing, flash attention; backward through the attention and
    qkv backward kernels into dx, the five weight slots and the two bias slots.
      qkvg = xn Wpack^T:         GEMM bound, bf16 (the pad columns past 3I + (1 or 2)H are not read by anyone).
      q, k, v, gate:             b200_qkv_post_fwd re-run on the saved qkvg with bg, bm, the rotary table and v_first: bit for bit.
      og, o, lse:                b200_attn_fwd re-run on the saved q, k, v, gate with the mask, dropout, seed and device seed: bit for bit.
      attention backward:        called with the incoming d_og and the forward's own q, k, v, o, lse, gate, mask, dropout, seed, softclamp,
                                 device seed and shared bitmask (the same buffers).
      d_qkvg (recorded):         b200_qkv_post_bwd re-run on the recorded dq, dk, dv, d_gate and the incoming d_v_extra: bit for bit,
                                 pad columns included; d_vfirst likewise.
      dx = d_qkvg Wpack:         GEMM bound over K = 3I + (1 or 2)H, bf16.
      dWq, dWk, dWv, dWg, dWm:   the row slices of d_qkvg^T xn (GEMM bound over K = T, fp32).
      dbg, dbm:                  column sums of the gate / mix logit columns of d_qkvg, gamma_(T-1)."""
    from e2_tts_pytorch_b200.modules import SOFTCLAMP
    ops = pkg.ops
    g = rng(seed)
    I, T = 64 * H, B * Np
    sc = Din ** -0.5
    xn = rnd((T, Din), g, grad=True)
    wq, wk, wv = (param((I, Din), g, sc) for _ in range(3))
    wg, bg = param((H, Din), g, sc), param((H,), g, 1.0)
    wm, bm = (param((H, Din), g, sc), param((H,), g, 1.0)) if has_mix else (None, None)
    vf = rnd((B, H, Np, 64), g, grad=True) if has_mix else None
    wpack = torch.cat([wq, wk, wv, wg] + ([wm] if has_mix else [])).detach().to(BF16)
    ncat = 3 * I + (2 if has_mix else 1) * H
    ld = (ncat + 7) // 8 * 8
    cs, sn = ops.rotary_table(Np, dev())
    mask = row_mask(B, Np, lens)
    bits = ops.attn_maskbits(mask, B, Np, dev()) if shared_bits else None
    sdev = seed_word(0x5DEECE66D) if use_seed_dev else None
    s = 0x1234567 + seed
    pool.begin(dev())
    og, v = ops.Attention.apply(xn, wq, wk, wv, wg, bg, wm, bm, vf, wpack, cs, sn, mask, B, Np, H, p_drop, s, SOFTCLAMP, sdev, bits)
    ctx = og.grad_fn
    (xn_s, qkvg, gate, vf_s, wp_s, cs_s, sn_s, bg_s, bm_s, q, k, v_s, o, lse, mask_s) = ctx.saved_tensors
    assert ctx.meta[:6] == (B, Np, H, ncat, ld, has_mix) and ctx.meta[6:9] == (p_drop, s, SOFTCLAMP) and same(ctx.meta[9], sdev)
    assert same(ctx.maskbits, bits)
    tag = f'B{B} Np{Np} H{H} Din{Din} mix={has_mix} extra={extra} p={p_drop}'
    # forward
    ref, acc = ref64(xn.detach(), wpack)
    cb(f'qkvg {tag}', qkvg[:, :ncat], ref, acc)
    q2, k2, v2 = (nans((B, H, Np, 64), BF16) for _ in range(3))
    gate2 = nans((T, H), F32)
    a = pkg.lib.make_args('b200_qkv_post_args', qkvg=qkvg, ld=ld, gate_bias=bg, mix_bias=bm, rot_cos=cs, rot_sin=sn, v_first=vf,
                          q=q2, k=k2, v=v2, gate=gate2, B=B, H=H, Np=Np, dim_head=64)
    pkg.lib.call('b200_qkv_post_fwd', a, ops._stream())
    for nm, got, want in (('q', q, q2), ('k', k, k2), ('v', v_s, v2), ('gate', gate, gate2), ('returned v', v, v2)):
        ce(f'{nm} {tag}', got, want)
    r = attn_fwd(pkg, q2, k2, v2, gate2, mask, SOFTCLAMP, p_drop, s, seed_dev=sdev)
    ce(f'og {tag}', og, r['og'])
    ce(f'o {tag}', o, r['o'])
    ce(f'lse {tag}', lse, r['lse'])
    # backward
    dog = rnd((T, I), g)
    dve = rnd((B, H, Np, 64), g) if extra else None
    rec.clear()
    torch.autograd.backward([og, v] if extra else [og], [dog, dve] if extra else [dog])
    slab_only(pool)
    (ab, _, (dq, dk, dv, dgt)), = rec.calls['_attn_core_bwd']
    assert torch.equal(ab[0], dog)
    for i, t in enumerate((q, k, v_s, o, lse, gate, mask)):
        assert same(ab[1 + i], t), f'attention backward argument {1 + i} {tag}'
    assert ab[8:11] == (p_drop, s, SOFTCLAMP) and same(ab[11], sdev) and same(ab[12], bits)
    d_qkvg = rec.calls['gemm'][0][0][0]
    assert d_qkvg.shape == (T, ld)
    d_qkvg2 = nans((T, ld), BF16)
    d_vf2 = nans((B, H, Np, 64), BF16) if has_mix else None
    a = pkg.lib.make_args('b200_qkv_post_args', qkvg=qkvg, ld=ld, gate_bias=bg, mix_bias=bm, rot_cos=cs, rot_sin=sn, v_first=vf,
                          gate=gate, dq=dq, dk=dk, dv=dv, dv_extra=dve, d_gate=dgt, d_qkvg=d_qkvg2, d_vfirst=d_vf2,
                          B=B, H=H, Np=Np, dim_head=64, dq_fp32=1)
    pkg.lib.call('b200_qkv_post_bwd', a, ops._stream())
    ce(f'd_qkvg {tag}', d_qkvg, d_qkvg2)
    if has_mix:
        ce(f'd_vfirst {tag}', vf.grad, d_vf2)
    dq_ = d_qkvg[:, :ncat]
    ref, acc = ref64(dq_, wpack.t())
    cb(f'dx {tag}', xn.grad, ref, acc)
    ref, acc = ref64(dq_.t(), xn.detach().t())
    for nm, w, lo, hi in (('wq', wq, 0, I), ('wk', wk, I, 2 * I), ('wv', wv, 2 * I, 3 * I), ('wg', wg, 3 * I, 3 * I + H),
                          ('wm', wm, 3 * I + H, 3 * I + 2 * H)):
        if w is not None:
            cf(f'd{nm} {tag}', w.grad, ref[lo:hi], acc[lo:hi])
    for nm, b, lo in (('bg', bg, 3 * I), ('bm', bm, 3 * I + H)):
        if b is not None:
            ref_b, acc_b = colsum_ref(d_qkvg[:, lo:lo + H])
            cf(f'd{nm} {tag}', b.grad, ref_b, acc_b)


def test_attention_cfg2_audio(pkg, rec, pool):
    """config 2, audio stream of a later layer: H = 8 with value-residual mix logits and v_first, the model's shared key bitmask,
    dropout 0.1 with a device seed word; ragged audio lengths behind the register tokens."""
    c = cfg2()
    B, Np = c['B'], c['Np']
    lens = [Np - (37 * b) % 500 for b in range(B)]
    attn_case(pkg, rec, pool, B=B, Np=Np, H=c['H'], Din=c['d'], lens=lens, has_mix=True, extra=False, p_drop=0.1, use_seed_dev=True,
              shared_bits=True, seed=1)


def test_attention_cfg2_text_first_layer(pkg, rec, pool):
    """config 2, text stream of layer 0: no mix logits, and its values feed every later layer (the extra value gradient d_v_extra)"""
    c = cfg2()
    B, Np = c['B'], c['Np']
    lens = [Np - (53 * b) % 700 for b in range(B)]
    attn_case(pkg, rec, pool, B=B, Np=Np, H=c['H'], Din=c['dt'], lens=lens, has_mix=False, extra=True, p_drop=0.0, use_seed_dev=False,
              shared_bits=True, seed=2)


@pytest.mark.parametrize('has_mix,extra', [(False, False), (True, True)])
def test_attention_small_odd(pkg, rec, pool, has_mix, extra):
    """B = 3, Np = 150, H = 2 (row pitch of the fused GEMM padded past 3I + (1 or 2)H), Din = 200 (a partial k-block), one element
    with only 4 valid keys; the node builds its own key bitmask"""
    H = 2
    ncat = 3 * 64 * H + (2 if has_mix else 1) * H
    assert (ncat + 7) // 8 * 8 > ncat
    attn_case(pkg, rec, pool, B=3, Np=150, H=H, Din=200, lens=[150, 97, 4], has_mix=has_mix, extra=extra, p_drop=0.0,
              use_seed_dev=False, shared_bits=False, seed=3 + has_mix)


# ============================================================================================================ OutProj
def outproj_case(pkg, rec, pool, *, B, Np, I, Dout, lens, with_cs, seed):
    """ops.OutProj: y = mask * cs[b] * (og Wout^T), and its backward.
      y:     GEMM bound, times the gate, the gate product rounds once (u |y|), bf16; masked rows exactly 0.
      dz (recorded, the backward GEMMs' operand) = dy * mask * cs[b]: one fp32 product, bf16 (masked rows exactly 0); without a
             gate it is dy * mask exactly.
      d_cs:  d_gate_ref. d_og = dz Wout: GEMM bound, bf16. dWout = dz^T og: GEMM bound over T, fp32."""
    ops = pkg.ops
    g = rng(seed)
    T = B * Np
    og = rnd((T, I), g, grad=True)
    w = param((Dout, I), g, I ** -0.5)
    wpack = w.detach().to(BF16)
    cs = (torch.rand(B, Dout, device=dev(), generator=g) + 0.5).requires_grad_() if with_cs else None
    mask = row_mask(B, Np, lens)
    mk = mask.reshape(T, 1).to(F64)
    csr = gate_rows(cs, Np) if with_cs else torch.ones((T, 1), device=dev(), dtype=F64)
    tag = f'B{B} Np{Np} I{I} D{Dout} cs={with_cs}'
    pool.begin(dev())
    y = ops.OutProj.apply(og, w, wpack, cs, mask, B, Np)
    assert y.grad_fn.meta == (B, Np)
    ref, acc = ref64(og.detach(), wpack)
    cb(f'y {tag}', y, ref * csr * mk, (acc * csr + U * (ref * csr).abs()) * mk)
    dy = rnd((T, Dout), g)
    rec.clear()
    y.backward(dy)
    slab_only(pool)
    dz = rec.calls['gemm'][0][0][0]
    want = dy.to(F64) * csr * mk
    if with_cs:
        cb(f'dz {tag}', dz, want, U * want.abs())
        ref, bound = d_gate_ref(dy, y.detach(), cs, B)
        cf(f'd_cs {tag}', cs.grad, ref, bound)
    else:
        ce(f'dz {tag}', dz, torch.where(mask.reshape(T, 1) != 0, dy, torch.zeros_like(dy)))
    ref, acc = ref64(dz, wpack.t())
    cb(f'd_og {tag}', og.grad, ref, acc)
    ref, acc = ref64(dz.t(), og.detach().t())
    cf(f'dW {tag}', w.grad, ref, acc)


def test_out_proj_cfg2(pkg, rec, pool):
    """config 2: the audio projection (gate per batch element) and the text projection (no gate, D = dt)"""
    c = cfg2()
    B, Np = c['B'], c['Np']
    lens = [Np - (41 * b) % 600 for b in range(B)]
    I = 64 * c['H']
    outproj_case(pkg, rec, pool, B=B, Np=Np, I=I, Dout=c['d'], lens=lens, with_cs=True, seed=10)
    outproj_case(pkg, rec, pool, B=B, Np=Np, I=I, Dout=c['dt'], lens=lens, with_cs=False, seed=11)


@pytest.mark.parametrize('with_cs', [True, False])
def test_out_proj_small_odd(pkg, rec, pool, with_cs):
    """B = 3, Np = 150: the batch boundaries of the gate rows fall inside the GEMM's 128-row tiles; the last element is fully masked"""
    outproj_case(pkg, rec, pool, B=3, Np=150, I=128, Dout=200, lens=[150, 61, 0], with_cs=with_cs, seed=12 + with_cs)


# ============================================================================================================ FeedForward
def ff_make(B, Np, Din, inner, with_cs, seed):
    g = rng(seed)
    nb = inner // 64
    P = dict(w1=param((2 * inner, Din), g, Din ** -0.5), b1=param((2 * inner,), g, 0.2), w2=param((Din, inner), g, inner ** -0.5),
             b2=param((Din,), g, 0.2), cs=(torch.rand(B, Din, device=dev(), generator=g) + 0.5).requires_grad_() if with_cs else None)
    P['w1p'] = pack_rows(P['w1'].detach(), nb).to(BF16)
    P['b1p'] = pack_rows(P['b1'].detach(), nb).contiguous()
    P['w2p'] = P['w2'].detach().to(BF16)
    P['g'] = g
    return P


def ff_apply(ops, P, xn, B, Np, p_drop, s, sdev):
    return ops.FeedForward.apply(xn, P['w1'], P['b1'], P['w2'], P['b2'], P['w1p'], P['b1p'], P['w2p'], P['cs'], B, Np, p_drop, s, sdev)


def ff_pool_refs(rec, y, dy, cs, B, nb):
    """references of the three gradients the FF backward draws from the zero pool: d_b2, d_cs and d_b1 (from the recorded dug)"""
    T = dy.shape[0]
    dug = rec.calls['gemm'][2][0][0]
    out = {}
    if cs is not None:
        t = dy.to(F64) * gate_rows(cs, T // B)
        out['b2'] = (t.sum(0), gamma(T + 1) * t.abs().sum(0))
        out['cs'] = d_gate_ref(dy, y, cs, B)
    else:
        out['b2'] = colsum_ref(dy)
    r, bd = colsum_ref(dug)
    out['b1'] = (unpack_rows(r, nb), unpack_rows(bd, nb))
    return out


def ff_case(pkg, rec, pool, *, B, Np, Din, inner, with_cs, p_drop, use_seed_dev, seed):
    """ops.FeedForward: GEGLU GEMM (+bias, dropout) -> out GEMM (+bias, gate), and its backward.
      ug = xn W1p^T + b1p (packed [u(64) | g(64)] blocks): GEMM bound + the bias add (u |ug|), bf16.
      h = dropout(u * gelu(g)) from the saved ug: the GEGLU epilogue bound of test_gpu_gemm_schedule (GELU polynomial 5e-7 |u|, three
          fp32 roundings, bf16), with the dropout pattern of seed + the device seed word; dropped units exactly 0.
      y = cs[b] (h W2^T + b2): GEMM bound, bias add and gate product (one rounding each), bf16.
      dz (recorded) = dy cs[b] (one product, bf16) or dy itself; d_b2 = sum dy cs[b] (gamma_(T+1), the rowgate kernel's fused sum) or
          the column sum of dy; d_cs: d_gate_ref.
      dh (recorded) = dz W2: GEMM bound, bf16; dW2 = dz^T h: GEMM bound over T.
      dug (recorded): b200_geglu_bwd re-run on dh, ug with the forward's dropout, seed and device seed: bit for bit.
      d_b1 = column sums of dug, un-interleaved; dx = dug W1p: GEMM bound; dW1 = un-interleaved dug^T xn: GEMM bound over T."""
    ops = pkg.ops
    nb = inner // 64
    assert nb > 1      # the interleave is visible
    P = ff_make(B, Np, Din, inner, with_cs, seed)
    g = P['g']
    T = B * Np
    xn = rnd((T, Din), g, grad=True)
    sdev = seed_word(0x2545F4914F6CDD1D) if use_seed_dev else None
    s = 0x7654321 + seed
    cs = P['cs']
    tag = f'B{B} Np{Np} Din{Din} inner{inner} cs={with_cs} p={p_drop} seed_dev={use_seed_dev}'
    pool.begin(dev())
    y = ff_apply(ops, P, xn, B, Np, p_drop, s, sdev)
    ctx = y.grad_fn
    assert ctx.meta[:5] == (B, Np, p_drop, s, inner) and same(ctx.meta[5], sdev)
    _, ug, h, y_s, _, _, cs_s = ctx.saved_tensors
    assert same(y_s, y) and same(cs_s, cs)
    ref, acc = ref64(xn.detach(), P['w1p'])
    z = ref + P['b1p'].to(F64)
    cb(f'ug {tag}', ug, z, acc + U * z.abs())
    zz = ug.to(F64).view(T, nb, 2, 64)
    u, gt = zz[:, :, 0].reshape(T, inner), zz[:, :, 1].reshape(T, inner)
    gelu = gt * 0.5 * (1 + torch.erf(gt / 2 ** 0.5))
    thresh16 = int(p_drop * 65536)
    s_eff = (s + (int(sdev.item()) if use_seed_dev else 0)) & (2 ** 64 - 1)
    kept = drop_mask(s_eff, T, inner) >= (thresh16 << 16)
    scale = 65536.0 / (65536 - thresh16)
    want = torch.where(kept, u * gelu * scale, torch.zeros_like(u))
    assert bool((h[~kept] == 0).all()), f'a dropped hidden unit is not zero {tag}'
    cf(f'h {tag}', h, want, (u.abs() * 5e-7 * scale + 4 * U * want.abs()) * (1 + U16) + U16 * want.abs())
    ref, acc = ref64(h, P['w2p'])
    z = ref + P['b2'].detach().to(F64)
    if with_cs:
        csr = gate_rows(cs, Np)
        cb(f'y {tag}', y, z * csr, (acc + U * z.abs()) * csr + U * (z * csr).abs())
    else:
        cb(f'y {tag}', y, z, acc + U * z.abs())
    dy = rnd((T, Din), g)
    rec.clear()
    y.backward(dy)
    slab_only(pool)
    calls = rec.calls['gemm']
    dz, dh, dug = calls[0][0][0], calls[0][2], calls[2][0][0]
    if with_cs:
        want = dy.to(F64) * csr
        cb(f'dz {tag}', dz, want, U * want.abs())
    else:
        ce(f'dz {tag}', dz, dy)
    refs = ff_pool_refs(rec, y.detach(), dy, cs, B, nb)
    cf(f'd_b2 {tag}', P['b2'].grad, *refs['b2'])
    if with_cs:
        cf(f'd_cs {tag}', cs.grad, *refs['cs'])
    ref, acc = ref64(dz, P['w2p'].t())
    cb(f'dh {tag}', dh, ref, acc)
    ref, acc = ref64(dz.t(), h.t())
    cf(f'dW2 {tag}', P['w2'].grad, ref, acc)
    dug2 = nans(tuple(ug.shape), BF16)
    pkg.lib.call('b200_geglu_bwd', dh, ug, dug2, None, T, inner, float(p_drop), int(s), sdev, ops._stream())
    ce(f'dug {tag}', dug, dug2)
    cf(f'd_b1 {tag}', P['b1'].grad, *refs['b1'])
    ref, acc = ref64(dug, P['w1p'].t())
    cb(f'dx {tag}', xn.grad, ref, acc)
    ref, acc = ref64(dug.t(), xn.detach().t())
    cf(f'dW1 {tag}', P['w1'].grad, unpack_rows(ref, nb), unpack_rows(acc, nb))


def test_feed_forward_cfg2_audio(pkg, rec, pool):
    """config 2 audio FF (inner = 4d) with the AdaLNZero gate, dropout 0.1 and a device seed word"""
    c = cfg2()
    ff_case(pkg, rec, pool, B=c['B'], Np=c['Np'], Din=c['d'], inner=c['inner'], with_cs=True, p_drop=0.1, use_seed_dev=True, seed=20)


def test_feed_forward_cfg2_text(pkg, rec, pool):
    """config 2 text FF: no gate (colscale None), dropout 0.1 without a device seed"""
    c = cfg2()
    ff_case(pkg, rec, pool, B=c['B'], Np=c['Np'], Din=c['dt'], inner=c['inner_t'], with_cs=False, p_drop=0.1, use_seed_dev=False,
            seed=21)


@pytest.mark.parametrize('with_cs,p_drop,use_seed_dev', [(True, 0.0, False), (False, 0.1, True)])
def test_feed_forward_small_odd(pkg, rec, pool, with_cs, p_drop, use_seed_dev):
    """B = 3, Np = 150, Din = 200, inner = 192 (three interleaved blocks)"""
    ff_case(pkg, rec, pool, B=3, Np=150, Din=200, inner=192, with_cs=with_cs, p_drop=p_drop, use_seed_dev=use_seed_dev,
            seed=22 + with_cs)


# ============================================================================================================ CrossCondition
def cross_case(pkg, rec, pool, *, T, D, Dt, has_at, with_dto, seed):
    """ops.CrossCondition on T*S rows: xo = x + [x | t] Wta^T, to = t + [x | t] Wat^T (or t itself without audio-to-text).
      xo, to: GEMM bound over K = D + Dt, the residual add (u |out|), bf16; without Wat, to is ts bit for bit.
      dx = dxo + [dxo | dto] Wstack[:, :D]  (without Wat: dxo + dxo Wta[:, :D]),
      dt = dto + [dxo | dto] Wstack[:, D:]  (without Wat: dto + dxo Wta[:, D:]; no residual when the text output has no consumer):
            GEMM bound, the residual add, bf16.
      dWta = dxo^T [x | t], dWat = dto^T [x | t]: GEMM bound over T*S rows, fp32."""
    ops = pkg.ops
    g = rng(seed)
    R, Kc = T * S, D + Dt
    xs = rnd((T, S, D), g, grad=True)
    ts = rnd((T, S, Dt), g, grad=True)
    w_ta = param((D, Kc), g, Kc ** -0.5)
    w_at = param((Dt, Kc), g, Kc ** -0.5) if has_at else None
    wstack = torch.cat([w_ta] + ([w_at] if has_at else [])).detach().to(BF16)
    tag = f'T{T} D{D} Dt{Dt} at={has_at} dto={with_dto}'
    pool.begin(dev())
    xo, to = ops.CrossCondition.apply(xs, ts, w_ta, w_at, wstack)
    x2, t2 = xs.detach().reshape(R, D), ts.detach().reshape(R, Dt)
    Acat = torch.cat([x2, t2], 1)
    ref, acc = ref64(Acat, wstack[:D])
    want = ref + x2.to(F64)
    cb(f'xo {tag}', xo, want, acc + U * want.abs())
    if has_at:
        ref, acc = ref64(Acat, wstack[D:])
        want = ref + t2.to(F64)
        cb(f'to {tag}', to, want, acc + U * want.abs())
    else:
        ce(f'to {tag}', to, ts)
    dxo = rnd((T, S, D), g)
    dto = rnd((T, S, Dt), g) if with_dto else None
    rec.clear()
    torch.autograd.backward([xo, to] if with_dto else [xo], [dxo, dto] if with_dto else [dxo])
    dxo2 = dxo.reshape(R, D)
    dto2 = dto.reshape(R, Dt) if with_dto else (torch.zeros((R, Dt), device=dev(), dtype=BF16) if has_at else None)
    dA = torch.cat([dxo2, dto2], 1) if has_at else dxo2
    K = dA.shape[1]
    for nm, got, lo, hi, res in (('dx', xs.grad, 0, D, dxo2), ('dt', ts.grad, D, Kc, dto2 if with_dto else None)):
        ref, acc = ref64(dA, wstack[:K, lo:hi].t())
        want = ref + (res.to(F64) if res is not None else 0)
        cb(f'{nm} {tag}', got, want, acc + U * want.abs())
    ref, acc = ref64(dxo2.t(), Acat.t())
    cf(f'dWta {tag}', w_ta.grad, ref, acc)
    if has_at:
        ref, acc = ref64(dto2.t(), Acat.t())
        cf(f'dWat {tag}', w_at.grad, ref, acc)


def test_cross_condition_cfg2(pkg, rec, pool):
    """config 2: a middle layer (both directions, both outputs consumed) and the last text layer (text_to_audio only, text output
    without a consumer: dto is None)"""
    c = cfg2()
    T = c['B'] * c['Np']
    cross_case(pkg, rec, pool, T=T, D=c['d'], Dt=c['dt'], has_at=True, with_dto=True, seed=30)
    cross_case(pkg, rec, pool, T=T, D=c['d'], Dt=c['dt'], has_at=False, with_dto=False, seed=31)


@pytest.mark.parametrize('has_at,with_dto', [(False, True), (True, False)])
def test_cross_condition_small_odd(pkg, rec, pool, has_at, with_dto):
    """T = 450 tokens x 4 streams, D = 192, Dt = 128 (the two-source GEMM switches sources on a 64-column k-block): without Wat but
    with a text gradient (its identity path must reach dt), and with Wat but no text gradient (zero-filled)"""
    cross_case(pkg, rec, pool, T=450, D=192, Dt=128, has_at=has_at, with_dto=with_dto, seed=32 + has_at)


# ============================================================================================================ SkipProj
def skip_case(pkg, rec, pool, *, T, D, seed):
    """ops.SkipProj: out = [x | skip] W^T over T*S rows (GEMM bound over K = 2D, bf16); dx = dy W[:, :D], dskip = dy W[:, D:]
    (GEMM bound, bf16); dW = dy^T [x | skip] (GEMM bound over T*S, fp32)."""
    ops = pkg.ops
    g = rng(seed)
    R = T * S
    xs, sk = rnd((T, S, D), g, grad=True), rnd((T, S, D), g, grad=True)
    w = param((D, 2 * D), g, (2 * D) ** -0.5)
    wpack = w.detach().to(BF16)
    tag = f'T{T} D{D}'
    out = ops.SkipProj.apply(xs, sk, w, wpack)
    Acat = torch.cat([xs.detach().reshape(R, D), sk.detach().reshape(R, D)], 1)
    ref, acc = ref64(Acat, wpack)
    cb(f'out {tag}', out, ref, acc)
    dy = rnd((T, S, D), g)
    out.backward(dy)
    dy2 = dy.reshape(R, D)
    for nm, got, lo in (('dx', xs.grad, 0), ('dskip', sk.grad, D)):
        ref, acc = ref64(dy2, wpack[:, lo:lo + D].t())
        cb(f'{nm} {tag}', got, ref, acc)
    ref, acc = ref64(dy2.t(), Acat.t())
    cf(f'dW {tag}', w.grad, ref, acc)


def test_skip_proj(pkg, rec, pool):
    c = cfg2()
    skip_case(pkg, rec, pool, T=c['B'] * c['Np'], D=c['d'], seed=40)
    skip_case(pkg, rec, pool, T=450, D=192, seed=41)


# ============================================================================================================ StemLinear
def stem_case(pkg, rec, pool, *, T, D, C, Kp, mode, seed):
    """ops.StemLinear over the packed stem operand A [T, Kp] (pad columns 0, as stem_prepare writes them):
      two sources: Wpack = [W_in | 0 | W_cond | 0] with the cond block at column Kp/2; concat: W_in over the first 2C columns;
      single (the DurationPredictor): W_in over the first C of Kp = C rounded up to 8.
      h = A Wpack^T + (b_in + b_cond): GEMM bound, the fp32 bias sum (u) and the bias add (u |h|), bf16.
      dW_in, dW_cond: the column blocks of d_h^T A at 0 and Kp/2 (GEMM bound over T, fp32); d_b_in = d_b_cond = column sums of d_h."""
    ops = pkg.ops
    g = rng(seed)
    two = mode == 'two'
    Cin = 2 * C if mode == 'concat' else C
    half = Kp // 2
    A_ = rnd((T, Kp), g)
    pad = torch.ones(Kp, device=dev(), dtype=torch.bool)
    pad[:Cin] = False
    if two:
        pad[half:half + C] = False
    A_[:, pad] = 0
    w_in, b_in = param((D, Cin), g, Cin ** -0.5), param((D,), g, 0.3)
    w_c, b_c = (param((D, C), g, C ** -0.5), param((D,), g, 0.3)) if two else (None, None)
    wpack = torch.zeros((D, Kp), device=dev(), dtype=BF16)
    wpack[:, :Cin] = w_in.detach().to(BF16)
    if two:
        wpack[:, half:half + C] = w_c.detach().to(BF16)
    tag = f'T{T} D{D} C{C} Kp{Kp} {mode}'
    pool.begin(dev())
    h = ops.StemLinear.apply(A_, w_in, b_in, w_c, b_c, wpack)
    assert h.grad_fn.meta == (D, Cin, two)
    ref, acc = ref64(A_, wpack)
    bias = b_in.detach().to(F64) + (b_c.detach().to(F64) if two else 0)
    want = ref + bias
    cb(f'h {tag}', h, want, acc + U * bias.abs() + U * want.abs())
    dh = rnd((T, D), g)
    h.backward(dh)
    slab_only(pool)
    ref, acc = ref64(dh.t(), A_.t())
    cf(f'dW_in {tag}', w_in.grad, ref[:, :Cin], acc[:, :Cin])
    rb, bb = colsum_ref(dh)
    cf(f'db_in {tag}', b_in.grad, rb, bb)
    if two:
        cf(f'dW_cond {tag}', w_c.grad, ref[:, half:half + C], acc[:, half:half + C])
        cf(f'db_cond {tag}', b_c.grad, rb, bb)


def test_stem_linear_cfg2(pkg, rec, pool):
    """config 2: 100 mel channels; E2TTS pads each source to Cp = C rounded up to 64 (so the cond block does not start at column C),
    with concat_cond one proj_in over cat(cond, x); the DurationPredictor's single proj_in over C rounded up to 8"""
    c = cfg2()
    T, D, C = c['B'] * c['N'], c['d'], 100
    Cp = (C + 63) // 64 * 64
    assert Cp != C
    stem_case(pkg, rec, pool, T=T, D=D, C=C, Kp=2 * Cp, mode='two', seed=50)
    stem_case(pkg, rec, pool, T=T, D=D, C=C, Kp=2 * Cp, mode='concat', seed=51)
    stem_case(pkg, rec, pool, T=T, D=D, C=C, Kp=(C + 7) // 8 * 8, mode='single', seed=52)


def test_stem_linear_c100_cp104(pkg, rec, pool):
    """two sources with C = 100 in Cp = 104 columns each: the cond block starts at 104, four columns past C"""
    stem_case(pkg, rec, pool, T=450, D=200, C=100, Kp=208, mode='two', seed=53)


# ============================================================================================================ PredHead / FlowLossHead
def head_bwd_checks(rec, tag, dp, y, w, b, wpack, C):
    """dy = dp Wpack (GEMM bound over C, bf16); dW = dp^T y (GEMM bound over T, fp32); db = column sums of dp"""
    ref, acc = ref64(dp[:, :C], wpack.t())
    cb(f'dy {tag}', y.grad, ref, acc)
    ref, acc = ref64(dp[:, :C].t(), y.detach().t())
    cf(f'dW {tag}', w.grad, ref, acc)
    cf(f'db {tag}', b.grad, *colsum_ref(dp[:, :C]))


def head_make(T, D, C, seed):
    g = rng(seed)
    y = rnd((T, D), g, grad=True)
    w, b = param((C, D), g, D ** -0.5), param((C,), g, 0.3)
    return g, y, w, b, w.detach().to(BF16)


def check_pred(tag, pred, y, wpack, b):
    """pred = y Wpack^T + b, fp32 out: GEMM bound and the bias add"""
    ref, acc = ref64(y.detach(), wpack)
    want = ref + b.detach().to(F64)
    cf(f'pred {tag}', pred, want, acc + U * want.abs())


@pytest.mark.parametrize('T', [None, 450])
def test_pred_head(pkg, rec, pool, T):
    """ops.PredHead: pred (fp32) and the backward from bf16(dpred) (recorded: bit for bit the round to nearest of dpred) into dy, dW,
    db; T = None is config 2 (B * N rows, d, 100 mels)"""
    c = cfg2()
    D = c['d'] if T is None else 200
    T = c['B'] * c['N'] if T is None else T
    C = 100
    g, y, w, b, wpack = head_make(T, D, C, 60 + T)
    tag = f'T{T} D{D}'
    pool.begin(dev())
    pred = pkg.ops.PredHead.apply(y, w, b, wpack)
    check_pred(tag, pred, y, wpack, b)
    dpred = torch.randn((T, C), device=dev(), generator=g)
    rec.clear()
    pred.backward(dpred)
    dp = rec.calls['gemm'][0][0][0]
    ce(f'dp {tag}', dp[:, :C], dpred.to(BF16))
    head_bwd_checks(rec, tag, dp, y, w, b, wpack, C)


@pytest.mark.parametrize('T,with_vel', [(None, True), (450, False)])
def test_flow_loss_head(pkg, rec, pool, T, with_vel):
    """ops.FlowLossHead: pred as PredHead; pred_data = x0 + pred bit for bit; the masked-MSE loss and its parts from the node's own
    pred (test_flow_loss's bounds: the flow and velocity means within (gamma_n + 6u) of themselves, the weighted sum 2u more);
    dpred (recorded) = bf16(2 dloss / n (d + w (pred - vt))) with the same per-term roundings as there, exactly 0 outside the span and in
    the pad columns; dy, dW, db from it as PredHead. Each batch element has its own span; one has none."""
    c = cfg2()
    B, N = (c['B'], c['N']) if T is None else (3, 150)
    D = c['d'] if T is None else 200
    T = B * N
    C = 100
    ldp = (C + 7) // 8 * 8
    g, y, w, b, wpack = head_make(T, D, C, 70 + T)
    x1, x0 = (torch.randn((T, C), device=dev(), generator=g) for _ in range(2))
    vt = torch.randn((T, C), device=dev(), generator=g) if with_vel else None
    span = torch.zeros((B, N), device=dev(), dtype=torch.bool)
    for i in range(B - 1):
        span[i, (7 * i) % N:(7 * i) % N + N // (2 + i)] = True
    span_u8 = span.to(U8).reshape(-1).contiguous()
    vw = 0.7
    tag = f'T{T} vel={with_vel}'
    pool.begin(dev())
    loss, pred, pred_data, parts = pkg.ops.FlowLossHead.apply(y, w, b, wpack, x1, x0, span_u8, vt, vw)
    check_pred(tag, pred, y, wpack, b)
    ce(f'pred_data {tag}', pred_data, x0 + pred)
    sm = span.reshape(-1)
    n = int(sm.sum()) * C
    w32 = float(torch.tensor(vw, dtype=F32))
    P = pred.to(F64)
    d = P - (x1.to(F64) - x0.to(F64))
    flow = (d ** 2)[sm].mean()
    dv = (P - vt.to(F64)) if with_vel else torch.zeros_like(d)
    vel = (dv ** 2)[sm].mean()
    tot = flow + w32 * vel
    e_flow, e_vel = flow * (gamma(n) + 6 * U), vel * (gamma(n) + 6 * U)
    cf(f'loss parts {tag}', parts, torch.stack([flow, vel]), torch.stack([e_flow, e_vel]))
    cf(f'loss {tag}', loss.reshape(1), tot.reshape(1), (e_flow + w32 * e_vel + 2 * U * tot).reshape(1))
    dloss = 0.37
    rec.clear()
    loss.backward(torch.tensor(dloss, device=dev()))
    dp = rec.calls['gemm'][0][0][0]
    assert dp.shape == (T, ldp)
    scale = 2 * dloss / n
    v = d + w32 * dv
    atol = abs(scale) * (2 * U * d.abs() + 3 * U * w32 * dv.abs() + 3 * U * v.abs())
    cb(f'dpred {tag}', dp[:, :C][sm], (scale * v)[sm], atol[sm])
    ce(f'dpred outside the span {tag}', dp[:, :C][~sm], torch.zeros_like(dp[:, :C][~sm]))
    ce(f'dpred pad columns {tag}', dp[:, C:], torch.zeros_like(dp[:, C:]))
    head_bwd_checks(rec, tag, dp, y, w, b, wpack, C)


# ============================================================================================================ FourierLinear
@pytest.mark.parametrize('small', [False, True])
def test_fourier_linear(pkg, rec, pool, small):
    """ops.FourierLinear: z = x W^T (GEMM bound, bf16, row pitch n rounded up to 8); out = b200_fourier_feat_fwd(z) re-run: bit for
    bit; dz (recorded) = b200_fourier_feat_bwd(d_out, z) re-run: bit for bit, pad columns included; dx = dz Wpack (GEMM bound over
    n, bf16); dW = dz^T x (GEMM bound over T, fp32). config 2 widths (LinearFourierEmbed(d).split_dims, Np rows per element) and a
    small case whose pitch is padded (n = 76 in 80 columns)."""
    from e2_tts_pytorch_b200.modules import LinearFourierEmbed
    ops = pkg.ops
    c = cfg2()
    if small:
        T, D, (df, dr) = 450, 200, (44, 32)
    else:
        T, D = c['B'] * c['Np'], c['d']
        df, dr = LinearFourierEmbed(D).split_dims
    n = df + dr
    ld = (n + 7) // 8 * 8
    assert (ld > n) == small
    g = rng(80 + small)
    x = rnd((T, D), g, grad=True)
    w = param((n, D), g, D ** -0.5)
    wpack = w.detach().to(BF16)
    tag = f'T{T} D{D} df{df} dr{dr}'
    out = ops.FourierLinear.apply(x, w, wpack, df, dr)
    ctx = out.grad_fn
    assert ctx.meta == (df, dr, ld)
    z = ctx.saved_tensors[2]
    ref, acc = ref64(x.detach(), wpack)
    cb(f'z {tag}', z[:, :n], ref, acc)
    out2 = nans((T, 2 * df + dr), BF16)
    pkg.lib.call('b200_fourier_feat_fwd', z, ld, out2, T, df, dr, ops._stream())
    ce(f'out {tag}', out, out2)
    dout = rnd((T, 2 * df + dr), g)
    rec.clear()
    out.backward(dout)
    dz = rec.calls['gemm'][0][0][0]
    dz2 = nans((T, ld), BF16)
    pkg.lib.call('b200_fourier_feat_bwd', dout, z, ld, dz2, T, df, dr, ops._stream())
    ce(f'dz {tag}', dz, dz2)
    ref, acc = ref64(dz[:, :n], wpack.t())
    cb(f'dx {tag}', x.grad, ref, acc)
    ref, acc = ref64(dz[:, :n].t(), x.detach().t())
    cf(f'dW {tag}', w.grad, ref, acc)


# ============================================================================================================ CondPack
def test_cond_pack(pkg):
    """ops.CondPack at config 2 (4 to_gamma projections per layer, the AdaLNZero ones with a bias): the forward hands back the packed
    stack unchanged; backward gives weight j the rows j*d..(j+1)*d of the packed weight gradient and bias m the segment (2m+1)*d of
    the packed bias gradient (the AdaLNZero gates sit on the odd segments), bit for bit."""
    c = cfg2()
    d, L = c['d'], bench.CONFIGS[2]['depth']
    n_w, n_b = 4 * L, 2 * L
    g = rng(90)
    W_out, b_out = param((n_w * d, d), g, 1.0, grad=False), param((n_w * d,), g, 1.0, grad=False)
    ws = [param((d, d), g, 1.0) for _ in range(n_w)]
    bs = [param((d,), g, 1.0) for _ in range(n_b)]
    Wo, bo = pkg.ops.CondPack.apply(W_out, b_out, d, n_w, *ws, *bs)
    ce('W out', Wo, W_out)
    ce('b out', bo, b_out)
    dW, db = torch.randn_like(W_out), torch.randn_like(b_out)
    torch.autograd.backward([Wo, bo], [dW, db])
    for j, w in enumerate(ws):
        ce(f'weight {j}', w.grad, dW[j * d:(j + 1) * d])
    for m, b in enumerate(bs):
        ce(f'bias {m}', b.grad, db[(2 * m + 1) * d:(2 * m + 2) * d])


# ============================================================================================================ hyper-connections, DwConv
def hc_leaves(P, inp, mode):
    names = ('gamma', 'afn', 'ascale', 'salpha', 'bfn', 'bscale', 'sbeta')
    params = [P[k].clone().requires_grad_() for k in names]
    ng = inp['ng'].clone().requires_grad_() if mode else None
    return params, ng


@pytest.mark.parametrize('mode', [0, 1, 2])
@pytest.mark.parametrize('fused', [False, True])
def test_hc_width_wiring(pkg, rec, pool, mode, fused):
    """ops.HcWidth / ops.HcDepthWidth: the forward equals b200_hc_width_fwd launched with the node's norm_mode and rows_per_batch,
    bit for bit (branch, streams, beta and the saved stats); the backward calls the width backward with the saved stats, the same
    parameters in order, norm_mode, rows_per_batch and the incoming gradients, and returns each of its results in the slot of the
    input it belongs to. T = 480 tokens of 3 elements (160 rows per batch, T * S a multiple of 64 as the fused backward needs), D = 200."""
    ops = pkg.ops
    T, D, rpb = 480, 200, 160
    assert ops.hc_can_fuse(T, S)
    P = hc_params(D, 100 + mode)
    inp = hc_inputs(T, D, rpb, mode, fused, 101 + mode)
    params, ng = hc_leaves(P, inp, mode)
    x = inp['x'].clone().requires_grad_()
    extra = ()
    if fused:
        y, bp = inp['y'].clone().requires_grad_(), inp['bp'].clone().requires_grad_()
        extra = (y, bp)
    pool.begin(dev())
    node = ops.HcDepthWidth if fused else ops.HcWidth
    branch, res, beta = node.apply(x, *extra, *params, ng, mode, rpb)
    ctx = branch.grad_fn
    assert ctx.meta == (mode, rpb)
    r = hc_fwd(pkg, P, inp['x'], mode, inp['ng'], rpb, inp['y'] if fused else None, inp['bp'] if fused else None)
    for nm, got in (('branch', branch), ('res', res), ('beta', beta)):
        ce(f'{nm} mode{mode} fused={fused}', got, r[nm])
    stats = ctx.saved_tensors[3 if fused else 1]
    ce(f'stats mode{mode} fused={fused}', stats, r['stats'])
    rec.clear()
    torch.autograd.backward([branch, res, beta], [inp['d_branch'], inp['d_res'], inp['d_beta']])
    slab_only(pool)
    (a, _, (d_x, d_y, d_bp, pg)), = rec.calls['_hc_width_bwd']
    assert same(a[0], x) and same(a[3], stats) and a[6:8] == (mode, rpb) and same(a[5], ng)
    assert all(same(p, q) for p, q in zip(a[4], params)) and len(a[4]) == 7
    for i, nm in ((8, 'd_branch'), (9, 'd_res'), (10, 'd_beta')):
        assert torch.equal(a[i], inp[nm]), nm
    if fused:
        assert same(a[1], extra[0]) and same(a[2], extra[1])
        ce('d_y', extra[0].grad, d_y)
        ce('d_beta_prev', extra[1].grad, d_bp)
    else:
        assert a[1] is None and a[2] is None
    ce('d_x', x.grad, d_x)
    for i, p in enumerate(params):
        ce(f'param {i}', p.grad, pg[i].reshape(p.shape))
    if mode:
        ce('norm gain', ng.grad, pg[7])
    else:
        assert pg[7] is None


def test_hc_depth(pkg):
    """ops.HcDepth: out = res + beta y (one product and one add, or one FMA: gamma_2, bf16); backward: d_res is the incoming gradient
    bit for bit, d_y = sum_s beta d_out (gamma_S, bf16), d_beta = sum_d d_out y (gamma_D, fp32). T = 450, D = 200, 4 streams."""
    T, D = 450, 200
    g = rng(110)
    res, y = rnd((T, S, D), g, grad=True), rnd((T, D), g, grad=True)
    beta = (torch.randn((T, S), device=dev(), generator=g) + 1).requires_grad_()
    out = pkg.ops.HcDepth.apply(res, y, beta)
    t = beta.detach().to(F64)[..., None] * y.detach().to(F64)[:, None]
    want = res.detach().to(F64) + t
    cb('out', out, want, gamma(2) * (res.detach().to(F64).abs() + t.abs()))
    d_out = rnd((T, S, D), g)
    out.backward(d_out)
    ce('d_res', res.grad, d_out)
    t = beta.detach().to(F64)[..., None] * d_out.to(F64)
    cb('d_y', y.grad, t.sum(1), gamma(S) * t.abs().sum(1))
    t = d_out.to(F64) * y.detach().to(F64)[:, None]
    cf('d_beta', beta.grad, t.sum(2), gamma(D) * t.abs().sum(2))


def test_dwconv_node(pkg, pool):
    """ops.DwConv on [B*Np, D] rows with the model's mask (B = 3, Np = 150, one element fully masked): the node passes B, Np and the
    mask to both launches and returns dweight in the parameter's [D, 1, k] shape; every output against dw_ref of
    test_gpu_conv_melspec_kernels with its bounds (zero initial accumulators, as the zero pool hands them out)."""
    B, Np, D, ks = 3, 150, 64, 31
    T = B * Np
    g = rng(120)
    x = rnd((T, D), g, grad=True)
    w = (torch.randn((D, 1, ks), device=dev(), generator=g) * ks ** -0.5).requires_grad_()
    b = param((D,), g, 0.5)
    mask = row_mask(B, Np, [150, 90, 0])
    pool.begin(dev())
    y = pkg.ops.DwConv.apply(x, w, b, mask, B, Np)
    assert y.grad_fn.meta == (B, Np)
    pre = y.grad_fn.saved_tensors[4]
    dy = rnd((T, D), g)
    y.backward(dy)
    slab_only(pool)
    m = mask.bool().cpu()
    r = dw_ref(h64(x).view(B, Np, D), m, h64(w).view(D, ks), h64(b), h64(dy).view(B, Np, D), h64(pre).view(B, Np, D))
    mm = m[..., None].expand(B, Np, D).reshape(T, D).to(dev())
    cb('pre', pre, r['conv'].reshape(T, D).to(dev()), r['e_pre'].reshape(T, D).to(dev()))
    for nm, got, key in (('y', y, 'y'), ('dx', x.grad, 'dx')):
        ref, e = r[key].reshape(T, D).to(dev()), r['e_' + key].reshape(T, D).to(dev())
        cb(nm, got.detach()[mm], ref[mm], e[mm])
        ce(f'{nm} masked rows', got.detach()[~mm], torch.zeros_like(got.detach()[~mm]))
    n = B * cdiv(Np, CV_TN) * CV_TN + 1
    assert w.grad.shape == w.shape
    cf('dweight', w.grad.view(D, ks), r['dW'].to(dev()), gamma(n) * r['dWabs'].to(dev()) + r['dWcar'].to(dev()))
    cf('dbias', b.grad, r['db'].to(dev()), gamma(n) * r['dbabs'].to(dev()) + r['dbcar'].to(dev()))


# ============================================================================================================ zero pool
def test_zero_pool_slices(pkg):
    """one step's slices (sizes around the 32-float alignment and 2-D shapes) are zero, 128-byte aligned, inside the slab and
    disjoint: each keeps its own fill after all are written"""
    ops = pkg.ops
    p = ops._ZeroPool()
    shapes = [1, 31, 32, 33, 100, 7, (3, 5), (200, 5), 4096, 5, (4, 5)]
    p.begin(dev())
    assert p.buf is None
    first = [p.zeros(s, dev()) for s in shapes]        # no slab yet: torch.zeros
    assert all(bool((t == 0).all()) for t in first)
    p.begin(dev())
    assert p.buf is not None
    got = [p.zeros(s, dev()) for s in shapes]
    lo, hi = p.buf.data_ptr(), p.buf.data_ptr() + 4 * p.buf.numel()
    spans = []
    for s, t in zip(shapes, got):
        assert tuple(t.shape) == (tuple(s) if isinstance(s, tuple) else (s,)) and t.dtype == F32
        ce(f'slice {s}', t, torch.zeros_like(t))
        a = t.data_ptr()
        assert a % 128 == 0 and lo <= a and a + 4 * t.numel() <= hi
        spans.append((a, a + 4 * t.numel()))
    spans.sort()
    for (a0, a1), (b0, b1) in zip(spans, spans[1:]):
        assert a1 <= b0, 'two slices of one step overlap'
    for i, t in enumerate(got):
        t.fill_(i + 1)
    for i, t in enumerate(got):
        assert bool((t == i + 1).all()), f'slice {i} was overwritten by another slice'


FF_POOL = dict(B=3, Np=150, Din=128, inner=128)


def ff_step(pkg, rec, P, xs, dys):
    """forwards of every x in xs in one step, one backward; -> (y, references of the pooled gradients) of each forward"""
    ops = pkg.ops
    B, Np = FF_POOL['B'], FF_POOL['Np']
    ops.zero_pool.begin(dev())
    ys = [ff_apply(ops, P, x, B, Np, 0.0, 0, None) for x in xs]
    rec.clear()
    torch.autograd.backward(ys, dys)
    return ys


def ff_single_refs(pkg, rec, P, x, dy):
    """the pooled gradients of one forward and backward, and their references (each gradient is then cleared)"""
    y, = ff_step(pkg, rec, P, [x], [dy])
    refs = ff_pool_refs(rec, y.detach(), dy, P['cs'], FF_POOL['B'], FF_POOL['inner'] // 64)
    for k in ('b1', 'b2', 'cs'):
        P[k].grad = None
    return refs


def summed(ra, rb):
    """two gradients added by autograd: each within its bound, and the fp32 sum rounds once"""
    return {k: (ra[k][0] + rb[k][0], ra[k][1] + rb[k][1] + U * ((ra[k][0] + rb[k][0]).abs() + ra[k][1] + rb[k][1])) for k in ra}


def check_pooled(P, refs, tag):
    for k in ('b1', 'b2', 'cs'):
        cf(f'd_{k} {tag}', P[k].grad, *refs[k])


@pytest.mark.parametrize('how', ['one_backward', 'two_steps'])
def test_zero_pool_accumulation(pkg, rec, pool, how):
    """FeedForward (gate, bias and GEGLU bias gradients all come from the pool): two forwards summed into one backward, or two steps
    without zeroing the gradients, give the sum of the two single-forward gradients (their bounds add, plus the rounding of the sum)"""
    c = FF_POOL
    P = ff_make(c['B'], c['Np'], c['Din'], c['inner'], True, 130)
    g = P['g']
    T = c['B'] * c['Np']
    xa, xb = rnd((T, c['Din']), g, grad=True), rnd((T, c['Din']), g, grad=True)
    da, db = rnd((T, c['Din']), g), rnd((T, c['Din']), g)
    ra = ff_single_refs(pkg, rec, P, xa, da)
    rb = ff_single_refs(pkg, rec, P, xb, db)
    if how == 'one_backward':
        ff_step(pkg, rec, P, [xa, xb], [da, db])
        slab_only(pool)
    else:
        ff_step(pkg, rec, P, [xa], [da])
        ff_step(pkg, rec, P, [xb], [db])
        slab_only(pool)
    check_pooled(P, summed(ra, rb), how)


def test_zero_pool_fallback(pkg, rec, monkeypatch):
    """a step whose demand exceeds the slab sized from the previous step: the accumulators that still fit come from the slab, the
    rest from torch.zeros, and every gradient is exact to its bound"""
    ops = pkg.ops
    p = ops._ZeroPool()
    monkeypatch.setattr(ops, 'zero_pool', p)
    c = FF_POOL
    small = ff_make(1, 64, 64, 128, True, 140)
    x = rnd((64, 64), small['g'], grad=True)
    p.begin(dev())
    ff_apply(ops, small, x, 1, 64, 0.0, 0, None).backward(rnd((64, 64), small['g']))
    P = ff_make(c['B'], c['Np'], 512, 2048, True, 141)
    T = c['B'] * c['Np']
    x = rnd((T, 512), P['g'], grad=True)
    dy = rnd((T, 512), P['g'])
    p.begin(dev())
    y = ff_apply(ops, P, x, c['B'], c['Np'], 0.0, 0, None)
    rec.clear()
    y.backward(dy)
    n = p.buf.numel()
    assert p.used > n, 'the step fits the slab: the fallback is not reached'
    inside = lambda t: p.buf.data_ptr() <= t.data_ptr() < p.buf.data_ptr() + 4 * n
    assert inside(P['cs'].grad) and inside(P['b2'].grad)     # the first two accumulators fit; the GEGLU bias one does not
    check_pooled(P, ff_pool_refs(rec, y.detach(), dy, P['cs'], c['B'], 2048 // 64), 'fallback')
