"""The head-dim-128 attention kernels of csrc/attn_tc.cu at the shapes where their schedules have edges, in every logit regime.

Forward (attn_fwd_wgmma_kernel<*, 128>): one CTA per (128-query tile, head, batch) on 64-key tiles through a 3-stage K / V ring; each
consumer warp picks its tanh evaluation (degree-5 polynomial, degree 9, or tanh.approx for the outliers) over its 16 query rows x 64
keys, with the dot products over all 128 dims, over the rows the TMA boxes read: past a head's end the next head's, past the tensor's
end zeros (attn_ref.warp_tile_amax, whose tiles are this kernel's).
Backward (attn_bwd_d128_wgmma_kernel): one CTA per (64-key tile, head, batch); the query tiles run in the order (j + kt) % nq through
a 3-stage Q / dO ring; warpgroup 0 computes S^T and warpgroup 1 dP^T and each hands the other half of its fragment over through one
fp32 exchange buffer, so warpgroup w scores query columns 32 w .. 32 w + 31; the lse / delta of the next query tile travel through a
two-slot buffer; each warpgroup adds its 64 dQ columns into dq as two 32-float TMA reduction boxes on a [B*H, N', 128] map. The
backward's per-warp choice between `tanh_poly2` everywhere and `tanh_poly2` / tanh.approx per element changes no value (both branches
evaluate `tanh_poly2` for |x| <= 0.5), so only the forward's degree-5 / degree-9 choice bears on isolation.

Every output starts NaN-filled and is held to the element-wise float64 bounds of attn_ref.restate (clamped and unclamped;
the Rv method of kernel_checks.py), the restatement itself to float64 autograd where the size allows. Rows without
a valid key give exactly o = 0, lse = -inf, dq = 0. Exact properties are held bit for bit. The host tests at the end feed the same
checks the restated values with one schedule fault injected each and require every fault to be rejected."""
import math

import pytest
import torch

import attn_ref
from attn_ref import TQ, TQB, assert_regime, attn_bwd, attn_fwd, attn_inputs, autograd64, dropout_keep, host_maskbits, restate
from kernel_checks import BF16, F32, F64, U, Rv, agree, check_b, check_e, check_f, dev, gamma, h64, pkg

DH = 128
TKB = 64            # keys per backward CTA
QDO_STAGES = 3      # the backward's Q / dO ring
H100_SMS = 132      # H100 SXM
W = 1e-3            # relative window of assert_regime around each polynomial threshold


# ------------------------------------------------------------------------------------------------------------------ launch rules
def fwd_grid(B, H, Np):
    return (-(-Np // TQ), H, B)


def fwd_last_query_tile(Np):
    """rows of the last forward query tile: up to 64 the second consumer warpgroup has no row of the head"""
    return Np - TQ * (fwd_grid(1, 1, Np)[0] - 1)


def bwd_grid(B, H, Np):
    return (-(-Np // TKB), H, B)


def bwd_last_key_tile(Np):
    return Np - TKB * (bwd_grid(1, 1, Np)[0] - 1)


def bwd_query_order(Np, kt):
    """the query tiles key-tile CTA kt visits, in order"""
    nq = -(-Np // TQB)
    return [(j + kt) % nq for j in range(nq)]


def ctas(grid):
    return grid[0] * grid[1] * grid[2]


def forward_choice_isolated(regime, uvalid):
    """a launch on a slice of the batch or of the heads makes, for every valid query row, the forward's choice of the big launch: the
    unclamped kernels choose nothing; in 'deg5' assert_regime has proven every warp tile, the neighbours' rows included, within the
    degree-5 range (zeros past the tensor's end keep it there); otherwise every valid warp tile must lie beyond that range, where
    the degree-9 and mixed paths evaluate the same polynomial per element"""
    if regime in ('big', 'deg5'):
        return True
    return bool((uvalid > 0.15 * (1 + W)).all())


# ------------------------------------------------------------------------------------------------------------------ cases
# (name, B, H, N', logit regime, softclamp (None: unclamped), dropout, per-batch masks, gate, per-(b, h) isolation)
CASES = [
    ('n33-b1-h1-deg5', 1, 1, 33, 'deg5', 50.0, 0.0, ('edges',), True, False),
    ('n64-b2-h3-deg9-nogate', 2, 3, 64, 'deg9', 50.0, 0.0, ('edges', 'tail'), False, False),
    ('n65-b2-h3-mixed-empty', 2, 3, 65, 'mixed', 50.0, 0.0, ('edges', 'empty'), True, True),
    ('n127-b3-h2-tanh', 3, 2, 127, 'tanh', 50.0, 0.0, ('tail', 'edges', 'random'), True, True),
    ('n160-b2-h2-unclamped-big-empty', 2, 2, 160, 'big', None, 0.0, ('random', 'empty'), True, True),
    ('n193-b2-h3-clamp64-sat', 2, 3, 193, 'sat', 64.0, 0.0, ('edges', 'random'), True, False),
    ('n255-b2-h2-mixed-dropout', 2, 2, 255, 'mixed', 50.0, 0.1, ('edges', 'tail'), True, False),
    ('n225-b2-h2-unclamped-big-dropout-nogate', 2, 2, 225, 'big', None, 0.1, ('tail', 'edges'), False, False),
    ('n385-b2-h2-mixed-nogate-empty', 2, 2, 385, 'mixed', 50.0, 0.0, ('edges', 'empty'), False, True),
    ('n448-b1-h2-deg9-unmasked', 1, 2, 448, 'deg9', 50.0, 0.0, ('none',), True, False),
    ('n577-b4-h16-mixed-dropout-waves', 4, 16, 577, 'mixed', 50.0, 0.1, ('tail', 'random', 'edges', 'none'), True, False),
    ('n1056-b2-h4-mixed', 2, 4, 1056, 'mixed', 50.0, 0.0, ('tail', 'random'), True, False),
    ('n2080-b1-h2-deg5', 1, 2, 2080, 'deg5', 50.0, 0.0, ('tail',), True, False),
]


def test_attention_d128_cases_cover_the_edges():
    """the cases above reach every edge of both schedules (checked on the host)"""
    Nps = [c[3] for c in CASES]
    assert {1, 32, 33, 63, 64} <= {bwd_last_key_tile(Np) for Np in Nps}           # keys in the last backward key tile
    nqs = {-(-Np // TQB) for Np in Nps}
    assert {1, 2, 3, 4} <= nqs and max(nqs) >= 7                                   # the Q / dO ring: never wraps, once, many times
    for Np in Nps:
        for kt in range(bwd_grid(1, 1, Np)[0]):
            assert sorted(bwd_query_order(Np, kt)) == list(range(-(-Np // TQB)))   # every CTA visits every query tile once
    assert any(Np % TQB == 1 and H > 1 for _, _, H, Np, *_ in CASES)               # a one-row last query tile next to another head
    assert {1, 64, 65, 127} <= {fwd_last_query_tile(Np) for Np in Nps}             # second consumer warpgroup idle or partial
    assert any(B * H * Np < TQB for _, B, H, Np, *_ in CASES)                      # the whole tensor inside one 64-row box
    n_ctas = [ctas(bwd_grid(B, H, Np)) for _, B, H, Np, *_ in CASES]
    assert min(n_ctas) < H100_SMS and max(n_ctas) > 2 * H100_SMS                  # below one wave, beyond two
    regimes = {(c[4], c[5]) for c in CASES}
    assert {'deg5', 'deg9', 'mixed', 'tanh'} <= {r for r, cl in regimes if cl == 50.0}
    assert ('sat', 64.0) in regimes and ('big', None) in regimes
    assert {'edges', 'tail', 'random', 'none', 'empty'} <= {k for c in CASES for k in c[7]}
    for unclamped in (False, True):
        sub = [c for c in CASES if (c[5] is None) == unclamped]
        assert any(c[6] > 0 and c[3] % 2 == 1 for c in sub)                        # dropout at odd N' (row pitch N' + 1)
        assert any(not c[8] for c in sub)                                          # no gate
        assert any(c[9] for c in sub)                                              # per-(b, h) isolation
    assert {1056, 2080} <= set(Nps)                                                # cfg2-like sequence lengths
    assert all(c[6] == 0 for c in CASES if c[9])                                   # isolation keeps the dropout counters: no dropout
    assert max(B * H * Np * Np for _, B, H, Np, *_ in CASES) <= 577 * 577 * 64     # the host float64 restatement stays affordable


# ------------------------------------------------------------------------------------------------------------------ checks
def delta_ref(r, gate, B, H, Np):
    """ws_delta = gate <dOg, o> with the kernel's own o: a 128-term fp32 dot product, then one product with the gate"""
    g4 = h64(gate).view(B, Np, H).permute(0, 2, 1) if gate is not None else torch.ones(B, H, Np, dtype=F64)
    return r['dgate_own'] * g4, gamma(DH + 1) * r['dgate_e'] / gamma(DH) * g4


def check_outputs(name, B, H, Np, gate, fw, bw, r):
    """every output of one forward + backward against the restatement r"""
    ok = r['row_ok']
    okq = ok[..., None].expand(B, H, Np, DH)
    zero = torch.zeros(B, H, Np, DH, dtype=F64)
    sel = lambda t: (torch.where(okq, t.v, zero), torch.where(okq, t.e, zero))
    merge = lambda t: t.permute(0, 2, 1, 3).reshape(B * Np, H * DH)
    check_b(f'{name} o', fw['o'], *sel(r['o']))
    ogv, oge = sel(r['og'])
    check_b(f'{name} og', fw['og'], merge(ogv), merge(oge))
    lse_k = fw['lse'].cpu()
    check_f(f'{name} lse', lse_k[ok].contiguous(), r['lse'].v[ok], r['lse'].e[ok])
    if gate is not None:
        okg = ok.permute(0, 2, 1).reshape(B * Np, H)
        dgo = torch.where(okg, r['dgate_own'].permute(0, 2, 1).reshape(B * Np, H), 0.)
        check_f(f'{name} d_gate', bw['d_gate'], dgo, r['dgate_e'].permute(0, 2, 1).reshape(B * Np, H))
    check_f(f'{name} ws_delta', bw['ws_delta'], *delta_ref(r, gate, B, H, Np))
    check_b(f'{name} ws_dO', bw['ws_dO'], r['dO'].v, U * r['dO'].v.abs())
    check_b(f'{name} dv', bw['dv'], r['dv'].v, r['dv'].e)
    check_b(f'{name} dk', bw['dk'], r['dk'].v, r['dk'].e)
    check_f(f'{name} dq', bw['dq'], *sel(r['dq']))
    # rows without a valid key: exactly zero output and dq, lse = -inf
    if not bool(ok.all()):
        assert bool(torch.isneginf(lse_k[~ok]).all()), f'{name}: lse of rows without a valid key'
        assert bool((fw['o'].cpu()[~ok] == 0).all()), f'{name}: o of rows without a valid key'
        assert bool((bw['dq'].cpu()[~ok] == 0).all()), f'{name}: dq of rows without a valid key'
        assert bool((fw['og'].cpu().view(B, Np, H, DH).permute(0, 2, 1, 3)[~ok] == 0).all()), f'{name}: og of rows without a valid key'


def run(pkg, q, k, v, gate, mask, dog, clamp, p_drop, seed, **kw):
    fw = attn_fwd(pkg, q, k, v, gate, mask, clamp, p_drop, seed, **kw)
    bw = attn_bwd(pkg, q, k, v, fw['o'], fw['lse'], gate, mask, dog, clamp, p_drop, seed, **kw)
    torch.cuda.synchronize()
    return fw, bw


@pytest.mark.gpu
@pytest.mark.parametrize('name,B,H,Np,regime,clamp,p_drop,masks,use_gate,iso', CASES, ids=[c[0] for c in CASES])
def test_attention_d128_schedule(pkg, name, B, H, Np, regime, clamp, p_drop, masks, use_gate, iso):
    seed = 8642097 + Np
    q, k, v, gate, m, mask, dog = attn_inputs(B, H, Np, regime, masks, use_gate, seed=Np * 29 + H, dh=DH)
    uvalid = assert_regime(regime, q, k, m, clamp)
    if p_drop > 0:
        assert Np % 2 == 1
    fw, bw = run(pkg, q, k, v, gate, mask, dog, clamp, p_drop, seed)
    assert torch.equal(fw['ws'].cpu(), host_maskbits(m, Np)), f'{name}: key bitmask'
    r = restate(q, k, v, gate, m, clamp, p_drop, seed, dog, fw['o'], fw['lse'])
    ok = r['row_ok']
    if B * H * Np * Np <= 3_000_000:
        ag = autograd64(q, k, v, gate, m, clamp, p_drop, seed, dog)
        for key in ('o', 'lse', 'dq', 'dk', 'dv'):
            s = ok if key in ('o', 'lse', 'dq') else torch.ones_like(ok)
            agree(f'{name} {key} (restatement vs float64 autograd)', Rv(r[key].v[s], r[key].e[s]), ag[key][s])
    check_outputs(name, B, H, Np, gate, fw, bw, r)
    if 'empty' in masks:
        assert not bool(ok.any(-1).any(-1).all())                                 # a batch element without a valid key
    if iso:
        # (E) each (b, h) launched alone (B = H = 1): its warp tiles read zeros past the head instead of the next head's rows
        assert clamp is None or bool((uvalid > 0.15 * (1 + W)).all())
        for b in range(B):
            for hh in range(H):
                sl = lambda t: t[b:b + 1, hh:hh + 1].contiguous()
                gs = gate.view(B, Np, H)[b, :, hh:hh + 1].contiguous() if gate is not None else None
                ms = mask[b:b + 1].contiguous() if mask is not None else None
                dogs = dog.view(B, Np, H, DH)[b, :, hh].contiguous()
                f1, b1 = run(pkg, sl(q), sl(k), sl(v), gs, ms, dogs, clamp, p_drop, seed)
                tag = f'{name} isolation b{b} h{hh}'
                check_e(f'{tag} o', f1['o'], sl(fw['o']))
                check_e(f'{tag} og', f1['og'], fw['og'].view(B, Np, H, DH)[b, :, hh])
                check_e(f'{tag} lse', f1['lse'], fw['lse'][b:b + 1, hh:hh + 1])
                check_e(f'{tag} dk', b1['dk'], sl(bw['dk']))
                check_e(f'{tag} dv', b1['dv'], sl(bw['dv']))
                if gate is not None:
                    check_e(f'{tag} d_gate', b1['d_gate'], bw['d_gate'].view(B, Np, H)[b, :, hh:hh + 1])
                okq = r['row_ok'][b:b + 1, hh:hh + 1, :, None]
                check_f(f'{tag} dq', b1['dq'], torch.where(okq, r['dq'].v[b:b + 1, hh:hh + 1], 0.),
                        torch.where(okq, r['dq'].e[b:b + 1, hh:hh + 1], 0.))
    if B > 1 and regime != 'deg9':
        # (E) batch element 0 launched alone (B = 1, the same (b, h) rows and dropout counters): only dq is summed in an order that
        # depends on the launch. ('deg9' cases may hold valid warp tiles on both sides of the degree-5 threshold.)
        assert forward_choice_isolated(regime, uvalid)
        sl = lambda t: t[0:1].contiguous()
        gs = gate.view(B, Np, H)[0].contiguous() if gate is not None else None
        dogs = dog.view(B, Np, H * DH)[0].contiguous()
        f1, b1 = run(pkg, sl(q), sl(k), sl(v), gs, sl(mask) if mask is not None else None, dogs, clamp, p_drop, seed)
        for key in ('dk', 'dv'):
            check_e(f'{name} alone {key}', b1[key], sl(bw[key]))
        if gate is not None:
            check_e(f'{name} alone d_gate', b1['d_gate'], bw['d_gate'].view(B, Np, H)[0])
        okq = r['row_ok'][0:1, ..., None]
        check_f(f'{name} alone dq', b1['dq'], torch.where(okq, r['dq'].v[0:1], 0.), torch.where(okq, r['dq'].e[0:1], 0.))


@pytest.mark.gpu
@pytest.mark.parametrize('clamp', [50.0, None])
def test_attention_d128_shared_bitmask_and_device_seed(pkg, clamp):
    """maskbits_ready = 1 with the bitmask of ops.attn_maskbits, and seed + *seed_dev wrapping mod 2^64, reproduce the per-call
    bitmask and the summed seed bit for bit (E); the ready bitmask is only read"""
    B, H, Np, p_drop = 3, 2, 193, 0.1
    q, k, v, gate, m, mask, dog = attn_inputs(B, H, Np, 'mixed', ('edges', 'tail', 'random'), True, seed=97, dh=DH)
    base, addend = 0x0123456789ABCDEF, 0xFEDCBA9876543211
    total = (base + addend) % 2 ** 64
    assert base + addend >= 2 ** 64
    ref_f, ref_b = run(pkg, q, k, v, gate, mask, dog, clamp, p_drop, total)
    shared = pkg.ops.attn_maskbits(mask, B, Np, dev())
    torch.cuda.synchronize()
    assert torch.equal(shared.cpu(), host_maskbits(m, Np))
    sd = torch.tensor([addend - 2 ** 64], dtype=torch.int64, device=dev())
    f, b = run(pkg, q, k, v, gate, None, dog, clamp, p_drop, base, ws=shared, ready=1, seed_dev=sd)   # keymask unused when ready
    assert torch.equal(shared.cpu(), host_maskbits(m, Np))
    for key in ('o', 'og', 'lse'):
        check_e(f'shared bitmask + device seed {key}', f[key], ref_f[key])
    for key in ('dk', 'dv', 'd_gate', 'ws_dO', 'ws_delta'):
        check_e(f'shared bitmask + device seed {key}', b[key], ref_b[key])
    keep = dropout_keep(total, B, H, Np, p_drop)
    assert 0.05 < 1 - float(keep.double().mean()) < 0.15                # the summed seed's dropout pattern is the one applied
    r = restate(q, k, v, gate, m, clamp, p_drop, total, dog, f['o'], f['lse'])
    check_outputs('device seed', B, H, Np, gate, f, b, r)


# ------------------------------------------------------------------------------------------------------------------ tightness
# A small head-dim-128 case on the host: the restated outputs pass the checks above, and each with one fault of the kind the
# backward schedule can make is rejected by them.
TB, TH, TN, TCLAMP, TDROP, TSEED = 2, 2, 65, 50.0, 0.1, 0x5EED5


def _host_case():
    q, k, v, gate, m, mask, dog = attn_inputs(TB, TH, TN, 'deg5', ('edges', 'random'), True, seed=17, dh=DH, device='cpu')
    r0 = restate(q, k, v, gate, m, TCLAMP, TDROP, TSEED, dog, torch.zeros(q.shape, dtype=BF16), torch.zeros(TB, TH, TN))
    o_k = r0['o'].v.to(BF16)                     # what a kernel within its bounds returns for the saved forward outputs
    lse_k = r0['lse'].v.to(F32)
    r = restate(q, k, v, gate, m, TCLAMP, TDROP, TSEED, dog, o_k, lse_k)
    assert bool(r['row_ok'].all())
    return (q, k, v, gate, m, dog, o_k, lse_k), r


@pytest.fixture(scope='module')
def host_case():
    return _host_case()


def _rejects(check, name, got, *ref):
    with pytest.raises(AssertionError):
        check(name, got, *ref)


def test_d128_checks_accept_the_restatement(host_case):
    """the unfaulted restated values pass every check the faults below must fail"""
    (q, k, v, gate, m, dog, o_k, lse_k), r = host_case
    check_b('dv', r['dv'].v.to(BF16), r['dv'].v, r['dv'].e)
    check_b('dk', r['dk'].v.to(BF16), r['dk'].v, r['dk'].e)
    check_f('dq', r['dq'].v.to(F32), r['dq'].v, r['dq'].e)
    dv, de = delta_ref(r, gate, TB, TH, TN)
    check_f('ws_delta', dv.to(F32), dv, de)


def _probs(q, k, m):
    """float64 softmax probabilities of the clamped logits and dP = dO V^T pick the positions where a fault shows most"""
    s = h64(q) @ h64(k).transpose(-1, -2) * DH ** -0.5
    lg = (TCLAMP * torch.tanh(s / TCLAMP)).masked_fill(~m[:, None, None, :], -math.inf)
    return torch.softmax(lg, -1)


@pytest.mark.parametrize('parity', [0, 1])
def test_d128_checks_reject_a_flipped_dropout_keep_bit(host_case, monkeypatch, parity):
    """one keep bit wrong at the even (parity 0) or odd (1) key of a hashed pair — the half a lane takes from its partner through
    the lane-pair shuffle — at a query column of warpgroup 1 (32 .. 63 of its tile), for dv and for dk"""
    (q, k, v, gate, m, dog, o_k, lse_k), r = host_case
    keep = dropout_keep(TSEED, TB, TH, TN, TDROP)
    p = _probs(q, k, m)
    dP = r['dO'].v @ h64(v).transpose(-1, -2)
    cols = (torch.arange(TN) % TQB >= 32)[:, None] & (torch.arange(TN) % 2 == parity)[None, :]
    for out, vis in (('dv', p), ('dk', p * dP.abs())):
        vis = torch.where(cols & m[:, None, None, :], vis, torch.zeros_like(vis))
        i = int(vis.flatten().argmax())
        flipped = keep.clone()
        flipped.view(-1)[i] = ~flipped.view(-1)[i]
        monkeypatch.setattr(attn_ref, 'dropout_keep', lambda *a: flipped)
        rf = restate(q, k, v, gate, m, TCLAMP, TDROP, TSEED, dog, o_k, lse_k)
        monkeypatch.undo()
        _rejects(check_b, f'flipped keep bit {out}', rf[out].v.to(BF16), r[out].v, r[out].e)


def test_d128_checks_reject_dq_landing_in_the_next_head(host_case):
    """the one-row last query tile's dq (N' % 64 == 1) added into row 0 of the next head instead of its own row"""
    (q, k, v, gate, m, dog, o_k, lse_k), r = host_case
    assert TN % TQB == 1
    dq = r['dq'].v.clone()
    dq[0, 1, 0] += dq[0, 0, TN - 1]
    _rejects(check_f, 'dq in the next head', dq.to(F32), r['dq'].v, r['dq'].e)


def test_d128_checks_reject_swapped_dq_boxes(host_case):
    """dq columns 32 .. 63 (warpgroup 0's second 32-float box) swapped with 64 .. 95 (warpgroup 1's first)"""
    (q, k, v, gate, m, dog, o_k, lse_k), r = host_case
    dq = r['dq'].v.clone()
    dq[..., 32:64], dq[..., 64:96] = r['dq'].v[..., 64:96], r['dq'].v[..., 32:64]
    _rejects(check_f, 'dq boxes swapped', dq.to(F32), r['dq'].v, r['dq'].e)


def test_d128_checks_reject_dv_without_keep_scale(host_case):
    """dv without the deferred 1 / (1 - p) of the dropped probabilities"""
    (q, k, v, gate, m, dog, o_k, lse_k), r = host_case
    ks = 65536 / (65536 - int(TDROP * 65536))
    _rejects(check_b, 'dv without 1 / (1 - p)', (r['dv'].v / ks).to(BF16), r['dv'].v, r['dv'].e)


def test_d128_checks_reject_delta_off_by_one_bf16_ulp(host_case):
    """delta of one row computed with one element of dO one bf16 ulp off, at the largest |dO o| of the tensor: the change is at least
    2^-8 of that term, the bound gamma_129 times a sum of 128 terms at most 2^-9.9 of it"""
    (q, k, v, gate, m, dog, o_k, lse_k), r = host_case
    dv, de = delta_ref(r, gate, TB, TH, TN)
    t = (r['dO'].v * h64(o_k)).abs()
    b, hh, i, e = (int(x) for x in (t == t.max()).nonzero()[0])
    x = float(r['dO'].v[b, hh, i, e])
    ulp = 2.0 ** (math.floor(math.log2(abs(x))) - 7)
    bad = dv.clone()
    bad[b, hh, i] += ulp * float(h64(o_k)[b, hh, i, e])
    _rejects(check_f, 'delta off by one ulp of dO', bad.to(F32), dv, de)
