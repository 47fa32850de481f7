"""GPU: the schedule of the attention backward kernel (csrc/attn_tc.cu) at the shapes where its edges lie.

Per 128-key CTA and 64-query tile, one consumer warpgroup reduces dQ over both warpgroups' dS^T tiles and adds it into dq with one
TMA tensor reduction on a [B*H, N', 64] map; a warpgroup whose 64 keys all lie at or past N' only keeps the barrier protocol. The cases
put 1, 32, 64, 65 and 127 valid keys into the last key tile (64 and 1 leave the second warpgroup without keys), a last query tile of
one row next to another head (a reduction at the wrong row or head coordinates lands in the neighbouring head's dq; the rows the box
covers past N' carry dS = 0, so these outputs cannot tell a clipped box from one that adds zeros there), grids below one wave and of
several waves, dropout at odd N' (the keep mask hashed once per key pair), clamped and unclamped. Every output of every head is held
to the element-wise float64 bounds of the restatement of tests/attn_ref.py, and a batch element launched alone gives
bit-identical dk, dv and d_gate: only dq is summed in an order that depends on the launch."""
import pytest
import torch

from attn_ref import assert_regime, attn_bwd, attn_fwd, attn_inputs, restate, unclamped_inputs
from kernel_checks import F64, check_b, check_e, check_f, pkg

pytestmark = pytest.mark.gpu

CLAMP = 50.0


def _run(pkg, unclamped, q, k, v, gate, mask, dog, p_drop, seed):
    clamp = None if unclamped else CLAMP
    fw = attn_fwd(pkg, q, k, v, gate, mask, clamp, p_drop, seed)
    bw = attn_bwd(pkg, q, k, v, fw['o'], fw['lse'], gate, mask, dog, clamp, p_drop, seed)
    torch.cuda.synchronize()
    return fw, bw


# (name, B, H, N', unclamped, dropout): key tiles of 128, query tiles of 64
CASES = [
    ('n129-last-key-tile-1-one-row-query-tile', 2, 3, 129, False, 0.0),
    ('n160-last-key-tile-32', 2, 2, 160, True, 0.0),
    ('n192-last-key-tile-64', 3, 2, 192, False, 0.0),
    ('n193-last-key-tile-65-dropout', 2, 3, 193, False, 0.1),
    ('n255-last-key-tile-127-dropout', 2, 2, 255, True, 0.1),
    ('n577-b4-h16-waves-dropout', 4, 16, 577, False, 0.1),
]


@pytest.mark.parametrize('name,B,H,Np,unclamped,p_drop', CASES, ids=[c[0] for c in CASES])
def test_attention_bwd_schedule(pkg, name, B, H, Np, unclamped, p_drop):
    seed = 424242 + Np
    if unclamped:
        q, k, v, gate, m, mask, dog = unclamped_inputs(B, H, Np, 'random', seed=Np * 13 + H)
    else:
        q, k, v, gate, m, mask, dog = attn_inputs(B, H, Np, 'mixed', ('tail', 'random'), True, seed=Np * 13 + H)
        # a batch element launched alone makes the same degree-5 / degree-9 choice per warp tile only outside the degree-5 range
        uvalid = assert_regime('mixed', q, k, m, CLAMP)
        assert bool((uvalid > 0.15 * (1 + 1e-3)).all())
    if p_drop > 0:
        assert Np % 2 == 1
    fw, bw = _run(pkg, unclamped, q, k, v, gate, mask, dog, p_drop, seed)
    if unclamped:
        r = restate(q, k, v, gate, m, None, p_drop, seed, dog, fw['o'], fw['lse'])
        okq = r['row_ok'][..., None].expand(B, H, Np, 64)
        zero = torch.zeros(B, H, Np, 64, dtype=F64)
        dq_v, dq_e = torch.where(okq, r['dq'].v, zero), torch.where(okq, r['dq'].e, zero)
    else:
        r = restate(q, k, v, gate, m, CLAMP, p_drop, seed, dog, fw['o'], fw['lse'])
        dq_v, dq_e = r['dq'].v, r['dq'].e
    check_b(f'{name} dv', bw['dv'], r['dv'].v, r['dv'].e)
    check_b(f'{name} dk', bw['dk'], r['dk'].v, r['dk'].e)
    check_f(f'{name} dq', bw['dq'], dq_v, dq_e)
    # batch element 0 launched alone (B = 1): the same (b, h) rows, dropout counters and key tiles
    gs = gate.view(B, Np, H)[0:1].reshape(Np, H).contiguous()
    dogs = dog.view(B, Np, H * 64)[0:1].reshape(Np, H * 64).contiguous()
    sl = lambda t: t[0:1].contiguous()
    f1, b1 = _run(pkg, unclamped, sl(q), sl(k), sl(v), gs, sl(mask), dogs, p_drop, seed)
    for key in ('dk', 'dv'):
        check_e(f'{name} alone {key}', b1[key], sl(bw[key]))
    check_e(f'{name} alone d_gate', b1['d_gate'], bw['d_gate'].view(B, Np, H)[0])
    check_f(f'{name} alone dq', b1['dq'], dq_v[0:1], dq_e[0:1])


def test_attention_bwd_schedule_cases_cover_the_edges():
    """the cases above reach every edge the schedule has (checked on the host)"""
    last_key_tile = {Np - 128 * ((Np - 1) // 128) for _, _, _, Np, _, _ in CASES}
    assert {1, 32, 64, 65, 127} <= last_key_tile
    assert any(Np % 64 == 1 and H > 1 for _, _, H, Np, _, _ in CASES)          # one-row last query tile next to another head
    ctas = [-(-Np // 128) * H * B for _, B, H, Np, _, _ in CASES]
    assert min(ctas) < 132 and max(ctas) > 2 * 132                             # below one wave and several waves of an H100 SXM
    assert {u for *_, u, _ in CASES} == {False, True} and any(p > 0 and Np % 2 for _, _, _, Np, _, p in CASES)
