"""The GLU epilogue of the wgmma GEMM (csrc/gemm.cu) through the staging slices and TMA tile stores, against its fragment-store path.

With 16-byte aligned bases for h (D), the pre-activations (D2) and glu_mult, the GLU GEMM writes u + bias, gate + bias and h as
64 x 64 slices through shared memory and TMA stores, with the tile's bias and glu_mult staged in shared memory by the producer. Output
bases that are 4- but not 16-byte aligned take the bf16x2 fragment stores. Both paths must give the same bits in h and in the
pre-activations, for every activation, with and without glu_mult, with dropout (host seed and device seed word), and on every tile.
Each case asserts:
  - h and the pre-activations are bit-identical between the two paths;
  - rows >= M and the pad columns of a wider pitch stay NaN on both paths (the TMA store clips at the tensor's extent);
and one test reads the GEMMTRACE line of each call in a child process, so that the comparison cannot pass by running one path twice.
"""
import os
import subprocess
import sys

import pytest
import torch

from kernel_checks import dev, operands, pkg  # noqa: F401

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16 = torch.bfloat16
PAD_ROWS = 3


def nan_buf(M, ld, off):
    """A NaN-filled [M + PAD_ROWS, ld] bf16 matrix whose base lies `off` elements past a 16-byte aligned allocation."""
    flat = torch.full(((M + PAD_ROWS) * ld + off,), float('nan'), device=dev(), dtype=BF16)
    return flat[off:].view(M + PAD_ROWS, ld)


def glu_call(pkg, M, N, K, *, act, mult, p=0.0, seed_dev=False, force_tile=0, ldd=None, ldd2=None, off=0, seed=11):
    """h [M + PAD_ROWS, ldd] and ug [M + PAD_ROWS, ldd2] from one GLU GEMM; off = 0 takes the TMA stores, off = 2 (4-byte aligned
    bases) the fragment stores. Operands are seeded by the shape, so both paths see the same inputs."""
    ldd = ldd or N // 2
    ldd2 = ldd2 or N
    torch.manual_seed(M * 7 + N * 3 + K)
    A = (torch.randn(M, K, device=dev()) * 0.5).to(BF16)
    W = (torch.randn(N, K, device=dev()) * 0.1).to(BF16)
    bias = torch.randn(N, device=dev()) * 0.3
    gm = 1 + 0.2 * torch.randn(N // 2, device=dev()) if mult else None
    sd = torch.tensor([12345], device=dev(), dtype=torch.int64) if seed_dev else None
    h, ug = nan_buf(M, ldd, off), nan_buf(M, ldd2, off)
    pkg.ops.gemm(A, W, M, N, K, out=h, ldd=ldd, D2=ug, ldd2=ldd2, bias=bias, geglu=act, dropout_p=p, seed=seed, seed_dev=sd,
                 glu_mult=gm, force_tile=force_tile)
    torch.cuda.synchronize()
    return h, ug


def bits(x):
    return x.contiguous().view(torch.int16)


def check_paths(pkg, M, N, K, **kw):
    h_t, ug_t = glu_call(pkg, M, N, K, off=0, **kw)
    h_f, ug_f = glu_call(pkg, M, N, K, off=2, **kw)
    assert h_t.data_ptr() % 16 == 0 and ug_t.data_ptr() % 16 == 0
    assert h_f.data_ptr() % 16 == 4 and ug_f.data_ptr() % 16 == 4
    for name, t, f, cols in (('h', h_t, h_f, N // 2), ('ug', ug_t, ug_f, N)):
        assert not bool(t[:M, :cols].isnan().any()), f'{name}: NaN inside the output'
        assert torch.equal(bits(t[:M, :cols]), bits(f[:M, :cols])), f'{name}: TMA and fragment paths differ'
        for path, x in (('tma', t), ('frag', f)):
            assert bool(x[M:].isnan().all()), f'{name} ({path}): rows >= M written'
            assert bool(x[:, cols:].isnan().all()), f'{name} ({path}): pad columns written'
    return h_t


@pytest.mark.parametrize('force_tile', [0, 1, 2, 3])
@pytest.mark.parametrize('mult', [False, True])
@pytest.mark.parametrize('act', [1, 2, 3])
def test_activation_tile(pkg, act, mult, force_tile):
    # M = 1000: a partial last 64-row band and 128-row tile; N = 384: the last 256-wide tile holds one 128-column group
    check_paths(pkg, 1000, 384, 192, act=act, mult=mult, p=0.1, force_tile=force_tile)


@pytest.mark.parametrize('seed_dev', [False, True])
@pytest.mark.parametrize('p', [0.0, 0.1, 0.25])
def test_dropout(pkg, p, seed_dev):
    h = check_paths(pkg, 520, 512, 128, act=1, mult=True, p=p, seed_dev=seed_dev)
    if p > 0:
        frac = float((h[:520, :256] == 0).float().mean())
        assert abs(frac - p) < 0.03, f'dropped fraction {frac} at p {p}'


@pytest.mark.parametrize('force_tile', [0, 1, 2, 3])
@pytest.mark.parametrize('M', [37, 64, 129])
def test_small_m_n128(pkg, M, force_tile):
    check_paths(pkg, M, 128, 64, act=2, mult=True, p=0.1, seed_dev=True, force_tile=force_tile)


@pytest.mark.parametrize('force_tile', [0, 1, 3])
def test_padded_pitch(pkg, force_tile):
    check_paths(pkg, 300, 640, 128, act=3, mult=True, p=0.25, ldd=320 + 24, ldd2=640 + 40, force_tile=force_tile)


@pytest.mark.parametrize('force_tile', [0, 1, 2])
def test_many_tiles_per_cta(pkg, force_tile):
    # more tiles than SMs at one k-block each: the per-tile bias / glu_mult hand-off between the producer and both consumer
    # warpgroups turns over many times in every CTA
    check_paths(pkg, 4100, 2048, 64, act=1, mult=True, p=0.1, seed_dev=True, force_tile=force_tile)


@pytest.mark.parametrize('act', [1, 2, 3])
def test_cfg2_text_shape(pkg, act):
    # the text feed-forward's FF-in GEMM of one cfg2 step: 16 x 1056 rows, inner 1024, K = 256
    check_paths(pkg, 16 * 1056, 2048, 256, act=act, mult=False, p=0.1, seed_dev=True)


_TRACE_CHILD = r'''
import sys, torch
sys.path.insert(0, sys.argv[1])
import e2_tts_pytorch_b200 as pkg
M, N, K = 200, 256, 64
A = torch.randn(M, K, device='cuda').to(torch.bfloat16)
W = torch.randn(N, K, device='cuda').to(torch.bfloat16)
for off in (0, 2):
    h = torch.empty(M * N // 2 + off, device='cuda', dtype=torch.bfloat16)[off:].view(M, N // 2)
    ug = torch.empty(M * N + off, device='cuda', dtype=torch.bfloat16)[off:].view(M, N)
    pkg.ops.gemm(A, W, M, N, K, out=h, D2=ug, ldd2=N, bias=torch.zeros(N, device='cuda'), geglu=2, dropout_p=0.1, seed=3)
    torch.cuda.synchronize()
    print('CALL', off, file=sys.stderr, flush=True)
'''


def test_path_taken(pkg):
    env = dict(os.environ, B200_GEMM_TRACE='1')
    r = subprocess.run([sys.executable, '-c', _TRACE_CHILD, ROOT], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stderr.splitlines() if ln.startswith('GEMMTRACE 200 256 64') or ln.startswith('CALL')]
    assert len(lines) == 4, r.stderr[-2000:]
    assert 'geglu=2' in lines[0] and lines[0].endswith('store=tma') and lines[1] == 'CALL 0', lines
    assert 'geglu=2' in lines[2] and lines[2].endswith('store=frag') and lines[3] == 'CALL 2', lines


def test_refusals_unchanged(pkg):
    M, N, K = 256, 256, 256
    A, B = operands(M, N, K, 1)
    h = torch.zeros(M, N // 2 + 8, device=dev(), dtype=BF16)
    ug = torch.zeros(M, N + 8, device=dev(), dtype=BF16)
    cases = [
        ('h pitch not a multiple of 8', 'GEGLU output pitch', dict(out=h, ldd=N // 2 + 4, D2=ug, ldd2=N)),
        ('pre-activation pitch not a multiple of 8', 'GEGLU output pitch', dict(out=h, ldd=N // 2, D2=ug, ldd2=N + 4)),
        ('N not a multiple of 128', 'GEGLU needs', dict(out=h, ldd=N // 2, D2=ug, ldd2=N, N=192)),
        ('bias not 16-byte aligned', 'GEGLU bias must be 16-byte aligned', dict(out=h, ldd=N // 2, D2=ug, ldd2=N,
                                                                              bias=torch.zeros(N + 4, device=dev())[1:])),
    ]
    for what, msg, kw in cases:
        n = kw.pop('N', N)
        with pytest.raises(RuntimeError, match=f'gemm: .*{msg}') as err:
            pkg.ops.gemm(A, B, M, n, K, geglu=True, **kw)
        assert 'b200_gemm failed' in str(err.value), what
    torch.cuda.synchronize()
    assert bool((h == 0).all()) and bool((ug == 0).all())
