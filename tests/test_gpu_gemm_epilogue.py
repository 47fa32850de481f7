"""The fused epilogue of the wgmma GEMM (csrc/gemm.cu) on each of its paths, held element by element to a float64 restatement.

Paths, chosen per call from the output and residual bases:
  TMA tile stores (bf16 D 16-byte aligned) with a TMA-staged residual (R 16-byte aligned): each 64 x 64 residual slice is loaded into
    the staging buffer its output slice uses next; a warpgroup's slice counter `nslice` picks the buffer (nslice & 1) and the parity
    of its barrier ((nslice >> 1) & 1), and it runs on across the tiles of the persistent CTA;
  TMA tile stores with a residual read from global memory inside the fragment loop (R 4- but not 16-byte aligned: resid_ldg);
  fragment stores (D not 16-byte aligned, bf16 rows of N % 8 != 0 columns, or fp32 D): store_pair, bf16x2 / float2 / scalar.
Every case runs the aligned and the 8-byte-offset D and R, and an fp32 D, and asserts:
  - each element within the float64 bound of `epilogue64` (kernel order: bias, GELU, gate, mask, residual; one fp32 rounding each);
  - path invariance: the four bf16 results are bit-identical, and equal to the fp32 result rounded to bf16 (round to nearest even,
    as pack_bf16 and __float2bfloat16_rn);
  - masked rows equal the residual bit for bit (+0.0 without one);
  - untouched memory: the output's pad columns and the rows past M stay NaN;
  - the residual's pad columns and rows past M are NaN, so a map or load with the wrong pitch or extent shows as a NaN.
Each schedule case asserts with `cta_tiles` the property it exists for (a tile that starts on an odd slice count, a warpgroup wholly
past M, ...). Products are computed on the device in float64 (`ref64`).
"""
import math

import pytest
import torch

from kernel_checks import (BF16, F32, F64, U, assert_close, check_bf16, cta_tiles, dev, item_shape, nan_out, odd_starts, operands,
                           pkg, ref64)

pytestmark = pytest.mark.gpu

GELU_SLOPE = 1.13   # max |gelu'(x)| = 1.1289 (at x = sqrt(2))
GELU_POLY = 5e-7    # absolute error of gemm.cu's gelu_erf2 in fp32 arithmetic


def rnd8(n):
    return (n + 7) // 8 * 8


def epilogue64(ref, acc, bias=None, colscale=None, rows_per_batch=0, rowmask=None, resid=None, act=0):
    """(want, bound) of the epilogue applied to ref64's (product, accumulation bound), in the kernel's order; each fp32 operation adds
    one rounding of the value it produces (taken at its largest magnitude |v| + e)."""
    v, e = ref, acc
    if bias is not None:
        v = v + bias.to(F64)
        e = e + U * (v.abs() + e)
    if act:
        g = v * 0.5 * (1 + torch.erf(v / math.sqrt(2)))
        e = GELU_SLOPE * e + GELU_POLY + U * g.abs()
        v = g
    if colscale is not None:
        cs = colscale.to(F64).repeat_interleave(rows_per_batch, 0)[:ref.shape[0]]
        v = v * cs
        e = cs.abs() * e + U * (v.abs() + cs.abs() * e)
    if rowmask is not None:
        mk = rowmask.to(F64)[:, None]
        v, e = v * mk, e * mk
    if resid is not None:
        v = v + resid.to(F64)
        e = e + U * (v.abs() + e)
    return v, e


def same_bits(name, got, want):
    it = torch.int16 if got.dtype == BF16 else torch.int32
    bad = got.contiguous().view(it) != want.contiguous().view(it)
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0, 0])
        idx = divmod(i, got.shape[1])
        raise AssertionError(f'{name}: {int(bad.sum())} of {bad.numel()} elements differ in their bits, first at {idx}: '
                             f'got {got.flatten()[i].item()!r}, want {want.flatten()[i].item()!r}')


def untouched(name, buf, M, c0, N):
    """everything of buf outside rows [0, M) x columns [c0, c0 + N) is still NaN"""
    assert bool(buf[M:].isnan().all()), f'{name}: a row past M was written'
    for side, cols in (('before', buf[:, :c0]), ('after', buf[:, c0 + N:])):
        hit = ~cols.isnan().all(0)
        assert not bool(hit.any()), f'{name}: {int(hit.sum())} columns {side} the output were written, rows {int((~cols.isnan()).any(1).sum())}'


def placed(vals, off, ld, extra_rows=3):
    """vals [M, n] copied into a NaN buffer [M + extra_rows, ld] at column off: (buffer, view of the values)"""
    M, n = vals.shape
    buf = nan_out(M + extra_rows, ld, fp32=vals.dtype == F32)
    buf[:M, off:off + n] = vals
    return buf, buf[:M, off:]


def run(pkg, name, M, N, K, *, seed, force_tile=0, a_mn=False, b_mn=False, K1=0, bias=False, rpb=0, mask=False, resid='own',
        ldd=None, ldr=None, rcol=0, act=0, ldf=None):
    """One GEMM with the requested epilogue, four ways (D and R each aligned or 8 bytes off; with act D is always aligned) plus an
    fp32 D of pitch ldf. resid: None, 'own' (a tensor of its own at column rcol of pitch ldr) or 'A' (the first A source itself,
    N == its K, ldr = lda). Returns the bf16 result."""
    A, B = operands(M, N, K, seed, scale=K ** -0.5)
    ref, acc = ref64(A, B)
    g = torch.Generator(device=dev()).manual_seed(seed + 1)
    bias_t = torch.randn(N, device=dev(), generator=g) if bias else None
    cs = torch.rand(-(-M // rpb), N, device=dev(), generator=g) + 0.5 if rpb else None
    mk = (torch.rand(M, device=dev(), generator=g) > 0.25).to(torch.uint8) if mask else None

    # A operand(s), K-major ones in NaN-padded buffers (the pad lies outside the operand maps)
    KA = K1 if K1 else K
    if a_mn:
        assert resid != 'A'
        At = A.t().contiguous()
        A1, lda, A2, lda2 = At[:KA].contiguous(), M, (At[KA:].contiguous() if K1 else None), M
    else:
        lda = rnd8(KA) + 8
        A1buf, A1 = placed(A[:, :KA], 0, lda, extra_rows=0)
        A2, lda2 = (A[:, K1:].contiguous(), K - K1) if K1 else (None, 0)
    Bin, ldb = (B.t().contiguous(), N) if b_mn else (B, K)

    if resid == 'A':
        assert N == KA and not a_mn
        rvals = A[:, :KA]
        rviews = [(A1, lda)]
    elif resid == 'own':
        rvals = torch.randn(M, N, device=dev(), generator=g).to(BF16)
        ldr = ldr or rnd8(rcol + N + 4) + 8
        rviews = [(placed(rvals, rcol + off, ldr)[1], ldr) for off in (0, 4)]   # R 16-byte aligned, then 8 bytes off
        assert rviews[0][0].data_ptr() % 16 == 0 and rviews[1][0].data_ptr() % 16 == 8
    else:
        rvals, rviews = None, [(None, 0)]

    want, bound = epilogue64(ref, acc, bias_t, cs, rpb, mk, rvals, act)
    ldd = ldd or rnd8(N + 4) + 8
    kw = dict(lda=lda, A2=A2, lda2=lda2, K1=K1, a_mn=a_mn, b_mn=b_mn, ldb=ldb, bias=bias_t, colscale=cs, rows_per_batch=rpb, rowmask=mk,
              force_tile=force_tile, act=act)
    masked = (mk == 0) if mask else None

    def check_masked(tag, got):
        if masked is not None and bool(masked.any()):
            exp = rvals[masked].to(got.dtype) if rvals is not None else torch.zeros_like(got[masked])
            same_bits(f'{tag}: masked rows', got[masked], exp)

    first = None
    for doff in ((0,) if act else (0, 4)):
        for R, ldr_ in rviews:
            rs = 'none' if R is None else 'aligned' if R.data_ptr() % 16 == 0 else '+8 B'
            tag = f'{name}: D {"aligned" if doff == 0 else "+8 B"}, R {rs}'
            dbuf = nan_out(M + 3, ldd)
            out = dbuf[:, doff:]
            assert (out.data_ptr() % 16 == 0) == (doff == 0)
            pkg.ops.gemm(A1, Bin, M, N, K, out=out, ldd=ldd, resid=R, ldr=ldr_, **kw)
            got = dbuf[:M, doff:doff + N]
            check_bf16(tag, got, want, bound)
            untouched(tag, dbuf, M, doff, N)
            check_masked(tag, got)
            if first is None:
                first = got.clone()
            else:
                same_bits(f'{tag}: against D aligned, R aligned', got, first)
    if not act:
        ldf = ldf or N + 1
        fbuf = nan_out(M + 3, ldf, fp32=True)
        pkg.ops.gemm(A1, Bin, M, N, K, out=fbuf, ldd=ldf, out_fp32=True, resid=rviews[0][0], ldr=rviews[0][1], **kw)
        tag = f'{name}: fp32 D, ldd {ldf}'
        got = fbuf[:M, :N]
        assert_close(tag, got, want, bound)
        untouched(tag, fbuf, M, 0, N)
        check_masked(tag, got)
        same_bits(f'{tag}: rounded to bf16, against the bf16 D', got.to(BF16), first)
    return first


# ---------------------------------------------------------------------------------------------- slice parity across tiles
# tile rows, N, force_tile, slices per warpgroup of the last tile column. 128 x 256: N - 256 in (0, 64], (64, 128], (128, 192],
# (192, 256]; 128 x 128: N - 128 in (0, 64], (64, 128]; 256 x 128 (two m64 blocks per warpgroup): N = 136 leaves an 8-wide last
# column, whose second residual slice is the next m64 block's (the r0 + 64 load of the mainloop).
@pytest.mark.parametrize('N,force_tile,slices', [
    (296, 3, 1), (360, 3, 2), (392, 3, 3), (512, 3, 4),
    (296, 0, 1), (392, 0, 3),
    (168, 1, 1), (200, 1, 2),
    (136, 2, 2), (136, 0, 2),
])
def test_slice_parity(pkg, N, force_tile, slices):
    K = 192
    rows, cols = item_shape(100000, N, force_tile)
    M = 199 * rows + 40        # more row tiles than SMs: CTAs run tiles of both columns; the last row tile's second warpgroup is past M
    assert item_shape(M, N, force_tile) == (rows, cols)
    ctas = cta_tiles(M, N, K, force_tile)
    last = [s for tiles in ctas for _, tn, s in tiles if tn == -(-N // cols) - 1]
    assert set(last) == {slices}
    if slices % 2:
        assert odd_starts(ctas) > 0, 'no tile starts on an odd slice count'
    run(pkg, f'parity {rows}x{cols} N {N}', M, N, K, seed=N + force_tile, force_tile=force_tile)


def test_cross_condition_forward_production(pkg):
    """CrossCondition forward at cfg2 with d = 320: x2 [4T, 320] and the text [4T, 256] as two A sources, + x2 as the residual. The
    128 x 256 tile's last column is 64 wide (one slice), so the tiles a CTA runs after one of those start on odd slice counts."""
    M, D, Dt = 4 * 16 * 1056, 320, 256
    assert item_shape(M, D) == (128, 256)
    ctas = cta_tiles(M, D, D + Dt)
    assert max(len(c) for c in ctas) >= 2 and odd_starts(ctas) > 0
    run(pkg, 'cross-condition forward', M, D, D + Dt, seed=3, K1=D, resid='A')


def test_cross_condition_backward_form(pkg):
    """two-source A, MN-major B (the CrossCondition backward's dx GEMM), + the first A source as the residual"""
    M, D, Dt = 2 * 16 * 1056, 320, 256
    ctas = cta_tiles(M, D, D + Dt)
    assert odd_starts(ctas) > 0
    run(pkg, 'cross-condition backward', M, D, D + Dt, seed=4, K1=D, b_mn=True, resid='A')


# ---------------------------------------------------------------------------------------------- row and K edges
@pytest.mark.parametrize('M,force_tile', [(20 * 128 + 40, 1), (10 * 256 + 40, 2), (20 * 128 + 40, 3), (40, 0), (40, 1), (40, 2), (40, 3)])
def test_row_edges(pkg, M, force_tile):
    """the last row tile's second warpgroup (or both m64 blocks of it) lies wholly past M and still waits on its residual barriers"""
    N, K = 392, 128
    rows, _ = item_shape(M, N, force_tile)
    assert M % rows == 40
    run(pkg, f'rows M {M} tile {force_tile}', M, N, K, seed=M + force_tile, force_tile=force_tile, bias=True, rpb=M, mask=True)


@pytest.mark.parametrize('K', [64, 128, 200, 1000])
def test_k_edges(pkg, K):
    """K = 64 and 128: both first residual loads go out in the tile's first k-block; 200 and 1000 end in a partial k-block"""
    for ft in (1, 2, 3):
        run(pkg, f'K {K} tile {ft}', 1000, 392, K, seed=K + ft, force_tile=ft, bias=True, mask=True)


# ---------------------------------------------------------------------------------------------- epilogue combinations
@pytest.mark.parametrize('a_mn,b_mn', [(False, False), (False, True), (True, False), (True, True)])
def test_residual_operand_majorness(pkg, a_mn, b_mn):
    for ft in (1, 2, 3):
        run(pkg, f'resid a_mn {a_mn} b_mn {b_mn} tile {ft}', 1096, 520, 320, seed=10 + ft + 4 * a_mn + 8 * b_mn, force_tile=ft,
            a_mn=a_mn, b_mn=b_mn)
    run(pkg, f'resid two-source a_mn {a_mn} b_mn {b_mn}', 1096, 520, 320, seed=30 + 4 * a_mn + 8 * b_mn, K1=192, a_mn=a_mn, b_mn=b_mn)


@pytest.mark.parametrize('rpb', [274, 1056, 0])
def test_bias_gate_mask_residual(pkg, rpb):
    """rows_per_batch 0 here stands for M: one gate row for all rows, as the Vocos pw2 GEMM calls it"""
    M = 2 * 1056 + 100
    rpb = rpb or M
    for ft in (0, 1, 2, 3):
        run(pkg, f'bias + gate + mask + resid, rpb {rpb}, tile {ft}', M, 392, 256, seed=rpb + ft, force_tile=ft, bias=True, rpb=rpb,
            mask=True)


@pytest.mark.parametrize('force_tile', [1, 2, 3])
def test_gelu_bias_gate_mask_residual(pkg, force_tile):
    """act = ACT_GELU with every other epilogue: one instantiation per tile (K-major only; D aligned, R aligned or not)"""
    M, N = 199 * item_shape(100000, 392, force_tile)[0] + 40, 392
    run(pkg, f'GELU tile {force_tile}', M, N, 192, seed=50 + force_tile, force_tile=force_tile, bias=True, rpb=1056, mask=True, act=1)
    # and without a residual: the plain TMA store path with the activation
    run(pkg, f'GELU no resid tile {force_tile}', 1000, N, 192, seed=60 + force_tile, force_tile=force_tile, bias=True, rpb=274,
        mask=True, resid=None, act=1)
    # N % 8 != 0: the activation on the fragment-store path
    run(pkg, f'GELU N 100 tile {force_tile}', 1000, 100, 192, seed=65 + force_tile, force_tile=force_tile, bias=True, rpb=274,
        mask=True, act=1)


@pytest.mark.parametrize('N', [99, 100, 321])
def test_output_width_not_whole_16_byte_units(pkg, N):
    """bf16 rows of N % 8 != 0 columns end in a partial 16-byte unit, which a TMA tile store would write past column N: such outputs
    leave from the fragments, and the columns after them stay untouched"""
    for ft in (1, 2, 3):
        run(pkg, f'N {N} plain tile {ft}', 1096, N, 192, seed=100 + N + ft, force_tile=ft, resid=None)
        run(pkg, f'N {N} epilogue tile {ft}', 1096, N, 192, seed=110 + N + ft, force_tile=ft, bias=True, rpb=274, mask=True)


# ---------------------------------------------------------------------------------------------- residual geometry
def test_residual_pitch_differs_from_output(pkg):
    for ft in (1, 2, 3):
        run(pkg, f'ldr != ldd tile {ft}', 1096, 520, 320, seed=70 + ft, force_tile=ft, ldd=536, ldr=600, bias=True, mask=True)


def test_residual_column_window(pkg):
    """the residual is columns [64, 64 + N) of a wider tensor (ldr > N, 16-byte aligned base)"""
    for ft in (1, 2, 3):
        run(pkg, f'resid window tile {ft}', 1096, 392, 320, seed=80 + ft, force_tile=ft, rcol=64, ldr=1024, rpb=274, mask=True)


def test_residual_is_the_a_operand(pkg):
    for ft in (1, 2, 3):
        run(pkg, f'resid = A tile {ft}', 1096, 320, 320, seed=90 + ft, force_tile=ft, resid='A', bias=True, mask=True)


# ---------------------------------------------------------------------------------------------- fp32 outputs
@pytest.mark.parametrize('N,ldf', [(100, 100), (100, 101), (99, 99), (257, 263), (1026, 1026), (1026, 1027)])
def test_fp32_output_full_epilogue(pkg, N, ldf):
    """fp32 D without split-K through store_pair: float2 stores where the pair is 8-byte aligned, scalar ones otherwise (odd ldd
    alternates them by row, odd N ends each row on a single column); N = 100 is the pred head's, 1026 the Vocos head's n_fft + 2"""
    for ft in (0, 2, 3):
        run(pkg, f'fp32 N {N} ldd {ldf} tile {ft}', 1000, N, 256, seed=N + ldf + ft, force_tile=ft, bias=True, rpb=274, mask=True, ldf=ldf)


# ---------------------------------------------------------------------------------------------- refusals
def test_refusals(pkg):
    M, N, K = 256, 256, 256
    A, B = operands(M, N, K, 1)
    f32 = torch.zeros(M, N, device=dev(), dtype=F32)
    out = torch.zeros(M, N, device=dev(), dtype=BF16)
    bias = torch.zeros(N, device=dev())
    cs = torch.ones(1, N, device=dev())
    mk = torch.ones(M, device=dev(), dtype=torch.uint8)
    R = torch.zeros(M, N + 16, device=dev(), dtype=BF16)
    cases = [
        ('split-K with a bias', 'split-K supports no epilogue', dict(out=f32, out_fp32=True, split_k=2, bias=bias)),
        ('split-K with a residual', 'split-K supports no epilogue', dict(out=f32, out_fp32=True, split_k=2, resid=R, ldr=N + 16)),
        ('split-K with a gate', 'split-K supports no epilogue', dict(out=f32, out_fp32=True, split_k=2, colscale=cs, rows_per_batch=M)),
        ('split-K with a mask', 'split-K supports no epilogue', dict(out=f32, out_fp32=True, split_k=2, rowmask=mk)),
        ('GLU with a residual', 'GEGLU needs', dict(out=out, ldd=N // 2, geglu=True, resid=R, ldr=N + 16)),
        ('GLU with a gate', 'GEGLU needs', dict(out=out, ldd=N // 2, geglu=True, colscale=cs, rows_per_batch=M)),
        ('GLU with a mask', 'GEGLU needs', dict(out=out, ldd=N // 2, geglu=True, rowmask=mk)),
        ('residual pitch not a multiple of 8', 'residual pitch', dict(out=out, resid=R, ldr=N + 4)),
        ('residual base not 4-byte aligned', 'residual must be 4-byte aligned', dict(out=out, resid=R[:, 1:], ldr=N + 16)),
    ]
    for what, msg, kw in cases:
        with pytest.raises(RuntimeError, match=f'gemm: .*{msg}') as err:
            pkg.ops.gemm(A, B, M, N, K, **kw)
        assert 'b200_gemm failed' in str(err.value), what
    torch.cuda.synchronize()
    # nothing was launched into the outputs
    assert bool((f32 == 0).all()) and bool((out == 0).all())
