"""The persistent tile schedule of the wgmma GEMM (csrc/gemm.cu): every work item (CTA tile x K split) computed exactly once.

Every output buffer is filled with NaN before the call, so an item the schedule skips (NaN stays) or a split-K item added twice (the
bound breaks) cannot pass. Each element is compared with a float64 product of the exact bf16 operands (computed on the device in
float64: the cfg2 shapes are too large for the host). Bounds:
  fp32 accumulation: the products of two bf16 values are exact in fp32, so a K-term inner product accumulated in fp32 in any order
  (k-blocks, wgmma k16 steps, split-K atomics) is within gamma_K * sum_k |a_k b_k| of the exact value (Higham, Accuracy and
  Stability of Numerical Algorithms, 2nd ed., eq. (3.5)); fp32 epilogue operations (bias, gate, residual add) round once each.
  bf16 outputs: one round-to-nearest of that fp32 value: + 2^-8 |value| (bf16 unit roundoff).
The tile and split-K selections are restated in kernel_checks (item_shape, work_items) so that each case can assert which side of a
threshold it is on.
"""
import math

import pytest
import torch

from kernel_checks import (BF16, F32, F64, U, U16, assert_close, check_bf16, dev, drop_mask, item_shape, nan_out, operands, pkg, ref64,
                           sms, work_items)

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------- checks
def run_plain(pkg, M, N, K, seed, force_tile=0, b_mn=False, a_mn=False):
    A, B = operands(M, N, K, seed)
    ref, acc = ref64(A, B)
    ld = (N + 7) // 8 * 8
    out = nan_out(M, ld)
    Ain = A.t().contiguous() if a_mn else A
    Bin = B.t().contiguous() if b_mn else B
    pkg.ops.gemm(Ain, Bin, M, N, K, a_mn=a_mn, b_mn=b_mn, out=out, ldd=ld, force_tile=force_tile)
    check_bf16(f'{M}x{N}x{K} tile {force_tile}', out[:, :N], ref, acc)


def run_dw(pkg, M, N, K, seed, split_k=-1, force_tile=0):
    """dW = dY^T X: both operands MN-major, fp32 out, split-K partials through atomics (the output is zeroed by the call)"""
    A, B = operands(M, N, K, seed)
    ref, acc = ref64(A, B)
    out = nan_out(M, N, fp32=True)
    pkg.ops.gemm(A.t().contiguous(), B.t().contiguous(), M, N, K, lda=M, ldb=N, a_mn=True, b_mn=True, out=out, ldd=N, out_fp32=True,
                 split_k=split_k, force_tile=force_tile)
    assert_close(f'dW {M}x{N}x{K} split {split_k}', out, ref, acc)


# ---------------------------------------------------------------------------------------------- cfg2 shapes
T2 = 16 * 1056     # cfg2 tokens: B16 x (1024 frames + 32 registers)


@pytest.mark.parametrize('M,N,K,b_mn', [
    (T2, 1552, 512, False),     # fused qkv (audio)
    (T2, 1552, 256, False),     # fused qkv (text, K = 256: four k-blocks per item)
    (T2, 1024, 256, True),      # text dX
    (T2, 512, 256, True),
    (T2, 512, 2048, False),     # FF-out
    (T2, 2048, 512, True),
])
def test_cfg2_plain_shapes(pkg, M, N, K, b_mn):
    assert item_shape(M, N) == (128, 256)
    run_plain(pkg, M, N, K, seed=M + N + K, b_mn=b_mn)


def test_cfg2_out_proj_gate_and_mask(pkg):
    """out-projection: AdaLN gate (per-batch column scale) + row mask"""
    M, N, K = T2, 512, 512
    A, B = operands(M, N, K, 5, scale=0.1)
    ref, acc = ref64(A, B)
    g = torch.Generator(device=dev()).manual_seed(6)
    cs = torch.rand(16, N, device=dev(), generator=g) + 0.5
    mask = (torch.rand(M, device=dev(), generator=g) > 0.1).to(torch.uint8)
    out = nan_out(M, N)
    pkg.ops.gemm(A, B, M, N, K, out=out, ldd=N, colscale=cs, rows_per_batch=1056, rowmask=mask)
    csr = cs.to(F64).repeat_interleave(1056, 0)
    mk = mask.to(F64)[:, None]
    # the fp32 product with the gate rounds once more: U |acc * cs|
    check_bf16('out-proj', out, ref * csr * mk, (acc * csr + U * (ref * csr).abs()) * mk)


@pytest.mark.parametrize('N,b_mn', [(512, False), (512, True), (256, False)])
def test_cfg2_cross_condition_two_source(pkg, N, b_mn):
    """cross-conditioning: 4T rows (4 residual streams), A = [audio (K1 = 512) | text (256)] from two sources, + residual"""
    M, K, K1 = 4 * T2, 768, 512
    A, B = operands(M, N, K, 7 + N, scale=0.05)
    ref, acc = ref64(A, B)
    A1, A2 = A[:, :K1].contiguous(), A[:, K1:].contiguous()
    g = torch.Generator(device=dev()).manual_seed(8)
    resid = torch.randn(M, N, device=dev(), generator=g).to(BF16)
    out = nan_out(M, N)
    Bin = B.t().contiguous() if b_mn else B
    pkg.ops.gemm(A1, Bin, M, N, K, lda=K1, A2=A2, lda2=K - K1, K1=K1, b_mn=b_mn, out=out, ldd=N, resid=resid, ldr=N)
    want = ref + resid.to(F64)
    check_bf16('cross-condition', out, want, acc + U * want.abs())


@pytest.mark.parametrize('M,N', [(512, 512), (4096, 512), (256, 1024)])
def test_cfg2_weight_gradient_split_k(pkg, M, N):
    K = T2
    n, split, per = work_items(M, N, K, split_k=-1)
    assert split > 1 and per >= 8
    run_dw(pkg, M, N, K, seed=M + N)


# ---------------------------------------------------------------------------------------------- schedule edge cases
def test_odd_items_per_cta_and_fewer_items_than_ctas(pkg):
    # 3 * SMs + 5 items of 128 x 128: five CTAs run four items, the rest three
    n = 3 * sms() + 5
    M, N, K = 128 * n, 128, 192
    assert work_items(M, N, K, force_tile=1)[0] == n
    run_plain(pkg, M, N, K, seed=1, force_tile=1)
    # fewer items than CTAs: the grid shrinks to the items
    M, N = 320, 256
    n = work_items(M, N, K, force_tile=1)[0]
    assert n < sms()
    run_plain(pkg, M, N, K, seed=2, force_tile=1)
    # a single item
    run_plain(pkg, 100, 128, K, seed=3, force_tile=1)


@pytest.mark.parametrize('K', [64, 200, 1000])
def test_k_one_block_and_tail(pkg, K):
    """K = 64 is one k-block per item; 200 and 1000 end in a partial k-block (zero-filled by the TMA)"""
    for ft in (0, 2):
        for N in (520, 248):
            run_plain(pkg, 1000, N, K, seed=K + ft + N, force_tile=ft)


@pytest.mark.parametrize('force_tile', [0, 1, 2, 3])
def test_every_force_tile(pkg, force_tile):
    M, K = 1096, 320
    for N in (520, 248):
        for i, (a_mn, b_mn) in enumerate(((False, False), (False, True), (True, False), (True, True))):
            run_plain(pkg, M, N, K, seed=40 + 4 * force_tile + i + N, force_tile=force_tile, a_mn=a_mn, b_mn=b_mn)
    run_dw(pkg, M, 520, K, seed=50 + force_tile, split_k=3, force_tile=force_tile)


def test_two_source_k_split_inside_items(pkg):
    """the switch from the first to the second A source falls inside every item's k-range, and inside a split-K split"""
    M, N, K, K1 = 1096, 520, 640, 192
    A, B = operands(M, N, K, 60)
    ref, acc = ref64(A, B)
    A1, A2 = A[:, :K1].contiguous(), A[:, K1:].contiguous()
    for ft in (0, 1, 2, 3):
        for n in (N, 256):
            out = nan_out(M, 528)
            pkg.ops.gemm(A1, B, M, n, K, lda=K1, A2=A2, lda2=K - K1, K1=K1, out=out, ldd=528, force_tile=ft)
            check_bf16(f'two-source tile {ft} N {n}', out[:, :n], ref[:, :n], acc[:, :n])
    # MN-major two-source A with split-K (the hyper-connection parameter GEMM form): 10 k-blocks in splits of 4, the switch after 3
    At1, At2 = A1.t().contiguous(), A2.t().contiguous()
    out = nan_out(M, N, fp32=True)
    pkg.ops.gemm(At1, B, M, N, K, lda=M, A2=At2, lda2=M, K1=K1, a_mn=True, out=out, ldd=N, out_fp32=True, split_k=3)
    assert work_items(M, N, K, split_k=3)[1:] == (3, 4)
    assert_close('two-source split-K', out, ref, acc)


def test_split_k_at_the_64_cap(pkg):
    M, N, K = 64, 128, 64 * 640
    n, split, per = work_items(M, N, K, split_k=-1)
    assert split == 64 and n == 64
    run_dw(pkg, M, N, K, seed=70)


# ---------------------------------------------------------------------------------------------- GEGLU + dropout
@pytest.mark.parametrize('M,N,K', [(T2, 4096, 512), (T2, 2048, 256), (1096, 512, 320), (1096, 512, 192)])
def test_geglu_dropout(pkg, M, N, K):
    p, seed = 0.1, 1234
    A, W = operands(M, N, K, 80 + K, scale=0.1)
    g = torch.Generator(device=dev()).manual_seed(81)
    bias = torch.randn(N, device=dev(), generator=g) * 0.1
    ref, acc = ref64(A, W)
    z = ref + bias.to(F64)
    D2 = nan_out(M, N)
    H = N // 2
    out = nan_out(M, H)
    pkg.ops.gemm(A, W, M, N, K, out=out, ldd=H, D2=D2, ldd2=N, bias=bias, geglu=True, dropout_p=p, seed=seed)
    check_bf16('GEGLU pre-activations', D2, z, acc + U * z.abs())
    # h from the saved bf16 pre-activations, as the kernel (and the backward) do: packed [u(64) | gate(64)] per 128 columns
    zz = D2.to(F64).view(M, N // 128, 2, 64)
    u, gt = zz[:, :, 0].reshape(M, H), zz[:, :, 1].reshape(M, H)
    gelu = gt * 0.5 * (1 + torch.erf(gt / math.sqrt(2)))
    thresh16 = int(p * 65536)
    kept = drop_mask(seed, M, H) >= (thresh16 << 16)
    scale = 65536.0 / (65536 - thresh16)
    want = torch.where(kept, u * gelu * scale, torch.zeros_like(u))
    # dropped elements are exactly zero; the kept ones carry the GELU polynomial's 5e-7 absolute error times |u| and three fp32 roundings
    got = out.to(F64)
    assert bool((got[~kept] == 0).all()), 'a dropped hidden unit is not zero'
    assert_close('GEGLU value', got, want, (u.abs() * 5e-7 * scale + 4 * U * want.abs()) * (1 + U16) + U16 * want.abs())
    nz = kept & (want.abs() > 1e-30)
    assert bool((got[nz] != 0).all()), 'a kept hidden unit is zero'
    frac = 1 - float(kept.double().mean())
    assert abs(frac - thresh16 / 65536) < 0.01


# ---------------------------------------------------------------------------------------------- output paths
@pytest.mark.parametrize('offset', [0, 4])
def test_bf16_output_base_alignment(pkg, offset):
    """bf16 outputs leave through the smem staging slices and TMA tile stores when the base is 16-byte aligned (offset 0), and as
    bf16x2 stores from the fragments otherwise (offset 4 elements = 8 bytes); the columns before the output stay untouched"""
    M, N, K = 1096, 520, 320
    A, B = operands(M, N, K, 90 + offset, scale=0.1)
    ref, acc = ref64(A, B)
    g = torch.Generator(device=dev()).manual_seed(91)
    bias = torch.randn(N, device=dev(), generator=g)
    mask = (torch.rand(M, device=dev(), generator=g) > 0.2).to(torch.uint8)
    buf = nan_out(M, 528 + 8)
    out = buf[:, offset:]
    assert (out.data_ptr() % 16 == 0) == (offset == 0)
    pkg.ops.gemm(A, B, M, N, K, out=out, ldd=528 + 8, bias=bias, rowmask=mask)
    mk = mask.to(F64)[:, None]
    want = (ref + bias.to(F64)) * mk
    check_bf16('bf16 out', out[:, :N], want, (acc + U * want.abs()) * mk)
    assert bool(buf[:, :offset].isnan().all()) and bool(buf[:, offset + N:].isnan().all())
