"""Element-wise float64 bounds for the kernel tests: the bound classes, the running-bound arithmetic `Rv`, the checks and the
fixtures every GPU test module shares (a module imports the `pkg` fixture by name).

Each entry point runs on the GPU and is compared, element by element, with a float64 restatement of the same operation computed
on the host from the exact bf16 / fp32 tensors the kernel received. Every bound belongs to one of three classes:
  E  bit-identical to the torch expression (copies, casts, packing, gathers: __float2bfloat16 and Tensor.to(torch.bfloat16) both
     round to nearest even).
  F  fp32 outputs: a sum of n terms is within gamma(n) * sum|terms| of the exact sum for ANY order of the additions (so for warp
     shuffles and atomics too), plus the documented error of the fp32 library functions and intrinsics the kernel calls (CUDA C++
     Programming Guide, appendix "Mathematical Functions": expf, sinf/cosf/sincosf, erff 2 ulp, log1pf 1 ulp, powf 4 ulp,
     __expf 2 + floor(1.173 |x|) ulp; correctly rounded + - * / and sqrtf).
  B  bf16 outputs: one round-to-nearest of an fp32 value within `atol` of the exact one (check_b).

The F bounds of a longer sequence of operations are carried by `Rv`: each intermediate of the kernel's sequence of operations is held
as its exact float64 value `v` and a bound `e` on the distance of the kernel's fp32 value from it. Each operation adds the propagated
error of its inputs (taken at the largest magnitude the computed inputs can have, |v| + e) and its own roundings (standard model
fl(a op b) = (a op b)(1 + d), |d| <= u; a sum or inner product of n terms in any order, warp shuffles and atomics included, is within
gamma_n sum|terms|: Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., (3.4)-(3.5)). A restatement checked against an
independent float64 reference must agree with it to a thousandth of its own bound (`agree`).
"""
import math

import numpy as np
import pytest
import torch

F64, BF16, F32 = torch.float64, torch.bfloat16, torch.float32
U = 2.0 ** -24      # fp32 unit roundoff (24-bit significand, round to nearest)
U16 = 2.0 ** -8     # bf16 unit roundoff (8-bit significand)


@pytest.fixture(scope='module')
def pkg():
    import e2_tts_pytorch_b200 as pkg
    assert torch.cuda.is_available()
    pkg.lib.load()
    return pkg


def dev():
    return torch.device('cuda:0')


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def stream():
    return torch.cuda.current_stream().cuda_stream


def nans(shape, dtype):
    return torch.full(shape, float('nan'), device=dev(), dtype=dtype)


def h64(t):
    return t.detach().to(F64).cpu()


def gen(seed):
    return torch.Generator().manual_seed(seed)


# ---------------------------------------------------------------------------------------------------------------------- bounds
def gamma(n):
    """Higham's gamma_n = n u / (1 - n u) (Accuracy and Stability of Numerical Algorithms, 2nd ed., eqs. (3.4), (4.4)): a sum of
    n + 1 terms, or an inner product of n terms, evaluated in fp32 in any order is within gamma_n * sum|terms| of the exact value."""
    return n * U / (1 - n * U)


def sig_err(a):
    """|sigmoidf_(fl(x + b)) - sigmoid(x + b)| for the kernels' 1 / (1 + __expf(-a)):  the fp32 add of logit and bias rounds
    (<= u|a|, sigmoid' <= 1/4); __expf(-a) is within 2 + floor(1.173|a|) ulp, i.e. 2(2 + 1.173|a|) u relative, which moves
    1 / (1 + e) by sigma (1 - sigma) times that (<= 1/4 of it); 1 + e and the division round once each (<= 2u sigma <= 2u)."""
    a = a.abs()
    return U * (a / 4 + (2 + 1.173 * a) / 2 + 2)


def _report(name, got, ref, bound):
    over = (got - ref).abs() - bound
    over = torch.where(torch.isnan(over), torch.full_like(over, math.inf), over)
    i = int(torch.argmax(over))
    idx = tuple(int(j) for j in np.unravel_index(i, tuple(ref.shape))) if ref.dim() else ()
    return (f'{name}: |got - ref| exceeds the bound at {idx}: got {got.flatten()[i].item():.9g}, ref {ref.flatten()[i].item():.9g}, '
            f'bound {bound.flatten()[i].item():.3g}; {int((over > 0).sum())} of {ref.numel()} elements')


def check_f(name, got, ref, bound):
    """element-wise |got - ref| <= bound (F: the caller derives the bound; NaN never passes)"""
    ref = ref.detach().to(F64).cpu()
    got = got.detach().to(F64).cpu().reshape(ref.shape)
    bound = torch.as_tensor(bound, dtype=F64).cpu().expand_as(ref)
    ok = (got - ref).abs() <= bound
    assert bool(ok.all()), _report(name, got, ref, bound)


def check_b(name, got, ref, atol):
    """B: got = bf16(v) with v an fp32 value, |v - ref| <= atol. Round to nearest with an 8-bit significand moves v by at most
    2^-8 |v|, so |got - ref| <= 2^-8 |v| + atol <= 2^-8 |ref| + (1 + 2^-8) atol."""
    assert got.dtype == BF16, got.dtype
    ref = ref.detach().to(F64).cpu()
    check_f(name, got, ref, U16 * ref.abs() + (1 + U16) * torch.as_tensor(atol, dtype=F64).cpu())


def check_e(name, got, want):
    """E: bit-identical, compared as integers (so +0 and -0 differ); bf16, fp32 and int32"""
    got, want = got.detach().cpu().contiguous(), want.detach().cpu().contiguous()
    assert got.dtype == want.dtype and got.shape == want.shape, (name, got.dtype, want.dtype, got.shape, want.shape)
    it = {BF16: torch.int16, F32: torch.int32, torch.int32: torch.int32}[got.dtype]
    bad = got.view(it) != want.view(it)
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        idx = tuple(int(j) for j in np.unravel_index(i, tuple(got.shape)))
        raise AssertionError(f'{name}: {int(bad.sum())} of {bad.numel()} elements differ, first at {idx}: '
                             f'got {got.flatten()[i].item()!r}, want {want.flatten()[i].item()!r}')


def check_zero(name, got):
    check_e(name, got, torch.zeros_like(got.cpu()))


def bf16_ulp(x):
    """spacing of bf16 numbers at |x| (8-bit significand; subnormal spacing 2^-133 below 2^-126)"""
    e = torch.floor(torch.log2(x.abs().clamp(min=2.0 ** -126)))
    return torch.pow(2.0, e - 7)


# ---------------------------------------------------------------------------------------------------------------- running bounds
class Rv:
    """exact float64 value v of an fp32 quantity of the kernel, and a bound e on |kernel value - v|"""

    def __init__(self, v, e=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e + torch.zeros_like(v)

    def mag(self):
        return self.v.abs() + self.e

    def __getitem__(self, i):
        return Rv(self.v[i], self.e[i])

    def reshape(self, *shape):
        return Rv(self.v.reshape(*shape), self.e.reshape(*shape))


def exact(t):
    return Rv(h64(t))


def _rnd(v, p, n=1):
    """n roundings of a result whose inputs carry the propagated error p"""
    return Rv(v, p + gamma(n) * (v.abs() + p))


def mul(a, b, n=1):
    return _rnd(a.v * b.v, a.mag() * b.e + a.e * b.v.abs(), n)


def add(a, b, n=1):
    return _rnd(a.v + b.v, a.e + b.e, n)


def neg(a):
    return Rv(-a.v, a.e)


def fma(a, b, c):
    return _rnd(a.v * b.v + c.v, a.mag() * b.e + a.e * b.v.abs() + c.e, 1)


def dots(pairs, n):
    """sum of inner products einsum(eq, a, b) over n terms in all, any order"""
    v = p = m = 0
    for eq, a, b in pairs:
        v = v + torch.einsum(eq, a.v, b.v)
        p = p + torch.einsum(eq, a.mag(), b.e) + torch.einsum(eq, a.e, b.v.abs())
        m = m + torch.einsum(eq, a.mag(), b.mag())
    return Rv(v, p + gamma(n) * m)


def dot(eq, a, b, n):
    return dots([(eq, a, b)], n)


def mono(a, f, rel, lo=None):
    """f monotone on [v - e, v + e] (clipped below at lo), result rounded with relative error rel"""
    v = f(a.v)
    x0 = a.v - a.e if lo is None else torch.clamp(a.v - a.e, min=lo)
    p = torch.maximum((f(a.v + a.e) - v).abs(), (f(x0) - v).abs())
    return Rv(v, p + rel * (v.abs() + p))


def to_bf16(a):
    return Rv(a.v, a.e + U16 * a.mag())


def ones_rv(*shape):
    return Rv(torch.ones(*shape, dtype=F64))


def agree(name, r, ref):
    """the restatement r computes the reference value to a thousandth of its bound; returns the bound to hold the kernel to"""
    ref = ref.detach().to(F64).cpu().reshape(r.v.shape)
    slack = 1e-3 * r.e + 1e-12 * ref.abs() + 1e-300
    bad = (r.v - ref).abs() > slack
    assert not bool(bad.any()), f'{name}: the float64 restatement disagrees with the reference ({int(bad.sum())} elements)'
    return ref, r.e + slack


def chk_f(name, got, r, ref):
    ref, bound = agree(name, r, ref)
    check_f(name, got, ref, bound)


def chk_b(name, got, r, ref):
    """r: the fp32 value before the kernel's final bf16 rounding"""
    ref, bound = agree(name, r, ref)
    check_b(name, got, ref, bound)


# ---------------------------------------------------------------------------------------------- GEMM outputs, compared on the device
# The references of GEMM-shaped outputs are computed on the device in float64: the cfg2 shapes are too large for the host.
def ref64(A, B):
    """exact-operand float64 product and the accumulation bound gamma_K * sum |a b|"""
    a, b = A.to(F64), B.to(F64)
    return a @ b.t(), gamma(A.shape[1]) * (a.abs() @ b.abs().t())


def operands(M, N, K, seed, scale=1.0):
    """bf16 A [M, K] and B [N, K] (B scaled), drawn on the device"""
    g = torch.Generator(device=dev()).manual_seed(seed)
    A = torch.randn(M, K, device=dev(), generator=g).to(BF16)
    B = (torch.randn(N, K, device=dev(), generator=g) * scale).to(BF16)
    return A, B


def nan_out(M, ld, fp32=False):
    return torch.full((M, ld), float('nan'), device=dev(), dtype=F32 if fp32 else BF16)


# ------------------------------------------------------------------------------- restated host selection of the GEMM (b200_gemm)
def item_shape(M, N, force_tile=0):
    """(rows, cols) of one CTA tile"""
    wide = force_tile == 3 or (force_tile == 0 and M >= 512 and N >= 256)
    if wide:
        return 128, 256
    return (128 if force_tile == 1 else (256 if (force_tile == 2 or M >= 256) else 128)), 128


def work_items(M, N, K, force_tile=0, split_k=1):
    """(work items, splits, k-blocks per split)"""
    r, c = item_shape(M, N, force_tile)
    tiles = -(-M // r) * -(-N // c)
    kb = -(-K // 64)
    split = split_k if split_k > 1 else 1
    if split_k < 0:
        units = sms()
        s_fill = (units + tiles // 2) // tiles
        while s_fill > 1 and tiles * s_fill > units:
            s_fill -= 1
        split = max(1, min(max(s_fill, 1), max(kb // 8, 1), 64))
    split = min(split, kb)
    per = -(-kb // split)
    split = -(-kb // per)
    return tiles * split, split, per


def cta_tiles(M, N, K, force_tile=0):
    """Per CTA of the persistent launch (no split-K), the tiles it runs in order: (tm, tn, slices), with `slices` the 64 x 64 output
    slices each consumer warpgroup stages for that tile. Work item w = blockIdx.x + i * grid, grid = min(items, SMs); tm = w % tiles_m,
    tn = w // tiles_m. A warpgroup's slice counter runs on across its CTA's tiles and picks the staging buffer (and residual barrier)
    by its parity."""
    r, c = item_shape(M, N, force_tile)
    tiles_m = -(-M // r)
    items = work_items(M, N, K, force_tile)[0]
    grid = min(items, sms())
    per_col = lambda tn: -(-min(c, N - tn * c) // 64) * (r // 128)
    return [[(w % tiles_m, w // tiles_m, per_col(w // tiles_m)) for w in range(b, items, grid)] for b in range(grid)]


def odd_starts(ctas):
    """number of tiles that begin on an odd slice count of their warpgroup (the staging buffer 1 and the barrier phase that go with it)"""
    n = 0
    for tiles in ctas:
        done = 0
        for _, _, s in tiles:
            n += done & 1
            done += s
    return n


def assert_close(name, got, ref, bound):
    got = got.to(F64)
    err = (got - ref).abs()
    bad = ~(err <= bound)            # NaN fails
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0, 0])
        idx = divmod(i, ref.shape[1])
        raise AssertionError(f'{name}: {int(bad.sum())} of {ref.numel()} elements out of bound, first at {idx}: '
                             f'got {got.flatten()[i].item():.9g}, ref {ref.flatten()[i].item():.9g}, bound {bound.flatten()[i].item():.3g}')


def check_bf16(name, got, ref, acc_bound, extra=0.0):
    """bf16 output: one rounding of an fp32 value within acc_bound (+ extra) of ref"""
    b = acc_bound + extra
    assert_close(name, got, ref, b + U16 * (ref.abs() + b))


def drop_mask(seed, rows, hidden):
    """kept (True) / dropped pattern of the GEGLU epilogue, restated in torch integer arithmetic (ptx.cuh drop_words):
    pair = (row * hidden + col) >> 1 (low 32 bits); x = pair * 0x9E3779B1 + seedmix; x ^= x >> 15; word = x * (0x85EBCA6B for even
    col, 0xC2B2AE35 for odd col), all mod 2^32; keep iff word >= thresh16 << 16."""
    M32 = 0xFFFFFFFF
    seedmix = (seed & M32) ^ (((seed >> 32) * 0x85EBCA77) & M32)
    r = torch.arange(rows, dtype=torch.int64, device=dev())[:, None]
    c = torch.arange(hidden, dtype=torch.int64, device=dev())[None, :]
    pair = ((r * hidden + c) >> 1) & M32
    x = (pair * 0x9E3779B1 + seedmix) & M32
    x = x ^ (x >> 15)
    word = torch.where(c % 2 == 0, (x * 0x85EBCA6B) & M32, (x * 0xC2B2AE35) & M32)
    return word
