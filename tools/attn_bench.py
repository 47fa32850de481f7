"""Developer tool (GPU): device time of the attention forward / backward kernels at a BASELINE shape, through the C ABI, for one
library build (B200_LIB selects it). usage: python tools/attn_bench.py [cfg2|cfg3] [iters] [variant]
variant (optional): 'unclamped' (no logit soft-clamp: the running-maximum kernels), 'nogate' (no head gate), 'plain' (neither);
without it, the reference's clamped, gated attention."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import e2_tts_pytorch_b200 as pkg
from e2_tts_pytorch_b200 import ops
dev = torch.device('cuda:0')
torch.manual_seed(0)
shape = sys.argv[1] if len(sys.argv) > 1 else 'cfg2'
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 20
variant = sys.argv[3] if len(sys.argv) > 3 else None
assert variant in (None, 'unclamped', 'nogate', 'plain'), variant
clamp = None if variant in ('unclamped', 'plain') else 50.0
B, H, Np = (16, 8, 1056) if shape == 'cfg2' else (8, 16, 2080)
bf = lambda *s: torch.randn(*s, device=dev).to(torch.bfloat16)
q, k, v = (bf(B, H, Np, 64).requires_grad_() for _ in range(3))
gate = torch.rand(B * Np, H, device=dev).requires_grad_() if variant not in ('nogate', 'plain') else None
m = torch.ones(B, Np, dtype=torch.uint8, device=dev)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
for drop in (0.1, 0.0):
    tf, tb = [], []
    for it in range(iters + 3):
        flush.zero_()
        e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        e[0].record()
        og = ops.AttnCore.apply(q, k, v, gate, m, drop, 7, clamp, None)
        e[1].record()
        w = torch.ones_like(og)
        flush.zero_()
        e[2].record()
        torch.autograd.grad(og, [q, k, v], w)
        e[3].record()
        torch.cuda.synchronize()
        if it >= 3:
            tf.append(e[0].elapsed_time(e[1]) * 1e3)
            tb.append(e[2].elapsed_time(e[3]) * 1e3)
    tf.sort(); tb.sort()
    fl = 4.0 * B * H * Np * Np * 64
    print(f'{os.path.basename(os.environ.get("B200_LIB", "default"))} {shape}{" " + variant if variant else ""} dropout {drop}: fwd (maskbits + kernel) median {tf[len(tf)//2]:.1f} us = {fl / tf[len(tf)//2] * 1e-6:.0f} TF/s, '
          f'bwd (prep + memset + kernel) median {tb[len(tb)//2]:.1f} us = {2.5 * fl / tb[len(tb)//2] * 1e-6:.0f} TF/s')
