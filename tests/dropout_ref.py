"""Dropout with known masks, for holding training steps with dropout on to the oracle of oracle/e2tts_oracle.py through its
`O.DROPOUT` hook (called as DROPOUT(name, x) on the attention probabilities, name `<prefix>.attn_dropout`, and on the GEGLU hidden,
name `<prefix>.ff.1`: the qualified names of the reference's nn.Dropout modules). Shared by tests/test_dropout_vs_reference.py,
oracle/make_reference_golden.py and tests/test_gpu_dropout_step.py.

Two mask recipes:
  * hashed (CPU): the kept set of a dropout module depends only on its qualified name, the input shape and the case seed (a
    torch.Generator seeded with zlib.crc32 of the three), kept elements scaled by 1 / (1 - p). oracle/make_reference_golden.py puts it in
    place of every nn.Dropout of the original e2_tts.py; `HashedDropout` gives the oracle the same masks.
  * the kernels' own (GPU): `SeedRecorder` records the host seed and the device seed word of every ops.Attention / ops.FeedForward
    call of a forward, keyed by the dropout module it belongs to (through the identity of the to_q / ff.0.proj weight it receives).
    `KernelMasks` rebuilds each call's keep mask from the effective seed (seed + device word) mod 2^64 with the float64 restatements
    of the kernels' hashes (attn_ref.dropout_keep, kernel_checks.drop_mask) and the kernels' keep scale 65536 / (65536 - thresh16).
"""
import zlib
from collections import namedtuple

import torch

from oracle import e2tts_oracle as O

M64 = 2 ** 64

# ---------------------------------------------------------------------------------------------------------------- hashed masks
P_REF = 0.25

# forward + backward cases of the original with dropout p = P_REF: class, seed, transformer kwargs, (batch, frames), lens, text,
# drop_text_cond. The masks of case `name` are seeded with its seed.
DROPOUT_CASES = {
    'depth2_lens': dict(cls='E2TTS', seed=111, tkw=dict(dim=128, depth=2, heads=2), mel=(2, 80), lens=[80, 51],
                        text=['abc', 'a longer text than the first'], drop=False),
    'text_dropped': dict(cls='E2TTS', seed=112, tkw=dict(dim=128, depth=2, heads=4), mel=(3, 64), lens=[64, 40, 17],
                         text=['one', 'two words', ''], drop=True),
    'residual1': dict(cls='E2TTS', seed=113, tkw=dict(dim=128, depth=2, heads=2, num_residual_streams=1), mel=(2, 64), lens=[64, 45],
                      text=['abc', 'defgh ij'], drop=False),
    'a2x128_t1x64': dict(cls='E2TTS', seed=114, tkw=dict(dim=128, depth=2, heads=2, dim_head=128, text_heads=1, text_dim_head=64),
                         mel=(2, 64), lens=[64, 37], text=['hello', 'xy z'], drop=False),
    'duration': dict(cls='DurationPredictor', seed=115, tkw=dict(dim=128, depth=2, heads=2), mel=(3, 72), lens=[72, 50, 31],
                     text=['abc', 'hello world', 'x']),
}
for _c in DROPOUT_CASES.values():
    _c.setdefault('drop', False)


def hashed_keep(name, shape, seed, p):
    """bool keep mask of dropout module `name` on an input of `shape` in case `seed`: P(keep) = 1 - p"""
    g = torch.Generator().manual_seed(zlib.crc32(f'{name}|{tuple(shape)}|{seed}'.encode()))
    return torch.rand(tuple(shape), generator=g) >= p


def hashed_drop(name, x, seed, p):
    return x * (hashed_keep(name, x.shape, seed, p).to(x.dtype) * (1.0 / (1.0 - p)))


class HashedDropout(torch.nn.Module):
    """in place of the reference's nn.Dropout `name`; appends `name` to `log` on every call"""

    def __init__(self, name, seed, p, log):
        super().__init__()
        self.name, self.seed, self.p, self.log = name, seed, p, log

    def forward(self, x):
        self.log.append(self.name)
        return hashed_drop(self.name, x, self.seed, self.p)


class HashedHook:
    """O.DROPOUT with the hashed masks of case `seed`; `names` lists the modules that dropped, in order"""

    def __init__(self, seed, p):
        self.seed, self.p, self.names = seed, p, []

    def __call__(self, name, x):
        self.names.append(name)
        return hashed_drop(name, x, self.seed, self.p)


# -------------------------------------------------------------------------------------------------------------- kernel masks
Call = namedtuple('Call', 'kind seed device_word p B Np width')   # width: heads (attention) or the GEGLU inner width (FF)


def keep_scale(p):
    """the kernels' scale of a kept element: 65536 / (65536 - thresh16), thresh16 = int(p * 65536) (P(drop) = thresh16 / 65536)"""
    t = int(p * 65536)
    return 65536.0 / (65536 - t)


def dropout_names(model):
    """{id(parameter): dropout module name} for the to_q weight of every attention and the ff.0.proj weight of every feed-forward"""
    out = {}
    for n, prm in model.named_parameters():
        for suffix, drop in (('.to_q.weight', '.attn_dropout'), ('.ff.0.proj.weight', '.ff.1')):
            if n.endswith(suffix):
                out[id(prm)] = n[:-len(suffix)] + drop
    return out


class SeedRecorder:
    """Inside the block, every ops.Attention / ops.FeedForward call of `model` is recorded as (dropout module name, Call) in
    `self.log`, every host seed draw of Transformer._forward_from_h (torch.randint(0, 2**62, (1,))) in `self.host`, and the
    final-normed transformer output of each forward (ops.FinalNorm) in `self.final`. `pin_host` makes those draws return it."""
    HOST_DRAW = (0, 2 ** 62, (1,))

    def __init__(self, pkg, model, pin_host=None):
        self.pkg, self.names, self.pin = pkg, dropout_names(model), pin_host
        self.log, self.host, self.final = [], [], []

    def calls(self, last=None):
        """{name: Call} of the last `last` calls (default: every call; a name recorded twice is an error)"""
        log = self.log if last is None else self.log[-last:]
        out = {}
        for name, c in log:
            assert name not in out, f'{name} ran twice'
            out[name] = c
        return out

    def __enter__(self):
        ops, rec = self.pkg.ops, self
        self.saved = ops.Attention, ops.FeedForward, ops.FinalNorm, torch.randint
        att, ff, fin, randint = self.saved

        class Attention:
            @staticmethod
            def apply(*a):
                sd = a[19]
                rec.log.append((rec.names[id(a[1])], Call('attn', int(a[17]), sd is not None, float(a[16]), a[13], a[14], a[15])))
                return att.apply(*a)

        class FeedForward:
            @staticmethod
            def apply(*a):
                sd = a[13]
                rec.log.append((rec.names[id(a[1])], Call('ff', int(a[12]), sd is not None, float(a[11]), a[9], a[10], a[1].shape[0] // 2)))
                return ff.apply(*a)

        class FinalNorm:
            @staticmethod
            def apply(*a):
                y = fin.apply(*a)
                rec.final.append(y)
                return y

        def draw(*a, **k):
            if a == self.HOST_DRAW and not k:
                out = randint(*a) if rec.pin is None else torch.tensor([rec.pin])
                rec.host.append(int(out.item()))
                return out
            return randint(*a, **k)

        ops.Attention, ops.FeedForward, ops.FinalNorm, torch.randint = Attention, FeedForward, FinalNorm, draw
        return self

    def __exit__(self, *a):
        ops = self.pkg.ops
        ops.Attention, ops.FeedForward, ops.FinalNorm, torch.randint = self.saved


class KernelMasks:
    """O.DROPOUT hook: the keep mask each recorded call drew, from effective seed (seed + word) mod 2^64 (+ `offset`: a negative
    control with every mask wrong), as the kernels scale it. `word` is the device seed word at the time of the step (used only
    by calls that had one)."""

    def __init__(self, calls, word=0, offset=0):
        self.calls, self.word, self.offset = calls, word, offset
        self.cache, self.used = {}, []

    def effective_seed(self, c):
        return (c.seed + (self.word if c.device_word else 0) + self.offset) % M64

    def keep(self, name, shape):
        """the mask the kernels draw for an input of the oracle's `shape`: [B, H, N', N'] probabilities (element
        ((b H + h) N' + i) stride + j of the attention hash) or a [B, N', inner] GEGLU hidden (row b N' + i, the natural hidden index)"""
        if name not in self.cache:
            from attn_ref import dropout_keep
            from kernel_checks import drop_mask
            c = self.calls[name]
            eff = self.effective_seed(c)
            if c.kind == 'attn':
                B, H, Np, _ = shape
                k = dropout_keep(eff, B, H, Np, c.p)
            else:
                B, Np, inner = shape
                k = (drop_mask(eff, B * Np, inner) >= (int(c.p * 65536) << 16)).cpu().view(B, Np, inner)
            self.cache[name] = k
        return self.cache[name]

    def __call__(self, name, x):
        self.used.append(name)
        c = self.calls[name]
        want = (c.B, c.width, c.Np) if c.kind == 'attn' else (c.B, c.Np, c.width)   # (B, H, N') or (B, N', inner)
        assert tuple(x.shape[:3]) == want, f'{name}: the kernel ran on {want}, the oracle drops a {tuple(x.shape)} input'
        return x * (self.keep(name, tuple(x.shape)).to(x.dtype) * keep_scale(c.p))


def splitmix64(w):
    """b200_seed_advance (csrc/lib.cu) in host integer arithmetic: the device seed word after one step of word `w`"""
    z = (w + 0x9E3779B97F4A7C15) % M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) % M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) % M64
    return z ^ (z >> 31)


def with_dropout(hook, fn, *a, **k):
    """fn(*a, **k) with O.DROPOUT = hook"""
    saved = O.DROPOUT
    O.DROPOUT = hook
    try:
        return fn(*a, **k)
    finally:
        O.DROPOUT = saved
