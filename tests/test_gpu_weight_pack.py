"""The weight pack (modules.WeightPack): the model whose forward the user calls refreshes ALL of its GEMM operands with ONE
b200_pack_weights launch per forward (sample(): one per call, for the whole ODE solve), and the packed operands follow the
parameters through in-place updates, new parameter storage, deep copies and CUDA-graph replays.

Every output is compared with a freshly built model loaded with the same state_dict, which packs from scratch. Forward
predictions are deterministic and must match bit for bit. The flow loss adds per-block partial sums with fp32 atomics
(DESIGN §5), so losses match to the rounding of that sum."""
import copy
import gc
import math
import random

import pytest
import torch

from conftest import rel_l2
from kernel_checks import U, dev, pkg
from oracle import e2tts_oracle as O

pytestmark = pytest.mark.gpu

B, N, C = 2, 96, 100
STEPS = 3           # sample(): 2 midpoint steps = 4 function evaluations, each a text pass and a null pass
TKW = dict(dim=128, depth=2, heads=2, dropout=0.0)
BUILD = {
    'e2tts': lambda pkg: pkg.E2TTS(transformer=dict(TKW), use_vocos=False),
    'interpolated_text': lambda pkg: pkg.E2TTS(transformer=dict(TKW), use_vocos=False, interpolated_text=True),
    'attn_fourier_embed_input': lambda pkg: pkg.E2TTS(transformer=dict(TKW, attn_fourier_embed_input=True), use_vocos=False),
    'duration': lambda pkg: pkg.DurationPredictor(transformer=dict(TKW)),
    'transformer': lambda pkg: pkg.Transformer(**TKW),
}


@pytest.fixture
def inp(pkg):
    """Seeded inputs and the pinned random draws of a training forward and of sample()."""
    g = torch.Generator().manual_seed(0)
    span = torch.zeros(B, N, dtype=torch.bool)
    span[:, 20:70] = True
    t = dict(mel=torch.randn(B, N, C, generator=g), x=torch.randn(B, N, TKW['dim'], generator=g),
             te=torch.randn(B, N, TKW['dim'] // 2, generator=g), y0=torch.randn(B, 48, C, generator=g))
    rand = dict(x0=torch.randn(B, N, C, generator=g), times=torch.rand(B, generator=g), span_mask=span,
                duration_rand_frac=torch.full((B,), 0.8))
    d = {k: v.to(dev()) for k, v in t.items()}
    d['text'] = pkg.list_str_to_tensor(['Hello', 'Goodbye']).to(dev())
    d['rand'] = dict({k: v.to(dev()) for k, v in rand.items()}, drop_text_cond=False)
    return d


@pytest.fixture
def pack_log(pkg, monkeypatch):
    """Every pack launch, and every ODE update (to place the launches inside sample()), in call order."""
    log, ops = [], pkg.ops
    pack_weights, axpy = ops.pack_weights, ops.axpy
    monkeypatch.setattr(ops, 'pack_weights', lambda *a: (log.append('pack'), pack_weights(*a))[1])
    monkeypatch.setattr(ops, 'axpy', lambda *a: (log.append('axpy'), axpy(*a))[1])
    return log


def build(pkg, kind, sd=None, seed=0):
    """`kind`'s model on the GPU in train mode, with `sd` loaded or else with every zero-initialised tensor randomised (so that
    every weight reaches the output)."""
    torch.manual_seed(seed)
    random.seed(seed)      # the hyper-connections draw their initial stream with python's randrange
    model = BUILD[kind](pkg)
    if sd is None:
        sd = O.randomize_zero_init({k: v.clone() for k, v in model.state_dict().items()}, seed=seed + 1)
    model.load_state_dict(sd)
    if hasattr(model, 'cond_drop_prob'):
        model.cond_drop_prob = 0.0
    return model.to(dev()).train()


def fresh(pkg, kind, model):
    return build(pkg, kind, sd=model.state_dict()) if model is not None else None


def run(pkg, kind, model, inp):
    """One training forward of `kind` on the pinned inputs -> {name: detached output}."""
    with pkg.inject_randomness(**inp['rand']):
        if kind == 'duration':
            out = dict(pred=model(inp['mel'], text=inp['text'], return_loss=False))
        elif kind == 'transformer':
            out = dict(pred=model(inp['x'], times=inp['rand']['times'], text_embed=inp['te']))
        else:
            o = model(inp['mel'], text=inp['text'])
            out = dict(pred=o.pred_flow, loss=o.loss)
    return {k: v.detach() for k, v in out.items()}


def sample(pkg, model, inp, null=None):
    with pkg.inject_randomness(y0=inp['y0']):
        return model.sample(inp['mel'][:, :16], text=inp['text'], duration=48, steps=STEPS, cfg_strength=1.0, cfg_null_model=null,
                            return_raw_output=True)


def assert_same(got, want):
    for k, w in want.items():
        if k == 'loss':
            # two orders of the same n_blocks positive fp32 additions are each within gamma(n_blocks) of the exact sum; the
            # division by the frame count rounds once in each
            nb = math.ceil(B * N * C / 256)
            tol = (2 * nb * U / (1 - nb * U) + 2 * U) * abs(float(w))
            assert abs(float(got[k]) - float(w)) <= tol, (k, float(got[k]), float(w))
        else:
            assert torch.equal(got[k], w), (k, rel_l2(got[k].cpu(), w.cpu()))


def perturb_(model, seed):
    """An optimiser-like in-place update of every parameter: 10 % relative noise."""
    g = torch.Generator(device=dev()).manual_seed(seed)
    with torch.no_grad():
        for p in model.parameters():
            p.mul_(1 + 0.1 * torch.randn(p.shape, generator=g, device=p.device))


@pytest.mark.parametrize('kind', list(BUILD))
def test_one_pack_launch_per_forward(pkg, inp, pack_log, kind):
    model = build(pkg, kind)
    for _ in range(2):       # the first forward builds the pack, the second reuses it
        pack_log.clear()
        run(pkg, kind, model, inp)
        assert pack_log == ['pack']


@pytest.mark.parametrize('null_model', [False, True])
def test_one_pack_launch_per_sample(pkg, inp, pack_log, null_model):
    """One launch per model before the solve, none inside any function evaluation."""
    model = build(pkg, 'e2tts')
    null = build(pkg, 'e2tts', seed=5) if null_model else None
    pack_log.clear()
    sample(pkg, model, inp, null)
    assert pack_log == ['pack'] * (2 if null_model else 1) + ['axpy'] * (2 * (STEPS - 1))


@pytest.mark.parametrize('update', ['in_place', 'new_storage'])
@pytest.mark.parametrize('kind', list(BUILD))
def test_forward_follows_parameter_updates(pkg, inp, kind, update):
    model = build(pkg, kind)
    before = run(pkg, kind, model, inp)
    assert_same(before, run(pkg, kind, fresh(pkg, kind, model), inp))
    old = [p.data for p in model.parameters()]      # the old storage stays alive, holding the old values
    if update == 'new_storage':
        for p in model.parameters():
            p.data = p.data.clone()
    perturb_(model, 1)
    after = run(pkg, kind, model, inp)
    assert_same(after, run(pkg, kind, fresh(pkg, kind, model), inp))
    k = next(iter(before))
    assert rel_l2(after[k].cpu(), before[k].cpu()) > 1e-2, 'the update must change the output'
    del old


@pytest.mark.parametrize('kind', ['e2tts', 'duration', 'transformer'])
def test_deepcopy_packs_its_own_weights(pkg, inp, kind):
    model = build(pkg, kind)
    want = run(pkg, kind, model, inp)         # the original's pack and rotary tables exist now
    gc.collect()                              # no collection of earlier garbage may free device memory inside the count
    gc.disable()
    try:
        n0 = torch.cuda.memory_stats(dev())['allocation.all.current']
        twin = copy.deepcopy(model)
        n_new = torch.cuda.memory_stats(dev())['allocation.all.current'] - n0
    finally:
        gc.enable()
    # one allocation per parameter and buffer: no packed operands, no rotary tables
    assert n_new == len([t for t in (*twin.parameters(), *twin.buffers()) if t.numel() > 0])
    perturb_(twin, 2)
    assert_same(run(pkg, kind, twin, inp), run(pkg, kind, fresh(pkg, kind, twin), inp))
    assert_same(run(pkg, kind, model, inp), want)


@pytest.mark.parametrize('null_model', [False, True])
def test_sample_follows_parameter_updates(pkg, inp, null_model):
    """sample() before and after an in-place update. The APG projection adds per-block fp64 partial sums with atomics, whose
    order can, rarely, move an fp32 result by one ulp, hence a tolerance instead of bit equality; a stale operand moves the
    output by more than 1e-2."""
    model = build(pkg, 'e2tts')
    null = build(pkg, 'e2tts', seed=5) if null_model else None

    def check():
        got = sample(pkg, model, inp, null)
        want = sample(pkg, fresh(pkg, 'e2tts', model), inp, fresh(pkg, 'e2tts', null))
        assert rel_l2(got.cpu(), want.cpu()) < 1e-4
        return got

    before = check()
    perturb_(model, 3)
    if null_model:
        perturb_(null, 4)
    after = check()
    assert rel_l2(after.cpu(), before.cpu()) > 1e-2


def test_graphed_step_follows_parameter_updates(pkg, inp):
    model = build(pkg, 'e2tts')
    with pkg.inject_randomness(**inp['rand']):
        step = pkg.GraphedTrainStep(model, inp['mel'], text=inp['text'])
        perturb_(model, 6)
        step()
    assert_same(dict(pred=step.out.pred_flow, loss=step.out.loss), run(pkg, 'e2tts', fresh(pkg, 'e2tts', model), inp))
    # the seed word GraphedTrainStep gave the model stays with it: a deep copy (an EMA model) has none
    assert model.transformer._seed_dev is not None
    assert copy.deepcopy(model).transformer._seed_dev is None
