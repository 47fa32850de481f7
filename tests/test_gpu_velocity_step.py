"""GPU: graphed training steps with the velocity-consistency term (e2_tts.py:1556-1589): GraphedTrainStep / BucketedTrainStep with
`velocity_consistency_model=`, the teacher's no-grad pass at t + delta captured ahead of the student's forward.

  * one graphed step with the randomness pinned, text kept and dropped, against eager forward(velocity_consistency_model=teacher) +
    backward: loss, flow part, velocity part and every gradient (model_checks.graphed_matches_eager's bounds);
  * `velocity=False` on that step against a step built without a teacher, and the launches of the two graphs: the velocity graph
    runs the plain graph's launches plus those of the eager teacher pass; the per-call refusals leave no launch behind;
  * FusedAdoptEMA.step + copy_ema_to between replays: the next replay reads the new teacher weights (packed inside the graph);
  * a teacher in training mode with dropout gets a new seed word, and so new masks, on every replay;
  * BucketedTrainStep (two buckets, k = 2, cond_drop_prob 0.25) against the eager loop over 10 optimiser steps, the teacher switched
    on when FusedAdoptEMA's EMA is initialised.
"""
import copy
import random

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2
from kernel_checks import dev, pkg  # noqa: F401  (pkg is a fixture)
from oracle import e2tts_oracle as O

pytestmark = pytest.mark.gpu


def _model(pkg, seed, weight=0.7, dropout=0.0, **kw):
    torch.manual_seed(seed)
    random.seed(seed)
    t = dict(dim=128, depth=2, heads=2, dropout=dropout, max_seq_len=256)
    m = pkg.E2TTS(transformer=t, use_vocos=False, velocity_consistency_weight=weight, **kw)
    m.load_state_dict(O.randomize_zero_init({k: v.clone() for k, v in m.state_dict().items()}, seed=seed + 1))
    return m.to(dev()).train()


def _inputs(pkg, drop=False, B=2, N=96, seed=5):
    g = torch.Generator().manual_seed(seed)
    mel = torch.randn(B, N, 100, generator=g).to(dev())
    text = pkg.list_str_to_tensor(['Hello there', 'Goodbye']).to(dev())
    span = torch.zeros(B, N, dtype=torch.bool)
    span[0, 10:70] = True
    span[1, 25:90] = True
    rnd = dict(x0=torch.randn(B, N, 100, generator=g).to(dev()), times=(0.9 * torch.rand(B, generator=g)).to(dev()),
               span_mask=span.to(dev()), drop_text_cond=drop)
    return mel, text, rnd


def _grads(model):
    return {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}


def _clear(model):
    for p in model.parameters():
        p.grad = None


def _parts(out):
    return float(out.loss), float(out.loss_breakdown.flow), float(out.loss_breakdown.velocity_consistency)


def _near(a, b):
    """model_checks.graphed_matches_eager's loss bound"""
    return abs(a - b) <= 1e-3 * abs(b) + 1e-5


def _close(tag, got_parts, got, want_parts, want):
    """loss, flow and velocity parts within 1e-3 |x| + 1e-5; the same parameters with a gradient, each within rel-L2 2e-3"""
    for name, a, b in zip(('loss', 'flow', 'velocity'), got_parts, want_parts):
        assert _near(a, b), (tag, name, a, b)
    assert set(got) == set(want), (tag, sorted(set(got) ^ set(want))[:5])
    for n in want:
        e = rel_l2(got[n].float().cpu(), want[n].float().cpu())
        assert e < 2e-3 or float(want[n].norm()) == 0, (tag, n, e)


def _eager(pkg, model, mel, text, rnd, teacher=None, delta=1e-3):
    """one eager step with the randomness pinned -> ((loss, flow, velocity), gradients); leaves no gradient behind"""
    kw = dict(velocity_consistency_model=teacher, velocity_consistency_delta=delta) if teacher is not None else {}
    with pkg.inject_randomness(**rnd):
        out = model(mel, text=text, **kw)
    out.loss.backward()
    parts, grads = _parts(out), _grads(model)
    del out     # an alive eager graph would drag the default stream into a later capture
    _clear(model)
    return parts, grads


@pytest.mark.parametrize('drop', [False, True], ids=['text', 'dropped'])
def test_graphed_step_with_teacher_matches_eager(pkg, drop):
    model = _model(pkg, 11, cond_drop_prob=1.0 if drop else 0.0)
    teacher = _model(pkg, 12).eval()
    mel, text, rnd = _inputs(pkg, drop)
    want_parts, want = _eager(pkg, model, mel, text, rnd, teacher)
    assert want_parts[2] > 0.1 * want_parts[1]       # the term matters in this case
    with pkg.inject_randomness(**rnd):
        step = pkg.GraphedTrainStep(model, mel, text=text, velocity_consistency_model=teacher, velocity_consistency_delta=1e-3)
    loss = step()
    torch.cuda.synchronize()
    got_parts = _parts(step.out)
    assert float(loss) == got_parts[0]
    print(f'{"dropped" if drop else "text"}: graphed {got_parts}, eager {want_parts}')
    _close('graphed with teacher vs eager', got_parts, {n: p.grad for n, p in model.named_parameters() if p.grad is not None},
           want_parts, want)
    assert all(p.grad is None for p in teacher.parameters())


def test_velocity_off_matches_the_step_without_teacher_and_launch_counts(pkg):
    model = _model(pkg, 21, cond_drop_prob=0.0)
    teacher = _model(pkg, 22).eval()
    mel, text, rnd = _inputs(pkg)
    # eager launches: the teacher pass is what a call with the teacher adds (counted after one call of each, past lazy set-up)
    _eager(pkg, model, mel, text, rnd, teacher)
    _eager(pkg, model, mel, text, rnd)
    n0 = pkg.lib.launch_count()
    _eager(pkg, model, mel, text, rnd, teacher)
    n1 = pkg.lib.launch_count()
    _eager(pkg, model, mel, text, rnd)
    n2 = pkg.lib.launch_count()
    teacher_pass = (n1 - n0) - (n2 - n1)
    assert teacher_pass > 0
    with pkg.inject_randomness(**rnd):
        with_t = pkg.GraphedTrainStep(model, mel, text=text, velocity_consistency_model=teacher, velocity_consistency_delta=1e-3)
        plain = pkg.GraphedTrainStep(model, mel, text=text)
    print(f'launches per replay: plain {plain.launches_per_step}, with teacher {with_t.launches}, eager teacher pass {teacher_pass}')
    assert with_t.launches[False] == plain.launches_per_step
    assert with_t.launches[True] == plain.launches_per_step + teacher_pass
    assert with_t.launches_per_step == with_t.launches[True]

    with_t(velocity=False)
    torch.cuda.synchronize()
    off_parts, off = _parts(with_t.out), _grads(model)
    assert off_parts[2] == 0.0
    plain()
    torch.cuda.synchronize()
    _close('velocity=False vs no teacher', off_parts, off, _parts(plain.out), _grads(model))
    with_t()                                           # back to the default: the teacher's graph, its gradients attached
    torch.cuda.synchronize()
    assert _parts(with_t.out)[2] > 0
    assert all(p.grad is g for p, g in with_t._grad_sets[True])

    # per-call refusals, before any launch
    n0 = pkg.lib.launch_count()
    with pytest.raises(ValueError, match='velocity=True on a step built without velocity_consistency_model'):
        plain(velocity=True)
    w = teacher.to_pred.weight
    w.data = w.data.clone()
    with pytest.raises(ValueError, match='new storage since capture'):
        with_t()
    assert pkg.lib.launch_count() == n0
    with_t(velocity=False)                             # the graph without the teacher still runs
    torch.cuda.synchronize()


def test_ema_refresh_between_replays_reaches_the_graph(pkg):
    model = _model(pkg, 31, cond_drop_prob=0.0)
    teacher = _model(pkg, 32).eval()
    mel, text, rnd = _inputs(pkg)
    delta = 0.05      # the teacher becomes a copy of the student: a visible step in t keeps its term away from zero
    with pkg.inject_randomness(**rnd):
        step = pkg.GraphedTrainStep(model, mel, text=text, flat_grads=True, velocity_consistency_model=teacher,
                                    velocity_consistency_delta=delta)
    opt = pkg.FusedAdoptEMA(list(model.parameters()), lr=1e-3, ema=True, ema_update_after_step=0, ema_update_every=1,
                            grad_sync=step.grad_sync)
    step()
    torch.cuda.synchronize()
    old_parts = _parts(step.out)
    before = [p.detach().clone() for p in teacher.parameters()]
    opt.step(step.grad_sync.flat)
    opt.copy_ema_to(teacher.parameters())
    torch.cuda.synchronize()
    assert not all(torch.equal(a, b) for a, b in zip(before, teacher.parameters()))
    step()
    torch.cuda.synchronize()
    got_parts, got = _parts(step.out), _grads(model)
    _clear(model)
    want_parts, want = _eager(pkg, model, mel, text, rnd, teacher, delta)
    print(f'EMA refresh: before {old_parts}, after {got_parts}, eager after {want_parts}')
    _close('replay after copy_ema_to vs eager', got_parts, got, want_parts, want)
    assert abs(got_parts[2] - old_parts[2]) > 100 * (1e-3 * abs(want_parts[2]) + 1e-5), 'the replay kept the old teacher'


def test_teacher_in_training_mode_draws_new_dropout_masks(pkg):
    model = _model(pkg, 41, cond_drop_prob=0.0)
    teacher = _model(pkg, 42, dropout=0.1).train()
    mel, text, rnd = _inputs(pkg)
    with pkg.inject_randomness(**rnd):
        step = pkg.GraphedTrainStep(model, mel, text=text, velocity_consistency_model=teacher, velocity_consistency_delta=1e-3)
    word = teacher.transformer._seed_dev
    assert word is not None and word is not model.transformer._seed_dev and step.teacher.seed_dev is word
    seeds, parts = [], []
    for _ in range(3):
        step()
        torch.cuda.synchronize()
        seeds.append(int(word.item()))
        parts.append(_parts(step.out))
    print(f'teacher seed words {seeds}, parts {parts}')
    assert len(set(seeds)) == 3
    for a, b in zip(parts, parts[1:]):
        assert abs(a[1] - b[1]) <= 1e-5 * abs(a[1]), 'the student (no dropout) changed between replays'
        assert abs(a[2] - b[2]) > 1e-4 * abs(a[2]), 'the teacher replayed the same dropout masks'


def test_bucketed_loop_with_ema_teacher_matches_eager(pkg):
    """10 optimiser steps of k = 2 micro-steps over buckets (96, 160), cond_drop_prob 0.25, the teacher (the EMA weights, copied
    after every optimiser step) switched on when FusedAdoptEMA's EMA is initialised (after step 3), both loops fed the same batches,
    the same CUDA-generator seeds and the same python coin.

    Bounds: the first micro-step is the graphed step of test_graphed_step_with_teacher_matches_eager (1e-3 |x| + 1e-5), and the
    first window's gradient is test_gpu_bucketed_step's accumulation bound (whole-gradient rel-L2 1e-2: the eager loop rounds its
    bf16 backward on loss / k, the graphs scale the fp32 gradient afterwards). From then on the two loops update from those
    slightly different gradients; Adopt normalises each element's update to about lr, so an element whose gradient is near zero
    may step either way, and the parameters drift apart by up to lr per step. With lr = 1e-4 over 9 updates the losses stay within
    2e-2 of each other. The velocity part is small (about 1e-3 of the loss: the teacher is the lagging EMA of the student and
    delta is 0.05), so it is held to itself: within 1e-1, where the drift enters both predictions it compares. A missing or stale
    teacher fails the first velocity step by far more (test_ema_refresh_between_replays_reaches_the_graph)."""
    B, k, n_opt, delta = 2, 2, 10, 0.05
    buckets = (96, 160)
    model_e = _model(pkg, 51, weight=0.5, cond_drop_prob=0.25)
    model_g = _model(pkg, 51, weight=0.5, cond_drop_prob=0.25)
    model_g.load_state_dict(model_e.state_dict())
    teacher_e, teacher_g = copy.deepcopy(model_e).eval(), copy.deepcopy(model_g).eval()
    opt_kw = dict(lr=1e-4, ema=True, ema_update_after_step=2, ema_update_every=1)
    step = pkg.BucketedTrainStep(model_g, B, buckets, grad_accumulation_steps=k, velocity_consistency_model=teacher_g,
                                 velocity_consistency_delta=delta)
    assert set(step.graphs) == set(step.velocity_graphs) == {(nb, d) for nb in buckets for d in (False, True)}
    opt_e = pkg.FusedAdoptEMA(list(model_e.parameters()), **opt_kw)
    opt_g = pkg.FusedAdoptEMA(list(model_g.parameters()), grad_sync=step.grad_sync, **opt_kw)

    g = torch.Generator().manual_seed(9)
    words = ['hello there', 'goodbye', 'a', 'the third one', 'x' * 30, 'good morning to you']
    data = []
    for i in range(k * n_opt):
        n = int(torch.randint(60, 161, (1,), generator=g))
        data.append((torch.randn(B, n, 100, generator=g).to(dev()), torch.tensor([n, n - 7], device=dev()),
                     [words[(i + j) % len(words)] for j in range(B)]))

    def eager_loop():
        random.seed(77)
        out_l = []
        for i, (mel, lens, text) in enumerate(data):
            torch.cuda.manual_seed(1000 + i)
            nb = step.plan.bucket(mel.shape[1])
            on = opt_e.ema_initted
            kw = dict(velocity_consistency_model=teacher_e, velocity_consistency_delta=delta) if on else {}
            out = model_e(F.pad(mel, (0, 0, 0, nb - mel.shape[1])), text=text, lens=lens, **kw)
            (out.loss / k).backward()
            out_l.append((float(out.loss), float(out.loss_breakdown.velocity_consistency), on))
            del out
            if (i + 1) % k == 0:
                if i + 1 == k:
                    out_l.append(_grads(model_e))
                opt_e.step()
                _clear(model_e)
                opt_e.copy_ema_to(teacher_e.parameters())
        return out_l

    def graphed_loop():
        random.seed(77)
        out_l = []
        for i, (mel, lens, text) in enumerate(data):
            torch.cuda.manual_seed(1000 + i)
            on = opt_g.ema_initted
            loss = step(mel, text=text, lens=lens, velocity=on)
            out_l.append((float(loss), float(step.velocity_loss), on))
            assert step.sync_gradients == ((i + 1) % k == 0)
            if step.sync_gradients:
                if i + 1 == k:
                    used = step.grad_sync.used.tolist()
                    out_l.append({n: v.detach().clone() for (n, _), v, u in zip(model_g.named_parameters(), step.grad_sync.grad_views, used)
                                  if u > 0})
                opt_g.step(step.grad_sync.flat)
                opt_g.copy_ema_to(teacher_g.parameters())
        return out_l

    want, got = eager_loop(), graphed_loop()
    torch.cuda.synchronize()
    grads_e, grads_g = want.pop(k), got.pop(k)
    assert set(grads_g) == set(grads_e), sorted(set(grads_g) ^ set(grads_e))[:5]
    names = sorted(grads_e)
    e_all = rel_l2(torch.cat([grads_g[n].double().flatten().cpu() for n in names]), torch.cat([grads_e[n].double().flatten().cpu() for n in names]))
    worst_l = worst_v = 0.0
    for i, ((lg, vg, on_g), (le, ve, on_e)) in enumerate(zip(got, want)):
        print(f'  micro-step {i:2d}: velocity {"on " if on_e else "off"} loss {lg:.6f} / {le:.6f}, velocity part {vg:.6g} / {ve:.6g}')
        if on_e:
            worst_v = max(worst_v, abs(vg - ve) / abs(ve))
        worst_l = max(worst_l, abs(lg - le) / abs(le))
    print(f'bucketed EMA loop: first-window gradient rel-L2 {e_all:.3g}, worst loss {worst_l:.3g}, worst velocity part {worst_v:.3g} '
          f'(relative to itself); launches {step.launches}')
    assert [w[2] for w in got] == [w[2] for w in want]
    assert sum(w[2] for w in want) >= 8, 'the teacher was switched on too late to test it'
    for (lg, vg, on), (le, ve, _) in zip(got, want):
        assert (vg > 0 and ve > 0) if on else (vg == 0.0 and ve == 0.0)
    assert _near(got[0][0], want[0][0]), (got[0], want[0])
    assert e_all < 1e-2
    assert worst_l < 2e-2 and worst_v < 1e-1
