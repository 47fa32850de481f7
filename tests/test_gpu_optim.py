"""GPU tests of the step around forward/backward (SURVEY §8e / §8f row 1): flat gradient gather, fused clip + Adopt + EMA kernel
against the PyTorch restatement in oracle/optim_oracle.py, and GraphedTrainStep's flat-gradient mode. Through the C ABI."""
import copy

import pytest
import torch

from conftest import rel_l2
from kernel_checks import dev, pkg
from oracle import optim_oracle as OO

pytestmark = pytest.mark.gpu


SHAPES = [(5,), (3, 7), (), (40000,), (16384,), (129, 515), (1,), (64, 64)]


@pytest.mark.parametrize('max_norm,wd', [(0.0, 0.0), (1.0, 0.0), (0.5, 1e-2)])
def test_fused_adopt_ema_vs_restatement(pkg, max_norm, wd):
    torch.manual_seed(0)
    params = [torch.nn.Parameter(torch.randn(s, device=dev())) for s in SHAPES]
    ref_params = [p.detach().cpu().clone() for p in params]
    opt = pkg.optim.FusedAdoptEMA(params, lr=3e-3, weight_decay=wd, max_grad_norm=max_norm, ema=True, ema_update_after_step=3, ema_update_every=2)
    ropt = OO.Adopt(ref_params, lr=3e-3, weight_decay=wd)
    rema = OO.EMA(ref_params, update_after_step=3, update_every=2)
    for step in range(12):
        grads = [torch.randn_like(p) * (0.1 + step) for p in params]
        skip = 3 if step in (0, 1, 6) else -1       # a parameter without a gradient on the FIRST and some later steps (text stream when the text is dropped)
        for i, (p, g) in enumerate(zip(params, grads)):
            p.grad = None if i == skip else g.clone()
        rg = [None if i == skip else g.cpu() for i, g in enumerate(grads)]
        if max_norm > 0:
            rg, total = OO.clip_grad_norm(rg, max_norm)
        opt.step()
        ropt.step(rg)
        rema.update()
        if max_norm > 0:
            assert abs(float(opt.grad_norm()) - float(total)) <= 1e-4 * float(total)
        for i, (p, rp) in enumerate(zip(params, ref_params)):
            assert rel_l2(p.detach().cpu(), rp) < 1e-5 or float((p.detach().cpu() - rp).abs().max()) < 1e-6, (step, i)
        for i, (e, re_) in enumerate(zip(opt.ema_parameters(), rema.ema)):
            assert float((e.cpu() - re_).abs().max()) < 1e-5 * max(1.0, float(re_.abs().max())), (step, i)
    for i, rp in enumerate(ref_params):
        st = ropt.state[i]
        o, n = opt.layout.offsets[i], opt.layout.numels[i]
        assert rel_l2(opt.m[o:o + n].cpu(), st['m'].flatten()) < 1e-4
        assert rel_l2(opt.v[o:o + n].cpu(), st['v'].flatten()) < 1e-4


def test_grad_sync_flattens_and_flags_unused(pkg):
    torch.manual_seed(1)
    params = [torch.nn.Parameter(torch.randn(s, device=dev())) for s in SHAPES]
    sync = pkg.optim.GradSync(params)
    grads = [torch.randn_like(p) for p in params]
    for i, (p, g) in enumerate(zip(params, grads)):
        p.grad = None if i == 3 else g
    flat = sync()
    assert flat.numel() == sync.layout.total
    for i, (p, g) in enumerate(zip(params, grads)):
        assert p.grad.data_ptr() == sync.grad_views[i].data_ptr()
        want = torch.zeros_like(g) if i == 3 else g
        assert torch.equal(p.grad, want), i
    assert sync.used.tolist() == [0.0 if i == 3 else 1.0 for i in range(len(params))]


def test_graphed_step_flat_grads_match_eager_and_feed_the_fused_optimizer(pkg):
    """GraphedTrainStep(flat_grads=True): after a replay p.grad are views of ONE flat buffer holding exactly the eager step's
    gradients; FusedAdoptEMA consumes that buffer; an EMA deepcopy of the model receives the EMA weights (trainer.py:170-174)."""
    torch.manual_seed(0)
    B, N = 2, 96
    from oracle import e2tts_oracle as O
    model = pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2, dropout=0.0), use_vocos=False)
    # (with the reference's zero-initialised cross-condition weights the text stream cannot reach the loss: half the gradients are 0)
    model.load_state_dict(O.randomize_zero_init({k: v.clone() for k, v in model.state_dict().items()}, seed=3))
    model.to(dev()).train()
    model.cond_drop_prob = 0.0
    ema_model = copy.deepcopy(model)       # EMA(model) deep-copies the module
    assert all(torch.equal(a, b) for a, b in zip(model.state_dict().values(), ema_model.state_dict().values()))
    mel = torch.randn(B, N, 100, device=dev())
    text = pkg.list_str_to_tensor(['Hello', 'Goodbye']).to(dev())
    x0, times = torch.randn(B, N, 100, device=dev()), torch.rand(B, device=dev())
    span = torch.zeros(B, N, dtype=torch.bool, device=dev())
    span[:, 20:70] = True
    with pkg.inject_randomness(x0=x0, times=times, span_mask=span, drop_text_cond=False):
        out = model(mel, text=text)
        out.loss.backward()
        want = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
        for p in model.parameters():
            p.grad = None
        del out
        step = pkg.GraphedTrainStep(model, mel, text=text, flat_grads=True)
        step()
    flat = step.grad_sync.flat
    lo, hi = flat.data_ptr(), flat.data_ptr() + flat.numel() * 4
    for n, p in model.named_parameters():
        assert lo <= p.grad.data_ptr() < hi, n
        if n in want:
            assert rel_l2(p.grad.float().cpu(), want[n].float().cpu()) < 2e-3 or float(want[n].norm()) == 0, n
    opt = pkg.optim.FusedAdoptEMA(list(model.parameters()), lr=1e-3, max_grad_norm=1.0, ema=True, ema_update_after_step=0, ema_update_every=1,
                                  grad_sync=step.grad_sync)
    before = [p.detach().clone() for p in model.parameters()]
    opt.step(flat)          # Adopt's first step: state init only
    assert all(torch.equal(a, b) for a, b in zip(before, model.parameters()))
    with pkg.inject_randomness(x0=x0, times=times, span_mask=span, drop_text_cond=False):
        step()
    opt.step(step.grad_sync.flat)
    moved = sum(int(not torch.equal(a, b)) for a, b in zip(before, model.parameters()))
    assert moved > 0.9 * len(before)
    opt.copy_ema_to(ema_model.parameters())
    for e, v in zip(ema_model.parameters(), opt.ema_parameters()):
        assert torch.equal(e, v)
    # the EMA copy is a working model of its own (separate packed-weight caches)
    ema_model.eval()
    with torch.no_grad():
        y = ema_model.sample(mel[:, :8], text=text, duration=24, steps=3, return_raw_output=True)
    assert torch.isfinite(y).all()
