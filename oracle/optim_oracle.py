"""CPU restatement of the optimiser-side step of the reference trainer — TEST INFRASTRUCTURE (only tests/ may import it).

What it restates (call sites in e2_tts_pytorch/trainer.py of the original project):
  * `clip_grad_norm_(model.parameters(), max_grad_norm)`  :272-273  (torch.nn.utils: total L2 norm, coef = max_norm / (norm + 1e-6), clamped to 1)
  * `Adopt(model.parameters(), lr=...)` :183 and `.step()` :275 — adam-atan2-pytorch (pyproject.toml:26), NOT vendored under
    the original project. PARITY UNPINNED: restated from the ADOPT algorithm (Taniguchi et al. 2024, "ADOPT: Modified Adam Can Converge
    with Any beta2 with the Optimal Rate", Algorithm 2 without the optional update clipping) as lucidrains' `adopt.py` implements it:
        first call : v = g^2, m = 0, parameters untouched
        afterwards : m <- lerp(m, g / max(sqrt(v), eps), 1 - beta1);  p <- p - lr m;  v <- lerp(v, g^2, 1 - beta2)
        weight decay (decoupled: wd / init_lr) multiplies p by (1 - lr wd) first; parameters whose grad is None are skipped
    defaults lr 1e-4, betas (0.9, 0.99), eps 1e-6, weight_decay 0.
  * `EMA(model, include_online_model=False)` :170-174 and `.update()` :279 — ema-pytorch (pyproject.toml:32), NOT vendored.
    PARITY UNPINNED: restated from its published update rule: step counter; every `update_every` steps: copy the online weights while
    step <= update_after_step (and once more on the first step after), then ema <- lerp(ema, online, 1 - decay) with
    decay = clamp(1 - (1 + epoch / inv_gamma)^-power, min_value, beta), epoch = max(step - update_after_step - 1, 0), decay 0 at epoch 0.
    defaults beta 0.9999, update_after_step 100, update_every 10, inv_gamma 1, power 2/3.
"""
import torch


def clip_grad_norm(grads, max_norm):
    gs = [g for g in grads if g is not None]
    total = torch.linalg.vector_norm(torch.stack([torch.linalg.vector_norm(g) for g in gs]))
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    return [None if g is None else g * coef for g in grads], total


class Adopt:
    def __init__(self, params, lr=1e-4, betas=(0.9, 0.99), eps=1e-6, weight_decay=0., decoupled_wd=True):
        self.params, self.lr, self.init_lr, self.betas, self.eps = params, lr, lr, betas, eps
        self.wd = weight_decay / lr if (decoupled_wd and weight_decay > 0) else weight_decay
        self.state = [None] * len(params)

    @torch.no_grad()
    def step(self, grads):
        b1, b2 = self.betas
        for i, (p, g) in enumerate(zip(self.params, grads)):
            if g is None:
                continue
            if self.wd > 0:
                p.mul_(1. - self.lr * self.wd)
            if self.state[i] is None:
                self.state[i] = dict(steps=0, m=torch.zeros_like(g), v=g * g)
                self.state[i]['steps'] = 1
                continue
            st = self.state[i]
            upd = g / st['v'].sqrt().clamp(min=self.eps)
            st['m'].lerp_(upd, 1. - b1)
            p.add_(st['m'], alpha=-self.lr)
            st['v'].lerp_(g * g, 1. - b2)
            st['steps'] += 1


class EMA:
    def __init__(self, params, beta=0.9999, update_after_step=100, update_every=10, inv_gamma=1.0, power=2. / 3., min_value=0.0):
        self.online = params
        self.ema = [p.detach().clone() for p in params]
        self.beta, self.update_after_step, self.update_every = beta, update_after_step, update_every
        self.inv_gamma, self.power, self.min_value = inv_gamma, power, min_value
        self.step, self.initted = 0, False

    def get_current_decay(self):   # evaluated AFTER update() has incremented self.step
        epoch = max(self.step - self.update_after_step - 1, 0)
        if epoch <= 0:
            return 0.0
        return min(max(1. - (1. + epoch / self.inv_gamma) ** -self.power, self.min_value), self.beta)

    def _copy(self):
        for e, p in zip(self.ema, self.online):
            e.copy_(p)

    @torch.no_grad()
    def update(self):
        step = self.step
        self.step += 1
        if step % self.update_every != 0:
            return
        if step <= self.update_after_step:
            self._copy()
            return
        if not self.initted:
            self._copy()
            self.initted = True
        decay = self.get_current_decay()
        for e, p in zip(self.ema, self.online):
            e.lerp_(p, 1. - decay)
