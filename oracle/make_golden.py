"""Mint the golden vectors under tests/golden/ by running the reference's OWN e2_tts.py (needs a checkout of the
original project). TEST INFRASTRUCTURE.

    E2TTS_REFERENCE_FILE=<original>/e2_tts_pytorch/e2_tts.py python oracle/make_golden.py

The reference draws its randomness internally (x0, times, span mask); oracle/load_reference.py records
those draws so they can be replayed into the oracle and the CUDA path. dropout=0 because dropout masks
cannot be replayed bit-for-bit across implementations (SURVEY §7 "hard parts").
Fixtures (fp32, torch.save):
  e2tts_d128_L2.pt     E2TTS fwd+bwd: state_dict, mel, text ids, lens, x0, times, span_mask -> loss, pred,
                       cond, parameter grads (full for the text-conditioned case, (norm,sum) per parameter for
                       the text-dropped case)
  sample_d128_L2.pt    E2TTS.sample 4-step midpoint end point (cfg_strength 1 -> cond + null pass + APG)
  duration_d128_L2.pt  DurationPredictor fwd+bwd (B=4, a prefix draw chosen for conditioning, see below): loss, full parameter
                       grads, and the return_loss=False prediction
  melspec.pt           MelSpec(wave) from torchaudio through the reference module
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.load_reference import load_reference, run_reference_forward  # noqa: E402
from oracle import e2tts_oracle as O  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden')
TKW = dict(dim=128, depth=2, heads=2)
REF_TKW = dict(dropout=0., max_seq_len=256, **TKW)
TEXT = ['Hello', 'Goodbye']


def main():
    ref = load_reference()
    os.makedirs(OUT, exist_ok=True)
    torch.manual_seed(0)
    model = ref.E2TTS(transformer=dict(**REF_TKW), use_vocos=False)
    sd = O.randomize_zero_init(model.state_dict(), seed=11)
    model.load_state_dict(sd)
    mel = torch.randn(2, 96, 100)
    lens = torch.tensor([96, 70])
    text_ids = O.list_str_to_tensor(TEXT)
    cases = {}
    for name, drop in (('text', False), ('drop', True)):
        torch.manual_seed(7)
        model.zero_grad()
        out, rec = run_reference_forward(ref, model, mel, TEXT, lens=lens, drop_text_cond=drop)
        out.loss.backward()
        grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
        if drop:  # keep the fixture small: full grads only for the text-conditioned case
            grads = {k: torch.stack((g.norm(), g.sum())) for k, g in grads.items()}
        cases[name] = dict(drop_text_cond=drop, loss=out.loss.detach(), pred=out.pred_flow.detach(),
                           cond=out.cond.detach(), pred_data=out.pred_data.detach(), grads=grads, **rec)
    torch.save(dict(transformer=TKW, max_seq_len=256, state_dict={k: v.clone() for k, v in model.state_dict().items()},
                    mel=mel, text=TEXT, text_ids=text_ids, lens=lens, cases=cases), os.path.join(OUT, 'e2tts_d128_L2.pt'))

    # sample(): record y0 (e2_tts.py:1418)
    model.eval()
    holder = {}

    class Rec:
        def __getattr__(self, n):
            return getattr(torch, n)

        def randn_like(self, *a, **k):
            holder['y0'] = torch.randn_like(*a, **k)
            return holder['y0'].clone()

    torch.manual_seed(3)
    cond = mel[:, :24]
    ref.torch = Rec()
    try:
        smp = model.sample(cond, text=TEXT, duration=64, steps=4, return_raw_output=True)
    finally:
        ref.torch = torch
    torch.save(dict(cond=cond, text_ids=text_ids, duration=64, steps=4, cfg_strength=1.0, y0=holder['y0'], out=smp),
               os.path.join(OUT, 'sample_d128_L2.pt'))

    # DurationPredictor. The loss reaches the backbone through a masked mean over a RANDOM PREFIX of every sequence
    # (e2_tts.py:1081-1086); with a short prefix the gradients of a few first-text-layer parameters are sums of nearly
    # cancelling terms, and rounding the fp32 oracle's OWN stage outputs to bf16 (O.STAGE_ROUND) flips them (round-1 fixture:
    # cosine 0.59 / -1.0 against itself). A bf16 path cannot be judged on such a case, so the fixture is minted on the first
    # torch seed whose prefix draw is well conditioned under that probe (every per-parameter cosine >= 0.997).
    torch.manual_seed(1)
    dp = ref.DurationPredictor(transformer=dict(**REF_TKW))
    dsd = O.randomize_zero_init(dp.state_dict(), seed=13)
    dp.load_state_dict(dsd)
    torch.manual_seed(21)
    dmel = torch.randn(4, 96, 100)
    dlens = torch.tensor([96, 70, 88, 80])
    dtext = ['Hello', 'Goodbye', 'Good morning', 'Hi']
    dtext_ids = O.list_str_to_tensor(dtext)

    def conditioning(rand_frac):
        res = []
        for rnd in (None, O.bf16_ste):
            O.STAGE_ROUND = rnd
            try:
                sdo = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in dsd.items()}
                O.duration_forward(sdo, O.TransformerCfg(cond_on_time=False, **TKW), dmel, dtext_ids, lens=dlens, rand_frac=rand_frac).backward()
            finally:
                O.STAGE_ROUND = None
            res.append({k: v.grad.double().flatten() for k, v in sdo.items() if v.grad is not None})
        total = torch.cat(list(res[0].values())).norm()
        worst = 1.0
        for k, a in res[0].items():
            if a.norm() >= 1e-4 * total:
                worst = min(worst, float(a @ res[1][k] / (a.norm() * res[1][k].norm() + 1e-30)))
        return worst

    for dseed in range(5, 200):
        torch.manual_seed(dseed)
        rand_frac = dmel.new_zeros(4).uniform_(0, 1)  # e2_tts.py:1082 draws exactly this after the seed
        if float(rand_frac.min()) >= 0.5 and conditioning(rand_frac) >= 0.997:
            break
    else:
        raise RuntimeError('no well-conditioned prefix draw found')
    print('duration fixture: seed', dseed, 'rand_frac', rand_frac.tolist())
    torch.manual_seed(dseed)
    loss = dp(dmel, text=dtext, lens=dlens)
    loss.backward()
    dgrads = {k: p.grad.clone() for k, p in dp.named_parameters() if p.grad is not None}
    dp.eval()
    with torch.no_grad():
        pred = dp(dmel, text=dtext, lens=dlens, return_loss=False)
    torch.save(dict(state_dict={k: v.clone() for k, v in dp.state_dict().items()}, mel=dmel, text=dtext, text_ids=dtext_ids, lens=dlens,
                    rand_frac=rand_frac, loss=loss.detach(), grads=dgrads, pred=pred, seed=dseed), os.path.join(OUT, 'duration_d128_L2.pt'))

    # MelSpec
    torch.manual_seed(9)
    wave = torch.randn(2, 256 * 24) * 0.3
    torch.save(dict(wave=wave, mel=ref.MelSpec()(wave)), os.path.join(OUT, 'melspec.pt'))
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)) // 1024, 'KiB')


if __name__ == '__main__':
    main()
