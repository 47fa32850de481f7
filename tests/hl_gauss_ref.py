"""The HL-Gauss classification head of DurationPredictor(hl_gauss_loss=dict(...), use_regression=False) (e2_tts.py:966-967,
1035-1040, 1107, 1111), restated twice for the tests. TEST INFRASTRUCTURE.

`HLGaussLoss` / `HLGaussLayer` restate hl-gauss-pytorch (SURVEY A.6) in both modes. tools/make_hl_gauss_golden.py binds the original
e2_tts.py's `HLGaussLayer` name to this one while the original runs: the restated leaf of oracle/ref_leaves/ takes the regression mode
only. Built in regression mode it has the leaf's parameters and draws the same random numbers.

`duration_forward` is the oracle's DurationPredictor.forward (oracle/e2tts_oracle.py, same stem, Transformer and masked mean) with the
head of `hl_gauss`: the classification head when it holds HLGaussLoss's keywords, the oracle's regression head when it is None.

UNPINNED details (upstream version dependent, no reference test pins them): the presence of the Linear bias, the Sequential wrapper
and its index 0 in classification mode, and the default sigma_to_bin_ratio (2.)."""
import math

import torch
import torch.nn.functional as F
from torch import nn

from oracle import e2tts_oracle as O

SIGMA_TO_BIN_RATIO = 2.


# ---------------------------------------------------------------------------------------------------------------------- hl-gauss-pytorch
class HLGaussLoss(nn.Module):
    def __init__(self, min_value, max_value, num_bins, sigma=None, sigma_to_bin_ratio=SIGMA_TO_BIN_RATIO, clamp_to_range=False):
        super().__init__()
        assert num_bins > 1
        assert max_value > min_value
        self.min_value, self.max_value, self.num_bins = min_value, max_value, num_bins
        support = torch.linspace(min_value, max_value, num_bins + 1).float()
        bin_size = (max_value - min_value) / num_bins
        self.sigma = sigma if sigma is not None else bin_size * sigma_to_bin_ratio
        self.clamp_to_range = clamp_to_range
        self.sigma_times_sqrt_two = math.sqrt(2.) * self.sigma
        self.register_buffer('support', support, persistent=False)
        self.register_buffer('centers', (support[:-1] + support[1:]) / 2, persistent=False)

    def transform_to_probs(self, target):
        assert self.sigma > 0.
        if self.clamp_to_range:
            target = target.clamp(min=self.min_value, max=self.max_value)
        cdf_evals = torch.special.erf((self.support - target.unsqueeze(-1)) / self.sigma_times_sqrt_two)
        z = cdf_evals[..., -1] - cdf_evals[..., 0]
        bin_probs = cdf_evals[..., 1:] - cdf_evals[..., :-1]
        return bin_probs / z.unsqueeze(-1)

    def transform_from_probs(self, probs):
        return (probs * self.centers).sum(dim=-1)

    def forward(self, logits, target=None):
        if target is None:
            return self.transform_from_probs(logits.softmax(dim=-1))
        return F.cross_entropy(logits, self.transform_to_probs(target))


class HLGaussLayer(nn.Module):
    def __init__(self, dim, *, hl_gauss_loss=None, use_regression=False, regress_activation=None):
        super().__init__()
        if isinstance(hl_gauss_loss, dict):
            hl_gauss_loss = HLGaussLoss(**hl_gauss_loss)
        self.hl_gauss_loss = hl_gauss_loss
        self.use_regression = use_regression
        assert use_regression or hl_gauss_loss is not None, '`hl_gauss_loss` must be passed in if not using regression'
        if use_regression:
            self.to_pred = nn.Sequential(nn.Linear(dim, 1), regress_activation or nn.Identity())
        else:
            self.to_pred = nn.Sequential(nn.Linear(dim, hl_gauss_loss.num_bins))

    def forward(self, embed, target=None):
        pred = self.to_pred(embed)
        if self.use_regression:
            pred = pred.squeeze(-1)
            if target is None:
                return pred
            return F.mse_loss(pred, target)
        return self.hl_gauss_loss(pred, target)


# ---------------------------------------------------------------------------------------------------------------------- oracle
def hl_gauss_probs(target, hl_gauss):
    """HLGaussLoss.transform_to_probs, functional: the Gaussian histogram of `target` [B] over `num_bins` bins of [min_value, max_value]
    in target's dtype; NaN where both ends of the cdf round to the same value (z = 0)."""
    lo, hi, nb = hl_gauss['min_value'], hl_gauss['max_value'], hl_gauss['num_bins']
    sigma = hl_gauss.get('sigma')
    sigma = sigma if sigma is not None else (hi - lo) / nb * hl_gauss.get('sigma_to_bin_ratio', SIGMA_TO_BIN_RATIO)
    support = torch.linspace(lo, hi, nb + 1, dtype=target.dtype, device=target.device)
    if hl_gauss.get('clamp_to_range', False):
        target = target.clamp(min=lo, max=hi)
    cdf = torch.special.erf((support - target[:, None]) / (math.sqrt(2.) * sigma))
    return (cdf[:, 1:] - cdf[:, :-1]) / (cdf[:, -1:] - cdf[:, :1])


def hl_gauss_centres(hl_gauss, dtype=torch.float32):
    support = torch.linspace(hl_gauss['min_value'], hl_gauss['max_value'], hl_gauss['num_bins'] + 1, dtype=dtype)
    return (support[:-1] + support[1:]) / 2


def duration_head(sd, pooled, target, hl_gauss):
    """HLGaussLayer on the pooled embedding, read from the state dict: the Softplus regression head with MSE (hl_gauss None) or the
    classification head of hl_gauss. The prediction when target is None, else the loss. A missing key, or weights whose rows are not
    the config's bins, raise KeyError."""
    w, bias = sd['hl_gauss_layer.to_pred.0.weight'], sd['hl_gauss_layer.to_pred.0.bias']
    if hl_gauss is None:
        pred = F.softplus(pooled @ w.t() + bias).squeeze(-1)
        return pred if target is None else F.mse_loss(pred, target)
    if w.shape[0] != hl_gauss['num_bins']:
        raise KeyError(f"hl_gauss_layer.to_pred.0.weight has {w.shape[0]} rows, the config {hl_gauss['num_bins']} bins")
    logits = pooled @ w.t() + bias
    if target is None:
        return (logits.softmax(-1) * hl_gauss_centres(hl_gauss, logits.dtype).to(logits.device)).sum(-1)
    return F.cross_entropy(logits, hl_gauss_probs(target.to(logits.dtype), hl_gauss))


def duration_forward(sd, cfg, mel, text, *, lens=None, rand_frac=None, return_loss=True, hl_gauss=None):
    """O.duration_forward (:1042-1113) with the head of `hl_gauss`: the prediction (:1107) or the loss against lens.float() (:1111)"""
    b, n, _ = mel.shape
    x = mel @ sd['proj_in.weight'].t() + sd['proj_in.bias']  # :1057
    te = O.character_embed(sd, text, n) if text is not None else None  # :1070
    if lens is None:
        lens = torch.full((b,), n, device=mel.device)
    mask = O.lens_to_mask(lens, n)
    if return_loss:  # :1081-1086
        rand_index = (rand_frac * lens).long()
        mask = mask & (torch.arange(n, device=mel.device)[None] < rand_index[:, None])
    emb = O.transformer_forward(sd, cfg, x, mask=mask, text_embed=te)
    num = (emb * mask[..., None]).sum(1)  # :212-224
    den = mask.float().sum(1).clamp(min=1.0)
    return duration_head(sd, num / den[:, None], lens.float() if return_loss else None, hl_gauss)
