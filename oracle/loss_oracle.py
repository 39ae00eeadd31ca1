# coding: utf-8
"""CPU oracle for the per-sample training criterion.  TEST INFRASTRUCTURE ONLY.

Restates, as plain torch CPU functions in the reference's op order, the three losses the reference trains with
(``reduce=False`` forms) and the masked mean its training step takes over them:
  * ``discretized_mix_logistic_loss`` (mixture.py:26-106),
  * ``mix_gaussian_loss`` (mixture.py:161-218, including the special case of 2 output channels),
  * the cross-entropy of the softmax head (train.py:346-362, nn.CrossEntropyLoss(reduction='none')),
  * ``criterion`` (train.py:727-748): head outputs ``[:, :, :-1]`` against targets ``[:, 1:]`` under the mask
    ``sequence_mask(lengths)[:, 1:]``.
``tests/golden/make_nll_golden.py`` writes the unmodified reference's losses to ``tests/golden/nll.npz`` and
``tests/test_forward_host.py`` checks these functions against them.  Every function returns (B,T) and accepts the
head outputs in float32 or float64 (the arithmetic follows the input's dtype).
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F


def _log_sum_exp(x):
    # mixture.py:17-23
    axis = len(x.size()) - 1
    m, _ = torch.max(x, dim=axis)
    m2, _ = torch.max(x, dim=axis, keepdim=True)
    return m + torch.log(torch.sum(torch.exp(x - m2), dim=axis))


def mol_nll(y_hat, y, num_classes=65536, log_scale_min=-16.0):
    """y_hat (B,3K,T), y (B,T) in [-1,1] -> (B,T)."""
    assert y_hat.dim() == 3 and y_hat.size(1) % 3 == 0
    nr_mix = y_hat.size(1) // 3
    y_hat = y_hat.transpose(1, 2)
    logit_probs = y_hat[:, :, :nr_mix]
    means = y_hat[:, :, nr_mix:2 * nr_mix]
    log_scales = torch.clamp(y_hat[:, :, 2 * nr_mix:3 * nr_mix], min=log_scale_min)
    y = y.unsqueeze(-1).to(y_hat.dtype).expand_as(means)
    centered_y = y - means
    inv_stdv = torch.exp(-log_scales)
    plus_in = inv_stdv * (centered_y + 1. / (num_classes - 1))
    cdf_plus = torch.sigmoid(plus_in)
    min_in = inv_stdv * (centered_y - 1. / (num_classes - 1))
    cdf_min = torch.sigmoid(min_in)
    log_cdf_plus = plus_in - F.softplus(plus_in)
    log_one_minus_cdf_min = -F.softplus(min_in)
    cdf_delta = cdf_plus - cdf_min
    mid_in = inv_stdv * centered_y
    log_pdf_mid = mid_in - log_scales - 2. * F.softplus(mid_in)
    inner_inner_cond = (cdf_delta > 1e-5).to(y_hat.dtype)
    inner_inner_out = inner_inner_cond * torch.log(torch.clamp(cdf_delta, min=1e-12)) + \
        (1. - inner_inner_cond) * (log_pdf_mid - np.log((num_classes - 1) / 2))
    inner_cond = (y > 0.999).to(y_hat.dtype)
    inner_out = inner_cond * log_one_minus_cdf_min + (1. - inner_cond) * inner_inner_out
    cond = (y < -0.999).to(y_hat.dtype)
    log_probs = cond * log_cdf_plus + (1. - cond) * inner_out
    log_probs = log_probs + F.log_softmax(logit_probs, -1)
    return -_log_sum_exp(log_probs)


def gauss_nll(y_hat, y, log_scale_min=-16.0):
    """y_hat (B,2,T) or (B,3K,T), y (B,T) -> (B,T)."""
    assert y_hat.dim() == 3
    C = y_hat.size(1)
    if C == 2:
        nr_mix = 1
    else:
        assert C % 3 == 0
        nr_mix = C // 3
    y_hat = y_hat.transpose(1, 2)
    if C == 2:
        logit_probs = None
        means = y_hat[:, :, 0:1]
        log_scales = torch.clamp(y_hat[:, :, 1:2], min=log_scale_min)
    else:
        logit_probs = y_hat[:, :, :nr_mix]
        means = y_hat[:, :, nr_mix:2 * nr_mix]
        log_scales = torch.clamp(y_hat[:, :, 2 * nr_mix:3 * nr_mix], min=log_scale_min)
    y = y.unsqueeze(-1).to(y_hat.dtype).expand_as(means)
    centered_y = y - means
    # torch.distributions.Normal(loc=0., scale=exp(log_scales)).log_prob(centered_y)
    scale = torch.exp(log_scales)
    var = scale ** 2
    log_probs = -((centered_y - 0.) ** 2) / (2 * var) - scale.log() - math.log(math.sqrt(2 * math.pi))
    if nr_mix > 1:
        log_probs = log_probs + F.log_softmax(logit_probs, -1)
        return -_log_sum_exp(log_probs)
    return -log_probs[:, :, 0]


def softmax_nll(y_hat, target):
    """y_hat (B,O,T) logits, target (B,T) classes -> (B,T): nn.CrossEntropyLoss(reduction='none')."""
    return F.cross_entropy(y_hat.unsqueeze(-1), target.long().unsqueeze(-1), reduction="none")[:, :, 0]


def per_sample(head_kind, y_hat, target, num_classes=65536, log_scale_min=-16.0):
    """head_kind: "mol", "gauss" or "softmax"."""
    if head_kind == "mol":
        return mol_nll(y_hat, target, num_classes=num_classes, log_scale_min=log_scale_min)
    if head_kind == "gauss":
        return gauss_nll(y_hat, target, log_scale_min=log_scale_min)
    return softmax_nll(y_hat, target)


def sequence_mask(lengths, max_len):
    # train.py sequence_mask: (B, max_len), True where t < lengths[b]
    return torch.arange(max_len).unsqueeze(0) < lengths.view(-1, 1)


def criterion(head_kind, y_hat, target, lengths=None, num_classes=65536, log_scale_min=-16.0, reduce=True):
    """train.py:727-748: the losses of y_hat[:, :, :-1] against target[:, 1:], masked mean over
    sequence_mask(lengths)[:, 1:] (every sample without lengths)."""
    T = y_hat.size(-1)
    losses = per_sample(head_kind, y_hat[:, :, :-1], target[:, 1:], num_classes=num_classes,
                        log_scale_min=log_scale_min)
    if not reduce:
        return losses
    if lengths is None:
        mask = torch.ones_like(losses)
    else:
        mask = sequence_mask(torch.as_tensor(lengths), T)[:, 1:].to(losses.dtype)
    return (losses * mask).sum() / mask.sum()
