# coding: utf-8
"""Generate tests/golden/nll.npz by running the UNMODIFIED reference's losses.

Needs a checkout of the reference (r9y9/wavenet_vocoder), found as oracle/stage_reference.py finds it (a directory
named ``reference`` or ``wavenet_vocoder`` next to this repository or above it) or named by WAVENET_VOCODER_REF:

    python tests/golden/make_nll_golden.py

Writes only ``nll.npz``: the reference's per-sample losses (``reduce=False``) of ``discretized_mix_logistic_loss``
(mixture.py:26-106), ``mix_gaussian_loss`` (mixture.py:161-218) and the cross-entropy of the softmax head
(train.py:346-362) on seeded head outputs and targets.  tests/test_forward_host.py compares oracle/loss_oracle.py with
them and tests/test_forward.py the device kernel.  The other golden files (make_golden.py) are left as they are:
``savez_compressed`` output is not byte-stable.
"""
import math
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.stage_reference import find_reference  # noqa: E402

REF_CHECKOUT = find_reference()
if REF_CHECKOUT is None:
    sys.exit("make_nll_golden.py needs a checkout of r9y9/wavenet_vocoder: set WAVENET_VOCODER_REF to its directory")
sys.path.insert(0, REF_CHECKOUT)
warnings.filterwarnings("ignore")

from wavenet_vocoder import mixture as ref_mixture     # noqa: E402  (the reference)

# nll.npz: the reference's per-sample losses (reduce=False) on seeded head outputs and targets.
# name: (head, out_channels, num_classes, log_scale_min)
NLL_CASES = {
    "mol_nc256": ("mol", 9, 256, -16.0),
    "mol_nc65536": ("mol", 9, 65536, -16.0),
    "mol_nc256_lsm7": ("mol", 30, 256, -7.0),
    "gauss_o2": ("gauss", 2, 65536, -7.0),
    "gauss_o9": ("gauss", 9, 65536, -16.0),
    "softmax_o256": ("softmax", 256, 256, -16.0),
}
NLL_B, NLL_T = 2, 96
Y_EDGE, Y_MARGIN, DELTA_MARGIN = 0.999, 1e-4, 0.1    # |y| - 0.999 and cdf_delta / 1e-5 - 1 stay this far from 0


def _mol_case(O, nc, lsm, gen):
    """Head outputs (B,O,T) and targets (B,T) for a MoL head.  Every sample puts all K components in one regime:
    the centre of the distribution, cdf_delta just above or just below 1e-5 (left tail, bins 3 logistic widths wide
    so that cdf_delta is computed without cancellation), the far tail (the log_pdf_mid branch), log-scales below
    log_scale_min (clamped), or a target beyond +-0.999."""
    K, B, T = O // 3, NLL_B, NLL_T
    half = 1.0 / (nc - 1)
    logits = torch.randn(B, K, T, generator=gen)
    y = (torch.rand(B, T, generator=gen) * 1.6 - 0.8)
    ls = torch.empty(B, K, T)
    centered = torch.empty(B, K, T)
    regimes = ["centre", "above", "below", "tail", "clamped", "edge"]
    for i in range(T):
        r = regimes[i % len(regimes)]
        for b in range(B):
            if r in ("above", "below") and lsm > -11.6 and nc > 256:
                r = "centre"
            if r == "centre" or r == "edge":
                # bins 1..4 logistic widths wide: narrower ones make cdf_plus - cdf_min cancel in fp32 (at 65536
                # classes and log-scales of -5..-2 the reference's own fp32 loss is 8e-5 off its float64 value)
                w = 1.0 + torch.rand(K, generator=gen) * 3
                ls[b, :, i] = -torch.log(w / (2 * half))
                centered[b, :, i] = torch.randn(K, generator=gen) * 2 * torch.exp(ls[b, :, i])
                if r == "edge":
                    y[b, i] = float(np.random.RandomState(i + 7 * b).choice([0.9995, 0.9985, -0.9995, -0.9985]))
            elif r in ("above", "below"):
                w = 3.0                                           # plus_in - min_in
                inv = w / (2 * half)
                target = (torch.rand(K, generator=gen) * 1.5 + 1.3) * 1e-5 if r == "above" else \
                    (torch.rand(K, generator=gen) * 4.0 + 3.0) * 1e-6
                plus = torch.log(target / (1 - math.exp(-w)))
                ls[b, :, i] = -math.log(inv)
                centered[b, :, i] = plus / inv - half
            elif r == "tail":
                ls[b, :, i] = torch.rand(K, generator=gen) * 2 - 6
                centered[b, :, i] = -(0.2 + torch.rand(K, generator=gen) * 0.3)
            else:                                                # clamped: raw log-scale below log_scale_min
                ls[b, :, i] = lsm - 1.0 - torch.rand(K, generator=gen) * 3
                centered[b, :, i] = torch.randn(K, generator=gen) * 2 * half
    y = y.float()

    def branch_delta(y_hat):
        # the branch quantity in fp32, recomputed from the stored tensors
        lsc = torch.clamp(y_hat[:, 2 * K:], min=lsm)
        c = y.unsqueeze(1) - y_hat[:, K:2 * K]
        inv = torch.exp(-lsc)
        return torch.sigmoid(inv * (c + half)) - torch.sigmoid(inv * (c - half))

    y_hat = torch.cat([logits, y.unsqueeze(1) - centered, ls], dim=1).float()
    # a component that landed near the threshold by chance is moved to the centre of its distribution
    near = (branch_delta(y_hat) / 1e-5 - 1).abs() < DELTA_MARGIN
    y_hat[:, K:2 * K][near] = y.unsqueeze(1).expand(B, K, T)[near]
    delta = branch_delta(y_hat)
    assert float((delta / 1e-5 - 1).abs().min()) >= DELTA_MARGIN, float((delta / 1e-5 - 1).abs().min())
    assert float((y.abs() - Y_EDGE).abs().min()) >= Y_MARGIN
    return y_hat, y, delta


def _gauss_case(O, lsm, gen):
    B, T = NLL_B, NLL_T
    K = 1 if O == 2 else O // 3
    y = torch.rand(B, T, generator=gen) * 1.8 - 0.9
    ls = torch.rand(B, K, T, generator=gen) * 4 - 5
    ls[:, :, ::4] = lsm - 1.0 - torch.rand(B, K, (T + 3) // 4, generator=gen) * 2      # clamped
    centered = torch.randn(B, K, T, generator=gen) * torch.exp(ls.clamp(min=lsm)) * 2
    means = y.unsqueeze(1) - centered
    if O == 2:
        return torch.cat([means, ls], dim=1).float(), y.float()
    logits = torch.randn(B, K, T, generator=gen)
    return torch.cat([logits, means, ls], dim=1).float(), y.float()


def make_nll():
    """tests/golden/nll.npz: the unmodified reference's per-sample losses (reduce=False) of every NLL_CASES case."""
    out = {"cases": np.array(list(NLL_CASES))}
    for n, (name, (head, O, nc, lsm)) in enumerate(NLL_CASES.items()):
        gen = torch.Generator().manual_seed(500 + n)
        if head == "mol":
            y_hat, y, delta = _mol_case(O, nc, lsm, gen)

            def ref_loss(y_hat, y):
                return ref_mixture.discretized_mix_logistic_loss(y_hat, y.unsqueeze(-1), num_classes=nc,
                                                                 log_scale_min=lsm, reduce=False)[:, :, 0]
            loss = ref_loss(y_hat, y)
            # a sample whose fp32 loss is not within 1e-6 of its float64 value (cancellation in c + 1/(nc-1) next to
            # a clamped log-scale) cannot pin a device kernel to 1e-5: its components move to the centre
            bad = (ref_loss(y_hat.double(), y.double()) - loss.double()).abs() > 1e-6 * loss.double().abs().clamp(min=1)
            K = O // 3
            means = y_hat[:, K:2 * K]
            means[bad.unsqueeze(1).expand_as(means)] = y.unsqueeze(1).expand_as(means)[bad.unsqueeze(1).expand_as(means)]
            loss = ref_loss(y_hat, y)
            gap = (ref_loss(y_hat.double(), y.double()) - loss.double()).abs() / loss.double().abs().clamp(min=1)
            assert float(gap.max()) <= 1e-6, float(gap.max())
            delta = torch.sigmoid(torch.exp(-y_hat[:, 2 * K:].clamp(min=lsm)) * (y.unsqueeze(1) - means + 1 / (nc - 1))) - \
                torch.sigmoid(torch.exp(-y_hat[:, 2 * K:].clamp(min=lsm)) * (y.unsqueeze(1) - means - 1 / (nc - 1)))
            assert float((delta / 1e-5 - 1).abs().min()) >= DELTA_MARGIN
            print("%-16s cdf_delta > 1e-5 on %d of %d components, |y| > 0.999 on %d samples" % (
                name, int((delta > 1e-5).sum()), delta.numel(), int((y.abs() > Y_EDGE).sum())))
        elif head == "gauss":
            y_hat, y = _gauss_case(O, lsm, gen)
            loss = ref_mixture.mix_gaussian_loss(y_hat, y.unsqueeze(-1), log_scale_min=lsm, reduce=False)[:, :, 0]
        else:
            y_hat = torch.randn(NLL_B, O, NLL_T, generator=gen) * 2
            y = torch.randint(0, O, (NLL_B, NLL_T), generator=gen)
            # train.py:346-362: MaskedCrossEntropyLoss's criterion on (B,C,T,1) against (B,T,1)
            loss = torch.nn.CrossEntropyLoss(reduction="none")(y_hat.unsqueeze(-1), y.unsqueeze(-1))[:, :, 0]
            y = y.to(torch.int32)
        assert bool(torch.isfinite(loss).all()), name
        out[name + ".y_hat"] = y_hat.numpy()
        out[name + ".y"] = y.numpy()
        out[name + ".loss"] = loss.detach().numpy()
        out[name + ".head"] = np.array(head)
        out[name + ".num_classes"] = np.int32(nc)
        out[name + ".log_scale_min"] = np.float32(lsm)
    np.savez_compressed(os.path.join(HERE, "nll.npz"), **out)


if __name__ == "__main__":
    make_nll()
