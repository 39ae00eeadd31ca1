# coding: utf-8
"""Teacher-forced scoring without a GPU:
  - oracle/loss_oracle.py equals the unmodified reference's per-sample losses stored in tests/golden/nll.npz, on every
    branch (cdf_delta on both sides of 1e-5 at 256 and 65536 classes, targets beyond +-0.999, clamped log-scales,
    Gaussian heads of 2, 3 and 3K channels, a one-component MoL head, softmax heads of 255 and 256 classes);
  - wn_nll and the stand-alone samplers refuse malformed arguments before they touch the device;
  - the library exports wn_forward and wn_nll, still reports ABI 3 and seven structs, and carries sm_90a code."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import loss_oracle as lo
from wavenet_vocoder_b200 import _native as N

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nll.npz")
HEADS = {"mol": N.WN_HEAD_MOL, "gauss": N.WN_HEAD_GAUSS, "softmax": N.WN_HEAD_SOFTMAX}


def nll_cases():
    z = np.load(GOLDEN, allow_pickle=False)
    return [str(n) for n in z["cases"]]


def nll_case(name):
    z = np.load(GOLDEN, allow_pickle=False)
    return dict(head=str(z[name + ".head"]), y_hat=torch.from_numpy(z[name + ".y_hat"]),
                y=torch.from_numpy(z[name + ".y"]), loss=torch.from_numpy(z[name + ".loss"]),
                num_classes=int(z[name + ".num_classes"]), log_scale_min=float(z[name + ".log_scale_min"]))


@pytest.mark.parametrize("name", nll_cases())
def test_oracle_losses_equal_reference(name):
    cs = nll_case(name)
    got = lo.per_sample(cs["head"], cs["y_hat"], cs["y"], num_classes=cs["num_classes"],
                        log_scale_min=cs["log_scale_min"])
    ref = cs["loss"]
    assert got.shape == ref.shape and got.dtype == torch.float32
    rel = float(((got - ref).abs() / ref.abs().clamp(min=1e-30)).max())
    assert rel <= 1e-6, rel


def test_golden_losses_reach_every_branch():
    seen = {"above": 0, "below": 0, "edge_hi": 0, "edge_lo": 0, "clamped": 0}
    for name in nll_cases():
        cs = nll_case(name)
        if cs["head"] != "mol":
            continue
        y_hat, y, K = cs["y_hat"], cs["y"], cs["y_hat"].size(1) // 3
        half = 1.0 / (cs["num_classes"] - 1)
        lsc = y_hat[:, 2 * K:].clamp(min=cs["log_scale_min"])
        c = y.unsqueeze(1) - y_hat[:, K:2 * K]
        delta = torch.sigmoid(torch.exp(-lsc) * (c + half)) - torch.sigmoid(torch.exp(-lsc) * (c - half))
        seen["above"] += int(((delta > 1e-5) & (delta < 1e-4)).sum())
        seen["below"] += int(((delta <= 1e-5) & (delta > 1e-6)).sum())
        seen["edge_hi"] += int((y > 0.999).sum())
        seen["edge_lo"] += int((y < -0.999).sum())
        seen["clamped"] += int((y_hat[:, 2 * K:] < cs["log_scale_min"]).sum())
    assert all(v > 0 for v in seen.values()), seen
    widths = {}
    for n in nll_cases():
        cs = nll_case(n)
        widths.setdefault(cs["head"], set()).add(cs["y_hat"].size(1))
    # a single Gaussian of 2 and of 3 channels, a one-component MoL, and an odd number of classes
    assert widths["gauss"] >= {2, 3, 9} and 3 in widths["mol"] and 255 in widths["softmax"], widths


def test_oracle_criterion_masks_as_train_py():
    cs = nll_case("mol_nc256")
    y_hat, y = cs["y_hat"], cs["y"]
    T = y.size(1)
    per = lo.criterion("mol", y_hat, y, num_classes=256, reduce=False)
    assert per.shape == (y.size(0), T - 1)
    lengths = torch.tensor([T, T // 2])
    want = (per[0].sum() + per[1, :T // 2 - 1].sum()) / (T - 1 + T // 2 - 1)
    got = lo.criterion("mol", y_hat, y, lengths=lengths, num_classes=256)
    assert torch.allclose(got, want, rtol=1e-6, atol=0)
    assert torch.allclose(lo.criterion("mol", y_hat, y, num_classes=256), per.mean(), rtol=1e-6, atol=0)


# ---- wn_nll refusals: every one returns before a kernel is launched, so none needs a device -------------------------
FAKE = C.c_void_p(16)       # never dereferenced: the argument checks come first


def nll_status(head=N.WN_HEAD_MOL, B=2, O=30, T=8, y=FAKE, cls=None, num_classes=256):
    return N.lib().wn_nll(FAKE, head, B, O, T, y, cls, num_classes, -16.0, FAKE, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(B=0), "B, O and T"),
    (dict(T=0), "B, O and T"),
    (dict(O=31), "3K channels"),
    (dict(head=N.WN_HEAD_GAUSS, O=4), "2 or 3K"),
    (dict(num_classes=1), "num_classes"),
    (dict(y=None), "target is required"),
    (dict(cls=FAKE), "not both"),
    (dict(head=N.WN_HEAD_SOFTMAX, O=256), "class_target"),
    (dict(head=N.WN_HEAD_SOFTMAX, O=256, y=None, cls=FAKE, B=-1), "B, O and T"),
    (dict(head=7), "head_kind"),
])
def test_wn_nll_refuses_malformed_arguments(kw, msg):
    rc = nll_status(**kw)
    assert rc == -1, rc
    assert msg in N.lib().wn_last_error().decode(), N.lib().wn_last_error()


@pytest.mark.parametrize("fn", ["wn_sample_mol", "wn_sample_gauss"])
@pytest.mark.parametrize("B,O,T", [(0, 3, 8), (2, 3, 0), (2, 0, 8), (-1, 3, 8), (2, -3, 8), (2, 3, -8)])
def test_samplers_refuse_empty_shapes(fn, B, O, T):
    """O = 0 passes the O % 3 check: without the shape check the kernel would read an empty head."""
    rc = getattr(N.lib(), fn)(FAKE, B, O, T, FAKE, FAKE, FAKE, None)
    assert rc == -1, rc
    assert "%s: B, O and T must be >= 1" % fn in N.lib().wn_last_error().decode(), N.lib().wn_last_error()


def test_forward_entry_points_without_an_abi_bump():
    lib = N.lib()
    for name in ("wn_forward", "wn_nll"):
        assert name in N.EXPORTS and hasattr(lib, name), name
    assert lib.wn_abi_version() == N.WN_ABI_VERSION == 3
    sizes = (C.c_int32 * 8)()
    assert lib.wn_struct_sizes(sizes, 8) == 7
    assert N.lib().wn_forward(None, None) == -1
    assert os.path.join(N.HERE, "csrc", "wn_dense.cuh") in N.HEADERS


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_library_carries_sm90a_code():
    out = subprocess.run(["cuobjdump", "--list-elf", N.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out, out
    syms = subprocess.run(["cuobjdump", "--dump-elf-symbols", N.LIB_PATH], capture_output=True, text=True).stdout
    assert "dense_gemm_kernel" in syms and "nll_kernel" in syms
