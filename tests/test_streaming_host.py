# coding: utf-8
"""Host side of streaming synthesis, without a GPU: the ABI-3 entry points and struct layouts, ABI-2 configs still
accepted, and wn_upsample_cone (the frame window a range of samples needs, and how many samples a prefix of frames
determines) against brute force on the PyTorch upsample networks."""
import ctypes as C

import pytest
import torch

from wavenet_vocoder_b200 import _native as N
from wavenet_vocoder_b200 import upsample as U
from wavenet_vocoder_b200.engine import make_config, upsample_cone, upsampler_struct

STREAM_EXPORTS = ["wn_stream_open", "wn_stream_generate", "wn_stream_position", "wn_stream_close", "wn_upsample_cone",
                  "wn_decode_stream"]


def test_abi3_exports_and_struct_sizes():
    lib = N.lib()
    assert lib.wn_abi_version() == 3
    for name in STREAM_EXPORTS:
        assert name in N.EXPORTS and hasattr(lib, name), name
    sizes = (C.c_int32 * 8)()
    assert lib.wn_struct_sizes(sizes, 8) == 7
    assert list(sizes)[:7] == [C.sizeof(t) for t in N.STRUCTS]
    assert lib.wn_struct_sizes(sizes, 5) == 5          # a version-2 binding asks for five


def test_config_of_abi_version_2_is_accepted():
    cfg = make_config(layers=4, stacks=2, residual_channels=16, gate_channels=32, skip_out_channels=16,
                      out_channels=30, kernel_size=3, cin_channels=8, gin_channels=-1, scalar_input=True,
                      output_distribution="Logistic")
    info = N.wn_plan_info()
    for version, rc in ((2, 0), (3, 0), (1, -1), (4, -1)):
        cfg.abi_version = version
        assert N.lib().wn_plan_only(C.byref(cfg), 1, 132, 232448, C.byref(info)) == rc, version


CASES = [([4, 4, 4, 4], 2, "ConvInUpsampleNetwork", 17),
         ([4, 5, 5, 3], 2, "ConvInUpsampleNetwork", 9),
         ([2, 4], 0, "ConvInUpsampleNetwork", 33),
         ([4, 4], 1, "UpsampleNetwork", 12),
         ([16, 16], 0, "UpsampleNetwork", 5)]
CH = 3


def net_for(scales, cin_pad, net):
    torch.manual_seed(0)
    m = getattr(U, net)(upsample_scales=scales, cin_pad=cin_pad, cin_channels=CH)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if n_.endswith("weight_g"):
                p.mul_(1.0 + 0.3 * torch.rand_like(p))
            if n_.endswith("weight_v"):
                p.add_(0.05 * torch.randn_like(p))
    return m.eval()


def run(m, c):
    with torch.no_grad():
        return m(c)[0]                                  # (C, T)


@pytest.mark.parametrize("scales,cin_pad,net,frames", CASES)
def test_cone_window_is_exact(scales, cin_pad, net, frames):
    """Frames outside the window do not touch the range; the first and the last frame of the window do."""
    m = net_for(scales, cin_pad, net)
    d = upsampler_struct(m, CH)
    F = frames + 2 * cin_pad
    gen = torch.Generator().manual_seed(1)
    c = torch.randn(1, CH, F, generator=gen)
    ref = run(m, c)
    T = ref.size(-1)
    assert upsample_cone(d["u"], F, True)[2] == T
    for t_lo, t_hi in [(0, 1), (0, T), (T - 1, T), (T // 3, T // 3 + 7), (T // 2, T - 2), (5, 6)]:
        f_lo, f_hi, _ = upsample_cone(d["u"], F, True, t_lo, t_hi)
        assert 0 <= f_lo < f_hi <= F
        for f in range(F):
            c2 = c.clone()
            c2[:, :, f] += 100.0
            diff = float((run(m, c2)[:, t_lo:t_hi] - ref[:, t_lo:t_hi]).abs().max())
            if f < f_lo or f >= f_hi:
                assert diff == 0.0, (t_lo, t_hi, f, f_lo, f_hi, diff)
            elif f in (f_lo, f_hi - 1):
                assert diff > 1e-3, (t_lo, t_hi, f, f_lo, f_hi, diff)      # shrinking the window by it would be wrong


@pytest.mark.parametrize("scales,cin_pad,net,frames", CASES)
def test_samples_ready_after_a_prefix_are_final(scales, cin_pad, net, frames):
    """The samples wn_upsample_cone calls ready after n frames are those of the full sequence, whatever follows.
    PyTorch's CPU convolution sums in an order that depends on the input length (1-2 ulp here), so the bound is 1e-6;
    a frame outside the cone would move them by the size of the continuation (x10)."""
    m = net_for(scales, cin_pad, net)
    d = upsampler_struct(m, CH)
    F = frames + 2 * cin_pad
    gen = torch.Generator().manual_seed(2)
    c = torch.randn(1, CH, F, generator=gen)
    ref = run(m, c)
    last = 0
    for n in range(1, F + 1):
        _, _, ready = upsample_cone(d["u"], n, False)
        assert last <= ready <= max(0, ref.size(-1))
        last = ready
        if ready == 0:
            continue
        for tail in (0, 1, 3):        # the prefix ending here, and two other continuations
            c2 = torch.cat([c[:, :, :n], torch.randn(1, CH, tail, generator=gen) * 10], dim=-1)
            got = run(m, c2)
            assert float((got[:, :ready] - ref[:, :ready]).abs().max()) <= 1e-6, (n, tail, ready)
    # with every frame known and final, everything is ready
    assert upsample_cone(d["u"], F, True)[2] == ref.size(-1)
