# coding: utf-8
"""Streaming synthesis on the GPU: an utterance made chunk by chunk (WaveNet.open_stream, wn_stream_* of the C ABI)
is bit-identical to the same utterance made by one incremental_forward call, for irregular splits, replayed and
Philox noise, batch tiles of 1, 3 and 4, both ring placements, conditioning frames pushed in groups, and interleaved
streams; StreamDecoder equals decode_device bit for bit; every misuse is refused."""
import ctypes as C

import pytest
import torch

from conftest import GOLDEN_CASES
from helpers import GoldenCase
from oracle import wavenet_oracle as orc
from wavenet_vocoder_b200 import WaveNet
from wavenet_vocoder_b200 import _native as N

pytestmark = pytest.mark.gpu


def model_of(kw, sd=None, seed=0):
    torch.manual_seed(seed)
    m = WaveNet(**kw)
    if sd is not None:
        m.load_state_dict(sd)
    else:
        with torch.no_grad():
            for n_, p in m.named_parameters():
                if n_.endswith(".bias"):
                    p.normal_(0, 0.05)
    return m.cuda().eval()


def max_dilation(kw):
    return 2 ** (kw["layers"] // kw["stacks"] - 1)


def irregular_split(T, maxdil):
    parts, left = [], T
    for p in (1, 7, 64, 2 * maxdil + 1):
        if left <= 0:
            break
        parts.append(min(p, left))
        left -= parts[-1]
    if left > 0:
        parts.append(left)
    return parts


def inputs_for(m, kw, B, T, gen):
    """initial input (defines B for models without conditioning), c (sample rate or frames), g."""
    O = kw["out_channels"]
    if kw.get("scalar_input", False):
        init = torch.rand(B, 1, 1, generator=gen) * 0.2 - 0.1
    else:
        init = torch.zeros(B, O, 1)
        init[:, 127] = 1.0
    c = None
    cin = kw.get("cin_channels", -1)
    if cin > 0:
        if kw.get("upsample_conditional_features", False):
            eng = m._get_engine()
            F = T // eng.ups_total + eng.ups_frames_lost + 2 * (eng.ups_indent // eng.ups_total)
            assert eng.upsampled_length(F) == T
            c = torch.randn(B, cin, F, generator=gen)
        else:
            c = torch.randn(B, cin, T, generator=gen)
    g = torch.randint(0, kw["n_speakers"], (B, 1), generator=gen) if kw.get("gin_channels", -1) > 0 else None
    return init, c, g


def one_shot(m, B, T, init, c, g, noise, seed):
    return m.incremental_forward(initial_input=init, c=c, g=g, T=T, noise=noise, seed=seed, return_params=True)


def chunked(m, kw, B, T, init, c, g, noise, seed, split=None):
    s = m.open_stream(B=B, g=g, initial_input=init, seed=seed, noise=noise, return_params=True)
    ys, ps = [], []
    if kw.get("upsample_conditional_features", False):
        # frames in irregular groups, then the tail
        F, f = c.size(-1), 0
        for n in (1, 2, 3, 5, 1):
            if f + n > F:
                break
            y, p = s.push_frames(c[:, :, f:f + n])
            ys.append(y), ps.append(p)
            f += n
        if f < F:
            y, p = s.push_frames(c[:, :, f:])
            ys.append(y), ps.append(p)
        y, p = s.finish()
        ys.append(y), ps.append(p)
    else:
        t = 0
        for n in split or irregular_split(T, max_dilation(kw)):
            y, p = s.generate(n, c=None if c is None else c[:, :, t:t + n])
            ys.append(y), ps.append(p)
            t += n
    assert s.t == T
    s.close()
    return torch.cat(ys, -1), torch.cat(ps, -1)


def assert_same(a, b):
    assert a[0].shape == b[0].shape and a[1].shape == b[1].shape
    assert torch.equal(a[0], b[0]), float((a[0].float() - b[0].float()).abs().max())
    assert torch.equal(a[1], b[1]), float((a[1] - b[1]).abs().max())


@pytest.mark.parametrize("noise_kind", ["replay", "philox"])
@pytest.mark.parametrize("B", [1, 3, 4])
@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_golden_cases_chunked_equal_one_shot(name, B, noise_kind):
    gc = GoldenCase(name)
    m = model_of(gc.kw, gc.sd)
    T = 160
    gen = torch.Generator().manual_seed(B)
    init, c, g = inputs_for(m, gc.kw, B, T, gen)
    noise = {k: v.cuda() for k, v in orc.predraw_noise(gc.cfg, B, T, 5).items()} if noise_kind == "replay" else None
    seed = None if noise is not None else 1234 + B
    assert m._get_engine().plan(B)["rings_in_smem"] == 1
    assert_same(chunked(m, gc.kw, B, T, init, c, g, noise, seed), one_shot(m, B, T, init, c, g, noise, seed))


CFG5 = dict(out_channels=30, layers=30, stacks=3, residual_channels=256, gate_channels=512, skip_out_channels=256,
            cin_channels=80, gin_channels=-1, scalar_input=True, output_distribution="Logistic", dropout=0.0)


def cfg_noise(kw, B, T, seed):
    cfg = orc.PathConfig(out_channels=kw["out_channels"], layers=kw["layers"], stacks=kw["stacks"],
                         residual_channels=kw["residual_channels"], gate_channels=kw["gate_channels"],
                         skip_out_channels=kw["skip_out_channels"], kernel_size=3, cin_channels=kw["cin_channels"],
                         gin_channels=-1, scalar_input=True, output_distribution="Logistic")
    return {k: v.cuda() for k, v in orc.predraw_noise(cfg, B, T, seed).items()}


@pytest.mark.parametrize("B", [1, 3])
def test_rings_in_global_memory(B):
    """Config 5's shape: its history rings do not fit in shared memory, so the stream state IS the rings."""
    m = model_of(CFG5)
    assert m._get_engine().plan(B)["rings_in_smem"] == 0
    T = 2 * max_dilation(CFG5) + 100
    gen = torch.Generator().manual_seed(3)
    init, c, g = inputs_for(m, CFG5, B, T, gen)
    for noise, seed in ((cfg_noise(CFG5, B, T, 8), None), (None, 77)):
        assert_same(chunked(m, CFG5, B, T, init, c, g, noise, seed), one_shot(m, B, T, init, c, g, noise, seed))


def upsample_model(scales, cin_pad, C=16):
    kw = dict(out_channels=30, layers=4, stacks=2, residual_channels=16, gate_channels=32, skip_out_channels=16,
              cin_channels=C, cin_pad=cin_pad, scalar_input=True, dropout=0.0, upsample_conditional_features=True,
              upsample_net="ConvInUpsampleNetwork",
              upsample_params={"upsample_scales": scales, "cin_channels": C, "cin_pad": cin_pad})
    m = model_of(kw)
    with torch.no_grad():
        for n_, p in m.upsample_net.named_parameters():
            if n_.endswith("weight_v"):
                p.add_(0.05 * torch.randn_like(p))
    return m, kw


@pytest.mark.parametrize("scales", [[4, 4, 4, 4], [4, 5, 5, 3]])
def test_push_frames_then_finish_equal_incremental_forward(scales):
    m, kw = upsample_model(scales, 2)
    eng = m._get_engine()
    assert m._native_upsample
    F = 4 + 5 + 2 * 2
    gen = torch.Generator().manual_seed(6)
    frames = torch.randn(2, kw["cin_channels"], F, generator=gen).cuda()
    T = eng.upsampled_length(F)
    ref = m.incremental_forward(c=frames, T=T, seed=11)
    s = m.open_stream(B=2, seed=11)
    outs, f = [], 0
    for n in (1, 3, 1, 2, 4, 2):
        y = s.push_frames(frames[:, :, f:f + n])
        f += n
        ready = eng.upsample_cone(f, False)[2]
        assert y.size(-1) == ready - sum(o.size(-1) for o in outs), (f, ready)
        assert s.t == ready
        outs.append(y)
    assert f == F
    outs.append(s.finish())
    got = torch.cat(outs, -1)
    assert got.shape == ref.shape and torch.equal(got, ref)


def test_interleaved_streams_equal_streams_alone():
    gc = GoldenCase("mol_cond")
    m = model_of(gc.kw, gc.sd)
    T = 120
    gen = torch.Generator().manual_seed(7)
    c1, c2 = torch.randn(1, 8, T, generator=gen).cuda(), torch.randn(3, 8, T, generator=gen).cuda()
    alone1 = m.incremental_forward(c=c1, T=T, seed=1)
    alone2 = m.incremental_forward(c=c2, T=T, seed=2)
    s1, s2 = m.open_stream(B=1, seed=1), m.open_stream(B=3, seed=2)
    o1, o2, t1, t2 = [], [], 0, 0
    for n1, n2 in ((5, 17), (40, 3), (75, 100)):
        o1.append(s1.generate(n1, c=c1[:, :, t1:t1 + n1]))
        o2.append(s2.generate(n2, c=c2[:, :, t2:t2 + n2]))
        t1, t2 = t1 + n1, t2 + n2
    assert torch.equal(torch.cat(o1, -1), alone1) and torch.equal(torch.cat(o2, -1)[:, :, :T], alone2)


@pytest.mark.parametrize("input_type", ["raw", "mulaw", "mulaw-quantize"])
def test_stream_decoder_equals_decode_device(input_type):
    from wavenet_vocoder_b200.dispatch import StreamDecoder, decode_device
    B, T = 3, 4000
    gen = torch.Generator().manual_seed(8)
    if input_type == "mulaw-quantize":
        y = torch.randn(B, 256, T, generator=gen).cuda()
    else:
        y = (torch.rand(B, 1, T, generator=gen) * 1.8 - 0.9).cuda()
    kw = dict(input_type=input_type, quantize_channels=256, postprocess="inv_preemphasis", global_gain_scale=0.9,
              preemphasis_coef=0.85)
    lengths = [T, T - 1700, 5]
    pcm, flt = decode_device(y, lengths, want_float=True, **kw)
    dec = StreamDecoder(B, "cuda", lengths=lengths, want_float=True, **kw)
    parts, t = [], 0
    for n in (1, 100, 1023, 1500, T - 2624):
        parts.append(dec(y[:, :, t:t + n]))
        t += n
    assert torch.equal(torch.cat([p[0] for p in parts], -1), pcm)
    assert torch.equal(torch.cat([p[1] for p in parts], -1), flt)


def test_misuse_is_refused_and_nothing_faults(monkeypatch):
    gc = GoldenCase("mol_cond")
    m = model_of(gc.kw, gc.sd)
    eng = m._get_engine()
    gen = torch.Generator().manual_seed(9)
    c = torch.randn(1, 8, 64, generator=gen).cuda()
    with pytest.raises(N.WnError, match="batch tile"):
        m.open_stream(B=5, seed=1)
    # teacher forcing inside a stream (the Python surface has no way to ask for it: straight through the C ABI)
    s = eng.open_stream(B=1, seed=1)
    ct = c.transpose(1, 2).contiguous()
    out, ts = torch.empty(1, 8, device="cuda"), torch.zeros(1, 2, device="cuda")
    a = N.wn_generate_args()
    a.B, a.T, a.c, a.out_scalar = 1, 8, ct.data_ptr(), out.data_ptr()
    a.T_test, a.test_scalar = 2, ts.data_ptr()
    assert N.lib().wn_stream_generate(s._s, C.byref(a), None) == -1
    assert b"teacher forcing" in N.lib().wn_last_error()
    # a chunk marked final, then one more
    y1, _ = s.generate(8, c=ct[:, :8], final=True)
    with pytest.raises(N.WnError, match="finalised"):
        s.generate(8, c=ct[:, 8:16])
    s.close()
    # the stream's first chunk equals the one-shot call, after all of the above
    assert torch.equal(y1.view(1, 1, 8), m.incremental_forward(c=c[:, :, :8], T=8, seed=1))
    # weights changed after the stream was opened
    s = m.open_stream(B=1, seed=3)
    s.generate(4, c=c[:, :, :4])
    with torch.no_grad():
        m.first_conv.bias.add_(0.01)
    with pytest.raises(N.WnError, match="weights changed"):
        s.generate(4, c=c[:, :, 4:8])
    s.close()
    # a frame window that does not cover the samples' cone
    mu, kw = upsample_model([4, 4], 1)
    eu = mu._get_engine()
    frames = torch.randn(1, 16, 12, generator=gen).cuda()
    su = eu.open_stream(B=1, seed=4)
    f_lo, f_hi, ready = eu.upsample_cone(12, True, 0, 40)
    assert (f_lo, ready) == (0, eu.upsampled_length(12))
    with pytest.raises(N.WnError, match="does not cover"):
        su.generate(40, c_frames=frames[:, :, :f_hi - 1], frame_offset=0, frames_total=12)
    with pytest.raises(N.WnError, match="not known yet"):
        su.generate(40, c_frames=frames[:, :, :3], frame_offset=0, frames_total=3)
    y, _ = su.generate(40, c_frames=frames[:, :, :f_hi], frame_offset=0, frames_total=12, final=False)
    su.close()
    ref = mu.incremental_forward(c=frames, T=eu.upsampled_length(12), seed=4)
    assert torch.equal(y.view(1, 1, 40), ref[:, :, :40])
    # engine 7 has no stream entry
    monkeypatch.setenv("WN_ENGINE", "7")
    m7 = model_of(gc.kw, gc.sd)
    with pytest.raises(N.WnError, match="engine 5"):
        m7.open_stream(B=1, seed=1)
