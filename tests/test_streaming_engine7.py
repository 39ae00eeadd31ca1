# coding: utf-8
"""Engine-7 streams on the GPU (WaveNet.open_stream(engine=7), wn_stream_open_args.engine = 7): up to 8 utterances in
one batch tile, chunk by chunk.  Every chunked run is bit-identical (outputs and head outputs) to one call on the same
engine-7 handle with the same noise and conditioning, for irregular splits, chunks of one sample across every ring
phase, replayed and Philox noise, tiles of 1, 2, 4 and 8 (partly filled), both ring placements, conditioning frames
pushed in groups, dense feedback, per-row speakers, and an engine-5 stream called in turn.  A Philox stream is tied to
the module's float64 forward(); StreamDecoder equals decode_device; every misuse is refused without a device fault."""
import ctypes as C

import pytest
import torch

from conftest import GOLDEN_CASES
from helpers import GoldenCase
from oracle import wavenet_oracle as orc
from test_streaming import CFG5, assert_same, cfg_noise, inputs_for, irregular_split, max_dilation, model_of
from wavenet_vocoder_b200 import WaveNet
from wavenet_vocoder_b200 import _native as N
from wavenet_vocoder_b200.engine import SynthesisEngine

pytestmark = pytest.mark.gpu


def model7(monkeypatch, kw, sd=None, seed=0):
    """A model whose own handle runs engine 7 (so incremental_forward is the one-shot call on the stream's handle)."""
    monkeypatch.setenv("WN_ENGINE", "7")
    m = model_of(kw, sd, seed)
    assert m._get_engine().plan(1)["engine"] == 7
    return m


def one_shot(m, B, T, init, c, g, noise, seed, **kw):
    return m.incremental_forward(initial_input=init, c=c, g=g, T=T, noise=noise, seed=seed, return_params=True, **kw)


def chunked(m, kw, B, T, init, c, g, noise, seed, split=None, **skw):
    s = m.open_stream(B=B, g=g, initial_input=init, seed=seed, noise=noise, return_params=True, engine=7, **skw)
    assert s._s.eng.plan(B)["engine"] == 7
    ys, ps = [], []
    if kw.get("upsample_conditional_features", False):
        F, f = c.size(-1), 0
        for n in (1, 2, 3, 5, 1):           # frames in irregular groups, then the tail
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


@pytest.mark.parametrize("noise_kind", ["replay", "philox"])
@pytest.mark.parametrize("B", [1, 3, 5, 8])
@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_golden_cases_chunked_equal_one_shot(name, B, noise_kind, monkeypatch):
    """Tiles of 1, 4 (3 rows), 8 (5 rows) and 8."""
    gc = GoldenCase(name)
    m = model7(monkeypatch, gc.kw, gc.sd)
    T = 160
    gen = torch.Generator().manual_seed(B)
    init, c, g = inputs_for(m, gc.kw, B, T, gen)
    noise = {k: v.cuda() for k, v in orc.predraw_noise(gc.cfg, B, T, 5).items()} if noise_kind == "replay" else None
    seed = None if noise is not None else 1234 + B
    plan = m._get_engine().plan(B)
    assert plan["rings_in_smem"] == 1 and plan["poll_warps"] == 0
    assert_same(chunked(m, gc.kw, B, T, init, c, g, noise, seed), one_shot(m, B, T, init, c, g, noise, seed))


@pytest.mark.parametrize("noise_kind", ["replay", "philox"])
def test_chunks_of_one_sample_at_every_ring_phase(noise_kind, monkeypatch):
    """A chunk boundary after each of the first 2*maxdil+2 steps: every phase of every history ring is a launch's
    first and last step once, so any state a step leaves for the next that the stream does not carry shows here."""
    gc = GoldenCase("mol_cond")
    m = model7(monkeypatch, gc.kw, gc.sd)
    B, n1 = 5, 2 * max_dilation(gc.kw) + 2
    T = n1 + 37
    gen = torch.Generator().manual_seed(2)
    init, c, g = inputs_for(m, gc.kw, B, T, gen)
    noise = {k: v.cuda() for k, v in orc.predraw_noise(gc.cfg, B, T, 6).items()} if noise_kind == "replay" else None
    seed = None if noise is not None else 99
    split = [1] * n1 + [T - n1]
    assert_same(chunked(m, gc.kw, B, T, init, c, g, noise, seed, split), one_shot(m, B, T, init, c, g, noise, seed))


@pytest.mark.parametrize("B", [2, 8])
def test_rings_in_global_memory(B, monkeypatch):
    """Config 5's shape: its history rings live in global memory, which IS the stream state.  Boundaries fall on
    different phases of the 1024-step ring of the last dilation."""
    m = model7(monkeypatch, CFG5)
    assert m._get_engine().plan(B)["rings_in_smem"] == 0
    D = 2 * max_dilation(CFG5)
    T = 2 * D + 300
    split = [1, 7, 64, D + 1, 700, T - (1 + 7 + 64 + D + 1 + 700)]
    gen = torch.Generator().manual_seed(3)
    init, c, g = inputs_for(m, CFG5, B, T, gen)
    for noise, seed in ((cfg_noise(CFG5, B, T, 8), None), (None, 77)):
        assert_same(chunked(m, CFG5, B, T, init, c, g, noise, seed, split), one_shot(m, B, T, init, c, g, noise, seed))


def test_config2_width_frames_pushed_in_groups(monkeypatch):
    """Config 2's widths (512 residual and gate channels, 24 layers, 80 conditioning channels) at B = 8, conditioning
    frames pushed in irregular groups and upsampled on the device, then finish()."""
    from test_gpu_parity import FULL
    kw = dict(FULL["cfg2_mol24"]["kw"], upsample_conditional_features=True, upsample_net="ConvInUpsampleNetwork",
              cin_pad=2, upsample_params={"upsample_scales": [4, 4, 4, 4], "cin_channels": 80, "cin_pad": 2})
    m = model7(monkeypatch, kw)
    eng = m._get_engine()
    assert m._native_upsample
    B, F = 8, 4 + 6
    gen = torch.Generator().manual_seed(4)
    frames = torch.randn(B, 80, F, generator=gen).cuda()
    T = eng.upsampled_length(F)
    ref = m.incremental_forward(c=frames, T=T, seed=11, return_params=True)
    s = m.open_stream(B=B, seed=11, return_params=True, engine=7)
    ys, ps, f = [], [], 0
    for n in (1, 3, 1, 2, 3):
        y, p = s.push_frames(frames[:, :, f:f + n])
        ys.append(y), ps.append(p)
        f += n
    assert f == F
    y, p = s.finish()
    ys.append(y), ps.append(p)
    assert sum(y.size(-1) for y in ys) == T
    assert_same((torch.cat(ys, -1), torch.cat(ps, -1)), ref)


def test_softmax_dense_feedback_and_dense_initial_input(monkeypatch):
    gc = GoldenCase("mulaw_softmax")
    m = model7(monkeypatch, gc.kw, gc.sd)
    B, T, O = 5, 150, gc.kw["out_channels"]
    gen = torch.Generator().manual_seed(5)
    init = torch.zeros(B, O, 1)
    init[:, 127] = 1.0
    dense = torch.softmax(torch.randn(B, O, 1, generator=gen), 1)
    noise = {k: v.cuda() for k, v in orc.predraw_noise(gc.cfg, B, T, 7).items()}
    split = irregular_split(T, max_dilation(gc.kw))
    # dense feedback (quantize=False): the fed-back vector is the whole softmax
    assert_same(chunked(m, gc.kw, B, T, init, None, None, None, 1, split, quantize=False),
                one_shot(m, B, T, init, None, None, None, 1, quantize=False))
    # a dense initial input (not one-hot), sampled classes after it
    assert_same(chunked(m, gc.kw, B, T, dense, None, None, noise, None, split),
                one_shot(m, B, T, dense, None, None, noise, None))


def test_gaussian_head_with_per_row_speakers(monkeypatch):
    """Config 3's shape: Gaussian head, speaker embedding, one speaker id per row."""
    from test_gpu_parity import FULL
    kw = FULL["cfg3_gauss_spk"]["kw"]
    m = model7(monkeypatch, kw)
    B, T = 8, 200
    gen = torch.Generator().manual_seed(6)
    c = torch.randn(B, kw["cin_channels"], T, generator=gen)
    g = torch.tensor([[0], [3], [5], [15], [3], [9], [1], [12]])
    init = torch.rand(B, 1, 1, generator=gen) * 0.2 - 0.1
    for noise, seed in (({"z": torch.randn(T, B, generator=gen).cuda()}, None), (None, 31)):
        assert_same(chunked(m, kw, B, T, init, c, g, noise, seed), one_shot(m, B, T, init, c, g, noise, seed))


def test_engine5_and_engine7_streams_called_in_turn():
    """One model (its handle runs engine 5): an engine-5 stream of 4 and an engine-7 stream of 8 (on the engine-7
    handle made for it) called alternately; each equals its own handle's one-shot call."""
    gc = GoldenCase("mol_cond")
    m = model_of(gc.kw, gc.sd)
    eng = m._get_engine()
    assert eng.plan(1)["engine"] == 5
    T = 200
    gen = torch.Generator().manual_seed(7)
    c5, c7 = torch.randn(4, 8, T, generator=gen).cuda(), torch.randn(8, 8, T, generator=gen).cuda()
    s5, s7 = m.open_stream(B=4, seed=1), m.open_stream(B=8, seed=2, engine=7)
    sib = eng.engine7()
    assert s7._s.eng is sib and sib.plan(8)["engine"] == 7 and sib.plan(8)["batch_tile"] == 8
    o5, o7, t5, t7 = [], [], 0, 0
    for n5, n7 in ((5, 17), (40, 3), (64, 90), (91, 90)):
        o5.append(s5.generate(n5, c=c5[:, :, t5:t5 + n5]))
        o7.append(s7.generate(n7, c=c7[:, :, t7:t7 + n7]))
        t5, t7 = t5 + n5, t7 + n7
    assert t5 == T and t7 == T
    assert torch.equal(torch.cat(o5, -1), m.incremental_forward(c=c5, T=T, seed=1))
    ref7, _ = sib.generate(B=8, T=T, c=c7.transpose(1, 2).contiguous(), seed=2)
    assert torch.equal(torch.cat(o7, -1), ref7.view(8, 1, T))
    s5.close(), s7.close()


def test_philox_stream_against_float64_forward():
    """Independent of engine 7's own one-shot call: the head outputs of a Philox stream of 8 rows against the
    module's float64 forward() teacher-forced on the stream's own waveform."""
    gc = GoldenCase("mol_cond")
    m = model_of(gc.kw, gc.sd)
    B, T = 8, 300
    gen = torch.Generator().manual_seed(8)
    init, c, g = inputs_for(m, gc.kw, B, T, gen)
    y, p = chunked(m, gc.kw, B, T, init, c, g, None, 4321)
    torch.manual_seed(0)
    m64 = WaveNet(**gc.kw)
    m64.load_state_dict(gc.sd)
    m64 = m64.double().eval()
    x = torch.cat([init.double(), y.cpu().double()[:, :, :-1]], dim=2)
    with torch.no_grad():
        ref = m64(x, c=c.double(), softmax=False)
    err = float((p.cpu().double() - ref).abs().max())
    print("engine-7 stream B=8 head outputs vs float64 forward(): max abs %.3g" % err)
    assert err <= 2e-5, err


def test_stream_decoder_over_engine7_stream():
    from wavenet_vocoder_b200.dispatch import StreamDecoder, decode_device
    gc = GoldenCase("mol_cond")
    m = model_of(gc.kw, gc.sd)
    B, T = 8, 400
    gen = torch.Generator().manual_seed(9)
    c = torch.randn(B, 8, T, generator=gen).cuda()
    kw = dict(input_type="mulaw", quantize_channels=256, postprocess="inv_preemphasis", global_gain_scale=0.9,
              preemphasis_coef=0.85)
    lengths = [T, T - 170, 5, 399, 200, T, 1, 300]
    s = m.open_stream(B=B, seed=5, engine=7)
    dec = StreamDecoder(B, "cuda", lengths=lengths, want_float=True, **kw)
    ys, parts, t = [], [], 0
    for n in (1, 100, 63, 200, 36):
        y = s.generate(n, c=c[:, :, t:t + n])
        ys.append(y)
        parts.append(dec(y))
        t += n
    s.close()
    ref, _ = m._get_engine().engine7().generate(B=B, T=T, c=c.transpose(1, 2).contiguous(), seed=5)
    assert torch.equal(torch.cat(ys, -1), ref.view(B, 1, T))
    pcm, flt = decode_device(ref.view(B, 1, T), lengths, want_float=True, **kw)
    assert torch.equal(torch.cat([q[0] for q in parts], -1), pcm)
    assert torch.equal(torch.cat([q[1] for q in parts], -1), flt)


def test_misuse_is_refused_and_nothing_faults():
    gc = GoldenCase("mol_cond")
    m = model_of(gc.kw, gc.sd)
    eng = m._get_engine()
    gen = torch.Generator().manual_seed(10)
    c = torch.randn(8, 8, 64, generator=gen).cuda()
    ct = c.transpose(1, 2).contiguous()
    with pytest.raises(N.WnError, match="1..8 utterances"):
        m.open_stream(B=9, seed=1, engine=7)
    with pytest.raises(N.WnError, match=r"wn_config\.engine = 7"):
        eng.open_stream(B=1, seed=1, engine=7)                  # an engine-7 stream on the engine-5 handle
    with pytest.raises(N.WnError, match="engine must be"):
        m.open_stream(B=1, seed=1, engine=6)
    ctor = dict(eng._ctor)
    with pytest.raises(N.WnError, match="engine must be"):
        SynthesisEngine(**dict(ctor, engine=3))
    # a handle with dedicated polling warps has no engine-7 stream kernel
    ep = SynthesisEngine(**dict(ctor, engine=7, poll_warps=4))
    assert ep.plan(1)["poll_warps"] == 4
    ep.load_state_dict(m.state_dict())
    with pytest.raises(N.WnError, match="compute warps poll"):
        ep.open_stream(B=1, seed=1, engine=7)
    ep.close()
    # teacher forcing through the C ABI
    s = m.open_stream(B=8, seed=1, engine=7)
    out, ts = torch.empty(8, 8, device="cuda"), torch.zeros(8, 2, device="cuda")
    a = N.wn_generate_args()
    a.B, a.T, a.c, a.out_scalar = 8, 8, ct.data_ptr(), out.data_ptr()
    a.T_test, a.test_scalar = 2, ts.data_ptr()
    assert N.lib().wn_stream_generate(s._s._s, C.byref(a), None) == -1
    assert b"teacher forcing" in N.lib().wn_last_error()
    # a chunk marked final, then one more
    y1, _ = s._s.generate(8, c=ct[:, :8], final=True)
    with pytest.raises(N.WnError, match="finalised"):
        s._s.generate(8, c=ct[:, 8:16])
    s.close()
    sib = eng.engine7()
    ref, _ = sib.generate(B=8, T=8, c=ct[:, :8].contiguous(), seed=1)
    assert torch.equal(y1, ref)
    # weights changed after the stream was opened
    s = m.open_stream(B=3, seed=3, engine=7)
    s.generate(4, c=c[:3, :, :4])
    with torch.no_grad():
        m.first_conv.bias.add_(0.01)
    with pytest.raises(N.WnError, match="weights changed"):
        s.generate(4, c=c[:3, :, 4:8])
    s.close()
    # after all of the above a fresh stream (on the reloaded engine-7 handle) equals its one-shot call
    s = m.open_stream(B=8, seed=12, engine=7)
    y = torch.cat([s.generate(n, c=c[:, :, t:t + n]) for t, n in ((0, 20), (20, 44))], -1)
    s.close()
    ref, _ = sib.generate(B=8, T=64, c=ct, seed=12)
    assert torch.equal(y, ref.view(8, 1, 64))
