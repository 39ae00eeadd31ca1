# coding: utf-8
"""Parity of the CUDA path (libwn.so through the WaveNet class surface / the C ABI) against
(a) the golden vectors written by the unmodified reference and (b) the CPU oracle on seeded
inputs.  Needs an H100; run with ``pytest -m gpu``.

Tolerances (fp32 path; BASELINE.json asks for <= 1e-4 RMS):
  head outputs ("distribution parameters"), teacher forced : max abs <= 2e-5 (observed ~1e-6)
  sampled waveform under replayed noise                     : RMS <= 1e-4
The reference's own criterion between its two code paths is 1e-4 abs (tests/test_model.py:362).
"""
import numpy as np
import pytest
import torch

from conftest import GOLDEN_CASES
from helpers import GoldenCase
from oracle import wavenet_oracle as orc

pytestmark = pytest.mark.gpu

PARAM_TOL = 2e-5
RMS_TOL = 1e-4


@pytest.fixture(params=[5, 7])
def engine(request, monkeypatch):
    """Both kernel organisations are parity-tested: 5 = the default (csrc/wn_kernel.cuh), 7 = the alternative
    (csrc/wn7_kernel.cuh).  The choice is read when the engine handle is created."""
    monkeypatch.setenv("WN_ENGINE", str(request.param))
    return request.param


def cuda_model(gc, **extra):
    from wavenet_vocoder_b200 import WaveNet
    kw = dict(gc.kw)
    kw.update(extra)
    m = WaveNet(**kw)
    m.load_state_dict(gc.sd)
    return m.cuda().eval()


def dev_noise(n):
    return {k: v.cuda() for k, v in n.items()}


TIE_MARGIN = 1e-4


def assert_class_ids_match(idx_got, logits_ref, e_noise, what=""):
    """Index work is bit-exact except at documented near-ties.  The sampled class of step t is
    argmax_i (p_i / sum p) / e_i  (OneHotCategorical, wavenet.py:334-335) with p = softmax(logits).  The kernel's
    logits differ from the reference's by ~1e-6 (summation order), so the winner can only change where the two
    largest ratios are within TIE_MARGIN (relative).  Assert: every step whose top-2 margin is >= TIE_MARGIN has
    the identical class id, and every differing step picked the reference's runner-up.
    idx_got (B,T) int; logits_ref (B,O,T); e_noise (T,B,O)."""
    p = torch.softmax(logits_ref.double(), dim=1)
    r = (p / p.sum(1, keepdim=True)) / e_noise.permute(1, 2, 0).double()          # (B,O,T)
    top = r.topk(2, dim=1)
    margin = (top.values[:, 0] - top.values[:, 1]) / top.values[:, 0]              # (B,T)
    ref_idx = top.indices[:, 0]
    diff = idx_got.long() != ref_idx
    clear = margin >= TIE_MARGIN
    assert not bool((diff & clear).any()), "%s: %d class ids differ at steps with a clear margin (min margin there %.3g)" % (
        what, int((diff & clear).sum()), float(margin[diff & clear].min()))
    assert bool((idx_got.long()[diff] == top.indices[:, 1][diff]).all()), what + ": a near-tie resolved to a third class"
    return int(diff.sum()), float(margin.min())


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_golden_teacher_forced(name, engine):
    gc = GoldenCase(name)
    m = cuda_model(gc)
    g = gc.t("g_ids")
    y, params = m.incremental_forward(test_inputs=gc.x_tf, c=gc.t("c_raw"), g=g, T=gc.T,
                                      noise=dev_noise(gc.noise_tf), return_params=True)
    ref = gc.t("params_tf")
    err = float((params.cpu() - ref).abs().max())
    assert params.shape == ref.shape
    assert err <= PARAM_TOL, err
    if gc.cfg.scalar_input:
        assert y.shape == (gc.B, 1, gc.T)
        assert float((y.cpu() - gc.t("y_tf")).abs().max()) <= 1e-4
    else:
        assert y.shape == (gc.B, gc.cfg.out_channels, gc.T)
        assert float(y.sum(1).min()) == 1.0 and float(y.sum(1).max()) == 1.0          # one-hot
        ndiff, _ = assert_class_ids_match(y.argmax(1).cpu(), ref, gc.noise_tf["e"], name)
        assert (y.argmax(1).cpu() != gc.t("y_tf").long()).sum().item() == ndiff       # the fixture agrees with the rule


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_golden_free_running_replayed_noise(name, engine):
    gc = GoldenCase(name)
    m = cuda_model(gc)
    g = gc.t("g_ids")
    y = m.incremental_forward(c=gc.t("c_raw"), g=g, T=gc.T, noise=dev_noise(gc.noise))
    ref = gc.t("y_free")
    if gc.cfg.scalar_input:
        assert y.shape == ref.shape
        rms = float(((y.cpu() - ref) ** 2).mean().sqrt())
        assert rms <= RMS_TOL, rms
    else:
        # free running: every step is checked on the kernel's OWN trajectory (teacher-force it into the oracle), so
        # one near-tie cannot hide later mismatches; and up to the first divergence the fixture must agree exactly
        got = y.argmax(1).cpu()
        first = torch.zeros(gc.B_free, gc.cfg.out_channels, 1)
        first[:, 127] = 1
        ti = torch.cat([first, y.cpu()[:, :, :-1]], dim=2)
        rec = []
        orc.incremental_forward(gc.cfg, gc.w, test_inputs=ti, T=gc.T, softmax=False, quantize=False, params_out=rec)
        ndiff, _ = assert_class_ids_match(got, torch.stack(rec, -1), gc.noise["e"], name + " (free running)")
        same = (got == ref.long())
        if ndiff == 0:
            assert bool(same.all())


def test_make_generation_fast_gives_same_result():
    gc = GoldenCase("mol_cond")
    m = cuda_model(gc)
    y1 = m.incremental_forward(c=gc.t("c_raw"), T=gc.T, noise=dev_noise(gc.noise))
    m.make_generation_fast_()
    assert "first_conv.weight" in m.state_dict()
    y2 = m.incremental_forward(c=gc.t("c_raw"), T=gc.T, noise=dev_noise(gc.noise))
    assert float((y1 - y2).abs().max()) <= 1e-5


@pytest.mark.parametrize("P", [4, 5, 8, 32])
def test_any_block_count_gives_same_head_outputs(P, engine):
    """The row partition must not change the result beyond fp32 reassociation."""
    from wavenet_vocoder_b200.engine import SynthesisEngine
    gc = GoldenCase("mol_cond")
    kw = gc.kw
    eng = SynthesisEngine(layers=kw["layers"], stacks=kw["stacks"], residual_channels=kw["residual_channels"],
                          gate_channels=kw["gate_channels"], skip_out_channels=kw["skip_out_channels"],
                          out_channels=kw["out_channels"], kernel_size=3, cin_channels=kw["cin_channels"],
                          gin_channels=-1, scalar_input=True, output_distribution="Logistic",
                          device=torch.device("cuda", 0), num_ctas=P)
    eng.load_state_dict(gc.sd)
    assert eng.plan(gc.B)["num_ctas"] == P
    c = gc.t("c_up").transpose(1, 2).contiguous()
    out, params = eng.generate(B=gc.B, T=gc.T, c=c, test_scalar=gc.x_tf.view(gc.B, gc.T),
                               noise=dev_noise(gc.noise_tf), want_params=True)
    assert float((params.cpu() - gc.t("params_tf")).abs().max()) <= PARAM_TOL
    eng.close()


@pytest.mark.parametrize("B", [1, 2, 3, 5, 8, 11])
def test_batch_tiles_and_chunks(B, engine):
    """Batch tiles 1/2/4/8 with padding rows, and B > 8 split into sequential launches: every
    utterance must equal what the oracle gives for it alone."""
    gc = GoldenCase("mol_cond")
    m = cuda_model(gc)
    T = 40
    gen = torch.Generator().manual_seed(B)
    c = torch.randn(B, gc.cfg.cin_channels, T, generator=gen)
    x = (torch.rand(B, 1, T, generator=gen) * 2 - 1) * 0.7
    noise = orc.predraw_noise(gc.cfg, B, T, 100 + B)
    y, params = m.incremental_forward(test_inputs=x, c=c, T=T, noise=dev_noise(noise), return_params=True)
    rec = []
    y_ref = orc.incremental_forward(gc.cfg, gc.w, test_inputs=x, c=c, T=T,
                                    noise=orc.replay_from_predrawn(gc.cfg, noise), params_out=rec)
    p_ref = torch.stack(rec, dim=-1)
    assert float((params.cpu() - p_ref).abs().max()) <= PARAM_TOL
    assert float((y.cpu() - y_ref).abs().max()) <= 1e-4
    # free running, same noise
    y2 = m.incremental_forward(c=c, T=T, noise=dev_noise(noise))
    y2_ref = orc.incremental_forward(gc.cfg, gc.w, c=c, T=T, noise=orc.replay_from_predrawn(gc.cfg, noise))
    assert float(((y2.cpu() - y2_ref) ** 2).mean().sqrt()) <= RMS_TOL


def test_teacher_forcing_prefix_then_free_running():
    """test_inputs shorter than T: forced for T' steps, then feeds back its own samples
    (wavenet.py:297-301)."""
    gc = GoldenCase("mixgauss")
    m = cuda_model(gc)
    T, Tp, B = 48, 17, 2
    gen = torch.Generator().manual_seed(5)
    x = (torch.rand(B, 1, Tp, generator=gen) * 2 - 1) * 0.5
    noise = orc.predraw_noise(gc.cfg, B, T, 77)
    y = m.incremental_forward(test_inputs=x, T=T, noise=dev_noise(noise))
    y_ref = orc.incremental_forward(gc.cfg, gc.w, test_inputs=x, T=T,
                                    noise=orc.replay_from_predrawn(gc.cfg, noise))
    assert y.shape == (B, 1, T)
    assert float(((y.cpu() - y_ref) ** 2).mean().sqrt()) <= RMS_TOL


def test_softmax_head_modes():
    gc = GoldenCase("mulaw_softmax")
    m = cuda_model(gc)
    # quantize=False returns probabilities / logits for every step (tests/test_model.py:352-355 in the reference)
    p = m.incremental_forward(test_inputs=gc.x_tf, T=gc.T, softmax=False, quantize=False)
    assert float((p.cpu() - gc.t("params_tf")).abs().max()) <= PARAM_TOL
    q = m.incremental_forward(test_inputs=gc.x_tf, T=gc.T, softmax=True, quantize=False)
    ref = torch.softmax(gc.t("params_tf"), dim=1)
    assert float((q.cpu() - ref).abs().max()) <= 1e-5
    # dense (non one-hot) teacher forcing rows go through the full first-conv GEMV
    soft = 0.9 * gc.x_tf + 0.1 / gc.cfg.out_channels
    rec = []
    orc.incremental_forward(gc.cfg, gc.w, test_inputs=soft, T=gc.T, softmax=False, quantize=False, params_out=rec)
    d = m.incremental_forward(test_inputs=soft, T=gc.T, softmax=False, quantize=False)
    assert float((d.cpu() - torch.stack(rec, -1)).abs().max()) <= PARAM_TOL
    # free running with probabilities fed back (quantize=False)
    f = m.incremental_forward(T=24, softmax=True, quantize=False)
    f_ref = orc.incremental_forward(gc.cfg, gc.w, T=24, softmax=True, quantize=False)
    assert float((f.cpu() - f_ref).abs().max()) <= 1e-5
    with pytest.raises(RuntimeError):
        m.incremental_forward(T=4, softmax=False, quantize=True)


def test_error_behaviour_matches_reference():
    gc = GoldenCase("mol_cond")
    m = cuda_model(gc)
    m.train()
    with pytest.raises(RuntimeError, match="eval mode"):          # conv.py:19-20
        m.incremental_forward(c=gc.t("c_raw"), T=gc.T)
    m.eval()
    with pytest.raises(RuntimeError):                             # local conditioning missing
        m.incremental_forward(T=8)
    with pytest.raises(AssertionError):                           # wavenet.py:276  c.size(-1) == T
        m2 = cuda_model(GoldenCase("mol_upsample"))
        m2.incremental_forward(c=GoldenCase("mol_upsample").t("c_raw"), T=7)


def test_philox_sampling_is_seed_reproducible_and_self_consistent():
    """Device RNG: same torch seed -> same waveform; feeding the waveform back as teacher-forcing
    input with the same seed must reproduce it bit for bit (each step sees identical inputs)."""
    gc = GoldenCase("mol_cond")
    m = cuda_model(gc)
    c = gc.t("c_raw")
    torch.manual_seed(11)
    y1 = m.incremental_forward(c=c, T=gc.T)
    torch.manual_seed(11)
    y2 = m.incremental_forward(c=c, T=gc.T)
    torch.manual_seed(12)
    y3 = m.incremental_forward(c=c, T=gc.T)
    assert torch.equal(y1, y2) and not torch.equal(y1, y3)
    assert float(y1.abs().max()) <= 1.0 and float(y1.std()) > 1e-3
    ti = torch.cat([torch.zeros(gc.B, 1, 1, device="cuda"), y1[:, :, :-1]], dim=2)
    y4 = m.incremental_forward(test_inputs=ti, c=c, T=gc.T, seed=0)
    torch.manual_seed(11)
    y5 = m.incremental_forward(test_inputs=ti, c=c, T=gc.T)
    assert torch.equal(y5, y1)
    assert y4.shape == y1.shape


def check_standalone_samplers(K, B, T):
    """The stand-alone MoL and Gaussian samplers on seeded (B, 3K, T) head outputs, and the single Gaussian on the
    first two channels, against the oracle's samplers on the same replayed noise."""
    from wavenet_vocoder_b200.mixture import sample_from_discretized_mix_logistic, sample_from_mix_gaussian
    gen = torch.Generator().manual_seed(3)
    y = torch.randn(B, 3 * K, T, generator=gen)
    y[:, 2 * K:] -= 2.0
    u1 = torch.empty(T, B, K).uniform_(1e-5, 1 - 1e-5, generator=gen)
    u2 = torch.empty(T, B).uniform_(1e-5, 1 - 1e-5, generator=gen)
    z = torch.randn(T, B, generator=gen)
    got = sample_from_discretized_mix_logistic(y.cuda(), noise={"u1": u1, "u2": u2}).cpu()
    # a single Gaussian of 3 channels draws no mixture indicator: the wrapper passes no u1
    got_g = sample_from_mix_gaussian(y.cuda(), noise={"u1": u1, "z": z} if K > 1 else {"z": z}).cpu()
    got_1 = sample_from_mix_gaussian(y[:, :2].contiguous().cuda(), noise={"z": z}).cpu()
    assert got.shape == got_g.shape == got_1.shape == (B, T)
    for t in range(T):
        yt = y[:, :, t].unsqueeze(1)
        ref = orc.sample_mol(yt, orc.ReplayNoise(uniform=[u1[t].unsqueeze(1), u2[t].unsqueeze(1)]))
        assert float((got[:, t:t + 1] - ref).abs().max()) <= 1e-5
        ref_g = orc.sample_gaussian(yt, orc.ReplayNoise(uniform=[u1[t].unsqueeze(1)] if K > 1 else [],
                                                        normal=[z[t].unsqueeze(1)]))
        assert float((got_g[:, t:t + 1] - ref_g).abs().max()) <= 1e-5
        ref_1 = orc.sample_gaussian(yt[:, :, :2], orc.ReplayNoise(normal=[z[t].unsqueeze(1)]))
        assert float((got_1[:, t:t + 1] - ref_1).abs().max()) <= 1e-5


def test_standalone_samplers_match_oracle():
    check_standalone_samplers(10, 3, 50)


# K = 1: a one-component MoL and the C == 3 Gaussian (mean y[1], log-scale y[2]); B x T = 771 leaves the last
# 256-thread block of the sampler kernel ragged
@pytest.mark.parametrize("K,B,T", [(1, 3, 50), (10, 3, 257), (1, 3, 257)])
def test_standalone_samplers_at_more_widths_match_oracle(K, B, T):
    check_standalone_samplers(K, B, T)


# ------------------------------------------------------------------------------------------------
# BASELINE.json configurations at full width, short T (the oracle needs ~6 ms per step)
# ------------------------------------------------------------------------------------------------
FULL = {
    "cfg1_mulaw256": dict(kw=dict(out_channels=256, layers=12, stacks=2, residual_channels=64, gate_channels=128,
                                  skip_out_channels=64, cin_channels=-1, gin_channels=-1, scalar_input=False,
                                  dropout=0.0), T=96),
    "cfg2_mol24": dict(kw=dict(out_channels=30, layers=24, stacks=4, residual_channels=512, gate_channels=512,
                               skip_out_channels=256, cin_channels=80, gin_channels=-1, scalar_input=True,
                               output_distribution="Logistic", dropout=0.0), T=96),
    "cfg3_gauss_spk": dict(kw=dict(out_channels=2, layers=24, stacks=4, residual_channels=128, gate_channels=256,
                                   skip_out_channels=128, cin_channels=80, gin_channels=16, n_speakers=16,
                                   use_speaker_embedding=True, scalar_input=True, output_distribution="Normal",
                                   dropout=0.0), T=96),
    "cfg5_mol30": dict(kw=dict(out_channels=30, layers=30, stacks=3, residual_channels=256, gate_channels=512,
                               skip_out_channels=256, cin_channels=80, gin_channels=-1, scalar_input=True,
                               output_distribution="Logistic", dropout=0.0), T=1100),
}


def full_case(name, seed=0):
    from wavenet_vocoder_b200 import WaveNet
    spec = FULL[name]
    kw = spec["kw"]
    torch.manual_seed(seed)
    m = WaveNet(**kw).eval()
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if n_.endswith(".bias"):
                p.normal_(0, 0.05)
        if kw["scalar_input"]:
            O = kw["out_channels"]
            b = m.last_conv_layers[3].bias
            if O == 2:
                b[1] -= 3.0
            else:
                b[2 * (O // 3):] -= 3.0
    cfg = orc.PathConfig(out_channels=kw["out_channels"], layers=kw["layers"], stacks=kw["stacks"],
                         residual_channels=kw["residual_channels"], gate_channels=kw["gate_channels"],
                         skip_out_channels=kw["skip_out_channels"], kernel_size=3,
                         cin_channels=kw["cin_channels"], gin_channels=kw["gin_channels"],
                         scalar_input=kw["scalar_input"], output_distribution=kw.get("output_distribution", "Logistic"))
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    w = orc.weights_from_state_dict(cfg, sd)
    return m, cfg, w, spec["T"]


@pytest.mark.parametrize("name", list(FULL))
def test_full_width_configs_against_oracle(name, engine):
    m, cfg, w, T = full_case(name)
    B = 1
    gen = torch.Generator().manual_seed(1)
    c = torch.randn(B, cfg.cin_channels, T, generator=gen) if cfg.cin_channels > 0 else None
    g_ids = torch.tensor([[5]]) if cfg.gin_channels > 0 else None
    g_vec = orc.embed_speaker(w, g_ids) if g_ids is not None else None
    noise = orc.predraw_noise(cfg, B, T, 9)
    rec = []
    with torch.no_grad():
        y_ref = orc.incremental_forward(cfg, w, c=c, g=g_vec, T=T, noise=orc.replay_from_predrawn(cfg, noise),
                                        params_out=rec)
    p_ref = torch.stack(rec, dim=-1)
    mc = m.cuda()
    # teacher forced on the oracle's own trajectory: per-step parity without error feedback
    if cfg.scalar_input:
        ti = torch.cat([torch.zeros(B, 1, 1), y_ref[:, :, :-1]], dim=2)
    else:
        first = torch.zeros(B, cfg.out_channels, 1)
        first[:, 127] = 1
        ti = torch.cat([first, y_ref[:, :, :-1]], dim=2)
    y_tf, params = mc.incremental_forward(test_inputs=ti, c=c, g=g_ids, T=T, noise=dev_noise(noise),
                                          return_params=True)
    perr = float((params.cpu() - p_ref).abs().max())
    assert perr <= 1e-4, perr
    # free running with the same noise
    y = mc.incremental_forward(c=c, g=g_ids, T=T, noise=dev_noise(noise))
    if cfg.scalar_input:
        assert float((y_tf.cpu() - y_ref).abs().max()) <= 2e-4
        rms = float(((y.cpu() - y_ref) ** 2).mean().sqrt())
        assert rms <= RMS_TOL, rms
    else:
        assert_class_ids_match(y_tf.argmax(1).cpu(), p_ref, noise["e"], name)
        first = torch.zeros(B, cfg.out_channels, 1)
        first[:, 127] = 1
        ti2 = torch.cat([first, y.cpu()[:, :, :-1]], dim=2)
        rec2 = []
        with torch.no_grad():
            orc.incremental_forward(cfg, w, test_inputs=ti2, T=T, softmax=False, quantize=False, params_out=rec2)
        assert_class_ids_match(y.argmax(1).cpu(), torch.stack(rec2, -1), noise["e"], name + " (free running)")
    print("%s: head-output max abs err %.3g" % (name, perr))


def test_config2_full_length_properties():
    """BASELINE config 2 at its full T=22050 (too long for the oracle): size-independent checks.
    (1) all samples finite and inside [-1,1]; (2) replaying the generated waveform as teacher
    forcing input with the same device seed reproduces it bit for bit; (3) two utterances run as
    a batch equal the same utterances run alone."""
    m, cfg, w, _ = full_case("cfg2_mol24")
    mc = m.cuda()
    T = 22050
    gen = torch.Generator().manual_seed(2)
    c = torch.randn(2, 80, T, generator=gen).cuda()
    y = mc.incremental_forward(c=c[:1], T=T, seed=1234)
    assert y.shape == (1, 1, T)
    assert bool(torch.isfinite(y).all()) and float(y.abs().max()) <= 1.0 and float(y.std()) > 1e-3
    ti = torch.cat([torch.zeros(1, 1, 1, device="cuda"), y[:, :, :-1]], dim=2)
    y_rep = mc.incremental_forward(test_inputs=ti, c=c[:1], T=T, seed=1234)
    assert torch.equal(y_rep, y)
    Ts = 4000
    yb = mc.incremental_forward(c=c[:, :, :Ts], T=Ts, seed=77)
    # philox streams are keyed by (seed, step, utterance index): row 0 alone must match row 0 of the batch
    y0 = mc.incremental_forward(c=c[:1, :, :Ts], T=Ts, seed=77)
    assert float((yb[:1] - y0).abs().max()) <= 1e-4


def test_c_abi_host_buffer_entry():
    """wn_generate_host: the same call with HOST buffers everywhere (copies inside, synchronous).
    Driven through ctypes exactly as INTEGRATION.md shows; checked against the golden vectors."""
    import ctypes as C
    from wavenet_vocoder_b200 import _native as N
    from wavenet_vocoder_b200.engine import make_config, weights_struct
    gc = GoldenCase("mol_cond")
    kw = gc.kw
    cfg = make_config(layers=kw["layers"], stacks=kw["stacks"], residual_channels=kw["residual_channels"],
                      gate_channels=kw["gate_channels"], skip_out_channels=kw["skip_out_channels"],
                      out_channels=kw["out_channels"], kernel_size=3, cin_channels=kw["cin_channels"],
                      gin_channels=-1, scalar_input=True, output_distribution="Logistic", device_index=0)
    h = C.c_void_p()
    N.check(N.lib().wn_create(C.byref(cfg), C.byref(h)))
    try:
        w, keep = weights_struct(gc.sd, cfg.layers, cfg.cin_channels, 0)
        N.check(N.lib().wn_load_weights(h, C.byref(w)))
        B, T, K = gc.B, gc.T, kw["out_channels"] // 3
        c = np.ascontiguousarray(gc.arr["c_up"].transpose(0, 2, 1)).astype(np.float32)       # (B,T,C)
        x_tf = np.ascontiguousarray(gc.arr["x_tf"].reshape(B, T)).astype(np.float32)
        u1 = np.ascontiguousarray(gc.noise_tf["u1"].numpy())
        u2 = np.ascontiguousarray(gc.noise_tf["u2"].numpy())
        out = np.zeros((B, T), np.float32)
        params = np.zeros((B, kw["out_channels"], T), np.float32)
        a = N.wn_generate_args()
        a.B, a.T, a.T_test = B, T, T
        a.c = c.ctypes.data
        a.test_scalar = x_tf.ctypes.data
        a.flags = N.WN_FLAG_SOFTMAX | N.WN_FLAG_QUANTIZE
        a.noise_kind = N.WN_NOISE_REPLAY
        a.noise_u1, a.noise_u2 = u1.ctypes.data, u2.ctypes.data
        a.out_scalar, a.params_out = out.ctypes.data, params.ctypes.data
        N.check(N.lib().wn_generate_host(h, C.byref(a)))
        assert float(np.abs(params - gc.arr["params_tf"]).max()) <= PARAM_TOL
        assert float(np.abs(out - gc.arr["y_tf"].reshape(B, T)).max()) <= 1e-4
        # argument errors come back as status codes with a message, not crashes
        a.c = None
        assert N.lib().wn_generate_host(h, C.byref(a)) == -1
        assert b"c is required" in N.lib().wn_last_error()
        info = N.wn_plan_info()
        N.check(N.lib().wn_get_plan(h, 1, C.byref(info)))
        assert info.launches >= 1 and info.exchanges_per_step == cfg.layers + 3
    finally:
        N.lib().wn_destroy(h)


# ------------------------------------------------------------------------------------------------
# The reference's own online == offline tests (tests/test_model.py:147-366 there: teacher-forced
# incremental_forward vs the batch forward(), atol 1e-4, warn-only) restated with synthetic inputs and
# a hard assert.  The batch side runs on a CPU copy of the module (plain fp32 PyTorch).
# ------------------------------------------------------------------------------------------------
ONLINE_OFFLINE = {
    "incremental_forward_correctness": dict(kw=dict(out_channels=256, layers=4, stacks=2, residual_channels=32,
                                                    gate_channels=32, skip_out_channels=32, scalar_input=False)),
    "local_conditioning": dict(kw=dict(out_channels=256, layers=4, stacks=2, residual_channels=32, gate_channels=32,
                                       skip_out_channels=32, cin_channels=2, scalar_input=False), c="sample"),
    "local_conditioning_upsample": dict(kw=dict(out_channels=256, layers=4, stacks=2, residual_channels=32,
                                                gate_channels=32, skip_out_channels=32, cin_channels=2,
                                                scalar_input=False, upsample_conditional_features=True,
                                                upsample_params={"upsample_scales": [2, 2], "cin_channels": 2}),
                                        c="frames"),
    "global_conditioning_with_embedding": dict(kw=dict(out_channels=256, layers=4, stacks=2, residual_channels=32,
                                                       gate_channels=32, skip_out_channels=32, gin_channels=16,
                                                       n_speakers=4, use_speaker_embedding=True, scalar_input=False),
                                               g="ids"),
    "global_conditioning_without_embedding": dict(kw=dict(out_channels=256, layers=4, stacks=2, residual_channels=32,
                                                          gate_channels=32, skip_out_channels=32, gin_channels=16,
                                                          use_speaker_embedding=False, scalar_input=False), g="vec"),
    "global_and_local_conditioning": dict(kw=dict(out_channels=256, layers=4, stacks=2, residual_channels=32,
                                                  gate_channels=32, skip_out_channels=32, cin_channels=2, gin_channels=16,
                                                  n_speakers=4, use_speaker_embedding=True, scalar_input=False),
                                          c="sample", g="ids"),
    "mixture_wavenet": dict(kw=dict(out_channels=30, layers=4, stacks=2, residual_channels=32, gate_channels=32,
                                    skip_out_channels=32, cin_channels=1, scalar_input=True), c="sample"),
}


@pytest.mark.parametrize("name", list(ONLINE_OFFLINE))
def test_online_equals_offline_like_the_reference(name):
    import copy
    from wavenet_vocoder_b200 import WaveNet
    spec = ONLINE_OFFLINE[name]
    kw = dict(spec["kw"], dropout=0.0)
    torch.manual_seed(3)
    cpu = WaveNet(**kw).eval()
    with torch.no_grad():
        for n_, p_ in cpu.named_parameters():
            if n_.endswith(".bias"):
                p_.normal_(0, 0.05)
    B, T = 2, 64
    gen = torch.Generator().manual_seed(8)
    if kw["scalar_input"]:
        x = (torch.rand(B, 1, T, generator=gen) * 2 - 1) * 0.9
    else:
        idx = torch.randint(0, 256, (B, T), generator=gen)
        x = torch.zeros(B, 256, T).scatter_(1, idx.unsqueeze(1), 1.0)
    c = g = None
    if spec.get("c") == "sample":
        c = torch.randn(B, kw["cin_channels"], T, generator=gen)
    elif spec.get("c") == "frames":
        c = torch.randn(B, kw["cin_channels"], T // 4, generator=gen)
    if spec.get("g") == "ids":
        g = torch.randint(0, kw["n_speakers"], (B, 1), generator=gen)
    elif spec.get("g") == "vec":
        g = torch.randn(B, kw["gin_channels"], 1, generator=gen)
    with torch.no_grad():
        y_offline = cpu(x, c=c, g=g, softmax=False)                               # batch forward
    gpu = copy.deepcopy(cpu).cuda()
    if kw["scalar_input"]:
        y, y_online = gpu.incremental_forward(test_inputs=x, c=c, g=g, T=T, return_params=True)
        assert y.shape == x.shape                                                 # tests/test_model.py:138,143
        y_free = gpu.incremental_forward(c=c, g=g, T=T)
        assert y_free.shape == x.shape
    else:
        y_online = gpu.incremental_forward(test_inputs=x, c=c, g=g, T=T, softmax=False, quantize=False)
    assert y_online.shape == y_offline.shape
    assert float((y_online.cpu() - y_offline).abs().max()) <= 1e-4                # the reference's own tolerance


def test_initial_input_like_eval_model(engine):
    """train.eval_model / synthesis.wavegen hand an explicit initial_input: (B,1,1) for scalar models,
    one-hot (B,1,Q) or (B,Q,1) for mu-law models (train.py:589-602 in the reference)."""
    gc = GoldenCase("mixgauss")
    m = cuda_model(gc)
    T, B = 40, 2
    noise = orc.predraw_noise(gc.cfg, B, T, 5)
    init = torch.tensor([[[0.3]], [[-0.6]]])                                       # (B,1,1)
    y = m.incremental_forward(initial_input=init, T=T, noise=dev_noise(noise))
    assert y.shape == (B, 1, T)
    for r in range(B):                                                             # each row against the oracle alone
        nr = {k: v[:, r:r + 1].contiguous() for k, v in noise.items()}
        y_ref = orc.incremental_forward(gc.cfg, gc.w, initial_input=init[r:r + 1], T=T,
                                        noise=orc.replay_from_predrawn(gc.cfg, nr))
        assert float(((y[r:r + 1].cpu() - y_ref) ** 2).mean().sqrt()) <= RMS_TOL
    # test_inputs override step 0 (wavenet.py:299-301): initial_input is then unused, whatever its shape
    n3 = orc.predraw_noise(gc.cfg, 3, 8, 6)
    ya = m.incremental_forward(initial_input=init, test_inputs=torch.zeros(3, 1, 4), T=8, noise=dev_noise(n3))
    yb = m.incremental_forward(test_inputs=torch.zeros(3, 1, 4), T=8, noise=dev_noise(n3))
    assert torch.equal(ya, yb)
    with pytest.raises(ValueError):
        m.incremental_forward(initial_input=torch.zeros(3, 1, 1), g=None, c=None, T=8,
                              noise=dev_noise(orc.predraw_noise(gc.cfg, 2, 8, 6)))
    gq = GoldenCase("mulaw_softmax")
    mq = cuda_model(gq)
    Q = gq.cfg.out_channels
    for layout in ("b1q", "bq1"):
        oh = torch.zeros(1, 1, Q)
        oh[:, :, 200] = 1
        init_q = oh if layout == "b1q" else oh.transpose(1, 2).contiguous()
        nz = orc.predraw_noise(gq.cfg, 1, 32, 6)
        yq = mq.incremental_forward(initial_input=init_q, T=32, noise=dev_noise(nz))
        yq_ref = orc.incremental_forward(gq.cfg, gq.w, initial_input=init_q, T=32,
                                         noise=orc.replay_from_predrawn(gq.cfg, nz))
        ti = torch.cat([init_q.view(1, 1, Q).transpose(1, 2), yq.cpu()[:, :, :-1]], dim=2)
        rec = []
        orc.incremental_forward(gq.cfg, gq.w, test_inputs=ti, T=32, softmax=False, quantize=False, params_out=rec)
        assert_class_ids_match(yq.argmax(1).cpu(), torch.stack(rec, -1), nz["e"], "initial_input " + layout)
    # per-utterance one-hot start classes and a dense (non one-hot) start vector are fed as given (wavenet.py:281-292)
    B2 = 3
    oh = torch.zeros(B2, 1, Q)
    for r, k in enumerate((5, 200, 77)):
        oh[r, 0, k] = 1
    nz = orc.predraw_noise(gq.cfg, B2, 24, 8)
    for init_q in (oh, 0.7 * oh + 0.3 / Q):
        p_got = mq.incremental_forward(initial_input=init_q, T=24, noise=dev_noise(nz), softmax=True, quantize=False)
        for r in range(B2):
            p_ref = orc.incremental_forward(gq.cfg, gq.w, initial_input=init_q[r:r + 1], T=24, softmax=True, quantize=False)
            assert float((p_got[r:r + 1].cpu() - p_ref).abs().max()) <= 1e-5


# ------------------------------------------------------------------------------------------------
# Batch tiles at BASELINE config 2's full width (what config 4 runs: 8 utterances per GPU in one launch), and a
# wide stack whose blocks own several row quads per job
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [2, 4, 8])
def test_config2_width_batch_tiles_against_oracle(B, engine):
    m, cfg, w, _ = full_case("cfg2_mol24")
    T = 64
    gen = torch.Generator().manual_seed(40 + B)
    c = torch.randn(B, cfg.cin_channels, T, generator=gen)
    noise = orc.predraw_noise(cfg, B, T, 50 + B)
    rec = []
    with torch.no_grad():
        y_ref = orc.incremental_forward(cfg, w, c=c, T=T, noise=orc.replay_from_predrawn(cfg, noise), params_out=rec)
    p_ref = torch.stack(rec, dim=-1)
    mc = m.cuda()
    assert mc._get_engine().plan(B)["batch_tile"] == min(B, 8 if engine == 7 else 4)      # engine 5 runs tiles of <= 4
    ti = torch.cat([torch.zeros(B, 1, 1), y_ref[:, :, :-1]], dim=2)
    y_tf, params = mc.incremental_forward(test_inputs=ti, c=c, T=T, noise=dev_noise(noise), return_params=True)
    perr = float((params.cpu() - p_ref).abs().max())
    assert perr <= PARAM_TOL * 2, perr
    assert float((y_tf.cpu() - y_ref).abs().max()) <= 2e-4
    y = mc.incremental_forward(c=c, T=T, noise=dev_noise(noise))
    rms = float(((y.cpu() - y_ref) ** 2).mean().sqrt())
    assert rms <= RMS_TOL, rms


@pytest.mark.parametrize("B", [1, 4])
def test_wide_stack_several_quads_per_owner(B, engine):
    """R = 768, G/2 = 384: every block owns 3 gate pairs / 6 residual rows / 9-step tiles (a wide layer whose per-block
    blob still double-buffers in shared memory)."""
    from wavenet_vocoder_b200 import WaveNet
    kw = dict(out_channels=30, layers=4, stacks=2, residual_channels=768, gate_channels=768, skip_out_channels=256,
              cin_channels=80, gin_channels=-1, scalar_input=True, output_distribution="Logistic", dropout=0.0)
    torch.manual_seed(21)
    m = WaveNet(**kw).eval()
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if n_.endswith(".bias"):
                p.normal_(0, 0.05)
        m.last_conv_layers[3].bias[20:] -= 3.0
    cfg = orc.PathConfig(out_channels=30, layers=4, stacks=2, residual_channels=768, gate_channels=768,
                         skip_out_channels=256, kernel_size=3, cin_channels=80, gin_channels=-1, scalar_input=True,
                         output_distribution="Logistic")
    w = orc.weights_from_state_dict(cfg, {k: v.detach().clone() for k, v in m.state_dict().items()})
    T = 40
    gen = torch.Generator().manual_seed(3)
    c = torch.randn(B, 80, T, generator=gen)
    noise = orc.predraw_noise(cfg, B, T, 4)
    rec = []
    with torch.no_grad():
        y_ref = orc.incremental_forward(cfg, w, c=c, T=T, noise=orc.replay_from_predrawn(cfg, noise), params_out=rec)
    mc = m.cuda()
    if engine == 5 and B == 4:
        # the default engine's shared-memory map has no room for two weight slots of this layer at a tile of 4: the
        # planner must say so (a clean status, not a crash)
        from wavenet_vocoder_b200._native import WnError
        with pytest.raises(WnError, match="shared memory too small"):
            mc.incremental_forward(c=c, T=T, noise=dev_noise(noise))
        return
    plan = mc._get_engine().plan(B)
    assert plan["rows_y"] == 3 and plan["rows_x"] == 6
    ti = torch.cat([torch.zeros(B, 1, 1), y_ref[:, :, :-1]], dim=2)
    _, params = mc.incremental_forward(test_inputs=ti, c=c, T=T, noise=dev_noise(noise), return_params=True)
    assert float((params.cpu() - torch.stack(rec, -1)).abs().max()) <= 1e-4


# ------------------------------------------------------------------------------------------------
# The TIMED path draws its noise on the device (Philox4x32-10 -> uniform / Box-Muller): its distribution against the
# oracle's sampler (torch RNG) on FIXED head outputs.  A model whose head output is a constant vector (all weights of the
# last 1x1 zero, the parameters in its bias) makes every step an independent draw from the same distribution.
# ------------------------------------------------------------------------------------------------
def const_head_model(kw, bias):
    from wavenet_vocoder_b200 import WaveNet
    torch.manual_seed(0)
    m = WaveNet(**kw).eval()
    with torch.no_grad():
        m.last_conv_layers[3].weight_g.mul_(0)        # w = g * v / |v| = 0
        m.last_conv_layers[3].bias.copy_(bias)
    return m.cuda()


def ks_two_sample(a, b):
    a, b = np.sort(a), np.sort(b)
    allv = np.concatenate([a, b])
    ca = np.searchsorted(a, allv, side="right") / a.size
    cb = np.searchsorted(b, allv, side="right") / b.size
    return float(np.abs(ca - cb).max())


def test_philox_mol_draws_follow_the_reference_sampler():
    K = 10
    kw = dict(out_channels=3 * K, layers=2, stacks=1, residual_channels=8, gate_channels=16, skip_out_channels=8,
              scalar_input=True, output_distribution="Logistic", dropout=0.0)
    gen = torch.Generator().manual_seed(1)
    logits = torch.randn(K, generator=gen)
    means = torch.linspace(-0.6, 0.6, K)
    log_scales = torch.full((K,), -5.5) + 0.3 * torch.randn(K, generator=gen)
    bias = torch.cat([logits, means, log_scales])
    m = const_head_model(kw, bias)
    B, T = 8, 25000                                                   # 2e5 independent draws
    y, params = m.incremental_forward(T=T, seed=123, initial_input=torch.zeros(B, 1, 1), return_params=True)
    assert float((params[:, :, ::997].cpu() - bias.view(1, -1, 1)).abs().max()) <= 1e-6      # the head really is constant
    got = y.reshape(-1).cpu().numpy()
    torch.manual_seed(5)
    n = got.size
    ref = orc.sample_mol(bias.view(1, 1, -1).expand(n, 1, -1).contiguous(), orc.GlobalNoise()).reshape(-1).numpy()
    # (a) component frequencies: nearest mean identifies the component (means are 0.13 apart, scales ~0.004)
    pick = lambda v: np.abs(v[:, None] - means.numpy()[None, :]).argmin(1)
    f_got = np.bincount(pick(got), minlength=K) / n
    f_ref = np.bincount(pick(ref), minlength=K) / n
    p_true = torch.softmax(logits, 0).numpy()
    sigma = np.sqrt(p_true * (1 - p_true) / n)
    assert np.all(np.abs(f_got - p_true) <= 5 * sigma + 2e-3), (f_got, p_true)
    assert np.all(np.abs(f_got - f_ref) <= 7 * sigma + 2e-3)
    # (b) moments and (c) Kolmogorov-Smirnov distance between the two samples (critical value 1.95*sqrt(2/n) at 1e-3)
    assert abs(got.mean() - ref.mean()) <= 5 * ref.std() / np.sqrt(n) * np.sqrt(2)
    assert abs(got.var() / ref.var() - 1.0) <= 0.02
    assert ks_two_sample(got, ref) <= 1.95 * np.sqrt(2.0 / n) * 1.5


def test_philox_gaussian_and_categorical_draws():
    # single Gaussian: Box-Muller normal vs torch normal
    kw = dict(out_channels=2, layers=2, stacks=1, residual_channels=8, gate_channels=16, skip_out_channels=8,
              scalar_input=True, output_distribution="Normal", dropout=0.0)
    bias = torch.tensor([0.1, -2.0])
    m = const_head_model(kw, bias)
    B, T = 8, 25000
    got = m.incremental_forward(T=T, seed=9, initial_input=torch.zeros(B, 1, 1)).reshape(-1).cpu().numpy()
    n = got.size
    sd = float(np.exp(-2.0))
    assert abs(got.mean() - 0.1) <= 5 * sd / np.sqrt(n)
    assert abs(got.std() / sd - 1.0) <= 0.01
    torch.manual_seed(2)
    ref = (torch.randn(n) * sd + 0.1).clamp(-1, 1).numpy()
    assert ks_two_sample(got, ref) <= 1.95 * np.sqrt(2.0 / n) * 1.5
    # categorical (softmax head): class frequencies vs the probabilities
    Q = 16
    kwq = dict(out_channels=Q, layers=2, stacks=1, residual_channels=8, gate_channels=16, skip_out_channels=8,
               scalar_input=False, dropout=0.0)
    logits = torch.randn(Q, generator=torch.Generator().manual_seed(3))
    mq = const_head_model(kwq, logits)
    init = torch.zeros(B, 1, Q)
    init[:, :, 0] = 1
    yq = mq.incremental_forward(T=T, seed=4, initial_input=init)
    idx = yq.argmax(1).reshape(-1).cpu().numpy()
    f = np.bincount(idx, minlength=Q) / idx.size
    p = torch.softmax(logits, 0).numpy()
    assert np.all(np.abs(f - p) <= 5 * np.sqrt(p * (1 - p) / idx.size) + 1e-3), (f, p)


# ------------------------------------------------------------------------------------------------
# Full-length runs with a strided oracle check: the kernel free-runs T samples (device noise, the timed path); windows
# of its OWN output are then teacher-forced into the oracle, preceded by one receptive field of history so that the
# oracle's zero-initialised queues have forgotten their start, and the head outputs of the window are compared.
# ------------------------------------------------------------------------------------------------
def strided_oracle_check(name, T, starts, win, tol):
    m, cfg, w, _ = full_case(name)
    rf = orc.receptive_field_size(cfg.layers, cfg.stacks, cfg.kernel_size)
    gen = torch.Generator().manual_seed(6)
    c = torch.randn(1, cfg.cin_channels, T, generator=gen)
    mc = m.cuda()
    y, params = mc.incremental_forward(c=c, T=T, seed=31, return_params=True)
    y, params = y.cpu(), params.cpu()
    assert bool(torch.isfinite(y).all()) and float(y.abs().max()) <= 1.0 and float(y.std()) > 1e-3
    worst = 0.0
    for t0 in starts:
        a = max(0, t0 - rf)                                        # oracle starts here with empty queues
        b = min(T, t0 + win)
        # input of step t is the sample of step t-1 (0 at t=0)
        prev = torch.cat([torch.zeros(1, 1, 1), y[:, :, :-1]], dim=2)[:, :, a:b]
        rec = []
        with torch.no_grad():
            orc.incremental_forward(cfg, w, test_inputs=prev, c=c[:, :, a:b], T=b - a,
                                    noise=orc.replay_from_predrawn(cfg, orc.predraw_noise(cfg, 1, b - a, 1)),
                                    params_out=rec)
        p_ref = torch.stack(rec, dim=-1)
        lo = t0 - a if a > 0 else 0
        err = float((params[:, :, a + lo:b] - p_ref[:, :, lo:]).abs().max())
        worst = max(worst, err)
        assert err <= tol, (name, t0, err)
    print("%s: strided oracle check over %d windows, worst head-output error %.3g" % (name, len(starts), worst))


def test_config2_full_length_strided_oracle():
    strided_oracle_check("cfg2_mol24", 22050, [0, 11000, 22050 - 256], 256, 2e-5 * 2.5)


def test_config5_long_form_strided_oracle():
    """BASELINE config 5: T = 240 000 (10 s at 24 kHz): tag arithmetic, 234 wraps of the largest history ring."""
    strided_oracle_check("cfg5_mol30", 240000, [0, 239000], 192, 2e-5 * 2.5)


def test_concurrent_half_grid_tiles_equal_sequential_tiles():
    """BASELINE config 4's per-GPU share (8 utterances) as two batch tiles of 4 running at the same time on two
    half-grid engines: the result must equal one full-grid call with the same seed (same Philox rows; the row
    partition only changes the fp32 summation order)."""
    m, cfg, w, _ = full_case("cfg2_mol24")
    mc = m.cuda()
    eng = mc._get_engine()
    if eng.plan(1)["engine"] != 5:
        pytest.skip("the concurrent-tile path is built on the default engine")
    B, T = 8, 48
    gen = torch.Generator().manual_seed(12)
    c = torch.randn(B, T, cfg.cin_channels, generator=gen).cuda()
    out = eng.generate_concurrent(B=B, T=T, c=c, seed=99)
    assert tuple(out.shape) == (B, T) and bool(torch.isfinite(out).all())
    ref, _ = eng.generate(B=B, T=T, c=c, seed=99)              # one engine, tiles one after the other, same Philox rows
    rms = float(((out - ref) ** 2).mean().sqrt())
    assert rms <= RMS_TOL, rms
    assert not torch.equal(out[:4], out[4:])
    # the class routes a free-running batch of more than one tile through the same path
    y = mc.incremental_forward(c=c.transpose(1, 2).contiguous(), T=T, seed=99)
    assert tuple(y.shape) == (B, 1, T)
    assert float(((y[:, 0] - ref) ** 2).mean().sqrt()) <= RMS_TOL
