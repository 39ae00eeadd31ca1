# coding: utf-8
"""The kernels on the model shapes of tests/shape_cases.py (kernel sizes 1, 2, 4 and 8, one layer, one-layer stacks,
a gate half of 640, residual / skip vectors of 1024, 128 conditioning channels, 34 mixtures, 1024 classes, and the
ragged shapes: vectors of 2 mod 4, heads of 3, 33 and 255, kernel sizes 5 to 7), on an H100:
  - teacher-forced head outputs against the fp32 oracle and against the module's float64 batch forward();
  - free running under replayed noise against the oracle (waveform RMS; class ids on the kernel's own trajectory);
  - streams: chunked == one shot bit for bit, chunk boundaries at different ring phases;
  - streams whose fed-back vector is dense (quantize=False), against incremental_forward with the same flags;
  - the upsampler at 128 channels and at its 8-scale limit, and the PyTorch path beyond it.
Every T is at least twice the largest ring delay so that every ring wraps; kernel_size 8 (delays up to 3584) is
checked over 8000 free-running steps by teacher-forcing the kernel's own output into the oracle."""
import pytest
import torch

from oracle import wavenet_oracle as orc
from helpers import GoldenCase
from shape_cases import MAX_B, NAMES, PARAM_TOL, ShapeCase, fresh_module, full_kw, max_delay, path_config
from test_gpu_parity import RMS_TOL, assert_class_ids_match
from test_shape_coverage_host import cfg_of, plan_status
from test_streaming import assert_same, chunked, inputs_for, model_of, one_shot
from test_upsample import TOL as UPS_TOL, model_for

pytestmark = pytest.mark.gpu


@pytest.fixture(params=[5, 7])
def engine(request, monkeypatch):
    """Both kernel organisations: 5 = the default (csrc/wn_kernel.cuh), 7 = the alternative (csrc/wn7_kernel.cuh).
    A case engine 7 does not plan at the test's batch is skipped for engine 7 with the planner's message."""
    monkeypatch.setenv("WN_ENGINE", str(request.param))
    params = getattr(request.node, "callspec", None)
    name = params.params.get("name") if params is not None else None
    if request.param == 7 and name is not None:
        B = params.params.get("B", MAX_B[name])
        rc, msg = plan_status(cfg_of(name), B)
        if rc != 0:
            pytest.skip("engine 7 does not plan %s at B=%d: %s" % (name, B, msg))
    return request.param


def dev_noise(n):
    return {k: v.cuda() for k, v in n.items()}


def gpu_T(name):
    return max(64, 2 * max_delay(full_kw(name)) + 16) if name != "k8_global" else 200


def cuda_model(sc, engine):
    """The case's module on the device, planned by the engine the test asks for (the `engine` fixture skips a case
    engine 7 does not plan; tests/test_shape_coverage_host.py checks the plans without a GPU)."""
    m = fresh_module(sc.kw, sc.sd).cuda()
    assert m._get_engine().plan(sc.B)["engine"] == engine
    return m


def onehot_start(B, O, classes=None):
    x = torch.zeros(B, O, 1)
    for r in range(B):
        x[r, classes[r] if classes else 127] = 1
    return x


BATCHES = [(n, B) for n in NAMES for B in (1, 3) if B <= MAX_B[n]]


@pytest.mark.parametrize("name,B", BATCHES)
def test_teacher_forced_head_outputs(name, B, engine):
    T = gpu_T(name)
    sc = ShapeCase(name, B=B, T=T)
    m = cuda_model(sc, engine)
    noise = orc.predraw_noise(sc.cfg, B, T, 3)
    _, params = m.incremental_forward(test_inputs=sc.x_tf, c=sc.t("c_up"), T=T, noise=dev_noise(noise),
                                      return_params=True)
    got = params.cpu()
    ref = sc.t("params_tf")
    assert got.shape == ref.shape
    err = float((got - ref).abs().max())
    err64 = float((got.double() - sc.forward64()).abs().max())
    print("%s B=%d engine %d: head-output max abs err %.3g vs oracle, %.3g vs float64 forward()" % (
        name, B, engine, err, err64))
    assert err <= PARAM_TOL[name], err
    assert err64 <= PARAM_TOL[name], err64


@pytest.mark.parametrize("name", NAMES)
def test_free_running_replayed_noise(name, engine):
    B, T = MAX_B[name], gpu_T(name)
    sc = ShapeCase(name, B=B, T=T, oracle=False)
    m = cuda_model(sc, engine)
    cfg, c = sc.cfg, sc.t("c_up")
    noise = orc.predraw_noise(cfg, B, T, 4)
    if cfg.scalar_input:
        y = m.incremental_forward(c=c, T=T, noise=dev_noise(noise)).cpu()
        with torch.no_grad():
            y_ref = orc.incremental_forward(cfg, sc.w, c=c, T=T, noise=orc.replay_from_predrawn(cfg, noise))
        assert y.shape == y_ref.shape
        rms = float(((y - y_ref) ** 2).mean().sqrt())
        assert float(y.std()) > 1e-3
        assert rms <= RMS_TOL, rms
        return
    # class ids: every step on the kernel's OWN trajectory, so one near-tie cannot hide later mismatches
    first = onehot_start(B, cfg.out_channels)
    y = m.incremental_forward(initial_input=first, T=T, noise=dev_noise(noise)).cpu()
    ti = torch.cat([first, y[:, :, :-1]], dim=2)
    rec = []
    with torch.no_grad():
        orc.incremental_forward(cfg, sc.w, test_inputs=ti, T=T, softmax=False, quantize=False, params_out=rec)
    assert_class_ids_match(y.argmax(1), torch.stack(rec, -1), noise["e"], name + " (free running)")


def test_kernel_size_8_long_form_against_oracle(engine):
    """Delays up to 3584: 8000 free-running steps (device noise) wrap the largest ring twice.  The kernel's own output
    is teacher-forced into the oracle from step 0 (the receptive field, 14 323, exceeds T: no later window could start
    with the oracle's queues empty and forgotten) and every step's head output is compared."""
    name, T = "k8_global", 8000
    sc = ShapeCase(name, B=1, T=T, oracle=False)
    m = cuda_model(sc, engine)
    c = sc.t("c_up")
    y, params = m.incremental_forward(c=c, T=T, seed=31, return_params=True)
    y, params = y.cpu(), params.cpu()
    assert bool(torch.isfinite(y).all()) and float(y.abs().max()) <= 1.0 and float(y.std()) > 1e-3
    prev = torch.cat([torch.zeros(1, 1, 1), y[:, :, :-1]], dim=2)
    rec = []
    with torch.no_grad():
        orc.incremental_forward(sc.cfg, sc.w, test_inputs=prev, c=c, T=T,
                                noise=orc.replay_from_predrawn(sc.cfg, orc.predraw_noise(sc.cfg, 1, T, 1)),
                                params_out=rec)
    p_ref = torch.stack(rec, dim=-1)
    err = (params - p_ref).abs().amax(dim=(0, 1))
    D = max_delay(sc.kw)
    print("%s engine %d: head-output max abs err %.3g over %d steps (%.3g after the first wrap of the %d ring)" % (
        name, engine, float(err.max()), T, float(err[D:].max()), D))
    assert float(err.max()) <= PARAM_TOL[name], float(err.max())


# ------------------------------------------------------------------------------------------------
# streams (engine 5)
# ------------------------------------------------------------------------------------------------
def ring_phase_split(T, D):
    """1, a prime, exactly the largest delay, then the rest: chunk boundaries at different ring phases."""
    parts = [1, 7] + ([D] if D > 0 else [])
    return parts + [T - sum(parts)]


@pytest.mark.parametrize("noise_kind", ["replay", "philox"])
@pytest.mark.parametrize("name,B", BATCHES)
def test_chunked_equals_one_shot(name, B, noise_kind):
    kw = full_kw(name)
    D = max_delay(kw)
    T = max(96, 2 * D + 64)
    sc = ShapeCase(name, B=B, T=T, oracle=False)
    m = fresh_module(sc.kw, sc.sd).cuda()
    assert m._get_engine().plan(B)["engine"] == 5
    gen = torch.Generator().manual_seed(B)
    init, c, g = inputs_for(m, kw, B, T, gen)
    noise = dev_noise(orc.predraw_noise(sc.cfg, B, T, 5)) if noise_kind == "replay" else None
    seed = None if noise is not None else 1234 + B
    split = ring_phase_split(T, D)
    assert_same(chunked(m, kw, B, T, init, c, g, noise, seed, split=split), one_shot(m, B, T, init, c, g, noise, seed))


def dense_feedback_model(name):
    if name == "mulaw_softmax":
        gc = GoldenCase(name)
        return model_of(gc.kw, gc.sd), gc.kw
    sc = ShapeCase(name, oracle=False)
    return fresh_module(sc.kw, sc.sd).cuda(), sc.kw


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("start", ["default", "dense"])
@pytest.mark.parametrize("softmax", [True, False])
@pytest.mark.parametrize("name", ["mulaw_softmax", "k4_softmax"])
def test_dense_feedback_stream_equals_one_shot(name, softmax, start, B):
    """quantize=False feeds back the dense vector (probabilities or logits) that the stream state keeps between
    chunks; from the default class and from a dense initial_input."""
    m, kw = dense_feedback_model(name)
    Q = kw["out_channels"]
    D = max_delay(dict(kw, kernel_size=kw.get("kernel_size", 3)))
    T = 2 * D + 64
    if start == "default":
        init_stream, init_ref = None, onehot_start(B, Q)
    else:
        init_stream = init_ref = 0.7 * onehot_start(B, Q, (5, 200, 77)) + 0.3 / Q
    ref = m.incremental_forward(initial_input=init_ref, T=T, softmax=softmax, quantize=False, return_params=True)
    s = m.open_stream(B=B, initial_input=init_stream, softmax=softmax, quantize=False, return_params=True)
    ys, ps = [], []
    for n in ring_phase_split(T, D):
        y, p = s.generate(n)
        ys.append(y), ps.append(p)
    assert s.t == T
    s.close()
    got = (torch.cat(ys, -1), torch.cat(ps, -1))
    assert got[0].shape == (B, Q, T)
    assert_same(got, ref)


# ------------------------------------------------------------------------------------------------
# the upsampler at its limits
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scales,C,frames", [([4, 4, 4, 4], 128, 17),       # 139 KB of dynamic shared memory
                                             ([2] * 8, 80, 9)])              # WNAUX_MAX_SCALES
def test_native_upsampler_at_its_limits(scales, C, frames):
    m = model_for(scales, 2, C=C)
    B = 3
    c = torch.randn(B, C, frames + 2 * 2, generator=torch.Generator().manual_seed(C))
    with torch.no_grad():
        ref = m.upsample_net(c)                                   # fp32 on the CPU
    m = m.cuda()
    eng = m._get_engine()
    T = ref.size(-1)
    assert m._native_upsample and eng.upsampled_length(c.size(-1)) == T
    got = eng.upsample(c.cuda(), T).cpu()
    assert tuple(got.shape) == (B, T, C)
    err = float((got.transpose(1, 2) - ref).abs().max())
    assert err <= UPS_TOL, err


def test_nine_scales_take_the_pytorch_upsampler():
    """Beyond 8 scales the native upsampler refuses the network: the module's own upsampler runs (in fp32) and the
    synthesis matches the oracle fed with the CPU module's upsampled conditioning."""
    m = model_for([2] * 9, 0, C=80)
    frames = torch.randn(1, 80, 2, generator=torch.Generator().manual_seed(9))
    with torch.no_grad():
        c_up = m.upsample_net(frames)
    T = c_up.size(-1)
    kw = dict(out_channels=30, layers=2, stacks=1, residual_channels=16, gate_channels=32, skip_out_channels=16,
              kernel_size=3, cin_channels=80, gin_channels=-1, scalar_input=True, output_distribution="Logistic")
    cfg = path_config(kw)
    w = orc.weights_from_state_dict(cfg, {k: v.detach().clone() for k, v in m.state_dict().items()})
    noise = orc.predraw_noise(cfg, 1, T, 2)
    rec = []
    with torch.no_grad():
        y_ref = orc.incremental_forward(cfg, w, c=c_up, T=T, noise=orc.replay_from_predrawn(cfg, noise), params_out=rec)
    m = m.cuda()
    m._get_engine()
    assert not m._native_upsample
    y, params = m.incremental_forward(c=frames, T=T, noise=dev_noise(noise), return_params=True)
    assert float((params.cpu() - torch.stack(rec, -1)).abs().max()) <= 2e-5
    assert float(((y.cpu() - y_ref) ** 2).mean().sqrt()) <= RMS_TOL
