# coding: utf-8
"""Every entry of the plan-variant matrix (tests/plan_variants.py) on an H100, on a handle of its own created under
the entry's knobs, checked two ways:
  (a) bit for bit against a handle of the default plan on the same shape, batch and inputs: the teacher-forced head
      outputs and samples, the free-running waveform (or class ids) and head outputs under replayed noise and under
      Philox; and for batch-tile entries whose rows sum in the same order at every tile, row 0 against the default
      plan run alone;
  (b) the teacher-forced head outputs against the module's float64 batch forward();
and, where the entry asks for it, bit for bit against its own long run at T = 1 and 2 (its first steps) and as a
stream cut into chunks of 1, 7 and 64 samples.  Entries whose knob changes the arithmetic or its order (the row
partition, a tile of 1) are compared with the default plan through (b) alone; the entry says why.  A race, a wrong
ring slot or a stale exchange line cannot hide inside (a)'s tolerance, because it has none."""
import os

import pytest
import torch

import plan_variants as pv
from oracle import wavenet_oracle as orc
from wavenet_vocoder_b200.engine import SynthesisEngine

pytestmark = pytest.mark.gpu

SEED = 4321
DEV = torch.device("cuda", 0)


class BaseData:
    """A base shape's weights and seeded inputs at the largest batch any entry runs it at; a batch of B takes the
    first B rows, so every run of the base sees the same utterances."""

    def __init__(self, base):
        spec = pv.BASES[base]
        self.base, self.kw = base, spec["kw"]
        self.T, self.T_tf = spec["T"], spec["T_tf"]
        self.B = max(e.B for e in pv.MATRIX if e.base == base)
        self.module = pv.make_module(base)
        self.sd = {k: v.detach().clone() for k, v in self.module.state_dict().items()}
        self.cfg = pv.path_config(base)
        kw, B, Tm = self.kw, self.B, max(self.T, self.T_tf)
        gen = torch.Generator().manual_seed(sum(map(ord, base)))
        if kw["scalar_input"]:
            self.x_tf = (torch.rand(B, self.T_tf, generator=gen) * 2 - 1) * 0.8
        else:
            self.x_tf = torch.randint(0, kw["out_channels"], (B, self.T_tf), generator=gen, dtype=torch.int32)
        self.c = torch.randn(B, kw["cin_channels"], Tm, generator=gen) if kw["cin_channels"] > 0 else None
        self.g_ids = torch.randint(0, kw["n_speakers"], (B, 1), generator=gen) if kw["gin_channels"] > 0 else None
        self.g = None
        if self.g_ids is not None:
            with torch.no_grad():
                self.g = self.module.embed_speakers(self.g_ids)[:, 0, :].contiguous()
        self.noise = orc.predraw_noise(self.cfg, B, Tm, 7)
        self._f64 = None

    def c_btc(self, B, t0, t1):
        return None if self.c is None else self.c[:B, :, t0:t1].transpose(1, 2).contiguous().to(DEV)

    def g_of(self, B):
        return None if self.g is None else self.g[:B].to(DEV)

    def noise_of(self, B, t0, t1):
        return {k: v[t0:t1, :B].contiguous().to(DEV) for k, v in self.noise.items()}

    def forward64(self):
        """Head outputs (B,O,T_tf) of the module's batch forward() in float64 on the teacher-forcing input."""
        if self._f64 is None:
            m = pv.make_module(self.base).double().eval()
            m.load_state_dict(self.sd)
            if self.kw["scalar_input"]:
                x = self.x_tf.double().unsqueeze(1)
            else:
                x = torch.zeros(self.B, self.kw["out_channels"], self.T_tf, dtype=torch.float64)
                x.scatter_(1, self.x_tf.long().unsqueeze(1), 1.0)
            c = None if self.c is None else self.c[:, :, :self.T_tf].double()
            with torch.no_grad():
                self._f64 = m(x, c=c, g=self.g_ids, softmax=False)
        return self._f64


@pytest.fixture(scope="module")
def bases():
    cache = {}

    def get(base):
        if base not in cache:
            cache[base] = BaseData(base)
        return cache[base]
    return get


def clear_knobs(monkeypatch):
    for k in list(os.environ):
        if k.startswith("WN_"):
            monkeypatch.delenv(k)


def new_engine(d, engine, env, cfg, monkeypatch):
    """A handle created (and, since the planner runs again at every launch, used) under exactly these knobs."""
    clear_knobs(monkeypatch)
    monkeypatch.setenv("WN_ENGINE", str(engine))
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    kw = d.kw
    eng = SynthesisEngine(layers=kw["layers"], stacks=kw["stacks"], residual_channels=kw["residual_channels"],
                          gate_channels=kw["gate_channels"], skip_out_channels=kw["skip_out_channels"],
                          out_channels=kw["out_channels"], kernel_size=kw["kernel_size"],
                          cin_channels=kw["cin_channels"], gin_channels=kw["gin_channels"],
                          scalar_input=kw["scalar_input"], output_distribution=kw.get("output_distribution", "Logistic"),
                          device=DEV, **cfg)
    eng.load_state_dict(d.sd)
    return eng


def cpu(r):
    return tuple(t.cpu() for t in r)


def one_shot(eng, d, B, T, tf=False, replay=True):
    """(out, params) of one call: teacher forced over T_tf steps, or free running over T steps."""
    if tf:
        x = d.x_tf[:B].to(DEV)
        forced = dict(test_scalar=x) if d.kw["scalar_input"] else dict(test_index=x)
        return cpu(eng.generate(B=B, T=T, c=d.c_btc(B, 0, T), g=d.g_of(B), noise=d.noise_of(B, 0, T),
                                want_params=True, **forced))
    if replay:
        return cpu(eng.generate(B=B, T=T, c=d.c_btc(B, 0, T), g=d.g_of(B), noise=d.noise_of(B, 0, T), want_params=True))
    return cpu(eng.generate(B=B, T=T, c=d.c_btc(B, 0, T), g=d.g_of(B), seed=SEED, want_params=True))


def runs(eng, d, B):
    return {"teacher-forced": one_shot(eng, d, B, d.T_tf, tf=True),
            "replayed noise": one_shot(eng, d, B, d.T),
            "philox": one_shot(eng, d, B, d.T, replay=False)}


def streamed(eng, d, B, replay):
    s = eng.open_stream(B=B, g=d.g_of(B), replay=replay, seed=None if replay else SEED)
    outs, params, t = [], [], 0
    split = list(pv.STREAM_SPLIT) + [d.T - sum(pv.STREAM_SPLIT)]
    for n in split:
        o, p = s.generate(n, c=d.c_btc(B, t, t + n), noise=d.noise_of(B, t, t + n) if replay else None,
                          want_params=True)
        outs.append(o)
        params.append(p)
        t += n
    assert s.t == d.T
    s.close()
    return torch.cat(outs, -1).cpu(), torch.cat(params, -1).cpu()


def assert_equal(got, ref, what):
    for name, a, b in zip(("samples", "head outputs"), got, ref):
        assert a.shape == b.shape, (what, name, a.shape, b.shape)
        if not torch.equal(a, b):
            diff = (a.double() - b.double()).abs()
            idx = (a != b).nonzero()[0].tolist()
            raise AssertionError("%s: %s differ from the reference at %d places, first at %s, max %.3g" % (
                what, name, int((a != b).sum()), idx, float(diff.max())))


_DEFAULTS = {}


def default_runs(d, B, engine, monkeypatch):
    """The same shape, batch and inputs on a handle of the default plan (one per base, batch and engine)."""
    key = (d.base, B, engine)
    if key not in _DEFAULTS:
        eng = new_engine(d, engine, {}, {}, monkeypatch)
        try:
            _DEFAULTS[key] = runs(eng, d, B)
        finally:
            eng.close()
    return _DEFAULTS[key]


@pytest.mark.parametrize("e", pv.MATRIX, ids=[e.id for e in pv.MATRIX])
def test_plan_variant(e, bases, monkeypatch):
    d = bases(e.base)
    ref = default_runs(d, e.B, e.engine, monkeypatch) if e.bit is None else None
    ref1 = default_runs(d, 1, e.engine, monkeypatch) if e.vs_b1 else None
    eng = new_engine(d, e.engine, e.env, e.cfg, monkeypatch)
    try:
        p = eng.plan(e.B)
        assert p["engine"] == e.engine
        for k, v in e.expect.items():
            assert p[k] == v, (e.id, k, p[k], v)
        got = runs(eng, d, e.B)
        # (b) float64 anchor
        err = float((got["teacher-forced"][1].double() - d.forward64()[:e.B]).abs().max())
        print("PV %s %s: teacher-forced head outputs vs float64 forward() max abs %.3g" % (e.base, e.id, err))
        assert err <= pv.TOL64[e.base], (e.id, err)
        # (a) bit identity with the default plan (or the entry's reference plan)
        if e.bit is None:
            for mode, r in got.items():
                assert_equal(r, ref[mode], "%s, %s" % (e.id, mode))
        if e.vs_b1:      # the reduction tree over the 32 lanes does not depend on the tile (reduce_scatter_multi)
            for mode, r in got.items():
                assert_equal((r[0][:1], r[1][:1]), ref1[mode], "%s, %s, row 0 against B = 1" % (e.id, mode))
        # the same handle: its first steps, and its stream
        if e.short:
            for T in pv.SHORT_T:
                for replay, mode in ((True, "replayed noise"), (False, "philox")):
                    o, p = one_shot(eng, d, e.B, T, replay=replay)
                    assert_equal((o, p), (got[mode][0][..., :T], got[mode][1][..., :T]),
                                 "%s, %s, T = %d" % (e.id, mode, T))
        if e.stream:
            for replay, mode in ((True, "replayed noise"), (False, "philox")):
                assert_equal(streamed(eng, d, e.B, replay), got[mode], "%s, %s, stream" % (e.id, mode))
    finally:
        eng.close()
