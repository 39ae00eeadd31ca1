# coding: utf-8
"""The plan-variant matrix of tests/plan_variants.py without a GPU:
  - every entry plans what it claims to test (ring depth, resident blobs, ring placement, replicas, polling warps,
    batch tile, engine) at every launch it makes, so that a knob that silently clamps to the default cannot leave its
    GPU test comparing the default plan with itself;
  - every synthesis kernel instantiation compiled into libwn.so is launched by a matrix entry or by a named existing
    test, so that a new instantiation without a test fails here;
  - every WN_* knob the library reads is in the matrix or exempt with a reason, and every planner field of wn_config
    is set by some entry;
  - engine 7's poll_warps range as include/wn.h states it."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

import plan_variants as pv
from conftest import ROOT
from wavenet_vocoder_b200 import _native as N
from wavenet_vocoder_b200.engine import make_config

SMEM = 232448
NSM = 132                 # SMs of an H100 SXM

# knobs read by the library that no entry sets, and why
EXEMPT = {
    "WN_PROF": "a diagnostic: per-block cycle counters, read back by wn_sync; the arithmetic is untouched",
    "WN_TIMEOUT_MS": "a diagnostic: the device watchdog's limit; only a stalled run reaches it",
    "WN_POLL_DEFAULT": "an alias: engine 7's poll_warps when neither the field nor WN_POLL_WARPS sets it",
}
CFG_FIELDS = ("num_ctas", "exchange_copies", "ring_slots", "poll_warps")


def cfg_of(kw, **fields):
    return make_config(layers=kw["layers"], stacks=kw["stacks"], residual_channels=kw["residual_channels"],
                       gate_channels=kw["gate_channels"], skip_out_channels=kw["skip_out_channels"],
                       out_channels=kw["out_channels"], kernel_size=kw["kernel_size"],
                       cin_channels=kw["cin_channels"], gin_channels=kw["gin_channels"],
                       scalar_input=kw["scalar_input"], output_distribution=kw.get("output_distribution", "Logistic"),
                       **fields)


def plan_only(kw, batch, **fields):
    info = N.wn_plan_info()
    N.check(N.lib().wn_plan_only(C.byref(cfg_of(kw, **fields)), batch, NSM, SMEM, C.byref(info)))
    return info.as_dict()


def set_env(monkeypatch, engine, env):
    for k in list(os.environ):
        if k.startswith("WN_"):
            monkeypatch.delenv(k)
    monkeypatch.setenv("WN_ENGINE", str(engine))
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def launches(kw, B, engine, stream, env, cfg=None):
    """[(plan, kernel)] of the launches one call makes: wn_generate splits B into batch tiles, a stream is one tile."""
    sizes = [B] if stream else pv.chunks(B, pv.max_tile(env, engine))
    out = []
    for b in sorted(set(sizes)):
        p = plan_only(kw, b, **(cfg or {}))
        out.append((p, pv.kernel_name(kw, p, engine, stream)))
    return out


def entry_launches(e, monkeypatch):
    set_env(monkeypatch, e.engine, e.env)
    kw = pv.BASES[e.base]["kw"]
    out = launches(kw, e.B, e.engine, False, e.env, e.cfg)
    if e.stream:
        out += launches(kw, e.B, e.engine, True, e.env, e.cfg)
    return out


@pytest.mark.parametrize("e", pv.MATRIX, ids=[e.id for e in pv.MATRIX])
def test_entry_plans_what_it_tests(e, monkeypatch):
    if e.stream:
        assert e.engine == 5 and e.B <= 4, "streams run on engine 5, one tile of at most 4"
    if e.vs_b1:      # the rows of a tile sum in the order of B = 1 only at a tile of 1 or with one element per thread
        kw = pv.BASES[e.base]["kw"]
        assert e.B > 1 and (pv.max_tile(e.env, e.engine) == 1 or
                            pv.variant(kw["residual_channels"], kw["gate_channels"] // 2) == (1, 1)), e.id
    kw = pv.BASES[e.base]["kw"]
    for p, kernel in entry_launches(e, monkeypatch):
        assert p["engine"] == e.engine
        for k, v in e.expect.items():
            assert p[k] == v, (e.id, k, p[k], v)
        nstream = p["blobs_per_step"] - p["resident_blobs"]
        assert (p["ring_slots"] > 0) == (nstream > 0)
        if any(k in e.env for k in ("WN_L2_PREFETCH", "WN_RING_SLOTS", "WN_RESIDENT")) or "ring_slots" in e.cfg:
            assert nstream > 0, "%s: nothing is streamed, the knob has nothing to act on" % e.id
        if e.engine == 7 and ("poll_warps" in e.cfg or "WN_POLL_WARPS" in e.env):
            assert kernel.endswith("false>"), "%s: the polling-warp kernel is not taken" % e.id
        # the variant follows R and G/2 (wn_host.cu launch_chunk's efor)
        if e.engine == 5:
            er, eg = pv.variant(kw["residual_channels"], kw["gate_channels"] // 2)
            assert ("<%d, %d, %d, " % (p["batch_tile"], er, eg)) in kernel


def test_streamed_blob_count_is_not_a_multiple_of_the_ring_depth(monkeypatch):
    """mbarrier phases when the ring depth does not divide the blobs streamed per step: at least one streamed entry
    per engine has nstream mod ring_slots != 0 (the ring slot of blob i drifts from step to step)."""
    for engine in (5, 7):
        drift = []
        for e in pv.MATRIX:
            if e.engine != engine:
                continue
            for p, _ in entry_launches(e, monkeypatch):
                nstream = p["blobs_per_step"] - p["resident_blobs"]
                if nstream > 0 and nstream % p["ring_slots"] != 0:
                    drift.append(e.id)
        assert drift, engine


def test_l2_prefetch_distances_cover_the_edges(monkeypatch):
    """D = 0, 2, 3, nstream - 1, nstream and above nstream on one base, each also at T = 1, 2 and in a stream."""
    by_base = {}
    for e in pv.MATRIX:
        if "WN_L2_PREFETCH" in e.env and e.B == 1:
            p = entry_launches(e, monkeypatch)[0][0]
            nstream = p["blobs_per_step"] - p["resident_blobs"]
            by_base.setdefault(e.base, set()).add(int(e.env["WN_L2_PREFETCH"]) - nstream)
            assert e.engine == 5 and e.short and e.stream
    rel = by_base["cfg2"]
    assert {-24, -22, -21, -1, 0} <= rel and max(rel) > 0, sorted(rel)


def library_kernels():
    path = N.LIB_PATH
    if not os.path.exists(path):
        pytest.skip("libwn.so is not built (run __graft_entry__.build())")
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm (binutils) is not installed: the kernel instantiations cannot be listed")
    out = subprocess.run([nm, "-C", path], capture_output=True, text=True, check=True).stdout
    return set(re.findall(r"(wn::wn_persistent_kernel<\d+, \d+, \d+, (?:true|false)>|"
                          r"wn7::wn7_kernel<\d+, (?:true|false)>)", out))


def test_every_kernel_instantiation_is_launched_by_a_test(monkeypatch):
    lib = library_kernels()
    assert any(k.startswith("wn::") for k in lib) and any(k.startswith("wn7::") for k in lib), sorted(lib)
    reached = {}
    for e in pv.MATRIX:
        for _, kernel in entry_launches(e, monkeypatch):
            reached.setdefault(kernel, []).append("tests/test_plan_variants.py::test_plan_variant[%s]" % e.id)
    for test, kw, B, engine, stream, env in pv.existing_launches():
        path, name = test.split("::")
        assert re.search(r"^def %s\(" % re.escape(name.split("[")[0]), open(os.path.join(ROOT, path)).read(), re.M), test
        set_env(monkeypatch, engine, env)
        for _, kernel in launches(kw, B, engine, False, env) + (launches(kw, B, engine, True, env) if stream else []):
            reached.setdefault(kernel, []).append(test)
    assert set(reached) <= lib, sorted(set(reached) - lib)
    missing = sorted(lib - set(reached))
    assert not missing, "kernel instantiations no test launches: %s" % missing


def test_every_knob_is_in_the_matrix_or_exempt():
    names = set()
    for d in (os.path.join(ROOT, "wavenet_vocoder_b200", "csrc"),):
        for f in os.listdir(d):
            names |= set(re.findall(r'env_int\("(WN_[A-Z0-9_]+)"', open(os.path.join(d, f)).read()))
    assert len(names) > 10, names
    used = {k for e in pv.MATRIX for k in e.env} | ({"WN_ENGINE"} if any(e.engine == 7 for e in pv.MATRIX) else set())
    missing = sorted(names - used - set(EXEMPT))
    assert not missing, "knobs neither tested nor exempt: %s" % missing
    assert not (set(EXEMPT) & used) and set(EXEMPT) <= names, "stale exemption"
    fields = {k for e in pv.MATRIX for k in e.cfg}
    assert set(CFG_FIELDS) - {"num_ctas"} <= fields, "wn_config fields no entry sets: %s" % (set(CFG_FIELDS) - fields)


def test_poll_warps_range(monkeypatch):
    """include/wn.h: poll_warps 2..8, larger values plan as 8, -1 = the compute warps poll; the field wins over
    WN_POLL_WARPS."""
    hdr = open(os.path.join(ROOT, "include", "wn.h")).read()
    assert re.search(r"poll_warps;\s*/\*[^*]*\(2\.\.8", hdr), "include/wn.h states another poll_warps range"
    set_env(monkeypatch, 7, {})
    kw = pv.BASES["cfg2"]["kw"]
    for asked, planned in ((-1, 0), (1, 2), (2, 2), (5, 5), (8, 8), (12, 8)):
        p = plan_only(kw, 1, poll_warps=asked)
        assert p["poll_warps"] == planned, (asked, p["poll_warps"])
    assert plan_only(kw, 1)["poll_warps"] == 0                     # the default: the compute warps poll
    monkeypatch.setenv("WN_POLL_WARPS", "4")
    assert plan_only(kw, 1)["poll_warps"] == 4
    assert plan_only(kw, 1, poll_warps=6)["poll_warps"] == 6
