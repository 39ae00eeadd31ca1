# coding: utf-8
"""Engine-7 streams without a GPU: wn_config.engine picks the plan as WN_ENGINE does and wins over it, bad values are
refused, the structs keep their sizes at ABI 3, every engine-7 stream kernel in libwn.so is launched by a named GPU
test, and the whole-utterance engine-7 kernels are still exactly the 8 of before."""
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
BASES = ("cfg1", "cfg2", "cfg3", "cfg5")
GPU_FILE = os.path.join("tests", "test_streaming_engine7.py")


def cfg_of(kw, **fields):
    return make_config(layers=kw["layers"], stacks=kw["stacks"], residual_channels=kw["residual_channels"],
                       gate_channels=kw["gate_channels"], skip_out_channels=kw["skip_out_channels"],
                       out_channels=kw["out_channels"], kernel_size=kw.get("kernel_size", 3),
                       cin_channels=kw.get("cin_channels", -1), gin_channels=kw.get("gin_channels", -1),
                       scalar_input=kw["scalar_input"], output_distribution=kw.get("output_distribution", "Logistic"),
                       **fields)


def plan_only(kw, batch, **fields):
    info = N.wn_plan_info()
    N.check(N.lib().wn_plan_only(C.byref(cfg_of(kw, **fields)), batch, NSM, SMEM, C.byref(info)))
    d = info.as_dict()
    d.pop("launches")
    return d


def clear_env(monkeypatch):
    for k in list(os.environ):
        if k.startswith("WN_"):
            monkeypatch.delenv(k)


@pytest.mark.parametrize("B", [1, 2, 4, 8])
@pytest.mark.parametrize("base", BASES)
def test_config_engine_field_plans_like_the_environment(base, B, monkeypatch):
    kw = pv.BASES[base]["kw"]
    clear_env(monkeypatch)
    default = plan_only(kw, B)
    assert default["engine"] == 5
    assert plan_only(kw, B, engine=5) == default
    monkeypatch.setenv("WN_ENGINE", "7")
    by_env = plan_only(kw, B)
    assert by_env["engine"] == 7 and by_env["batch_tile"] == B
    assert plan_only(kw, B, engine=7) == by_env
    assert plan_only(kw, B, engine=5) == default            # the field wins over WN_ENGINE
    monkeypatch.delenv("WN_ENGINE")
    assert plan_only(kw, B, engine=7) == by_env


@pytest.mark.parametrize("value", [-1, 1, 6, 8, 70])
def test_unknown_engine_values_are_refused(value, monkeypatch):
    clear_env(monkeypatch)
    kw = pv.BASES["cfg2"]["kw"]
    cfg = cfg_of(kw, engine=value)
    info = N.wn_plan_info()
    assert N.lib().wn_plan_only(C.byref(cfg), 1, NSM, SMEM, C.byref(info)) == -1
    assert b"wn_config.engine" in N.lib().wn_last_error()
    pl = N.Wn7Plan()
    assert N.lib().wn_plan_passes(C.byref(cfg), 1, NSM, SMEM, C.cast(C.byref(pl), C.POINTER(C.c_int32)),
                                  C.sizeof(pl) // 4, None, 0) == -1
    buf = (C.c_float * 16)()
    assert N.lib().wn_pack_cta(C.byref(cfg), 1, NSM, SMEM, None, 0, buf, 16) == -1


def test_plan_passes_is_engine_7s_for_either_engine(monkeypatch):
    clear_env(monkeypatch)
    kw = pv.BASES["cfg2"]["kw"]
    ref_plan, ref_passes = N.plan_passes(cfg_of(kw), 8)
    for e in (5, 7):
        pl, ps = N.plan_passes(cfg_of(kw, engine=e), 8)
        assert bytes(pl) == bytes(ref_plan) and [bytes(p) for p in ps] == [bytes(p) for p in ref_passes]


def test_struct_sizes_and_abi_unchanged():
    L = N.lib()
    assert L.wn_abi_version() == N.WN_ABI_VERSION == 3
    sizes = (C.c_int32 * 7)()
    assert L.wn_struct_sizes(sizes, 7) == 7
    assert list(sizes) == [C.sizeof(t) for t in N.STRUCTS]
    # the new fields sit where a reserved slot was: sizes and every other offset as before
    assert C.sizeof(N.wn_config) == 24 * 4 and N.wn_config.engine.offset == 17 * 4
    assert N.wn_stream_open_args.engine.offset + 4 == N.wn_stream_open_args.reserved.offset
    assert len(N.wn_config().reserved) == 6 and len(N.wn_stream_open_args().reserved) == 5


def stream_launches():
    """(test name in the GPU file, model keywords, B) of every engine-7 stream the GPU tests open."""
    from helpers import GoldenCase
    golden = {n: dict(GoldenCase(n).kw) for n in ("mol_cond", "mulaw_softmax")}
    c2, c3, c5 = pv.BASES["cfg2"]["kw"], pv.BASES["cfg3"]["kw"], pv.BASES["cfg5"]["kw"]
    out = [("test_golden_cases_chunked_equal_one_shot", golden["mol_cond"], B) for B in (1, 3, 5, 8)]
    out += [("test_chunks_of_one_sample_at_every_ring_phase", golden["mol_cond"], 5),
            ("test_rings_in_global_memory", c5, 2), ("test_rings_in_global_memory", c5, 8),
            ("test_config2_width_frames_pushed_in_groups", c2, 8),
            ("test_softmax_dense_feedback_and_dense_initial_input", golden["mulaw_softmax"], 5),
            ("test_gaussian_head_with_per_row_speakers", c3, 8),
            ("test_engine5_and_engine7_streams_called_in_turn", golden["mol_cond"], 8),
            ("test_philox_stream_against_float64_forward", golden["mol_cond"], 8),
            ("test_stream_decoder_over_engine7_stream", golden["mol_cond"], 8),
            ("test_misuse_is_refused_and_nothing_faults", golden["mol_cond"], 8)]
    return out


def library_symbols():
    path = N.LIB_PATH
    if not os.path.exists(path):
        pytest.skip("libwn.so is not built (run __graft_entry__.build())")
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm (binutils) is not installed: the kernel instantiations cannot be listed")
    return subprocess.run([nm, "-C", path], capture_output=True, text=True, check=True).stdout


def test_every_stream_kernel_is_launched_by_a_named_gpu_test(monkeypatch):
    out = library_symbols()
    lib = set(re.findall(r"wn7::wn7_stream_kernel<\d+>", out))
    assert lib, "no engine-7 stream kernel in libwn.so"
    src = open(os.path.join(ROOT, GPU_FILE)).read()
    clear_env(monkeypatch)
    reached = {}
    for test, kw, B in stream_launches():
        assert re.search(r"^def %s\(" % re.escape(test), src, re.M), test
        p = plan_only(kw, B, engine=7)
        assert p["engine"] == 7 and p["poll_warps"] == 0
        reached.setdefault("wn7::wn7_stream_kernel<%d>" % p["batch_tile"], []).append(test)
    assert set(reached) == lib, (sorted(reached), sorted(lib))


def test_config5_rings_are_in_global_memory_for_engine_7(monkeypatch):
    """test_rings_in_global_memory of the GPU file relies on it."""
    clear_env(monkeypatch)
    for B in (2, 8):
        assert plan_only(pv.BASES["cfg5"]["kw"], B, engine=7)["rings_in_smem"] == 0


def test_whole_utterance_engine7_kernels_unchanged():
    out = library_symbols()
    got = set(re.findall(r"wn7::wn7_kernel<\d+, (?:true|false)>", out))
    assert got == {"wn7::wn7_kernel<%d, %s>" % (bt, s) for bt in (1, 2, 4, 8) for s in ("true", "false")}
