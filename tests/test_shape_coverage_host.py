# coding: utf-8
"""The model shapes of tests/shape_cases.py without a GPU:
  - the planner's numbers for each case, so that every GPU case provably reaches the code its comment names (a
    partly filled older-tap quad, no rings, one blob to the tail, streamed weight slots, rings in global memory), and
    the two refusals come back as clean statuses with their messages;
  - the packed per-block images replayed by the independent interpreters of tests/test_host_packing.py (engine 5)
    and tests/test_host_packing_v7.py (engine 7) reproduce the oracle's teacher-forced head outputs;
  - the oracle against the module's batch forward() in float64.  The golden vectors pin the oracle to the reference
    at kernel_size 3 only: this is what makes it a valid yardstick for the other kernel sizes and shapes."""
import ctypes as C

import numpy as np
import pytest

import test_host_packing as hp5
import test_host_packing_v7 as hp7
from shape_cases import NAMES, ShapeCase, full_kw, max_delay
from wavenet_vocoder_b200 import _native as N

REPLAY_TOL = 2e-5
ORACLE64_TOL = 5e-6          # fp32 oracle against float64: observed <= 1e-6 on every case
T_HOST = 40


def cdiv(a, b):
    return -(-a // b)


def cfg_of(name, num_ctas=0):
    return hp5.cfg_for(ShapeKw(name), num_ctas=num_ctas)


class ShapeKw:
    """Just enough of a case for cfg_for."""

    def __init__(self, name):
        self.kw = full_kw(name)


def plan_status(cfg, batch):
    info = N.wn_plan_info()
    rc = N.lib().wn_plan_only(C.byref(cfg), batch, hp5.NSM, hp5.SMEM, C.byref(info))
    return rc, (info.as_dict() if rc == 0 else N.lib().wn_last_error().decode())


# what each case must reach, by batch: the planner's numbers
EXPECT = {
    "k1": {1: dict(num_ctas=32)},
    "k2": {1: dict(num_ctas=32)},
    "k4_softmax": {1: dict(num_ctas=32)},
    "k8_global": {1: dict(num_ctas=64, rings_in_smem=0), 4: dict(num_ctas=64, rings_in_smem=0)},
    "L1": {1: dict(num_ctas=32, blobs_per_step=2)},
    "dil1": {1: dict(num_ctas=32)},
    "eg8": {1: dict(num_ctas=128, resident_blobs=3, ring_slots=0),
            4: dict(num_ctas=128, resident_blobs=0, ring_slots=2)},
    "wide_rs": {1: dict(num_ctas=128)},
    "mol_k34": {1: dict(num_ctas=32)},
    "softmax_wide": {1: dict(num_ctas=64), 4: dict(num_ctas=64)},
    "gauss3_r6": {1: dict(num_ctas=6, rows_x=1, rows_skip=2, rows_head_b=1)},
    "mol_k1": {1: dict(num_ctas=10, rows_x=1, rows_skip=2, rows_head_b=1)},
    "mol_k11": {1: dict(num_ctas=26, rows_x=1, rows_skip=1, rows_head_b=2)},
    "softmax_255": {1: dict(num_ctas=18, rows_x=2, rows_skip=2, rows_head_b=15)},
}
RAGGED = ("gauss3_r6", "mol_k1", "mol_k11", "softmax_255")
# a block count that divides none of the gate half, residual, skip and head (gauss3_r6 has 6 gate pairs, so at most
# 6 blocks)
RAGGED_CTAS = {"gauss3_r6": 4, "mol_k1": 4, "mol_k11": 7, "softmax_255": 7}


def ragged(n, P):
    """n rows over P blocks: the planner sizes every block for ceil(n / P) rows (rows_*), and unless P divides n some
    blocks own fewer (wn_part), so their row quads are partly filled, or none."""
    return n != P * cdiv(n, P)


@pytest.mark.parametrize("name", NAMES)
def test_plan_reaches_what_the_case_is_for(name, monkeypatch):
    monkeypatch.setenv("WN_ENGINE", "5")
    kw = full_kw(name)
    cfg = cfg_of(name)
    L, G2, R, S, O, kwid = kw["layers"], kw["gate_channels"] // 2, kw["residual_channels"], kw["skip_out_channels"], \
        kw["out_channels"], kw["kernel_size"]
    for batch in (1, 2, 3, 4):
        rc, p = plan_status(cfg, batch)
        if name == "wide_rs" and batch > 2:            # a tile of 4
            assert rc == -1 and "shared memory too small for two weight slots" in p, p
            continue
        assert rc == 0, p
        P = p["num_ctas"]
        assert p["exchanges_per_step"] == L + 3 and p["blobs_per_step"] == L + 1
        assert (p["rows_y"], p["rows_x"], p["rows_skip"], p["rows_head_a"], p["rows_head_b"]) == \
            (cdiv(G2, P), cdiv(R, P), cdiv(S, P), cdiv(S, P), cdiv(O, P))
        assert p["smem_bytes"] <= hp5.SMEM
        assert p["resident_blobs"] + p["ring_slots"] >= min(L + 1, 2)
        for k, v in EXPECT[name].get(batch, dict(num_ctas=EXPECT[name][1]["num_ctas"])).items():
            assert p[k] == v, (name, batch, k, p[k], v)
        # the older-tap group: (kw-1) * RA rows packed in quads of 4
        rows_d = (kwid - 1) * 2 * p["rows_y"]
        if name == "k1":
            assert rows_d == 0
        elif name == "k2":
            assert rows_d == 2                       # one quad, half filled
        elif name == "k4_softmax":
            assert rows_d == 6                       # two quads, the second half filled
        elif name == "k8_global":
            assert rows_d == 14 and max_delay(kw) == 3584
        elif name == "gauss3_r6":
            assert rows_d == 8                       # two full quads
        elif name == "mol_k11":
            assert rows_d == 12                      # three full quads
        elif name == "softmax_255":
            assert rows_d == 10                      # three quads, the third half filled
        if name in RAGGED:
            # some blocks own fewer rows than the plan's per-block share, or none
            assert any(ragged(n, P) for n in (R, S, O)), (name, P)
            # residual, gate half and skip of 2 mod 4, and an odd head
            assert (R % 4, G2 % 4, S % 4, O % 2) == (2, 2, 2, 1), name
    if name in ("softmax_wide", "softmax_255"):
        rc, msg = plan_status(cfg, 8)
        assert rc == -1 and "too many rows per block for this batch tile" in msg, msg
    if name == "softmax_255":
        # 15 head rows per block: 60 (row, utterance) items at a tile of 4, just under the 64 a block finalises
        rc, p = plan_status(cfg, 4)
        assert rc == 0 and p["batch_tile"] == 4 and p["rows_head_b"] * 4 == 60, p
    if name == "eg8":
        # at a tile of 4 nothing is resident: every blob goes through the two streamed slots each step
        rc, p = plan_status(cfg, 4)
        assert p["streamed_bytes_per_step"] > 0


_CASE_CACHE = {}


def host_case(name):
    if name not in _CASE_CACHE:
        _CASE_CACHE[name] = ShapeCase(name, B=1, T=T_HOST)
    return _CASE_CACHE[name]


def replay_ctas(name):
    """Block counts to replay the packed image at: the default; 5 where the default is 32; for the ragged shapes, a
    count at which every vector is ragged."""
    rc, p = plan_status(cfg_of(name), 1)
    assert rc == 0, p
    out = [p["num_ctas"]]
    extra = RAGGED_CTAS.get(name, 5 if out[0] == 32 else None)
    if extra is not None:
        rc, msg = plan_status(cfg_of(name, num_ctas=extra), 1)
        assert rc == 0, (name, extra, msg)
        out.append(extra)
    return out


@pytest.mark.parametrize("name", NAMES)
def test_engine5_packed_image_replays_oracle(name, monkeypatch):
    monkeypatch.setenv("WN_ENGINE", "5")
    sc = host_case(name)
    Ps = replay_ctas(name)
    if EXPECT[name][1]["num_ctas"] == 32:
        assert 5 in Ps
    if name in RAGGED:
        kw = full_kw(name)
        P = RAGGED_CTAS[name]
        assert P in Ps and all(ragged(kw[k] // (2 if k == "gate_channels" else 1), P) for k in (
            "gate_channels", "residual_channels", "skip_out_channels", "out_channels")), (name, P)
    for P in Ps:
        got = hp5.PackedModel(sc, P).run_teacher_forced(0)
        err = float(np.abs(got - sc.arr["params_tf"][0]).max())
        assert err <= REPLAY_TOL, (name, P, err)


@pytest.mark.parametrize("name", NAMES)
def test_engine7_packed_image_replays_oracle(name, monkeypatch):
    monkeypatch.setenv("WN_ENGINE", "7")
    rc, p = plan_status(cfg_of(name), 1)
    if rc != 0:
        pytest.skip("engine 7 does not plan %s: %s" % (name, p))
    sc = host_case(name)
    for P in replay_ctas(name):
        got = hp7.PackedModel(sc, P).run_teacher_forced(0)
        err = float(np.abs(got - sc.arr["params_tf"][0]).max())
        assert err <= REPLAY_TOL, (name, P, err)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_float64_batch_forward(name):
    """Long enough that the oldest tap of the most dilated layer reads a real input, not the zero history."""
    D = max_delay(full_kw(name))
    sc = ShapeCase(name, B=2, T=max(48, D + 200 if D > 1000 else 2 * D + 8))
    ref = sc.forward64().numpy()
    got = sc.arr["params_tf"]
    assert got.shape == ref.shape
    err = float(np.abs(got.astype(np.float64) - ref).max())
    print("%s: oracle vs float64 forward() max abs err %.3g" % (name, err))
    assert err <= ORACLE64_TOL, err
