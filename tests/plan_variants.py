# coding: utf-8
"""The plan-variant matrix: model shapes x batch x knob settings that move the synthesis kernel's pipeline without
changing the model -- the weight ring's depth and resident / streamed split, the L2 prefetch distance, history rings in
global memory, exchange replicas and layout, warp order and poll timing, engine 7's polling warps and the batch
tile.  Shared by tests/test_plan_variants_host.py (every entry's plan and the kernel instantiation it launches, without
a GPU) and tests/test_plan_variants.py (every entry on an H100, against the default plan of the same shape and against
float64 forward()).

Every knob is read when a handle is planned, so each entry runs on a handle of its own created under its settings.
An entry is checked bit for bit against the default plan (``bit`` is None) wherever the knob only moves data or
changes timing; ``bit`` holds the reason where the per-element arithmetic or its order changes, and the entry is then
held against float64 forward() alone."""
from shape_cases import full_kw
from test_gpu_parity import FULL

# Base shapes.  T: free-running length, at least twice the largest history-ring delay so that every ring wraps;
# T_tf: teacher-forced length, anchored against float64 forward() (config 5's 1024-step rings are wrapped by the
# free-running runs, which need no host reference).
BASES = {
    # softmax head: 64 blocks, all 13 blobs resident, one-hot feedback
    "cfg1": dict(kw=FULL["cfg1_mulaw256"]["kw"], T=160),
    # config 2 width: 128 blocks, 1 resident blob, 24 streamed through 4 slots, rings in shared memory, variant <4, 2>
    "cfg2": dict(kw=FULL["cfg2_mol24"]["kw"], T=160),
    # global conditioning: 16 resident blobs, 9 streamed through 4 slots, variant <1, 1>
    "cfg3": dict(kw=FULL["cfg3_gauss_spk"]["kw"], T=160),
    # 4 resident blobs, 27 streamed through 4 slots, rings in global memory, variant <2, 2>
    "cfg5": dict(kw=FULL["cfg5_mol30"]["kw"], T=2100, T_tf=256),
    # gate half 640, variant <8, 8>: at a tile of 2 or 4 every blob streams through two slots
    "eg8": dict(kw=dict(full_kw("eg8")), T=96),
    # ragged: kernel size 7, 81 conditioning channels, 33 MoL head rows; largest ring delay 48
    "mol_k11": dict(kw=dict(full_kw("mol_k11")), T=112),
}
for _b in BASES.values():
    _b["kw"] = dict(_b["kw"], dropout=0.0)
    _b["kw"].setdefault("kernel_size", 3)
    _b["kw"].setdefault("cin_channels", -1)
    _b["kw"].setdefault("gin_channels", -1)
    _b.setdefault("T_tf", _b["T"])

# head-output bound against float64 forward(): test_forward.py / shape_cases.py's, 1e-4 for the 512-wide stacks
TOL64 = {"cfg1": 2e-5, "cfg2": 1e-4, "cfg3": 2e-5, "cfg5": 1e-4, "eg8": 1e-4, "mol_k11": 2e-5}

# a stream is cut into chunks of 1, 7 and 64 samples, then the rest
STREAM_SPLIT = (1, 7, 64)
# lengths at which the first L2 prefetch loop covers most of the launch
SHORT_T = (1, 2)

NUM_CTAS_WHY = "the row partition changes, and with it every GEMV's summation order"
TILE1_WHY = ("at a tile of 1 a thread owns pairs of adjacent vector elements, at 2, 4 and 8 every 128th one "
             "(wn_kernel.cuh elem): where a thread holds two or more elements its partial sums differ in the last bits")


class Entry:
    """One matrix entry.  env: knob environment; cfg: wn_config fields; expect: plan fields (wn_plan_info) that must
    hold at every launch of the entry; bit: None, or why the entry is held against float64 alone; short: also run
    at T = 1 and 2 (against the first steps of its own long run); stream: also run as a stream in chunks (engine 5,
    B <= 4), against its own one-shot run; vs_b1: row 0 also equals the default plan at B = 1 bit for bit (every
    element of a row is summed in the same order whatever the tile: the tile is 1, or a thread holds one element
    of each vector)."""

    def __init__(self, id, base, B=1, engine=5, env=None, cfg=None, expect=None, bit=None, short=False, stream=False,
                 vs_b1=False):
        self.id, self.base, self.B, self.engine = id, base, B, engine
        self.env = {k: str(v) for k, v in (env or {}).items()}
        self.cfg = dict(cfg or {})
        self.expect = dict(expect or {})
        self.bit, self.short, self.stream, self.vs_b1 = bit, short, stream, vs_b1

    def __repr__(self):
        return self.id


def _e(*a, **k):
    return Entry(*a, **k)


def _l2pf(base, D, expect, **k):
    return _e("%s_l2pf%d" % (base, D), base, env={"WN_L2_PREFETCH": D}, expect=expect, short=True, stream=True, **k)


_C2 = dict(rings_in_smem=1)          # config 2 at B = 1 by default: 1 resident blob + 4 ring slots, rings in shared memory
_C2S = dict(resident_blobs=1, ring_slots=4, **_C2)

MATRIX = [
    # ---------------- engine 5, config 2 width
    # ring depth (the fit maximum is 5: the default's 4 slots + its 1 resident blob)
    _e("cfg2_ring2_env", "cfg2", env={"WN_RING_SLOTS": 2}, expect=dict(ring_slots=2, resident_blobs=3)),
    _e("cfg2_ring3_env", "cfg2", env={"WN_RING_SLOTS": 3}, expect=dict(ring_slots=3, resident_blobs=2)),
    _e("cfg2_ring5_env", "cfg2", env={"WN_RING_SLOTS": 5}, expect=dict(ring_slots=5, resident_blobs=0)),
    _e("cfg2_ring2_cfg", "cfg2", cfg=dict(ring_slots=2), expect=dict(ring_slots=2, resident_blobs=3)),
    _e("cfg2_ring3_cfg", "cfg2", cfg=dict(ring_slots=3), expect=dict(ring_slots=3, resident_blobs=2), short=True),
    _e("cfg2_ring5_cfg", "cfg2", cfg=dict(ring_slots=5), expect=dict(ring_slots=5, resident_blobs=0)),
    # every blob streamed (25 through 4 slots: the ring phase drifts by one slot per step)
    _e("cfg2_resident0", "cfg2", env={"WN_RESIDENT": 0}, expect=dict(ring_slots=4, resident_blobs=0), stream=True),
    _e("cfg2_ring_gmem", "cfg2", env={"WN_RING_SMEM": 0}, expect=dict(rings_in_smem=0, ring_slots=4), stream=True),
    # L2 prefetch distance: 0, 2, 3, nstream - 1, nstream and above nstream (clamped to it)
    _l2pf("cfg2", 0, _C2S), _l2pf("cfg2", 2, _C2S), _l2pf("cfg2", 3, _C2S), _l2pf("cfg2", 23, _C2S),
    _l2pf("cfg2", 24, _C2S), _l2pf("cfg2", 40, _C2S),
    _e("cfg2_l2persist0", "cfg2", env={"WN_L2_PERSIST": 0}, expect=_C2S),
    _e("cfg2_l2persist1", "cfg2", env={"WN_L2_PERSIST": 1}, expect=_C2S),
    # exchange replicas: 2, 4 and the cap (64 finaliser threads / 4 items per block)
    _e("cfg2_ncopy2_env", "cfg2", env={"WN_NCOPY": 2}, expect=dict(exchange_copies=2)),
    _e("cfg2_ncopy16_env", "cfg2", env={"WN_NCOPY": 16}, expect=dict(exchange_copies=16)),
    _e("cfg2_ncopy4_cfg", "cfg2", cfg=dict(exchange_copies=4), expect=dict(exchange_copies=4)),
    _e("cfg2_ncopy16_cfg", "cfg2", cfg=dict(exchange_copies=16), expect=dict(exchange_copies=16)),
    _e("cfg2_warp_reverse", "cfg2", env={"WN_WARP_REVERSE": 1}, expect=_C2S),
    _e("cfg2_gate_cycles", "cfg2", env={"WN_GATE_CYCLES": 3000}, expect=_C2S),
    # block count: 64; 100 = 3 gate rows per block (a half-filled quad), no resident blob, 3 ring slots
    _e("cfg2_ctas64", "cfg2", env={"WN_NUM_CTAS": 64}, expect=dict(num_ctas=64), bit=NUM_CTAS_WHY),
    _e("cfg2_ctas100", "cfg2", env={"WN_NUM_CTAS": 100},
       expect=dict(num_ctas=100, rows_y=3, resident_blobs=0, ring_slots=3), bit=NUM_CTAS_WHY),
    # batch tile at B = 8: 8 launches of 1, 4 of 2, one of 8 (all 25 blobs streamed, rings in global memory); the
    # default runs 2 of 4.  Tiles of 2, 4 and 8 give the same bits; a tile of 1 equals B = 1 run alone
    _e("cfg2_tile1", "cfg2", B=8, env={"WN_MAX_TILE": 1}, expect=dict(batch_tile=1), bit=TILE1_WHY, vs_b1=True),
    _e("cfg2_tile2", "cfg2", B=8, env={"WN_MAX_TILE": 2}, expect=dict(batch_tile=2)),
    _e("cfg2_tile8", "cfg2", B=8, env={"WN_MAX_TILE": 8},
       expect=dict(batch_tile=8, resident_blobs=0, rings_in_smem=0)),
    # streams at tiles of 2 and 4
    _e("cfg2_b2_ring3", "cfg2", B=2, env={"WN_RING_SLOTS": 3}, expect=dict(batch_tile=2, ring_slots=3),
       short=True, stream=True),
    _e("cfg2_b4_l2pf2", "cfg2", B=4, env={"WN_L2_PREFETCH": 2}, expect=dict(batch_tile=4), stream=True),

    # ---------------- engine 5, config 3 (global conditioning)
    _e("cfg3_resident15", "cfg3", env={"WN_RESIDENT": 15}, expect=dict(resident_blobs=15, ring_slots=4),
       stream=True),
    _e("cfg3_ring3", "cfg3", env={"WN_RING_SLOTS": 3}, expect=dict(resident_blobs=17, ring_slots=3)),
    _l2pf("cfg3", 3, dict(resident_blobs=16, ring_slots=4)),
    _e("cfg3_b2_ncopy2", "cfg3", B=2, env={"WN_NCOPY": 2}, expect=dict(batch_tile=2, exchange_copies=2),
       stream=True),

    # ---------------- engine 5, config 5 (rings in global memory)
    _e("cfg5_ring2", "cfg5", env={"WN_RING_SLOTS": 2}, expect=dict(ring_slots=2, resident_blobs=6)),
    _e("cfg5_resident0", "cfg5", env={"WN_RESIDENT": 0}, expect=dict(ring_slots=4, resident_blobs=0)),
    _l2pf("cfg5", 2, dict(ring_slots=4, resident_blobs=4, rings_in_smem=0)),
    _e("cfg5_b2_ring3", "cfg5", B=2, env={"WN_RING_SLOTS": 3}, expect=dict(batch_tile=2, ring_slots=3),
       stream=True),
    _e("cfg5_tile8", "cfg5", B=8, env={"WN_MAX_TILE": 8}, expect=dict(batch_tile=8)),

    # ---------------- engine 5, gate half 640
    _e("eg8_b3_l2pf3", "eg8", B=3, env={"WN_L2_PREFETCH": 3}, expect=dict(batch_tile=4, resident_blobs=0,
                                                                           ring_slots=2), short=True, stream=True),
    _e("eg8_b4_warp_reverse", "eg8", B=4, env={"WN_WARP_REVERSE": 1}, expect=dict(resident_blobs=0, ring_slots=2)),
    _e("eg8_b2_warp_reverse", "eg8", B=2, env={"WN_WARP_REVERSE": 1}, expect=dict(batch_tile=2, resident_blobs=3),
       stream=True),
    _e("eg8_tile8", "eg8", B=8, env={"WN_MAX_TILE": 8}, expect=dict(batch_tile=8)),

    # ---------------- engine 5, ragged rows: 7 blocks divide none of the vectors.  Each block is sized for 4 gate
    # pairs (RA = 8), 3 residual, 4 skip and 5 head rows; gate 26 = 5 x 4 + 2 x 3, residual 18 = 4 x 3 + 3 x 2,
    # skip 22 = 4 + 6 x 3, head 33 = 5 x 5 + 2 x 4
    _e("mol_k11_ctas7", "mol_k11", env={"WN_NUM_CTAS": 7},
       expect=dict(num_ctas=7, rows_y=4, rows_x=3, rows_skip=4, rows_head_b=5), bit=NUM_CTAS_WHY),

    # ---------------- engine 5, softmax head: replicas, layout, warp order
    _e("cfg1_ncopy4_env", "cfg1", env={"WN_NCOPY": 4}, expect=dict(exchange_copies=4, resident_blobs=13)),
    _e("cfg1_ncopy16_env", "cfg1", env={"WN_NCOPY": 16}, expect=dict(exchange_copies=16)),
    _e("cfg1_ncopy2_cfg", "cfg1", cfg=dict(exchange_copies=2), expect=dict(exchange_copies=2)),
    _e("cfg1_xc_layout", "cfg1", env={"WN_XC_SHIFT": 2, "WN_XSTRIDE": 32}, stream=True),
    _e("cfg1_warp_reverse", "cfg1", env={"WN_WARP_REVERSE": 1}),
    _e("cfg1_gate_cycles", "cfg1", env={"WN_GATE_CYCLES": 3000}),
    # R = G/2 = 64: a thread holds one element of each vector at every tile, so row 0 equals B = 1 run alone
    _e("cfg1_tile8", "cfg1", B=8, env={"WN_MAX_TILE": 8}, expect=dict(batch_tile=8), vs_b1=True),
]

# ---------------- engine 7: polling warps 2, 4, 8 at every batch tile, set through the field and the environment
for _i, (_B, _npw) in enumerate([(B, n) for B in (1, 2, 4, 8) for n in (2, 4, 8)]):
    _via_cfg = _i % 2 == 0
    MATRIX.append(_e("e7_cfg2_b%d_poll%d_%s" % (_B, _npw, "cfg" if _via_cfg else "env"), "cfg2", B=_B, engine=7,
                     cfg=dict(poll_warps=_npw) if _via_cfg else None,
                     env=None if _via_cfg else {"WN_POLL_WARPS": _npw},
                     expect=dict(poll_warps=_npw, batch_tile=_B)))
MATRIX += [
    _e("e7_cfg2_spread0", "cfg2", engine=7, env={"WN_EX_SPREAD": 0}),
    _e("e7_cfg2_spread2", "cfg2", engine=7, env={"WN_EX_SPREAD": 2}),
    _e("e7_cfg2_spread3", "cfg2", engine=7, env={"WN_EX_SPREAD": 3}),
    _e("e7_cfg2_defer_gate0", "cfg2", engine=7, env={"WN_DEFER_GATE": 0}),
    _e("e7_cfg2_warp_reverse0", "cfg2", engine=7, env={"WN_WARP_REVERSE": 0}),
    _e("e7_cfg2_backoff", "cfg2", engine=7, env={"WN_BACKOFF_NS": 300}),
    _e("e7_cfg2_poll4_backoff", "cfg2", engine=7, env={"WN_POLL_WARPS": 4, "WN_BACKOFF_NS": 300},
       expect=dict(poll_warps=4)),
    _e("e7_cfg2_poll4_gate_cycles", "cfg2", engine=7, env={"WN_POLL_WARPS": 4, "WN_GATE_CYCLES": 3000},
       expect=dict(poll_warps=4)),
    _e("e7_cfg2_ring3", "cfg2", engine=7, env={"WN_RING_SLOTS": 3}, expect=dict(ring_slots=3)),
    _e("e7_cfg2_ring2_cfg", "cfg2", engine=7, cfg=dict(ring_slots=2), expect=dict(ring_slots=2)),
    _e("e7_cfg2_resident0", "cfg2", engine=7, env={"WN_RESIDENT": 0}, expect=dict(resident_blobs=0)),
    _e("e7_cfg2_ring_gmem", "cfg2", engine=7, env={"WN_RING_SMEM": 0}, expect=dict(rings_in_smem=0)),
    _e("e7_cfg2_ctas100", "cfg2", engine=7, env={"WN_NUM_CTAS": 100}, expect=dict(num_ctas=100), bit=NUM_CTAS_WHY),
    _e("e7_cfg1_poll4", "cfg1", engine=7, cfg=dict(poll_warps=4), expect=dict(poll_warps=4)),
    _e("e7_cfg1_b4_poll2", "cfg1", B=4, engine=7, env={"WN_POLL_WARPS": 2}, expect=dict(poll_warps=2, batch_tile=4)),
    _e("e7_cfg3_poll8", "cfg3", engine=7, env={"WN_POLL_WARPS": 8}, expect=dict(poll_warps=8)),
]

BY_ID = {e.id: e for e in MATRIX}
assert len(BY_ID) == len(MATRIX), "duplicate matrix ids"

def _golden_kw(name):
    from helpers import GoldenCase
    kw = dict(GoldenCase(name).kw)
    kw.setdefault("kernel_size", 3)
    kw.setdefault("cin_channels", -1)
    kw.setdefault("gin_channels", -1)
    return kw


def existing_launches():
    """Kernel instantiations that tests outside this matrix already launch (they are not run again here): (test id,
    model keywords, B, engine, stream, env) of each test's launches.  The host test plans them to confirm."""
    mol = _golden_kw("mol_cond")
    eg8 = dict(full_kw("eg8"))
    c2, c5 = BASES["cfg2"]["kw"], BASES["cfg5"]["kw"]
    out = []
    for B in (1, 2, 3, 8):
        for eng in (5, 7):
            out.append(("tests/test_gpu_parity.py::test_batch_tiles_and_chunks[%d-%d]" % (eng, B), mol, B, eng, False,
                        {}))
    out += [
        ("tests/test_gpu_parity.py::test_config2_width_batch_tiles_against_oracle[5-4]", c2, 4, 5, False, {}),
        ("tests/test_shape_coverage.py::test_teacher_forced_head_outputs[5-eg8-1]", eg8, 1, 5, False, {}),
        ("tests/test_shape_coverage.py::test_chunked_equals_one_shot[eg8-1-replay]", eg8, 1, 5, True, {}),
        ("tests/test_shape_coverage.py::test_chunked_equals_one_shot[eg8-3-replay]", eg8, 3, 5, True, {}),
        ("tests/test_streaming.py::test_golden_cases_chunked_equal_one_shot[mol_cond-1-replay]", mol, 1, 5, True, {}),
        ("tests/test_streaming.py::test_golden_cases_chunked_equal_one_shot[mol_cond-3-replay]", mol, 3, 5, True, {}),
        ("tests/test_streaming.py::test_rings_in_global_memory[1]", c5, 1, 5, True, {}),
        ("tests/test_streaming.py::test_rings_in_global_memory[3]", c5, 3, 5, True, {}),
    ]
    return out


def chunks(B, tile):
    """Batch sizes of the launches wn_generate makes for B utterances at batch tile `tile`."""
    return [min(tile, B - b0) for b0 in range(0, B, tile)]


def efor(K):
    """Elements per thread of a 128-thread group for a vector of K (wn_host.cu launch_chunk)."""
    return 1 if K <= 128 else (2 if K <= 256 else (4 if K <= 512 else 8))


def variant(R, G2):
    er, eg = efor(R), efor(G2)
    if er == 1 and eg == 1:
        return 1, 1
    if er <= 2 and eg <= 2:
        return 2, 2
    if er <= 4 and eg <= 2:
        return 4, 2
    return 8, 8


def kernel_name(kw, plan, engine, stream):
    """The kernel instantiation a launch with this plan takes, as `nm -C` spells its host stub."""
    if engine == 7:
        return "wn7::wn7_kernel<%d, %s>" % (plan["batch_tile"], "true" if plan["poll_warps"] == 0 else "false")
    er, eg = variant(kw["residual_channels"], kw["gate_channels"] // 2)
    return "wn::wn_persistent_kernel<%d, %d, %d, %s>" % (plan["batch_tile"], er, eg, "true" if stream else "false")


def max_tile(env, engine):
    return max(1, min(8, int(env.get("WN_MAX_TILE", 8 if engine == 7 else 4))))


def make_module(base):
    """The seeded CPU module of a base shape (eval mode), built as full_case / shape_cases.make_module build it."""
    if base in ("eg8", "mol_k11"):
        from shape_cases import make_module as shape_module
        return shape_module(base)
    from test_gpu_parity import full_case
    name = {"cfg1": "cfg1_mulaw256", "cfg2": "cfg2_mol24", "cfg3": "cfg3_gauss_spk", "cfg5": "cfg5_mol30"}[base]
    return full_case(name)[0]


def path_config(base):
    from shape_cases import path_config as pc
    return pc(BASES[base]["kw"])
