# coding: utf-8
"""ctypes binding of libwn.so (include/wn.h) and the in-tree build recipe.

The library is the product; this module only loads it.  There is deliberately no fallback: if
the shared object is missing or cannot be loaded, every entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.path.join(HERE, "libwn.so")
SOURCES = [os.path.join(HERE, "csrc", "wn_host.cu")]
HEADERS = [os.path.join(HERE, "csrc", f) for f in ("wn_plan.h", "wn_kernel.cuh", "wn7_plan.h", "wn7_kernel.cuh", "wn7_kernel_body.cuh",
                                                     "wn7_host.cuh", "wn_aux.cuh",
                                                     "wn_dense.cuh")] + [os.path.join(ROOT, "include", "wn.h")]

WN_ABI_VERSION = 3
WN_INPUT_SCALAR, WN_INPUT_ONEHOT = 0, 1
WN_HEAD_MOL, WN_HEAD_GAUSS, WN_HEAD_SOFTMAX = 0, 1, 2
WN_NOISE_REPLAY, WN_NOISE_PHILOX = 0, 1
WN_FLAG_SOFTMAX, WN_FLAG_QUANTIZE = 1, 2

_f32p = C.POINTER(C.c_float)
_i32p = C.POINTER(C.c_int32)


class wn_config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "abi_version", "layers", "stacks", "residual_channels", "gate_channels", "skip_channels",
        "out_channels", "kernel_size", "cin_channels", "gin_channels", "input_kind", "head_kind",
        "device", "num_ctas", "exchange_copies", "ring_slots", "poll_warps", "engine")] + [("reserved", C.c_int32 * 6)]


class wn_layer_weights(C.Structure):
    _fields_ = [(n, _f32p) for n in ("conv_w", "conv_b", "cond_w", "gcond_w", "out_w", "out_b",
                                     "skip_w", "skip_b")]


class wn_weights(C.Structure):
    _fields_ = [(n, _f32p) for n in ("first_w", "first_b", "last_a_w", "last_a_b", "last_b_w",
                                     "last_b_b")] + [("layers", C.POINTER(wn_layer_weights))]


class wn_generate_args(C.Structure):
    _fields_ = [
        ("B", C.c_int32), ("T", C.c_int32),
        ("c", C.c_void_p), ("c_frames", C.c_void_p), ("n_frames", C.c_int32), ("g", C.c_void_p), ("initial", C.c_void_p),
        ("initial_index", C.c_int32), ("initial_rows", C.c_void_p), ("initial_dense", C.c_void_p),
        ("T_test", C.c_int32),
        ("test_scalar", C.c_void_p), ("test_index", C.c_void_p), ("test_dense", C.c_void_p),
        ("flags", C.c_uint32), ("noise_kind", C.c_int32), ("seed", C.c_uint64),
        ("noise_u1", C.c_void_p), ("noise_u2", C.c_void_p), ("noise_z", C.c_void_p),
        ("noise_e", C.c_void_p),
        ("out_scalar", C.c_void_p), ("out_index", C.c_void_p), ("out_dense", C.c_void_p),
        ("params_out", C.c_void_p), ("stream", C.c_void_p),
        ("philox_row0", C.c_int32),
        ("reserved", C.c_int32 * 7),
    ]


class wn_upsampler(C.Structure):
    _fields_ = [("channels", C.c_int32), ("n_scales", C.c_int32), ("scales", _i32p), ("filters", _f32p),
                ("conv_in_w", _f32p), ("conv_in_ks", C.c_int32), ("indent", C.c_int32), ("reserved", C.c_int32 * 5)]


class wn_stream_open_args(C.Structure):
    _fields_ = [("B", C.c_int32), ("g", C.c_void_p), ("initial", C.c_void_p), ("initial_index", C.c_int32),
                ("initial_rows", C.c_void_p), ("initial_dense", C.c_void_p), ("flags", C.c_uint32),
                ("noise_kind", C.c_int32), ("seed", C.c_uint64), ("philox_row0", C.c_int32), ("stream", C.c_void_p),
                ("engine", C.c_int32), ("reserved", C.c_int32 * 5)]


class wn_stream_chunk(C.Structure):
    _fields_ = [("frame_offset", C.c_int64), ("frames_total", C.c_int64), ("final", C.c_int32),
                ("reserved", C.c_int32 * 5)]

WN_DECODE_RAW, WN_DECODE_MULAW, WN_DECODE_MULAW_QUANTIZE = 0, 1, 2


class wn_plan_info(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "num_ctas", "threads_per_cta", "batch_tile", "rows_y", "rows_x", "rows_skip", "rows_head_a",
        "rows_head_b", "resident_blobs", "ring_slots", "blobs_per_step", "exchange_copies",
        "exchanges_per_step", "rings_in_smem")] + [(n, C.c_int64) for n in (
            "smem_bytes", "layer_blob_bytes", "head_blob_bytes", "packed_bytes_per_cta",
            "weight_bytes_per_step", "flops_per_sample", "streamed_bytes_per_step", "launches",
            "cond_packed_bytes_per_cta", "bias_packed_bytes_per_cta", "num_clusters", "cluster_size",
            "num_passes", "engine", "poll_warps")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "reserved"}


# the structs in wn_struct_sizes order
STRUCTS = (wn_config, wn_weights, wn_generate_args, wn_plan_info, wn_upsampler, wn_stream_open_args, wn_stream_chunk)


class Wn7Pass(C.Structure):
    """Mirror of struct Wn7Pass (csrc/wn7_plan.h): one warp pass = two complete rows x nit k-steps."""
    _fields_ = [("w_off", C.c_int32), ("nit", C.c_int16), ("x_off", C.c_int16), ("idx", C.c_int16),
                ("job", C.c_int8), ("deferred", C.c_int8)]


_NKIND, _NCW = 5, 8


class Wn7Plan(C.Structure):
    """Mirror of struct Wn7Plan (csrc/wn7_plan.h); filled by wn_plan_passes."""
    _fields_ = ([(n, C.c_int32) for n in ("L", "per_stack", "R", "G", "G2", "S", "O", "kw", "C", "gin", "input_kind",
                                          "head_kind", "Kmix")] + [("skip_scale", C.c_float)] +
                [(n, C.c_int32) for n in ("P", "BT", "npw", "my", "mx", "ms", "mo", "xoff", "xin_vals", "NS")] +
                [(n, C.c_int64) for n in ("slot_pairs", "ex_pairs")] +
                [(n, C.c_int32) for n in ("ex_a", "ex_b", "gate_cycles", "backoff_ns")] +
                [("npass", C.c_int32),
                 ("pass_begin", (C.c_int32 * _NCW) * _NKIND), ("pass_count", (C.c_int32 * _NCW) * _NKIND),
                 ("pass_crit", (C.c_int32 * _NCW) * _NKIND), ("has_deferred", C.c_int32 * _NKIND)] +
                [(n, C.c_int32) for n in ("fb_floats", "lb_floats", "tb_floats", "slot_floats")] +
                [("cta_w_floats", C.c_int64)] +
                [(n, C.c_int32) for n in ("nblobs", "nres", "nring", "bo_zb", "bo_xb", "bo_sb", "bo_ha", "bo_hb",
                                          "cta_b_floats", "qA")] +
                [("cta_cw_floats", C.c_int64), ("ring_in_smem", C.c_int32), ("ring_pos_total", C.c_int64)] +
                [(n, C.c_int32) for n in ("sm_bar", "sm_misc", "sm_pass", "sm_ringtab", "sm_xin", "sm_sb", "sm_pre",
                                          "sm_cond", "sm_bias", "sm_skipacc", "sm_xown", "sm_hs", "sm_noise", "sm_in",
                                          "sm_x0w", "sm_ring", "sm_slots", "smem_bytes", "nthreads")])


def plan_passes(cfg, batch=1, num_sms=132, smem=232448):
    """(Wn7Plan, [Wn7Pass]) the planner produces for `cfg` (no GPU needed)."""
    pl = Wn7Plan()
    n = lib().wn_plan_passes(C.byref(cfg), batch, num_sms, smem, C.cast(C.byref(pl), _i32p), C.sizeof(pl) // 4, None, 0)
    if n < 0:
        check(n)
    ps = (Wn7Pass * max(n, 1))()
    n = lib().wn_plan_passes(C.byref(cfg), batch, num_sms, smem, C.cast(C.byref(pl), _i32p), C.sizeof(pl) // 4,
                             C.cast(ps, C.c_void_p), n)
    if n < 0:
        check(n)
    return pl, list(ps)[:n]


# every symbol include/wn.h declares (tests check the .so exports all of them)
EXPORTS = ["wn_abi_version", "wn_struct_sizes", "wn_last_error", "wn_create", "wn_destroy", "wn_load_weights",
           "wn_generate", "wn_sync", "wn_generate_host", "wn_get_plan", "wn_plan_only",
           "wn_pack_cta", "wn_plan_passes", "wn_load_upsampler", "wn_upsample", "wn_decode", "wn_sample_mol", "wn_sample_gauss",
           "wn_stream_open", "wn_stream_generate", "wn_stream_position", "wn_stream_close", "wn_upsample_cone",
           "wn_decode_stream", "wn_forward", "wn_nll"]


# entry points an older build of ABI 3 may lack (bound when present)
OPTIONAL_EXPORTS = ("wn_struct_sizes", "wn_forward", "wn_nll")


def nvcc_command(out=LIB_PATH):
    return ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
            "--shared", "-Xcompiler", "-fPIC", "-o", out] + SOURCES


def needs_build():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(f) > t for f in SOURCES + HEADERS)


def build(force=False, verbose=False):
    """Compile libwn.so in-tree for sm_90a (nvcc cross-compiles without a GPU)."""
    if not force and not needs_build():
        return LIB_PATH
    cmd = nvcc_command()
    if verbose:
        print(" ".join(cmd), file=sys.stderr)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    return LIB_PATH


_lib = None


def lib():
    """Load libwn.so (building it first only if nvcc is available and it is missing).  A library that is
    present is loaded as it is: the tree may be read-only at run time, so rebuilding a stale one is left to
    build()."""
    global _lib
    if _lib is not None:
        return _lib
    alt = os.environ.get("WN_LIB_PATH")      # A/B experiments: load another build of the same ABI as it is
    if alt:
        return _bind(C.CDLL(alt))
    if not os.path.exists(LIB_PATH):
        try:
            build()
        except FileNotFoundError:
            pass
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("libwn.so not found at %s: run `python -c 'import __graft_entry__ as g; "
                           "g.build()'` (needs nvcc). There is no CPU fallback." % LIB_PATH)
    if needs_build():
        import warnings
        warnings.warn("%s is older than its sources under csrc/ and is loaded as it is; run __graft_entry__.build() "
                      "to rebuild it" % LIB_PATH, RuntimeWarning, stacklevel=2)
    return _bind(C.CDLL(LIB_PATH))


def _bind(L):
    global _lib
    L.wn_abi_version.restype = C.c_int32
    L.wn_last_error.restype = C.c_char_p
    L.wn_create.argtypes = [C.POINTER(wn_config), C.POINTER(C.c_void_p)]
    L.wn_destroy.argtypes = [C.c_void_p]
    L.wn_load_weights.argtypes = [C.c_void_p, C.POINTER(wn_weights)]
    L.wn_generate.argtypes = [C.c_void_p, C.POINTER(wn_generate_args)]
    L.wn_generate_host.argtypes = [C.c_void_p, C.POINTER(wn_generate_args)]
    L.wn_sync.argtypes = [C.c_void_p]
    L.wn_get_plan.argtypes = [C.c_void_p, C.c_int32, C.POINTER(wn_plan_info)]
    L.wn_plan_only.argtypes = [C.POINTER(wn_config), C.c_int32, C.c_int32, C.c_int64, C.POINTER(wn_plan_info)]
    L.wn_pack_cta.argtypes = [C.POINTER(wn_config), C.c_int32, C.c_int32, C.c_int64, C.POINTER(wn_weights),
                              C.c_int32, _f32p, C.c_int64]
    L.wn_plan_passes.argtypes = [C.POINTER(wn_config), C.c_int32, C.c_int32, C.c_int64, _i32p, C.c_int32,
                                 C.c_void_p, C.c_int32]
    L.wn_load_upsampler.argtypes = [C.c_void_p, C.POINTER(wn_upsampler)]
    L.wn_upsample.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    L.wn_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_float,
                            C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    L.wn_sample_mol.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p]
    L.wn_sample_gauss.argtypes = L.wn_sample_mol.argtypes
    L.wn_stream_open.argtypes = [C.c_void_p, C.POINTER(wn_stream_open_args), C.POINTER(C.c_void_p)]
    L.wn_stream_generate.argtypes = [C.c_void_p, C.POINTER(wn_generate_args), C.POINTER(wn_stream_chunk)]
    L.wn_stream_position.argtypes = [C.c_void_p]
    L.wn_stream_close.argtypes = [C.c_void_p]
    _i64p = C.POINTER(C.c_int64)
    L.wn_upsample_cone.argtypes = [C.POINTER(wn_upsampler), C.c_int64, C.c_int32, C.c_int64, C.c_int64, _i64p, _i64p,
                                   _i64p]
    L.wn_decode_stream.argtypes = L.wn_decode.argtypes[:-1] + [C.c_void_p, C.c_void_p]
    if hasattr(L, "wn_forward"):           # added to ABI 3 without a version bump: detected by presence
        L.wn_forward.argtypes = [C.c_void_p, C.POINTER(wn_generate_args)]
        L.wn_nll.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                             C.c_float, C.c_void_p, C.c_void_p]
    for n in EXPORTS:
        if n in OPTIONAL_EXPORTS and not hasattr(L, n):
            continue                       # an older build of the same ABI (A/B experiments through WN_LIB_PATH)
        fn = getattr(L, n)
        if n != "wn_last_error":
            fn.restype = C.c_int64 if n == "wn_stream_position" else C.c_int32
    if L.wn_abi_version() != WN_ABI_VERSION:
        raise RuntimeError("libwn.so ABI version mismatch")
    sizes = (C.c_int32 * len(STRUCTS))()
    if hasattr(L, "wn_struct_sizes"):
        L.wn_struct_sizes.argtypes = [C.POINTER(C.c_int32), C.c_int32]
    if hasattr(L, "wn_struct_sizes") and L.wn_struct_sizes(sizes, len(STRUCTS)) == len(STRUCTS):
        mine = [C.sizeof(t) for t in STRUCTS]
        if list(sizes) != mine:
            raise RuntimeError("libwn.so struct layout mismatch: library %s, binding %s" % (list(sizes), mine))
    _lib = L
    return L


class WnError(RuntimeError):
    pass


def check(rc):
    if rc != 0:
        raise WnError("libwn: %s (status %d)" % (lib().wn_last_error().decode("utf-8", "replace"), rc))
