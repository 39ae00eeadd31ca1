// wn_host.cu — libwn.so: planner, weight packer and the C ABI declared in include/wn.h.
// Built for sm_90a only:  nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo ...
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/wn.h"
#include "wn_plan.h"
#include "wn_kernel.cuh"
#include "wn7_plan.h"
#include "wn7_kernel.cuh"
#include "wn_aux.cuh"
#include "wn_dense.cuh"

// ------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------
static thread_local std::string g_err;
static int32_t fail(int32_t code, const std::string& msg) {
    g_err = msg;
    return code;
}
#define CUDA_TRY(expr)                                                                          \
    do {                                                                                        \
        cudaError_t e_ = (expr);                                                                \
        if (e_ != cudaSuccess) {                                                                \
            return fail(WN_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_));       \
        }                                                                                       \
    } while (0)

// restores the caller's current CUDA device on scope exit (the library must not change it as a side effect)
struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        if (prev != dev) cudaSetDevice(dev); else prev = -1;
    }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

static int env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return (v && *v) ? atoi(v) : dflt;
}

// ------------------------------------------------------------------------------------------
// planner (pure host arithmetic; exercised without a GPU through wn_plan_only / wn_pack_cta)
// ------------------------------------------------------------------------------------------
static int align_up(long long v, int a) { return (int)(((v + a - 1) / a) * a); }

static int32_t build_plan(const wn_config& c, int batch, int num_sms, long long smem_cap, WnPlan& pl,
                          std::vector<int>& ringtab) {
    memset(&pl, 0, sizeof(pl));
    // version 3 only added entry points: a version-2 caller's structs are the same
    if (c.abi_version != WN_ABI_VERSION && c.abi_version != 2) return fail(WN_ERR_INVALID, "wn_config.abi_version mismatch");
    if (c.layers < 1 || c.stacks < 1 || c.layers % c.stacks != 0)
        return fail(WN_ERR_INVALID, "layers must be a positive multiple of stacks (wavenet.py:117)");
    if (c.gate_channels < 2 || (c.gate_channels & 1)) return fail(WN_ERR_INVALID, "gate_channels must be even");
    if (c.kernel_size < 1 || c.kernel_size > 8) return fail(WN_ERR_INVALID, "kernel_size out of range [1,8]");
    if (c.residual_channels < 1 || c.skip_channels < 1 || c.out_channels < 1)
        return fail(WN_ERR_INVALID, "channel counts must be positive");
    const int maxK = WN_MAXE * 128;
    if (c.residual_channels > maxK || c.gate_channels / 2 > maxK || c.skip_channels > maxK || c.out_channels > maxK)
        return fail(WN_ERR_INVALID, "a stage vector exceeds 1024 entries (unsupported shape)");
    if (c.cin_channels < 0 || c.cin_channels > 32 * WN_MAX_CI)
        return fail(WN_ERR_INVALID, "cin_channels must be in [0,128]");
    if (c.gin_channels < 0) return fail(WN_ERR_INVALID, "gin_channels must be >= 0");
    if (c.layers / c.stacks > 20) return fail(WN_ERR_INVALID, "dilation 2^(layers/stacks) too large");
    if (c.input_kind == WN_INPUT_SCALAR) {
        if (c.head_kind == WN_HEAD_MOL) {
            if (c.out_channels % 3 != 0) return fail(WN_ERR_INVALID, "MoL head needs out_channels % 3 == 0 (mixture.py:130)");
        } else if (c.head_kind == WN_HEAD_GAUSS) {
            if (c.out_channels != 2 && c.out_channels % 3 != 0)
                return fail(WN_ERR_INVALID, "Gaussian head needs out_channels == 2 or % 3 == 0 (mixture.py:229-234)");
        } else
            return fail(WN_ERR_INVALID, "scalar input needs a MoL or Gaussian head (wavenet.py:322-330)");
    } else if (c.input_kind == WN_INPUT_ONEHOT) {
        if (c.head_kind != WN_HEAD_SOFTMAX) return fail(WN_ERR_INVALID, "one-hot input needs the softmax head");
    } else
        return fail(WN_ERR_INVALID, "bad input_kind");
    if (batch < 1) return fail(WN_ERR_INVALID, "batch must be >= 1");
    if (num_sms < 1) return fail(WN_ERR_INVALID, "no SMs");

    pl.L = c.layers;
    pl.per_stack = c.layers / c.stacks;
    pl.R = c.residual_channels;
    pl.G = c.gate_channels;
    pl.G2 = c.gate_channels / 2;
    pl.S = c.skip_channels;
    pl.O = c.out_channels;
    pl.kw = c.kernel_size;
    pl.C = c.cin_channels;
    pl.gin = c.gin_channels;
    pl.input_kind = c.input_kind;
    pl.head_kind = c.head_kind;
    pl.Kmix = (c.head_kind == WN_HEAD_SOFTMAX) ? 0 : (c.out_channels == 2 ? 1 : c.out_channels / 3);
    pl.skip_scale = (float)sqrt(1.0 / (double)c.layers);
    pl.BT = batch <= 1 ? 1 : (batch <= 2 ? 2 : (batch <= 4 ? 4 : 8));
    const int BT = pl.BT;

    // ---- how many blocks: every block must own at least one gate pair
    int P = c.num_ctas > 0 ? c.num_ctas : env_int("WN_NUM_CTAS", 0);
    if (P <= 0) {
        const int cap = std::min(num_sms, pl.G2);
        const int per = wn_ceil_div(pl.G2, cap);
        P = wn_ceil_div(pl.G2, per);
    }
    if (P > num_sms) return fail(WN_ERR_INVALID, "num_ctas exceeds the SM count (blocks must be co-resident)");
    if (P > pl.G2) return fail(WN_ERR_INVALID, "num_ctas exceeds gate_channels/2");
    pl.P = P;
    pl.NYm = wn_ceil_div(pl.G2, P);
    pl.NXm = wn_ceil_div(pl.R, P);
    pl.NSm = wn_ceil_div(pl.S, P);
    pl.NAm = wn_ceil_div(pl.S, P);
    pl.NBm = wn_ceil_div(pl.O, P);
    pl.RA = 2 * pl.NYm;
    pl.NQ_A = wn_ceil_div(pl.RA, 4);
    pl.RA4 = 4 * pl.NQ_A;
    pl.NQ_D = wn_ceil_div((pl.kw - 1) * pl.RA, 4);
    pl.NQ_BO = wn_ceil_div(pl.NXm, 4);
    pl.NQ_BS = wn_ceil_div(pl.NSm, 4);
    pl.NQ_HA = wn_ceil_div(pl.NAm, 4);
    pl.NQ_HB = wn_ceil_div(pl.NBm, 4);
    // ---- blobs
    int o = 0;
    pl.fb_Zx = o; o += pl.NQ_A * pl.R * 4;
    pl.fb_zb = o; o += pl.RA4;
    pl.fb_floats = align_up(o, 4);
    o = 0;
    pl.lb_Zy = o; o += pl.NQ_A * pl.G2 * 4;
    pl.lb_Zx = o; o += pl.NQ_A * pl.R * 4;
    pl.lb_Xo = o; o += pl.NQ_BO * pl.G2 * 4;
    pl.lb_Td = o; o += pl.NQ_D * pl.R * 4;
    pl.lb_Sk = o; o += pl.NQ_BS * pl.G2 * 4;
    pl.lb_zb = o; o += pl.RA4;
    pl.lb_xb = o; o += 4 * pl.NQ_BO;
    pl.lb_sb = o; o += 4 * pl.NQ_BS;
    pl.lb_floats = align_up(o, 4);
    o = 0;
    pl.tb_Td = o;  o += pl.NQ_D * pl.R * 4;
    pl.tb_Sk = o;  o += pl.NQ_BS * pl.G2 * 4;
    pl.tb_sb = o;  o += 4 * pl.NQ_BS;
    pl.tb_Ha = o;  o += pl.NQ_HA * pl.S * 4;
    pl.tb_Hab = o; o += 4 * pl.NQ_HA;
    pl.tb_Hb = o;  o += pl.NQ_HB * pl.S * 4;
    pl.tb_Hbb = o; o += 4 * pl.NQ_HB;
    pl.tb_floats = align_up(o, 4);
    pl.slot_floats = align_up(std::max(pl.fb_floats, std::max(pl.L > 1 ? pl.lb_floats : 0, pl.tb_floats)), 32);
    pl.cta_w_floats = (long long)pl.fb_floats + (long long)(pl.L - 1) * pl.lb_floats + pl.tb_floats;
    pl.nblobs = pl.L + 1;
    pl.cta_cw_floats = (long long)pl.L * pl.NQ_A * pl.C * 4;

    // ---- exchange map
    pl.NE = pl.L + 3;
    int nc = c.exchange_copies > 0 ? c.exchange_copies : env_int("WN_NCOPY", 0);
    // every (row, utterance) item of a broadcast is finalised by one thread per replica inside a
    // 64-thread group, so items * replicas <= 64
    const int max_items = std::max(std::max(pl.NYm, pl.NXm), std::max(pl.NSm, std::max(pl.NAm, pl.NBm))) * BT;
    if (max_items > 64) return fail(WN_ERR_INVALID, "too many rows per block for this batch tile (use more blocks)");
    if (nc <= 0) nc = 1;   // scattered replica stores cost more than they save
    nc = std::min(nc, 64 / max_items);
    pl.ncopy = std::max(1, std::min(nc, P));
    if ((pl.G2 & 1) || (pl.R & 1) || (pl.S & 1))
        return fail(WN_ERR_INVALID, "residual, gate/2 and skip channel counts must be even (16-byte exchange loads)");
    pl.ex_yx = 0;
    pl.ex_sk = pl.L * (pl.G2 + pl.R);
    pl.ex_h1 = pl.ex_sk + pl.S;
    pl.ex_h2 = pl.ex_h1 + pl.S;
    pl.ex_elems = pl.ex_h2 + pl.O;
    pl.xc_shift = env_int("WN_XC_SHIFT", 5);          // 32 pairs (256 bytes) per chunk ...
    pl.xstride = env_int("WN_XSTRIDE", WN_XSTRIDE);   // ... 4352 bytes apart; WN_XC_SHIFT=2 WN_XSTRIDE=32 = one sector per 256-byte granule
    pl.copy_stride_pairs = ((((long long)pl.ex_elems * BT) >> pl.xc_shift) + 2) * pl.xstride + 96;

    // ---- history rings: tap k (0 = oldest) is consumed (kw-1-k)*d steps later
    ringtab.assign((size_t)pl.L * std::max(pl.kw - 1, 0) * 2, 0);
    long long pos = 0;
    for (int l = 0; l < pl.L; ++l)
        for (int k = 0; k < pl.kw - 1; ++k) {
            const int D = (pl.kw - 1 - k) * wn_dilation(pl, l);
            ringtab[((size_t)l * (pl.kw - 1) + k) * 2] = (int)pos;
            ringtab[((size_t)l * (pl.kw - 1) + k) * 2 + 1] = D;
            pos += D;
        }
    pl.ring_pos_total = pos;
    const long long ring_bytes = pos * pl.RA4 * BT * 4;

    // ---- shared memory map
    auto layout = [&](bool ring_smem) -> long long {
        long long off = 0;
        auto take = [&](long long bytes, int al) {
            off = ((off + al - 1) / al) * al;
            long long r = off;
            off += bytes;
            return (int)r;
        };
        pl.sm_bar = take((long long)(2 * pl.nblobs + 8) * 8, 16);
        pl.sm_misc = take(16, 16);
        pl.sm_in = take((long long)BT * 8 + (pl.input_kind == WN_INPUT_ONEHOT ? (long long)BT * pl.O * 4 : 0), 16);
        pl.sm_ringtab = take((long long)ringtab.size() / 2 * 3 * 4 + 16, 16);   // (offset, delay, position) per (layer, tap)
        pl.sm_xs = take(2LL * (pl.R + pl.G2) * BT * 4, 16);   // stash of (x, y), double buffered by stage parity
        const int nq1 = std::max(pl.NQ_A + pl.NQ_BO, std::max(pl.NQ_BS, std::max(pl.NQ_HA, pl.NQ_HB)));
        pl.red1_floats = nq1 * 4 * BT * 4 + 4;                // partial sums of the 4 warps of a group
        pl.sm_red1 = take(2LL * pl.red1_floats * 4, 16);
        // + NQ_BO quads that no kernel writes: without them the fit below changes (config 5 at a batch tile of 8 would
        // keep 3 blobs resident instead of 2), and the resident / streamed split is a tuning decision of its own
        pl.red2_floats = (pl.NQ_D + pl.NQ_BS + pl.NQ_BO) * 4 * BT * 4 + 4;
        pl.sm_red2 = take(2LL * pl.red2_floats * 4, 16);      // two buffers each, alternating by stage
        pl.sm_sb = take(2LL * pl.L * pl.RA4 * BT * 4, 16);     // static part + per-step pre-sum table
        pl.sm_cond = take(pl.C > 0 ? 2LL * pl.L * pl.RA4 * BT * 4 : 16, 16);
        pl.sm_skipacc = take((long long)(pl.NSm * BT + 8 * pl.NQ_BS) * 4 + 16, 16);   // running skip sum + 2 bias stashes
        pl.sm_hs = take((long long)pl.O * BT * 4, 16);
        pl.sm_noise = take((long long)BT * (pl.O + 2) * 4, 16);
        pl.sm_first = take(2LL * pl.R * 4, 16);
        pl.sm_ring = take(ring_smem ? ring_bytes : 16, 16);
        pl.sm_slots = take(0, 128);
        return off;
    };
    const long long slot_bytes = (long long)pl.slot_floats * 4;
    const int want_ring_smem = env_int("WN_RING_SMEM", -1);
    bool ring_smem = (want_ring_smem != 0) && ring_bytes <= 96 * 1024;
    long long fixed = layout(ring_smem);
    long long fit = (smem_cap - fixed) / slot_bytes;
    if (ring_smem && want_ring_smem < 0 && fit < std::min<long long>(pl.nblobs, 3)) {
        ring_smem = false;
        fixed = layout(false);
        fit = (smem_cap - fixed) / slot_bytes;
    }
    pl.ring_in_smem = ring_smem ? 1 : 0;
    if (fit >= pl.nblobs) {
        pl.nres = pl.nblobs;
        pl.nring = 0;
    } else {
        if (fit < 2) return fail(WN_ERR_INVALID, "shared memory too small for two weight slots (use more blocks)");
        int nr = c.ring_slots > 0 ? c.ring_slots : env_int("WN_RING_SLOTS", 4);
        nr = (int)std::max<long long>(2, std::min<long long>(nr, fit));
        pl.nring = nr;
        pl.nres = (int)fit - nr;
        const int force_res = env_int("WN_RESIDENT", -1);
        if (force_res >= 0 && force_res < pl.nres) pl.nres = force_res;
    }
    pl.smem_bytes = (int)(pl.sm_slots + (long long)(pl.nres + pl.nring) * slot_bytes);
    if (pl.smem_bytes > smem_cap) return fail(WN_ERR_INVALID, "shared memory map exceeds the per-block limit");
    return WN_OK;
}

// the work of one step, which depends on the model shape only: both kernel organisations report the same numbers
static void fill_work(const wn_config& c, wn_plan_info* out) {
    const int64_t R = c.residual_channels, G = c.gate_channels, G2 = G / 2, S = c.skip_channels, O = c.out_channels;
    const int64_t L = c.layers, kw = c.kernel_size, C = c.cin_channels;
    const int64_t cin0 = (c.input_kind == WN_INPUT_SCALAR) ? 1 : O;
    // SURVEY.md 8(d): MAC = C0*R + L*(G*kw*R + G*C + S*G/2 + R*G/2) + S*S + O*S ; weights = MAC + biases
    const int64_t mac = cin0 * R + L * (G * kw * R + G * C + S * G2 + R * G2) + S * S + O * S;
    const int64_t biases = R + L * (G + S + R) + S + O;
    out->flops_per_sample = 2 * mac;
    out->weight_bytes_per_step = 4 * (mac + biases);
}

static void fill_info(const wn_config& c, const WnPlan& pl, wn_plan_info* out) {
    memset(out, 0, sizeof(*out));
    out->num_ctas = pl.P;
    out->threads_per_cta = WN_NTHREADS;
    out->batch_tile = pl.BT;
    out->rows_y = pl.NYm;
    out->rows_x = pl.NXm;
    out->rows_skip = pl.NSm;
    out->rows_head_a = pl.NAm;
    out->rows_head_b = pl.NBm;
    out->resident_blobs = pl.nres;
    out->ring_slots = pl.nring;
    out->blobs_per_step = pl.nblobs;
    out->exchange_copies = pl.ncopy;
    out->exchanges_per_step = pl.NE;
    out->rings_in_smem = pl.ring_in_smem;
    out->smem_bytes = pl.smem_bytes;
    out->layer_blob_bytes = (int64_t)pl.lb_floats * 4;
    out->head_blob_bytes = (int64_t)pl.tb_floats * 4;
    out->packed_bytes_per_cta = (int64_t)pl.cta_w_floats * 4;
    out->cond_packed_bytes_per_cta = (int64_t)pl.cta_cw_floats * 4;
    out->engine = 5;
    fill_work(c, out);
    int64_t streamed = 0;
    for (int i = pl.nres; i < pl.nblobs; ++i) streamed += wn_blob_floats(pl, i) * 4LL;
    out->streamed_bytes_per_step = streamed * pl.P;
}

// ------------------------------------------------------------------------------------------
// packer
// ------------------------------------------------------------------------------------------
static inline void put_q(float* grp, int K, int rowidx, int k, float v) {
    grp[((size_t)(rowidx >> 2) * K + k) * 4 + (rowidx & 3)] = v;
}

// Host-side folding for the one-broadcast-per-layer schedule (done once per weight upload, fp64):
//   V_l = sqrt(.5) * W_l[:, :, kw-1]                 (l >= 1; modules.py:162 scale moved into the weight)
//   M_l = V_{l+1} . Wo_l          (G x G/2)         (conv1x1_out of layer l folded into layer l+1)
//   zb_l = conv_b_l + V_l . bo_{l-1}
struct Folded {
    std::vector<std::vector<float>> V, M, zb;     // per layer (V[0] is the plain current tap)
};

static void fold_layers(int L, int G, int R, int G2, int kw, const wn_weights& w, Folded& f) {
    const float rs2 = 0.70710678118654752440f;
    f.V.assign(L, {});
    f.M.assign(L, {});
    f.zb.assign(L, {});
    for (int l = 0; l < L; ++l) {
        const wn_layer_weights& lw = w.layers[l];
        f.V[l].resize((size_t)G * R);
        for (int g = 0; g < G; ++g)
            for (int r = 0; r < R; ++r) {
                const float wv = lw.conv_w[(size_t)g * kw * R + (size_t)(kw - 1) * R + r];
                f.V[l][(size_t)g * R + r] = (l == 0) ? wv : wv * rs2;
            }
        f.zb[l].resize(G);
        for (int g = 0; g < G; ++g) f.zb[l][g] = lw.conv_b ? lw.conv_b[g] : 0.f;
        if (l == 0) continue;
        const wn_layer_weights& pw = w.layers[l - 1];
        f.M[l - 1].resize((size_t)G * G2);
        std::vector<double> acc(G2);
        for (int g = 0; g < G; ++g) {
            std::fill(acc.begin(), acc.end(), 0.0);
            double bacc = 0.0;
            const float* vrow = &f.V[l][(size_t)g * R];
            for (int r = 0; r < R; ++r) {
                const double v = vrow[r];
                const float* orow = pw.out_w + (size_t)r * G2;
                for (int j = 0; j < G2; ++j) acc[j] += v * (double)orow[j];
                if (pw.out_b) bacc += v * (double)pw.out_b[r];
            }
            for (int j = 0; j < G2; ++j) f.M[l - 1][(size_t)g * G2 + j] = (float)acc[j];
            f.zb[l][g] = (float)((double)f.zb[l][g] + bacc);
        }
    }
}

// packed image of block `p`: first blob, L-1 layer blobs, tail blob (all zero-padded)
static void pack_cta(const WnPlan& pl, const wn_weights& w, const Folded& f, int p, float* out) {
    memset(out, 0, (size_t)pl.cta_w_floats * sizeof(float));
    int y0, ny, x0, nx, s0, ns, a0, na, b0, nb;
    wn_part(pl.G2, pl.P, p, y0, ny);
    wn_part(pl.R, pl.P, p, x0, nx);
    wn_part(pl.S, pl.P, p, s0, ns);
    wn_part(pl.S, pl.P, p, a0, na);
    wn_part(pl.O, pl.P, p, b0, nb);
    const int R = pl.R, G2 = pl.G2, kw = pl.kw, S = pl.S, L = pl.L;
    // the gate rows this block evaluates: a_j, b_j interleaved (modules.py:138 split)
    auto grow = [&](int rr) { return (rr & 1) ? G2 + y0 + (rr >> 1) : y0 + (rr >> 1); };
    auto pack_taps = [&](float* grp, int layer) {       // older taps of `layer` (conv.py:56-61: col = k*R + r)
        const float* cw = w.layers[layer].conv_w;
        for (int rr = 0; rr < 2 * ny; ++rr)
            for (int tap = 0; tap < kw - 1; ++tap)
                for (int k = 0; k < R; ++k)
                    put_q(grp, R, tap * pl.RA + rr, k, cw[(size_t)grow(rr) * kw * R + (size_t)tap * R + k]);
    };
    auto pack_skip = [&](float* grp, float* bias, int layer) {
        const wn_layer_weights& lw = w.layers[layer];
        for (int r = 0; r < ns; ++r) {
            for (int k = 0; k < G2; ++k) put_q(grp, G2, r, k, lw.skip_w[(size_t)(s0 + r) * G2 + k]);
            bias[r] = lw.skip_b ? lw.skip_b[s0 + r] : 0.f;
        }
    };
    {   // stage 0
        float* blob = out;
        for (int rr = 0; rr < 2 * ny; ++rr) {
            for (int k = 0; k < R; ++k) put_q(blob + pl.fb_Zx, R, rr, k, f.V[0][(size_t)grow(rr) * R + k]);
            blob[pl.fb_zb + rr] = f.zb[0][grow(rr)];
        }
    }
    for (int s = 1; s < L; ++s) {
        float* blob = out + wn_blob_off(pl, s);
        const wn_layer_weights& pw = w.layers[s - 1];
        for (int rr = 0; rr < 2 * ny; ++rr) {
            const int g = grow(rr);
            for (int k = 0; k < G2; ++k) put_q(blob + pl.lb_Zy, G2, rr, k, f.M[s - 1][(size_t)g * G2 + k]);
            for (int k = 0; k < R; ++k) put_q(blob + pl.lb_Zx, R, rr, k, f.V[s][(size_t)g * R + k]);
            blob[pl.lb_zb + rr] = f.zb[s][g];
        }
        for (int r = 0; r < nx; ++r) {
            for (int k = 0; k < G2; ++k) put_q(blob + pl.lb_Xo, G2, r, k, pw.out_w[(size_t)(x0 + r) * G2 + k]);
            blob[pl.lb_xb + r] = pw.out_b ? pw.out_b[x0 + r] : 0.f;
        }
        pack_taps(blob + pl.lb_Td, s - 1);
        pack_skip(blob + pl.lb_Sk, blob + pl.lb_sb, s - 1);
    }
    float* tb = out + wn_blob_off(pl, L);
    pack_taps(tb + pl.tb_Td, L - 1);
    pack_skip(tb + pl.tb_Sk, tb + pl.tb_sb, L - 1);
    for (int r = 0; r < na; ++r) {
        const float* row = w.last_a_w + (size_t)(a0 + r) * S;
        for (int k = 0; k < S; ++k) put_q(tb + pl.tb_Ha, S, r, k, row[k]);
        tb[pl.tb_Hab + r] = w.last_a_b ? w.last_a_b[a0 + r] : 0.f;
    }
    for (int r = 0; r < nb; ++r) {
        const float* row = w.last_b_w + (size_t)(b0 + r) * S;
        for (int k = 0; k < S; ++k) put_q(tb + pl.tb_Hb, S, r, k, row[k]);
        tb[pl.tb_Hbb + r] = w.last_b_b ? w.last_b_b[b0 + r] : 0.f;
    }
}

static void pack_cw_cta(const WnPlan& pl, const wn_weights& w, int p, float* out) {
    if (pl.C <= 0) return;
    memset(out, 0, (size_t)pl.cta_cw_floats * sizeof(float));
    int y0, ny;
    wn_part(pl.G2, pl.P, p, y0, ny);
    for (int l = 0; l < pl.L; ++l) {
        const float* cwm = w.layers[l].cond_w;
        float* grp = out + (size_t)l * pl.NQ_A * pl.C * 4;
        for (int j = 0; j < ny; ++j)
            for (int ab = 0; ab < 2; ++ab) {
                const int rr = 2 * j + ab, grow = ab ? pl.G2 + y0 + j : y0 + j;
                for (int ch = 0; ch < pl.C; ++ch) put_q(grp, pl.C, rr, ch, cwm[(size_t)grow * pl.C + ch]);
            }
    }
}

static int32_t check_weights(const wn_config& c, const wn_weights* w) {
    if (!w || !w->first_w || !w->first_b || !w->last_a_w || !w->last_a_b || !w->last_b_w || !w->last_b_b || !w->layers)
        return fail(WN_ERR_INVALID, "wn_weights: missing tensor");
    for (int l = 0; l < c.layers; ++l) {
        const wn_layer_weights& lw = w->layers[l];
        if (!lw.conv_w || !lw.conv_b || !lw.out_w || !lw.out_b || !lw.skip_w || !lw.skip_b)
            return fail(WN_ERR_INVALID, "wn_weights: missing layer tensor");
        if (c.cin_channels > 0 && !lw.cond_w) return fail(WN_ERR_INVALID, "wn_weights: cond_w required (cin_channels > 0)");
        if (c.gin_channels > 0 && !lw.gcond_w) return fail(WN_ERR_INVALID, "wn_weights: gcond_w required (gin_channels > 0)");
    }
    return WN_OK;
}

#include "wn7_host.cuh"

// which kernel organisation: 5 (default) = critical / deferred warp groups, values polled straight into the registers
// of the threads that use them, quad-major GEMV + butterfly + one group barrier (csrc/wn_kernel.cuh); 7 = the
// alternative: row-pair passes finalised inside the warp, up to 8 utterances per launch (csrc/wn7_kernel.cuh).
// Both are parity-tested.  On an H100 SXM (700 W) 7 is 20 % slower at B = 1 (config 2) and 46 % faster for 8
// utterances (config 4), which it runs in one launch (DESIGN.md 7).
// wn_config.engine: 0 = WN_ENGINE (7, else 5); 5 or 7 = that engine, whatever WN_ENGINE says.
static int32_t engine_choice(const wn_config& c, int* engine) {
    if (c.engine == 0) *engine = env_int("WN_ENGINE", 5) == 7 ? 7 : 5;
    else if (c.engine == 5 || c.engine == 7) *engine = c.engine;
    else return fail(WN_ERR_INVALID, "wn_config.engine must be 0 (WN_ENGINE, else 5), 5 or 7; got " + std::to_string(c.engine));
    return WN_OK;
}

// ------------------------------------------------------------------------------------------
// handle
// ------------------------------------------------------------------------------------------
struct WnHandle {
    wn_config cfg;
    int engine = 7;
    Wn7Plan base7;                // plan for BT=1 (grid, passes and blob layout are batch independent)
    std::vector<Wn7Pass> passes7;
    float* d_bpack = nullptr;
    Wn7Pass* d_passes = nullptr;
    bool attr7_set[12] = {};      // [0, 8): whole utterances (BT x polling warps or not), [8, 12): the stream kernels
    // local-conditioning upsampler (wn_load_upsampler)
    bool have_ups = false;
    wnaux::UpsampleDesc ups;
    int ups_C = 0, ups_ks = 0, ups_total = 1;
    float *d_ups_filters = nullptr, *d_ups_convw = nullptr;
    float* d_cup = nullptr;  size_t cup_bytes = 0;     // (B,T,C) upsampled conditioning
    float* d_hfr = nullptr;  size_t hfr_bytes = 0;     // (B,F',C) frames after conv_in
    bool ups_attr = false;
    int num_sms = 0;
    long long smem_cap = 0;
    bool have_weights = false;
    uint64_t weight_gen = 0;      // bumped by every weight / upsampler upload: an open stream made with older ones stops
    WnPlan base;                  // plan for BT=1 (partition + blob layout are batch independent)
    std::vector<int> ringtab;
    float *d_wpack = nullptr, *d_cwpack = nullptr, *d_wg = nullptr, *d_first_w = nullptr, *d_first_b = nullptr;
    int* d_ringtab = nullptr;
    int* d_err = nullptr;
    uint2* d_xbuf = nullptr;   size_t xbuf_bytes = 0;
    float* d_ring = nullptr;   size_t ring_bytes = 0;
    float* d_gbias = nullptr;  size_t gbias_bytes = 0;
    void* d_scratch = nullptr; size_t scratch_bytes = 0;   // wn_generate_host staging
    long long* d_prof = nullptr; size_t prof_bytes = 0;    // WN_PROF=1 cycle counters
    cudaStream_t last_stream = nullptr;
    bool pending = false;
    int64_t launches = 0;
    bool attr_set[28] = {};       // [0, 16): whole utterances, [16, 28): the stream instantiations
    size_t l2_persist_bytes = 0, l2_window_max = 0;   // persisting-L2 carve-out
    int l2_mode = 0;                                  // WN_L2_PERSIST: 1 = packed weights, 2 = exchange buffer
    size_t l2_bytes = 0, l2_carve_bytes = 0;          // L2 size; the carve-out this handle asked for
    int last_l2_pf = 0;                               // L2 prefetch distance of the last launch (WN_PROF report)
    size_t wpack_bytes = 0;
    float* d_dense = nullptr;  size_t dense_bytes = 0;    // unfolded fp32 matrices of the batch forward (DenseLayout)
    float* d_fwd = nullptr;    size_t fwd_bytes = 0;      // wn_forward activation scratch
};

template <typename T>
static int32_t ensure(T** ptr, size_t* have, size_t need) {
    if (*have >= need && *ptr) return WN_OK;
    if (*ptr) cudaFree(*ptr);
    *ptr = nullptr;
    *have = 0;
    CUDA_TRY(cudaMalloc((void**)ptr, need));
    *have = need;
    return WN_OK;
}

static int max_tile(int engine) { return std::max(1, std::min(8, env_int("WN_MAX_TILE", engine == 7 ? 8 : 4))); }
static int bt_index(int BT) { return BT == 1 ? 0 : BT == 2 ? 1 : BT == 4 ? 2 : 3; }

// One launch of a stream (wn_stream_generate): the stream's state buffer and where the launch starts.
struct StreamCtx {
    float* state;          // rings then feedback (wn_kernel.cuh WnPtrs::state); rings in global memory live in it
    int state_load;        // 0 for the first chunk: zero history, feedback from initial*
    unsigned t_base;       // absolute step of the chunk's first sample
    const float* gbias;    // Wg . g, computed at open (NULL without global conditioning)
};

// How many streamed blobs the weight warp keeps in flight into L2 ahead of its shared-memory ring (wn_kernel.cuh
// tma_loop).  The ring already puts each copy about nring stages ahead of its use; one more blob of lead through L2
// is what measured best on an H100 (DESIGN.md 7: config 2 is 89.0 us/sample at D = 1, 89.6 at 2, 90.7 at 3, 92.6
// at 6 and 102.9 at 8 against 94.4 at 0): prefetched blobs that wait longer in L2 evict each other, the exchange
// and the conditioning weights.  D is capped by the grid-wide blob stages (P blocks x one blob) that fit in the L2
// left once the persisting carve-out (the exchange buffer), history rings kept in global memory, the conditioning
// weights (re-read every step) and a 2 MB margin are taken out; a handle counts on the share of that L2 its grid has
// of the SMs, so the two half-grid handles of generate_concurrent, which run at the same time, split it.
// WN_L2_PREFETCH=<D> overrides it (0: no prefetch).
static int l2_prefetch_distance(const WnHandle* h, const WnPlan& pl) {
    const int nstream = pl.nblobs - pl.nres;
    if (nstream <= 0) return 0;
    const int forced = env_int("WN_L2_PREFETCH", -1);
    if (forced >= 0) return std::min(forced, nstream);
    long long blob = 0;
    for (int i = pl.nres; i < pl.nblobs; ++i) blob = std::max<long long>(blob, wn_blob_floats(pl, i) * 4LL);
    const long long rings = pl.ring_in_smem ? 0 : (long long)pl.P * pl.ring_pos_total * pl.RA4 * pl.BT * 4;
    long long budget = (long long)h->l2_bytes - (long long)h->l2_carve_bytes - rings - (long long)pl.P * pl.cta_cw_floats * 4 -
                       (2LL << 20);
    budget = budget * pl.P / std::max(h->num_sms, pl.P);
    if (budget <= 0) return 0;
    const int lead = 1;
    return (int)std::min<long long>(std::min<long long>(budget / (pl.P * blob), lead), nstream);
}

// The per-call pointers and scalars of a launch of utterances [b0, b0 + Bc) of the call `a`; WnPtrs and Wn7Ptrs name
// them alike.  C: conditioning channels, O: head outputs, K: mixture components.
template <typename Ptrs>
static void set_call_args(Ptrs& pp, const wn_generate_args* a, int b0, int Bc, int C, int O, int K) {
    const int T = a->T, Tt = a->T_test;
    pp.c = a->c ? a->c + (size_t)b0 * T * C : nullptr;
    pp.initial = a->initial ? a->initial + b0 : nullptr;
    pp.initial_dense = a->initial_dense ? a->initial_dense + (size_t)b0 * O : nullptr;
    pp.initial_rows = a->initial_rows ? a->initial_rows + b0 : nullptr;
    pp.test_scalar = a->test_scalar ? a->test_scalar + (size_t)b0 * Tt : nullptr;
    pp.test_index = a->test_index ? a->test_index + (size_t)b0 * Tt : nullptr;
    pp.test_dense = a->test_dense ? a->test_dense + (size_t)b0 * Tt * O : nullptr;
    // noise is (T, Btotal, .): the kernel indexes with the total batch, so shift by the row
    pp.u1 = a->noise_u1 ? a->noise_u1 + (size_t)b0 * K : nullptr;
    pp.u2 = a->noise_u2 ? a->noise_u2 + b0 : nullptr;
    pp.z = a->noise_z ? a->noise_z + b0 : nullptr;
    pp.e = a->noise_e ? a->noise_e + (size_t)b0 * O : nullptr;
    pp.out_scalar = a->out_scalar ? a->out_scalar + (size_t)b0 * T : nullptr;
    pp.out_index = a->out_index ? a->out_index + (size_t)b0 * T : nullptr;
    pp.out_dense = a->out_dense ? a->out_dense + (size_t)b0 * O * T : nullptr;
    pp.params_out = a->params_out ? a->params_out + (size_t)b0 * O * T : nullptr;
    pp.B = Bc;
    pp.Btot = a->B;
    pp.b0 = b0 + a->philox_row0;          // only the Philox counters use it (wn_kernel.cuh fetch_noise)
    pp.T = T;
    pp.T_test = Tt;
    pp.initial_index = a->initial_index < 0 ? 127 : a->initial_index;   // wavenet.py:286
    pp.flags = a->flags;
    pp.noise_kind = a->noise_kind;
    pp.seed = a->seed;
    pp.timeout_cycles = (long long)env_int("WN_TIMEOUT_MS", 2000) * 1500000LL;
}

static int32_t launch_chunk(WnHandle* h, const wn_generate_args* a, int b0, int Bc, cudaStream_t st,
                            const StreamCtx* sc = nullptr) {
    WnPlan pl;
    std::vector<int> rt;
    int32_t rc = build_plan(h->cfg, Bc, h->num_sms, h->smem_cap, pl, rt);
    if (rc) return rc;
    if (pl.P != h->base.P || pl.lb_floats != h->base.lb_floats)
        return fail(WN_ERR_STATE, "plan changed between weight upload and generate");
    pl.l2_pf = h->last_l2_pf = l2_prefetch_distance(h, pl);
    const int BT = pl.BT;
    const wn_config& c = h->cfg;

    // exchange replicas: zeroed every call so stale tags can never match
    const size_t xb = (size_t)pl.ncopy * pl.copy_stride_pairs * sizeof(uint2);
    rc = ensure(&h->d_xbuf, &h->xbuf_bytes, xb);
    if (rc) return rc;
    CUDA_TRY(cudaMemsetAsync(h->d_xbuf, 0, xb, st));
    if (!pl.ring_in_smem && !sc) {         // a stream's global-memory rings are its state buffer (zeroed at open)
        const size_t rb = std::max<size_t>(16, (size_t)pl.P * pl.ring_pos_total * pl.RA4 * BT * sizeof(float));
        rc = ensure(&h->d_ring, &h->ring_bytes, rb);
        if (rc) return rc;
        CUDA_TRY(cudaMemsetAsync(h->d_ring, 0, rb, st));
    }
    WnPtrs pp;
    memset(&pp, 0, sizeof(pp));
    if (sc) {
        pp.state = sc->state;
        pp.state_load = sc->state_load;
        pp.t_base = sc->t_base;
        pp.gbias = sc->gbias;
    } else if (c.gin_channels > 0) {
        if (!a->g) return fail(WN_ERR_INVALID, "g is required (gin_channels > 0), cf. train.py:72-80 sanity_check");
        const size_t gb = (size_t)Bc * pl.L * pl.G * sizeof(float);
        rc = ensure(&h->d_gbias, &h->gbias_bytes, gb);
        if (rc) return rc;
        wn::wn_gbias_kernel<<<dim3(pl.L, Bc), 128, 0, st>>>(h->d_wg, a->g + (size_t)b0 * c.gin_channels, h->d_gbias,
                                                          pl.L, pl.G, c.gin_channels);
        CUDA_TRY(cudaGetLastError());
        h->launches++;
        pp.gbias = h->d_gbias;
    }
    pp.wpack = h->d_wpack;
    pp.cwpack = h->d_cwpack;
    pp.first_w = h->d_first_w;
    pp.first_b = h->d_first_b;
    pp.xbuf = h->d_xbuf;
    pp.ring_g = (sc && !pl.ring_in_smem) ? sc->state : h->d_ring;
    pp.ringtab = h->d_ringtab;
    pp.err = h->d_err;
    set_call_args(pp, a, b0, Bc, pl.C, pl.O, pl.Kmix);
    pp.warp_reverse = env_int("WN_WARP_REVERSE", 0);
    pp.gate_cycles = env_int("WN_GATE_CYCLES", 0);
    pp.prof = nullptr;
    if (env_int("WN_PROF", 0)) {
#ifndef WN_STAGE_PROF
        return fail(WN_ERR_INVALID, "WN_PROF: this libwn.so has no stage counters; scripts/stage_prof.py builds one with "
                                    "-DWN_STAGE_PROF");
#endif
        const size_t pb = (size_t)pl.P * WN_PROF_SLOTS * sizeof(long long);
        rc = ensure(&h->d_prof, &h->prof_bytes, pb);
        if (rc) return rc;
        CUDA_TRY(cudaMemsetAsync(h->d_prof, 0, pb, st));
        pp.prof = h->d_prof;
    }

    void* kargs[2] = {(void*)&pl, (void*)&pp};
    // kernel variants: <batch tile, elements of x per thread, elements of y per thread> (128-thread groups)
    auto efor = [](int K) { return K <= 128 ? 1 : (K <= 256 ? 2 : (K <= 512 ? 4 : 8)); };
    const int er = efor(pl.R), eg = efor(pl.G2);
    const int var = (er == 1 && eg == 1) ? 0 : ((er <= 2 && eg <= 2) ? 1 : ((er <= 4 && eg <= 2) ? 2 : 3));
    const void* fn = nullptr;
    // stream launches take the STREAM instantiations (wn_kernel.cuh Engine); a stream holds at most one tile of 4
#define WN_PICK(BT_, S_)                                                                \
    fn = var == 0 ? (const void*)wn::wn_persistent_kernel<BT_, 1, 1, S_>               \
       : var == 1 ? (const void*)wn::wn_persistent_kernel<BT_, 2, 2, S_>               \
       : var == 2 ? (const void*)wn::wn_persistent_kernel<BT_, 4, 2, S_>               \
                  : (const void*)wn::wn_persistent_kernel<BT_, 8, 8, S_>
    if (sc && BT > 4) return fail(WN_ERR_INVALID, "a stream holds at most 4 utterances");
    switch (BT) {
        case 1: if (sc) WN_PICK(1, true); else WN_PICK(1, false); break;
        case 2: if (sc) WN_PICK(2, true); else WN_PICK(2, false); break;
        case 4: if (sc) WN_PICK(4, true); else WN_PICK(4, false); break;
        default: WN_PICK(8, false); break;
    }
#undef WN_PICK
    const int ai = bt_index(BT) * 4 + var + (sc ? 16 : 0);
    if (!h->attr_set[ai]) {
        CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_cap));
        h->attr_set[ai] = true;
    }
    // cooperative launch: the runtime refuses to start unless all P blocks are co-resident,
    // which the spin-wait exchanges require
    cudaLaunchConfig_t lc;
    memset(&lc, 0, sizeof(lc));
    lc.gridDim = dim3(pl.P);
    lc.blockDim = dim3(WN_NTHREADS);
    lc.dynamicSmemBytes = (size_t)pl.smem_bytes;
    lc.stream = st;
    cudaLaunchAttribute la[2];
    int na = 0;
    la[na].id = cudaLaunchAttributeCooperative;
    la[na].val.cooperative = 1;
    ++na;
    if (h->l2_mode == 1 && h->l2_persist_bytes > 0 && h->wpack_bytes > 0) {
        const size_t win = std::min(h->wpack_bytes, h->l2_window_max);
        la[na].id = cudaLaunchAttributeAccessPolicyWindow;
        la[na].val.accessPolicyWindow.base_ptr = (void*)h->d_wpack;
        la[na].val.accessPolicyWindow.num_bytes = win;
        la[na].val.accessPolicyWindow.hitRatio = (float)std::min(1.0, (double)h->l2_persist_bytes / (double)win);
        la[na].val.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
        la[na].val.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
        ++na;
    } else if (h->l2_mode == 2 && h->l2_persist_bytes > 0) {
        // keep the exchange buffer (a few MB, every line touched once per generated sample) in the persisting part of
        // L2: the 112 MB/sample weight stream otherwise evicts it between two steps
        la[na].id = cudaLaunchAttributeAccessPolicyWindow;
        la[na].val.accessPolicyWindow.base_ptr = (void*)h->d_xbuf;
        la[na].val.accessPolicyWindow.num_bytes = std::min(xb, h->l2_window_max);
        la[na].val.accessPolicyWindow.hitRatio = 1.0f;
        la[na].val.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
        la[na].val.accessPolicyWindow.missProp = cudaAccessPropertyNormal;
        ++na;
    }
    lc.attrs = la;
    lc.numAttrs = na;
    CUDA_TRY(cudaLaunchKernelExC(&lc, fn, kargs));
    h->launches++;
    return WN_OK;
}

static void fill_info7(const wn_config& c, const Wn7Plan& pl, wn_plan_info* out) {
    memset(out, 0, sizeof(*out));
    out->num_ctas = pl.P;
    out->threads_per_cta = pl.nthreads;
    out->batch_tile = pl.BT;
    out->rows_y = pl.my;
    out->rows_x = pl.mx;
    out->rows_skip = pl.ms;
    out->rows_head_a = pl.ms;
    out->rows_head_b = pl.mo;
    out->resident_blobs = pl.nres;
    out->ring_slots = pl.nring;
    out->blobs_per_step = pl.nblobs;
    out->exchange_copies = 1;
    out->exchanges_per_step = pl.NS;
    out->rings_in_smem = pl.ring_in_smem;
    out->smem_bytes = pl.smem_bytes;
    out->layer_blob_bytes = (int64_t)pl.lb_floats * 4;
    out->head_blob_bytes = (int64_t)pl.tb_floats * 4;
    out->packed_bytes_per_cta = (int64_t)pl.cta_w_floats * 4;
    out->cond_packed_bytes_per_cta = (int64_t)pl.cta_cw_floats * 4;
    out->bias_packed_bytes_per_cta = (int64_t)pl.cta_b_floats * 4;
    out->num_clusters = pl.P;
    out->cluster_size = 1;
    out->poll_warps = pl.npw;
    out->num_passes = pl.npass;
    out->engine = 7;
    fill_work(c, out);
    int64_t streamed = 0;
    for (int i = pl.nres; i < pl.nblobs; ++i) streamed += wn7_blob_floats(pl, i) * 4LL;
    out->streamed_bytes_per_step = streamed * pl.P;
}

// c_frames (B,C,F) -> h->d_cup (B,T,C).  A stream passes a window: c_frames starts at utterance frame f_off, level 0
// of the utterance has n0 rows (WNAUX_UNBOUNDED until the last frame is known) and the output starts at sample t_off.
static int32_t run_upsampler(WnHandle* h, const float* c_frames, int B, int F, int T, cudaStream_t st, int f_off = 0,
                             int n0 = -1, int t_off = 0) {
    const int C = h->ups_C;
    const int Fo = F - (h->ups_ks > 0 ? h->ups_ks - 1 : 0);
    if (n0 < 0) n0 = Fo;
    int32_t rc = ensure(&h->d_hfr, &h->hfr_bytes, (size_t)B * Fo * C * sizeof(float));
    if (rc) return rc;
    rc = ensure(&h->d_cup, &h->cup_bytes, (size_t)B * T * C * sizeof(float));
    if (rc) return rc;
    const long long n = (long long)B * Fo * C;
    const int blocks = (int)std::min<long long>((n + 255) / 256, 4096);
    if (h->ups_ks > 0)
        wnaux::conv_in_kernel<<<blocks, 256, 0, st>>>(c_frames, h->d_ups_convw, h->d_hfr, B, C, F, h->ups_ks);
    else
        wnaux::frames_to_fc_kernel<<<blocks, 256, 0, st>>>(c_frames, h->d_hfr, B, C, F);
    CUDA_TRY(cudaGetLastError());
    constexpr int TS = 256;
    const size_t smem = 2ull * (TS / 2 + 8) * C * sizeof(float);
    if (!h->ups_attr) {
        CUDA_TRY(cudaFuncSetAttribute(wnaux::upsample_kernel<TS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        h->ups_attr = true;
    }
    wnaux::upsample_kernel<TS><<<dim3((T + TS - 1) / TS, B), 256, smem, st>>>(h->d_hfr, h->d_ups_filters, h->ups, C, Fo,
                                                                            f_off, n0, t_off, T, h->d_cup);
    CUDA_TRY(cudaGetLastError());
    h->launches += 2;
    return WN_OK;
}

static const void* kernel7_for(int BT, bool self, bool stream) {
    if (stream) {       // wn7_kernel.cuh: streams run on handles whose compute warps poll
        switch (BT) {
            case 1: return (const void*)wn7::wn7_stream_kernel<1>;
            case 2: return (const void*)wn7::wn7_stream_kernel<2>;
            case 4: return (const void*)wn7::wn7_stream_kernel<4>;
            default: return (const void*)wn7::wn7_stream_kernel<8>;
        }
    }
    if (self) {
        switch (BT) {
            case 1: return (const void*)wn7::wn7_kernel<1, true>;
            case 2: return (const void*)wn7::wn7_kernel<2, true>;
            case 4: return (const void*)wn7::wn7_kernel<4, true>;
            default: return (const void*)wn7::wn7_kernel<8, true>;
        }
    }
    switch (BT) {
        case 1: return (const void*)wn7::wn7_kernel<1, false>;
        case 2: return (const void*)wn7::wn7_kernel<2, false>;
        case 4: return (const void*)wn7::wn7_kernel<4, false>;
        default: return (const void*)wn7::wn7_kernel<8, false>;
    }
}

static int32_t prepare_kernel7(WnHandle* h, int BT, bool self, bool stream) {
    const int ai = bt_index(BT) + (stream ? 8 : (self ? 4 : 0));
    if (h->attr7_set[ai]) return WN_OK;
    const void* fn = kernel7_for(BT, self, stream);
    CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_cap));
    h->attr7_set[ai] = true;
    return WN_OK;
}

static int32_t launch_chunk7(WnHandle* h, const wn_generate_args* a, int b0, int Bc, cudaStream_t st,
                             const StreamCtx* sc = nullptr) {
    Wn7Plan pl;
    std::vector<Wn7Pass> passes;
    std::vector<int> rt;
    int32_t rc = build_plan7(h->cfg, Bc, h->num_sms, h->smem_cap, pl, passes, rt);
    if (rc) return rc;
    if (pl.P != h->base7.P || pl.lb_floats != h->base7.lb_floats || pl.npass != h->base7.npass)
        return fail(WN_ERR_STATE, "plan changed between weight upload and generate");
    const int BT = pl.BT;
    const wn_config& c = h->cfg;
    const size_t xb = (size_t)pl.ex_pairs * sizeof(uint2);
    rc = ensure(&h->d_xbuf, &h->xbuf_bytes, xb);
    if (rc) return rc;
    CUDA_TRY(cudaMemsetAsync(h->d_xbuf, 0, xb, st));     // zeroed every call so stale tags can never match
    if (sc && pl.npw != 0) return fail(WN_ERR_INVALID, "an engine-7 stream needs a handle whose compute warps poll");
    if (!pl.ring_in_smem && !sc) {         // a stream's global-memory rings are its state buffer (zeroed at open)
        const size_t rb = std::max<size_t>(16, (size_t)pl.P * pl.ring_pos_total * 4 * pl.qA * BT * sizeof(float));
        rc = ensure(&h->d_ring, &h->ring_bytes, rb);
        if (rc) return rc;
        CUDA_TRY(cudaMemsetAsync(h->d_ring, 0, rb, st));
    }
    Wn7Ptrs pp;
    memset(&pp, 0, sizeof(pp));
    if (sc) {
        pp.state = sc->state;
        pp.state_load = sc->state_load;
        pp.t_base = sc->t_base;
        pp.gbias = sc->gbias;
    } else if (c.gin_channels > 0) {
        if (!a->g) return fail(WN_ERR_INVALID, "g is required (gin_channels > 0), cf. train.py:72-80 sanity_check");
        const size_t gb = (size_t)Bc * pl.L * pl.G * sizeof(float);
        rc = ensure(&h->d_gbias, &h->gbias_bytes, gb);
        if (rc) return rc;
        wn::wn_gbias_kernel<<<dim3(pl.L, Bc), 128, 0, st>>>(h->d_wg, a->g + (size_t)b0 * c.gin_channels, h->d_gbias,
                                                          pl.L, pl.G, c.gin_channels);
        CUDA_TRY(cudaGetLastError());
        h->launches++;
        pp.gbias = h->d_gbias;
    }
    pp.wpack = h->d_wpack;
    pp.cwpack = h->d_cwpack;
    pp.bpack = h->d_bpack;
    pp.passes = h->d_passes;
    pp.warp_reverse = env_int("WN_WARP_REVERSE", 1);
    pp.defer_gate = env_int("WN_DEFER_GATE", 1);
    pp.first_w = h->d_first_w;
    pp.first_b = h->d_first_b;
    pp.xbuf = h->d_xbuf;
    pp.ring_g = (sc && !pl.ring_in_smem) ? sc->state : h->d_ring;
    pp.ringtab = h->d_ringtab;
    pp.err = h->d_err;
    set_call_args(pp, a, b0, Bc, pl.C, pl.O, pl.Kmix);
    pp.prof = nullptr;
    if (env_int("WN_PROF", 0)) {
        const size_t pb = (size_t)pl.P * 16 * sizeof(long long);
        rc = ensure(&h->d_prof, &h->prof_bytes, pb);
        if (rc) return rc;
        CUDA_TRY(cudaMemsetAsync(h->d_prof, 0, pb, st));
        pp.prof = h->d_prof;
    }
    rc = prepare_kernel7(h, BT, pl.npw == 0, sc != nullptr);
    if (rc) return rc;
    void* kargs[2] = {(void*)&pl, (void*)&pp};
    // cooperative launch: the runtime refuses to start unless all P blocks are co-resident, which the
    // spin-wait exchanges require
    cudaLaunchConfig_t lc;
    memset(&lc, 0, sizeof(lc));
    lc.gridDim = dim3(pl.P);
    lc.blockDim = dim3(pl.nthreads);
    lc.dynamicSmemBytes = (size_t)pl.smem_bytes;
    lc.stream = st;
    cudaLaunchAttribute la[2];
    int na = 0;
    la[na].id = cudaLaunchAttributeCooperative;
    la[na].val.cooperative = 1;
    ++na;
    if (h->l2_mode == 2 && h->l2_persist_bytes > 0) {
        la[na].id = cudaLaunchAttributeAccessPolicyWindow;
        la[na].val.accessPolicyWindow.base_ptr = (void*)h->d_xbuf;
        la[na].val.accessPolicyWindow.num_bytes = std::min(xb, h->l2_window_max);
        la[na].val.accessPolicyWindow.hitRatio = 1.0f;
        la[na].val.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
        la[na].val.accessPolicyWindow.missProp = cudaAccessPropertyNormal;
        ++na;
    }
    lc.attrs = la;
    lc.numAttrs = na;
    CUDA_TRY(cudaLaunchKernelExC(&lc, kernel7_for(BT, pl.npw == 0, sc != nullptr), kargs));
    h->launches++;
    return WN_OK;
}

// ------------------------------------------------------------------------------------------
// teacher-forced batch forward (wn_forward): csrc/wn_dense.cuh
// ------------------------------------------------------------------------------------------
// The dense image holds the fp32 matrices as they arrive in wn_weights (row-major M x K), not folded: per layer
// [conv_w | cond_w] (G x kw*R+C), conv_b (G), [out_w ; skip_w] (R+S x G/2), [out_b ; skip_b] (R+S); then last_a_w,
// last_a_b, last_b_w, last_b_b.  Every piece starts at a multiple of 4 floats.
struct DenseLayout {
    size_t gate_w, gate_b, os_w, os_b, per_layer;   // offsets within one layer
    size_t la_w, la_b, lb_w, lb_b, total;            // offsets of the head, total floats
};

static DenseLayout dense_layout(const wn_config& c) {
    auto al = [](size_t v) { return (v + 3) / 4 * 4; };
    const size_t R = c.residual_channels, G = c.gate_channels, G2 = G / 2, S = c.skip_channels, O = c.out_channels;
    const size_t Kg = (size_t)c.kernel_size * R + c.cin_channels;
    DenseLayout d;
    d.gate_w = 0;
    d.gate_b = al(G * Kg);
    d.os_w = d.gate_b + al(G);
    d.os_b = d.os_w + al((R + S) * G2);
    d.per_layer = d.os_b + al(R + S);
    d.la_w = (size_t)c.layers * d.per_layer;
    d.la_b = d.la_w + al(S * S);
    d.lb_w = d.la_b + al(S);
    d.lb_b = d.lb_w + al(O * S);
    d.total = d.lb_b + al(O);
    return d;
}

static void pack_dense(const wn_config& c, const wn_weights& w, std::vector<float>& img) {
    const DenseLayout d = dense_layout(c);
    const size_t R = c.residual_channels, G = c.gate_channels, G2 = G / 2, S = c.skip_channels, O = c.out_channels;
    const size_t kwR = (size_t)c.kernel_size * R, Cc = c.cin_channels, Kg = kwR + Cc;
    img.assign(d.total, 0.f);
    auto put = [&](size_t off, const float* src, size_t n) { memcpy(img.data() + off, src, n * sizeof(float)); };
    for (int l = 0; l < c.layers; ++l) {
        const wn_layer_weights& lw = w.layers[l];
        const size_t base = (size_t)l * d.per_layer;
        for (size_t row = 0; row < G; ++row) {
            put(base + d.gate_w + row * Kg, lw.conv_w + row * kwR, kwR);
            if (Cc) put(base + d.gate_w + row * Kg + kwR, lw.cond_w + row * Cc, Cc);
        }
        put(base + d.gate_b, lw.conv_b, G);
        put(base + d.os_w, lw.out_w, R * G2);
        put(base + d.os_w + R * G2, lw.skip_w, S * G2);
        put(base + d.os_b, lw.out_b, R);
        put(base + d.os_b + R, lw.skip_b, S);
    }
    put(d.la_w, w.last_a_w, S * S);
    put(d.la_b, w.last_a_b, S);
    put(d.lb_w, w.last_b_w, O * S);
    put(d.lb_b, w.last_b_b, O);
}

// the conditioning inputs of a call (c or c_frames, g); window_frames: c_frames is a window of the utterance (a stream
// chunk, checked by the caller), not all of it
static int32_t validate_cond(const WnHandle* h, const wn_generate_args* a, bool window_frames) {
    const wn_config& c = h->cfg;
    if (a->c && a->c_frames) return fail(WN_ERR_INVALID, "give either c (sample rate) or c_frames, not both");
    if (c.cin_channels > 0 && !a->c && !a->c_frames) return fail(WN_ERR_INVALID, "c is required (cin_channels > 0), cf. train.py:82-87");
    if (c.cin_channels == 0 && (a->c || a->c_frames)) return fail(WN_ERR_INVALID, "c given but the model has no local conditioning");
    if (a->c_frames && window_frames) {
        if (!h->have_ups) return fail(WN_ERR_STATE, "c_frames given but no upsampler was loaded (wn_load_upsampler)");
    } else if (a->c_frames) {
        if (!h->have_ups) return fail(WN_ERR_STATE, "c_frames given but no upsampler was loaded (wn_load_upsampler)");
        const long long Fo = (long long)a->n_frames - (h->ups_ks > 0 ? h->ups_ks - 1 : 0);
        if (Fo < 1 || Fo * h->ups_total - 2LL * h->ups.indent != (long long)a->T)
            return fail(WN_ERR_INVALID, "upsampled conditioning length != T (wavenet.py:276)");
    }
    if (c.gin_channels == 0 && a->g) return fail(WN_ERR_INVALID, "g given but the model has no global conditioning");
    return WN_OK;
}

static int32_t validate_forward(const WnHandle* h, const wn_generate_args* a) {
    const wn_config& c = h->cfg;
    if (!a) return fail(WN_ERR_INVALID, "null args");
    if (a->B < 1 || a->T < 1) return fail(WN_ERR_INVALID, "B and T must be >= 1");
    if (a->T_test != a->T) return fail(WN_ERR_INVALID, "wn_forward: T_test must equal T (every step is teacher forced)");
    const int nx = (a->test_scalar != nullptr) + (a->test_index != nullptr) + (a->test_dense != nullptr);
    if (nx != 1) return fail(WN_ERR_INVALID, "wn_forward: give exactly one of test_scalar, test_index, test_dense");
    if (c.input_kind == WN_INPUT_SCALAR && !a->test_scalar)
        return fail(WN_ERR_INVALID, "wn_forward: a scalar-input model takes test_scalar");
    if (c.input_kind == WN_INPUT_ONEHOT && a->test_scalar)
        return fail(WN_ERR_INVALID, "wn_forward: a one-hot-input model takes test_index or test_dense");
    if (a->noise_u1 || a->noise_u2 || a->noise_z || a->noise_e)
        return fail(WN_ERR_INVALID, "wn_forward draws no noise: noise_u1, noise_u2, noise_z and noise_e must be NULL");
    if (a->out_scalar || a->out_index || a->out_dense)
        return fail(WN_ERR_INVALID, "wn_forward writes params_out only: out_scalar, out_index and out_dense must be NULL");
    if (a->initial || a->initial_rows || a->initial_dense)
        return fail(WN_ERR_INVALID, "wn_forward: initial, initial_rows and initial_dense must be NULL (every step is "
                                    "teacher forced)");
    if (!a->params_out) return fail(WN_ERR_INVALID, "wn_forward: params_out required");
    if (a->flags & ~WN_FLAG_SOFTMAX) return fail(WN_ERR_INVALID, "wn_forward: only WN_FLAG_SOFTMAX applies");
    if (c.gin_channels > 0 && !a->g) return fail(WN_ERR_INVALID, "g is required (gin_channels > 0)");
    return validate_cond(h, a, false);
}

// ------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------
extern "C" {

int32_t wn_abi_version(void) { return WN_ABI_VERSION; }
int32_t wn_struct_sizes(int32_t* out, int32_t n) {
    const int32_t v[7] = {(int32_t)sizeof(wn_config), (int32_t)sizeof(wn_weights), (int32_t)sizeof(wn_generate_args),
                          (int32_t)sizeof(wn_plan_info), (int32_t)sizeof(wn_upsampler),
                          (int32_t)sizeof(wn_stream_open_args), (int32_t)sizeof(wn_stream_chunk)};
    int32_t k = 0;
    for (; k < 7 && k < n; ++k) out[k] = v[k];
    return k;
}
const char* wn_last_error(void) { return g_err.c_str(); }

int32_t wn_plan_only(const wn_config* cfg, int32_t batch, int32_t num_sms, int64_t smem_per_cta, wn_plan_info* out) {
    if (!cfg || !out) return fail(WN_ERR_INVALID, "null argument");
    int engine = 5;
    if (int32_t rce = engine_choice(*cfg, &engine)) return rce;
    if (engine == 7) {
        Wn7Plan pl6;
        std::vector<Wn7Pass> ps;
        std::vector<int> rt6;
        int32_t rc6 = build_plan7(*cfg, batch, num_sms, smem_per_cta, pl6, ps, rt6);
        if (rc6) return rc6;
        fill_info7(*cfg, pl6, out);
        return WN_OK;
    }
    WnPlan pl;
    std::vector<int> rt;
    int32_t rc = build_plan(*cfg, batch, num_sms, smem_per_cta, pl, rt);
    if (rc) return rc;
    fill_info(*cfg, pl, out);
    return WN_OK;
}

int32_t wn_plan_passes(const wn_config* cfg, int32_t batch, int32_t num_sms, int64_t smem_per_cta, int32_t* plan_words,
                       int32_t max_plan_words, void* passes, int32_t max_passes) {
    if (!cfg) return fail(WN_ERR_INVALID, "null argument");
    int engine = 5;            // the pass table is engine 7's whichever engine the config picks; a bad value is refused
    if (int32_t rce = engine_choice(*cfg, &engine)) return rce;
    Wn7Plan pl;
    std::vector<Wn7Pass> ps;
    std::vector<int> rt;
    int32_t rc = build_plan7(*cfg, batch, num_sms, smem_per_cta, pl, ps, rt);
    if (rc) return rc;
    if (plan_words) {
        const int n = std::min<int>(max_plan_words, (int)(sizeof(Wn7Plan) / 4));
        memcpy(plan_words, &pl, (size_t)n * 4);
    }
    if (passes) {
        if (max_passes < pl.npass) return fail(WN_ERR_INVALID, "pass buffer too small");
        memcpy(passes, ps.data(), ps.size() * sizeof(Wn7Pass));
    }
    return pl.npass;
}

int32_t wn_pack_cta(const wn_config* cfg, int32_t batch, int32_t num_sms, int64_t smem_per_cta, const wn_weights* w,
                    int32_t cta, float* packed, int64_t packed_floats) {
    if (!cfg || !packed) return fail(WN_ERR_INVALID, "null argument");
    int engine = 5;
    if (int32_t rce = engine_choice(*cfg, &engine)) return rce;
    if (engine == 7) {
        Wn7Plan pl6;
        std::vector<Wn7Pass> ps;
        std::vector<int> rt6;
        int32_t rc6 = build_plan7(*cfg, batch, num_sms, smem_per_cta, pl6, ps, rt6);
        if (rc6) return rc6;
        rc6 = check_weights(*cfg, w);
        if (rc6) return rc6;
        if (cta < 0 || cta >= pl6.P) return fail(WN_ERR_INVALID, "cta out of range");
        if (packed_floats < pl6.cta_w_floats) return fail(WN_ERR_INVALID, "packed buffer too small");
        Folded fo;
        fold_layers(pl6.L, pl6.G, pl6.R, pl6.G2, pl6.kw, *w, fo);
        pack7_cta(pl6, ps, *w, fo, cta, packed);
        long long off = pl6.cta_w_floats;
        if (packed_floats >= off + pl6.cta_cw_floats) {
            pack7_cw(pl6, *w, cta, packed + off);
            off += pl6.cta_cw_floats;
            if (packed_floats >= off + pl6.cta_b_floats) pack7_bias(pl6, *w, fo, cta, packed + off);
        }
        return WN_OK;
    }
    WnPlan pl;
    std::vector<int> rt;
    int32_t rc = build_plan(*cfg, batch, num_sms, smem_per_cta, pl, rt);
    if (rc) return rc;
    rc = check_weights(*cfg, w);
    if (rc) return rc;
    if (cta < 0 || cta >= pl.P) return fail(WN_ERR_INVALID, "cta out of range");
    if (packed_floats < pl.cta_w_floats) return fail(WN_ERR_INVALID, "packed buffer too small");
    Folded fo;
    fold_layers(pl.L, pl.G, pl.R, pl.G2, pl.kw, *w, fo);
    pack_cta(pl, *w, fo, cta, packed);
    if (packed_floats >= pl.cta_w_floats + pl.cta_cw_floats) pack_cw_cta(pl, *w, cta, packed + pl.cta_w_floats);
    return WN_OK;
}

int32_t wn_create(const wn_config* cfg, void** handle) {
    if (!cfg || !handle) return fail(WN_ERR_INVALID, "null argument");
    *handle = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(WN_ERR_CUDA, std::string("no CUDA device: ") + cudaGetErrorString(e) +
                                     " (libwn has no CPU path; it needs an sm_90 GPU)");
    if (cfg->device < 0 || cfg->device >= ndev) return fail(WN_ERR_INVALID, "device ordinal out of range");
    DeviceGuard guard(cfg->device);
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(WN_ERR_CUDA, "libwn.so is built for sm_90a only; found compute capability " +
                                     std::to_string(prop.major) + "." + std::to_string(prop.minor));
    int coop = 0;
    CUDA_TRY(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, cfg->device));
    if (!coop) return fail(WN_ERR_CUDA, "device does not support cooperative launch");
    int engine = 5;
    if (int32_t rce = engine_choice(*cfg, &engine)) return rce;
    WnHandle* h = new WnHandle();
    h->cfg = *cfg;
    h->engine = engine;
    h->num_sms = prop.multiProcessorCount;
    h->smem_cap = (long long)prop.sharedMemPerBlockOptin;
    h->l2_bytes = (size_t)prop.l2CacheSize;
    int32_t rc;
    if (h->engine == 7) {
        rc = build_plan7(h->cfg, 1, h->num_sms, h->smem_cap, h->base7, h->passes7, h->ringtab);
    } else {
        rc = build_plan(h->cfg, 1, h->num_sms, h->smem_cap, h->base, h->ringtab);
    }
    if (rc) {
        delete h;
        return rc;
    }
    h->l2_mode = env_int("WN_L2_PERSIST", 2);
    if (h->l2_mode > 0 && prop.persistingL2CacheMaxSize > 0) {
        // WN_L2_PERSIST=2 (default): the exchange buffer (a few MB, every line written and read once per generated
        // sample) lives in a 16 MB persisting carve-out of the 50 MB L2, so the 112 MB/sample weight stream cannot
        // evict it between two steps.  On an H100 SXM the three settings are within 1 % of each other (DESIGN.md 7).
        // This sets cudaLimitPersistingL2CacheSize for the device (process-wide).
        // =1 pins as much of the packed weight image as allowed instead; =0: nothing.
        const size_t want = h->l2_mode == 2 ? std::min<size_t>((size_t)prop.persistingL2CacheMaxSize, 16u << 20)
                                             : (size_t)prop.persistingL2CacheMaxSize;
        if (cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want) == cudaSuccess) {
            h->l2_carve_bytes = want;
            h->l2_persist_bytes = (size_t)prop.persistingL2CacheMaxSize;
            h->l2_window_max = (size_t)prop.accessPolicyMaxWindowSize;
        } else {
            cudaGetLastError();
        }
    }
    // freeze the partition so every batch tile agrees with the packing
    if (h->engine == 7) {
        h->cfg.num_ctas = h->base7.P;
        h->cfg.poll_warps = h->base7.npw == 0 ? -1 : h->base7.npw;
    } else {
        h->cfg.num_ctas = h->base.P;
        h->cfg.exchange_copies = h->base.ncopy;
    }
    if (cudaMalloc((void**)&h->d_err, 16) != cudaSuccess || cudaMemset(h->d_err, 0, 16) != cudaSuccess) {
        delete h;
        return fail(WN_ERR_CUDA, "cudaMalloc failed");
    }
    *handle = h;
    return WN_OK;
}

int32_t wn_destroy(void* handle) {
    WnHandle* h = (WnHandle*)handle;
    if (!h) return WN_OK;
    DeviceGuard guard(h->cfg.device);
    cudaDeviceSynchronize();
    cudaFree(h->d_bpack); cudaFree(h->d_passes);
    cudaFree(h->d_ups_filters); cudaFree(h->d_ups_convw); cudaFree(h->d_cup); cudaFree(h->d_hfr);
    cudaFree(h->d_wpack); cudaFree(h->d_cwpack); cudaFree(h->d_wg); cudaFree(h->d_first_w); cudaFree(h->d_first_b);
    cudaFree(h->d_ringtab); cudaFree(h->d_err); cudaFree(h->d_xbuf); cudaFree(h->d_ring); cudaFree(h->d_gbias);
    cudaFree(h->d_scratch);
    cudaFree(h->d_prof);
    cudaFree(h->d_dense); cudaFree(h->d_fwd);
    delete h;
    return WN_OK;
}

int32_t wn_load_weights(void* handle, const wn_weights* w) {
    WnHandle* h = (WnHandle*)handle;
    if (!h) return fail(WN_ERR_INVALID, "null handle");
    int32_t rc = check_weights(h->cfg, w);
    if (rc) return rc;
    DeviceGuard guard(h->cfg.device);
    h->weight_gen++;
    const wn_config& c = h->cfg;
    auto upload =[&](float** dst, const std::vector<float>& src) -> int32_t {
        if (*dst) cudaFree(*dst);
        *dst = nullptr;
        CUDA_TRY(cudaMalloc((void**)dst, std::max<size_t>(16, src.size() * sizeof(float))));
        if (!src.empty()) CUDA_TRY(cudaMemcpy(*dst, src.data(), src.size() * sizeof(float), cudaMemcpyHostToDevice));
        return WN_OK;
    };
    struct Shape { int L, G, R, G2, kw, O, P; } pl;
    if (h->engine == 7) {
        const Wn7Plan& p6 = h->base7;
        pl = {p6.L, p6.G, p6.R, p6.G2, p6.kw, p6.O, p6.P};
        Folded fo;
        fold_layers(pl.L, pl.G, pl.R, pl.G2, pl.kw, *w, fo);
        std::vector<float> img((size_t)p6.P * p6.cta_w_floats), cw((size_t)p6.P * p6.cta_cw_floats),
            bs((size_t)p6.P * p6.cta_b_floats);
        for (int p = 0; p < p6.P; ++p) {
            pack7_cta(p6, h->passes7, *w, fo, p, img.data() + (size_t)p * p6.cta_w_floats);
            pack7_cw(p6, *w, p, cw.data() + (size_t)p * p6.cta_cw_floats);
            pack7_bias(p6, *w, fo, p, bs.data() + (size_t)p * p6.cta_b_floats);
        }
        if ((rc = upload(&h->d_wpack, img))) return rc;
        h->wpack_bytes = img.size() * sizeof(float);
        if ((rc = upload(&h->d_cwpack, cw))) return rc;
        if ((rc = upload(&h->d_bpack, bs))) return rc;
        if (h->d_passes) cudaFree(h->d_passes);
        h->d_passes = nullptr;
        CUDA_TRY(cudaMalloc((void**)&h->d_passes, std::max<size_t>(16, h->passes7.size() * sizeof(Wn7Pass))));
        CUDA_TRY(cudaMemcpy(h->d_passes, h->passes7.data(), h->passes7.size() * sizeof(Wn7Pass), cudaMemcpyHostToDevice));
    } else {
        const WnPlan& p5 = h->base;
        pl = {p5.L, p5.G, p5.R, p5.G2, p5.kw, p5.O, p5.P};
        std::vector<float> img((size_t)p5.P * p5.cta_w_floats);
        {
            Folded fo;
            fold_layers(pl.L, pl.G, pl.R, pl.G2, pl.kw, *w, fo);
            for (int p = 0; p < p5.P; ++p) pack_cta(p5, *w, fo, p, img.data() + (size_t)p * p5.cta_w_floats);
        }
        if ((rc = upload(&h->d_wpack, img))) return rc;
        h->wpack_bytes = img.size() * sizeof(float);
        std::vector<float> cw((size_t)p5.P * p5.cta_cw_floats);
        for (int p = 0; p < p5.P; ++p) pack_cw_cta(p5, *w, p, cw.data() + (size_t)p * p5.cta_cw_floats);
        if ((rc = upload(&h->d_cwpack, cw))) return rc;
    }
    std::vector<float> wg;
    if (c.gin_channels > 0) {
        wg.resize((size_t)pl.L * pl.G * c.gin_channels);
        for (int l = 0; l < pl.L; ++l)
            memcpy(wg.data() + (size_t)l * pl.G * c.gin_channels, w->layers[l].gcond_w,
                   (size_t)pl.G * c.gin_channels * sizeof(float));
    }
    if ((rc = upload(&h->d_wg, wg))) return rc;
    std::vector<float> fw;
    if (c.input_kind == WN_INPUT_SCALAR) {
        fw.assign(w->first_w, w->first_w + pl.R);
    } else {   // (R,O) -> [O][R]: a one-hot input selects one contiguous column
        fw.resize((size_t)pl.O * pl.R);
        for (int r = 0; r < pl.R; ++r)
            for (int o = 0; o < pl.O; ++o) fw[(size_t)o * pl.R + r] = w->first_w[(size_t)r * pl.O + o];
    }
    if ((rc = upload(&h->d_first_w, fw))) return rc;
    std::vector<float> fb(w->first_b, w->first_b + pl.R);
    if ((rc = upload(&h->d_first_b, fb))) return rc;
    if (h->d_ringtab) cudaFree(h->d_ringtab);
    h->d_ringtab = nullptr;
    CUDA_TRY(cudaMalloc((void**)&h->d_ringtab, std::max<size_t>(16, h->ringtab.size() * sizeof(int))));
    if (!h->ringtab.empty())
        CUDA_TRY(cudaMemcpy(h->d_ringtab, h->ringtab.data(), h->ringtab.size() * sizeof(int), cudaMemcpyHostToDevice));
    {   // the unfolded matrices wn_forward reads: uploaded with the packed image, so neither path can see stale weights
        std::vector<float> dense;
        pack_dense(c, *w, dense);
        if ((rc = upload(&h->d_dense, dense))) return rc;
        h->dense_bytes = dense.size() * sizeof(float);
    }
    h->have_weights = true;
    return WN_OK;
}

// window_frames: c_frames is a window of the utterance (a stream chunk, checked by the caller), not all of it
static int32_t validate_args(const WnHandle* h, const wn_generate_args* a, bool window_frames = false) {
    const wn_config& c = h->cfg;
    if (!a) return fail(WN_ERR_INVALID, "null args");
    if (a->B < 1 || a->T < 1) return fail(WN_ERR_INVALID, "B and T must be >= 1");
    if ((long long)a->T * (c.layers + 3LL) >= 0xFFFFFFF0LL) return fail(WN_ERR_INVALID, "T too large for 32-bit tags");
    int32_t rc = validate_cond(h, a, window_frames);
    if (rc) return rc;
    if (a->T_test < 0 || a->T_test > a->T) return fail(WN_ERR_INVALID, "T_test must be in [0,T] (wavenet.py:258)");
    if (c.input_kind == WN_INPUT_SCALAR) {
        if (!a->out_scalar) return fail(WN_ERR_INVALID, "out_scalar required");
        if (a->T_test > 0 && !a->test_scalar) return fail(WN_ERR_INVALID, "test_scalar required when T_test > 0");
    } else {
        const bool quant = (a->flags & WN_FLAG_QUANTIZE) != 0, soft = (a->flags & WN_FLAG_SOFTMAX) != 0;
        if (quant && !soft)
            return fail(WN_ERR_INVALID, "quantize without softmax feeds logits to OneHotCategorical (wavenet.py:332-335): unsupported");
        if (quant && !a->out_index) return fail(WN_ERR_INVALID, "out_index required with QUANTIZE");
        if (!quant && !a->out_dense) return fail(WN_ERR_INVALID, "out_dense required without QUANTIZE");
        if (a->T_test > 0 && !a->test_index && !a->test_dense) return fail(WN_ERR_INVALID, "test_index or test_dense required when T_test > 0");
        // the reference's default start class is 127 (wavenet.py:286) and indexing a smaller model with it raises
        const int start = a->initial_index < 0 ? 127 : a->initial_index;
        if (a->T_test == 0 && !a->initial_rows && !a->initial_dense && start >= c.out_channels)
            return fail(WN_ERR_INVALID, "initial_index out of range (the default start class is 127, wavenet.py:286)");
    }
    if (a->noise_kind == WN_NOISE_REPLAY) {
        const bool quant = (a->flags & WN_FLAG_QUANTIZE) != 0;
        if (c.head_kind == WN_HEAD_MOL && (!a->noise_u1 || !a->noise_u2)) return fail(WN_ERR_INVALID, "replay noise u1,u2 required (MoL)");
        if (c.head_kind == WN_HEAD_GAUSS && !a->noise_z) return fail(WN_ERR_INVALID, "replay noise z required (Gaussian)");
        if (c.head_kind == WN_HEAD_GAUSS && c.out_channels > 3 && !a->noise_u1) return fail(WN_ERR_INVALID, "replay noise u1 required (Gaussian mixture)");
        if (c.head_kind == WN_HEAD_SOFTMAX && quant && !a->noise_e) return fail(WN_ERR_INVALID, "replay noise e required (softmax)");
    } else if (a->noise_kind != WN_NOISE_PHILOX)
        return fail(WN_ERR_INVALID, "bad noise_kind");
    return WN_OK;
}

int32_t wn_generate(void* handle, const wn_generate_args* a) {
    WnHandle* h = (WnHandle*)handle;
    if (!h) return fail(WN_ERR_INVALID, "null handle");
    if (!h->have_weights) return fail(WN_ERR_STATE, "wn_generate before wn_load_weights");
    int32_t rc = validate_args(h, a);
    if (rc) return rc;
    DeviceGuard guard(h->cfg.device);
    cudaStream_t st = (cudaStream_t)a->stream;
    wn_generate_args up_args;
    if (a->c_frames) {
        rc = run_upsampler(h, a->c_frames, a->B, a->n_frames, a->T, st);
        if (rc) return rc;
        up_args = *a;
        up_args.c = h->d_cup;
        up_args.c_frames = nullptr;
        a = &up_args;
    }
    // batch tiles: up to 8 utterances share one launch (one pass over the weights per step for all of them)
    const int tile = max_tile(h->engine);
    for (int b0 = 0; b0 < a->B; b0 += tile) {
        const int Bc = std::min(tile, a->B - b0);
        rc = h->engine == 7 ? launch_chunk7(h, a, b0, Bc, st) : launch_chunk(h, a, b0, Bc, st);
        if (rc) return rc;
    }
    h->last_stream = st;
    h->pending = true;
    return WN_OK;
}

int32_t wn_sync(void* handle) {
    WnHandle* h = (WnHandle*)handle;
    if (!h) return fail(WN_ERR_INVALID, "null handle");
    DeviceGuard guard(h->cfg.device);
    CUDA_TRY(cudaStreamSynchronize(h->last_stream));
    h->pending = false;
    int err[4] = {0, 0, 0, 0};
    CUDA_TRY(cudaMemcpy(err, h->d_err, sizeof(err), cudaMemcpyDeviceToHost));
    if (h->d_prof && env_int("WN_PROF", 0)) {
        std::vector<long long> pc(h->prof_bytes / sizeof(long long));
        CUDA_TRY(cudaMemcpy(pc.data(), h->d_prof, h->prof_bytes, cudaMemcpyDeviceToHost));
        if (h->engine != 7) {
            // the per-block stage profile (wn_kernel.cuh, WN_PROF_SLOTS), one line per block for scripts/stage_prof.py
            const int P = (int)(pc.size() / WN_PROF_SLOTS);
            for (int p = 0; p < P; ++p) {
                fprintf(stderr, "WN_PROF_BLOCK %d", p);
                for (int i = 0; i < WN_PROF_SLOTS; ++i) fprintf(stderr, " %lld", pc[(size_t)p * WN_PROF_SLOTS + i]);
                fprintf(stderr, "\n");
            }
            fprintf(stderr, "WN_PROF L2 prefetch distance %d blobs\n", h->last_l2_pf);
        } else {
            const char* names7[4] = {"W0.acquire_blob+pre", "W0.wait_input", "W0.critical_passes", "W0.deferred+release"};
            const int P = (int)(pc.size() / 16);
            for (int i = 8; i < 12; ++i) {
                long long mn = pc[i], mx = pc[i], sum = 0;
                for (int p = 0; p < P; ++p) { mn = std::min(mn, pc[p * 16 + i]); mx = std::max(mx, pc[p * 16 + i]); sum += pc[p * 16 + i]; }
                fprintf(stderr, "WN_PROF %-20s mean %12.0f  min %12lld  max %12lld cycles\n", names7[i - 8], (double)sum / P, mn, mx);
            }
        }
    }
    if (err[0] != 0) {
        cudaMemset(h->d_err, 0, sizeof(err));
        char buf[160];
        snprintf(buf, sizeof(buf), "device watchdog: block %d thread %d stuck waiting on 0x%08x", err[2], err[3],
                 (unsigned)err[1]);
        return fail(WN_ERR_DEVICE, buf);
    }
    return WN_OK;
}

int32_t wn_get_plan(void* handle, int32_t batch, wn_plan_info* out) {
    WnHandle* h = (WnHandle*)handle;
    if (!h || !out) return fail(WN_ERR_INVALID, "null argument");
    const int bt = std::min(std::max(batch, 1), max_tile(h->engine));
    if (h->engine == 7) {
        Wn7Plan pl6;
        std::vector<Wn7Pass> ps;
        std::vector<int> rt6;
        int32_t rc6 = build_plan7(h->cfg, bt, h->num_sms, h->smem_cap, pl6, ps, rt6);
        if (rc6) return rc6;
        fill_info7(h->cfg, pl6, out);
        out->launches = h->launches;
        return WN_OK;
    }
    WnPlan pl;
    std::vector<int> rt;
    int32_t rc = build_plan(h->cfg, bt, h->num_sms, h->smem_cap, pl, rt);
    if (rc) return rc;
    fill_info(h->cfg, pl, out);
    out->launches = h->launches;
    return WN_OK;
}

// Host-buffer variant: stage inputs to the device, run, copy results back (synchronous).
int32_t wn_generate_host(void* handle, const wn_generate_args* a) {
    WnHandle* h = (WnHandle*)handle;
    if (!h) return fail(WN_ERR_INVALID, "null handle");
    if (!h->have_weights) return fail(WN_ERR_STATE, "wn_generate_host before wn_load_weights");
    int32_t rc = validate_args(h, a);
    if (rc) return rc;
    DeviceGuard guard(h->cfg.device);
    const wn_config& c = h->cfg;
    const size_t B = a->B, T = a->T, O = c.out_channels, Tt = a->T_test;
    const size_t K = (c.head_kind == WN_HEAD_SOFTMAX) ? 0 : (O == 2 ? 1 : O / 3);
    struct Item { const void* src; void* dst_host; size_t bytes; size_t off; };
    std::vector<Item> in, out;
    size_t total = 0;
    auto add = [&](std::vector<Item>& v, const void* src, void* dsth, size_t bytes) {
        if ((!src && !dsth) || bytes == 0) return (size_t)-1;
        total = (total + 255) / 256 * 256;
        v.push_back({src, dsth, bytes, total});
        total += bytes;
        return v.back().off;
    };
    const size_t o_c = add(in, a->c, nullptr, B * T * (size_t)c.cin_channels * 4);
    const size_t o_cf = add(in, a->c_frames, nullptr, B * (size_t)c.cin_channels * (size_t)std::max(a->n_frames, 0) * 4);
    const size_t o_g = add(in, a->g, nullptr, B * (size_t)c.gin_channels * 4);
    const size_t o_init = add(in, a->initial, nullptr, B * 4);
    const size_t o_irow = add(in, a->initial_rows, nullptr, B * 4);
    const size_t o_iden = add(in, a->initial_dense, nullptr, B * O * 4);
    const size_t o_ts = add(in, a->test_scalar, nullptr, B * Tt * 4);
    const size_t o_ti = add(in, a->test_index, nullptr, B * Tt * 4);
    const size_t o_td = add(in, a->test_dense, nullptr, B * Tt * O * 4);
    const size_t o_u1 = add(in, a->noise_u1, nullptr, T * B * K * 4);
    const size_t o_u2 = add(in, a->noise_u2, nullptr, T * B * 4);
    const size_t o_z = add(in, a->noise_z, nullptr, T * B * 4);
    const size_t o_e = add(in, a->noise_e, nullptr, T * B * O * 4);
    const size_t o_os = add(out, nullptr, a->out_scalar, B * T * 4);
    const size_t o_oi = add(out, nullptr, a->out_index, B * T * 4);
    const size_t o_od = add(out, nullptr, a->out_dense, B * O * T * 4);
    const size_t o_po = add(out, nullptr, a->params_out, B * O * T * 4);
    rc = ensure(&h->d_scratch, &h->scratch_bytes, total + 256);
    if (rc) return rc;
    char* base = (char*)h->d_scratch;
    cudaStream_t st = (cudaStream_t)a->stream;
    for (const Item& it : in) CUDA_TRY(cudaMemcpyAsync(base + it.off, it.src, it.bytes, cudaMemcpyHostToDevice, st));
    wn_generate_args d = *a;
    auto dp = [&](size_t off) -> char* { return off == (size_t)-1 ? nullptr : base + off; };
    d.c = (const float*)dp(o_c);
    d.c_frames = (const float*)dp(o_cf);
    d.g = (const float*)dp(o_g);
    d.initial = (const float*)dp(o_init);
    d.initial_rows = (const int32_t*)dp(o_irow);
    d.initial_dense = (const float*)dp(o_iden);
    d.test_scalar = (const float*)dp(o_ts);
    d.test_index = (const int32_t*)dp(o_ti);
    d.test_dense = (const float*)dp(o_td);
    d.noise_u1 = (const float*)dp(o_u1);
    d.noise_u2 = (const float*)dp(o_u2);
    d.noise_z = (const float*)dp(o_z);
    d.noise_e = (const float*)dp(o_e);
    d.out_scalar = (float*)dp(o_os);
    d.out_index = (int32_t*)dp(o_oi);
    d.out_dense = (float*)dp(o_od);
    d.params_out = (float*)dp(o_po);
    rc = wn_generate(handle, &d);
    if (rc) return rc;
    for (const Item& it : out) CUDA_TRY(cudaMemcpyAsync(it.dst_host, base + it.off, it.bytes, cudaMemcpyDeviceToHost, st));
    return wn_sync(handle);
}

// the geometry of an upsampler (everything but its weights); *filter_floats = taps of all smoothing filters
static int32_t ups_desc(const wn_upsampler* u, wnaux::UpsampleDesc& d, long long& total, int& filter_floats) {
    if (u->n_scales < 1 || u->n_scales > WNAUX_MAX_SCALES || !u->scales)
        return fail(WN_ERR_INVALID, "upsampler needs 1..8 scales and their filters");
    if (u->conv_in_ks < 0 || u->indent < 0) return fail(WN_ERR_INVALID, "bad conv_in / indent");
    memset(&d, 0, sizeof(d));
    d.n_scales = u->n_scales;
    d.indent = u->indent;
    int off = 0;
    total = 1;
    for (int j = 0; j < u->n_scales; ++j) {
        const int s = u->scales[j];
        if (s < 2 || s > 4096) return fail(WN_ERR_INVALID, "every upsample scale must be in [2,4096]");
        d.scales[j] = s;
        d.foff[j] = off;
        d.rscale[j] = (float)(1.0 / (double)s);
        off += 2 * s + 1;
        total *= s;
        if (total > (1 << 24)) return fail(WN_ERR_INVALID, "total upsample scale too large");
    }
    filter_floats = off;
    return WN_OK;
}

// Frames [*f_lo, *f_hi) that samples [t_lo, t_hi) need and the samples known from the start (*n_ready), given
// n_frames received (final: all of them).  Mirrors upsample_kernel's index table (wnaux::cone_rows).
static int32_t ups_cone(const wnaux::UpsampleDesc& d, long long total, int ks, long long n_frames, bool final,
                        long long t_lo, long long t_hi, long long* f_lo, long long* f_hi, long long* n_ready) {
    const int lost = ks > 0 ? ks - 1 : 0;
    const long long Fo = n_frames - lost;                 // rows of level 0 (conv_in outputs) known
    *f_lo = *f_hi = 0;
    *n_ready = 0;
    if (t_lo < 0 || t_hi < t_lo) return fail(WN_ERR_INVALID, "bad sample range");
    if (Fo < 1) return t_hi > t_lo ? fail(WN_ERR_INVALID, "no sample is known before conv_in has its first window") : WN_OK;
    if (Fo * total >= WNAUX_UNBOUNDED) return fail(WN_ERR_INVALID, "utterance too long for the upsampler's 32-bit indices");
    const int n0 = final ? (int)Fo : WNAUX_UNBOUNDED;
    const long long full = std::max(0LL, Fo * total - 2LL * d.indent);   // the length if the utterance ended here
    int lo, hi;
    bool inside;
    if (final) {
        *n_ready = full;
    } else {
        // the cone grows with t, so the known samples are a prefix: bisect for its length
        long long a = 0, b = full;
        while (a < b) {
            const long long m = (a + b + 1) / 2;
            wnaux::cone_rows(d, n0, (int)Fo, (int)(m - 1), (int)m, &lo, &hi, &inside);
            if (inside) a = m; else b = m - 1;
        }
        *n_ready = a;
    }
    if (t_hi > t_lo) {
        if (t_hi > full) return fail(WN_ERR_INVALID, "sample range beyond the upsampled length of the frames");
        wnaux::cone_rows(d, n0, (int)Fo, (int)t_lo, (int)t_hi, &lo, &hi, &inside);
        *f_lo = lo;
        *f_hi = (long long)hi + lost + 1;
    }
    return WN_OK;
}

int32_t wn_upsample_cone(const wn_upsampler* u, int64_t n_frames, int32_t final, int64_t t_lo, int64_t t_hi,
                         int64_t* f_lo, int64_t* f_hi, int64_t* n_ready) {
    if (!u || !f_lo || !f_hi || !n_ready) return fail(WN_ERR_INVALID, "null argument");
    wnaux::UpsampleDesc d;
    long long total, a, b, r;
    int nf;
    int32_t rc = ups_desc(u, d, total, nf);
    if (rc) return rc;
    rc = ups_cone(d, total, u->conv_in_ks, n_frames, final != 0, t_lo, t_hi, &a, &b, &r);
    *f_lo = a;
    *f_hi = b;
    *n_ready = r;
    return rc;
}

int32_t wn_load_upsampler(void* handle, const wn_upsampler* u) {
    WnHandle* h = (WnHandle*)handle;
    if (!h) return fail(WN_ERR_INVALID, "null handle");
    DeviceGuard guard(h->cfg.device);
    h->have_ups = false;
    h->weight_gen++;
    if (!u) return WN_OK;
    if (u->channels != h->cfg.cin_channels || u->channels < 1) return fail(WN_ERR_INVALID, "upsampler channels != cin_channels");
    if (u->n_scales < 1 || u->n_scales > WNAUX_MAX_SCALES || !u->scales || !u->filters)
        return fail(WN_ERR_INVALID, "upsampler needs 1..8 scales and their filters");
    if ((u->conv_in_w != nullptr) != (u->conv_in_ks > 0) || u->indent < 0) return fail(WN_ERR_INVALID, "bad conv_in / indent");
    long long total = 1;
    int off = 0;
    int32_t rc = ups_desc(u, h->ups, total, off);
    if (rc) return rc;
    h->ups_total = (int)total;
    h->ups_C = u->channels;
    h->ups_ks = u->conv_in_ks;
    if (h->d_ups_filters) cudaFree(h->d_ups_filters);
    h->d_ups_filters = nullptr;
    CUDA_TRY(cudaMalloc((void**)&h->d_ups_filters, (size_t)off * sizeof(float)));
    CUDA_TRY(cudaMemcpy(h->d_ups_filters, u->filters, (size_t)off * sizeof(float), cudaMemcpyHostToDevice));
    if (h->d_ups_convw) cudaFree(h->d_ups_convw);
    h->d_ups_convw = nullptr;
    if (u->conv_in_ks > 0) {
        const size_t nw = (size_t)u->channels * u->channels * u->conv_in_ks;
        CUDA_TRY(cudaMalloc((void**)&h->d_ups_convw, nw * sizeof(float)));
        CUDA_TRY(cudaMemcpy(h->d_ups_convw, u->conv_in_w, nw * sizeof(float), cudaMemcpyHostToDevice));
    }
    h->have_ups = true;
    return WN_OK;
}

int32_t wn_upsample(void* handle, const float* c_frames, int32_t B, int32_t n_frames, int32_t T, float* out, void* stream) {
    WnHandle* h = (WnHandle*)handle;
    if (!h || !c_frames || !out) return fail(WN_ERR_INVALID, "null argument");
    if (!h->have_ups) return fail(WN_ERR_STATE, "no upsampler was loaded (wn_load_upsampler)");
    const long long Fo = (long long)n_frames - (h->ups_ks > 0 ? h->ups_ks - 1 : 0);
    if (B < 1 || Fo < 1 || Fo * h->ups_total - 2LL * h->ups.indent != (long long)T)
        return fail(WN_ERR_INVALID, "upsampled conditioning length != T (wavenet.py:276)");
    DeviceGuard guard(h->cfg.device);
    int32_t rc = run_upsampler(h, c_frames, B, n_frames, T, (cudaStream_t)stream);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(out, h->d_cup, (size_t)B * T * h->ups_C * sizeof(float), cudaMemcpyDeviceToDevice,
                             (cudaStream_t)stream));
    return WN_OK;
}

int32_t wn_decode_stream(const float* y_scalar, const int32_t* y_index, int32_t B, int32_t T, const int32_t* lengths,
                         int32_t input_type, int32_t quantize_channels, float preemphasis_coef, float global_gain_scale,
                         float* out_float, int16_t* out_pcm16, float* carry, void* stream) {
    if (B < 1 || T < 1) return fail(WN_ERR_INVALID, "B and T must be >= 1");
    if (!out_float && !out_pcm16) return fail(WN_ERR_INVALID, "no output buffer");
    if (input_type == WN_DECODE_MULAW_QUANTIZE ? !y_index : !y_scalar) return fail(WN_ERR_INVALID, "missing input for this input_type");
    if (input_type < 0 || input_type > 2) return fail(WN_ERR_INVALID, "bad input_type");
    if (input_type != WN_DECODE_RAW && quantize_channels < 2) return fail(WN_ERR_INVALID, "quantize_channels must be >= 2");
    wnaux::decode_kernel<1024><<<B, 256, 0, (cudaStream_t)stream>>>(y_scalar, y_index, T, lengths, input_type,
                                                                    (float)(quantize_channels - 1), preemphasis_coef,
                                                                    global_gain_scale, out_float, (short*)out_pcm16, carry);
    CUDA_TRY(cudaGetLastError());
    return WN_OK;
}

int32_t wn_decode(const float* y_scalar, const int32_t* y_index, int32_t B, int32_t T, const int32_t* lengths,
                  int32_t input_type, int32_t quantize_channels, float preemphasis_coef, float global_gain_scale,
                  float* out_float, int16_t* out_pcm16, void* stream) {
    return wn_decode_stream(y_scalar, y_index, B, T, lengths, input_type, quantize_channels, preemphasis_coef,
                            global_gain_scale, out_float, out_pcm16, nullptr, stream);
}

// ------------------------------------------------------------------------------------------
// streams
// ------------------------------------------------------------------------------------------
struct WnStream {
    WnHandle* h = nullptr;
    int B = 0;
    int engine = 5;                // the kernel organisation the chunks run on (wn_stream_open_args.engine)
    uint64_t weight_gen = 0;       // the handle's weights this stream was opened with
    wn_stream_open_args open;      // initial* point into d_init (copies made at open)
    float* d_state = nullptr;      // P x rings, then the feedback (WnPtrs::state / Wn7Ptrs::state)
    float* d_gbias = nullptr;
    float* d_init = nullptr;
    long long t = 0;               // absolute step of the next sample
    bool final = false;
};

int32_t wn_stream_open(void* handle, const wn_stream_open_args* a, void** stream) {
    WnHandle* h = (WnHandle*)handle;
    if (!h || !a || !stream) return fail(WN_ERR_INVALID, "null argument");
    *stream = nullptr;
    if (!h->have_weights) return fail(WN_ERR_STATE, "wn_stream_open before wn_load_weights");
    if (a->engine != 0 && a->engine != 5 && a->engine != 7)
        return fail(WN_ERR_INVALID, "wn_stream_open_args.engine must be 0 or 5 (engine 5) or 7; got " + std::to_string(a->engine));
    const int engine = a->engine == 7 ? 7 : 5;
    if (engine == 5) {
        if (h->engine != 5)
            return fail(WN_ERR_INVALID, "this stream runs on engine 5 but the handle runs engine 7 (WN_ENGINE=7 or "
                                        "wn_config.engine = 7): open it with wn_stream_open_args.engine = 7");
        const int tile = std::min(4, max_tile(5));
        if (a->B < 1 || a->B > tile)
            return fail(WN_ERR_INVALID, "a stream holds 1.." + std::to_string(tile) + " utterances (one batch tile)");
    } else {
        if (h->engine != 7)
            return fail(WN_ERR_INVALID, "an engine-7 stream needs a handle that runs engine 7 (wn_config.engine = 7); "
                                        "this one runs engine 5");
        if (h->base7.npw != 0)
            return fail(WN_ERR_INVALID, "an engine-7 stream needs a handle whose compute warps poll (poll_warps 0 or -1); "
                                        "this one has " + std::to_string(h->base7.npw) + " polling warps");
        const int tile = max_tile(7);
        if (a->B < 1 || a->B > tile)
            return fail(WN_ERR_INVALID, "an engine-7 stream holds 1.." + std::to_string(tile) +
                                            " utterances (one batch tile)");
    }
    const wn_config& c = h->cfg;
    if (c.gin_channels > 0 && !a->g) return fail(WN_ERR_INVALID, "g is required (gin_channels > 0), cf. train.py:72-80 sanity_check");
    if (c.gin_channels == 0 && a->g) return fail(WN_ERR_INVALID, "g given but the model has no global conditioning");
    if (a->noise_kind != WN_NOISE_REPLAY && a->noise_kind != WN_NOISE_PHILOX) return fail(WN_ERR_INVALID, "bad noise_kind");
    DeviceGuard guard(c.device);
    // the state buffer: every block's history rings, then the feedback of the next step
    size_t state_floats = 0;
    int L = 0, G = 0, O = 0;
    if (engine == 5) {
        WnPlan pl;
        std::vector<int> rt;
        int32_t rc = build_plan(c, a->B, h->num_sms, h->smem_cap, pl, rt);
        if (rc) return rc;
        state_floats = (size_t)pl.P * wn_state_ring_floats(pl) + wn_state_feedback_floats(pl);
        L = pl.L, G = pl.G, O = pl.O;
    } else {
        Wn7Plan pl;
        std::vector<Wn7Pass> ps;
        std::vector<int> rt;
        int32_t rc = build_plan7(c, a->B, h->num_sms, h->smem_cap, pl, ps, rt);
        if (rc) return rc;
        state_floats = (size_t)pl.P * wn7_state_ring_floats(pl) + wn7_state_feedback_floats(pl);
        L = pl.L, G = pl.G, O = pl.O;
    }
    cudaStream_t st = (cudaStream_t)a->stream;
    WnStream* s = new WnStream();
    s->h = h;
    s->B = a->B;
    s->engine = engine;
    s->weight_gen = h->weight_gen;
    s->open = *a;
    auto bail = [&](int32_t code) {
        cudaFree(s->d_state); cudaFree(s->d_gbias); cudaFree(s->d_init);
        delete s;
        return code;
    };
    if (cudaMalloc((void**)&s->d_state, state_floats * sizeof(float)) != cudaSuccess ||
        cudaMalloc((void**)&s->d_init, ((size_t)2 + O) * a->B * sizeof(float)) != cudaSuccess)
        return bail(fail(WN_ERR_NOMEM, "cudaMalloc of the stream state failed"));
    if (cudaMemsetAsync(s->d_state, 0, state_floats * sizeof(float), st) != cudaSuccess)
        return bail(fail(WN_ERR_CUDA, "cudaMemsetAsync of the stream state failed"));
    // the step-0 inputs are copied: the caller's buffers may go once open returns
    float* init = s->d_init;
    int32_t* init_rows = (int32_t*)(s->d_init + a->B);
    float* init_dense = s->d_init + 2 * a->B;
    auto copy = [&](void* dst, const void* src, size_t bytes) {
        return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st) == cudaSuccess;
    };
    if ((a->initial && !copy(init, a->initial, a->B * sizeof(float))) ||
        (a->initial_rows && !copy(init_rows, a->initial_rows, a->B * sizeof(int32_t))) ||
        (a->initial_dense && !copy(init_dense, a->initial_dense, (size_t)a->B * O * sizeof(float))))
        return bail(fail(WN_ERR_CUDA, "copying the initial input failed"));
    s->open.initial = a->initial ? init : nullptr;
    s->open.initial_rows = a->initial_rows ? init_rows : nullptr;
    s->open.initial_dense = a->initial_dense ? init_dense : nullptr;
    s->open.g = nullptr;
    if (c.gin_channels > 0) {
        // Wg . g once per stream (modules.py:148-152 recomputes it every step although g is constant)
        if (cudaMalloc((void**)&s->d_gbias, (size_t)a->B * L * G * sizeof(float)) != cudaSuccess)
            return bail(fail(WN_ERR_NOMEM, "cudaMalloc of the stream's global-conditioning bias failed"));
        wn::wn_gbias_kernel<<<dim3(L, a->B), 128, 0, st>>>(h->d_wg, a->g, s->d_gbias, L, G, c.gin_channels);
        h->launches++;
    }
    if (cudaStreamSynchronize(st) != cudaSuccess || cudaGetLastError() != cudaSuccess)
        return bail(fail(WN_ERR_CUDA, "stream set-up failed"));
    *stream = s;
    return WN_OK;
}

int32_t wn_stream_generate(void* stream, const wn_generate_args* chunk, const wn_stream_chunk* where) {
    WnStream* s = (WnStream*)stream;
    if (!s || !chunk) return fail(WN_ERR_INVALID, "null argument");
    WnHandle* h = s->h;
    if (s->final) return fail(WN_ERR_STATE, "the stream was finalised: no chunk may follow its final one");
    if (h->weight_gen != s->weight_gen)
        return fail(WN_ERR_STATE, "the handle's weights changed since the stream was opened (wn_load_weights)");
    if (chunk->B != s->B) return fail(WN_ERR_INVALID, "chunk B differs from the B the stream was opened with");
    if (chunk->g || chunk->initial || chunk->initial_rows || chunk->initial_dense)
        return fail(WN_ERR_INVALID, "g and the initial input belong to wn_stream_open, not to a chunk");
    if (chunk->T_test != 0 || chunk->test_scalar || chunk->test_index || chunk->test_dense)
        return fail(WN_ERR_INVALID, "teacher forcing is not supported in a stream");
    if (chunk->T >= 1 && s->t + chunk->T > (1LL << 32))
        return fail(WN_ERR_INVALID, "absolute step beyond 2^32 (the Philox step counter is 32-bit)");
    wn_generate_args a = *chunk;
    a.initial = s->open.initial;
    a.initial_index = s->open.initial_index;
    a.initial_rows = s->open.initial_rows;
    a.initial_dense = s->open.initial_dense;
    a.flags = s->open.flags;
    a.noise_kind = s->open.noise_kind;
    a.seed = s->open.seed;
    a.philox_row0 = s->open.philox_row0;
    int32_t rc = validate_args(h, &a, true);
    if (rc) return rc;
    DeviceGuard guard(h->cfg.device);
    cudaStream_t st = (cudaStream_t)a.stream;
    if (a.c_frames) {
        if (!where) return fail(WN_ERR_INVALID, "c_frames in a stream needs its wn_stream_chunk (frame offset, frames so far)");
        if (where->frame_offset < 0 || a.n_frames < 1 || where->frame_offset + a.n_frames > where->frames_total)
            return fail(WN_ERR_INVALID, "the frame window lies outside the frames received so far");
        long long f_lo, f_hi, n_ready;
        rc = ups_cone(h->ups, h->ups_total, h->ups_ks, where->frames_total, where->final != 0, 0, 0, &f_lo, &f_hi,
                      &n_ready);
        if (rc) return rc;
        if (s->t + a.T > n_ready)
            return fail(WN_ERR_INVALID, "samples [" + std::to_string(s->t) + "," + std::to_string(s->t + a.T) +
                                            ") are not known yet from " + std::to_string(where->frames_total) +
                                            " frames (" + std::to_string(n_ready) + " are)");
        rc = ups_cone(h->ups, h->ups_total, h->ups_ks, where->frames_total, where->final != 0, s->t, s->t + a.T, &f_lo,
                      &f_hi, &n_ready);
        if (rc) return rc;
        if (f_lo < where->frame_offset || f_hi > where->frame_offset + a.n_frames)
            return fail(WN_ERR_INVALID, "the frame window [" + std::to_string(where->frame_offset) + "," +
                                            std::to_string(where->frame_offset + a.n_frames) + ") does not cover frames [" +
                                            std::to_string(f_lo) + "," + std::to_string(f_hi) + ") the chunk needs");
        const int lost = h->ups_ks > 0 ? h->ups_ks - 1 : 0;
        const int n0 = where->final ? (int)(where->frames_total - lost) : WNAUX_UNBOUNDED;
        rc = run_upsampler(h, a.c_frames, a.B, a.n_frames, a.T, st, (int)where->frame_offset, n0, (int)s->t);
        if (rc) return rc;
        a.c = h->d_cup;
        a.c_frames = nullptr;
    }
    StreamCtx sc;
    sc.state = s->d_state;
    sc.state_load = s->t > 0 ? 1 : 0;
    sc.t_base = (unsigned)s->t;
    sc.gbias = s->d_gbias;
    rc = s->engine == 7 ? launch_chunk7(h, &a, 0, a.B, st, &sc) : launch_chunk(h, &a, 0, a.B, st, &sc);
    if (rc) return rc;
    s->t += a.T;
    if (where && where->final) s->final = true;
    h->last_stream = st;
    h->pending = true;
    return WN_OK;
}

int64_t wn_stream_position(void* stream) {
    WnStream* s = (WnStream*)stream;
    return s ? (int64_t)s->t : (int64_t)fail(WN_ERR_INVALID, "null stream");
}

int32_t wn_stream_close(void* stream) {
    WnStream* s = (WnStream*)stream;
    if (!s) return WN_OK;
    DeviceGuard guard(s->h->cfg.device);
    cudaDeviceSynchronize();           // a chunk in flight still reads and writes the state
    cudaFree(s->d_state);
    cudaFree(s->d_gbias);
    cudaFree(s->d_init);
    delete s;
    return WN_OK;
}

int32_t wn_sample_mol(const float* y_bot, int32_t B, int32_t O, int32_t T, const float* u1_tbk, const float* u2_tb,
                      float* out_bt, void* stream) {
    if (!y_bot || !u1_tbk || !u2_tb || !out_bt) return fail(WN_ERR_INVALID, "null argument");
    if (B < 1 || T < 1 || O < 1) return fail(WN_ERR_INVALID, "wn_sample_mol: B, O and T must be >= 1");
    if (O % 3 != 0) return fail(WN_ERR_INVALID, "out_channels % 3 != 0 (mixture.py:130)");
    const int n = B * T;
    wn::wn_sample_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(y_bot, B, O, T, u1_tbk, u2_tb, out_bt, 0);
    CUDA_TRY(cudaGetLastError());
    return WN_OK;
}

int32_t wn_sample_gauss(const float* y_bot, int32_t B, int32_t O, int32_t T, const float* u1_tbk, const float* z_tb,
                        float* out_bt, void* stream) {
    if (!y_bot || !z_tb || !out_bt) return fail(WN_ERR_INVALID, "null argument");
    if (B < 1 || T < 1 || O < 1) return fail(WN_ERR_INVALID, "wn_sample_gauss: B, O and T must be >= 1");
    if (O != 2 && O % 3 != 0) return fail(WN_ERR_INVALID, "out_channels must be 2 or a multiple of 3 (mixture.py:229-234)");
    if (O > 3 && !u1_tbk) return fail(WN_ERR_INVALID, "u1 required for a mixture");
    const int n = B * T;
    wn::wn_sample_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(y_bot, B, O, T, u1_tbk, z_tb, out_bt, 1);
    CUDA_TRY(cudaGetLastError());
    return WN_OK;
}

int32_t wn_forward(void* handle, const wn_generate_args* a) {
    WnHandle* h = (WnHandle*)handle;
    if (!h) return fail(WN_ERR_INVALID, "null handle");
    if (!h->have_weights || !h->d_dense) return fail(WN_ERR_STATE, "wn_forward before wn_load_weights");
    int32_t rc = validate_forward(h, a);
    if (rc) return rc;
    DeviceGuard guard(h->cfg.device);
    const wn_config& c = h->cfg;
    cudaStream_t st = (cudaStream_t)a->stream;
    const int B = a->B, T = a->T, L = c.layers, R = c.residual_channels, G = c.gate_channels, G2 = G / 2;
    const int S = c.skip_channels, O = c.out_channels, kw = c.kernel_size, Cc = c.cin_channels;
    const int per_stack = L / c.stacks;
    // scratch: X (B,R,T) | Y, then the head's hidden layer (B,max(G/2,S),T) | skip sum (B,S,T) | c^T (B,C,T) |
    // a dense one-hot input transposed (B,O,T)
    auto al = [](size_t v) { return (v + 63) / 64 * 64; };
    const size_t BT = (size_t)B * T;
    const size_t oY = al(BT * R), oS = oY + al(BT * std::max(G2, S)), oC = oS + al(BT * S), oD = oC + al(BT * Cc);
    const size_t need = (oD + (a->test_dense ? al(BT * O) : 0) + 64) * sizeof(float);
    if (ensure(&h->d_fwd, &h->fwd_bytes, need)) {
        cudaGetLastError();
        return fail(WN_ERR_NOMEM, "wn_forward: cannot allocate " + std::to_string(need) + " bytes of activation scratch");
    }
    float *X = h->d_fwd, *Y = h->d_fwd + oY, *skip = h->d_fwd + oS, *cT = h->d_fwd + oC, *xdT = h->d_fwd + oD;
    int64_t launches = 0;
    const float* cond = a->c;
    if (a->c_frames) {
        rc = run_upsampler(h, a->c_frames, B, a->n_frames, T, st);
        if (rc) return rc;
        cond = h->d_cup;
    }
    if (Cc > 0) {
        wnd::transpose_tc_kernel<<<dim3((T + 31) / 32, (Cc + 31) / 32, B), dim3(32, 8), 0, st>>>(cond, cT, T, Cc);
        CUDA_TRY(cudaGetLastError());
        ++launches;
    }
    const float* gb = nullptr;
    if (c.gin_channels > 0) {         // W_g . g once per call, as the synthesis path does
        rc = ensure(&h->d_gbias, &h->gbias_bytes, (size_t)B * L * G * sizeof(float));
        if (rc) return rc;
        wn::wn_gbias_kernel<<<dim3(L, B), 128, 0, st>>>(h->d_wg, a->g, h->d_gbias, L, G, c.gin_channels);
        CUDA_TRY(cudaGetLastError());
        ++launches;
        gb = h->d_gbias;
    }
    if (a->test_dense) {
        wnd::transpose_tc_kernel<<<dim3((T + 31) / 32, (O + 31) / 32, B), dim3(32, 8), 0, st>>>(a->test_dense, xdT, T, O);
        CUDA_TRY(cudaGetLastError());
        ++launches;
    }
    {
        const long long n = (long long)BT * R;
        const int blocks = (int)std::min<long long>((n + 255) / 256, 1 << 16);
        wnd::first_conv_kernel<<<blocks, 256, 0, st>>>(a->test_scalar, a->test_index, a->test_dense ? xdT : nullptr,
                                                       h->d_first_w, h->d_first_b, X, B, R, O, T);
        CUDA_TRY(cudaGetLastError());
        ++launches;
    }
    const DenseLayout d = dense_layout(c);
    for (int l = 0; l < L; ++l) {
        const float* lw = h->d_dense + (size_t)l * d.per_layer;
        wnd::DenseGemm p;
        memset(&p, 0, sizeof(p));
        p.A = lw + d.gate_w;
        p.M = G;
        p.K = kw * R + Cc;
        p.T = T;
        p.X = X;
        p.cT = Cc > 0 ? cT : nullptr;
        p.R = R;
        p.kw = kw;
        p.dil = 1 << (l % per_stack);
        p.Cc = Cc;
        p.kwR = kw * R;
        p.bias = lw + d.gate_b;
        p.gbias = gb ? gb + (size_t)l * G : nullptr;
        p.gstride = (long long)L * G;
        p.G2 = G2;
        p.out = Y;
        CUDA_TRY((wnd::launch_dense_gemm<wnd::B_GATE, wnd::EPI_GATE>(p, B, st)));
        wnd::DenseGemm q;
        memset(&q, 0, sizeof(q));
        q.A = lw + d.os_w;
        q.M = R + S;
        q.K = G2;
        q.T = T;
        q.Bsrc = Y;
        q.R = R;
        q.bias = lw + d.os_b;
        q.out = X;
        q.out2 = skip;
        q.first = l == 0;
        CUDA_TRY((wnd::launch_dense_gemm<wnd::B_PLAIN, wnd::EPI_RESSKIP>(q, B, st)));
        launches += 2;
    }
    {   // relu(skip * sqrt(1/L)) -> last_a -> relu -> last_b (wavenet.py:207-210)
        wnd::DenseGemm p;
        memset(&p, 0, sizeof(p));
        p.A = h->d_dense + d.la_w;
        p.M = S;
        p.K = S;
        p.T = T;
        p.Bsrc = skip;
        p.brelu = 1;
        p.bscale = (float)std::sqrt(1.0 / L);
        p.bias = h->d_dense + d.la_b;
        p.out = Y;
        CUDA_TRY((wnd::launch_dense_gemm<wnd::B_PLAIN, wnd::EPI_RELU_BIAS>(p, B, st)));
        wnd::DenseGemm q;
        memset(&q, 0, sizeof(q));
        q.A = h->d_dense + d.lb_w;
        q.M = O;
        q.K = S;
        q.T = T;
        q.Bsrc = Y;
        q.bias = h->d_dense + d.lb_b;
        q.out = a->params_out;
        CUDA_TRY((wnd::launch_dense_gemm<wnd::B_PLAIN, wnd::EPI_BIAS>(q, B, st)));
        launches += 2;
    }
    if (a->flags & WN_FLAG_SOFTMAX) {
        const int blocks = (int)std::min<long long>(((long long)BT + 255) / 256, 1 << 16);
        wnd::col_softmax_kernel<<<blocks, 256, 0, st>>>(a->params_out, B, O, T);
        CUDA_TRY(cudaGetLastError());
        ++launches;
    }
    h->launches += launches;
    h->last_stream = st;
    h->pending = true;
    return WN_OK;
}

int32_t wn_nll(const float* y_bot, int32_t head_kind, int32_t B, int32_t O, int32_t T, const float* y_target,
               const int32_t* class_target, int32_t num_classes, float log_scale_min, float* out_bt, void* stream) {
    if (!y_bot || !out_bt) return fail(WN_ERR_INVALID, "wn_nll: null argument");
    if (B < 1 || T < 1 || O < 1) return fail(WN_ERR_INVALID, "wn_nll: B, O and T must be >= 1");
    if (y_target && class_target) return fail(WN_ERR_INVALID, "wn_nll: give y_target or class_target, not both");
    if (!y_target && !class_target) return fail(WN_ERR_INVALID, "wn_nll: a target is required");
    if (num_classes < 2) return fail(WN_ERR_INVALID, "wn_nll: num_classes must be >= 2");
    if (head_kind == WN_HEAD_MOL) {
        if (O % 3 != 0) return fail(WN_ERR_INVALID, "wn_nll: a MoL head has 3K channels (mixture.py:44)");
    } else if (head_kind == WN_HEAD_GAUSS) {
        if (O != 2 && O % 3 != 0) return fail(WN_ERR_INVALID, "wn_nll: a Gaussian head has 2 or 3K channels (mixture.py:176-181)");
    } else if (head_kind != WN_HEAD_SOFTMAX) {
        return fail(WN_ERR_INVALID, "wn_nll: bad head_kind");
    }
    if (head_kind == WN_HEAD_SOFTMAX ? !class_target : !y_target)
        return fail(WN_ERR_INVALID, head_kind == WN_HEAD_SOFTMAX ? "wn_nll: a softmax head takes class_target"
                                                                  : "wn_nll: a MoL or Gaussian head takes y_target");
    wnd::NllArgs na;
    memset(&na, 0, sizeof(na));
    na.y = y_bot;
    na.yt = y_target;
    na.ct = class_target;
    na.out = out_bt;
    na.head = head_kind == WN_HEAD_MOL ? wnd::NLL_MOL : head_kind == WN_HEAD_GAUSS ? wnd::NLL_GAUSS : wnd::NLL_SOFTMAX;
    na.B = B;
    na.O = O;
    na.T = T;
    na.log_scale_min = log_scale_min;
    na.half_bin = (float)(1.0 / (num_classes - 1));
    na.log_half_nc = (float)std::log((num_classes - 1) / 2.0);
    const long long n = (long long)B * T;
    const int blocks = (int)std::min<long long>((n + 255) / 256, 1 << 16);
    wnd::nll_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(na);
    CUDA_TRY(cudaGetLastError());
    return WN_OK;
}

}  // extern "C"
