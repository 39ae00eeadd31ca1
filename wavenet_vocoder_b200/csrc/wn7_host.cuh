// wn7_host.cuh — planner and weight packer of the synthesis kernel (included by wn_host.cu).
// Pure host arithmetic: exercised without a GPU through wn_plan_only / wn_pack_cta / wn_plan_passes.
#pragma once
#include "wn7_plan.h"

static int align_up7(long long v, int a) { return (int)(((v + a - 1) / a) * a); }

struct JobSpec7 {
    int job, npasses, x_off, klen, deferred;
};

static int32_t build_plan7(const wn_config& c, int batch, int num_sms, long long smem_cap, Wn7Plan& pl,
                           std::vector<Wn7Pass>& passes, std::vector<int>& ringtab) {
    memset(&pl, 0, sizeof(pl));
    passes.clear();
    if (c.abi_version != WN_ABI_VERSION && c.abi_version != 2) return fail(WN_ERR_INVALID, "wn_config.abi_version mismatch");
    if (c.layers < 1 || c.stacks < 1 || c.layers % c.stacks != 0)
        return fail(WN_ERR_INVALID, "layers must be a positive multiple of stacks (wavenet.py:117)");
    if (c.gate_channels < 2 || (c.gate_channels & 1)) return fail(WN_ERR_INVALID, "gate_channels must be even");
    if (c.kernel_size < 1 || c.kernel_size > 8) return fail(WN_ERR_INVALID, "kernel_size out of range [1,8]");
    if (c.residual_channels < 1 || c.skip_channels < 1 || c.out_channels < 1)
        return fail(WN_ERR_INVALID, "channel counts must be positive");
    if (c.residual_channels > 8192 || c.gate_channels > 16384 || c.skip_channels > 8192 || c.out_channels > 8192)
        return fail(WN_ERR_INVALID, "channel count too large (unsupported shape)");
    if (c.cin_channels < 0 || c.cin_channels > 32 * WN7_MAX_CI)
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
    if ((c.gate_channels / 2) & 1 || c.residual_channels & 1 || c.skip_channels & 1)
        return fail(WN_ERR_INVALID, "residual, gate/2 and skip channel counts must be even (16-byte exchange loads)");
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
    pl.NS = pl.L + 3;
    const int BT = pl.BT;

    // ---- how many blocks: every block must own at least one gate pair
    int P = c.num_ctas > 0 ? c.num_ctas : env_int("WN_NUM_CTAS", 0);
    if (P <= 0) {
        const int cap = std::min(num_sms, pl.G2);
        const int per = wn7_ceil_div(pl.G2, cap);
        P = wn7_ceil_div(pl.G2, per);
    }
    if (P > num_sms) return fail(WN_ERR_INVALID, "num_ctas exceeds the SM count (blocks must be co-resident)");
    if (P > pl.G2) return fail(WN_ERR_INVALID, "num_ctas exceeds gate_channels/2");
    pl.P = P;
    auto even = [](int v) { return (v + 1) & ~1; };
    pl.my = wn7_ceil_div(pl.G2, P);
    pl.mx = even(wn7_ceil_div(pl.R, P));
    pl.ms = even(wn7_ceil_div(pl.S, P));
    pl.mo = even(wn7_ceil_div(pl.O, P));
    pl.qA = wn7_ceil_div(2 * pl.my, 4);
    pl.xoff = align_up7(pl.G2, 4);
    // polling warps: one 16-byte load (2 pairs) per lane for the (y, x) vector of one utterance, capped
    {
        // poll_warps: -1 (or WN_POLL_WARPS=-1 / "self") = compute warps 0..3 poll themselves; 0 = choose
        int want = c.poll_warps != 0 ? c.poll_warps : env_int("WN_POLL_WARPS", 0);
        if (want == 0) want = env_int("WN_POLL_DEFAULT", -1);
        if (want < 0) pl.npw = 0;
        else pl.npw = std::max(2, std::min(WN7_MAX_NPW, want));
    }
    pl.nthreads = 32 * (pl.npw + WN7_NCW + 3);

    // ---- passes.  Jobs of a stage kind in order (critical first); every pass is two rows, passes are dealt
    // round-robin over the compute warps continuing across jobs.
    const int G2 = pl.G2, R = pl.R, S = pl.S, xoff = pl.xoff;
    const int npA = pl.my, npB = pl.mx / 2, npD = (pl.kw - 1) * pl.my, npS = pl.ms / 2, npHB = pl.mo / 2;
    std::vector<std::vector<JobSpec7>> kinds(WN7_NKIND);
    kinds[WN7_K_FIRST] = {{WN7_J_A0, npA, xoff, R, 0}};
    kinds[WN7_K_LAYER] = {{WN7_J_A, npA, 0, xoff + R, 0},
                          {WN7_J_B, npB, 0, G2, 0},
                          {WN7_J_D, npD, xoff, R, 1},
                          {WN7_J_S, npS, 0, G2, 1}};
    kinds[WN7_K_TAIL] = {{WN7_J_SL, npS, 0, G2, 0}, {WN7_J_D, npD, xoff, R, 1}};
    kinds[WN7_K_HEAD1] = {{WN7_J_HA, npS, 0, S, 0}};
    kinds[WN7_K_HEAD2] = {{WN7_J_HB, npHB, 0, S, 0}};
    int xin_vals = 128;
    int blob_fill[3] = {0, 0, 0};
    auto blob_of_kind = [](int k) { return k == WN7_K_FIRST ? 0 : (k == WN7_K_LAYER ? 1 : 2); };
    for (int k = 0; k < WN7_NKIND; ++k) {
        std::vector<std::vector<Wn7Pass>> per_warp(WN7_NCW);
        std::vector<int> ncrit(WN7_NCW, 0);
        int rr = 0;
        for (const JobSpec7& js : kinds[k]) {
            if (js.npasses == 0 || js.klen == 0) continue;
            const int nit = wn7_ceil_div(js.klen, 128);
            xin_vals = std::max(xin_vals, js.x_off + 128 * nit);
            if (js.deferred) pl.has_deferred[k] = 1;
            for (int q = 0; q < js.npasses; ++q) {
                Wn7Pass ps;
                memset(&ps, 0, sizeof(ps));
                ps.nit = (int16_t)nit;
                ps.x_off = (int16_t)js.x_off;
                ps.deferred = (int8_t)js.deferred;
                ps.job = (int8_t)js.job;
                // gate pairs / taps are indexed by pair, plain rows by the first row of the pass
                ps.idx = (int16_t)((js.job == WN7_J_A0 || js.job == WN7_J_A || js.job == WN7_J_D) ? q : 2 * q);
                const int w = rr % WN7_NCW;
                ++rr;
                per_warp[w].push_back(ps);
                if (!js.deferred) ncrit[w] = (int)per_warp[w].size();
            }
        }
        for (int w = 0; w < WN7_NCW; ++w) {
            pl.pass_begin[k][w] = (int)passes.size();
            pl.pass_count[k][w] = (int)per_warp[w].size();
            pl.pass_crit[k][w] = ncrit[w];
            for (Wn7Pass& ps : per_warp[w]) {
                int& fill = blob_fill[blob_of_kind(k)];
                ps.w_off = fill;
                fill += ps.nit * 2 * 32 * 4;
                passes.push_back(ps);
            }
        }
    }
    pl.npass = (int)passes.size();
    if (pl.npass > 4096) return fail(WN_ERR_INVALID, "too many passes (unsupported shape)");
    if (xin_vals > 32000) return fail(WN_ERR_INVALID, "stage vector too long");
    pl.xin_vals = align_up7(xin_vals, 4);
    pl.fb_floats = align_up7(blob_fill[0], 4);
    pl.lb_floats = align_up7(blob_fill[1], 4);
    pl.tb_floats = align_up7(blob_fill[2], 4);
    pl.slot_floats = align_up7(std::max(pl.fb_floats, std::max(pl.L > 1 ? pl.lb_floats : 0, pl.tb_floats)), 32);
    pl.cta_w_floats = (long long)pl.fb_floats + (long long)(pl.L - 1) * pl.lb_floats + pl.tb_floats;
    pl.nblobs = pl.L + 1;
    pl.cta_cw_floats = (long long)pl.L * pl.qA * pl.C * 4;
    // ---- biases
    int bo = 0;
    pl.bo_zb = bo; bo += pl.L * 2 * pl.my;
    pl.bo_xb = bo; bo += pl.L * pl.mx;
    pl.bo_sb = bo; bo += pl.L * pl.ms;
    pl.bo_ha = bo; bo += pl.ms;
    pl.bo_hb = bo; bo += pl.mo;
    pl.cta_b_floats = align_up7(bo, 4);

    // ---- exchange map (pairs): one slot per stage, vector order == xin order, slots on 256-byte boundaries
    {
        // WN_EX_SPREAD: 0 contiguous; 1 (default) = 4 pairs (one 32-byte sector) per 256-byte granule; 3 = 8 pairs
        // (64 bytes) per granule.  A contiguous vector sits on a handful of L2 slices and its 128 x npw*32 polling
        // lanes queue there.
        const int sp = env_int("WN_EX_SPREAD", 1);
        pl.ex_a = sp == 1 ? 2 : (sp == 3 ? 3 : (sp == 2 ? 1 : 0));
        pl.ex_b = sp == 0 ? 0 : (sp == 2 ? 4 : 5);
        const long long linear = (long long)std::max(std::max(xoff + R, S), pl.O) * BT + 2;
        pl.slot_pairs = align_up7((((linear >> pl.ex_a) + 1) << pl.ex_b) + 32, 32);
        pl.ex_pairs = (long long)pl.NS * pl.slot_pairs + 32;
        pl.gate_cycles = env_int("WN_GATE_CYCLES", 0);
        pl.backoff_ns = env_int("WN_BACKOFF_NS", 0);
    }

    // ---- history rings: tap k (0 = oldest) is consumed (kw-1-k)*d steps later; one position = 4qA*BT floats
    ringtab.assign((size_t)pl.L * std::max(pl.kw - 1, 0) * 2, 0);
    long long pos = 0;
    for (int l = 0; l < pl.L; ++l)
        for (int k = 0; k < pl.kw - 1; ++k) {
            const int D = (pl.kw - 1 - k) * wn7_dilation(pl, l);
            ringtab[((size_t)l * (pl.kw - 1) + k) * 2] = (int)pos;
            ringtab[((size_t)l * (pl.kw - 1) + k) * 2 + 1] = D;
            pos += D;
        }
    pl.ring_pos_total = pos;
    const long long ring_bytes = pos * 4 * pl.qA * BT * 4;

    // ---- shared memory map
    auto layout = [&](bool ring_smem) -> long long {
        long long off = 0;
        auto take = [&](long long bytes, int al) {
            off = ((off + al - 1) / al) * al;
            long long r = off;
            off += bytes;
            return (int)r;
        };
        const long long tab = (long long)pl.L * 4 * pl.qA * BT * 4;
        pl.sm_bar = take((long long)(2 * pl.nblobs + 20) * 8, 16);
        pl.sm_misc = take(16, 16);
        pl.sm_in = take((long long)BT * 8 + (pl.input_kind == WN_INPUT_ONEHOT ? (long long)BT * pl.O * 4 : 0), 16);
        pl.sm_pass = take((long long)pl.npass * (long long)sizeof(Wn7Pass), 16);
        pl.sm_ringtab = take((long long)ringtab.size() / 2 * 3 * 4 + 16, 16);
        pl.sm_xin = take(2LL * pl.xin_vals * BT * 4, 16);
        pl.sm_sb = take(tab, 16);
        pl.sm_pre = take(tab, 16);
        pl.sm_cond = take(pl.C > 0 ? 2 * tab : 16, 16);
        pl.sm_bias = take((long long)pl.cta_b_floats * 4, 16);
        pl.sm_skipacc = take((long long)pl.ms * BT * 4, 16);
        pl.sm_xown = take((long long)2 * pl.mx * BT * 4, 16);
        pl.sm_hs = take((long long)(pl.O * BT + 2) * 4, 16);
        pl.sm_noise = take((long long)BT * (pl.O + 2) * 4, 16);
        pl.sm_x0w = take((long long)2 * R * 4, 16);
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

// ------------------------------------------------------------------------------------------
// packer
// ------------------------------------------------------------------------------------------
// element of the matrix a pass multiplies: row r (0/1) of pass `ps` of block p in stage `stage`, column = entry k
// of the stage input vector ([y | pad | x] for the layer stages, [S] for the head stages).  0 for padding.
struct Pack7 {
    const Wn7Plan& pl;
    const wn_weights& w;
    const Folded& f;
    int p;
    int y0, ny, x0, nx, s0, ns, a0, na, b0, nb;
    Pack7(const Wn7Plan& pl_, const wn_weights& w_, const Folded& f_, int p_) : pl(pl_), w(w_), f(f_), p(p_) {
        wn7_part(pl.G2, pl.P, p, y0, ny);
        wn7_part(pl.R, pl.P, p, x0, nx);
        wn7_part(pl.S, pl.P, p, s0, ns);
        wn7_part(pl.S, pl.P, p, a0, na);
        wn7_part(pl.O, pl.P, p, b0, nb);
    }
    int ycol(int k) const { return (k >= 0 && k < pl.G2) ? k : -1; }
    int xcol(int k) const { return (k >= pl.xoff && k < pl.xoff + pl.R) ? k - pl.xoff : -1; }
    int scol(int k) const { return (k >= 0 && k < pl.S) ? k : -1; }
    float elem(const Wn7Pass& ps, int stage, int r, int k) const {
        const int R = pl.R, G2 = pl.G2, kw = pl.kw, S = pl.S;
        int col;
        switch (ps.job) {
            case WN7_J_A0: {
                if (ps.idx >= ny || (col = xcol(k)) < 0) return 0.f;
                const int row = r ? G2 + y0 + ps.idx : y0 + ps.idx;
                return f.V[0][(size_t)row * R + col];
            }
            case WN7_J_A: {
                if (ps.idx >= ny) return 0.f;
                const int row = r ? G2 + y0 + ps.idx : y0 + ps.idx;
                if ((col = ycol(k)) >= 0) return f.M[stage - 1][(size_t)row * G2 + col];
                if ((col = xcol(k)) >= 0) return f.V[stage][(size_t)row * R + col];
                return 0.f;
            }
            case WN7_J_B: {
                const int j = ps.idx + r;
                if (j >= nx || (col = ycol(k)) < 0) return 0.f;
                return w.layers[stage - 1].out_w[(size_t)(x0 + j) * G2 + col];
            }
            case WN7_J_D: {
                const int tap = ps.idx / pl.my, i = ps.idx % pl.my;
                if (i >= ny || (col = xcol(k)) < 0) return 0.f;
                const int row = r ? G2 + y0 + i : y0 + i;
                return w.layers[stage - 1].conv_w[(size_t)row * kw * R + (size_t)tap * R + col];   // conv.py:56-61: col = k*R + r
            }
            case WN7_J_S:
            case WN7_J_SL: {
                const int j = ps.idx + r;
                if (j >= ns || (col = ycol(k)) < 0) return 0.f;
                return w.layers[stage - 1].skip_w[(size_t)(s0 + j) * G2 + col];
            }
            case WN7_J_HA: {
                const int j = ps.idx + r;
                if (j >= na || (col = scol(k)) < 0) return 0.f;
                return w.last_a_w[(size_t)(a0 + j) * S + col];
            }
            default: {
                const int j = ps.idx + r;
                if (j >= nb || (col = scol(k)) < 0) return 0.f;
                return w.last_b_w[(size_t)(b0 + j) * S + col];
            }
        }
    }
};

// packed image of block `p`: first blob, L-1 layer blobs, tail blob; tiles in pass order, [j][row][lane][4 k]
static void pack7_cta(const Wn7Plan& pl, const std::vector<Wn7Pass>& passes, const wn_weights& w, const Folded& f, int p,
                      float* out) {
    memset(out, 0, (size_t)pl.cta_w_floats * sizeof(float));
    Pack7 pk(pl, w, f, p);
    auto pack_kind = [&](int kind, int stage, float* blob) {
        for (int wv = 0; wv < WN7_NCW; ++wv)
            for (int i = 0; i < pl.pass_count[kind][wv]; ++i) {
                const Wn7Pass& ps = passes[pl.pass_begin[kind][wv] + i];
                float* tile = blob + ps.w_off;
                for (int j = 0; j < ps.nit; ++j)
                    for (int r = 0; r < 2; ++r)
                        for (int lane = 0; lane < 32; ++lane) {
                            float* dst = tile + (((size_t)j * 2 + r) * 32 + lane) * 4;
                            const int k0 = ps.x_off + 4 * (lane + 32 * j);
                            for (int kk = 0; kk < 4; ++kk) dst[kk] = pk.elem(ps, stage, r, k0 + kk);
                        }
            }
    };
    pack_kind(WN7_K_FIRST, 0, out);
    for (int s = 1; s < pl.L; ++s) pack_kind(WN7_K_LAYER, s, out + wn7_blob_off(pl, s));
    float* tb = out + wn7_blob_off(pl, pl.L);
    pack_kind(WN7_K_TAIL, pl.L, tb);
    pack_kind(WN7_K_HEAD1, pl.L + 1, tb);
    pack_kind(WN7_K_HEAD2, pl.L + 2, tb);
}

// biases of the rows block p owns
static void pack7_bias(const Wn7Plan& pl, const wn_weights& w, const Folded& f, int p, float* out) {
    memset(out, 0, (size_t)pl.cta_b_floats * sizeof(float));
    Pack7 pk(pl, w, f, p);
    for (int l = 0; l < pl.L; ++l) {
        for (int i = 0; i < pk.ny; ++i) {
            out[pl.bo_zb + l * 2 * pl.my + 2 * i] = f.zb[l][pk.y0 + i];
            out[pl.bo_zb + l * 2 * pl.my + 2 * i + 1] = f.zb[l][pl.G2 + pk.y0 + i];
        }
        if (l >= 1)
            for (int j = 0; j < pk.nx; ++j)
                out[pl.bo_xb + l * pl.mx + j] = w.layers[l - 1].out_b ? w.layers[l - 1].out_b[pk.x0 + j] : 0.f;
        for (int j = 0; j < pk.ns; ++j)
            out[pl.bo_sb + l * pl.ms + j] = w.layers[l].skip_b ? w.layers[l].skip_b[pk.s0 + j] : 0.f;
    }
    for (int j = 0; j < pk.na; ++j) out[pl.bo_ha + j] = w.last_a_b ? w.last_a_b[pk.a0 + j] : 0.f;
    for (int j = 0; j < pk.nb; ++j) out[pl.bo_hb + j] = w.last_b_b ? w.last_b_b[pk.b0 + j] : 0.f;
}

// conditioning rows of block p: [L][qA][C][4], gate rows a_i, b_i interleaved
static void pack7_cw(const Wn7Plan& pl, const wn_weights& w, int p, float* out) {
    if (pl.C <= 0) return;
    memset(out, 0, (size_t)pl.cta_cw_floats * sizeof(float));
    int y0, ny;
    wn7_part(pl.G2, pl.P, p, y0, ny);
    for (int l = 0; l < pl.L; ++l) {
        const float* cwm = w.layers[l].cond_w;
        float* grp = out + (size_t)l * pl.qA * pl.C * 4;
        for (int ro = 0; ro < 2 * ny; ++ro) {
            const int row = (ro & 1) ? pl.G2 + y0 + (ro >> 1) : y0 + (ro >> 1);
            for (int ch = 0; ch < pl.C; ++ch) grp[((size_t)(ro >> 2) * pl.C + ch) * 4 + (ro & 3)] = cwm[(size_t)row * pl.C + ch];
        }
    }
}
