// wn_plan.h — the execution plan shared by the host planner/packer and the persistent kernel.
//
// One generated sample is a chain of small matrix-vector "stages" with a strict serial
// dependency (reference wavenet.py:296-336).  The engine spreads every stage over P cooperating
// thread blocks (one per SM): block p owns a fixed slice of the OUTPUT rows of every matrix, so
// its weights never move between SMs, and the stage outputs (a few hundred floats) are exchanged
// through tagged slots in L2.  This header fixes (a) which rows a block owns, (b) the layout of
// the per-block packed weight image ("blobs", one per layer plus one for the head), (c) the
// shared-memory map, and (d) the exchange-slot map.  All of it is plain arithmetic on the model
// shape so the host tests can check the packer without a GPU.
#pragma once
#include <stdint.h>

#ifndef WN_HD
#ifdef __CUDACC__
#define WN_HD __host__ __device__ __forceinline__
#else
#define WN_HD inline
#endif
#endif

#define WN_NT 256                 // compute threads per block (8 warps)
#define WN_NWARP (WN_NT / 32)
#define WN_AUX_WARPS 2            // +1 weight-streaming (TMA) warp, +1 conditioning warp
#define WN_NTHREADS (WN_NT + 32 * WN_AUX_WARPS)
#define WN_MAXE 8                 // a stage input vector has at most WN_MAXE*128 entries (128-thread groups)
#define WN_MAX_BT 8               // utterances processed together by one launch
#define WN_MAX_CI 4               // local-conditioning channels <= 32*WN_MAX_CI

struct WnPlan {
    // ---- model shape (wavenet.py:98-111)
    int L, per_stack, R, G, G2, S, O, kw, C, gin, input_kind, head_kind, Kmix;
    // ---- partition: P blocks; max rows a block owns in each matrix
    int P;
    int NYm;      // gate pairs (rows j and j+G/2 of the dilated conv, modules.py:138)
    int NXm;      // rows of conv1x1_out  (modules.py:160)
    int NSm;      // rows of conv1x1_skip (modules.py:157)
    int NAm;      // rows of last_conv_layers[1]
    int NBm;      // rows of last_conv_layers[3]
    int RA;       // 2*NYm : rows of the dilated conv a block evaluates (a_j, b_j interleaved)
    // row quads per group ("quad-major" layout [quad][k][4 rows], one 16-byte smem load feeds 4 rows)
    int NQ_A, NQ_D, NQ_BO, NQ_BS, NQ_HA, NQ_HB;
    // ---- blobs (offsets in floats).  Stage s of a step evaluates layer s from (y_{s-1}, x_{s-1}):
    //   z_s = M_{s-1} y_{s-1} + V_s x_{s-1} + ...   with V_s = sqrt(.5) W_s[:,:,kw-1],  M_{s-1} = V_s Wo_{s-1}
    // so conv1x1_out of layer s-1 is folded into the current tap of layer s and one broadcast per
    // layer (y_s and x_s together) is enough.
    // first blob (stage 0): current tap of layer 0 + bias
    int fb_Zx, fb_zb, fb_floats;
    // layer blob (stage s = 1..L-1)
    int lb_Zy;      // M_{s-1} rows          [NQ_A][G2][4]
    int lb_Zx;      // V_s rows              [NQ_A][R][4]
    int lb_Xo;      // conv1x1_out_{s-1} rows [NQ_BO][G2][4]  (the residual stream itself, published as x_s)
    int lb_Td;      // older taps of layer s-1 [NQ_D][R][4]   (deferred: queued for steps t+d, t+2d ...)
    int lb_Sk;      // conv1x1_skip_{s-1} rows [NQ_BS][G2][4] (deferred)
    int lb_zb, lb_xb, lb_sb;   // biases: conv_b_s + V_s bo_{s-1} | bo_{s-1} | bs_{s-1}
    int lb_floats;
    // tail blob (stage L + head): older taps and skip rows of layer L-1, then the two head matrices
    int tb_Td, tb_Sk, tb_sb, tb_Ha, tb_Hab, tb_Hb, tb_Hbb, tb_floats;
    int slot_floats;            // shared-memory slot size (>= every blob)
    long long cta_w_floats;     // packed floats per block = fb + (L-1)*lb + tb
    int nblobs;                 // L + 1 per step
    int nres;                   // blobs [0,nres) stay resident in shared memory for the whole call
    int nring;                  // the others stream through nring slots every step
    int l2_pf;                  // streamed blobs the weight warp prefetches into L2 ahead of its ring copies (0: none)
    // ---- conditioning weights (kept in L2, read by the conditioning warp): [L][NQ_A][C][4]
    long long cta_cw_floats;
    // ---- exchange: element offsets (multiply by BT for pairs) of each vector inside one copy.
    // exchange s (0..L-1) carries y_s (G2) then x_s (R); then skip (S), head hidden (S), head out (O)
    int NE;                     // exchanges per step = L+3
    int ncopy;
    int ex_yx, ex_sk, ex_h1, ex_h2, ex_elems;
    long long copy_stride_pairs;
    // ---- batch tile
    int BT;
    // ---- history rings of the older-tap products
    int ring_in_smem;
    long long ring_pos_total;   // sum over (layer, tap) of the delay; one position = RA4*BT floats
    int RA4;                    // 4*NQ_A
    // ---- shared memory map (byte offsets)
    int sm_bar, sm_misc, sm_ringtab, sm_xs, sm_red1, sm_red2, sm_sb, sm_cond, sm_skipacc, sm_hs,
        sm_noise, sm_in, sm_first, sm_ring, sm_slots, smem_bytes;
    int red1_floats;            // one of the two critical-partials buffers (alternating by stage)
    int red2_floats;            // one of the two deferred-partials buffers
    float skip_scale;           // sqrt(1/L), wavenet.py:313
    int xc_shift, xstride;      // exchange layout: 2^xc_shift pairs per chunk, chunks xstride pairs apart
};
WN_HD long long wn_pair_index_(const WnPlan& pl, long long lin) {
    return (long long)(((unsigned long long)lin >> pl.xc_shift) * (unsigned long long)pl.xstride +
                       ((unsigned long long)lin & ((1ull << pl.xc_shift) - 1ull)));
}

// balanced split of `rows` over P blocks: block p owns [base, base+cnt)
WN_HD void wn_part(int rows, int P, int p, int& base, int& cnt) {
    int q = rows / P, r = rows % P;
    base = p * q + (p < r ? p : r);
    cnt = q + (p < r ? 1 : 0);
}

WN_HD int wn_ceil_div(int a, int b) { return (a + b - 1) / b; }
// Exchange layout: the L2 slice hash takes higher address bits, so a contiguous few-KB vector
// would sit on a handful of slices and all P readers would queue there.  Pairs are therefore
// stored in 256-byte chunks (32 pairs: what one warp polls with one load) spaced 4352 bytes apart.
#define WN_XCHUNK 32
#define WN_XSTRIDE 544
#define wn_pair_index(lin) wn_pair_index_(pl, (lin))
WN_HD long long wn_pair_index_(const struct WnPlan& pl, long long lin);
WN_HD int wn_dilation(const WnPlan& pl, int l) { return 1 << (l % pl.per_stack); }
// exchange ids within a step (tag = t*(L+3) + id + 1)
WN_HD int wn_eid_yx(int s) { return s; }              // (y_s, x_s), s = 0..L-1
WN_HD int wn_eid_sk(const WnPlan& pl) { return pl.L; }
WN_HD int wn_eid_h1(const WnPlan& pl) { return pl.L + 1; }
WN_HD int wn_eid_h2(const WnPlan& pl) { return pl.L + 2; }
// float offset of blob i inside a block's packed image, and its size
WN_HD long long wn_blob_off(const WnPlan& pl, int i) {
    return i == 0 ? 0 : (long long)pl.fb_floats + (long long)(i - 1) * pl.lb_floats;
}
WN_HD int wn_blob_floats(const WnPlan& pl, int i) {
    return i == 0 ? pl.fb_floats : (i < pl.L ? pl.lb_floats : pl.tb_floats);
}
