// wn7_kernel.cuh — the persistent sm_90a synthesis kernel.
//
// One launch == one WaveNet.incremental_forward() call (reference wavenet.py:215-343): the whole T-step loop,
// including the sampler, runs on the device.  P thread blocks (one per SM, cooperative launch) each own a fixed slice
// of the output rows of every matrix (wn7_plan.h).
//
// Stages of one generated sample (the algebra is the reference's, re-associated on the host):
//   stage 0      : x_0 (first 1x1 conv of the fed-back sample, wavenet.py:308; every block evaluates it locally) ->
//                  current tap of layer 0 -> tanh*sigmoid -> publish y_0
//   stage s < L  : from (y_{s-1}, x_{s-1}):  z_s = M_{s-1} y_{s-1} + V_s x_{s-1} + bias + conditioning + queued older
//                  taps, with V_s = sqrt(.5) W_s[:,:,kw-1] and M_{s-1} = V_s Wo_{s-1} folded on the host (conv1x1_out of
//                  layer s-1 rides inside the current tap of layer s: ONE exchange per layer),
//                  x_s = (Wo_{s-1} y_{s-1} + bo + x_{s-1}) sqrt(.5)  (modules.py:160-162) -> publish (y_s, x_s).
//                  Deferred (off the critical path): the OLDER taps' products W_{s-1}[:,:,k<kw-1] x_{s-1}(t), queued for
//                  steps t+d, t+2d (replaces the input shift register of conv.py:32-44 by a queue of output
//                  products), and conv1x1_skip_{s-1}, accumulated in layer order (wavenet.py:312).
//   stage L      : skip rows of the last layer -> total skip * sqrt(1/L) -> ReLU -> publish
//   stage L+1,+2 : last_conv_layers (wavenet.py:315-319)
// then every block reads the O head outputs and evaluates the sampler (mixture.py) redundantly from identical noise, so
// the sample itself needs no broadcast.
//
// Exchange: every value travels as an 8-byte (value, tag) pair (tag = global stage index + 1) written with one
// st.relaxed.gpu and read with 16-byte ld.relaxed.gpu (two pairs): data and "ready" flag are one word -- no fence, no
// separate barrier, one L2 write + one L2 read per hop.
//
// Warp roles:
//   pollers (npw) : copy the stage vector from L2 into shared memory, ONE 16-byte coherent load per lane where the
//                   vector allows (a lane's coherent loads do not overlap), then release it with an
//                   mbarrier; also evaluate x_0 and run the sampler.
//   compute (8)   : passes (wn7_plan.h): two complete rows per warp from shared-memory weights, 32-lane butterfly,
//                   finalisation (bias, gate, residual, ReLU, ring / skip bookkeeping) and st.relaxed.gpu publish by the
//                   lanes the butterfly ends in.  Critical passes first, deferred ones (queued taps, skip rows) after.
//   HK            : once per step: ring positions, next step's pre-sum table (bias + conditioning + queued taps).
//   TMA           : streams the packed weight blobs global -> shared with cp.async.bulk + mbarrier (SASS UBLKCP).
//   COND          : local-conditioning projection of the block's gate rows, one step ahead.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include "wn7_plan.h"

struct Wn7Ptrs {
    const float* wpack;        // [P][cta_w_floats]
    const float* cwpack;       // [P][cta_cw_floats]
    const float* bpack;        // [P][cta_b_floats]
    const Wn7Pass* passes;     // [npass]
    const float* gbias;        // [B][L][G] = Wg_l . g_b   (NULL without global conditioning)
    const float* first_w;      // scalar input: [R];  one-hot input: transposed [O][R]
    const float* first_b;      // [R]
    uint2* xbuf;               // exchange pairs
    float* ring_g;             // [P][ring floats] when the history rings do not fit in shared memory
    const int* ringtab;        // [L*(kw-1)*2] : (offset in positions, delay D)
    int* err;                  // [4] device fault word, what, block, thread
    // ---- per call
    const float* c;
    const float* initial;
    const float* initial_dense;   // one-hot input: (B,O) dense start vector or NULL
    const int* initial_rows;      // one-hot input: (B) start class per utterance or NULL
    const float* test_scalar;
    const int* test_index;
    const float* test_dense;
    const float* u1;
    const float* u2;
    const float* z;
    const float* e;
    float* out_scalar;
    int* out_index;
    float* out_dense;
    float* params_out;
    int B, Btot, b0, T, T_test, initial_index;   // B rows in this launch; noise is strided by Btot
    unsigned flags;
    int noise_kind;
    unsigned long long seed;
    long long timeout_cycles;
    long long* prof;           // optional [P][16] cycle counters
    int warp_reverse;          // 1: logical warp = (warps-1) - physical warp
    int defer_gate;            // 1: deferred passes start only after every compute warp has published its critical rows
    // ---- streaming (wn_stream_generate, wn7_stream_kernel): a launch continues an utterance at absolute step t_base
    unsigned t_base;           // absolute step of local step 0 (Philox counters, ring positions)
    float* state;              // [P][ring floats] rings then the feedback [BT] s_in, [BT] s_idx, [BT][O] s_dense
    int state_load;            // 1: rings and step-0 feedback come from `state`; 0: zero rings, feedback from initial*
};

// floats of a stream's state: the history rings of one block, then (once) the feedback of the next step
__host__ __device__ inline long long wn7_state_ring_floats(const Wn7Plan& pl) {
    return pl.ring_pos_total * 4 * pl.qA * pl.BT;
}
__host__ __device__ inline long long wn7_state_feedback_floats(const Wn7Plan& pl) {
    return 2LL * pl.BT + (pl.input_kind != 0 ? (long long)pl.BT * pl.O : 0);
}

#define WN7_FLAG_SOFTMAX 1u
#define WN7_FLAG_QUANTIZE 2u

namespace wn7 {

// ------------------------------------------------------------------------------------------
// PTX helpers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// TMA 1-D bulk copy global -> shared, completion counted in bytes on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ uint4 ld_pair2(const uint2* p) {
    uint4 v;
    asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_pair(uint2* p, float v, uint32_t tag) {
    asm volatile("st.relaxed.gpu.global.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(__float_as_uint(v)), "r"(tag) : "memory");
}
__device__ __forceinline__ int ld_flag(const int* p) {
    int v;
    asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

__host__ __device__ constexpr int ilog2c(int v) { return v <= 1 ? 0 : 1 + ilog2c(v >> 1); }

// Philox4x32-10 (counter-based; the same (seed, step, utterance, slot) gives the same draw in every block, which
// is what lets all blocks sample redundantly)
__device__ __forceinline__ uint4 philox4(uint4 ctr, uint2 key) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z;
        ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
        key.x += 0x9E3779B9u;
        key.y += 0xBB67AE85u;
    }
    return ctr;
}
__device__ __forceinline__ float u01(uint32_t r) {   // (0,1), then mapped like uniform_(1e-5, 1-1e-5)
    const float u = ((r >> 8) + 0.5f) * (1.0f / 16777216.0f);
    return 1e-5f + u * (1.0f - 2e-5f);
}

// slow path of every spin loop: has another block faulted / have we waited too long?
__device__ __forceinline__ bool check_abort_slow(volatile int* s_abort, int* err, long long timeout, uint32_t what, int p,
                                              long long& t0) {
    if (*s_abort) return true;
    if (ld_flag(err) != 0) {
        *s_abort = 1;
        return true;
    }
    const long long now = clock64();
    if (t0 == 0) {
        t0 = now;
        return false;
    }
    if (now - t0 > timeout) {
        if (atomicCAS(err, 0, 1) == 0) {
            err[1] = (int)what;
            err[2] = p;
            err[3] = (int)threadIdx.x;
        }
        *s_abort = 1;
        return true;
    }
    return false;
}

// 32-lane butterfly: every level that still has more than one value also halves the value set.  Afterwards value v
// (v < NV) sits in v[0] of lane v*32/NV (and of the lanes up to the next value's).
template <int NV>
__device__ __forceinline__ void reduce32(float (&v)[NV], int lane) {
    int n = NV;
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        if (n > 1) {
            n >>= 1;
            const bool hi = (lane & off) != 0;
#pragma unroll
            for (int i = 0; i < NV / 2; ++i) {
                if (i < n) {
                    const float send = hi ? v[i] : v[i + n];
                    const float keep = hi ? v[i + n] : v[i];
                    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
                }
            }
        } else {
            v[0] += __shfl_xor_sync(0xffffffffu, v[0], off);
        }
    }
}

#define WN7_NSP 4                 // compute warps that poll when there are no dedicated polling warps

// SELF: no dedicated polling warps -- compute warps 0..WN7_NSP-1 poll the vector themselves (their share each), meet
// at a named barrier and go straight into their passes; the other compute warps are released through the mbarrier.
// STREAM: the kernel of wn_stream_generate (absolute steps, history and feedback in a state buffer); a separate
// __global__ (wn7_stream_kernel), so the whole-utterance kernels compile exactly as without it.
template <int BT, bool SELF, bool STREAM = false>
struct Engine {
    static constexpr int NV = 2 * BT;          // values of one pass: 2 rows x BT utterances, index r*BT + b
    const Wn7Plan& pl;
    const Wn7Ptrs& pp;
    unsigned char* sm;
    int tid, warp, lane, p;
    // Shared-memory regions are addressed through accessors that recompute `sm + offset` from the plan (a uniform
    // constant-bank load) instead of ~30 pointer members that would stay live in registers across the whole loop.
    template <typename T> __device__ __forceinline__ T* at(int off) const { return reinterpret_cast<T*>(sm + off); }
    __device__ __forceinline__ uint64_t* bar_full_() const { return at<uint64_t>(pl.sm_bar); }
    __device__ __forceinline__ uint64_t* bar_empty_() const { return bar_full_() + pl.nres + pl.nring; }
    __device__ __forceinline__ uint64_t* bar_cfull_() const { return bar_empty_() + (pl.nring > 0 ? pl.nring : 1); }
    __device__ __forceinline__ uint64_t* bar_cempty_() const { return bar_cfull_() + 2; }
    __device__ __forceinline__ uint64_t* bar_in_() const { return bar_cfull_() + 4; }
    __device__ __forceinline__ uint64_t* bar_free_() const { return bar_cfull_() + 6; }
    __device__ __forceinline__ uint64_t* bar_pre_() const { return bar_cfull_() + 8; }
    __device__ __forceinline__ uint64_t* bar_x0_() const { return bar_cfull_() + 9; }
    __device__ __forceinline__ uint64_t* bar_ps_() const { return bar_cfull_() + 10; }
    __device__ __forceinline__ uint64_t* bar_dstep_() const { return bar_cfull_() + 11; }
    __device__ __forceinline__ uint64_t* bar_crit_() const { return bar_cfull_() + 12; }      // [2]
    __device__ __forceinline__ volatile int* s_abort_() const { return at<volatile int>(pl.sm_misc); }
    __device__ __forceinline__ volatile int* s_skipcnt_() const { return at<volatile int>(pl.sm_misc) + 1; }   // skip-row passes_() completed
    __device__ __forceinline__ Wn7Pass* passes_() const { return at<Wn7Pass>(pl.sm_pass); }
    __device__ __forceinline__ int* ringtab_() const { return at<int>(pl.sm_ringtab); }       // [e][3]: offset, delay, t mod delay
    __device__ __forceinline__ float* xin_() const { return at<float>(pl.sm_xin); }
    __device__ __forceinline__ float* sb_() const { return at<float>(pl.sm_sb); }
    __device__ __forceinline__ float* pre_() const { return at<float>(pl.sm_pre); }
    __device__ __forceinline__ float* cond_() const { return at<float>(pl.sm_cond); }
    __device__ __forceinline__ float* bias_() const { return at<float>(pl.sm_bias); }
    __device__ __forceinline__ float* skipacc_() const { return at<float>(pl.sm_skipacc); }
    __device__ __forceinline__ float* xown_() const { return at<float>(pl.sm_xown); }
    __device__ __forceinline__ float* x0own_() const { return at<float>(pl.sm_xown) + pl.mx * BT; }
    __device__ __forceinline__ float* hs_() const { return at<float>(pl.sm_hs); }
    __device__ __forceinline__ float* noise_() const { return at<float>(pl.sm_noise); }
    __device__ __forceinline__ float* x0w_() const { return at<float>(pl.sm_x0w); }
    __device__ __forceinline__ float* slots_() const { return at<float>(pl.sm_slots); }
    __device__ __forceinline__ volatile float* ring_() const {
        return pl.ring_in_smem ? at<volatile float>(pl.sm_ring)
                               : (volatile float*)(pp.ring_g + (size_t)p * pl.ring_pos_total * 4 * pl.qA * BT);
    }
    __device__ __forceinline__ float* s_in_() const { return at<float>(pl.sm_in); }                  // [BT] scalar feedback
    __device__ __forceinline__ int* s_idx_() const { return at<int>(pl.sm_in) + BT; }                // [BT] class feedback
    __device__ __forceinline__ float* s_dense_() const { return at<float>(pl.sm_in) + 2 * BT; }      // [BT][O] dense feedback
    bool dead;
    // rows this block owns
    int y0, ny, x0r, nx, s0, ns, a0, na, b0, nb;

    __device__ Engine(const Wn7Plan& pl_, const Wn7Ptrs& pp_, unsigned char* sm_) : pl(pl_), pp(pp_), sm(sm_) {
        // logical warp = last physical warp first: the SM's issue arbiter prefers the highest warp id among eligible
        // warps, and the critical compute warps are the first logical ones
        lane = threadIdx.x & 31;
        warp = pp.warp_reverse ? (pl.nthreads / 32 - 1) - (int)(threadIdx.x >> 5) : (int)(threadIdx.x >> 5);
        tid = warp * 32 + lane;
        p = blockIdx.x;
        dead = false;
        wn7_part(pl.G2, pl.P, p, y0, ny);
        wn7_part(pl.R, pl.P, p, x0r, nx);
        wn7_part(pl.S, pl.P, p, s0, ns);
        wn7_part(pl.S, pl.P, p, a0, na);
        wn7_part(pl.O, pl.P, p, b0, nb);
    }

    // ---- watchdog: a stuck wait sets the device fault word and makes every block unwind
    __device__ __forceinline__ bool check_abort(uint32_t what, long long& t0) {
        return check_abort_slow(s_abort_(), pp.err, pp.timeout_cycles, what, p, t0);
    }
    // Waits are WARP-COLLECTIVE (all 32 lanes call them together) and return a warp-uniform verdict, so that a
    // watchdog abort never leaves some lanes of a warp behind in a later shuffle or vote.  `relaxed` waits
    // (anything off the critical path) back off with nanosleep.
    template <bool relaxed = false>
    __device__ __forceinline__ bool wait_bar(uint64_t* bar, uint32_t parity, uint32_t what) {
        if (!dead) {
            uint32_t spins = 0;
            long long t0 = 0;
            while (!mbar_try_wait(bar, parity)) {
                if (relaxed) __nanosleep(64);
                if (((++spins) & (relaxed ? 63u : 255u)) == 0 && check_abort(what, t0)) {
                    dead = true;
                    break;
                }
            }
        }
        dead = __any_sync(0xffffffffu, dead);
        return !dead;
    }
    // single-lane variant (the TMA lane)
    template <bool relaxed = false>
    __device__ __forceinline__ bool wait_bar_lane(uint64_t* bar, uint32_t parity, uint32_t what) {
        if (dead) return false;
        uint32_t spins = 0;
        long long t0 = 0;
        while (!mbar_try_wait(bar, parity)) {
            if (relaxed) __nanosleep(64);
            if (((++spins) & (relaxed ? 63u : 255u)) == 0 && check_abort(what, t0)) {
                dead = true;
                return false;
            }
        }
        return true;
    }
    __device__ __forceinline__ void wait_count(volatile int* cnt, int need, uint32_t what) {
        if (!dead) {
            uint32_t spins = 0;
            long long t0 = 0;
            while (*cnt < need) {
                if (((++spins) & 255u) == 0 && check_abort(what, t0)) {
                    dead = true;
                    break;
                }
            }
            __threadfence_block();
        }
        dead = __any_sync(0xffffffffu, dead);
    }
    // barrier over the polling warps with a watchdog (a plain bar.sync would hang if one of them aborted)
    uint32_t ps_par = 0;
    __device__ __forceinline__ void poller_sync() {
        if constexpr (SELF) {
            // named barrier over the polling compute warps that also OR-reduces the abort flag: every thread always
            // reaches it (all spin loops have a watchdog), so an abort cannot leave a warp behind
            uint32_t r;
            asm volatile(
                "{\n\t.reg .pred p, q;\n\t"
                "setp.ne.u32 p, %1, 0;\n\t"
                "bar.red.or.pred q, 1, %2, p;\n\t"
                "selp.u32 %0, 1, 0, q;\n\t}"
                : "=r"(r)
                : "r"((uint32_t)dead), "n"(32 * WN7_NSP)
                : "memory");
            dead = r != 0;
        } else {
            __syncwarp();
            if (!dead && lane == 0) mbar_arrive(bar_ps_());          // one arrival per polling warp
            wait_bar(bar_ps_(), ps_par, 0x00200000u);
            ps_par ^= 1u;
        }
    }
    __device__ __forceinline__ int n_poll_warps() const { return SELF ? WN7_NSP : pl.npw; }
    // `slot` = pair offset of the stage slot, `i` = linear pair index inside it
    __device__ __forceinline__ void publish(long long slot, long long i, float v, uint32_t tag) {
        st_pair(pp.xbuf + slot + wn7_phys(pl, i), v, tag);
    }

    // ======================================================================================
    // weight streaming warp
    // ======================================================================================
    __device__ void tma_loop() {
        if (lane != 0) return;
        const float* base = pp.wpack + (size_t)p * pl.cta_w_floats;
        for (int i = 0; i < pl.nres; ++i) {
            const uint32_t bytes = (uint32_t)wn7_blob_floats(pl, i) * 4u;
            mbar_expect_tx(&bar_full_()[i], bytes);
            bulk_g2s(slots_() + (size_t)i * pl.slot_floats, base + wn7_blob_off(pl, i), bytes, &bar_full_()[i]);
        }
        const int nstream = pl.nblobs - pl.nres;
        if (nstream <= 0) return;
        const uint32_t total = (uint32_t)pp.T * (uint32_t)nstream;
        int i = pl.nres;
        uint32_t s = 0, u = 0;
        for (uint32_t js = 0; js < total; ++js) {
            if (u > 0) {
                if (!wait_bar_lane<true>(&bar_empty_()[s], (u - 1) & 1u, 0x40000000u | s)) return;
            }
            const uint32_t bytes = (uint32_t)wn7_blob_floats(pl, i) * 4u;
            uint64_t* fb = &bar_full_()[pl.nres + s];
            mbar_expect_tx(fb, bytes);
            bulk_g2s(slots_() + (size_t)(pl.nres + s) * pl.slot_floats, base + wn7_blob_off(pl, i), bytes, fb);
            if (++i == pl.nblobs) i = pl.nres;
            if (++s == (uint32_t)pl.nring) { s = 0; ++u; }
        }
    }

    // ======================================================================================
    // conditioning warp: cond_()[t&1][l][row][b] = Wc_l[the block's gate rows] . c_t  (modules.py:141-145), one step
    // ahead; the weights come straight from L2 (they are read once per step)
    // ======================================================================================
    __device__ void cond_loop() {
        const int C = pl.C, L = pl.L, T = pp.T, B = pp.B, RA4 = 4 * pl.qA;
        constexpr int NVC = 4 * BT;                 // one row QUAD x BT utterances (the passes use row pairs)
        constexpr int M = ilog2c(NVC);
        const float* cw = pp.cwpack + (size_t)p * pl.cta_cw_floats;
        for (int t = 0; t < T; ++t) {
            const int par = t & 1, u = t >> 1;
            if (u > 0) {
                if (!wait_bar<true>(&bar_cempty_()[par], (u - 1) & 1u, 0x20000000u)) return;
            }
            float ct[BT][WN7_MAX_CI];
#pragma unroll
            for (int b = 0; b < BT; ++b)
#pragma unroll
                for (int i = 0; i < WN7_MAX_CI; ++i) {
                    const int ch = lane + 32 * i;
                    ct[b][i] = (b < B && ch < C) ? __ldg(pp.c + ((size_t)b * T + t) * C + ch) : 0.f;
                }
            float* dst = cond_() + (size_t)par * L * RA4 * BT;
            for (int l = 0; l < L; ++l) {
                for (int q = 0; q < pl.qA; ++q) {
                    float acc[NVC];
#pragma unroll
                    for (int v = 0; v < NVC; ++v) acc[v] = 0.f;
                    const float* wq = cw + ((size_t)(l * pl.qA + q) * C) * 4;
#pragma unroll
                    for (int i = 0; i < WN7_MAX_CI; ++i) {
                        const int ch = lane + 32 * i;
                        if (ch < C) {
                            const float4 w4 = __ldg(reinterpret_cast<const float4*>(wq + (size_t)ch * 4));
#pragma unroll
                            for (int b = 0; b < BT; ++b) {
                                acc[0 * BT + b] = fmaf(w4.x, ct[b][i], acc[0 * BT + b]);
                                acc[1 * BT + b] = fmaf(w4.y, ct[b][i], acc[1 * BT + b]);
                                acc[2 * BT + b] = fmaf(w4.z, ct[b][i], acc[2 * BT + b]);
                                acc[3 * BT + b] = fmaf(w4.w, ct[b][i], acc[3 * BT + b]);
                            }
                        }
                    }
                    // full-warp butterfly (32 lanes): one more level than reduce16
                    {
                        int n = NVC;
#pragma unroll
                        for (int off = 16; off >= 1; off >>= 1) {
                            if (n > 1) {
                                n >>= 1;
                                const bool hi = (lane & off) != 0;
#pragma unroll
                                for (int i = 0; i < NVC / 2; ++i) {
                                    if (i < n) {
                                        const float send = hi ? acc[i] : acc[i + n];
                                        const float keep = hi ? acc[i + n] : acc[i];
                                        acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
                                    }
                                }
                            } else {
                                acc[0] += __shfl_xor_sync(0xffffffffu, acc[0], off);
                            }
                        }
                    }
                    if ((lane & ((32 >> M) - 1)) == 0) {
                        const int v = lane >> (5 - M);   // = row_in_quad*BT + b
                        dst[((size_t)l * RA4 + q * 4 + v / BT) * BT + (v % BT)] = acc[0];
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&bar_cfull_()[par]);
        }
    }

    // ======================================================================================
    // sampler (one warp per utterance; every block computes the same thing)
    // ======================================================================================
    __device__ __forceinline__ void warp_argmax(float& best, int& bi) {
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, off);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
            if (ob > best || (ob == best && oi < bi)) {
                best = ob;
                bi = oi;
            }
        }
    }
    // noise_() for step t of utterance b into noise_()[b][*]; layout [u1(0..K-1) | u2 or z] or [e(0..O-1)]
    __device__ void fetch_noise(int t, int b) {
        float* nz = noise_() + (size_t)b * (pl.O + 2);
        const int B = pp.Btot, K = pl.Kmix, O = pl.O;
        const uint32_t ub = (uint32_t)(pp.b0 + b);
        const uint32_t tc = (STREAM ? pp.t_base : 0u) + (uint32_t)t;   // Philox counts absolute steps; replay is per launch
        const bool replay = pp.noise_kind == 0;
        const uint2 key = make_uint2((uint32_t)pp.seed, (uint32_t)(pp.seed >> 32));
        if (b >= pp.B) {   // padding row of the batch tile: harmless constants
            for (int i = lane; i < O + 2; i += 32) nz[i] = 0.5f;
            return;
        }
        if (pl.head_kind == 2) {
            for (int i = lane; i < O; i += 32) {
                float e;
                if (replay) e = pp.e ? __ldg(pp.e + ((size_t)t * B + b) * O + i) : 1.0f;
                else {
                    const uint4 r = philox4(make_uint4(tc, ub, (uint32_t)i, 2u), key);
                    e = -logf(u01(r.x));
                }
                nz[i] = e;
            }
            return;
        }
        const bool mix = (pl.head_kind == 0) || (K > 1);
        if (mix) {
            for (int i = lane; i < K; i += 32) {
                float u;
                if (replay) u = __ldg(pp.u1 + ((size_t)t * B + b) * K + i);
                else u = u01(philox4(make_uint4(tc, ub, (uint32_t)i, 0u), key).x);
                nz[i] = u;
            }
        }
        if (lane == 0) {
            float v;
            if (pl.head_kind == 0) {
                if (replay) v = __ldg(pp.u2 + (size_t)t * B + b);
                else v = u01(philox4(make_uint4(tc, ub, 0u, 1u), key).x);
            } else {
                if (replay) v = __ldg(pp.z + (size_t)t * B + b);
                else {
                    const uint4 r = philox4(make_uint4(tc, ub, 0u, 1u), key);
                    v = sqrtf(-2.f * logf(u01(r.x))) * cospif(2.f * u01(r.y));   // Box-Muller
                }
            }
            nz[K] = v;
        }
    }
    // draw sample of utterance b from hs_()[:, b]; sets the feedback for step t+1 and writes outputs
    __device__ void sample_utt(int t, int b) {
        const int O = pl.O, K = pl.Kmix, T = pp.T;
        const float* nz = noise_() + (size_t)b * (pl.O + 2);
        const bool writer = (p == 0);
        if (pl.head_kind == 2) {
            const bool softmax = (pp.flags & WN7_FLAG_SOFTMAX) != 0, quant = (pp.flags & WN7_FLAG_QUANTIZE) != 0;
            // F.softmax (wavenet.py:332): exp(h - max) / sum
            if (softmax) {
                float m = -INFINITY;
                for (int i = lane; i < O; i += 32) m = fmaxf(m, hs_()[i * BT + b]);
#pragma unroll
                for (int off = 16; off >= 1; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
                float s = 0.f;
                for (int i = lane; i < O; i += 32) {
                    const float e = expf(hs_()[i * BT + b] - m);
                    hs_()[i * BT + b] = e;
                    s += e;
                }
#pragma unroll
                for (int off = 16; off >= 1; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
                for (int i = lane; i < O; i += 32) hs_()[i * BT + b] = hs_()[i * BT + b] / s;
            }
            if (quant) {
                // OneHotCategorical(p).sample() (wavenet.py:334-335): renormalise, argmax(p / Exp(1))
                float sp = 0.f;
                for (int i = lane; i < O; i += 32) sp += hs_()[i * BT + b];
#pragma unroll
                for (int off = 16; off >= 1; off >>= 1) sp += __shfl_xor_sync(0xffffffffu, sp, off);
                float best = -INFINITY;
                int bi = 0x7fffffff;
                for (int i = lane; i < O; i += 32) {
                    const float r = (hs_()[i * BT + b] / sp) / nz[i];
                    if (r > best) {
                        best = r;
                        bi = i;
                    }
                }
                warp_argmax(best, bi);
                if (bi >= O) bi = 0;
                if (lane == 0) {
                    if (writer && b < pp.B) pp.out_index[(size_t)b * T + t] = bi;
                    s_idx_()[b] = (t + 1 < pp.T_test && b < pp.B) ? (pp.test_index ? pp.test_index[(size_t)b * pp.T_test + t + 1] : -1)
                                                               : bi;
                }
            } else {
                for (int i = lane; i < O; i += 32) {
                    const float v = hs_()[i * BT + b];
                    if (writer && b < pp.B) pp.out_dense[((size_t)b * O + i) * T + t] = v;
                    s_dense_()[b * O + i] = v;
                }
                if (lane == 0)
                    s_idx_()[b] = (t + 1 < pp.T_test && b < pp.B && pp.test_index)
                                   ? pp.test_index[(size_t)b * pp.T_test + t + 1] : -1;
            }
            // teacher forcing with dense rows overrides the feedback
            if (t + 1 < pp.T_test && pp.test_dense != nullptr && b < pp.B) {
                for (int i = lane; i < O; i += 32)
                    s_dense_()[b * O + i] = pp.test_dense[((size_t)b * pp.T_test + t + 1) * O + i];
                if (lane == 0) s_idx_()[b] = -1;
            }
            return;
        }
        // ---- scalar heads
        float mean, ls;
        const bool mix = (pl.head_kind == 0) || (K > 1);
        if (mix) {
            // Gumbel-max over the K mixture logits (mixture.py:138-140 / :247-249)
            float best = -INFINITY;
            int bi = 0x7fffffff;
            for (int i = lane; i < K; i += 32) {
                const float g = hs_()[i * BT + b] - logf(-logf(nz[i]));
                if (g > best) {
                    best = g;
                    bi = i;
                }
            }
            warp_argmax(best, bi);
            if (bi >= K) bi = 0;
            mean = hs_()[(K + bi) * BT + b];        // mixture.py:143-146 one-hot select
            ls = hs_()[(2 * K + bi) * BT + b];
        } else if (O == 2) {
            mean = hs_()[0 * BT + b];               // mixture.py:258-259
            ls = hs_()[1 * BT + b];
        } else {
            mean = hs_()[1 * BT + b];               // mixture.py:260-261 (C == 3)
            ls = hs_()[2 * BT + b];
        }
        float xv;
        if (pl.head_kind == 0) {
            const float u = nz[K];
            // mixture.py:152  x = mu + exp(s) * (log u - log(1-u)); separate roundings as in torch
            xv = __fadd_rn(mean, __fmul_rn(expf(ls), __fsub_rn(logf(u), logf(__fsub_rn(1.0f, u)))));
        } else {
            // mixture.py:265-267  Normal(mu, exp(s)).sample() == z * sigma + mu
            xv = __fadd_rn(__fmul_rn(nz[K], expf(ls)), mean);
        }
        xv = fminf(fmaxf(xv, -1.0f), 1.0f);      // mixture.py:154 / :269
        if (lane == 0) {
            if (writer && b < pp.B) pp.out_scalar[(size_t)b * T + t] = xv;
            s_in_()[b] = (t + 1 < pp.T_test && b < pp.B) ? pp.test_scalar[(size_t)b * pp.T_test + t + 1] : xv;
        }
    }

    // ======================================================================================
    // pollers
    // ======================================================================================
    // copy pairs [p0, p0+npairs) of exchange slot `src` into xin_() (utterance-major) once every tag equals `tag`;
    // lane pl_ of NPL takes 16-byte loads j = pl_, pl_+NPL, ... (4 of them in flight per retry round)
    __device__ void poll_pairs(const uint2* __restrict__ src, int p0, int npairs, uint32_t tag, float* __restrict__ xb, int pl_,
                               int NPL) {
        const int nld = (npairs + 1) >> 1;
        const int xv = pl.xin_vals;
        for (int j0 = pl_; j0 < nld; j0 += 4 * NPL) {
            uint4 q[4];
            uint32_t spins = 0;
            long long t0 = 0;
            while (true) {
                uint32_t bad = 0;
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int j = j0 + u * NPL;
                    if (j < nld) q[u] = ld_pair2(src + wn7_phys(pl, p0 + 2 * j));
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int j = j0 + u * NPL;
                    if (j < nld) bad |= (q[u].y ^ tag) | ((2 * j + 1 < npairs) ? (q[u].w ^ tag) : 0u);
                }
                if (bad == 0) break;
                if (pl.backoff_ns > 0) __nanosleep(pl.backoff_ns);
                if (((++spins) & 63u) == 0 && check_abort(tag, t0)) {
                    dead = true;
                    break;
                }
            }
            if (dead) break;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int j = j0 + u * NPL;
                if (j < nld) {
                    const int i0 = p0 + 2 * j;                       // pair index = k*BT + b
                    if constexpr (BT == 1) {
                        xb[i0] = __uint_as_float(q[u].x);
                        if (2 * j + 1 < npairs) xb[i0 + 1] = __uint_as_float(q[u].z);
                    } else {
                        xb[(i0 % BT) * xv + i0 / BT] = __uint_as_float(q[u].x);
                        if (2 * j + 1 < npairs) xb[((i0 + 1) % BT) * xv + (i0 + 1) / BT] = __uint_as_float(q[u].z);
                    }
                }
            }
        }
        dead = __any_sync(0xffffffffu, dead);
    }
    // x_0 = first 1x1 conv of the fed-back sample (wavenet.py:308): all R entries -> xb[b][xoff + k], and the rows the
    // block owns -> x0own_()
    __device__ void write_x0(float* __restrict__ xb, int pl_, int NPL, bool own_too) {
        const int R = pl.R, O = pl.O, xv = pl.xin_vals;
        const int n = R * BT, nown = pl.mx * BT;
        for (int i = pl_; i < n + (own_too ? nown : 0); i += NPL) {
            const bool own = i >= n;
            const int k = (own ? i - n : i) % (own ? pl.mx : R), b = (own ? i - n : i) / (own ? pl.mx : R);
            const int g = own ? (k < nx ? x0r + k : -1) : k;
            float v = 0.f;
            if (g >= 0) {
                if (pl.input_kind == 0) {
                    v = fmaf(x0w_()[g], s_in_()[b], x0w_()[R + g]);
                } else {
                    const int idx = min(s_idx_()[b], O - 1);          // class ids are range-checked on the host where it can
                    if (idx >= 0) {
                        v = __ldg(pp.first_w + (size_t)idx * R + g) + x0w_()[R + g];   // one-hot input: a column gather
                    } else {
                        float a = 0.f;
                        for (int o = 0; o < O; ++o) a = fmaf(__ldg(pp.first_w + (size_t)o * R + g), s_dense_()[b * O + o], a);
                        v = a + x0w_()[R + g];
                    }
                }
            }
            if (own) x0own_()[k * BT + b] = v;
            else xb[b * xv + pl.xoff + k] = v;
        }
    }
    // all head outputs of step t -> hs_(), then the sampler (sets the feedback of step t+1)
    __device__ void read_head_and_sample(int t, int pl_, int NPL) {
        const int npairs = pl.O * BT;                      // pair index o*BT + b == hs_() index
        const uint32_t tag = (uint32_t)t * (uint32_t)pl.NS + (uint32_t)(pl.L + 2) + 1u;
        const uint2* src = pp.xbuf + wn7_ex_off(pl, pl.L + 2);
        const int nld = (npairs + 1) >> 1;
        for (int j = pl_; j < nld; j += NPL) {
            const bool two = 2 * j + 1 < npairs;
            uint4 q;
            uint32_t spins = 0;
            long long t0 = 0;
            while (true) {
                q = ld_pair2(src + wn7_phys(pl, 2 * j));
                if (q.y == tag && (!two || q.w == tag)) break;
                if (pl.backoff_ns > 0) __nanosleep(pl.backoff_ns);
                if (((++spins) & 63u) == 0 && check_abort(tag, t0)) {
                    dead = true;
                    break;
                }
            }
            if (dead) break;
            hs_()[2 * j] = __uint_as_float(q.x);
            if (two) hs_()[2 * j + 1] = __uint_as_float(q.z);
        }
        dead = __any_sync(0xffffffffu, dead);
        poller_sync();
        if (dead) return;
        if (p == 0 && pp.params_out != nullptr) {
            const int O = pl.O, T = pp.T;
            for (int i = pl_; i < O * BT; i += NPL) {
                const int o = i / BT, b = i % BT;
                if (b < pp.B) pp.params_out[((size_t)b * O + o) * T + t] = hs_()[i];
            }
            if (pl.head_kind == 2) {                         // the softmax sampler overwrites hs_() in place
                poller_sync();
                if (dead) return;
            }
        }
        for (int b = warp; b < BT; b += n_poll_warps()) {      // polling warps are warps 0..n-1 in both modes
            sample_utt(t, b);
            if (t + 1 < pp.T) fetch_noise(t + 1, b);
        }
        poller_sync();
    }

    // poller duties of stage s of step t (global stage n), in two phases: the rare heavy work first (sampler of the
    // previous step, x_0), then only the coherent loads -- so that a compute warp that polls can hold its preloaded
    // weights in registers across the second phase
    __device__ __forceinline__ void poll_stage_head(int t, int s, float* __restrict__ xb, int pl_, int NPL) {
        if (s == 0) {
            if (t > 0) read_head_and_sample(t - 1, pl_, NPL);
            if (dead) return;
            write_x0(xb, pl_, NPL, true);
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_x0_());     // x_0 at the rows this block owns is in place (read in stage 1)
        } else if (s == 1) {
            write_x0(xb, pl_, NPL, false);              // x_0 is evaluated locally
        }
    }
    __device__ __forceinline__ void poll_stage_loads(int s, uint32_t n, float* __restrict__ xb, int pl_, int NPL) {
        if (s == 0) return;
        const uint2* src = pp.xbuf + wn7_ex_off(pl, s - 1);
        if (s <= pl.L) {
            poll_pairs(src, 0, pl.G2 * BT, n, xb, pl_, NPL);
            if (dead || s == 1) return;
            poll_pairs(src, pl.xoff * BT, pl.R * BT, n, xb, pl_, NPL);
        } else {
            poll_pairs(src, 0, pl.S * BT, n, xb, pl_, NPL);
        }
    }

    __device__ void poll_loop() {
        const int NPL = 32 * pl.npw;
        const int pl_ = warp * 32 + lane, NS = pl.NS, T = pp.T;
        const int xin_floats = pl.xin_vals * BT;
        uint32_t n = 0;
        long long t_prev = clock64();
        for (int t = 0; t < T && !dead; ++t) {
            for (int s = 0; s < NS; ++s, ++n) {
                const int par = n & 1;
                if (n >= 2) {
                    if (!wait_bar(&bar_free_()[par], ((n >> 1) - 1) & 1u, 0x10000000u | (uint32_t)s)) break;
                }
                float* xb = xin_() + (size_t)par * xin_floats;
                // gate: the next vector cannot be complete earlier than the local chain + one L2 hop after this one, and
                // polling earlier only loads the L2 slices the publishers are writing to
                if (pl.gate_cycles > 0) { while (clock64() - t_prev < pl.gate_cycles) {} }
                poll_stage_head(t, s, xb, pl_, NPL);
                if (!dead) poll_stage_loads(s, n, xb, pl_, NPL);
                if (dead) break;
                __syncwarp();
                if (lane == 0) mbar_arrive(&bar_in_()[par]);     // one arrival per polling warp
                t_prev = clock64();
            }
        }
        if (!dead) read_head_and_sample(T - 1, pl_, NPL);
    }

    // ======================================================================================
    // compute warps
    // ======================================================================================
    int rs_slot = 0;
    uint32_t rs_par = 0;
    __device__ __forceinline__ const float* acquire_blob(int t, int i) {
        if (i < pl.nres) {
            if (t == 0) wait_bar(&bar_full_()[i], 0, 0x80000000u | (uint32_t)i);
            return slots_() + (size_t)i * pl.slot_floats;
        }
        const int slot = pl.nres + rs_slot;
        wait_bar(&bar_full_()[slot], rs_par, 0x80000000u | (uint32_t)i);
        return slots_() + (size_t)slot * pl.slot_floats;
    }
    __device__ __forceinline__ void release_blob(int i) {
        if (i >= pl.nres) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&bar_empty_()[rs_slot]);
            if (++rs_slot == pl.nring) {
                rs_slot = 0;
                rs_par ^= 1u;
            }
        }
    }
    // modules.py:154  tanh(a) * sigmoid(g) with a single division:
    //   (1 - e^{-2a}) / ((1 + e^{-2a}) (1 + e^{-g}));  |a| is clamped where tanh has saturated in fp32.
    __device__ __forceinline__ static float gate(float a, float g) {
        const float ac = fminf(fmaxf(a, -15.0f), 15.0f);
        const float ea = expf(-2.0f * ac), eg = expf(-g);
        return (1.0f - ea) / ((1.0f + ea) * (1.0f + eg));
    }

    // One pass: two complete rows.  Lane l handles k = x_off + 4*(l + 32 j) .. +3 of both rows for every utterance,
    // the butterfly leaves value (row r, utterance b) in lane (r*BT + b) * 32/NV, and those lanes finalise.
    __device__ __forceinline__ void fma_step(const float4& wa, const float4& wb, const float* __restrict__ x, int xv,
                                             float (&acc)[NV], float (&acc2)[NV]) {
#pragma unroll
        for (int b = 0; b < BT; ++b) {
            const float4 x4 = *reinterpret_cast<const float4*>(x + (size_t)b * xv);
            if constexpr (BT == 1) {
                // one utterance: two independent chains per row keep the FMA pipe busy
                acc[0] = fmaf(wa.x, x4.x, acc[0]);
                acc2[0] = fmaf(wa.y, x4.y, acc2[0]);
                acc[0] = fmaf(wa.z, x4.z, acc[0]);
                acc2[0] = fmaf(wa.w, x4.w, acc2[0]);
                acc[1] = fmaf(wb.x, x4.x, acc[1]);
                acc2[1] = fmaf(wb.y, x4.y, acc2[1]);
                acc[1] = fmaf(wb.z, x4.z, acc[1]);
                acc2[1] = fmaf(wb.w, x4.w, acc2[1]);
            } else {
                acc[b] = fmaf(wa.x, x4.x, acc[b]);
                acc[b] = fmaf(wa.y, x4.y, acc[b]);
                acc[b] = fmaf(wa.z, x4.z, acc[b]);
                acc[b] = fmaf(wa.w, x4.w, acc[b]);
                acc[BT + b] = fmaf(wb.x, x4.x, acc[BT + b]);
                acc[BT + b] = fmaf(wb.y, x4.y, acc[BT + b]);
                acc[BT + b] = fmaf(wb.z, x4.z, acc[BT + b]);
                acc[BT + b] = fmaf(wb.w, x4.w, acc[BT + b]);
            }
        }
    }
    __device__ __forceinline__ void run_pass(const Wn7Pass& ps, const float* __restrict__ blob, const float* __restrict__ xb,
                                             int s, uint32_t tag) {
        float acc[NV], acc2[NV];
#pragma unroll
        for (int v = 0; v < NV; ++v) { acc[v] = 0.f; acc2[v] = 0.f; }
        run_pass_tail(ps, blob, xb, s, tag, 0, acc, acc2);
    }
    // k-steps [j0, nit) with the weights read from shared memory, then the butterfly and the finalisation
    __device__ __forceinline__ void run_pass_tail(const Wn7Pass& ps, const float* __restrict__ blob, const float* __restrict__ xb,
                                                  int s, uint32_t tag, int j0, float (&acc)[NV], float (&acc2)[NV]) {
        const float4* __restrict__ w = reinterpret_cast<const float4*>(blob + ps.w_off) + lane;
        const float* __restrict__ x = xb + ps.x_off + 4 * lane;
        const int xv = pl.xin_vals;
        const int nit = ps.nit;
        for (; j0 < nit; j0 += 4) {
            float4 wa[4], wb[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (j0 + u < nit) {
                    wa[u] = w[(j0 + u) * 64];
                    wb[u] = w[(j0 + u) * 64 + 32];
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (j0 + u < nit) fma_step(wa[u], wb[u], x + (j0 + u) * 128, xv, acc, acc2);
        }
        if constexpr (BT == 1) {
            acc[0] += acc2[0];
            acc[1] += acc2[1];
        }
        reduce32<NV>(acc, lane);
        constexpr int LPV = 32 / NV;                      // lanes per value
        const float mine = acc[0];
        // the second row's value of the same utterance sits 16 lanes up
        const float other = __shfl_down_sync(0xffffffffu, mine, 16);
        if ((lane & (LPV - 1)) != 0) return;
        const int v = lane / LPV, r = v / BT, b = v % BT;
        const int job = ps.job, idx = ps.idx, RA4 = 4 * pl.qA;
        const float RSQRT2 = 0.70710678118654752440f;         // math.sqrt(0.5), modules.py:162
        const long long ex = wn7_ex_off(pl, s);
        switch (job) {
            case WN7_J_A0:
            case WN7_J_A: {
                if (r != 0 || idx >= ny) break;
                const float a = mine + pre_()[((size_t)s * RA4 + 2 * idx) * BT + b];
                const float g = other + pre_()[((size_t)s * RA4 + 2 * idx + 1) * BT + b];
                publish(ex, (long long)(y0 + idx) * BT + b, gate(a, g), tag);
            } break;
            case WN7_J_B: {
                // modules.py:160-162  x_s = (conv1x1_out(y_{s-1}) + x_{s-1}) * sqrt(0.5)
                const int j = idx + r;
                if (j >= nx) break;
                const float o = mine + bias_()[pl.bo_xb + s * pl.mx + j];
                const float xp = (s == 1) ? x0own_()[j * BT + b] : xown_()[j * BT + b];
                const float xn = (o + xp) * RSQRT2;
                publish(ex, (long long)(pl.xoff + x0r + j) * BT + b, xn, tag);
                xown_()[j * BT + b] = xn;
            } break;
            case WN7_J_D: {
                // older-tap products of layer s-1 -> history ring_() (consumed at steps t+d, t+2d, conv.py:32-44)
                const int tap = idx / pl.my, i = idx % pl.my;
                const int e = ((s - 1) * (pl.kw - 1) + tap) * 3;
                ring_()[((size_t)ringtab_()[e] + ringtab_()[e + 2]) * RA4 * BT + (2 * i + r) * BT + b] = mine;
            } break;
            case WN7_J_S: {
                // skip rows of layer s-1, accumulated in layer order (wavenet.py:312)
                const int j = idx + r;
                if (j >= ns) break;
                const float h = mine + bias_()[pl.bo_sb + (s - 1) * pl.ms + j];
                skipacc_()[j * BT + b] = (s == 1) ? h : skipacc_()[j * BT + b] + h;
            } break;
            case WN7_J_SL: {
                // (s_0 + ... + s_{L-2}) + s_{L-1}, * sqrt(1/L), first ReLU of the head (wavenet.py:312-315)
                const int j = idx + r;
                if (j >= ns) break;
                float tot = mine + bias_()[pl.bo_sb + (pl.L - 1) * pl.ms + j];
                if (pl.L >= 2) tot = skipacc_()[j * BT + b] + tot;
                publish(ex, (long long)(s0 + j) * BT + b, fmaxf(tot * pl.skip_scale, 0.f), tag);
            } break;
            case WN7_J_HA: {
                const int j = idx + r;
                if (j >= na) break;
                publish(ex, (long long)(a0 + j) * BT + b, fmaxf(mine + bias_()[pl.bo_ha + j], 0.f), tag);
            } break;
            default: {   // WN7_J_HB
                const int j = idx + r;
                if (j >= nb) break;
                publish(ex, (long long)(b0 + j) * BT + b, mine + bias_()[pl.bo_hb + j], tag);
            } break;
        }
    }

    __device__ void comp_loop() {
        const int cw = warp - wn7_warp_comp(pl), NS = pl.NS, L = pl.L, T = pp.T;
        const int xin_floats = pl.xin_vals * BT;
        const bool prof = (pp.prof != nullptr) && cw == 0 && lane == 0;
        long long pc[4] = {0, 0, 0, 0}, tc = 0;
#define WN7_TICK(i) if (prof) { const long long now_ = clock64(); pc[i] += now_ - tc; tc = now_; }
        // skip-row passes_() per layer stage (all warps): the tail stage waits for all of them
        int nskip = 0;
        for (int w = 0; w < WN7_NCW; ++w)
            for (int i = 0; i < pl.pass_count[WN7_K_LAYER][w]; ++i)
                if (passes_()[pl.pass_begin[WN7_K_LAYER][w] + i].job == WN7_J_S) ++nskip;
        uint32_t n = 0, nd = 0;
        long long t_prev = clock64();
        const float* blob = nullptr;
        for (int t = 0; t < T && !dead; ++t) {
            if (prof) tc = clock64();
            for (int s = 0; s < NS; ++s, ++n) {
                const int par = n & 1, kind = wn7_kind(pl, s);
                if (s <= L) blob = acquire_blob(t, s);
                if (s == 0) wait_bar(bar_pre_(), (uint32_t)t & 1u, 0x02000000u);          // pre_()-sums of this step are built
                if (s == 1) wait_bar(bar_x0_(), (uint32_t)t & 1u, 0x02000001u);           // x_0 at the owned rows is in place
                const int begin = pl.pass_begin[kind][cw], cnt = pl.pass_count[kind][cw], crit = pl.pass_crit[kind][cw];
                float* xb = xin_() + (size_t)par * xin_floats;
                const bool i_poll = SELF && cw < WN7_NSP;
                if (i_poll) {
                    // this warp is one of the pollers: the buffer must be free, then the rare heavy part of the duty
                    if (n >= 2) {
                        if (!wait_bar(&bar_free_()[par], ((n >> 1) - 1) & 1u, 0x10000000u | (uint32_t)s)) break;
                    }
                    poll_stage_head(t, s, xb, cw * 32 + lane, 32 * WN7_NSP);
                    if (dead) break;
                }
                WN7_TICK(0);
                if (i_poll) {
                    if (pl.gate_cycles > 0) { while (clock64() - t_prev < pl.gate_cycles) {} }
                    poll_stage_loads(s, n, xb, cw * 32 + lane, 32 * WN7_NSP);     // its share of the vector ...
                    poller_sync();                                                // ... then the group barrier
                    if (dead) break;
                    if (lane == 0) mbar_arrive(&bar_in_()[par]);     // releases the compute warps that do not poll
                    t_prev = clock64();
                } else {
                    if (!wait_bar(&bar_in_()[par], (n >> 1) & 1u, 0x08000000u | (uint32_t)s)) break;
                }
                WN7_TICK(1);
                bool had_skip = false;
                if (kind == WN7_K_TAIL && L >= 2) {
                    // skip rows of layers 0..L-2 are accumulated by the deferred passes_() of stages 1..L-1
                    bool need = false;
                    for (int i = 0; i < cnt; ++i) need |= passes_()[begin + i].job == WN7_J_SL;
                    if (need) wait_count(s_skipcnt_(), (t * (L - 1) + (L - 1)) * nskip, 0x02000002u);
                    if (dead) break;
                }
                const bool gate_def = pp.defer_gate && pl.has_deferred[kind];
                const int cpar = nd & 1;                  // bar_crit is used only in the stages that have deferred passes
                if (gate_def && crit == 0) { __syncwarp(); if (lane == 0) mbar_arrive(&bar_crit_()[cpar]); }
                for (int i = 0; i < cnt; ++i) {
                    const Wn7Pass& ps = passes_()[begin + i];
                    if (gate_def && i == crit) {
                        // the deferred products are not needed before the next step: let the critical rows of every warp of
                        // this SM leave first (they share the issue slots)
                        if (!wait_bar<true>(&bar_crit_()[cpar], (nd >> 1) & 1u, 0x00400000u | (uint32_t)s)) break;
                    }
                    run_pass(ps, blob, xb, s, n + 1u);
                    had_skip |= ps.job == WN7_J_S;
                    if (i + 1 == crit) {
                        WN7_TICK(2);
                        if (gate_def) { __syncwarp(); if (lane == 0) mbar_arrive(&bar_crit_()[cpar]); }
                    }
                }
                if (dead) break;
                if (gate_def) ++nd;
                __syncwarp();
                if (had_skip) {
                    __threadfence_block();
                    if (lane == 0) {
                        int c = 0;
                        for (int i = 0; i < cnt; ++i) c += passes_()[begin + i].job == WN7_J_S;
                        atomicAdd((int*)s_skipcnt_(), c);
                    }
                }
                if (lane == 0) mbar_arrive(&bar_free_()[par]);
                if (s < L || s == NS - 1) release_blob(wn7_blob_of_stage(pl, s));
                if (s == L) {
                    // every deferred product of this step is in its ring_(): HK may advance the rings and build the next table
                    __threadfence_block();
                    if (lane == 0) mbar_arrive(bar_dstep_());
                }
                WN7_TICK(3);
            }
        }
        if (SELF && cw < WN7_NSP && !dead) read_head_and_sample(T - 1, cw * 32 + lane, 32 * WN7_NSP);
        if (prof) {
            for (int i = 0; i < 4; ++i) pp.prof[(size_t)p * 16 + 8 + i] = pc[i];
        }
#undef WN7_TICK
    }

    // ======================================================================================
    // housekeeping warp: ring_() positions and the pre_()-sum table, once per step
    // ======================================================================================
    // Everything of z_l(t) that does not depend on step t's exchanges: (folded) bias_() + global conditioning +
    // local-conditioning projection + the queued products of the older taps.
    __device__ void build_pre(int t) {
        const int L = pl.L, RA4 = 4 * pl.qA, kw = pl.kw, n = L * RA4 * BT;
        if (pl.C > 0) wait_bar<true>(&bar_cfull_()[t & 1], (uint32_t)(t >> 1) & 1u, 0x01000000u);
        if (dead) return;
        const float* cd = cond_() + (size_t)(t & 1) * L * RA4 * BT;
        for (int i = lane; i < n; i += 32) {
            const int l = i / (RA4 * BT), rem = i % (RA4 * BT);
            float v = sb_()[i];
            if (pl.C > 0) v += cd[i];
            for (int k = 0; k < kw - 1; ++k) {
                const int e = (l * (kw - 1) + k) * 3;
                v += ring_()[((size_t)ringtab_()[e] + ringtab_()[e + 2]) * RA4 * BT + rem];
            }
            pre_()[i] = v;
        }
        __syncwarp();
        if (lane == 0) {
            if (pl.C > 0) mbar_arrive(&bar_cempty_()[t & 1]);
            mbar_arrive(bar_pre_());
        }
    }
    __device__ void hk_loop() {
        const int L = pl.L, T = pp.T, kw = pl.kw;
        build_pre(0);
        for (int t = 0; t < T && !dead; ++t) {
            if (!wait_bar<true>(bar_dstep_(), (uint32_t)t & 1u, 0x00800000u)) break;
            // advance the ring_() positions to (t+1) mod delay, then the pre_()-sums of step t+1
            for (int i = lane; i < L * (kw - 1); i += 32) {
                const int pos = ringtab_()[i * 3 + 2] + 1;
                ringtab_()[i * 3 + 2] = (pos == ringtab_()[i * 3 + 1]) ? 0 : pos;
            }
            __threadfence_block();
            __syncwarp();
            if (t + 1 < T) build_pre(t + 1);
        }
    }
};

// ------------------------------------------------------------------------------------------
// kernel entry
// ------------------------------------------------------------------------------------------
// Stream epilogue (every thread, after the block barrier that follows the role loops): the rings in shared memory and
// block 0's feedback of the step after the launch.  Nothing else carries over a step: the stage buffers xin / xown /
// x0own / hs / noise are filled before they are read within the step, skipacc restarts at layer 1, the pre-sum table
// and the conditioning double buffer are rebuilt per step by HK and COND, and the exchange tags count local steps.
template <int BT>
__device__ __noinline__ void wn7_store_state(const Wn7Plan& pl, const Wn7Ptrs& pp, unsigned char* sm) {
    const int tid = (int)threadIdx.x, NT = (int)blockDim.x, p = (int)blockIdx.x;
    const long long ring_n = wn7_state_ring_floats(pl);
    if (pl.ring_in_smem) {
        const volatile float* ring = reinterpret_cast<const volatile float*>(sm + pl.sm_ring);
        float* dst = pp.state + (size_t)p * ring_n;
        for (long long i = tid; i < ring_n; i += NT) dst[i] = ring[i];
    }
    if (p == 0) {
        const float* s_in = reinterpret_cast<const float*>(sm + pl.sm_in);      // layout of Engine's s_in_ / s_idx_ / s_dense_
        const int* s_idx = reinterpret_cast<const int*>(s_in + BT);
        const float* s_dense = reinterpret_cast<const float*>(s_idx + BT);
        float* fb = pp.state + (size_t)pl.P * ring_n;
        for (int b = tid; b < BT; b += NT) {
            fb[b] = s_in[b];
            fb[BT + b] = __int_as_float(s_idx[b]);
        }
        if (pl.input_kind != 0)
            for (int i = tid; i < BT * pl.O; i += NT) fb[2 * BT + i] = s_dense[i];
    }
}

template <int BT, bool SELF>
__global__ void __launch_bounds__(32 * ((SELF ? 0 : WN7_MAX_NPW) + WN7_NCW + 3), 1)
wn7_kernel(const __grid_constant__ Wn7Plan pl, const __grid_constant__ Wn7Ptrs pp) {
    constexpr bool STREAM = false;
#include "wn7_kernel_body.cuh"
}

// wn_stream_generate's kernel: handles whose compute warps poll (SELF), BT = 1, 2, 4, 8
template <int BT>
__global__ void __launch_bounds__(32 * (WN7_NCW + 3), 1)
wn7_stream_kernel(const __grid_constant__ Wn7Plan pl, const __grid_constant__ Wn7Ptrs pp) {
    constexpr bool SELF = true, STREAM = true;
#include "wn7_kernel_body.cuh"
}

}  // namespace wn7
