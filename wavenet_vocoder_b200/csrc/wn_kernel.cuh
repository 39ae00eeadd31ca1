// wn_kernel.cuh — the persistent sm_90a synthesis kernel.
//
// One launch == one WaveNet.incremental_forward() call (reference wavenet.py:215-343): the whole
// T-step loop, including the sampler, runs on the device.  P thread blocks (one per SM,
// cooperative launch) each own a fixed slice of the output rows of every matrix (wn_plan.h).
//
// Per generated sample the blocks run L+3 "stages", each ending in ONE broadcast:
//   stage 0      : x_0 (first 1x1 conv of the fed-back sample, computed by every block) ->
//                  its rows of the current tap of layer 0 -> tanh*sigmoid -> publish y_0
//   stage s<L    : wait for (y_{s-1}, x_{s-1}); then for layer s (modules.py:112-163)
//                    z_s = M_{s-1} y_{s-1} + V_s x_{s-1} + bias + conditioning + queued older taps
//                  where V_s = sqrt(.5) W_s[:,:,kw-1] and M_{s-1} = V_s Wo_{s-1} were folded on the host
//                  (conv1x1_out of the previous layer rides inside the current tap, so the reference's
//                  two dependent GEMVs per layer need one broadcast instead of two), and
//                    x_s = (Wo_{s-1} y_{s-1} + bo + x_{s-1}) sqrt(.5)        (its rows; the residual stream)
//                  -> publish (y_s, x_s) together.
//                  Deferred, off the critical path while the broadcast travels: the OLDER taps'
//                  products W_{s-1}[:,:,k<kw-1] . x_{s-1}(t), queued for steps t+d, t+2d (this replaces
//                  the reference's input shift register, conv.py:32-44, by a queue of OUTPUT partials
//                  private to the block), and its rows of conv1x1_skip_{s-1}, accumulated in layer
//                  order like wavenet.py:312.
//   stage L      : skip rows of the last layer -> total skip * sqrt(1/L) -> ReLU -> publish
//   head 1, 2    : wavenet.py:315-319, one broadcast each
// then the sampler (mixture.py), which every block evaluates redundantly from the same noise so
// no further broadcast is needed.
//
// Inside a block the 8 compute warps are split in two groups that run concurrently:
//   critical group (warps 0-3): wait for the broadcast -> current-tap rows -> gate -> publish.
//       Nothing else sits between two broadcasts.
//   deferred group (warps 4-7): takes (y_{s-1}, x_{s-1}) from a shared-memory stash left by the critical
//       group and does everything that is only needed later (queued older-tap products, skip rows).
// plus one warp that streams weights (TMA) and one that projects the local conditioning.
//
// Exchange protocol: every value travels as an 8-byte (value, tag) pair (tag = step*NE+id+1), written with
// one 8-byte store and polled with 8/16-byte loads, so data and "ready" flag are one atomic word: no
// fences, no separate barrier, one L2 write + one L2 read per hop.  What the code is shaped by:
//   * an L1-bypassing coherent load (SASS LDG.E.64/128.STRONG.GPU) is a round trip to L2 for the issuing
//     warp, and several of them from one warp do not overlap -> the poll time is (loads per thread) x one
//     L2 round trip: the vector is read by the 128 threads of the critical group, and with one utterance per
//     launch each thread owns PAIRS of adjacent elements fetched by one 16-byte load (3 loads per thread for
//     config 2) rather than one warp per quad (24 loads per lane), TMA bulk-copy or cp.async polling;
//   * replicas of a value written by different threads cost more in scattered stores than they save: one
//     copy (`ncopy` = 1; the replica mechanism is kept for experiments);
//   * the pairs are spread over L2 slices (wn_pair_index).
//
// Weights: fp32, packed per block by the host ("blobs").  A dedicated warp streams the blobs
// into shared memory with TMA bulk copies (cp.async.bulk + mbarrier complete_tx) through a ring
// of slots, running ahead of the compute warps; blobs that fit stay resident for the whole call.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include "wn_plan.h"

struct WnPtrs {
    const float* wpack;        // [P][cta_w_floats]
    const float* cwpack;       // [P][cta_cw_floats]
    const float* gbias;        // [B][L][G] = Wg_l . g_b   (NULL without global conditioning)
    const float* first_w;      // scalar input: [R];  one-hot input: transposed [O][R]
    const float* first_b;      // [R]
    uint2* xbuf;               // exchange replicas
    float* ring_g;             // [P][ring floats] when the history rings do not fit in smem
    const int* ringtab;        // [L*(kw-1)*2] : (offset in positions, delay D)
    int* err;                  // [4] device fault word, last tag, block, info
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
    long long* prof;           // [P][WN_PROF_SLOTS] stage profile (-DWN_STAGE_PROF builds only, scripts/stage_prof.py)
    int warp_reverse;          // 1: logical warp = 9 - physical warp (the issue arbiter favours high warp ids)
    int gate_cycles;           // the critical group does not poll an exchange earlier than this after its own publish
    // ---- streaming (wn_stream_generate): a launch continues an utterance at absolute step t_base
    unsigned t_base;           // absolute step of local step 0 (Philox counters, ring positions); 0 for a whole utterance
    float* state;              // NULL, or [P][ring floats] rings then the feedback [BT] s_in, [BT] s_idx, [BT][O] s_dense
    int state_load;            // 1: rings and step-0 feedback come from `state`; 0: zero rings, feedback from initial*
};

// floats of the stream state that follow the rings: the feedback of the next step
__host__ __device__ inline long long wn_state_feedback_floats(const WnPlan& pl) {
    return 2LL * pl.BT + (pl.input_kind != 0 ? (long long)pl.BT * pl.O : 0);
}
__host__ __device__ inline long long wn_state_ring_floats(const WnPlan& pl) {
    return (long long)pl.ring_pos_total * pl.RA4 * pl.BT;       // per block
}

#define WN_FLAG_SOFTMAX_ 1u
#define WN_FLAG_QUANTIZE_ 2u

namespace wn {

// ------------------------------------------------------------------------------------------
// PTX helpers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
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
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
// the same copy with an L2 cache policy (createpolicy) attached to its reads
__device__ __forceinline__ void bulk_g2s_hint(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t pol) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
            smem_u32(dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
        : "memory");
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
// ask L2 to fetch [src, src+bytes) from global memory (bytes a multiple of 16); no shared memory, no completion
__device__ __forceinline__ void prefetch_l2(const void* src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint2 ld_pair(const uint2* p) {
    uint2 v;
    asm volatile("ld.relaxed.gpu.global.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint4 ld_pair2(const uint2* p) {
    uint4 v;
    asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p)
                 : "memory");
    return v;
}
__device__ __forceinline__ void st_pair(uint2* p, float v, uint32_t tag) {
    asm volatile("st.relaxed.gpu.global.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(__float_as_uint(v)), "r"(tag)
                 : "memory");
}
__device__ __forceinline__ int ld_flag(const int* p) {
    int v;
    asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// named barrier over the WN_NT compute threads only (aux warps never join), OR-reducing a flag
__device__ __forceinline__ bool bar_or(bool pred) {
    uint32_t r;
    asm volatile(
        "{\n\t.reg .pred p, q;\n\t"
        "setp.ne.u32 p, %1, 0;\n\t"
        "bar.red.or.pred q, 1, %2, p;\n\t"
        "selp.u32 %0, 1, 0, q;\n\t}"
        : "=r"(r)
        : "r"((uint32_t)pred), "n"(WN_NT)
        : "memory");
    return r != 0;
}

// named barrier `ID` over `N` threads, OR-reducing a flag
template <int ID, int N>
__device__ __forceinline__ bool bar_or_n(bool pred) {
    uint32_t r;
    asm volatile(
        "{\n\t.reg .pred p, q;\n\t"
        "setp.ne.u32 p, %1, 0;\n\t"
        "bar.red.or.pred q, %2, %3, p;\n\t"
        "selp.u32 %0, 1, 0, q;\n\t}"
        : "=r"(r)
        : "r"((uint32_t)pred), "n"(ID), "n"(N)
        : "memory");
    return r != 0;
}

// The barrier at which the two compute groups of a block meet (id 3, all WN_NT compute threads).  The groups arrive
// from two different loops, which PTX allows (a barrier is its id, not its instruction) but compute-sanitizer's
// synccheck reports as divergence: -DWN_SINGLE_BARRIER_SITE compiles ONE out-of-line instance for that tool.
// The shipped build inlines it: the out-of-line call is on the critical path of every stage.
#ifdef WN_SINGLE_BARRIER_SITE
__device__ __noinline__ bool bar_groups(bool pred) { return bar_or_n<3, WN_NT>(pred); }
#else
__device__ __forceinline__ bool bar_groups(bool pred) { return bar_or_n<3, WN_NT>(pred); }
#endif

// NA independent value sets reduced in lock step (the shuffles of different sets overlap)
template <int NA, int NV>
__device__ __forceinline__ void reduce_scatter_multi(float (&v)[NA][NV], int lane) {
    int n = NV;
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        if (n > 1) {
            n >>= 1;
            const bool hi = (lane & off) != 0;
#pragma unroll
            for (int a = 0; a < NA; ++a) {
#pragma unroll
                for (int i = 0; i < NV / 2; ++i) {
                    if (i < n) {
                        const float send = hi ? v[a][i] : v[a][i + n];
                        const float keep = hi ? v[a][i + n] : v[a][i];
                        v[a][i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
                    }
                }
            }
        } else {
#pragma unroll
            for (int a = 0; a < NA; ++a) v[a][0] += __shfl_xor_sync(0xffffffffu, v[a][0], off);
        }
    }
}

template <int NV>
__device__ __forceinline__ void reduce_scatter(float (&v)[NV], int lane) {
    // butterfly over the 32 lanes; while more than one value is left each step also halves the
    // value set, so NV values cost NV-1+... shuffles instead of 5*NV.  Afterwards v[0] of lane
    // l is the warp-wide sum of value (l >> (5 - log2 NV)).
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

__host__ __device__ constexpr int ilog2c(int v) { return v <= 1 ? 0 : 1 + ilog2c(v >> 1); }

// Philox4x32-10 (counter-based; the same (seed, step, utterance, slot) gives the same draw in
// every block, which is what lets all blocks sample redundantly)
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


// slow path of every spin loop: has another block faulted / have we waited too long?  `t0` is the clock of the
// wait's first check (0 before it); returns the value to pass next time, or -1 to abort.  Passed by value: a
// reference would put it on the stack, and every wait of the stage loop would begin with a local-memory store.
__device__ __noinline__ long long wn_check_abort(volatile int* s_abort, int* err, long long timeout, uint32_t what,
                                                 int p, long long t0) {
    if (*s_abort) return -1;
    if (ld_flag(err) != 0) {
        *s_abort = 1;
        return -1;
    }
    const long long now = clock64();
    if (t0 == 0) return now;
    if (now - t0 > timeout) {
        if (atomicCAS(err, 0, 1) == 0) {
            err[1] = (int)what;
            err[2] = p;
            err[3] = (int)threadIdx.x;
        }
        *s_abort = 1;
        return -1;
    }
    return t0;
}

// Stage profile (scripts/stage_prof.py): cycle counters per block, compiled only with -DWN_STAGE_PROF so that the
// shipped kernels keep no counter state across the step loop.  Lane 0 of each warp adds its own phases:
//   critical warp w   [w*13, w*13+13)  stages 1..L-1: acquire+pre, poll, stash, weight load+FMA issue, wait for the
//                                      FMA results (and so for the weight reads they consume), shuffle reduce,
//                                      quad_store, barrier (arrival -> release), finalize, publish, wait for the
//                                      deferred group; then stages 0, L and the head; then the step tail
//   critical skew     52: sum over stages 1..L-1 of (last - first arrival at the group barrier), 53: stages counted,
//                     54+w: stages at which warp w arrived last
//   deferred warp w   [58+w*6, 58+w*6+6): wait for the stash, unstash, weight load+FMA+reduce+store, barrier,
//                                      finalize (ring / skip writes), the rest of the step
//   82, 83: TMA warp cycles spent waiting for a free ring slot, and in total; 84, 85: the same for the
//   conditioning warp
#define WN_PROF_SLOTS 96
enum { WN_PC_ACQ, WN_PC_POLL, WN_PC_STASH, WN_PC_FMA, WN_PC_READY, WN_PC_REDUCE, WN_PC_STORE, WN_PC_BAR, WN_PC_FIN,
       WN_PC_PUB, WN_PC_DDONE, WN_PC_HEAD, WN_PC_TAIL, WN_PC_CRIT };
enum { WN_PD_WAIT, WN_PD_UNSTASH, WN_PD_GEMV, WN_PD_BAR, WN_PD_FIN, WN_PD_REST, WN_PC_DEF };
enum { WN_PS_SKEW = 4 * WN_PC_CRIT, WN_PS_DEF = WN_PS_SKEW + 6, WN_PS_TMA = WN_PS_DEF + 4 * WN_PC_DEF,
       WN_PS_COND = WN_PS_TMA + 2 };
static_assert(WN_PS_COND + 2 <= WN_PROF_SLOTS, "stage profile slots");
#ifdef WN_STAGE_PROF
#define WN_PROF_DECL(N) const bool prof_ = (pp.prof != nullptr) && lane == 0; long long pc_[N] = {}, tc_ = 0;
#define WN_PROF_START() if (prof_) tc_ = clock64();
#define WN_TICK(i) if (prof_) { const long long now_ = clock64(); pc_[i] += now_ - tc_; tc_ = now_; }
// the same after a shared-memory store of `v`: the store, and so the clock read behind it, waits until v is computed
#define WN_TICK_AFTER(i, sink, v) if (prof_) { *reinterpret_cast<volatile float*>(sink) = (v); } WN_TICK(i)
#define WN_PROF_STORE(base, N) if (prof_) { for (int i_ = 0; i_ < (N); ++i_) pp.prof[(size_t)p * WN_PROF_SLOTS + (base) + i_] = pc_[i_]; }
#else
#define WN_PROF_DECL(N)
#define WN_PROF_START()
#define WN_TICK(i)
#define WN_TICK_AFTER(i, sink, v)
#define WN_PROF_STORE(base, N)
#endif

// ------------------------------------------------------------------------------------------
#define WN_NTC 128                 // threads of one compute group (4 warps)
#define WN_GW 4                    // warps per group
#define WN_DISPATCH_E(EV, ...)                                \
    switch (EV) {                                             \
        case 1: { constexpr int E = 1; __VA_ARGS__ } break;   \
        case 2: { constexpr int E = 2; __VA_ARGS__ } break;   \
        case 4: { constexpr int E = 4; __VA_ARGS__ } break;   \
        default: { constexpr int E = 8; __VA_ARGS__ } break;  \
    }

// STREAM: the kernel of wn_stream_generate (absolute steps, history and feedback in a state buffer).  A separate
// instantiation too: any code after the step loops changes the register allocation of the loops (the config-2 kernel
// then spills in its hot loop and loses 9 % on an H100 SXM at 400 W), so the whole-utterance kernels compile as before.
template <int BT, int ER, int EG, bool STREAM = false>
struct Engine {
    static constexpr int NV = 4 * BT;
    static constexpr int NA = (BT >= 8) ? 1 : 2;     // quads reduced together (their shuffle chains overlap)
    const WnPlan& pl;
    const WnPtrs& pp;
    unsigned char* sm;
    int tid, warp, lane, p;
    int gt, gw;                    // thread / warp index inside the compute group
    uint64_t *bar_full, *bar_empty, *bar_cfull, *bar_cempty;
    volatile int* s_abort;
    volatile int* s_stash_cnt;     // stashes published by the critical group (monotonic)
    volatile int* s_ddone_cnt;     // deferred-group warps finished, summed over stages (monotonic)
    int* ringtab;
    float *xs, *ys, *red1, *red2, *sb, *pre, *cond, *skipacc, *hs, *noise, *first, *slots;
    volatile float* ring;
    float* s_in;     // [BT] scalar feedback
    int* s_idx;      // [BT] class feedback
    float* s_dense;  // [BT][O] dense feedback (only without QUANTIZE)
    bool dead;

    __device__ Engine(const WnPlan& pl_, const WnPtrs& pp_, unsigned char* sm_)
        : pl(pl_), pp(pp_), sm(sm_) {
        // logical thread index: the SM's issue arbiter prefers the highest warp id among eligible warps, so the
        // critical group (logical warps 0-3) is mapped onto the highest physical warps when warp_reverse is set
        lane = threadIdx.x & 31;
        warp = pp.warp_reverse ? (WN_NTHREADS / 32 - 1) - (int)(threadIdx.x >> 5) : (int)(threadIdx.x >> 5);
        tid = warp * 32 + lane;
        p = blockIdx.x;
        gt = tid & (WN_NTC - 1);
        gw = warp & (WN_GW - 1);
        const int nslots = pl.nres + pl.nring;
        bar_full = reinterpret_cast<uint64_t*>(sm + pl.sm_bar);
        bar_empty = bar_full + nslots;
        bar_cfull = bar_empty + (pl.nring > 0 ? pl.nring : 1);
        bar_cempty = bar_cfull + 2;
        s_abort = reinterpret_cast<volatile int*>(sm + pl.sm_misc);
        s_stash_cnt = s_abort + 1;
        s_ddone_cnt = s_abort + 2;
        s_in = reinterpret_cast<float*>(sm + pl.sm_in);
        s_idx = reinterpret_cast<int*>(s_in + BT);
        s_dense = reinterpret_cast<float*>(s_idx + BT);
        ringtab = reinterpret_cast<int*>(sm + pl.sm_ringtab);
        xs = reinterpret_cast<float*>(sm + pl.sm_xs);
        ys = xs + 2 * pl.R * BT;
        red1 = reinterpret_cast<float*>(sm + pl.sm_red1);
        red2 = reinterpret_cast<float*>(sm + pl.sm_red2);
        sb = reinterpret_cast<float*>(sm + pl.sm_sb);
        pre = sb + (size_t)pl.L * pl.RA4 * BT;
        cond = reinterpret_cast<float*>(sm + pl.sm_cond);
        skipacc = reinterpret_cast<float*>(sm + pl.sm_skipacc);
        hs = reinterpret_cast<float*>(sm + pl.sm_hs);
        noise = reinterpret_cast<float*>(sm + pl.sm_noise);
        first = reinterpret_cast<float*>(sm + pl.sm_first);
        slots = reinterpret_cast<float*>(sm + pl.sm_slots);
        if (pl.ring_in_smem)
            ring = reinterpret_cast<volatile float*>(sm + pl.sm_ring);
        else
            ring = pp.ring_g + (size_t)p * pl.ring_pos_total * pl.RA4 * BT;
        dead = false;
    }

    // ---- watchdog: a stuck wait sets the device fault word and makes every block unwind
    __device__ __forceinline__ bool check_abort(uint32_t what, long long& t0) {
        t0 = wn_check_abort(s_abort, pp.err, pp.timeout_cycles, what, p, t0);
        return t0 < 0;
    }
    // `relaxed` waits (anything off the critical path) back off with nanosleep so that they do not
    // take issue slots and LSU bandwidth from the critical warp of the same SM sub-partition
    template <bool relaxed = false>
    __device__ __forceinline__ bool wait_bar(uint64_t* bar, uint32_t parity, uint32_t what) {
        uint32_t spins = 0;
        long long t0 = 0;
        while (!mbar_try_wait(bar, parity)) {
            if (relaxed) __nanosleep(64);
            if (((++spins) & (relaxed ? 63u : 255u)) == 0 && check_abort(what, t0)) return false;
        }
        return true;
    }
    // monotonic shared-memory counter (cross-group hand-off inside the block)
    template <bool relaxed = false>
    __device__ __forceinline__ void wait_count(volatile int* cnt, int need, uint32_t what) {
        uint32_t spins = 0;
        long long t0 = 0;
        while (*cnt < need) {
            if (relaxed) __nanosleep(32);
            if (((++spins) & (relaxed ? 63u : 255u)) == 0 && check_abort(what, t0)) {
                dead = true;
                return;
            }
        }
        __threadfence_block();
    }

    // ---- wait for a broadcast vector: thread owns elements k = gt + j*WN_NTC.
    // Which element of a K-vector is slot j of this thread.  With one utterance per launch a thread owns
    // PAIRS of adjacent elements so that one 16-byte load fetches two (value, tag) pairs: every L1-bypassing
    // coherent load is a round trip to L2 for the issuing warp and they do not overlap, so the
    // number of loads per thread is what sets the poll time.
    template <int E>
    __device__ __forceinline__ int elem(int j) const {
        if constexpr (BT == 1 && (E % 2) == 0) return 2 * gt + 2 * WN_NTC * (j >> 1) + (j & 1);
        else return gt + j * WN_NTC;
    }
    // `src` is the base of the block's replica, `e0` the first element of the vector
    template <int E>
    __device__ __forceinline__ uint32_t load_vec(const uint2* __restrict__ src, int e0, int K, uint32_t tag,
                                                 float (&x)[E][BT]) {
        uint32_t bad = 0;
        if constexpr (BT == 1 && (E % 2) == 0) {
            uint4 raw[E / 2];
#pragma unroll
            for (int j = 0; j < E / 2; ++j) {
                const int k = elem<E>(2 * j);
                raw[j] = make_uint4(0u, tag, 0u, tag);
                if (k < K) raw[j] = ld_pair2(src + wn_pair_index((long long)(e0 + k)));
            }
#pragma unroll
            for (int j = 0; j < E / 2; ++j) {
                bad |= (raw[j].y ^ tag) | ((elem<E>(2 * j) + 1 < K) ? (raw[j].w ^ tag) : 0u);
                x[2 * j][0] = __uint_as_float(raw[j].x);
                x[2 * j + 1][0] = __uint_as_float(raw[j].z);
            }
        } else {
#pragma unroll
            for (int j = 0; j < E; ++j) {
                const int k = elem<E>(j);
                if (k < K) {
                    const uint2* s = src + wn_pair_index((long long)(e0 + k) * BT);
                    if constexpr (BT == 1) {
                        const uint2 v = ld_pair(s);
                        x[j][0] = __uint_as_float(v.x);
                        bad |= v.y ^ tag;
                    } else {
#pragma unroll
                        for (int b = 0; b < BT; b += 2) {
                            const uint4 v = ld_pair2(s + b);
                            x[j][b] = __uint_as_float(v.x);
                            bad |= v.y ^ tag;
                            x[j][b + 1] = __uint_as_float(v.z);
                            bad |= v.w ^ tag;
                        }
                    }
                } else {
#pragma unroll
                    for (int b = 0; b < BT; ++b) x[j][b] = 0.f;
                }
            }
        }
        return bad;
    }
    // At a tile of 1 the polls are warp-uniform: every lane repeats its loads until the whole warp's elements have
    // arrived, and the watchdog's verdict is shared.  A lane that left the loop on its own would run the GEMV in a
    // divergent branch while other lanes of its warp still poll, and the warp's shuffle reduction would wait for the
    // last of them (every critical-group thread calls every poll, so all 32 lanes are here).  Larger tiles keep
    // per-lane polls: with the votes, -Xptxas -v shows more spill in <4,2,2>, <4,4,2,true> and <8,2,2>.
    static constexpr bool WARP_POLL = BT == 1;
    __device__ __forceinline__ static bool poll_all(bool mine) {
        if constexpr (WARP_POLL) return __all_sync(0xffffffffu, mine);
        else return mine;
    }
    __device__ __forceinline__ static bool poll_any(bool mine) {
        if constexpr (WARP_POLL) return __any_sync(0xffffffffu, mine);
        else return mine;
    }
    template <int E>
    __device__ __forceinline__ void poll_vec(const uint2* __restrict__ src, int e0, int K, uint32_t tag,
                                             float (&x)[E][BT]) {
        uint32_t spins = 0;
        long long t0 = 0;
        while (!poll_all(load_vec<E>(src, e0, K, tag, x) == 0)) {
            if (((++spins) & 63u) == 0 && poll_any(check_abort(tag, t0))) {
                dead = true;
                return;
            }
        }
    }
    // two vectors of the same exchange (y then x): all loads of an attempt are in flight together
    template <int EA, int EB>
    __device__ __forceinline__ void poll_vec2(const uint2* __restrict__ src, int ea, int KA, float (&a)[EA][BT],
                                              int eb, int KB, float (&b)[EB][BT], uint32_t tag) {
        uint32_t spins = 0;
        long long t0 = 0;
        while (true) {
            const uint32_t bad = load_vec<EA>(src, ea, KA, tag, a) | load_vec<EB>(src, eb, KB, tag, b);
            if (poll_all(bad == 0)) return;
            if (((++spins) & 63u) == 0 && poll_any(check_abort(tag, t0))) {
                dead = true;
                return;
            }
        }
    }
    template <int E>
    __device__ __forceinline__ void stash(float* dst, int K, const float (&x)[E][BT]) {
#pragma unroll
        for (int j = 0; j < E; ++j) {
            const int k = elem<E>(j);
            if (k < K) {
#pragma unroll
                for (int b = 0; b < BT; ++b) dst[k * BT + b] = x[j][b];
            }
        }
    }
    template <int E>
    __device__ __forceinline__ void unstash(const float* src, int K, float (&x)[E][BT]) {
#pragma unroll
        for (int j = 0; j < E; ++j) {
            const int k = elem<E>(j);
#pragma unroll
            for (int b = 0; b < BT; ++b) x[j][b] = (k < K) ? src[k * BT + b] : 0.f;
        }
    }

    // ---- one row quad (4 rows x K) times the thread's slice of the input vector, accumulated
    __device__ __forceinline__ static void fma_k(float4 w4, const float (&xk)[BT], float (&acc)[NV]) {
#pragma unroll
        for (int b = 0; b < BT; ++b) {
            acc[0 * BT + b] = fmaf(w4.x, xk[b], acc[0 * BT + b]);
            acc[1 * BT + b] = fmaf(w4.y, xk[b], acc[1 * BT + b]);
            acc[2 * BT + b] = fmaf(w4.z, xk[b], acc[2 * BT + b]);
            acc[3 * BT + b] = fmaf(w4.w, xk[b], acc[3 * BT + b]);
        }
    }
    template <int E>
    __device__ __forceinline__ void quad_fma(const float* __restrict__ wq /* [K][4] */, int K,
                                             const float (&x)[E][BT], float (&acc)[NV]) {
#pragma unroll
        for (int j = 0; j < E; ++j) {
            const int k = elem<E>(j);
            if (k < K) fma_k(*reinterpret_cast<const float4*>(wq + (size_t)k * 4), x[j], acc);
        }
    }

    // ---- layer stages 1..L-1: the weights of the first pass of NA quads are read into registers before the poll
    // (the ring slot is full once acquire_blob returns), so that after the exchange arrives only FMAs are left.
    // Weight w of that pass, w = h*(EG+ER) + j, is the float4 that multiplies y element j (j < EG; gate quads: M_{s-1},
    // residual quads: conv1x1_out_{s-1}) or x element j-EG (gate quads only: V_s) in quad h.  The first NPRE of them
    // are preloaded; the others are read from shared memory when they are used.  The kernel is held to 168 registers
    // (320 threads, one block per SM): -Xptxas -v shows no more stack or spill than without the preload only for a
    // tile of 1 with EG + ER <= 6 outside the stream kernels (config 2 is <1,4,2,false>); the other instantiations
    // read the weights as they multiply.
    static constexpr int NW0 = NA * (EG + ER);
    static constexpr int NPRE = (BT == 1 && !STREAM && EG + ER <= 6) ? (NW0 < 8 ? NW0 : 8) : 0;
    static constexpr int NPRE_A = NPRE > 0 ? NPRE : 1;
    __device__ __forceinline__ const float* w0y(const float* W, int h, int NQ_A) const {
        return h < NQ_A ? W + pl.lb_Zy + (size_t)h * pl.G2 * 4 : W + pl.lb_Xo + (size_t)(h - NQ_A) * pl.G2 * 4;
    }
    __device__ __forceinline__ void preload0(const float* W, int NQ_A, int nqc, float4 (&wp)[NPRE_A]) {
#pragma unroll
        for (int w = 0; w < NPRE; ++w) {
            const int h = w / (EG + ER), j = w % (EG + ER);
            const float* src = nullptr;
            if (j < EG) {
                const int k = elem<EG>(j);
                if (h < nqc && k < pl.G2) src = w0y(W, h, NQ_A) + (size_t)k * 4;
            } else {
                const int k = elem<ER>(j - EG);
                if (h < NQ_A && k < pl.R) src = W + pl.lb_Zx + ((size_t)h * pl.R + k) * 4;
            }
            wp[w] = src ? *reinterpret_cast<const float4*>(src) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    // the first pass: quad h sums y[0..EG) then x[0..ER), the order quad_fma sums in
    __device__ __forceinline__ void pass0(const float* W, int NQ_A, int nqc, const float4 (&wp)[NPRE_A],
                                          const float (&yr)[EG][BT], const float (&xr)[ER][BT], float (&acc)[NA][NV]) {
#pragma unroll
        for (int h = 0; h < NA; ++h) {
#pragma unroll
            for (int v = 0; v < NV; ++v) acc[h][v] = 0.f;
#pragma unroll
            for (int j = 0; j < EG; ++j) {
                const int k = elem<EG>(j), w = h * (EG + ER) + j;
                if (h < nqc && k < pl.G2)
                    fma_k(w < NPRE ? wp[w] : *reinterpret_cast<const float4*>(w0y(W, h, NQ_A) + (size_t)k * 4), yr[j],
                          acc[h]);
            }
#pragma unroll
            for (int j = 0; j < ER; ++j) {
                const int k = elem<ER>(j), w = h * (EG + ER) + EG + j;
                if (h < NQ_A && k < pl.R)
                    fma_k(w < NPRE ? wp[w] : *reinterpret_cast<const float4*>(W + pl.lb_Zx + ((size_t)h * pl.R + k) * 4),
                          xr[j], acc[h]);
            }
        }
    }
    // after the warp reduction lane (v << (5-M)) holds value v of the quad; warp gw's partial goes
    // to red[(q*NV + v)*4 + gw]
    __device__ __forceinline__ void quad_store(const float (&acc)[NV], int q, float* __restrict__ red) {
        constexpr int M = ilog2c(NV);
        if ((lane & ((32 >> M) - 1)) == 0) red[(q * NV + (lane >> (5 - M))) * WN_GW + gw] = acc[0];
    }
    __device__ __forceinline__ float red_sum(const float* red, int rowidx, int b) const {
        const int v = (rowidx >> 2) * NV + (rowidx & 3) * BT + b;
        const float4 a = *reinterpret_cast<const float4*>(red + v * WN_GW);
        return (a.x + a.y) + (a.z + a.w);
    }
    // simple GEMV over NQ quads, two quads per pass so that their shuffle chains overlap
    template <int E>
    __device__ __forceinline__ void gemv(const float* __restrict__ w, int NQ, int K, const float (&x)[E][BT],
                                         float* __restrict__ red, int q0 = 0) {
        for (int q = 0; q < NQ; q += NA) {
            float acc[NA][NV];
#pragma unroll
            for (int h = 0; h < NA; ++h) {
#pragma unroll
                for (int v = 0; v < NV; ++v) acc[h][v] = 0.f;
                if (q + h < NQ) quad_fma<E>(w + (size_t)(q + h) * K * 4, K, x, acc[h]);
            }
            reduce_scatter_multi<NA, NV>(acc, lane);
#pragma unroll
            for (int h = 0; h < NA; ++h)
                if (q + h < NQ) quad_store(acc[h], q0 + q + h, red);
        }
    }
    __device__ __forceinline__ void publish(int elem, int b, int copy, float v, uint32_t tag) {
        st_pair(pp.xbuf + (size_t)copy * pl.copy_stride_pairs + wn_pair_index((long long)elem * BT + b), v, tag);
    }

    // ---- weight slots.  Every compute warp walks the blobs 0..L of every step in order; the ones that
    // stream go through the ring, tracked by a running (slot, parity) pair (no divisions).
    int rs_slot = 0;
    uint32_t rs_par = 0;
    __device__ __forceinline__ const float* acquire_blob(int t, int i) {
        if (i < pl.nres) {
            if (t == 0 && !wait_bar(&bar_full[i], 0, 0x80000000u | (uint32_t)i)) dead = true;
            return slots + (size_t)i * pl.slot_floats;
        }
        const int slot = pl.nres + rs_slot;
        if (!wait_bar(&bar_full[slot], rs_par, 0x80000000u | (uint32_t)i)) dead = true;
        return slots + (size_t)slot * pl.slot_floats;
    }
    __device__ __forceinline__ void release_blob(int t, int i) {
        if (i >= pl.nres) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&bar_empty[rs_slot]);
            if (++rs_slot == pl.nring) {
                rs_slot = 0;
                rs_par ^= 1u;
            }
        }
    }

    // ======================================================================================
    // weight streaming warp.  The streamed blobs (nres..L, every step) go through the shared-memory ring;
    // the ring can only be pl.nring blobs deep, so in addition the warp asks L2 to fetch the blob pl.l2_pf
    // places further along the same sequence (wrapping into the next step, never past the last step of the
    // launch) before it issues each copy.  The ring copies read with an evict-first policy: a blob already
    // in shared memory leaves L2 before the prefetched blobs that are still to be copied.
    // ======================================================================================
    __device__ void tma_loop() {
        if (lane != 0) return;
        const float* base = pp.wpack + (size_t)p * pl.cta_w_floats;
        for (int i = 0; i < pl.nres; ++i) {
            const uint32_t bytes = (uint32_t)wn_blob_floats(pl, i) * 4u;
            mbar_expect_tx(&bar_full[i], bytes);
            bulk_g2s(slots + (size_t)i * pl.slot_floats, base + wn_blob_off(pl, i), bytes, &bar_full[i]);
        }
        const int nstream = pl.nblobs - pl.nres;
        if (nstream <= 0) return;
        const uint32_t total = (uint32_t)pp.T * (uint32_t)nstream;
        const uint32_t dist = (uint32_t)pl.l2_pf < total ? (uint32_t)pl.l2_pf : total;
        int ipf = pl.nres;          // next blob to prefetch: dist blobs ahead of i
        for (uint32_t k = 0; k < dist; ++k) {
            prefetch_l2(base + wn_blob_off(pl, ipf), (uint32_t)wn_blob_floats(pl, ipf) * 4u);
            if (++ipf == pl.nblobs) ipf = pl.nres;
        }
        const uint64_t pol = l2_policy_evict_first();
        int i = pl.nres;
#ifdef WN_STAGE_PROF
        const long long t_begin = clock64();
        long long t_wait = 0;
#endif
        for (uint32_t js = 0; js < total; ++js) {
            const uint32_t s = js % (uint32_t)pl.nring, u = js / (uint32_t)pl.nring;
            if (u > 0) {
#ifdef WN_STAGE_PROF
                const long long t_w = clock64();
#endif
                if (!wait_bar<true>(&bar_empty[s], (u - 1) & 1u, 0x40000000u | s)) return;
#ifdef WN_STAGE_PROF
                t_wait += clock64() - t_w;
#endif
            }
            if (dist > 0 && js + dist < total) {
                prefetch_l2(base + wn_blob_off(pl, ipf), (uint32_t)wn_blob_floats(pl, ipf) * 4u);
                if (++ipf == pl.nblobs) ipf = pl.nres;
            }
            const uint32_t bytes = (uint32_t)wn_blob_floats(pl, i) * 4u;
            uint64_t* fb = &bar_full[pl.nres + s];
            mbar_expect_tx(fb, bytes);
            bulk_g2s_hint(slots + (size_t)(pl.nres + s) * pl.slot_floats, base + wn_blob_off(pl, i), bytes, fb, pol);
            if (++i == pl.nblobs) i = pl.nres;
        }
#ifdef WN_STAGE_PROF
        if (pp.prof != nullptr) {
            pp.prof[(size_t)p * WN_PROF_SLOTS + WN_PS_TMA] = t_wait;
            pp.prof[(size_t)p * WN_PROF_SLOTS + WN_PS_TMA + 1] = clock64() - t_begin;
        }
#endif
    }

    // ======================================================================================
    // conditioning warp: cond[t&1][l][row][b] = Wc_l[rows] . c_t  (modules.py:141-145), one step
    // ahead of the compute warps; weights come straight from L2 (they are read once per step)
    // ======================================================================================
    __device__ void cond_loop() {
        const int C = pl.C, L = pl.L, T = pp.T, B = pp.B;
        constexpr int NV = 4 * BT;
        constexpr int M = ilog2c(NV);
        const float* cw = pp.cwpack + (size_t)p * pl.cta_cw_floats;
#ifdef WN_STAGE_PROF
        const long long t_begin = clock64();
        long long t_wait = 0;
#endif
        for (int t = 0; t < T; ++t) {
            const int par = t & 1, u = t >> 1;
            if (u > 0) {
#ifdef WN_STAGE_PROF
                const long long t_w = clock64();
#endif
                if (!wait_bar<true>(&bar_cempty[par], (u - 1) & 1u, 0x20000000u)) return;
#ifdef WN_STAGE_PROF
                t_wait += clock64() - t_w;
#endif
            }
            float ct[BT][WN_MAX_CI];
#pragma unroll
            for (int b = 0; b < BT; ++b)
#pragma unroll
                for (int i = 0; i < WN_MAX_CI; ++i) {
                    const int ch = lane + 32 * i;
                    ct[b][i] = (b < B && ch < C) ? __ldg(pp.c + ((size_t)b * T + t) * C + ch) : 0.f;
                }
            float* dst = cond + (size_t)par * L * pl.RA4 * BT;
            for (int l = 0; l < L; ++l) {
                for (int q = 0; q < pl.NQ_A; ++q) {
                    float acc[NV];
#pragma unroll
                    for (int v = 0; v < NV; ++v) acc[v] = 0.f;
                    const float* wq = cw + ((size_t)(l * pl.NQ_A + q) * C) * 4;
#pragma unroll
                    for (int i = 0; i < WN_MAX_CI; ++i) {
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
                    reduce_scatter<NV>(acc, lane);
                    if ((lane & ((32 >> M) - 1)) == 0) {
                        const int v = lane >> (5 - M);   // = row_in_quad*BT + b
                        dst[((size_t)l * pl.RA4 + q * 4 + v / BT) * BT + (v % BT)] = acc[0];
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&bar_cfull[par]);
        }
#ifdef WN_STAGE_PROF
        if (pp.prof != nullptr && lane == 0) {
            pp.prof[(size_t)p * WN_PROF_SLOTS + WN_PS_COND] = t_wait;
            pp.prof[(size_t)p * WN_PROF_SLOTS + WN_PS_COND + 1] = clock64() - t_begin;
        }
#endif
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
    // noise for step t of utterance b into noise[b][*]; layout [u1(0..K-1) | u2 or z] or [e(0..O-1)]
    __device__ void fetch_noise(int t, int b) {
        float* nz = noise + (size_t)b * (pl.O + 2);
        const int B = pp.Btot, K = pl.Kmix, O = pl.O;
        const uint32_t ub = (uint32_t)(pp.b0 + b);
        const bool replay = pp.noise_kind == 0;
        const uint2 key = make_uint2((uint32_t)pp.seed, (uint32_t)(pp.seed >> 32));
        const uint32_t tc = (STREAM ? pp.t_base : 0u) + (uint32_t)t;   // Philox counts absolute steps; replay is per launch
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
    // draw sample of utterance b from hs[:, b]; sets the feedback for step t+1 and writes outputs
    __device__ void sample_utt(int t, int b) {
        const int O = pl.O, K = pl.Kmix, T = pp.T;
        const float* nz = noise + (size_t)b * (pl.O + 2);
        const bool writer = (p == 0);
        if (pl.head_kind == 2) {
            const bool softmax = (pp.flags & WN_FLAG_SOFTMAX_) != 0, quant = (pp.flags & WN_FLAG_QUANTIZE_) != 0;
            // F.softmax (wavenet.py:332): exp(h - max) / sum
            if (softmax) {
                float m = -INFINITY;
                for (int i = lane; i < O; i += 32) m = fmaxf(m, hs[i * BT + b]);
#pragma unroll
                for (int off = 16; off >= 1; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
                float s = 0.f;
                for (int i = lane; i < O; i += 32) {
                    const float e = expf(hs[i * BT + b] - m);
                    hs[i * BT + b] = e;
                    s += e;
                }
#pragma unroll
                for (int off = 16; off >= 1; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
                for (int i = lane; i < O; i += 32) hs[i * BT + b] = hs[i * BT + b] / s;
            }
            if (quant) {
                // OneHotCategorical(p).sample() (wavenet.py:334-335): renormalise, argmax(p / Exp(1))
                float sp = 0.f;
                for (int i = lane; i < O; i += 32) sp += hs[i * BT + b];
#pragma unroll
                for (int off = 16; off >= 1; off >>= 1) sp += __shfl_xor_sync(0xffffffffu, sp, off);
                float best = -INFINITY;
                int bi = 0x7fffffff;
                for (int i = lane; i < O; i += 32) {
                    const float r = (hs[i * BT + b] / sp) / nz[i];
                    if (r > best) {
                        best = r;
                        bi = i;
                    }
                }
                warp_argmax(best, bi);
                if (bi >= O) bi = 0;
                if (lane == 0) {
                    if (writer && b < pp.B) pp.out_index[(size_t)b * T + t] = bi;
                    s_idx[b] = (t + 1 < pp.T_test && b < pp.B) ? (pp.test_index ? pp.test_index[(size_t)b * pp.T_test + t + 1] : -1)
                                                               : bi;
                }
            } else {
                for (int i = lane; i < O; i += 32) {
                    const float v = hs[i * BT + b];
                    if (writer && b < pp.B) pp.out_dense[((size_t)b * O + i) * T + t] = v;
                    s_dense[b * O + i] = v;
                }
                if (lane == 0)
                    s_idx[b] = (t + 1 < pp.T_test && b < pp.B && pp.test_index)
                                   ? pp.test_index[(size_t)b * pp.T_test + t + 1] : -1;
            }
            // teacher forcing with dense rows overrides the feedback
            if (t + 1 < pp.T_test && pp.test_dense != nullptr && b < pp.B) {
                for (int i = lane; i < O; i += 32)
                    s_dense[b * O + i] = pp.test_dense[((size_t)b * pp.T_test + t + 1) * O + i];
                if (lane == 0) s_idx[b] = -1;
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
                const float g = hs[i * BT + b] - logf(-logf(nz[i]));
                if (g > best) {
                    best = g;
                    bi = i;
                }
            }
            warp_argmax(best, bi);
            if (bi >= K) bi = 0;
            mean = hs[(K + bi) * BT + b];        // mixture.py:143-146 one-hot select
            ls = hs[(2 * K + bi) * BT + b];
        } else if (O == 2) {
            mean = hs[0 * BT + b];               // mixture.py:258-259
            ls = hs[1 * BT + b];
        } else {
            mean = hs[1 * BT + b];               // mixture.py:260-261 (C == 3)
            ls = hs[2 * BT + b];
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
            s_in[b] = (t + 1 < pp.T_test && b < pp.B) ? pp.test_scalar[(size_t)b * pp.T_test + t + 1] : xv;
        }
    }

    // ======================================================================================
    // compute groups
    // ======================================================================================
    __device__ __forceinline__ static int efor(int K) {
        return K <= WN_NTC ? 1 : (K <= 2 * WN_NTC ? 2 : (K <= 4 * WN_NTC ? 4 : 8));
    }

    // x_0 = first 1x1 conv of the fed-back sample (wavenet.py:308); every block computes all of it
    __device__ __forceinline__ void make_x0(float (&x)[ER][BT]) {
        const int R = pl.R, O = pl.O;
#pragma unroll
        for (int j = 0; j < ER; ++j) {
            const int k = elem<ER>(j);
#pragma unroll
            for (int b = 0; b < BT; ++b) x[j][b] = 0.f;
            if (k < R) {
                if (pl.input_kind == 0) {
#pragma unroll
                    for (int b = 0; b < BT; ++b) x[j][b] = fmaf(first[k], s_in[b], first[R + k]);
                } else {
#pragma unroll
                    for (int b = 0; b < BT; ++b) {
                        const int idx = min(s_idx[b], O - 1);      // class ids are range-checked on the host where it can
                        if (idx >= 0) {
                            // one-hot input: the GEMV is a column gather
                            x[j][b] = __ldg(pp.first_w + (size_t)idx * R + k) + first[R + k];
                        } else {
                            float a = 0.f;
                            for (int o = 0; o < O; ++o)
                                a = fmaf(__ldg(pp.first_w + (size_t)o * R + k), s_dense[b * O + o], a);
                            x[j][b] = a + first[R + k];
                        }
                    }
                }
            }
        }
    }
    // modules.py:154  tanh(a) * sigmoid(g) with a single division:
    //   (1 - e^{-2a}) / ((1 + e^{-2a}) (1 + e^{-g}));  |a| is clamped where tanh has saturated in fp32.
    // Absolute error ~1e-7 (the subtraction 1 - e^{-2a} loses relative, not absolute, accuracy near 0).
    __device__ __forceinline__ static float gate(float a, float g) {
        const float ac = fminf(fmaxf(a, -15.0f), 15.0f);
        const float ea = expf(-2.0f * ac), eg = expf(-g);
        return (1.0f - ea) / ((1.0f + ea) * (1.0f + eg));
    }
    // Everything of z_l(t) that does not depend on step t's broadcasts: (folded) bias + global conditioning
    // + local conditioning projection + the queued products of the older taps.  The deferred group builds
    // the whole table for step `t` while the critical group is still in the head of step t-1.
    __device__ void build_pre(int t) {
        const int L = pl.L, RA4 = pl.RA4, kw = pl.kw, n = L * pl.RA * BT;
        if (pl.C > 0) {
            if (!wait_bar<true>(&bar_cfull[t & 1], (uint32_t)(t >> 1) & 1u, 0x10000000u)) dead = true;
        }
        const float* cd = cond + (size_t)(t & 1) * L * RA4 * BT;
        for (int i = gt; i < n; i += WN_NTC) {
            const int b = i % BT, rr = (i / BT) % pl.RA, l = i / (BT * pl.RA);
            const int idx = (l * RA4 + rr) * BT + b;
            float v = sb[idx];
            if (pl.C > 0) v += cd[idx];
            for (int k = 0; k < kw - 1; ++k) {
                const int e = (l * (kw - 1) + k) * 3;
                int pos = ringtab[e + 2];
                if (t > 0) { ++pos; if (pos == ringtab[e + 1]) pos = 0; }     // the table still holds (t-1) mod delay
                v += ring[((size_t)ringtab[e] + pos) * RA4 * BT + rr * BT + b];
            }
            pre[idx] = v;
        }
        __syncwarp();
        if (pl.C > 0) {
            // the conditioning warp may refill cond[t&1] once all four deferred warps are done with it
            if (lane == 0) mbar_arrive(&bar_cempty[t & 1]);
        }
    }

    // --------------------------------------------------------------------------------------
    // critical group (warps 0-3)
    // --------------------------------------------------------------------------------------
    __device__ void crit_loop() {
        const int L = pl.L, R = pl.R, G2 = pl.G2, S = pl.S, O = pl.O, T = pp.T, P = pl.P, ncopy = pl.ncopy;
        int y0, ny, x0r, nx, s0, ns, a0, na, b0, nb;
        wn_part(G2, P, p, y0, ny);
        wn_part(R, P, p, x0r, nx);
        wn_part(S, P, p, s0, ns);
        wn_part(S, P, p, a0, na);
        wn_part(O, P, p, b0, nb);
        const int ES = efor(S), EO = efor(O);
        const uint2* xin = pp.xbuf + (size_t)(p % ncopy) * pl.copy_stride_pairs;
        const uint32_t NEID = (uint32_t)L + 3u;
        const int YX = G2 + R;
        const float RSQRT2 = 0.70710678118654752440f;         // math.sqrt(0.5), modules.py:162
        const int NQ_A = pl.NQ_A, NQ_BO = pl.NQ_BO, nqc = NQ_A + NQ_BO;
        // finalizer roles: threads [0,64) publish gate outputs (and skip / head rows), [64,128) the
        // residual rows; local index u -> (item, replica)
        const int fl = gt & 63;
        const bool grpA = gt < 64;
        auto role = [&](int nitems, int& item, int& copy) {
            item = -1; copy = 0;
            if (nitems > 0 && fl < nitems * ncopy) { item = fl % nitems; copy = fl / nitems; }
        };
        int it_y, cp_y, it_x, cp_x, it_s, cp_s, it_a, cp_a, it_b, cp_b;
        role(ny * BT, it_y, cp_y);
        role(nx * BT, it_x, cp_x);
        role(ns * BT, it_s, cp_s);
        role(na * BT, it_a, cp_a);
        role(nb * BT, it_b, cp_b);
        if (!grpA) it_y = it_s = it_a = it_b = -1;
        if (grpA) it_x = -1;
        const int pa_idx = it_y >= 0 ? (2 * (it_y / BT)) * BT + (it_y % BT) : 0;   // [row a_j][b]; row b_j is BT further
        float xr[ER][BT], yr[EG][BT];
        WN_PROF_DECL(WN_PC_CRIT)
#ifdef WN_STAGE_PROF
        // arrival at the group barrier (low 32 bits of the clock), by stage parity: the last 4 of the 2*nblobs+8
        // mbarrier words, which no mbarrier uses (no static shared memory: it would shrink the dynamic map)
        volatile uint32_t* s_arrive = reinterpret_cast<volatile uint32_t*>(bar_full + 2 * pl.nblobs + 4);
        long long skew = 0, nskew = 0, nlast[WN_GW] = {};
#endif
        int nstash = 0;      // stashes published so far == deferred stages started
        int ndone = 0;       // deferred stages this group has waited for
        long long t_pub = clock64();
        if (bar_groups(false)) return;      // the deferred group has built the pre-sums of step 0

        for (int t = 0; t < T; ++t) {
            const uint32_t tagbase = (uint32_t)t * NEID + 1u;
            WN_PROF_START();
            bool step_dead = false;
            do {
                make_x0(xr);
                WN_TICK(WN_PC_TAIL);
                // ------------------------------------------------------------ stage 0: layer 0 from x_0
                {
                    const float* W = acquire_blob(t, 0);
                    float pre_a = 0.f, pre_b = 0.f;
                    if (it_y >= 0) { pre_a = pre[pa_idx]; pre_b = pre[pa_idx + BT]; }
                    float* r1 = red1;                                   // partials buffers alternate by stage
                    gemv<ER>(W + pl.fb_Zx, NQ_A, R, xr, r1);
                    if (bar_or_n<1, WN_NTC>(dead)) { step_dead = true; break; }
                    if (it_y >= 0) {
                        const int fr = it_y / BT, fb = it_y % BT;
                        const float a = red_sum(r1, 2 * fr, fb) + pre_a;
                        const float g = red_sum(r1, 2 * fr + 1, fb) + pre_b;
                        publish(pl.ex_yx + y0 + fr, fb, cp_y, gate(a, g), tagbase + wn_eid_yx(0));
                    }
                    release_blob(t, 0);
                    t_pub = clock64();
                    WN_TICK(WN_PC_HEAD);
                }
                // ------------------------------------------------------------ stages 1..L-1
                for (int s = 1; s < L; ++s) {
                    const float* W = acquire_blob(t, s);
                    float pre_a = 0.f, pre_b = 0.f;
                    if (it_y >= 0) { pre_a = pre[pa_idx + s * pl.RA4 * BT]; pre_b = pre[pa_idx + s * pl.RA4 * BT + BT]; }
                    float4 wp[NPRE_A];
                    if constexpr (NPRE > 0) preload0(W, NQ_A, nqc, wp);
                    WN_TICK(WN_PC_ACQ);
                    {
                        const int e0 = pl.ex_yx + (s - 1) * YX;
                        const uint32_t tag = tagbase + wn_eid_yx(s - 1);
                        if (pp.gate_cycles > 0) { while (clock64() - t_pub < pp.gate_cycles) {} }
                        if (s >= 2) poll_vec2<EG, ER>(xin, e0, G2, yr, e0 + G2, R, xr, tag);
                        else poll_vec<EG>(xin, e0, G2, tag, yr);      // x_0 is already in registers
                    }
                    WN_TICK(WN_PC_POLL);
                    float* xst = xs + (size_t)(s & 1) * R * BT;
                    float* r1 = red1 + (size_t)(s & 1) * pl.red1_floats;
                    stash<ER>(xst, R, xr);
                    stash<EG>(ys + (size_t)(s & 1) * G2 * BT, G2, yr);
                    WN_TICK(WN_PC_STASH);
                    // gate pre-activations of layer s (quads [0,NQ_A)) and residual rows x_s (quads [NQ_A,nqc))
                    for (int q = 0; q < nqc; q += NA) {
                        float acc[NA][NV];
                        if (NPRE > 0 && q == 0) {
                            pass0(W, NQ_A, nqc, wp, yr, xr, acc);
                        } else {
#pragma unroll
                            for (int h = 0; h < NA; ++h) {
#pragma unroll
                                for (int v = 0; v < NV; ++v) acc[h][v] = 0.f;
                                const int qq = q + h;
                                if (qq < NQ_A) {
                                    quad_fma<EG>(W + pl.lb_Zy + (size_t)qq * G2 * 4, G2, yr, acc[h]);
                                    quad_fma<ER>(W + pl.lb_Zx + (size_t)qq * R * 4, R, xr, acc[h]);
                                } else if (qq < nqc) {
                                    quad_fma<EG>(W + pl.lb_Xo + (size_t)(qq - NQ_A) * G2 * 4, G2, yr, acc[h]);
                                }
                            }
                        }
                        WN_TICK(WN_PC_FMA);
                        WN_TICK_AFTER(WN_PC_READY, r1 + (size_t)q * NV * WN_GW + gw, acc[NA - 1][NV - 1]);
                        reduce_scatter_multi<NA, NV>(acc, lane);
                        WN_TICK(WN_PC_REDUCE);
#pragma unroll
                        for (int h = 0; h < NA; ++h)
                            if (q + h < nqc) quad_store(acc[h], q + h, r1);
                        WN_TICK(WN_PC_STORE);
                    }
#ifdef WN_STAGE_PROF
                    if (prof_) s_arrive[(s & 1) * WN_GW + gw] = (uint32_t)tc_;
#endif
                    if (bar_or_n<1, WN_NTC>(dead)) { step_dead = true; break; }
                    WN_TICK(WN_PC_BAR);
#ifdef WN_STAGE_PROF
                    if (prof_ && gw == 0) {
                        const uint32_t a0 = s_arrive[(s & 1) * WN_GW];
                        int lo = 0, hi = 0, last = 0;
                        for (int w = 1; w < WN_GW; ++w) {
                            const int a = (int)(s_arrive[(s & 1) * WN_GW + w] - a0);
                            lo = min(lo, a);
                            if (a > hi) { hi = a; last = w; }
                        }
                        skew += hi - lo;
                        ++nskew;
                        ++nlast[last];
                    }
#endif
                    // stash complete (the barrier ordered every thread's writes).  The last thread of the group hands
                    // it over: it publishes nothing unless a block owns 64 rows of a vector, whereas thread 0 publishes
                    // a gate output, and the fence would delay that publish in every stage.
                    if (gt == WN_NTC - 1) {
                        __threadfence_block();
                        *s_stash_cnt = nstash + 1;
                    }
                    ++nstash;
                    const uint32_t tag = tagbase + wn_eid_yx(s);
                    float vy = 0.f, vx = 0.f;
                    if (it_y >= 0) {
                        const int fr = it_y / BT, fb = it_y % BT;
                        const float a = red_sum(r1, 2 * fr, fb) + pre_a;
                        const float g = red_sum(r1, 2 * fr + 1, fb) + pre_b;
                        vy = gate(a, g);
                    }
                    if (it_x >= 0) {
                        // modules.py:160-162  x_s = (conv1x1_out(y_{s-1}) + x_{s-1}) * sqrt(0.5)
                        const int fr = it_x / BT, fb = it_x % BT;
                        const float o = red_sum(r1, NQ_A * 4 + fr, fb) + W[pl.lb_xb + fr];
                        vx = (o + xst[(x0r + fr) * BT + fb]) * RSQRT2;
                    }
                    WN_TICK(WN_PC_FIN);
                    if (it_y >= 0) publish(pl.ex_yx + s * YX + y0 + it_y / BT, it_y % BT, cp_y, vy, tag);
                    if (it_x >= 0) publish(pl.ex_yx + s * YX + G2 + x0r + it_x / BT, it_x % BT, cp_x, vx, tag);
                    release_blob(t, s);
                    t_pub = clock64();
                    WN_TICK(WN_PC_PUB);
                    // the stash of stage s+1 reuses the buffer of stage s-1: the deferred group must be done with it
                    if (s >= 2) { wait_count(s_ddone_cnt, WN_GW * (ndone + 1), 0x08000000u); ++ndone; }
                    WN_TICK(WN_PC_DDONE);
                }
                if (step_dead) break;
                // ------------------------------------------------------------ stage L: skip of the last layer
                const float* H = acquire_blob(t, L);
                {
                    const int e0 = pl.ex_yx + (L - 1) * YX;
                    const uint32_t tag = tagbase + wn_eid_yx(L - 1);
                    if (L >= 2) poll_vec2<EG, ER>(xin, e0, G2, yr, e0 + G2, R, xr, tag);
                    else poll_vec<EG>(xin, e0, G2, tag, yr);
                }
                stash<ER>(xs + (size_t)(L & 1) * R * BT, R, xr);
                float* r1 = red1 + (size_t)(L & 1) * pl.red1_floats;
                gemv<EG>(H + pl.tb_Sk, pl.NQ_BS, G2, yr, r1);
                if (bar_or_n<1, WN_NTC>(dead)) { step_dead = true; break; }
                if (gt == WN_NTC - 1) {     // not a publisher of the skip rows (see the layer stages)
                    __threadfence_block();
                    *s_stash_cnt = nstash + 1;
                }
                ++nstash;
                // skip rows of layers 0..L-2 were accumulated by the deferred group: wait for its stage L-1
                if (L >= 2) { wait_count(s_ddone_cnt, WN_GW * (ndone + 1), 0x08000001u); ++ndone; }
                if (it_s >= 0) {
                    // (s_0 + ... + s_{L-2}) + s_{L-1}, * sqrt(1/L), first ReLU of the head (wavenet.py:312-315)
                    const int fr = it_s / BT, fb = it_s % BT;
                    float tot = red_sum(r1, fr, fb) + H[pl.tb_sb + fr];
                    if (L >= 2) tot = skipacc[it_s] + tot;
                    publish(pl.ex_sk + s0 + fr, fb, cp_s, fmaxf(tot * pl.skip_scale, 0.f), tagbase + wn_eid_sk(pl));
                }
                // ---------------------------------------------------------------- head (wavenet.py:315-319)
                float* r1a = red1 + (size_t)((L + 1) & 1) * pl.red1_floats;
                if (na > 0) {
                    WN_DISPATCH_E(ES, { float h[E][BT];
                                        poll_vec<E>(xin, pl.ex_sk, S, tagbase + wn_eid_sk(pl), h);
                                        gemv<E>(H + pl.tb_Ha, pl.NQ_HA, S, h, r1a); });
                }
                if (bar_or_n<1, WN_NTC>(dead)) { step_dead = true; break; }
                if (it_a >= 0) {
                    const int fr = it_a / BT, fb = it_a % BT;
                    publish(pl.ex_h1 + a0 + fr, fb, cp_a, fmaxf(red_sum(r1a, fr, fb) + H[pl.tb_Hab + fr], 0.f), tagbase + wn_eid_h1(pl));
                }
                if (nb > 0) {
                    WN_DISPATCH_E(ES, { float h[E][BT];
                                        poll_vec<E>(xin, pl.ex_h1, S, tagbase + wn_eid_h1(pl), h);
                                        gemv<E>(H + pl.tb_Hb, pl.NQ_HB, S, h, r1); });
                }
                if (bar_or_n<1, WN_NTC>(dead)) { step_dead = true; break; }
                if (it_b >= 0) {
                    const int fr = it_b / BT, fb = it_b % BT;
                    publish(pl.ex_h2 + b0 + fr, fb, cp_b, red_sum(r1, fr, fb) + H[pl.tb_Hbb + fr], tagbase + wn_eid_h2(pl));
                }
                release_blob(t, L);
                {
                    WN_DISPATCH_E(EO, { float h[E][BT];
                                        poll_vec<E>(xin, pl.ex_h2, O, tagbase + wn_eid_h2(pl), h);
                                        stash<E>(hs, O, h); });
                }
                WN_TICK(WN_PC_HEAD);
            } while (false);
            // ---- both groups meet: sampler (one warp per utterance), then the next step
            if (bar_groups(dead || step_dead)) return;
            // the deferred group finished its stage L before this barrier
            if (L >= 1) ++ndone;
            step_tail(t);
            if (bar_groups(false)) return;
            WN_TICK(WN_PC_TAIL);
        }
        WN_PROF_STORE(gw * WN_PC_CRIT, WN_PC_CRIT)
#ifdef WN_STAGE_PROF
        if (prof_ && gw == 0) {
            long long* out = pp.prof + (size_t)p * WN_PROF_SLOTS;
            out[WN_PS_SKEW] = skew;
            out[WN_PS_SKEW + 1] = nskew;
            for (int w = 0; w < WN_GW; ++w) out[WN_PS_SKEW + 2 + w] = nlast[w];
        }
#endif
    }

    // head outputs are in hs: optional dump, sampling, feedback for the next step (all 8 compute warps)
    __device__ __forceinline__ void step_tail(int t) {
        const int O = pl.O, T = pp.T;
        if (p == 0 && pp.params_out != nullptr) {
            for (int i = tid; i < O * BT; i += WN_NT) {
                const int o = i / BT, b = i % BT;
                if (b < pp.B) pp.params_out[((size_t)b * O + o) * T + t] = hs[i];
            }
            // the softmax sampler overwrites hs in place: finish the copy first (block-uniform)
            if (pl.head_kind == 2) bar_groups(false);
        }
        if (warp < BT) {
            sample_utt(t, warp);
#ifndef WN_NO_SAMPLER_SYNCWARP
            __syncwarp();                 // every lane has read step t's draws before they are overwritten
#endif
            if (t + 1 < T) fetch_noise(t + 1, warp);
        }
        // advance the ring positions to (t+1) mod delay
        for (int i = WN_NT - 1 - tid; i < pl.L * (pl.kw - 1); i += WN_NT) {
            const int pos = ringtab[i * 3 + 2] + 1;
            ringtab[i * 3 + 2] = (pos == ringtab[i * 3 + 1]) ? 0 : pos;
        }
    }

    // --------------------------------------------------------------------------------------
    // deferred group (warps 4-7): queued older-tap products and skip rows, one stage behind
    // --------------------------------------------------------------------------------------
    __device__ void def_loop() {
        const int L = pl.L, R = pl.R, G2 = pl.G2, T = pp.T, P = pl.P, kw = pl.kw;
        int s0, ns;
        wn_part(pl.S, P, p, s0, ns);
        const int NQ_D = pl.NQ_D, NQ_BS = pl.NQ_BS, nqd = (kw > 1 ? NQ_D : 0) + NQ_BS;
        const int qoff = (kw > 1 ? NQ_D : 0);
        const int nring_items = (kw - 1) * pl.RA * BT, nskip_items = ns * BT;
        float xr[ER][BT], yr[EG][BT];
        WN_PROF_DECL(WN_PC_DEF)
        int nstash = 0;

        // one deferred stage: `Td` = older taps of `layer` (uses x), `Sk`/`skb` = skip rows of `layer`
        // (uses y; nullptr in the tail stage, where the critical group evaluates them itself)
        auto stage = [&](int t, int s, int layer, const float* Td, const float* Sk, const float* skb) {
            wait_count<true>(s_stash_cnt, nstash + 1, 0x04000000u);
            ++nstash;
            WN_TICK(WN_PD_WAIT);
            unstash<ER>(xs + (size_t)(s & 1) * R * BT, R, xr);
            if (Sk) unstash<EG>(ys + (size_t)(s & 1) * G2 * BT, G2, yr);
            WN_TICK(WN_PD_UNSTASH);
            float* red = red2 + (size_t)(s & 1) * pl.red2_floats;
            const int nq = Sk ? nqd : qoff;
            for (int q = 0; q < nq; q += NA) {
                float acc[NA][NV];
#pragma unroll
                for (int h = 0; h < NA; ++h) {
#pragma unroll
                    for (int v = 0; v < NV; ++v) acc[h][v] = 0.f;
                    const int qq = q + h;
                    if (qq < qoff) quad_fma<ER>(Td + (size_t)qq * R * 4, R, xr, acc[h]);
                    else if (qq < nq) quad_fma<EG>(Sk + (size_t)(qq - qoff) * G2 * 4, G2, yr, acc[h]);
                }
                reduce_scatter_multi<NA, NV>(acc, lane);
#pragma unroll
                for (int h = 0; h < NA; ++h)
                    if (q + h < nq) quad_store(acc[h], q + h, red);
            }
            WN_TICK(WN_PD_GEMV);
            const bool d = bar_or_n<2, WN_NTC>(dead);
            WN_TICK(WN_PD_BAR);
            if (!d) {
                // older-tap products of `layer` -> history ring (consumed at steps t+d, t+2d, conv.py:32-44)
                for (int f = gt; f < nring_items; f += WN_NTC) {
                    const int dr = f / BT, db = f % BT, tap = dr / pl.RA, rr = dr % pl.RA;
                    const int e = (layer * (kw - 1) + tap) * 3;
                    ring[((size_t)ringtab[e] + ringtab[e + 2]) * pl.RA4 * BT + rr * BT + db] = red_sum(red, dr, db);
                }
                // skip rows, accumulated in layer order (wavenet.py:312)
                if (Sk) {
                    for (int f = gt; f < nskip_items; f += WN_NTC) {
                        const int fr = f / BT, fb = f % BT;
                        const float h = red_sum(red, qoff * 4 + fr, fb) + skb[fr];
                        skipacc[f] = (layer == 0) ? h : skipacc[f] + h;
                    }
                }
            }
            __threadfence_block();
            __syncwarp();
            if (lane == 0) atomicAdd((int*)s_ddone_cnt, 1);
            WN_TICK(WN_PD_FIN);
            return d;
        };

        build_pre(0);
        if (bar_groups(dead)) return;
        for (int t = 0; t < T; ++t) {
            WN_PROF_START();
            bool step_dead = false;
            release_blob(t, 0);                       // stage 0 has no deferred work
            for (int s = 1; s < L && !step_dead; ++s) {
                const float* W = acquire_blob(t, s);
                step_dead = stage(t, s, s - 1, W + pl.lb_Td, W + pl.lb_Sk, W + pl.lb_sb);
                release_blob(t, s);
            }
            if (!step_dead) {
                const float* H = acquire_blob(t, L);
                step_dead = stage(t, L, L - 1, H + pl.tb_Td, nullptr, nullptr);
                release_blob(t, L);
            }
            if (!step_dead && t + 1 < T) {
                // all rings of step t are written (group barrier inside stage()): pre-sums of step t+1
                if (bar_or_n<2, WN_NTC>(dead)) step_dead = true;
                else build_pre(t + 1);
            }
            if (bar_groups(dead || step_dead)) return;
            step_tail(t);
            if (bar_groups(false)) return;
            WN_TICK(WN_PD_REST);
        }
        WN_PROF_STORE(WN_PS_DEF + gw * WN_PC_DEF, WN_PC_DEF)
    }
};

// ------------------------------------------------------------------------------------------
// Stream epilogue (compute threads only).  Both loops end every step on a group barrier after the deferred group's
// ring writes and the sampler's feedback, so the rings and the feedback of step T are final here.  Nothing else
// carries over a step: skipacc restarts at layer 0, stash / partials / pre-sums are per stage.
// ------------------------------------------------------------------------------------------
template <int BT>
__device__ __noinline__ void wn_store_state(const WnPlan& pl, const WnPtrs& pp, unsigned char* sm) {
    const int warp = pp.warp_reverse ? (WN_NTHREADS / 32 - 1) - (int)(threadIdx.x >> 5) : (int)(threadIdx.x >> 5);
    const int tid = warp * 32 + (int)(threadIdx.x & 31), p = blockIdx.x;
    if (tid >= WN_NT) return;
    const long long ring_n = wn_state_ring_floats(pl);
    if (pl.ring_in_smem) {
        const volatile float* ring = reinterpret_cast<const volatile float*>(sm + pl.sm_ring);
        float* dst = pp.state + (size_t)p * ring_n;
        for (long long i = tid; i < ring_n; i += WN_NT) dst[i] = ring[i];
    }
    if (p == 0) {
        const float* s_in = reinterpret_cast<const float*>(sm + pl.sm_in);      // layout of Engine's s_in / s_idx / s_dense
        const int* s_idx = reinterpret_cast<const int*>(s_in + BT);
        const float* s_dense = reinterpret_cast<const float*>(s_idx + BT);
        float* fb = pp.state + (size_t)pl.P * ring_n;
        for (int b = tid; b < BT; b += WN_NT) {
            fb[b] = s_in[b];
            fb[BT + b] = __int_as_float(s_idx[b]);
        }
        if (pl.input_kind != 0)
            for (int i = tid; i < BT * pl.O; i += WN_NT) fb[2 * BT + i] = s_dense[i];
    }
}

// ------------------------------------------------------------------------------------------
// kernel entry
// ------------------------------------------------------------------------------------------
template <int BT, int ER, int EG, bool STREAM = false>
__global__ void __launch_bounds__(WN_NTHREADS, 1)
wn_persistent_kernel(const __grid_constant__ WnPlan pl, const __grid_constant__ WnPtrs pp) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    Engine<BT, ER, EG, STREAM> eng(pl, pp, smem_raw);
    const int tid = eng.tid, p = blockIdx.x;      // logical thread index (see Engine)
    const int nslots = pl.nres + pl.nring;
    if (tid == 0) {
        for (int i = 0; i < nslots; ++i) mbar_init(&eng.bar_full[i], 1);
        for (int i = 0; i < pl.nring; ++i) mbar_init(&eng.bar_empty[i], WN_NWARP);
        for (int i = 0; i < 2; ++i) {
            mbar_init(&eng.bar_cfull[i], 1);
            mbar_init(&eng.bar_cempty[i], WN_GW);
        }
        *eng.s_abort = 0;
        *eng.s_stash_cnt = 0;
        *eng.s_ddone_cnt = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // zero the history (== the reference's zero-initialised queue, conv.py:35-36) and scratch; a continued stream
    // loads the history its previous launch stored instead (rings in global memory ARE the state buffer: nothing to do)
    const long long ring_n = wn_state_ring_floats(pl);
    if (pl.ring_in_smem) {
        const float* src = (STREAM && pp.state_load) ? pp.state + (size_t)p * ring_n : nullptr;
        for (long long i = tid; i < ring_n; i += WN_NTHREADS) eng.ring[i] = src ? src[i] : 0.f;
    }
    for (int i = tid; i < pl.NSm * BT + 4; i += WN_NTHREADS) eng.skipacc[i] = 0.f;
    for (int i = tid; i < pl.L * (pl.kw - 1); i += WN_NTHREADS) {
        eng.ringtab[i * 3] = pp.ringtab[i * 2];           // offset of the ring (in positions)
        eng.ringtab[i * 3 + 1] = pp.ringtab[i * 2 + 1];   // delay D
        eng.ringtab[i * 3 + 2] = STREAM ? (int)(pp.t_base % (unsigned)pp.ringtab[i * 2 + 1]) : 0;   // (absolute t) mod D
    }
    for (int k = tid; k < pl.R; k += WN_NTHREADS) {
        eng.first[k] = (pl.input_kind == 0) ? pp.first_w[k] : 0.f;
        eng.first[pl.R + k] = pp.first_b[k];
    }
    {
        // static part of the pre-activation: (folded) conv bias + global-conditioning projection
        // (modules.py:148-152 recomputes Wg.g every step although g is constant; fold it once)
        int y0, ny;
        wn_part(pl.G2, pl.P, p, y0, ny);
        const float* blob0 = pp.wpack + (size_t)p * pl.cta_w_floats;
        const int n = pl.L * pl.RA4 * BT;
        for (int i = tid; i < n; i += WN_NTHREADS) {
            const int b = i % BT, rr = (i / BT) % pl.RA4, l = i / (BT * pl.RA4);
            float v = 0.f;
            if (rr < pl.RA && (rr >> 1) < ny) {
                v = blob0[wn_blob_off(pl, l) + (l == 0 ? pl.fb_zb : pl.lb_zb) + rr];
                if (pp.gbias != nullptr && b < pp.B) {
                    const int grow = (rr & 1) ? pl.G2 + y0 + (rr >> 1) : y0 + (rr >> 1);
                    v += pp.gbias[((size_t)b * pl.L + l) * pl.G + grow];
                }
            }
            eng.sb[i] = v;
        }
    }
    // feedback for step 0 (wavenet.py:281-301)
    if (tid < BT) {
        const int b = tid;
        float v = 0.f;
        int idx = -1;
        if (b < pp.B) {
            if (pl.input_kind == 0) {
                if (pp.T_test > 0) v = pp.test_scalar[(size_t)b * pp.T_test];
                else if (pp.initial) v = pp.initial[b];
            } else {
                if (pp.T_test > 0) idx = pp.test_index ? pp.test_index[(size_t)b * pp.T_test] : -1;
                else if (pp.initial_dense) idx = -1;
                else if (pp.initial_rows) idx = pp.initial_rows[b];
                else idx = pp.initial_index;
            }
        } else if (pl.input_kind != 0) idx = 0;
        const float* fb = (STREAM && pp.state_load) ? pp.state + (size_t)pl.P * ring_n : nullptr;   // the last launch's
        eng.s_in[b] = fb ? fb[b] : v;
        eng.s_idx[b] = fb ? __float_as_int(fb[BT + b]) : idx;
    }
    if (pl.input_kind != 0) {
        const float* dsrc = nullptr;
        size_t stride = 0;
        if (pp.T_test > 0 && pp.test_dense != nullptr) { dsrc = pp.test_dense; stride = (size_t)pp.T_test * pl.O; }
        else if (pp.T_test == 0 && pp.initial_dense != nullptr) { dsrc = pp.initial_dense; stride = (size_t)pl.O; }
        const float* fb = (STREAM && pp.state_load) ? pp.state + (size_t)pl.P * ring_n + 2 * BT : nullptr;
        for (int i = tid; i < BT * pl.O; i += WN_NTHREADS) {
            const int b = i / pl.O, o = i % pl.O;
            eng.s_dense[i] = fb ? fb[i] : ((dsrc && b < pp.B) ? dsrc[(size_t)b * stride + o] : 0.f);
        }
    }
    const int warp = tid >> 5;
    if (warp < BT && warp < WN_NWARP) eng.fetch_noise(0, warp);
    __syncthreads();
    if (warp == WN_NWARP) {
        eng.tma_loop();
        return;
    }
    if (warp == WN_NWARP + 1) {
        if (pl.C > 0) eng.cond_loop();
        return;
    }
    if (warp < WN_GW) eng.crit_loop();
    else eng.def_loop();
    if constexpr (STREAM) wn_store_state<BT>(pl, pp, smem_raw);
}

// gbias[b][l][row] = Wg_l[row,:] . g_b   (modules.py:148-152), once per call
__global__ void wn_gbias_kernel(const float* __restrict__ wg, const float* __restrict__ g, float* __restrict__ out,
                                int L, int G, int gin) {
    const int l = blockIdx.x, b = blockIdx.y;
    for (int row = threadIdx.x; row < G; row += blockDim.x) {
        const float* w = wg + ((size_t)l * G + row) * gin;
        float a = 0.f;
        for (int i = 0; i < gin; ++i) a = fmaf(w[i], g[(size_t)b * gin + i], a);
        out[((size_t)b * L + l) * G + row] = a;
    }
}

// stand-alone samplers over (B,O,T): the reference's mixture.py entry points
__global__ void wn_sample_kernel(const float* __restrict__ y, int B, int O, int T, const float* __restrict__ u1,
                                 const float* __restrict__ n2, float* __restrict__ out, int gauss) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * T) return;
    const int b = i / T, t = i % T;
    const float* yb = y + (size_t)b * O * T + t;
    float mean, ls;
    const int K = (O == 2) ? 1 : O / 3;
    if (K > 1 || (!gauss)) {
        float best = -INFINITY;
        int bi = 0;
        for (int k = 0; k < K; ++k) {
            const float gk = yb[(size_t)k * T] - logf(-logf(u1[((size_t)t * B + b) * K + k]));
            if (gk > best) {
                best = gk;
                bi = k;
            }
        }
        mean = yb[(size_t)(K + bi) * T];
        ls = yb[(size_t)(2 * K + bi) * T];
    } else if (O == 2) {
        mean = yb[0];
        ls = yb[(size_t)T];
    } else {
        mean = yb[(size_t)T];
        ls = yb[(size_t)2 * T];
    }
    const float v = n2[(size_t)t * B + b];
    float xv;
    if (!gauss) xv = __fadd_rn(mean, __fmul_rn(expf(ls), __fsub_rn(logf(v), logf(__fsub_rn(1.0f, v)))));
    else xv = __fadd_rn(__fmul_rn(v, expf(ls)), mean);
    out[i] = fminf(fmaxf(xv, -1.0f), 1.0f);
}

}  // namespace wn
