// wn_dense.cuh — the teacher-forced batch forward (reference WaveNet.forward, wavenet.py:177-213) and the per-sample
// training criterion (mixture.py:26-106, :161-218; train.py:346-405), hand-written for sm_90a.
//
// Under teacher forcing every time step is independent, so a layer is two dense GEMMs over the B*T columns:
//   gate     Z = [W_conv | W_c] (G x kw*R+C) . [X_taps ; c^T]         epilogue Y = tanh(a + ..) * sigmoid(b + ..)  (B,G/2,T)
//   out/skip   [W_out ; W_skip] (R+S x G/2) . Y                       epilogue X <- (acc + out_b + X) * sqrt(1/2), skip (+)=
// and the head is two more (relu(skip * sqrt(1/L)) in the operand load, relu in the first epilogue).  Row k*R + r of
// X_taps is X[r, t - (kw-1-k)*d], zero for a negative time (the causal padding of modules.py:53-68).  Activations are
// channel-major per utterance, (B, ch, T), so that N is time and the operand loads along N are contiguous.
//
// Precision: 3xTF32 on mma.sync m16n8k8.  Each fp32 operand x is split into big = tf32(x) and small = tf32(x - big),
// and the product is accumulated in fp32 as small*big + big*small + big*big: what the dropped small*small term and the
// rounding of small cost is ~2^-22 relative per product, the same order as fp32 FMA, so the fp32 engine's parity bounds
// hold.  Plain TF32 (2^-11) would not.  (TF32 wgmma wants both operands K-major; the activation operand here is
// N-major, which is why this is mma.sync.)
//
// A column tile never crosses utterances and there is no split-K and no atomic: every output is one thread's fixed
// sequence of operations, so results are deterministic and row b of a batch equals the utterance computed alone.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

namespace wnd {

constexpr int BM = 64, BN = 128, BK = 16, STAGES = 3, NTHREADS = 256;
constexpr int AS = BK + 4;      // A tile row stride (floats): fragment loads hit 32 distinct banks
constexpr int BS = BN + 8;      // B tile row stride
constexpr int CS = BN + 4;      // epilogue staging row stride
constexpr int A_STAGE = BM * AS, B_STAGE = BK * BS;
constexpr int SMEM_FLOATS = STAGES * (A_STAGE + B_STAGE);   // 41 472 bytes: static shared memory, no opt-in
static_assert(BM * CS <= SMEM_FLOATS, "epilogue staging must fit in the pipeline buffers");

enum { B_PLAIN = 0, B_GATE = 1 };                                         // how the K x N operand is gathered
enum { EPI_GATE = 0, EPI_RESSKIP = 1, EPI_RELU_BIAS = 2, EPI_BIAS = 3 };  // what the epilogue does

struct DenseGemm {
    const float* A;            // M x K row-major weights (for EPI_GATE: G rows, tile rows paired i / i + G/2)
    int M, K, T;
    const float* Bsrc;         // B_PLAIN: (B, K, T)
    const float* X;            // B_GATE: residual input (B, R, T)
    const float* cT;           // B_GATE: local conditioning (B, Cc, T) or NULL
    int R, kw, dil, Cc, kwR;   // B_GATE: K = kw*R + Cc
    float bscale;              // operand transform relu(v * bscale) when brelu
    int brelu;
    const float* bias;         // per output row
    const float* gbias;        // EPI_GATE: W_g . g of utterance b at gbias[b * gstride + row], or NULL
    long long gstride;
    int G2;                    // EPI_GATE: gate half
    float* out;                // EPI_GATE: Y (B,G2,T); EPI_RESSKIP: X (B,R,T) in place; else (B,M,T)
    float* out2;               // EPI_RESSKIP: skip sum (B, M-R, T)
    int first;                 // EPI_RESSKIP: the first layer writes the skip sum instead of adding to it
};

__device__ __forceinline__ void cp4(float* dst, const float* src, bool valid) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(d), "l"(src), "r"(valid ? 4 : 0));
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ void split_tf32(float x, uint32_t& big, uint32_t& small) {
    uint32_t hi, lo;
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(hi) : "f"(x));
    const float rest = x - __uint_as_float(hi);
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(lo) : "f"(rest));
    big = hi;
    small = lo;
}

__device__ __forceinline__ void mma_tf32(float* c, const uint32_t* a, const uint32_t* b) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// One block = a BM x BN tile of one utterance (blockIdx.z); 8 warps of 32 x 32; a 3-stage cp.async pipeline of
// 4-byte copies (a dilation shift of 1..3 floats breaks 16-byte alignment, and out-of-range elements -- the causal
// padding, the ragged edges of M, K and T -- are zero-filled by a source size of 0).
template <int BMODE, int EPI>
__global__ void __launch_bounds__(NTHREADS) dense_gemm_kernel(const __grid_constant__ DenseGemm p) {
    __shared__ __align__(16) float sm[SMEM_FLOATS];
    float* As = sm;
    float* Bs = sm + STAGES * A_STAGE;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, tq = lane & 3;
    const int wm = warp & 1, wn = warp >> 1;
    const int n0 = blockIdx.x * BN, mt = blockIdx.y, b = blockIdx.z;
    const int T = p.T, K = p.K;
    const int nk = (K + BK - 1) / BK;

    // this thread's A rows (fixed over k): tile rows (tid>>4) + 16 i, column tid & 15
    const int akk = tid & 15;
    const float* arow[4];
    bool aok[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int lr = (tid >> 4) + 16 * i;
        int row;
        bool ok;
        if (EPI == EPI_GATE) {          // rows [0, BM/2) of the tile are gate rows j, rows [BM/2, BM) are rows G/2 + j
            const int j = mt * (BM / 2) + (lr < BM / 2 ? lr : lr - BM / 2);
            ok = j < p.G2;
            row = lr < BM / 2 ? j : p.G2 + j;
        } else {
            row = mt * BM + lr;
            ok = row < p.M;
        }
        arow[i] = p.A + (size_t)(ok ? row : 0) * K;
        aok[i] = ok;
    }
    // this thread's B column (fixed): tid & 127, rows (tid>>7) + 2 i
    const int bn = tid & (BN - 1);
    const int t = n0 + bn;
    const bool tok = t < T;

    auto load_tile = [&](int stage, int kt) {
        const int k0 = kt * BK;
        float* as = As + stage * A_STAGE;
        float* bs = Bs + stage * B_STAGE;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int lr = (tid >> 4) + 16 * i, k = k0 + akk;
            const bool ok = aok[i] && k < K;
            cp4(as + lr * AS + akk, ok ? arow[i] + k : p.A, ok);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int kk = (tid >> 7) + 2 * i, k = k0 + kk;
            const float* src = p.A;
            bool ok = false;
            if (BMODE == B_PLAIN) {
                ok = tok && k < K;
                if (ok) src = p.Bsrc + ((size_t)b * K + k) * T + t;
            } else if (k < p.kwR) {
                const int tap = k / p.R, r = k - tap * p.R;
                const int ts = t - (p.kw - 1 - tap) * p.dil;
                ok = tok && ts >= 0;
                if (ok) src = p.X + ((size_t)b * p.R + r) * T + ts;
            } else if (k < K) {
                ok = tok;
                if (ok) src = p.cT + ((size_t)b * p.Cc + (k - p.kwR)) * T + t;
            }
            cp4(bs + kk * BS + bn, src, ok);
        }
    };

    float acc[2][4][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < nk) load_tile(s, s);
        cp_commit();
    }
    for (int kt = 0; kt < nk; ++kt) {
        cp_wait<STAGES - 2>();
        __syncthreads();
        const float* as = As + (kt % STAGES) * A_STAGE;
        const float* bs = Bs + (kt % STAGES) * B_STAGE;
#pragma unroll
        for (int ks = 0; ks < BK; ks += 8) {
            uint32_t ab[2][4], asl[2][4];
#pragma unroll
            for (int mf = 0; mf < 2; ++mf) {
                const float* ap = as + (wm * 32 + mf * 16 + g) * AS + ks + tq;
                split_tf32(ap[0], ab[mf][0], asl[mf][0]);
                split_tf32(ap[8 * AS], ab[mf][1], asl[mf][1]);
                split_tf32(ap[4], ab[mf][2], asl[mf][2]);
                split_tf32(ap[8 * AS + 4], ab[mf][3], asl[mf][3]);
            }
            uint32_t bb[4][2], bsl[4][2];
#pragma unroll
            for (int nf = 0; nf < 4; ++nf) {
                const float* bp = bs + (ks + tq) * BS + wn * 32 + nf * 8 + g;
                float v0 = bp[0], v1 = bp[4 * BS];
                if (p.brelu) {
                    v0 = fmaxf(v0 * p.bscale, 0.f);
                    v1 = fmaxf(v1 * p.bscale, 0.f);
                }
                split_tf32(v0, bb[nf][0], bsl[nf][0]);
                split_tf32(v1, bb[nf][1], bsl[nf][1]);
            }
#pragma unroll
            for (int mf = 0; mf < 2; ++mf)
#pragma unroll
                for (int nf = 0; nf < 4; ++nf) {
                    mma_tf32(acc[mf][nf], asl[mf], bb[nf]);
                    mma_tf32(acc[mf][nf], ab[mf], bsl[nf]);
                    mma_tf32(acc[mf][nf], ab[mf], bb[nf]);
                }
        }
        const int nxt = kt + STAGES - 1;
        if (nxt < nk) load_tile(nxt % STAGES, nxt);
        cp_commit();
    }
    cp_wait<0>();
    __syncthreads();

    // stage the accumulator tile in shared memory, then finish it with the threads laid along N (coalesced)
    float* Cs = sm;
#pragma unroll
    for (int mf = 0; mf < 2; ++mf)
#pragma unroll
        for (int nf = 0; nf < 4; ++nf) {
            const int r = wm * 32 + mf * 16 + g, c = wn * 32 + nf * 8 + 2 * tq;
            Cs[r * CS + c] = acc[mf][nf][0];
            Cs[r * CS + c + 1] = acc[mf][nf][1];
            Cs[(r + 8) * CS + c] = acc[mf][nf][2];
            Cs[(r + 8) * CS + c + 1] = acc[mf][nf][3];
        }
    __syncthreads();
    constexpr int ROWS = EPI == EPI_GATE ? BM / 2 : BM;
    for (int e = tid; e < ROWS * BN; e += NTHREADS) {
        const int lr = e / BN, n = e % BN, tt = n0 + n;
        if (tt >= T) continue;
        const float v = Cs[lr * CS + n];
        if (EPI == EPI_GATE) {                                   // modules.py:138-154
            const int j = mt * (BM / 2) + lr;
            if (j >= p.G2) continue;
            float za = v + p.bias[j], zb = Cs[(lr + BM / 2) * CS + n] + p.bias[p.G2 + j];
            if (p.gbias) {
                const float* gb = p.gbias + (size_t)b * p.gstride;
                za += gb[j];
                zb += gb[p.G2 + j];
            }
            p.out[((size_t)b * p.G2 + j) * T + tt] = tanhf(za) * (1.f / (1.f + expf(-zb)));
        } else if (EPI == EPI_RESSKIP) {                         // modules.py:156-163, wavenet.py:203-206
            const int row = mt * BM + lr;
            if (row >= p.M) continue;
            const float z = v + p.bias[row];
            if (row < p.R) {
                float* xp = p.out + ((size_t)b * p.R + row) * T + tt;
                *xp = (z + *xp) * 0.70710678118654752f;
            } else {
                const int S = p.M - p.R;
                float* sp = p.out2 + ((size_t)b * S + (row - p.R)) * T + tt;
                *sp = p.first ? z : *sp + z;
            }
        } else {                                                 // wavenet.py:207-210
            const int row = mt * BM + lr;
            if (row >= p.M) continue;
            float z = v + p.bias[row];
            if (EPI == EPI_RELU_BIAS) z = fmaxf(z, 0.f);
            p.out[((size_t)b * p.M + row) * T + tt] = z;
        }
    }
}

// grid: column tiles of one utterance on x (up to 2^31 - 1), row tiles on y, utterances on z
template <int BMODE, int EPI>
inline cudaError_t launch_dense_gemm(const DenseGemm& p, int B, cudaStream_t st) {
    const int rows = EPI == EPI_GATE ? p.G2 : p.M, per = EPI == EPI_GATE ? BM / 2 : BM;
    const dim3 grid((unsigned)((p.T + BN - 1) / BN), (unsigned)((rows + per - 1) / per), (unsigned)B);
    dense_gemm_kernel<BMODE, EPI><<<grid, NTHREADS, 0, st>>>(p);
    return cudaGetLastError();
}

// (B, T, C) -> (B, C, T): the conditioning (and a dense one-hot input) in the channel-major layout of the GEMMs
__global__ void transpose_tc_kernel(const float* __restrict__ in, float* __restrict__ out, int T, int C) {
    __shared__ float tile[32][33];
    const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32, b = blockIdx.z;
    const float* src = in + (size_t)b * T * C;
    float* dst = out + (size_t)b * C * T;
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int tt = t0 + i, c = c0 + threadIdx.x;
        if (tt < T && c < C) tile[i][threadIdx.x] = src[(size_t)tt * C + c];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int c = c0 + i, tt = t0 + threadIdx.x;
        if (tt < T && c < C) dst[(size_t)c * T + tt] = tile[threadIdx.x][i];
    }
}

// First 1x1 conv (wavenet.py:196) -> X (B,R,T).  fw is the handle's first-conv image: (R) for scalar input, [O][R]
// for one-hot input.  A class id is a column gather; a dense one-hot row (transposed to (B,O,T)) is an fp32 FMA chain
// from zero, so an exactly one-hot row gives the gathered value bit for bit.  A class id outside [0,O) gives NaN.
__global__ void first_conv_kernel(const float* __restrict__ xs, const int* __restrict__ xi, const float* __restrict__ xdT,
                                  const float* __restrict__ fw, const float* __restrict__ fb, float* __restrict__ X, int B,
                                  int R, int O, int T) {
    const long long n = (long long)B * R * T;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int tt = (int)(i % T), r = (int)((i / T) % R);
        const long long b = i / ((long long)R * T);
        float v;
        if (xs) {
            v = fmaf(fw[r], xs[b * T + tt], fb[r]);
        } else if (xi) {
            const int k = xi[b * T + tt];
            v = (k >= 0 && k < O) ? fw[(size_t)k * R + r] + fb[r] : __int_as_float(0x7fc00000);
        } else {
            float a = 0.f;
            for (int o = 0; o < O; ++o) a = fmaf(fw[(size_t)o * R + r], xdT[((size_t)b * O + o) * T + tt], a);
            v = a + fb[r];
        }
        X[i] = v;
    }
}

// softmax over the channel axis of (B,O,T), in place (wavenet.py:213)
__global__ void col_softmax_kernel(float* __restrict__ y, int B, int O, int T) {
    const long long n = (long long)B * T;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / T;
        float* col = y + (size_t)b * O * T + (i - b * T);
        float m = -INFINITY;
        for (int o = 0; o < O; ++o) m = fmaxf(m, col[(size_t)o * T]);
        float s = 0.f;
        for (int o = 0; o < O; ++o) s += expf(col[(size_t)o * T] - m);
        for (int o = 0; o < O; ++o) col[(size_t)o * T] = expf(col[(size_t)o * T] - m) / s;
    }
}

// ---- per-sample negative log-likelihood (the reference's losses with reduce=False) --------------------------------
enum { NLL_MOL = 0, NLL_GAUSS = 1, NLL_SOFTMAX = 2 };

__device__ __forceinline__ float softplus_t(float x) { return x > 20.f ? x : log1pf(expf(x)); }   // F.softplus
__device__ __forceinline__ float sigmoid_t(float x) { return 1.f / (1.f + expf(-x)); }

struct NllArgs {
    const float* y;        // (B,O,T)
    const float* yt;       // (B,T) targets in [-1,1]  (MoL, Gaussian)
    const int* ct;         // (B,T) classes            (softmax)
    float* out;            // (B,T)
    int head, B, O, T;
    float log_scale_min;
    float half_bin;        // 1 / (num_classes - 1)
    float log_half_nc;     // log((num_classes - 1) / 2)
};

// log-probability of component k before the mixture weights: mixture.py:53-99 (MoL) or :196-204 (Gaussian)
__device__ __forceinline__ float component_lp(const NllArgs& a, const float* col, long long T, int K, int k, float yv) {
    if (a.head == NLL_MOL) {
        const float mean = col[(K + k) * T];
        const float lsc = fmaxf(col[(2 * K + k) * T], a.log_scale_min);
        const float centered = yv - mean;
        const float inv_stdv = expf(-lsc);
        const float plus_in = inv_stdv * (centered + a.half_bin);
        const float cdf_plus = sigmoid_t(plus_in);
        const float min_in = inv_stdv * (centered - a.half_bin);
        const float cdf_min = sigmoid_t(min_in);
        const float log_cdf_plus = plus_in - softplus_t(plus_in);
        const float log_one_minus_cdf_min = -softplus_t(min_in);
        const float cdf_delta = cdf_plus - cdf_min;
        const float mid_in = inv_stdv * centered;
        const float log_pdf_mid = mid_in - lsc - 2.f * softplus_t(mid_in);
        const float inner_inner = cdf_delta > 1e-5f ? logf(fmaxf(cdf_delta, 1e-12f)) : log_pdf_mid - a.log_half_nc;
        const float inner = yv > 0.999f ? log_one_minus_cdf_min : inner_inner;
        return yv < -0.999f ? log_cdf_plus : inner;
    }
    // Normal(0, exp(log_scale)).log_prob(y - mean), torch/distributions/normal.py
    const int mi = a.O == 2 ? 0 : K + k, li = a.O == 2 ? 1 : 2 * K + k;
    const float lsc = fmaxf(col[li * T], a.log_scale_min);
    const float centered = yv - col[mi * T];
    const float scale = expf(lsc);
    const float var = scale * scale;
    return -(centered * centered) / (2.f * var) - logf(scale) - 0.91893853320467274f;
}

__global__ void nll_kernel(const __grid_constant__ NllArgs a) {
    const long long n = (long long)a.B * a.T, T = a.T;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / T;
        const float* col = a.y + (size_t)b * a.O * T + (i - b * T);
        if (a.head == NLL_SOFTMAX) {                        // nn.CrossEntropyLoss(reduction='none'), train.py:346-362
            const int k = a.ct[i];
            if (k < 0 || k >= a.O) {
                a.out[i] = __int_as_float(0x7fc00000);
                continue;
            }
            float m = -INFINITY;
            for (int o = 0; o < a.O; ++o) m = fmaxf(m, col[o * T]);
            float s = 0.f;
            for (int o = 0; o < a.O; ++o) s += expf(col[o * T] - m);
            a.out[i] = -((col[k * T] - m) - logf(s));
            continue;
        }
        const float yv = a.yt[i];
        const int K = a.O == 2 ? 1 : a.O / 3;
        if (K == 1 && a.head == NLL_GAUSS) {                 // mixture.py:206-216: no mixture weights
            a.out[i] = -component_lp(a, col, T, 1, 0, yv);
            continue;
        }
        // log_softmax of the mixture logits (mixture.py:101, :207)
        float lm = -INFINITY;
        for (int k = 0; k < K; ++k) lm = fmaxf(lm, col[k * T]);
        float ls = 0.f;
        for (int k = 0; k < K; ++k) ls += expf(col[k * T] - lm);
        const float lnorm = logf(ls);
        // log_sum_exp over the components (mixture.py:17-23): max first, then the sum
        float m = -INFINITY;
        for (int k = 0; k < K; ++k) m = fmaxf(m, component_lp(a, col, T, K, k, yv) + ((col[k * T] - lm) - lnorm));
        float s = 0.f;
        for (int k = 0; k < K; ++k) s += expf(component_lp(a, col, T, K, k, yv) + ((col[k * T] - lm) - lnorm) - m);
        a.out[i] = -(m + logf(s));
    }
}

}  // namespace wnd
