// wn_aux.cuh — the two steps either side of the synthesis kernel (SURVEY.md 8(f-1), 8(f-2)), hand-written:
//
//   * local-conditioning upsampler (reference upsample.py:29-85, called at wavenet.py:274-276):
//     conv_in (C x C x (2*cin_pad+1), no bias) over mel frames, then per scale s a nearest-neighbour
//     stretch by s and a 1 x (2s+1) smoothing filter (the same filter for every channel), writing the
//     sample-rate conditioning directly in the (B,T,C) layout the synthesis kernel reads;
//   * output decode (synthesis.py:66-84, evaluate.py:43-48,247-251, audio.py:57-58): inverse mu-law
//     (class index or companded scalar; nnmnkwii.preprocessing inv_mulaw / inv_mulaw_quantize),
//     inv_preemphasis (a serial one-pole IIR, scipy.signal.lfilter([1],[1,-coef]) in float32), division by
//     global_gain_scale, clip to [-1,1], (x*32767) truncated to int16.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include <algorithm>

namespace wnaux {

#define WNAUX_MAX_SCALES 8

struct UpsampleDesc {
    int n_scales;
    int scales[WNAUX_MAX_SCALES];
    int foff[WNAUX_MAX_SCALES];      // offset of filter j (2*s_j+1 taps) in `filters`
    float rscale[WNAUX_MAX_SCALES];  // (float)(1.0 / s_j): F.interpolate's nearest index is floor(dst * rscale)
    int indent;                      // samples trimmed at both ends (cin_pad * prod(scales), upsample.py:35,59-60)
};

// h[b][f][ch] = sum_{ci,k} w[ch][ci][k] * c[b][ci][f+k]    (nn.Conv1d, no padding, no bias; upsample.py:76,83)
__global__ void conv_in_kernel(const float* __restrict__ c, const float* __restrict__ w, float* __restrict__ h, int B, int C,
                               int F, int ks) {
    const int Fo = F - ks + 1;
    const long long n = (long long)B * Fo * C;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int ch = (int)(i % C), f = (int)((i / C) % Fo), b = (int)(i / ((long long)C * Fo));
        const float* wr = w + (size_t)ch * C * ks;
        const float* cb = c + (size_t)b * C * F + f;
        float a = 0.f;
        for (int ci = 0; ci < C; ++ci)
            for (int k = 0; k < ks; ++k) a = fmaf(wr[ci * ks + k], cb[(size_t)ci * F + k], a);
        h[i] = a;
    }
}
// (B,C,F) -> (B,F,C) when there is no conv_in (plain UpsampleNetwork)
__global__ void frames_to_fc_kernel(const float* __restrict__ c, float* __restrict__ h, int B, int C, int F) {
    const long long n = (long long)B * F * C;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int ch = (int)(i % C), f = (int)((i / C) % F), b = (int)(i / ((long long)C * F));
        h[i] = c[((size_t)b * C + ch) * F + f];
    }
}

// One block = one tile of TS output samples of one utterance.  The levels below the last one are evaluated for
// the index range the tile needs and kept in shared memory ([index][channel]); the last level goes straight to
// global memory in (B,T,C) layout.
//   level j:  a_j[u] = sum_{k=0}^{2s} w_j[k] * st[u + k - s],   st[v] = a_{j-1}[min(floor(v * rscale), n_{j-1}-1)] for
//   0 <= v < n_j, 0 outside (Conv2d padding (0, s), upsample.py:41-43; Stretch2d upsample.py:19-21)
// Windows (streaming): `h` holds rows [f_off, f_off+Fw) of level 0, whose full length is n0 (WNAUX_UNBOUNDED while more
// frames may follow), and output sample i is sample t_off + i of the whole utterance.  Every index, the zero padding
// and the clamp are those of the whole sequence, so a window equals the same samples of a one-shot upsample.
#define WNAUX_UNBOUNDED (1 << 30)
template <int TS>
__global__ void upsample_kernel(const float* __restrict__ h /* (B,Fw,C) */, const float* __restrict__ filters,
                                const __grid_constant__ UpsampleDesc d, int C, int Fw, int f_off, int n0, int t_off,
                                int T_out, float* __restrict__ out /* (B,T_out,C) */) {
    extern __shared__ float sm[];
    const int b = blockIdx.y, t0 = blockIdx.x * TS;
    const int J = d.n_scales;
    // length of every level and the index range this tile needs from it (block-uniform: one thread fills the table)
    __shared__ int n[WNAUX_MAX_SCALES + 1], lo[WNAUX_MAX_SCALES + 1], hi[WNAUX_MAX_SCALES + 1];
    if (threadIdx.x == 0) {
        n[0] = n0;
        for (int j = 1; j <= J; ++j) n[j] = n0 >= WNAUX_UNBOUNDED ? WNAUX_UNBOUNDED : n[j - 1] * d.scales[j - 1];
        lo[J] = t_off + t0 + d.indent;
        hi[J] = t_off + min(t0 + TS, T_out) - 1 + d.indent;
        for (int j = J; j >= 1; --j) {
            const int s = d.scales[j - 1];
            const int vlo = max(lo[j] - s, 0), vhi = min(hi[j] + s, n[j] - 1);
            lo[j - 1] = min((int)floorf((float)vlo * d.rscale[j - 1]), n[j - 1] - 1);
            hi[j - 1] = min((int)floorf((float)vhi * d.rscale[j - 1]), n[j - 1] - 1);
        }
    }
    __syncthreads();
    // level 0 window from global memory
    float* cur = sm;
    float* nxt = sm + (size_t)(TS / 2 + 8) * C;      // every scale >= 2: a lower level's window is <= TS/2 + 3 entries
    {
        const int len = hi[0] - lo[0] + 1;
        for (int i = threadIdx.x; i < len * C; i += blockDim.x)
            cur[i] = h[((size_t)b * Fw + (lo[0] - f_off)) * C + i];
    }
    __syncthreads();
    for (int j = 1; j <= J; ++j) {
        const int s = d.scales[j - 1];
        const float* w = filters + d.foff[j - 1];
        const float rs = d.rscale[j - 1];
        const int len = hi[j] - lo[j] + 1;
        const bool last = (j == J);
        for (int i = threadIdx.x; i < len * C; i += blockDim.x) {
            const int u = lo[j] + i / C, ch = i % C;
            float a = 0.f;
            for (int k = 0; k <= 2 * s; ++k) {
                const int v = u + k - s;
                if (v >= 0 && v < n[j]) {
                    const int src = min((int)floorf((float)v * rs), n[j - 1] - 1);
                    a = fmaf(w[k], cur[(size_t)(src - lo[j - 1]) * C + ch], a);
                }
            }
            if (last) out[((size_t)b * T_out + (u - d.indent - t_off)) * C + ch] = a;
            else nxt[i] = a;
        }
        __syncthreads();
        float* t = cur; cur = nxt; nxt = t;
    }
}

// Host mirror of the table upsample_kernel builds: rows [*r_lo, *r_hi] of level 0 that output samples [t_lo, t_hi)
// read when level 0 has n0 rows (WNAUX_UNBOUNDED: no right edge).  *inside: no index of that cone reaches past the
// first n_in rows of level 0 at any level (neither the zero padding nor the clamp of a sequence that ends there), so
// the samples are the same for every sequence that starts with those n_in rows.
inline void cone_rows(const UpsampleDesc& d, int n0, int n_in, int t_lo, int t_hi, int* r_lo, int* r_hi, bool* inside) {
    const int J = d.n_scales;
    int n[WNAUX_MAX_SCALES + 1], m[WNAUX_MAX_SCALES + 1];
    n[0] = n0;
    m[0] = n_in;
    for (int j = 1; j <= J; ++j) {
        n[j] = n0 >= WNAUX_UNBOUNDED ? WNAUX_UNBOUNDED : n[j - 1] * d.scales[j - 1];
        m[j] = m[j - 1] * d.scales[j - 1];
    }
    int lo = t_lo + d.indent, hi = t_hi - 1 + d.indent;
    bool ok = hi < m[J];
    for (int j = J; j >= 1; --j) {
        const int s = d.scales[j - 1];
        const int vlo = std::max(lo - s, 0), vhi = std::min(hi + s, n[j] - 1);
        ok = ok && hi + s < m[j];
        lo = std::min((int)floorf((float)vlo * d.rscale[j - 1]), n[j - 1] - 1);
        hi = std::min((int)floorf((float)vhi * d.rscale[j - 1]), n[j - 1] - 1);
        ok = ok && (int)floorf((float)vhi * d.rscale[j - 1]) < m[j - 1];
    }
    *r_lo = lo;
    *r_hi = hi;
    *inside = ok;
}

// ---- decode -------------------------------------------------------------------------------------------------
enum { DEC_RAW = 0, DEC_MULAW = 1, DEC_MULAW_QUANTIZE = 2 };

// One block per utterance; chunks of CH samples: pointwise inverse companding by all threads, the one-pole
// recursion by thread 0 (y[n] = x[n] + coef*y[n-1], each operation rounded to float32 exactly like
// scipy.signal.lfilter's float32 loop), then gain / clip / int16 by all threads.
// `carry` (B, or NULL for a zero start): coef * y[-1] on entry, coef * y[T-1] on exit, so that consecutive chunks of an
// utterance decode to the bits one call over the whole utterance gives.
template <int CH>
__global__ void decode_kernel(const float* __restrict__ y_scalar, const int* __restrict__ y_index, int T, const int* __restrict__ lengths,
                              int kind, float mu, float coef, float gain, float* __restrict__ out_float,
                              short* __restrict__ out_pcm, float* __restrict__ carry = nullptr) {
    __shared__ float chunk[CH];
    __shared__ float carry_s;
    const int b = blockIdx.x;
    const int len = lengths ? min(lengths[b], T) : T;
    if (threadIdx.x == 0) carry_s = carry ? carry[b] : 0.f;
    __syncthreads();
    for (int base = 0; base < T; base += CH) {
        const int nthis = min(CH, T - base);
        for (int i = threadIdx.x; i < nthis; i += blockDim.x) {
            float v;
            if (kind == DEC_MULAW_QUANTIZE) {
                // nnmnkwii inv_mulaw_quantize: y = 2*float(idx)/mu - 1, then inv_mulaw
                v = __fsub_rn(__fdiv_rn(__fmul_rn(2.0f, (float)y_index[(size_t)b * T + base + i]), mu), 1.0f);
            } else {
                v = y_scalar[(size_t)b * T + base + i];
            }
            if (kind != DEC_RAW) {
                // nnmnkwii inv_mulaw: sign(y) * (1/mu) * ((1+mu)^|y| - 1)
                const float sgn = (v > 0.f) ? 1.f : ((v < 0.f) ? -1.f : 0.f);
                v = __fmul_rn(__fmul_rn(sgn, __fdiv_rn(1.0f, mu)), __fsub_rn(powf(__fadd_rn(1.0f, mu), fabsf(v)), 1.0f));
            }
            chunk[i] = v;
        }
        __syncthreads();
        if (coef != 0.f && threadIdx.x == 0) {
            float z = carry_s;                       // = coef * y[n-1]
            for (int i = 0; i < nthis; ++i) {
                const float yv = __fadd_rn(z, chunk[i]);
                chunk[i] = yv;
                z = __fmul_rn(coef, yv);
            }
            carry_s = z;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < nthis; i += blockDim.x) {
            float v = chunk[i];
            if (gain > 0.f) v = __fdiv_rn(v, gain);                       // synthesis.py:80-82
            const size_t o = (size_t)b * T + base + i;
            const bool inside = base + i < len;
            if (out_float) out_float[o] = inside ? v : 0.f;
            if (out_pcm) {
                const float cl = fminf(fmaxf(v, -1.0f), 1.0f);            // evaluate.py:247
                out_pcm[o] = inside ? (short)(int)__fmul_rn(cl, 32767.0f) : (short)0;   // evaluate.py:43-48
            }
        }
        __syncthreads();
    }
    if (carry && threadIdx.x == 0) carry[b] = carry_s;
}

}  // namespace wnaux
