// xbench_stream.cu — skeleton of the synthesis kernel's weight stream (no model, no exchange).
// P blocks; each streams its own slice of a packed image laid out like the packer's ([P][blob image], 23 layer
// blobs of 36,912 bytes and one tail blob of 28,720 bytes per step: config 2 at P = 128, 112.3 MB per step) into
// shared memory with cp.async.bulk through a 4-slot mbarrier ring.  One consumer warp takes each blob, holds it for
// a fixed number of cycles ("work") and releases the slot.  The producer optionally asks L2 to fetch the blob D
// ahead (cp.async.bulk.prefetch.L2) before it copies the current one, and optionally marks the shared-memory copy
// evict-first in L2.  Reports the consumer's wait per blob, the time per step and the bytes per second achieved.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o xbench_stream scripts/xbench_stream.cu
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cuda_runtime.h>

#define NSTREAM 24              // streamed blobs per step (blob 0 of 25 stays resident in the real kernel)
#define LAYER_BYTES 36912u
#define TAIL_BYTES 28720u
#define NRING 4
#define SLOT_BYTES 36992u       // LAYER_BYTES rounded up to 128

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t n) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(n) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* b) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* b, uint32_t par) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(b)), "r"(par) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar, bool evict_first,
                                         uint64_t pol) {
    if (evict_first)
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                     ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol) : "memory");
    else
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void prefetch_l2(const void* src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint32_t blob_bytes(int j) { return j < NSTREAM - 1 ? LAYER_BYTES : TAIL_BYTES; }

__device__ int g_abort = 0;
// a wait that takes longer than this (or another thread's abort) ends the run instead of hanging it
__device__ __forceinline__ bool timed_out(long long t0) {
    if (clock64() - t0 > 400000000LL || *((volatile int*)&g_abort)) { g_abort = 1; return true; }
    return false;
}

__global__ void __launch_bounds__(64, 1)
stream(const char* image, long long cta_bytes, int steps, int dist, int evict_first, int work, long long* out) {
    extern __shared__ __align__(128) unsigned char smem[];
    uint64_t* full = (uint64_t*)smem;
    uint64_t* empty = full + NRING;
    unsigned char* slots = smem + 128;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const char* base = image + (size_t)blockIdx.x * cta_bytes;
    if (threadIdx.x == 0) {
        for (int s = 0; s < NRING; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int total = steps * NSTREAM;
    if (warp == 0) {                                            // producer
        if (lane != 0) return;
        uint64_t pol = 0;
        asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
        for (int k = 0; k < dist && k < total; ++k) prefetch_l2(base + (size_t)(k % NSTREAM) * LAYER_BYTES, blob_bytes(k % NSTREAM));
        for (int js = 0; js < total; ++js) {
            const int s = js % NRING, u = js / NRING;
            if (u > 0) {
                const long long tw = clock64();
                bool ok = true;
                while (!mbar_try_wait(&empty[s], (u - 1) & 1)) if (timed_out(tw)) { ok = false; break; }
                if (!ok) return;
            }
            if (dist > 0 && js + dist < total) {
                const int j = (js + dist) % NSTREAM;
                prefetch_l2(base + (size_t)j * LAYER_BYTES, blob_bytes(j));
            }
            const int j = js % NSTREAM;
            mbar_expect_tx(&full[s], blob_bytes(j));
            bulk_g2s(slots + (size_t)s * SLOT_BYTES, base + (size_t)j * LAYER_BYTES, blob_bytes(j), &full[s], evict_first, pol);
        }
    } else {                                                    // consumer
        long long wait = 0;
        uint32_t acc = 0;
        const long long t0 = clock64();
        for (int js = 0; js < total; ++js) {
            const int s = js % NRING, u = js / NRING;
            const long long tw = clock64();
            bool ok = true;
            while (!mbar_try_wait(&full[s], u & 1)) if (timed_out(tw)) { ok = false; break; }
            if (!ok) break;
            wait += clock64() - tw;
            acc += ((const uint32_t*)(slots + (size_t)s * SLOT_BYTES))[lane];    // touch the blob
            const long long tb = clock64();
            while (clock64() - tb < work) {}
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
        }
        if (lane == 0) {
            out[blockIdx.x * 2] = wait;
            out[blockIdx.x * 2 + 1] = clock64() - t0 + (acc == 0x9e3779b9u);
        }
    }
}

int main(int argc, char** argv) {
    setvbuf(stdout, NULL, _IONBF, 0);
    const int P = argc > 1 ? atoi(argv[1]) : 128, steps = argc > 2 ? atoi(argv[2]) : 200;
    const long long cta_bytes = (long long)(NSTREAM - 1) * LAYER_BYTES + TAIL_BYTES;
    const double step_bytes = (double)cta_bytes * P;
    char* image; long long* out;
    cudaMalloc(&image, (size_t)cta_bytes * P);
    cudaMalloc(&out, (size_t)P * 2 * sizeof(long long));
    cudaMemset(image, 1, (size_t)cta_bytes * P);
    const int smem = 128 + NRING * SLOT_BYTES;
    cudaFuncSetAttribute(stream, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
    printf("%s, %d SMs, L2 %d MB; P=%d blocks, %.1f MB streamed per step, %d-slot ring, %d steps per run\n", prop.name,
           prop.multiProcessorCount, prop.l2CacheSize >> 20, P, step_bytes / 1e6, NRING, steps);
    long long* h = (long long*)malloc((size_t)P * 2 * sizeof(long long));
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int work : {0, 3000})
        for (int ef = 0; ef < 2; ++ef)
            for (int dist = 0; dist <= 8; ++dist) {
                float best = 1e30f, ms = 0.f;
                double wait = 0.0;
                for (int rep = 0; rep < 3; ++rep) {                 // first run warms up; best of the other two
                    cudaEventRecord(e0);
                    stream<<<P, 64, smem>>>(image, cta_bytes, steps, dist, ef, work, out);
                    cudaEventRecord(e1);
                    cudaError_t e = cudaEventSynchronize(e1);
                    if (e != cudaSuccess || cudaGetLastError() != cudaSuccess) { printf("launch failed: %s\n", cudaGetErrorString(e)); return 1; }
                    int ab = 0; cudaMemcpyFromSymbol(&ab, g_abort, sizeof(int));
                    if (ab) { printf("WATCHDOG fired: work=%d evict_first=%d D=%d\n", work, ef, dist); return 1; }
                    cudaEventElapsedTime(&ms, e0, e1);
                    if (rep > 0 && ms < best) {
                        best = ms;
                        cudaMemcpy(h, out, (size_t)P * 2 * sizeof(long long), cudaMemcpyDeviceToHost);
                        wait = 0.0;
                        for (int p = 0; p < P; ++p) wait += (double)h[2 * p];
                        wait /= (double)P * steps * NSTREAM;
                    }
                }
                printf("work %4d cycles/blob  evict_first %d  D=%d : %7.2f us/step  %6.0f GB/s  wait %6.0f cycles/blob\n", work,
                       ef, dist, best * 1e3 / steps, step_bytes * steps / (best * 1e-3) / 1e9, wait);
            }
    return 0;
}
