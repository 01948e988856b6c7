// bw_probe.cu -- HBM bandwidth ceilings for the access shapes the scan kernels use (development tool, not product).
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tools/bw_probe tools/bw_probe.cu
// Prints GB/s for: plain 16-byte streaming read, streaming copy, cp.async staged read (the k_decode_lcp shape),
// bulk-TMA (cp.async.bulk) staged read, bulk-TMA copy through shared memory, cudaMemcpy D2D, and the k_gather shape
// (2320 B every 10368 B) copied by a bulk-TMA ring, with 32-byte aligned stores, and register-staged by whole warps.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

__device__ __forceinline__ uint4 ldg_stream(const uint4 *p)
{
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void stg_stream(uint4 *p, const uint4 &v)
{
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

template <int U>
__global__ void k_read(const uint4 *__restrict__ src, size_t n, uint32_t *out)
{
    uint32_t acc = 0;
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride * U) {
        uint4 v[U];
#pragma unroll
        for (int j = 0; j < U; j++) v[j] = (i + j * stride < n) ? ldg_stream(src + i + j * stride) : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int j = 0; j < U; j++) acc += v[j].x ^ v[j].y ^ v[j].z ^ v[j].w;
    }
    if (acc == 0x12345678u) *out = acc;
}

template <int U>
__global__ void k_copy(const uint4 *__restrict__ src, uint4 *__restrict__ dst, size_t n)
{
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride * U) {
        uint4 v[U];
#pragma unroll
        for (int j = 0; j < U; j++)
            if (i + j * stride < n) v[j] = ldg_stream(src + i + j * stride);
#pragma unroll
        for (int j = 0; j < U; j++)
            if (i + j * stride < n) stg_stream(dst + i + j * stride, v[j]);
    }
}

// per-warp cp.async ring: each warp streams CH-chunk pieces, STAGES deep, and only touches one word per piece
template <int CH, int STAGES>
__global__ void k_cpasync(const uint4 *__restrict__ src, size_t n, uint32_t *out)
{
    extern __shared__ uint4 sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    uint4 *buf = sm + (size_t)warp * STAGES * CH;
    const size_t pieces = n / CH;
    const size_t stride = (size_t)gridDim.x * nw;
    size_t p = (size_t)blockIdx.x * nw + warp;
    uint32_t acc = 0;
    auto issue = [&](size_t piece, int st) {
        if (piece < pieces) {
            const uint4 *s = src + piece * CH;
            for (int c = lane; c < CH; c += 32) {
                uint32_t d = (uint32_t)__cvta_generic_to_shared(buf + st * CH + c);
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(s + c) : "memory");
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    for (int s = 0; s < STAGES - 1; s++) issue(p + s * stride, s);
    for (int it = 0; p < pieces; p += stride, it++) {
        issue(p + (STAGES - 1) * stride, (it + STAGES - 1) % STAGES);
        asm volatile("cp.async.wait_group %0;" ::"n"(STAGES - 1) : "memory");
        __syncwarp();
        acc += buf[(it % STAGES) * CH + lane].x;
        __syncwarp();
    }
    if (acc == 0x12345678u) *out = acc;
}

__device__ __forceinline__ void mbar_init(uint64_t *bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    asm volatile(
        "{\n .reg .pred p;\n WAIT_LOOP:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n @p bra DONE;\n bra WAIT_LOOP;\n DONE:\n}\n" ::"r"(
            (uint32_t)__cvta_generic_to_shared(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     (uint32_t)__cvta_generic_to_shared(dst)),
                 "l"(src), "r"(bytes), "r"((uint32_t)__cvta_generic_to_shared(bar))
                 : "memory");
}
__device__ __forceinline__ void bulk_s2g(void *dst, const void *src, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"((uint32_t)__cvta_generic_to_shared(src)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}

// warp-cooperative, register-staged copy of the gather shape: each warp moves KV pieces of CH chunks at a time (read at a
// stride of `sstride` chunks, written every `dstride` chunks), every 16-byte load issued before the first store, no
// shared memory
template <int CH, int KV>
__global__ void k_warp_gather(const uint4 *__restrict__ src, uint4 *__restrict__ dst, size_t pieces, size_t sstride,
                              size_t dstride)
{
    constexpr int PER = (CH + 31) / 32;
    const int lane = threadIdx.x & 31;
    const size_t nw = (size_t)gridDim.x * (blockDim.x >> 5);
    for (size_t p = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); p < pieces; p += nw * KV) {
        uint4 v[KV][PER];
#pragma unroll
        for (int k = 0; k < KV; k++)
#pragma unroll
            for (int j = 0; j < PER; j++) {
                const int c = lane + 32 * j;
                if (p + k * nw < pieces && c < CH) v[k][j] = ldg_stream(src + (p + k * nw) * sstride + c);
            }
#pragma unroll
        for (int k = 0; k < KV; k++)
#pragma unroll
            for (int j = 0; j < PER; j++) {
                const int c = lane + 32 * j;
                if (p + k * nw < pieces && c < CH) stg_stream(dst + (p + k * nw) * dstride + c, v[k][j]);
            }
    }
}

// per-warp bulk-TMA ring. COPY: also store every piece back to dst with a bulk store (every `dst_stride` chunks; 0: CH).
template <int CH, int STAGES, bool COPY>
__global__ void k_bulk(const uint4 *__restrict__ src, uint4 *__restrict__ dst, size_t n, uint32_t *out,
                       size_t src_stride, size_t dst_stride)
{
    extern __shared__ __align__(128) uint4 sm[];
    __shared__ uint64_t bars[16 * STAGES];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    uint4 *buf = sm + (size_t)warp * STAGES * CH;
    uint64_t *bar = bars + warp * STAGES;
    if (lane == 0)
        for (int s = 0; s < STAGES; s++) mbar_init(bar + s, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncwarp();
    const size_t sstep = src_stride ? src_stride : CH;  // source pieces every `sstep` chunks (gather shape)
    const size_t pieces = src_stride ? n / src_stride : n / CH;
    const size_t stride = (size_t)gridDim.x * nw;
    size_t p = (size_t)blockIdx.x * nw + warp;
    uint32_t acc = 0;
    constexpr int D = COPY ? STAGES - 2 : STAGES - 1;  // prefetch distance
    auto issue = [&](size_t piece, int it) {
        if (piece < pieces && lane == 0) {
            const int st = it % STAGES;
            if (COPY) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");  // buffer st was stored 2 its ago
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            mbar_expect_tx(bar + st, CH * 16);
            bulk_g2s(buf + st * CH, src + piece * sstep, CH * 16, bar + st);
        }
    };
    for (int s = 0; s < D; s++) issue(p + s * stride, s);
    for (int it = 0; p < pieces; p += stride, it++) {
        issue(p + D * stride, it + D);
        const int st = it % STAGES;
        mbar_wait(bar + st, (it / STAGES) & 1);
        if (COPY) {
            if (lane == 0) bulk_s2g(dst + p * (dst_stride ? dst_stride : CH), buf + st * CH, CH * 16);
        } else {
            acc += buf[st * CH + lane].x;
        }
        __syncwarp();
    }
    if (COPY && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    if (acc == 0x12345678u) *out = acc;
}

template <typename F>
static float timeit(F f, int reps = 5)
{
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    f();
    CK(cudaDeviceSynchronize());
    float best = 1e30f;
    for (int r = 0; r < reps; r++) {
        cudaEventRecord(a);
        f();
        cudaEventRecord(b);
        CK(cudaEventSynchronize(b));
        float ms;
        cudaEventElapsedTime(&ms, a, b);
        if (ms < best) best = ms;
    }
    return best;
}

int main()
{
    const size_t bytes = (size_t)1 << 30;  // 1 GiB source, 1 GiB destination: far larger than the 50 MB L2
    const size_t n = bytes / 16;
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    uint4 *src, *dst;
    uint32_t *out;
    CK(cudaMalloc(&src, bytes));
    CK(cudaMalloc(&dst, bytes));
    CK(cudaMalloc(&out, 4));
    CK(cudaMemset(src, 1, bytes));
    CK(cudaMemset(dst, 0, bytes));
    const double GB = bytes / 1e9;
    float ms;
    for (int g : {sms * 4, sms * 8, sms * 16}) {
        ms = timeit([&] { k_read<4><<<g, 256>>>(src, n, out); });
        printf("read  U=4 grid=%5d            : %8.1f GB/s\n", g, GB / (ms / 1e3));
        ms = timeit([&] { k_read<8><<<g, 256>>>(src, n, out); });
        printf("read  U=8 grid=%5d            : %8.1f GB/s\n", g, GB / (ms / 1e3));
    }
    for (int g : {sms * 4, sms * 8}) {
        ms = timeit([&] { k_copy<4><<<g, 256>>>(src, dst, n); });
        printf("copy  U=4 grid=%5d (r+w)      : %8.1f GB/s\n", g, 2 * GB / (ms / 1e3));
        ms = timeit([&] { k_copy<8><<<g, 256>>>(src, dst, n); });
        printf("copy  U=8 grid=%5d (r+w)      : %8.1f GB/s\n", g, 2 * GB / (ms / 1e3));
    }
    ms = timeit([&] { cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice); });
    printf("cudaMemcpy D2D (r+w)              : %8.1f GB/s\n", 2 * GB / (ms / 1e3));
    {
        constexpr int CH = 576;
        auto run = [&](auto kern, int warps, int stages, const char *name) {
            size_t smem = (size_t)warps * stages * CH * 16;
            CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            float t = timeit([&] { kern<<<sms, warps * 32, smem>>>(src, n, out); });
            printf("%-34s: %8.1f GB/s\n", name, GB / (t / 1e3));
        };
        run(k_cpasync<CH, 2>, 12, 2, "cp.async ring 12w x 2st x 9KB read");
        run(k_cpasync<CH, 2>, 8, 2, "cp.async ring  8w x 2st x 9KB read");
        run(k_cpasync<CH, 3>, 8, 3, "cp.async ring  8w x 3st x 9KB read");
    }
    {
        constexpr int CH = 576;
        auto run = [&](auto kern, int warps, int stages, bool copy, const char *name) {
            size_t smem = (size_t)warps * stages * CH * 16;
            CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            float t = timeit([&] { kern<<<sms, warps * 32, smem>>>(src, dst, n, out, (size_t)0, (size_t)0); });
            printf("%-34s: %8.1f GB/s\n", name, (copy ? 2 : 1) * GB / (t / 1e3));
        };
        run(k_bulk<CH, 2, false>, 12, 2, false, "bulk TMA ring 12w x 2st x 9KB read");
        run(k_bulk<CH, 3, false>, 8, 3, false, "bulk TMA ring  8w x 3st x 9KB read");
        run(k_bulk<CH, 4, true>, 6, 4, true, "bulk TMA copy  6w x 4st x 9KB r+w");
    }
    {
        constexpr int CH = 160;  // 2.5 KB pieces: one kv of the gather
        auto run = [&](auto kern, int warps, int stages, const char *name) {
            size_t smem = (size_t)warps * stages * CH * 16;
            CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            float t = timeit([&] { kern<<<sms, warps * 32, smem>>>(src, dst, n, out, (size_t)0, (size_t)0); });
            printf("%-34s: %8.1f GB/s\n", name, 2 * GB / (t / 1e3));
            t = timeit([&] { kern<<<sms * 2, warps * 32, smem>>>(src, dst, n, out, (size_t)0, (size_t)0); });
            printf("%-34s: %8.1f GB/s (2 CTA/SM)\n", name, 2 * GB / (t / 1e3));
        };
        run(k_bulk<CH, 4, true>, 8, 4, "bulk TMA copy  8w x 4st x 2.5KB");
        run(k_bulk<CH, 6, true>, 8, 6, "bulk TMA copy  8w x 6st x 2.5KB");
    }
    {
        // the gather shape: 2.3 KB pieces read at a 10 KB stride (one winner out of five records), written contiguously
        constexpr int CH = 145;
        size_t smem = (size_t)8 * 8 * CH * 16;
        auto kern = k_bulk<CH, 8, true>;
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const size_t sstride = 648;  // chunks between consecutive source pieces (10368 B)
        const size_t pieces = n / sstride;
        float t = timeit([&] { kern<<<sms, 8 * 32, smem>>>(src, dst, n, out, sstride, (size_t)0); });
        printf("bulk TMA gather-shaped copy 2320B every 10368B: %8.1f GB/s (r+w of the bytes moved)\n",
               2.0 * pieces * CH * 16 / 1e9 / (t / 1e3));
        // the same, written every 2336 B: every store starts on a 32-byte sector (what a sector-aligned layout would buy)
        t = timeit([&] { kern<<<sms, 8 * 32, smem>>>(src, dst, n, out, sstride, (size_t)146); });
        printf("bulk TMA gather-shaped, 32B-aligned stores      : %8.1f GB/s\n", 2.0 * pieces * CH * 16 / 1e9 / (t / 1e3));
        // the ring the gather runs today: 6 stages of 2320 B per warp, 8 warps, two CTAs per SM
        constexpr int ST6 = 6;
        auto k6 = k_bulk<CH, ST6, true>;
        const size_t smem6 = (size_t)8 * ST6 * CH * 16;
        CK(cudaFuncSetAttribute(k6, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem6));
        t = timeit([&] { k6<<<sms * 2, 8 * 32, smem6>>>(src, dst, n, out, sstride, (size_t)0); });
        printf("bulk TMA gather-shaped 8w x 6st, 2 CTA/SM       : %8.1f GB/s\n", 2.0 * pieces * CH * 16 / 1e9 / (t / 1e3));
        // register-staged, warp-cooperative
        for (int g : {sms * 4, sms * 8, sms * 16}) {
            t = timeit([&] { k_warp_gather<CH, 1><<<g, 256>>>(src, dst, pieces, sstride, CH); });
            printf("register-staged gather-shaped KV=1 grid=%5d : %8.1f GB/s\n", g, 2.0 * pieces * CH * 16 / 1e9 / (t / 1e3));
            t = timeit([&] { k_warp_gather<CH, 2><<<g, 256>>>(src, dst, pieces, sstride, CH); });
            printf("register-staged gather-shaped KV=2 grid=%5d : %8.1f GB/s\n", g, 2.0 * pieces * CH * 16 / 1e9 / (t / 1e3));
        }
    }
    printf("done\n");
    return 0;
}
