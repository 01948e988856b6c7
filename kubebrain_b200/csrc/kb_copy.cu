// kb_copy.cu -- the answer every reader shares: the kb_result lifecycle, an answer's buffers and per-kv view arrays, and
// the copy of its kvs into the response arena, behind a job table (kb_batch.cu, kb_page.cu):
//   k_gather_jobs -> k_gather    padded [internal key][value] pairs
//   k_wire_jobs -> k_wire_copy   etcd protobuf elements (kb_wire.cuh)
// The job kernels run on the lane stream, the copy on the copy stream (range batches and pages) or on the lane stream
// (point reads).  The host frames the elements with kb_wire_range_head / _tail and kb_wire_watch_head.
#include <algorithm>

#include "kb_scan.cuh"
#include "kb_wire.cuh"

namespace {

// ------------------------------------------------------------------------------------------------
// k_gather: one warp per emitted kv; key (internal key, padded) then value (padded), 16-byte vector copies
// ------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(256)
k_gather_jobs(StoreDev st, const ReqDev *__restrict__ reqs, uint32_t nreq, const uint64_t *__restrict__ job_first,
              const uint64_t *__restrict__ arena_base, const uint32_t *__restrict__ sel,
              const uint64_t *__restrict__ slot, GatherJob *__restrict__ jobs, GatherOut out)
{
    const uint64_t n_kvs = job_first[nreq];  // written by k_req_finalize
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n_kvs; k += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = nreq;  // request of kv k: last q with job_first[q] <= k
    while (hi - lo > 1) {
        uint32_t mid = (lo + hi) >> 1;
        if (job_first[mid] <= k) lo = mid; else hi = mid;
    }
    const uint32_t q = lo;
    const uint64_t s = reqs[q].sel_base + (k - job_first[q]);
    const uint32_t rec = sel[s];
    const uint64_t dst_byte = arena_base[q] + slot[s];
    const uint32_t kl = st.klen[rec], vl = st.vlen[rec];
    GatherJob j;
    j.dst16 = dst_byte >> 4;
    j.vsrc16 = st.voff16[rec];
    j.ksrc16 = st.koff16[rec];
    j.nk = (kl + 15) >> 4;
    j.nv = (vl + 15) >> 4;
    j.kl = kl;
    jobs[k] = j;
    out.rec_idx[k] = rec;
    out.key_off[k] = dst_byte + 4;
    out.key_len[k] = kl - 13;
    out.val_off[k] = dst_byte + (uint64_t)j.nk * 16;
    out.val_len[k] = vl;
    out.rev[k] = be64_bytes((const uint8_t *)(st.kslab + j.ksrc16) + kl - 8);
    }
}

// ---- k_gather: copy of every winner's [internal key, padded][value, padded] into the response arena, staged through
// registers.  One warp per kv: every lane loads up to GATHER_U 16-byte chunks of the pair (all loads of a round are
// issued before its first store), then stores them; a kv larger than 32 x GATHER_U chunks takes several rounds.  Blocks
// of 32 jobs are handed out through a global counter (zeroed by the kernel that builds the jobs), so a CTA that starts
// late -- the SM was still busy with another stream's kernel -- simply takes fewer blocks.
// No shared memory and 40 registers: the copy runs beside the next batch's short kernels and the fan-out CTA instead of
// holding the SM's shared memory (the bulk-TMA ring it replaces held 2 x 111 KB per SM), and on a 2 320-byte kv it is
// faster with the GPU to itself too (profiles/h100_ab_gather.txt).
constexpr int GATHER_WARPS = 8;
constexpr int GATHER_U = 5;  // chunks per lane and round: 160 chunks (2560 B), a typical kv in one round

__device__ __forceinline__ uint4 ldg_evict_first(const uint4 *p, uint64_t pol)
{
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ void stg_evict_first(uint4 *p, const uint4 &v, uint64_t pol)
{
    asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y),
                 "r"(v.z), "r"(v.w), "l"(pol)
                 : "memory");
}

__global__ void __launch_bounds__(GATHER_WARPS * 32, 6)  // 40 registers: two CTAs fit beside the fan-out CTA and the short kernels
k_gather(StoreDev st, const GatherJob *__restrict__ jobs, const uint64_t *__restrict__ n_kvs_dev, uint4 *__restrict__ arena,
         unsigned long long *__restrict__ work_ctr)
{
    static_assert(sizeof(GatherJob) == 32, "lanes 0..7 hold the eight words of a job");
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n_kvs = *n_kvs_dev;
    const uint64_t l2pol = l2_evict_first_policy();  // both directions stream: the copy must not flush L2 for its neighbours
    for (;;) {
        unsigned long long b = 0;
        if (lane == 0) b = atomicAdd(work_ctr, 32ull);
        const uint64_t base = __shfl_sync(0xffffffffu, b, 0);
        if (base >= n_kvs) break;
        const uint32_t cnt = n_kvs - base < 32 ? (uint32_t)(n_kvs - base) : 32u;
        // word (lane & 7) of the current job; the next kv's is loaded while this one is copied
        const uint32_t *jw = (const uint32_t *)(jobs + base) + (lane & 7);
        uint32_t w = __ldg(jw);
        for (uint32_t j = 0; j < cnt; j++) {
            const uint64_t dst16 = ((uint64_t)__shfl_sync(0xffffffffu, w, 1) << 32) | __shfl_sync(0xffffffffu, w, 0);
            const uint64_t vsrc16 = ((uint64_t)__shfl_sync(0xffffffffu, w, 3) << 32) | __shfl_sync(0xffffffffu, w, 2);
            const uint32_t ksrc16 = __shfl_sync(0xffffffffu, w, 4);
            const uint32_t nk = __shfl_sync(0xffffffffu, w, 5), n = nk + __shfl_sync(0xffffffffu, w, 6);
            if (j + 1 < cnt) w = __ldg(jw + 8 * (j + 1));
            for (uint32_t c0 = 0; c0 < n; c0 += 32 * GATHER_U) {
                uint4 v[GATHER_U];
#pragma unroll
                for (int u = 0; u < GATHER_U; u++) {
                    const uint32_t c = c0 + lane + 32 * u;
                    if (c < n) v[u] = ldg_evict_first(c < nk ? st.kslab + ksrc16 + c : st.vslab + vsrc16 + (c - nk), l2pol);
                }
#pragma unroll
                for (int u = 0; u < GATHER_U; u++) {
                    const uint32_t c = c0 + lane + 32 * u;
                    if (c < n) stg_evict_first(arena + dst16 + c, v[u], l2pol);
                }
            }
        }
    }
}

// thread per emitted kv: where its element goes and what the per-kv view arrays say
__global__ void __launch_bounds__(256)
k_wire_jobs(StoreDev st, const ReqDev *__restrict__ reqs, uint32_t nreq, const uint64_t *__restrict__ job_first,
            const uint64_t *__restrict__ arena_base, const uint32_t *__restrict__ sel,
            const uint64_t *__restrict__ slot, int wire, WireJob *__restrict__ jobs, WireOut out)
{
    const uint64_t n_kvs = job_first[nreq];
    if (n_kvs == 0 && blockIdx.x == 0 && threadIdx.x == 0) out.elem_off[0] = 0;
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n_kvs;
         k += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t lo = 0, hi = nreq;  // request of kv k: last q with job_first[q] <= k
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (job_first[mid] <= k) lo = mid; else hi = mid;
        }
        const uint32_t q = lo;
        const uint64_t s = reqs[q].sel_base + (k - job_first[q]);
        const uint32_t rec = sel[s];
        const uint64_t E = arena_base[q] + slot[s];
        const uint32_t kl = st.klen[rec], vl = st.vlen[rec];
        const uint32_t ksrc16 = st.koff16[rec];
        const uint64_t rev = be64_bytes((const uint8_t *)(st.kslab + ksrc16) + kl - 8);
        const WireSizes ws = wire_sizes(kl - 13, vl, rev, wire);
        __align__(16) uint8_t h1[32], h2[32];
        uint32_t n1, n2;
#pragma unroll
        for (int b = 0; b < 32; b++) h1[b] = h2[b] = 0;
        wire_headers(ws, wire, h1, n1, h2, n2);
        const uint64_t vsrc16 = st.voff16[rec];
        WireJob j;
        j.loc = make_uint4((uint32_t)E, (uint32_t)(E >> 32), (uint32_t)vsrc16, (uint32_t)(vsrc16 >> 32));
        j.len = make_uint4(ksrc16, ws.ul, vl, n1 | (n2 << 8));
        j.h1[0] = ((const uint4 *)h1)[0];
        j.h1[1] = ((const uint4 *)h1)[1];
        j.h2[0] = ((const uint4 *)h2)[0];
        j.h2[1] = ((const uint4 *)h2)[1];
        jobs[k] = j;
        out.rec_idx[k] = rec;
        out.rev[k] = rev;
        out.key_off[k] = E + n1;
        out.key_len[k] = ws.ul;
        out.val_off[k] = E + n1 + ws.ul + n2;
        out.val_len[k] = vl;
        out.elem_off[k] = E;
        if (k == n_kvs - 1) out.elem_off[n_kvs] = E + ws.elem;
    }
}

// bytes [lo, hi) of a 16-byte chunk as a mask (0xff per selected byte); lo/hi are clamped to [0,16]
__device__ __forceinline__ uint4 byte_mask16(int lo, int hi)
{
    lo = max(lo, 0);
    hi = min(hi, 16);
    uint32_t w[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int a = max(lo - 4 * k, 0), b = min(hi - 4 * k, 4);  // byte range inside word k
        uint32_t m = 0;
        if (b > a) {
            const uint32_t upto_b = b >= 4 ? 0xffffffffu : ((1u << (8 * b)) - 1u);
            const uint32_t upto_a = a >= 4 ? 0xffffffffu : ((1u << (8 * a)) - 1u);
            m = upto_b & ~upto_a;
        }
        w[k] = m;
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// 16 bytes starting `s` bytes (0..15) into the 32-byte pair (lo, hi)
__device__ __forceinline__ uint4 funnel16(const uint4 &lo, const uint4 &hi, uint32_t s)
{
    const uint32_t w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
    const uint32_t ws = s >> 2, bs = (s & 3) * 8;
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        uint32_t a = 0, b = 0;
#pragma unroll
        for (int t = 0; t < 4; t++) {  // ws is 0..3: select without dynamic register indexing
            if (ws == (uint32_t)t) {
                a = w[t + k];
                b = w[t + k + 1 < 8 ? t + k + 1 : 7];
            }
        }
        o[k] = __funnelshift_r(a, b, bs);
    }
    return make_uint4(o[0], o[1], o[2], o[3]);
}

// the part of the element's chunk [e0, e0+16) that comes from a global-memory segment: segment bytes
// [begin, begin+len) of the element are bytes [skip, skip+len) behind the 16-byte aligned pointer `base`
template <bool SMEM>
__device__ __forceinline__ uint4 wire_ld(const uint4 *p)
{
    return SMEM ? *p : __ldg(p);  // staged copy in shared memory, or the slab itself
}

template <bool SMEM, typename I>
__device__ __forceinline__ void seg_mem(uint4 &acc, I e0, I begin, uint32_t len, const uint4 *base, uint32_t skip)
{
    const I lo = begin - e0, hi = begin + (I)len - e0;  // segment range in chunk coordinates
    if (hi <= 0 || lo >= 16 || len == 0) return;
    const I t = (I)skip + (e0 - begin);  // source byte of chunk byte 0 (may be negative)
    const I ci = t >> 4;                          // floor
    const uint32_t s = (uint32_t)(t & 15);
    const I last = ((I)skip + len - 1) >> 4;  // last chunk holding segment bytes
    uint4 a = make_uint4(0, 0, 0, 0), b = a;
    if (ci >= 0 && ci <= last) a = wire_ld<SMEM>(base + ci);
    if (s != 0 && ci + 1 >= 0 && ci + 1 <= last) b = wire_ld<SMEM>(base + ci + 1);
    const uint4 v = funnel16(a, b, s);
    const uint4 m = byte_mask16((int)max(lo, (I)0), (int)min(hi, (I)16));
    acc.x |= v.x & m.x;
    acc.y |= v.y & m.y;
    acc.z |= v.z & m.z;
    acc.w |= v.w & m.w;
}

// ... and the part that comes from a short header (at most 32 bytes, held in two registers quads): chunk byte j is
// header byte j - lo, i.e. the 16 bytes at offset 16 - lo of the 64-byte string [16 zero bytes | h_lo | h_hi | 16 zero]
template <typename I>
__device__ __forceinline__ void seg_reg(uint4 &acc, I e0, I begin, uint32_t len, const uint4 &h_lo, const uint4 &h_hi)
{
    const I lo = begin - e0, hi = lo + (I)len;
    if (hi <= 0 || lo >= 16 || len == 0) return;
    const int o = 16 - (int)lo;  // 1 .. 47
    const uint4 z = make_uint4(0, 0, 0, 0);
    const int q = o >> 4;
    const uint4 a = q == 0 ? z : q == 1 ? h_lo : h_hi;
    const uint4 b = q == 0 ? h_lo : q == 1 ? h_hi : z;
    const uint4 v = funnel16(a, b, (uint32_t)(o & 15));
    const uint4 m = byte_mask16((int)max(lo, (I)0), (int)min(hi, (I)16));
    acc.x |= v.x & m.x;
    acc.y |= v.y & m.y;
    acc.z |= v.z & m.z;
    acc.w |= v.w & m.w;
}

constexpr int WIRE_WARPS = 8;

// 16 bytes starting 4*WS + bs/8 bytes into the pair (a, b): the word offset is a compile-time constant, the bit shift
// inside a word (bs = 0, 8, 16, 24) is a run-time operand of the funnel shift
template <int WS>
__device__ __forceinline__ uint4 funnel16_w(const uint4 &a, const uint4 &b, uint32_t bs)
{
    const uint32_t w0 = WS == 0 ? a.x : WS == 1 ? a.y : WS == 2 ? a.z : a.w;
    const uint32_t w1 = WS == 0 ? a.y : WS == 1 ? a.z : WS == 2 ? a.w : b.x;
    const uint32_t w2 = WS == 0 ? a.z : WS == 1 ? a.w : WS == 2 ? b.x : b.y;
    const uint32_t w3 = WS == 0 ? a.w : WS == 1 ? b.x : WS == 2 ? b.y : b.z;
    const uint32_t w4 = WS == 0 ? b.x : WS == 1 ? b.y : WS == 2 ? b.z : b.w;
    return make_uint4(__funnelshift_r(w0, w1, bs), __funnelshift_r(w1, w2, bs), __funnelshift_r(w2, w3, bs),
                      __funnelshift_r(w3, w4, bs));
}

// Interior chunks [c_lo, c_hi) of a destination that lie entirely inside one source segment: chunk c holds source
// bytes [t0 + 16 (c - c_lo), +16) behind `base`, so the byte shift is the same for all of them.  Per chunk: two
// 16-byte loads (the second is the neighbour lane's first), four funnel shifts, one 16-byte store; two chunks per
// lane and step.
template <bool SMEM, int WS, typename I>
__device__ __forceinline__ void copy_interior_w(uint4 *__restrict__ dst0, I c_lo, I c_hi,
                                                const uint4 *src, uint32_t bs, uint32_t lane)
{
    const I n = c_hi - c_lo;
    uint4 *d = dst0 + c_lo;
    for (I i = lane; i < n; i += 64) {
        const bool two = i + 32 < n;
        const uint4 a0 = wire_ld<SMEM>(src + i), b0 = wire_ld<SMEM>(src + i + 1);
        const uint4 a1 = two ? wire_ld<SMEM>(src + i + 32) : a0, b1 = two ? wire_ld<SMEM>(src + i + 33) : b0;
        stg_stream(d + i, funnel16_w<WS>(a0, b0, bs));
        if (two) stg_stream(d + i + 32, funnel16_w<WS>(a1, b1, bs));
    }
}

template <bool SMEM, typename I>
__device__ __forceinline__ void copy_interior(uint4 *__restrict__ dst0, I c_lo, I c_hi, const uint4 *base, I t0,
                                              uint32_t lane)
{
    if (c_hi <= c_lo) return;
    const uint4 *src = base + (t0 >> 4);
    const uint32_t s = (uint32_t)(t0 & 15), bs = (s & 3) * 8;
    switch (s >> 2) {  // warp-uniform
        case 0: copy_interior_w<SMEM, 0, I>(dst0, c_lo, c_hi, src, bs, lane); break;
        case 1: copy_interior_w<SMEM, 1, I>(dst0, c_lo, c_hi, src, bs, lane); break;
        case 2: copy_interior_w<SMEM, 2, I>(dst0, c_lo, c_hi, src, bs, lane); break;
        default: copy_interior_w<SMEM, 3, I>(dst0, c_lo, c_hi, src, bs, lane); break;
    }
}

// One element, by one warp.  The destination is produced in aligned 16-byte chunks.  Chunks that lie entirely inside
// the user key or inside the value (all but a handful) take the uniform-shift fast path; the few boundary chunks
// (headers, segment seams, the element's first and last chunk, which it shares with its neighbours) are assembled
// from the four segments [header | user key | rev + value header | value] and fall back to byte stores where they
// are partial.  ksrc points at the internal key (user key at +4), vsrc at the value; both 16-byte aligned.
// KSMEM / VSMEM: the key / the value is read from its staged copy in shared memory, else from the slab itself.
template <bool KSMEM, bool VSMEM, typename I>
__device__ __forceinline__ void wire_emit_element(const uint4 &loc, const uint4 &len, const uint4 &h1a, const uint4 &h1b,
                                                  const uint4 &h2a, const uint4 &h2b, const uint4 *ksrc,
                                                  const uint4 *vsrc, uint8_t *__restrict__ arena, uint32_t lane)
{
    const uint64_t dst = ((uint64_t)loc.y << 32) | loc.x;
    const uint32_t ul = len.y, vl = len.z, n1 = len.w & 0xffu, n2 = (len.w >> 8) & 0xffu;
    const I total = (I)n1 + ul + n2 + vl;
    const I lead = (I)(dst & 15);
    uint4 *dst0 = (uint4 *)(arena + (dst - lead));
    const I nchunks = (lead + total + 15) >> 4;
    const I b_key = n1, b_h2 = b_key + ul, b_val = b_h2 + n2;
    // interior chunk ranges of the two source segments (chunk c covers element bytes [16 c - lead, +16))
    const I ck_lo = (b_key + lead + 15) >> 4;
    const I ck_hi = max(ck_lo, (b_key + (I)ul + lead) >> 4);
    const I cv_lo = max(ck_hi, (b_val + lead + 15) >> 4);
    const I cv_hi = max(cv_lo, (b_val + (I)vl + lead) >> 4);
    copy_interior<KSMEM, I>(dst0, ck_lo, ck_hi, ksrc, 4 + (ck_lo * 16 - lead - b_key), lane);
    copy_interior<VSMEM, I>(dst0, cv_lo, cv_hi, vsrc, cv_lo * 16 - lead - b_val, lane);
    // boundary chunks: [0, ck_lo) u [ck_hi, cv_lo) u [cv_hi, nchunks)
    const I nb0 = ck_lo, nb1 = cv_lo - ck_hi, nb2 = nchunks - cv_hi;
    for (I i = lane; i < nb0 + nb1 + nb2; i += 32) {
        const I c = i < nb0 ? i : i < nb0 + nb1 ? ck_hi + (i - nb0) : cv_hi + (i - nb0 - nb1);
        const I e0 = c * 16 - lead;
        uint4 acc = make_uint4(0, 0, 0, 0);
        seg_reg<I>(acc, e0, 0, n1, h1a, h1b);
        seg_mem<KSMEM, I>(acc, e0, b_key, ul, ksrc, 4);
        seg_reg<I>(acc, e0, b_h2, n2, h2a, h2b);
        seg_mem<VSMEM, I>(acc, e0, b_val, vl, vsrc, 0);
        if (e0 >= 0 && e0 + 16 <= total) {
            stg_stream(dst0 + c, acc);
        } else {
            uint8_t *d = (uint8_t *)(dst0 + c);
#pragma unroll
            for (int b = 0; b < 16; b++)
                if (e0 + b >= 0 && e0 + b < total) d[b] = (uint8_t)byte_of(acc, b);
        }
    }
}

__device__ __forceinline__ uint32_t wsmem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void wmbar_wait(uint64_t *bar, uint32_t parity, unsigned int *err_flag)
{
    dmbar_wait(bar, parity, err_flag);  // bounded: see kb_internal.cuh
}

constexpr int WIRE_MAX_STAGES = 8;
constexpr uint32_t WIRE_JOB_CHUNKS = sizeof(WireJob) / 16;  // 6
constexpr uint32_t WIRE_WARP_CHUNKS = 880;                  // shared memory per warp: two CTAs of 8 warps per SM

// k_wire_copy: warp per element, sources staged by the copy engine.  Lane 0 runs `stages - 1` elements ahead and
// issues, per element, three bulk (TMA) copies into the warp's ring slot -- the 96-byte job, the internal key, the
// value -- completing on the slot's mbarrier; the whole warp then assembles the element from shared memory
// (wire_emit_element<true, true>) and writes it with 16-byte stores.  The loads in flight are therefore independent of
// the registers, exactly as in k_gather; only the unaligned destination forces the bytes through the lanes.  An element
// too large for a slot is copied straight from the slabs (wire_emit_element<false, false>).
// HOSTV: the value heap is mapped host memory (KB_CFG_HOST_VALUES).  The bulk copy is used for HBM sources only: a slot
// stages the job and the key, and the value is read straight from the heap (wire_emit_element<true, false>).
template <bool HOSTV>
__global__ void __launch_bounds__(WIRE_WARPS * 32, 2)
k_wire_copy(StoreDev st, const WireJob *__restrict__ jobs, const uint64_t *__restrict__ n_kvs_dev,
            uint8_t *__restrict__ arena, uint32_t slot_chunks, uint32_t stages, unsigned int *__restrict__ err_flag)
{
    extern __shared__ __align__(128) uint4 wbuf[];  // WIRE_WARPS x stages x slot_chunks
    __shared__ uint64_t wbars[WIRE_WARPS * WIRE_MAX_STAGES];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint4 *ring = wbuf + (size_t)warp * stages * slot_chunks;
    uint64_t *bar = wbars + warp * WIRE_MAX_STAGES;
    if (lane == 0) {
        for (uint32_t s = 0; s < stages; s++)
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(wsmem_u32(bar + s)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    const uint64_t n_kvs = *n_kvs_dev;
    const uint64_t kstride = (uint64_t)gridDim.x * WIRE_WARPS;
    const uint64_t k0 = (uint64_t)blockIdx.x * WIRE_WARPS + warp;
    const uint32_t room = slot_chunks - WIRE_JOB_CHUNKS - 1;  // chunks of key + value a slot can stage

    // lane 0: issue the copies of element k into ring slot `slot`
    auto issue = [&](uint64_t k, uint32_t slot) {
        const uint4 *jp = (const uint4 *)(jobs + k);
        const uint4 loc = __ldg(jp), len = __ldg(jp + 1);
        const uint32_t nkc = (4 + len.y + 15) >> 4, nvc = HOSTV ? 0 : (len.z + 15) >> 4;  // chunks staged
        const bool fits = nkc + nvc <= room;
        uint4 *sl = ring + (size_t)slot * slot_chunks;
        const uint32_t b = wsmem_u32(bar + slot);
        // the slot was last read (generic proxy) by the warp before the __syncwarp that precedes this call
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b),
                     "r"((WIRE_JOB_CHUNKS + (fits ? nkc + nvc : 0)) * 16)
                     : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                         wsmem_u32(sl)),
                     "l"(jp), "r"(WIRE_JOB_CHUNKS * 16), "r"(b)
                     : "memory");
        if (fits) {
            const uint64_t vsrc16 = ((uint64_t)loc.w << 32) | loc.z;
            if (nkc)
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                                 wsmem_u32(sl + WIRE_JOB_CHUNKS)),
                             "l"(st.kslab + len.x), "r"(nkc * 16), "r"(b)
                             : "memory");
            if (nvc)
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                                 wsmem_u32(sl + WIRE_JOB_CHUNKS + nkc)),
                             "l"(st.vslab + vsrc16), "r"(nvc * 16), "r"(b)
                             : "memory");
        }
    };

    uint64_t k_issue = k0, k_proc = k0;
    uint32_t s_issue = 0, s_proc = 0, ph = 0;
    // prologue: fill all but one slot
    for (uint32_t i = 0; i + 1 < stages && k_issue < n_kvs; i++, k_issue += kstride) {
        if (lane == 0) issue(k_issue, s_issue);
        if (++s_issue == stages) s_issue = 0;
    }
    for (; k_proc < n_kvs; k_proc += kstride) {
        if (k_issue < n_kvs) {  // the slot freed by the previous step (a __syncwarp ended that step)
            if (lane == 0) issue(k_issue, s_issue);
            if (++s_issue == stages) s_issue = 0;
            k_issue += kstride;
        }
        wmbar_wait(bar + s_proc, ph, err_flag);
        const uint4 *sl = ring + (size_t)s_proc * slot_chunks;
        const uint4 loc = sl[0], len = sl[1], h1a = sl[2], h1b = sl[3], h2a = sl[4], h2b = sl[5];
        const uint32_t nkc = (4 + len.y + 15) >> 4, nvc = HOSTV ? 0 : (len.z + 15) >> 4;
        if (nkc + nvc <= room) {
            if constexpr (HOSTV) {  // a value of any length: long long offsets
                const uint64_t vsrc16 = ((uint64_t)loc.w << 32) | loc.z;
                wire_emit_element<true, false, long long>(loc, len, h1a, h1b, h2a, h2b, sl + WIRE_JOB_CHUNKS,
                                                          st.vslab + vsrc16, arena, lane);
            } else {
                wire_emit_element<true, true, int>(loc, len, h1a, h1b, h2a, h2b, sl + WIRE_JOB_CHUNKS,
                                                   sl + WIRE_JOB_CHUNKS + nkc, arena, lane);
            }
        } else {
            const uint64_t vsrc16 = ((uint64_t)loc.w << 32) | loc.z;
            wire_emit_element<false, false, long long>(loc, len, h1a, h1b, h2a, h2b, st.kslab + len.x, st.vslab + vsrc16,
                                                       arena, lane);
        }
        __syncwarp();  // every lane is done reading the slot before lane 0 refills it
        if (++s_proc == stages) {
            s_proc = 0;
            ph ^= 1;
        }
    }
}

// ring geometry of k_wire_copy for a store whose largest padded [key][value] pair is `max_kv_chunks`
static inline void wire_geometry(uint32_t max_kv_chunks, uint32_t *slot_chunks, uint32_t *stages)
{
    const uint32_t room = max_kv_chunks < 32 ? 32 : max_kv_chunks > 160 ? 160 : max_kv_chunks;
    const uint32_t slot = WIRE_JOB_CHUNKS + room + 1;  // job | key + value | one chunk of slack for the shifted reads
    uint32_t s = WIRE_WARP_CHUNKS / slot;
    s = s < 3 ? 3 : s > (uint32_t)WIRE_MAX_STAGES ? (uint32_t)WIRE_MAX_STAGES : s;
    *slot_chunks = slot;
    *stages = s;
}

}  // namespace

kb_result *kb_result_new(ResultKind kind, int out_mode)
{
    kb_result *r = new kb_result();
    r->kind = kind;
    r->out_mode = out_mode;
    return r;
}

// the device meta and arena back to their pools
void result_put_device(kb_ctx *ctx, kb_result *res)
{
    pool_put_dev(ctx, res->d_meta);
    res->d_meta = DBuf();
    pool_put_arena(ctx, res->d_arena, res->kind == ResultKind::point_read);
    res->d_arena = DBuf();
}

void result_release_locked(kb_ctx *ctx, kb_result *res)
{
    if (!res) return;
    if (ctx) {
        pool_put_host(ctx, res->h_meta);
        pool_put_host(ctx, res->h_arena);
        result_put_device(ctx, res);
        if (res->done_ev) ctx->ev_pool.push_back(res->done_ev);
    }
    delete res;
}

int result_to_host(kb_ctx *ctx, kb_result *res, cudaStream_t s, std::initializer_list<D2HPiece> pieces,
                   uint64_t arena_bytes, const char *what)
{
    size_t meta = 0;
    for (const D2HPiece &p : pieces) meta += p.bytes;
    int rc = KB_OK;
    cudaError_t e = res->done_ev ? cudaStreamWaitEvent(s, res->done_ev, 0) : cudaSuccess;
    if (meta) {
        pool_put_host(ctx, res->h_meta);
        res->h_meta = HBuf();
        rc = pool_get_host(ctx, meta + 64, &res->h_meta);
    }
    if (rc == KB_OK && arena_bytes) rc = pool_get_host(ctx, arena_bytes + 16, &res->h_arena);
    if (rc == KB_OK) {
        size_t off = 0;
        for (const D2HPiece &p : pieces) {
            if (p.bytes && e == cudaSuccess)
                e = cudaMemcpyAsync((uint8_t *)res->h_meta.p + off, p.src, p.bytes, cudaMemcpyDeviceToHost, s);
            off += p.bytes;
        }
        if (arena_bytes && e == cudaSuccess)
            e = cudaMemcpyAsync(res->h_arena.p, res->d_arena.p, arena_bytes, cudaMemcpyDeviceToHost, s);
    }
    const cudaError_t es = cudaStreamSynchronize(s);  // also after a failure: nothing may still be writing the buffers
    if (e == cudaSuccess) e = es;
    if (rc == KB_OK && e != cudaSuccess) rc = kb_cuda_fail(ctx, e, what);
    result_put_device(ctx, res);
    return rc;
}

extern "C" void kb_result_free(kb_ctx *ctx, kb_result *res)
{
    if (!res) return;
    if (ctx) {
        std::lock_guard<std::mutex> g(ctx->mu);
        result_release_locked(ctx, res);
    } else {
        delete res;
    }
}

// gather of `n_jobs` (upper bound; the count is the table's kvs) copy jobs into `arena`
int launch_gather(kb_ctx *ctx, cudaStream_t strm, const GatherJob *d_jobs, const JobTable &tab, uint4 *arena,
                  uint64_t n_jobs, uint64_t alg_bytes)
{
    // two CTAs per SM (16 warps, one 2.3 KB kv each in flight) reach the copy rate; a third takes HBM from the fan-out,
    // and one showed no gain (profiles/h100_ab.txt)
    const unsigned ggrid =
        (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((n_jobs + GATHER_WARPS * 32 - 1) / (GATHER_WARPS * 32), 2 * ctx->n_sms));
    KB_LAUNCH_S(ctx, strm, "k_gather", alg_bytes,
                (k_gather<<<ggrid, GATHER_WARPS * 32, 0, strm>>>(ctx->st, d_jobs, tab.n_kvs(), arena, tab.work_ctr)));
    return KB_OK;
}

// The context's error flag, as a lane batch's rows or a page cut published it (its HostPub's error word): raised by an
// EARLIER wire copy of this context and never cleared
int pub_err_check(kb_ctx *ctx, const HostPub &pub)
{
    if (pub.err() == 0) return KB_OK;
    return kb_fail(ctx, KB_ECUDA, "range scan: an earlier wire copy of this context timed out on a bulk copy (the "
                                  "context's error flag stays raised)");
}

// the per-kv view arrays of an answer of at most `cap` kvs inside one device buffer of cap * (wire ? 44 : 36) + 72 bytes;
// returns the element offsets (wire modes: cap + 1 entries)
uint64_t *om_layout(void *om, uint64_t cap, int wire, GatherOut &go)
{
    go.rev = (uint64_t *)om;
    go.key_off = go.rev + cap;
    go.val_off = go.key_off + cap;
    uint64_t *elem_off = go.val_off + cap;
    go.rec_idx = (uint32_t *)(wire ? elem_off + cap + 1 : elem_off);
    go.key_len = go.rec_idx + cap;
    go.val_len = go.key_len + cap;
    return elem_off;
}

// A new result (held by `res`) and the buffers of its answer: an arena of arena_bytes (none when 0) and, for a range
// answer (batch or page) of at most cap_kvs kvs, its per-kv arrays (res->d_meta, laid out into go; *elem_off: the element
// offsets).  A point-read result takes only the arena, from the point-read pool.
int answer_new(kb_ctx *ctx, HeldResult &res, ResultKind kind, int out_mode, int wire, uint64_t cap_kvs,
               uint64_t arena_bytes, GatherOut *go, uint64_t **elem_off)
{
    res.p = kb_result_new(kind, out_mode);
    res.p->wire = wire;
    if (!arena_bytes) return KB_OK;
    if (cap_kvs) {
        KB_TRY(pool_get_dev(ctx, cap_kvs * (wire ? 44 : 36) + 64 + 8, &res.p->d_meta));
        *elem_off = om_layout(res.p->d_meta.p, cap_kvs, wire, *go);
    }
    return pool_get_arena(ctx, arena_bytes, &res.p->d_arena, kind == ResultKind::point_read);
}

// out_mode -> the base mode (KB_OUT_*) and the wire mode (KB_WIRE_*_I); KB_EINVAL when both wire flags are set.  Each
// entry point checks which combinations it accepts.
int split_out_mode(int out_mode, int *base, int *wire)
{
    const int flags = out_mode & (KB_WIRE_ETCD_KVS | KB_WIRE_ETCD_EVENTS);
    *base = out_mode & ~(KB_WIRE_ETCD_KVS | KB_WIRE_ETCD_EVENTS);
    *wire = flags == KB_WIRE_ETCD_KVS ? KB_WIRE_KVS_I : flags == KB_WIRE_ETCD_EVENTS ? KB_WIRE_EVENTS_I : 0;
    return flags == (KB_WIRE_ETCD_KVS | KB_WIRE_ETCD_EVENTS) ? KB_EINVAL : KB_OK;
}

// the job buffer launch_copy needs for n kvs
size_t copy_jobs_bytes(uint64_t n, int wire) { return n * (wire ? sizeof(WireJob) : sizeof(GatherJob)); }

// the copy on stream sg starts behind the copy jobs enqueued on L.stream
int copy_after_jobs(kb_ctx *ctx, ScanLane &L, cudaStream_t sg)
{
    if (sg == L.stream) return KB_OK;
    KB_CUDA(ctx, cudaEventRecord(L.ev_jobs, L.stream));
    KB_CUDA(ctx, cudaStreamWaitEvent(sg, L.ev_jobs, 0));
    return KB_OK;
}

// the end of a copy just enqueued on the copy stream sg: recorded in ev_copied (its JobSet's ev_gather) and in
// res->done_ev, which completes the answer (kb_result_wait, kb_sync)
int copy_done(kb_ctx *ctx, cudaStream_t sg, cudaEvent_t ev_copied, kb_result *res)
{
    KB_CUDA(ctx, cudaEventRecord(ev_copied, sg));
    KB_TRY(ev_take(ctx, &res->done_ev));
    KB_CUDA(ctx, cudaEventRecord(res->done_ev, sg));
    return KB_OK;
}

// The copy of an answer whose job table (job_first[nreq + 1] | arena_base[nreq + 1] | work counter) is being written on
// L.stream: the copy jobs (into d_jobs) and the per-kv arrays on L.stream, the copy into res->d_arena on stream sg.  A
// range answer copies on the copy stream and passes ev_copied (its JobSet's ev_gather): the end of the copy is recorded
// there and in res->done_ev.  A point-read answer copies on the lane stream itself (ev_copied = nullptr): the batch
// publishes its rows behind the copy, so the arena is complete when they arrive.
int launch_copy(kb_ctx *ctx, ScanLane &L, cudaStream_t sg, void *d_jobs, cudaEvent_t ev_copied, const ReqDev *d_reqs,
                uint32_t nreq, const JobTable &tab, const uint32_t *sel, const uint64_t *slot, uint64_t cap_kvs, int wire,
                const GatherOut &go, uint64_t *d_elem_off, kb_result *res)
{
    const uint64_t *d_jobfirst = tab.job_first, *d_arenabase = tab.arena_base;
    const unsigned jgrid = (unsigned)std::min<uint64_t>((cap_kvs + 255) / 256, (uint64_t)ctx->n_sms * 8);
    if (wire) {
        WireOut wo;
        wo.rec_idx = go.rec_idx;
        wo.rev = go.rev;
        wo.key_off = go.key_off;
        wo.key_len = go.key_len;
        wo.val_off = go.val_off;
        wo.val_len = go.val_len;
        wo.elem_off = d_elem_off;
        WireJob *d_wj = (WireJob *)d_jobs;
        KB_LAUNCH_S(ctx, L.stream, "k_wire_jobs", cap_kvs * 20,
                    (k_wire_jobs<<<jgrid, 256, 0, L.stream>>>(ctx->st, d_reqs, nreq, d_jobfirst, d_arenabase, sel, slot,
                                                              wire, d_wj, wo)));
        KB_TRY(copy_after_jobs(ctx, L, sg));
        uint32_t slot_chunks, wstages;
        wire_geometry(ctx->max_kv_chunks, &slot_chunks, &wstages);
        const size_t wsmem = (size_t)WIRE_WARPS * wstages * slot_chunks * 16;
        // the context's value placement picks the kernel
        auto *kernel = ctx->host_values ? k_wire_copy<true> : k_wire_copy<false>;
        if (!ctx->wire_attr_set) {
            cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(WIRE_WARPS * WIRE_WARP_CHUNKS * 16));
            ctx->wire_attr_set = true;
        }
        const unsigned wgrid =
            (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((cap_kvs + WIRE_WARPS - 1) / WIRE_WARPS, 2 * (uint64_t)ctx->n_sms));
        KB_LAUNCH_S(ctx, sg, "k_wire_copy", 0,
                    (kernel<<<wgrid, WIRE_WARPS * 32, wsmem, sg>>>(ctx->st, d_wj, tab.n_kvs(), (uint8_t *)res->d_arena.p,
                                                                 slot_chunks, wstages, (unsigned int *)ctx->d_ctrs.p + 8)));
    } else {
        GatherJob *d_gj = (GatherJob *)d_jobs;
        KB_LAUNCH_S(ctx, L.stream, "k_gather_jobs", cap_kvs * 20,
                    (k_gather_jobs<<<jgrid, 256, 0, L.stream>>>(ctx->st, d_reqs, nreq, d_jobfirst, d_arenabase, sel, slot,
                                                                d_gj, go)));
        KB_TRY(copy_after_jobs(ctx, L, sg));
        KB_TRY(launch_gather(ctx, sg, d_gj, tab, (uint4 *)res->d_arena.p, cap_kvs, 0));
    }
    return ev_copied ? copy_done(ctx, sg, ev_copied, res) : KB_OK;
}

// The per-kv arrays and the arena of an answer of nk > 0 kvs and nbytes arena bytes become the result's: KB_OUT_HOST
// copies them to pinned host memory (and hands the device meta and arena back), KB_OUT_DEVICE keeps them in HBM
int answer_finish(kb_ctx *ctx, kb_result *res, const GatherOut &go, const uint64_t *d_elem_off, uint64_t nk,
                  uint64_t nbytes, kb_tp &tseg)
{
    const int wire = res->wire;
    if (res->out_mode == KB_OUT_HOST) {
        // per-kv arrays: six strided pieces of the capacity-sized device layout -> one compact host layout, on the
        // host-copy stream behind this batch's gather (which waited for the per-kv arrays): a later batch's gather (already
        // queued on the copy stream when batches are submitted ahead) does not sit between the answer and the host
        const int rc = result_to_host(ctx, res, ctx->stream_h,
                                      {{go.rev, nk * 8}, {go.key_off, nk * 8}, {go.val_off, nk * 8},
                                       {d_elem_off, wire ? (nk + 1) * 8 : 0}, {go.rec_idx, nk * 4}, {go.key_len, nk * 4},
                                       {go.val_len, nk * 4}},
                                      nbytes, "range D2H");
        kb_seg(ctx, "host:range_d2h", tseg);
        KB_TRY(rc);
        uint8_t *hm = (uint8_t *)res->h_meta.p;
        res->rev = (const uint64_t *)hm;
        res->key_off = res->rev + nk;
        res->val_off = res->key_off + nk;
        res->elem_off = wire ? res->val_off + nk : nullptr;
        res->rec_idx = (const uint32_t *)(res->val_off + nk + (wire ? nk + 1 : 0));
        res->key_len = res->rec_idx + nk;
        res->val_len = res->key_len + nk;
    } else {
        res->rev = go.rev;
        res->key_off = go.key_off;
        res->val_off = go.val_off;
        res->rec_idx = go.rec_idx;
        res->key_len = go.key_len;
        res->val_len = go.val_len;
        res->elem_off = wire ? d_elem_off : nullptr;
    }
    return KB_OK;
}

extern "C" int kb_result_wait(kb_ctx *ctx, const kb_result *res, void *cuda_stream)
{
    if (!ctx || !res) return KB_EINVAL;
    if (!res->done_ev) return KB_OK;
    cudaSetDevice(ctx->device);
    if (cuda_stream) {
        KB_CUDA(ctx, cudaStreamWaitEvent((cudaStream_t)cuda_stream, res->done_ev, 0));
    } else {
        KB_CUDA(ctx, cudaEventSynchronize(res->done_ev));
    }
    return KB_OK;
}

// ---- framing of the wire elements (host): etcdserverpb.ResponseHeader{revision} (pkg/server/etcd/kv.go:253-257) is
// field 1 of both responses; a header with revision 0 is still emitted (non-nil message of length 0)
static uint64_t host_put_varint(uint8_t *out, uint64_t v)
{
    uint64_t n = 0;
    while (v >= 0x80) {
        out[n++] = (uint8_t)(v | 0x80);
        v >>= 7;
    }
    out[n++] = (uint8_t)v;
    return n;
}

static uint64_t host_put_header(uint64_t header_rev, uint8_t *out)
{
    uint8_t body[12];
    uint64_t nb = 0;
    if (header_rev) {
        body[nb++] = 0x18;  // ResponseHeader.revision = 3, varint
        nb += host_put_varint(body + nb, header_rev);
    }
    uint64_t w = 0;
    out[w++] = 0x0a;  // field 1, length-delimited
    w += host_put_varint(out + w, nb);
    memcpy(out + w, body, nb);
    return w + nb;
}

extern "C" uint64_t kb_wire_range_head(uint64_t header_rev, uint8_t *out)
{
    return out ? host_put_header(header_rev, out) : 0;
}

extern "C" uint64_t kb_wire_range_tail(int more, int64_t count, uint8_t *out)
{
    if (!out) return 0;
    uint64_t w = 0;
    if (more) {  // RangeResponse.more = 3
        out[w++] = 0x18;
        out[w++] = 1;
    }
    if (count) {  // RangeResponse.count = 4
        out[w++] = 0x20;
        w += host_put_varint(out + w, (uint64_t)count);
    }
    return w;
}

extern "C" uint64_t kb_wire_watch_head(uint64_t header_rev, int canceled, const uint8_t *reason, uint64_t reason_len,
                                       uint8_t *out)
{
    if (!out || (reason_len && !reason)) return 0;
    uint64_t w = host_put_header(header_rev, out);
    if (canceled) {  // WatchResponse.canceled = 4
        out[w++] = 0x20;
        out[w++] = 1;
    }
    if (reason_len) {  // WatchResponse.cancel_reason = 6
        out[w++] = 0x32;
        w += host_put_varint(out + w, reason_len);
        memcpy(out + w, reason, reason_len);
        w += reason_len;
    }
    return w;
}
