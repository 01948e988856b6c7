// kb_decode.cuh -- the per-record scan summary and k_decode_lcp, the per-batch pass over it (included by kb_scan.cu).
//
// Every examined record is reduced to one 32-bit meta word:
//   bits 0..15  LCP with the preceding key (common-prefix length, the input of the "same user key" test)
//   bits 16..23 decode / visibility / tombstone / compaction-class flags (KB_M_*)
//
// Replaces coder.Decode (pkg/backend/coder/normal.go:58-70) and the per-record front half of worker.run
// (pkg/backend/scanner/scanner.go:430-453, 471-491, 566-591): decode, TTL expiry, revision visibility,
// tombstone test, deleted-flag revision-record test.
//
// Most of that word depends on the store alone: the LCP with the record in front (in directory order), whether the key
// decodes, the revision, the tombstone literal, the value's leading 8 bytes of a revision record.  Those facts are kept
// beside the directory as the scan summary (StoreDev::srev / sword, 12 bytes per record), built when a store is loaded
// or restored and patched by kb_apply_batch for the records a batch touches (k_summarize).  The per-batch pass then only
// compares the summary's revision against the request's read revision and the sweep's timeout revision: an
// element-wise kernel that reads 12 bytes and writes 4 per record, where the raw keys cost ~280.
#pragma once

#include "kb_internal.cuh"

namespace {

constexpr uint32_t MAGIC_LE = 0x8b80fb57u;  // bytes 57 fb 80 8b (coder/normal.go:26)

__device__ __forceinline__ uint32_t bswap32(uint32_t x) { return __byte_perm(x, 0, 0x0123); }

// Summary of record i of `st` against record i - 1 (record 0 gets KB_LCP_INF; the pass replaces the LCP of every
// request's first record by KB_LCP_INF anyway), computed by one warp; `lane` 0 stores it.
//   sword: the LCP in bits 0..15; KB_M_DEC_OK / KB_M_REV0 / KB_S_TOMBV (the value is "tombstone", util.go:28) at the
//          meta word's positions; KB_S_VL9, KB_S_VL8, KB_S_EVENTS (the user key contains "/events/") above them
//   srev:  the key's revision; for a revision record (revision 0) with a value of at least 8 bytes, the value's first
//          8 bytes big-endian (scanner.go:476-491, 566-591); 0 when the key does not decode
// The lanes compare 32 chunks of the two keys at a time and test 32 start positions of "/events/" at a time, so a
// record costs a few dependent round trips whatever its key length (the write path summarizes a few hundred records
// per batch, the load path all of them).
__device__ __forceinline__ void summarize_record(const StoreDev &st, uint32_t i, uint32_t lane, uint64_t *srev, uint32_t *sword)
{
    const unsigned FULLM = 0xffffffffu;
    const uint4 *kp = st.kslab + st.koff16[i];
    const uint32_t len = st.klen[i];
    uint32_t lcp = KB_LCP_INF;
    if (i > 0) {
        const uint4 *pp = st.kslab + st.koff16[i - 1];
        const uint32_t m = min(len, (uint32_t)st.klen[i - 1]);
        lcp = m;
        for (uint32_t c0 = 0; c0 * 16 < m; c0 += 32) {
            const uint32_t c = c0 + lane;
            const int p = c * 16 < m ? first_diff16(kp[c], pp[c]) : 16;
            const unsigned diff = __ballot_sync(FULLM, p < 16);
            if (diff) {
                const int src = __ffs(diff) - 1;
                lcp = min(m, (c0 + src) * 16 + (uint32_t)__shfl_sync(FULLM, p, src));
                break;
            }
        }
    }
    const uint8_t *kb = (const uint8_t *)kp;
    const uint32_t vl = st.vlen[i];
    uint32_t w = lcp;
    uint64_t s = 0;
    if (vl == 9) w |= KB_S_VL9;
    if (vl >= 8) w |= KB_S_VL8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (vl >= 8) v = st.vslab[st.voff16[i]];
    if (vl == 9 && v.x == 0x626d6f74u && v.y == 0x6e6f7473u && (v.z & 0xffu) == 0x65u) w |= KB_S_TOMBV;
    if (len >= 13 && ((const uint32_t *)kp)[0] == MAGIC_LE && kb[len - 9] == 0x24) {  // coder.Decode (normal.go:58-70)
        w |= KB_M_DEC_OK;
        s = be64_bytes(kb + len - 8);
        if (s == 0) {
            w |= KB_M_REV0;
            if (vl >= 8) s = ((uint64_t)bswap32(v.x) << 32) | bswap32(v.y);
        }
        // bytes.Contains(rawKey, "/events/") over the user key kb[4 .. len - 9)
        const uint8_t *uk = kb + 4;
        const uint32_t n = len - 13;
        bool found = false;
        for (uint32_t p = lane; p + 8 <= n && !found; p += 32) found = be64_bytes(uk + p) == 0x2f6576656e74732full;
        if (__any_sync(FULLM, found)) w |= KB_S_EVENTS;
    }
    if (lane == 0) {
        *srev = s;
        *sword = w;
    }
}

// summary of records idx[0 .. n) (idx == nullptr: of records 0 .. n) into srev / sword, warp per record
__global__ void __launch_bounds__(256)
k_summarize(StoreDev st, const uint32_t *__restrict__ idx, uint32_t n, uint64_t *__restrict__ srev, uint32_t *__restrict__ sword)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < n; t += warps) {
        const uint32_t i = idx ? idx[t] : (uint32_t)t;
        summarize_record(st, i, lane, srev + i, sword + i);
    }
}

// One meta word per examined record from the summary: tile per CTA, four records per thread, every load of the thread
// issued before the first use.  Bit for bit what decoding the raw key and value gives (summarize_record holds the
// store-only half of that decision).
__global__ void __launch_bounds__(256, 8)
k_decode_lcp(StoreDev st, const TileDev *__restrict__ tiles, ScanMode mode, uint32_t *__restrict__ meta)
{
    constexpr int PER = KB_TILE / 256;
    const TileDev &tile = tiles[blockIdx.x];
    const uint32_t rec0 = tile.rec0, n = tile.n, flat0 = tile.flat0, lo = tile.lo;
    const uint64_t read_rev = tile.read_rev;
    uint32_t w[PER];
    uint64_t s[PER];
#pragma unroll
    for (int j = 0; j < PER; j++) {
        const uint32_t r = j * 256 + threadIdx.x;
        w[j] = r < n ? __ldg(st.sword + rec0 + r) : 0u;
        s[j] = r < n ? __ldg(st.srev + rec0 + r) : 0ull;
    }
#pragma unroll
    for (int j = 0; j < PER; j++) {
        const uint32_t r = j * 256 + threadIdx.x;
        if (r >= n) break;
        const uint32_t lcp = rec0 + r == lo ? KB_LCP_INF : (w[j] & KB_M_LCP_MASK);  // a request's first record has no prev
        uint32_t flags = 0;
        if (w[j] & KB_M_DEC_OK) {
            const bool rev0 = (w[j] & KB_M_REV0) != 0;
            const uint64_t rev = rev0 ? 0 : s[j];
            flags = w[j] & (KB_M_DEC_OK | KB_M_REV0);
            bool expired = false;
            if (mode.ttl_scan && (w[j] & KB_S_EVENTS)) {  // compactIfExpired scanner.go:566-591
                if (rev0) {
                    if ((w[j] & KB_S_VL8) && s[j] <= mode.timeout_rev) {
                        expired = true;
                        flags |= KB_M_TTLREV;
                    }
                } else if (rev <= mode.timeout_rev) {
                    expired = true;
                    flags |= KB_M_TTLOBJ;
                }
            }
            if (!expired && rev <= read_rev) {  // scanner.go:451-453
                flags |= KB_M_TRIG;
                if (w[j] & KB_S_TOMBV) flags |= KB_M_TOMB;
                bool prevok = true;
                if (mode.compact && rev0 && (w[j] & KB_S_VL9)) {  // scanner.go:476-491
                    if (s[j] > read_rev)
                        prevok = false;  // `continue` without updating prev (Q5)
                    else
                        flags |= KB_M_REVDEL;
                }
                if (prevok) flags |= KB_M_PREVOK;
            }
        }
        meta[flat0 + r] = lcp | flags;
    }
}

}  // namespace
