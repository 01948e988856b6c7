// kb_decode.cuh -- k_decode_lcp, the per-batch pass over the scan summary (included by kb_scan.cu).
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
// or restored and patched by kb_apply_batch for the records a batch touches (kb_store.cu summarize_record /
// k_summarize build it).  The per-batch pass then only
// compares the summary's revision against the request's read revision and the sweep's timeout revision: an
// element-wise kernel that reads 12 bytes and writes 4 per record, where the raw keys cost ~280.
#pragma once

#include "kb_internal.cuh"

namespace {

// One meta word per examined record from the summary: tile per CTA, four records per thread, every load of the thread
// issued before the first use.  Bit for bit what decoding the raw key and value gives (summarize_record in kb_store.cu
// holds the store-only half of that decision).
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
