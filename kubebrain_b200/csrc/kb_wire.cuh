// kb_wire.cuh -- the element format of the scan answer as etcd protobuf elements, written by the device: the element
// sizes the scan sizes answers with (kb_scan.cu, kb_batch.cu) and the job kb_copy.cu's k_wire_jobs / k_wire_copy build
// and copy.
//
// Replaces the per-kv materialisation of the etcd-compatible server: kvToEtcdKv (pkg/server/etcd/backendshim.go:427-436)
// + the gogo-protobuf Marshal of etcdserverpb.RangeResponse.kvs (List, backendshim.go:269-282) or of
// etcdserverpb.WatchResponse.events (range stream, backendshim.go:349-363; batches cut by receiver.go:119-138).
// A protobuf message is the concatenation of its fields, so the device writes the repeated-field ELEMENTS back to
// back (one per emitted kv, reference order) and the host only prepends / appends the few header and trailer bytes
// (kb_wire_range_head / _tail / kb_wire_watch_head): nothing is re-materialised per kv on the CPU.
//
//   KVS    element:  12 <len(kv)>  kv                       kv = [0a <ul> user key] [18 <rev>] [2a <vl> value]
//   EVENTS element:  5a <len(ev)>  ev,  ev = 12 <len(kv)> kv      (proto3: empty key / value and rev 0 are omitted)
//
// Field numbers: go.etcd.io/etcd/api/v3 v3.5.2 (reference go.mod:28), pinned by tests/test_wire.py.
#pragma once

#include "kb_internal.cuh"

namespace {

__device__ __forceinline__ uint32_t varint_len(uint64_t v) { return v ? (uint32_t)(70 - __clzll((long long)v)) / 7u : 1u; }

struct WireSizes {
    uint32_t ul, vl;
    uint64_t rev;
    uint64_t body, kv, elem;  // mvccpb.KeyValue body, kv field (tag + len + body), whole element
};

__device__ __forceinline__ WireSizes wire_sizes(uint32_t ul, uint32_t vl, uint64_t rev, int wire)
{
    WireSizes s;
    s.ul = ul;
    s.vl = vl;
    s.rev = rev;
    s.body = (ul ? 1 + varint_len(ul) + (uint64_t)ul : 0) + (rev ? 1 + varint_len(rev) : 0) +
             (vl ? 1 + varint_len(vl) + (uint64_t)vl : 0);
    s.kv = 1 + varint_len(s.body) + s.body;
    s.elem = wire == KB_WIRE_KVS_I ? s.kv : 1 + varint_len(s.kv) + s.kv;
    return s;
}

// response bytes of one emitted record: padded [key][value] in the arena modes, element bytes in the wire modes
__device__ __forceinline__ uint64_t kv_resp_bytes(const StoreDev &st, uint32_t rec, int wire)
{
    const uint32_t kl = st.klen[rec], vl = st.vlen[rec];
    if (!wire) return (uint64_t)pad16(kl) + pad16(vl);
    const uint64_t rev = be64_bytes((const uint8_t *)(st.kslab + st.koff16[rec]) + kl - 8);
    return wire_sizes(kl - 13, vl, rev, wire).elem;
}

struct __align__(16) WireJob {  // 96 bytes: six 16-byte loads, the same for every lane of the warp that copies it
    uint4 loc;     // {dst lo, dst hi, vsrc16 lo, vsrc16 hi}: first arena byte of the element, value slab chunk
    uint4 len;     // {ksrc16, ul, vl, n1 | n2 << 8}: key slab chunk (magic | user key | '$' | rev), lengths
    uint4 h1[2];   // bytes in front of the user key: [5a len] 12 len [0a len]   (n1 of them)
    uint4 h2[2];   // bytes between user key and value: [18 rev] [2a len]        (n2 of them)
};

struct WireOut {
    uint32_t *rec_idx;
    uint64_t *rev;
    uint64_t *key_off;
    uint32_t *key_len;
    uint64_t *val_off;
    uint32_t *val_len;
    uint64_t *elem_off;  // n_kvs + 1
};

__device__ __forceinline__ uint32_t put_varint(uint8_t *p, uint64_t v)
{
    uint32_t n = 0;
    while (v >= 0x80) {
        p[n++] = (uint8_t)(v | 0x80);
        v >>= 7;
    }
    p[n++] = (uint8_t)v;
    return n;
}

// the bytes in front of the user key and between the user key and the value
__device__ __forceinline__ void wire_headers(const WireSizes &s, int wire, uint8_t *h1, uint32_t &n1, uint8_t *h2,
                                             uint32_t &n2)
{
    n1 = 0;
    if (wire == KB_WIRE_EVENTS_I) {
        h1[n1++] = 0x5a;
        n1 += put_varint(h1 + n1, s.kv);
    }
    h1[n1++] = 0x12;
    n1 += put_varint(h1 + n1, s.body);
    if (s.ul) {
        h1[n1++] = 0x0a;
        n1 += put_varint(h1 + n1, s.ul);
    }
    n2 = 0;
    if (s.rev) {
        h2[n2++] = 0x18;
        n2 += put_varint(h2 + n2, s.rev);
    }
    if (s.vl) {
        h2[n2++] = 0x2a;
        n2 += put_varint(h2 + n2, s.vl);
    }
}

}  // namespace
