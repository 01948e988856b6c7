// kubebrain.hpp -- C++ host-side mirror of the reference's Go interfaces for the hot path, on top of the C ABI
// (include/kb_b200.h).  The reference is compiled Go and no Go toolchain exists in the build image, so this is the
// compiled-language host layer: same names, argument meaning and error behaviour as
//   coder.Coder          pkg/backend/coder/interface.go:18-28, normal.go:25-70, rev.go:22-47
//   scanner.Scanner      pkg/backend/scanner/interface.go:24-37
//   backend.Backend      pkg/backend/backend.go:44-84 (List / Count / ListByStream / Compact / compaction borders)
//   Ring                 pkg/backend/ring.go:24-118
// Header-only; link with -lkbb200.  Errors that the reference returns as `error` are thrown as kb::Error.
#pragma once

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <functional>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/kb_b200.h"

namespace kb {

using Bytes = std::string;  // byte strings

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string &m) : std::runtime_error(m), code(c) {}
};

// ---------------------------------------------------------------------------------------------------------
// coder
// ---------------------------------------------------------------------------------------------------------
struct NormalCoder {
    static constexpr const char *kMagic = "\x57\xfb\x80\x8b";  // normal.go:26
    static constexpr char kSplit = '$';                        // normal.go:31

    Bytes EncodeObjectKey(const Bytes &userKey, uint64_t revision) const
    {  // normal.go:42-50
        Bytes k(kMagic, 4);
        k += userKey;
        k.push_back(kSplit);
        for (int i = 7; i >= 0; i--) k.push_back((char)((revision >> (8 * i)) & 0xff));
        return k;
    }
    Bytes EncodeRevisionKey(const Bytes &userKey) const { return EncodeObjectKey(userKey, 0); }  // normal.go:53-55

    // normal.go:58-70; returns false (the reference returns an error) on bad magic / split byte / short key
    bool Decode(const Bytes &internalKey, Bytes *userKey, uint64_t *revision) const
    {
        if (internalKey.size() < 13) return false;  // Go would panic on the slice expressions
        if (std::memcmp(internalKey.data(), kMagic, 4) != 0) return false;
        if (internalKey[internalKey.size() - 9] != kSplit) return false;
        uint64_t r = 0;
        for (size_t i = internalKey.size() - 8; i < internalKey.size(); i++) r = (r << 8) | (uint8_t)internalKey[i];
        *revision = r;
        *userKey = internalKey.substr(4, internalKey.size() - 13);
        return true;
    }
};

// rev.go:32-47
inline bool ParseRevision(const Bytes &v, uint64_t *rev, bool *isTombstone)
{
    if (v.size() != 8 && v.size() != 9) return false;  // ErrInvalidRevFormat
    uint64_t r = 0;
    for (int i = 0; i < 8; i++) r = (r << 8) | (uint8_t)v[i];
    *rev = r;
    *isTombstone = v.size() == 9;
    return true;
}

// pkg/backend/util.go:70-83
inline Bytes PrefixEnd(const Bytes &prefix)
{
    Bytes end = prefix;
    for (size_t i = end.size(); i-- > 0;) {
        if ((uint8_t)end[i] < 0xff) {
            end[i] = (char)((uint8_t)end[i] + 1);
            end.resize(i + 1);
            return end;
        }
    }
    return Bytes(1, '\0');  // noPrefixEnd
}

// ---------------------------------------------------------------------------------------------------------
// Ring (pkg/backend/ring.go:24-118); T is the cached event type
// ---------------------------------------------------------------------------------------------------------
template <typename Event>
class Ring {
   public:
    explicit Ring(int l) : l_(l), arr_(l) {}
    void Add(const Event &e)
    {
        arr_[index(e_)] = e;
        if (e_ == s_ + l_) s_++;
        e_++;
    }
    int Size() const { return l_; }
    void Reset() { s_ = e_ = 0; }
    struct FindRet {
        bool empty = false, high = false, low = false;
        Event newest{}, oldest{};
        std::vector<Event> events;
    };
    // FindEvents: events from (inclusive) revision; Event must expose .Revision
    FindRet FindEvents(uint64_t revision) const
    {
        FindRet ret;
        if (e_ == 0) {
            ret.empty = true;
            return ret;
        }
        ret.newest = arr_[index(e_ - 1)];
        ret.oldest = arr_[index(s_)];
        if (revision > ret.newest.Revision) {
            ret.high = true;
            return ret;
        }
        if (revision < ret.oldest.Revision) {
            ret.low = true;
            return ret;
        }
        int64_t lo = 0, hi = e_ - s_;
        while (lo < hi) {  // sort.Search
            int64_t mid = lo + (hi - lo) / 2;
            if (arr_[index(s_ + mid)].Revision >= revision) hi = mid; else lo = mid + 1;
        }
        for (int64_t i = lo; i < e_ - s_; i++) ret.events.push_back(arr_[index(s_ + i)]);
        return ret;
    }

   private:
    int index(int64_t i) const { return (int)(i % l_); }
    int64_t s_ = 0, e_ = 0;
    int l_;
    std::vector<Event> arr_;
};

// ---------------------------------------------------------------------------------------------------------
// Engine / Scanner / Backend over the C ABI
// ---------------------------------------------------------------------------------------------------------
struct KeyValue {  // v2rpc.KeyValue
    Bytes Key, Value;
    uint64_t Revision = 0;
    bool operator==(const KeyValue &o) const { return Key == o.Key && Value == o.Value && Revision == o.Revision; }
};

class Engine {
   public:
    // flags: KB_CFG_* (KB_CFG_HOST_VALUES keeps the value heap in mapped pinned host memory)
    explicit Engine(int device = 0, uint32_t flags = 0)
    {
        const kb_config cfg{(uint32_t)sizeof(kb_config), flags};
        int rc = kb_open(device, &cfg, &ctx_);
        if (rc != KB_OK) throw Error(rc, "kb_open failed: no usable CUDA device (there is no CPU fallback)");
    }
    ~Engine() { kb_close(ctx_); }
    Engine(const Engine &) = delete;
    Engine &operator=(const Engine &) = delete;
    kb_ctx *ctx() const { return ctx_; }
    void Check(int rc) const
    {
        if (rc != KB_OK) throw Error(rc, kb_last_error(ctx_));
    }
    // items must be sorted by internal key (the storage.Iter contract)
    void LoadSorted(const std::vector<std::pair<Bytes, Bytes>> &items)
    {
        Bytes keys, vals;
        std::vector<uint64_t> ko{0}, vo{0};
        for (auto &kv : items) {
            keys += kv.first;
            vals += kv.second;
            ko.push_back(keys.size());
            vo.push_back(vals.size());
        }
        static const uint8_t z = 0;
        Check(kb_load_sorted(ctx_, keys.empty() ? &z : (const uint8_t *)keys.data(), ko.data(),
                             vals.empty() ? &z : (const uint8_t *)vals.data(), vo.data(), items.size()));
    }
    // snapshot file in device layout (restart without re-iterating the engine)
    void Dump(const std::string &path) { Check(kb_dump(ctx_, path.c_str())); }
    void Restore(const std::string &path) { Check(kb_restore(ctx_, path.c_str())); }
    // one committed storage.BatchWrite (pkg/storage/interface.go:62-84): Put / Del in order, last op on a key wins
    struct WriteOp {
        bool del;
        Bytes key, val;
    };
    void ApplyBatch(const std::vector<WriteOp> &ops)
    {
        std::vector<kb_write_op> raw(ops.size());
        for (size_t i = 0; i < ops.size(); i++) {
            raw[i].type = ops[i].del ? KB_OP_DEL : KB_OP_PUT;
            raw[i].key = (const uint8_t *)ops[i].key.data();
            raw[i].key_len = ops[i].key.size();
            raw[i].val = (const uint8_t *)ops[i].val.data();
            raw[i].val_len = ops[i].val.size();
        }
        Check(kb_apply_batch(ctx_, raw.data(), raw.size()));
    }

   private:
    kb_ctx *ctx_ = nullptr;
};

struct StreamRangeResponse {  // v2rpc.StreamRangeResponse
    uint64_t Revision = 0;
    std::vector<KeyValue> Kvs;
    bool More = false;
    std::string Err;
};

struct Victim {
    uint32_t Record;
    uint8_t Class;
};

// one delete call of a compaction sweep as the engine executes it: the internal key, and for classes 3 / 4 (DelCurrent)
// the value the sweep read -- delete only if the engine still holds it
struct VictimKey {
    Bytes Key, Guard;
    uint32_t Record;
    uint8_t Class;
};

class Scanner {  // scanner.Scanner
   public:
    static constexpr int kRangeStreamBatch = 300;  // scanner.go:43
    explicit Scanner(Engine &e) : e_(e) {}
    Engine &engine() { return e_; }

    std::vector<KeyValue> Range(const Bytes &start, const Bytes &end, uint64_t revision, int64_t limit)
    {  // scanner.go:83-119
        kb_range_req rq{(const uint8_t *)start.data(), start.size(), (const uint8_t *)end.data(), end.size(), revision, limit};
        kb_result *res = nullptr;
        e_.Check(kb_range_batch(e_.ctx(), &rq, 1, KB_OUT_HOST, &res));
        kb_range_view v;
        kb_range_view_get(res, &v);
        std::vector<KeyValue> out(v.n_kvs);
        for (uint64_t i = 0; i < v.n_kvs; i++) {
            out[i].Key.assign((const char *)v.bytes + v.key_off[i], v.key_len[i]);
            out[i].Value.assign((const char *)v.bytes + v.val_off[i], v.val_len[i]);
            out[i].Revision = v.rev[i];
        }
        kb_result_free(e_.ctx(), res);
        return out;
    }

    // The etcd-compatible answers, serialised: what backendShim.List (pkg/server/etcd/backendshim.go:269-282) hands to
    // gRPC as an etcdserverpb.RangeResponse; the kv elements are written by the device, only head and tail are added here.
    Bytes RangeResponseWire(const Bytes &start, const Bytes &end, uint64_t revision, int64_t limit, uint64_t headerRev,
                            bool more)
    {
        kb_range_req rq{(const uint8_t *)start.data(), start.size(), (const uint8_t *)end.data(), end.size(), revision, limit};
        kb_result *res = nullptr;
        e_.Check(kb_range_batch(e_.ctx(), &rq, 1, KB_OUT_HOST | KB_WIRE_ETCD_KVS, &res));
        kb_range_view v;
        kb_range_view_get(res, &v);
        uint8_t head[32], tail[32];
        const uint64_t nh = kb_wire_range_head(headerRev, head);
        const uint64_t nt = kb_wire_range_tail(more ? 1 : 0, (int64_t)v.n_kvs + (more ? 1 : 0), tail);
        Bytes out((const char *)head, nh);
        if (v.n_bytes) out.append((const char *)v.bytes, v.n_bytes);
        out.append((const char *)tail, nt);
        kb_result_free(e_.ctx(), res);
        return out;
    }

    // ... and the range stream (backendshim.go:329-368): one serialised etcdserverpb.WatchResponse per 300-kv batch
    // (header revision 0: forked receivers never get readRev, receiver.go:162-166), then the cancel message
    std::vector<Bytes> RangeStreamWire(const Bytes &start, const Bytes &end, uint64_t revision)
    {
        std::vector<Bytes> out;
        uint8_t head[64];
        kb_range_req rq{(const uint8_t *)start.data(), start.size(), (const uint8_t *)end.data(), end.size(), revision, 0};
        kb_result *res = nullptr;
        std::string err;
        int rc = kb_range_batch(e_.ctx(), &rq, 1, KB_OUT_HOST | KB_WIRE_ETCD_EVENTS, &res);
        if (rc != KB_OK) {
            err = kb_last_error(e_.ctx());
        } else {
            kb_range_view v;
            kb_range_view_get(res, &v);
            const uint64_t nh = kb_wire_watch_head(0, 0, nullptr, 0, head);
            for (uint64_t i = 0; i < v.n_kvs; i += kRangeStreamBatch) {
                const uint64_t j = std::min<uint64_t>(v.n_kvs, i + kRangeStreamBatch);
                Bytes m((const char *)head, nh);
                m.append((const char *)v.bytes + v.elem_off[i], v.elem_off[j] - v.elem_off[i]);
                out.push_back(std::move(m));
            }
            kb_result_free(e_.ctx(), res);
        }
        std::vector<uint8_t> endm(64 + err.size());
        const uint64_t ne = kb_wire_watch_head(revision, 1, (const uint8_t *)err.data(), err.size(), endm.data());
        out.emplace_back((const char *)endm.data(), ne);
        return out;
    }

    // f(view) for every page of one range stream; returns the error text of a failed open or next ("" when none)
    template <class F>
    std::string EachPage(const Bytes &start, const Bytes &end, uint64_t revision, int mode, uint64_t pageBytes, F &&f)
    {
        kb_range_req rq{(const uint8_t *)start.data(), start.size(), (const uint8_t *)end.data(), end.size(), revision, 0};
        kb_range_stream *s = nullptr;
        if (kb_range_stream_open(e_.ctx(), &rq, mode, kRangeStreamBatch, &s) != KB_OK) return kb_last_error(e_.ctx());
        std::string err;
        for (;;) {
            kb_result *page = nullptr;
            if (kb_range_stream_next(e_.ctx(), s, pageBytes, &page) != KB_OK) {
                err = kb_last_error(e_.ctx());
                break;
            }
            if (!page) break;
            kb_range_view v;
            kb_range_view_get(page, &v);
            f(v);
            kb_result_free(e_.ctx(), page);
        }
        kb_range_stream_close(e_.ctx(), s);
        return err;
    }

    int Count(const Bytes &start, const Bytes &end, uint64_t revision)
    {  // scanner.go:121-126
        kb_range_req rq{(const uint8_t *)start.data(), start.size(), (const uint8_t *)end.data(), end.size(), revision, 0};
        kb_result *res = nullptr;
        e_.Check(kb_range_batch(e_.ctx(), &rq, 1, KB_OUT_COUNT, &res));
        kb_range_view v;
        kb_range_view_get(res, &v);
        int c = (int)v.req_count[0];
        kb_result_free(e_.ctx(), res);
        return c;
    }

    // scanner.go:129-145: 300-kv batches with More=true, then the end marker.  The batches come from forked receivers
    // whose readRev is never set (receiver.go:162-166): their header revision is 0 (Q7).
    std::vector<StreamRangeResponse> RangeStream(const Bytes &start, const Bytes &end, uint64_t revision)
    {
        std::vector<StreamRangeResponse> out;
        StreamRangeResponse last;
        last.Revision = revision;
        try {
            auto kvs = Range(start, end, revision, 0);
            for (size_t i = 0; i < kvs.size(); i += kRangeStreamBatch) {
                StreamRangeResponse r;
                r.Revision = 0;
                r.More = true;
                r.Kvs.assign(kvs.begin() + i, kvs.begin() + std::min(kvs.size(), i + kRangeStreamBatch));
                out.push_back(std::move(r));
            }
        } catch (const Error &e) {
            last.Err = e.what();  // getListStreamEnd scanner.go:179-192
        }
        out.push_back(last);
        return out;
    }

    // RangeStream and RangeStreamWire with the answer fetched page by page (kb_range_stream_*): the same messages, while
    // no buffer holds more than one page of whole 300-kv batches within pageBytes
    static constexpr uint64_t kRangeStreamPageBytes = 64ull << 20;

    std::vector<StreamRangeResponse> RangeStreamPaged(const Bytes &start, const Bytes &end, uint64_t revision,
                                                      uint64_t pageBytes = kRangeStreamPageBytes)
    {
        std::vector<StreamRangeResponse> out;
        StreamRangeResponse last;
        last.Revision = revision;
        last.Err = EachPage(start, end, revision, KB_OUT_HOST, pageBytes, [&](const kb_range_view &v) {
            for (uint64_t i = 0; i < v.n_kvs; i += kRangeStreamBatch) {
                StreamRangeResponse r;
                r.More = true;
                for (uint64_t k = i; k < std::min<uint64_t>(v.n_kvs, i + kRangeStreamBatch); k++) {
                    KeyValue kv;
                    kv.Key.assign((const char *)v.bytes + v.key_off[k], v.key_len[k]);
                    kv.Value.assign((const char *)v.bytes + v.val_off[k], v.val_len[k]);
                    kv.Revision = v.rev[k];
                    r.Kvs.push_back(std::move(kv));
                }
                out.push_back(std::move(r));
            }
        });
        out.push_back(last);
        return out;
    }

    std::vector<Bytes> RangeStreamWirePaged(const Bytes &start, const Bytes &end, uint64_t revision,
                                            uint64_t pageBytes = kRangeStreamPageBytes)
    {
        std::vector<Bytes> out;
        uint8_t head[64];
        const uint64_t nh = kb_wire_watch_head(0, 0, nullptr, 0, head);
        const std::string err =
            EachPage(start, end, revision, KB_OUT_HOST | KB_WIRE_ETCD_EVENTS, pageBytes, [&](const kb_range_view &v) {
                for (uint64_t i = 0; i < v.n_kvs; i += kRangeStreamBatch) {
                    const uint64_t j = std::min<uint64_t>(v.n_kvs, i + kRangeStreamBatch);
                    Bytes m((const char *)head, nh);
                    m.append((const char *)v.bytes + v.elem_off[i], v.elem_off[j] - v.elem_off[i]);
                    out.push_back(std::move(m));
                }
            });
        std::vector<uint8_t> endm(64 + err.size());
        const uint64_t ne = kb_wire_watch_head(revision, 1, (const uint8_t *)err.data(), err.size(), endm.data());
        out.emplace_back((const char *)endm.data(), ne);
        return out;
    }

    // scanner.go:195-199 -> ordered delete calls; *count = worker.run's count
    std::vector<Victim> Compact(const Bytes &start, const Bytes &end, uint64_t revision, uint64_t timeoutRevision = 0,
                                bool supportTTL = true, uint64_t *count = nullptr)
    {
        kb_result *res = nullptr;
        e_.Check(kb_compact_sweep(e_.ctx(), (const uint8_t *)start.data(), start.size(), (const uint8_t *)end.data(),
                                  end.size(), revision, timeoutRevision, supportTTL ? 1 : 0, KB_OUT_HOST, &res));
        kb_compact_view v;
        kb_compact_view_get(res, &v);
        std::vector<Victim> out(v.n_victims);
        for (uint64_t i = 0; i < v.n_victims; i++) out[i] = Victim{v.victim_idx[i], v.victim_class[i]};
        if (count) *count = v.count;
        kb_result_free(e_.ctx(), res);
        return out;
    }

    // Compact's delete calls as keys (+ guards), page by page (kb_compact_stream_*): apply(page) gets each page of whole
    // groups of `group` victims within pageBytes arena bytes and may commit its deletes before the next page is made.
    // *count = worker.run's count.
    void CompactPaged(const Bytes &start, const Bytes &end, uint64_t revision,
                      const std::function<void(const std::vector<VictimKey> &)> &apply, uint64_t timeoutRevision = 0,
                      bool supportTTL = true, uint64_t pageBytes = 64ull << 20, uint64_t group = 1024,
                      uint64_t *count = nullptr)
    {
        kb_compact_stream *cs = nullptr;
        e_.Check(kb_compact_stream_open(e_.ctx(), (const uint8_t *)start.data(), start.size(), (const uint8_t *)end.data(),
                                        end.size(), revision, timeoutRevision, supportTTL ? 1 : 0, group, &cs));
        if (count) kb_compact_stream_info(cs, nullptr, count, nullptr);
        struct Closer {
            kb_ctx *ctx;
            kb_compact_stream *s;
            ~Closer() { kb_compact_stream_close(ctx, s); }
        } closer{e_.ctx(), cs};
        for (;;) {
            kb_result *page = nullptr;
            e_.Check(kb_compact_stream_next(e_.ctx(), cs, pageBytes, &page));
            if (!page) return;
            kb_compact_page_view v;
            kb_compact_page_view_get(page, &v);
            std::vector<VictimKey> out(v.n);
            for (uint64_t i = 0; i < v.n; i++)
                out[i] = VictimKey{Bytes((const char *)v.bytes + v.key_off[i], v.key_len[i]),
                                   Bytes((const char *)v.bytes + v.guard_off[i], v.guard_len[i]), v.rec_idx[i],
                                   v.victim_class[i]};
            kb_result_free(e_.ctx(), page);
            apply(out);
        }
    }

   private:
    Engine &e_;
};

struct RangeResponse {
    uint64_t Revision = 0;
    std::vector<KeyValue> Kvs;
    bool More = false;
};

class Backend {  // the read half of backend.Backend
   public:
    // partition_bytes == 0: GetPartitions returns the interval whole; > 0: it cuts the interval on the device into at most
    // max_partitions partitions of about partition_bytes answer bytes each
    Backend(Engine &e, std::string prefix, std::vector<std::string> skipped = {}, uint64_t partition_bytes = 0,
            uint64_t max_partitions = 64)
        : scanner_(e), prefix_(std::move(prefix)), skipped_(std::move(skipped)), partition_bytes_(partition_bytes),
          max_partitions_(max_partitions)
    {
    }
    uint64_t GetCurrentRevision() const { return rev_; }
    void SetCurrentRevision(uint64_t r) { rev_ = r; }

    // range.go:34-81 Backend.Get: *found=false for a missing key, a key created after `revision`, or a deleted key
    uint64_t Get(const Bytes &key, uint64_t revision, KeyValue *kv, bool *found)
    {
        kb_get_req rq{(const uint8_t *)key.data(), key.size(), revision};
        kb_result *res = nullptr;
        scanner_.engine().Check(kb_get_batch(scanner_.engine().ctx(), &rq, 1, KB_OUT_HOST, &res));
        kb_get_view v;
        kb_get_view_get(res, &v);
        uint64_t cur = rev_;
        *found = v.status[0] == KB_GET_FOUND;
        if (*found) {
            kv->Key = key;
            kv->Value.assign((const char *)v.bytes + v.val_off[0], v.val_len[0]);
            kv->Revision = v.mod_rev[0];
            if (v.mod_rev[0] > cur) cur = v.mod_rev[0];
        }
        kb_result_free(scanner_.engine().ctx(), res);
        return cur;
    }

    // backendShim.Get's answer, serialised (backendshim.go:235-254): the RangeResponse with the read's kv element, written
    // by the device, or none for a missing / deleted key; header revision = max(current, mod_revision) when found
    Bytes GetResponseWire(const Bytes &key, uint64_t revision)
    {
        kb_get_req rq{(const uint8_t *)key.data(), key.size(), revision};
        kb_pending *p = nullptr;
        kb_result *res = nullptr;
        kb_ctx *ctx = scanner_.engine().ctx();
        scanner_.engine().Check(kb_get_submit(ctx, &rq, 1, KB_OUT_HOST | KB_WIRE_ETCD_KVS, &p));
        scanner_.engine().Check(kb_get_collect(ctx, p, &res));
        kb_get_view v;
        const uint64_t *eo = nullptr;
        kb_get_view_get(res, &v);
        kb_get_elem_off(res, &eo);
        const bool found = v.status[0] == KB_GET_FOUND;
        uint8_t head[32], tail[32];
        const uint64_t nh = kb_wire_range_head(found && v.mod_rev[0] > rev_ ? v.mod_rev[0] : rev_, head);
        const uint64_t nt = kb_wire_range_tail(0, found ? 1 : 0, tail);
        Bytes out((const char *)head, nh);
        if (found) out.append((const char *)v.bytes + eo[0], eo[1] - eo[0]);
        out.append((const char *)tail, nt);
        kb_result_free(ctx, res);
        return out;
    }

    // Get of many (key, revision) reads in one batch: one answer per read, in order (Found = false for a missing key, a
    // key created after the revision, or a deleted key)
    struct GetAnswer {
        bool Found = false;
        KeyValue Kv;
    };
    std::vector<GetAnswer> GetMany(const std::vector<std::pair<Bytes, uint64_t>> &reads)
    {
        std::vector<kb_get_req> rq(reads.size());
        for (size_t i = 0; i < reads.size(); i++)
            rq[i] = kb_get_req{(const uint8_t *)reads[i].first.data(), reads[i].first.size(), reads[i].second};
        kb_result *res = nullptr;
        scanner_.engine().Check(kb_get_batch(scanner_.engine().ctx(), rq.data(), rq.size(), KB_OUT_HOST, &res));
        kb_get_view v;
        kb_get_view_get(res, &v);
        std::vector<GetAnswer> out(reads.size());
        for (size_t i = 0; i < reads.size(); i++) {
            if (v.status[i] != KB_GET_FOUND) continue;
            out[i].Found = true;
            out[i].Kv.Key = reads[i].first;
            out[i].Kv.Value.assign((const char *)v.bytes + v.val_off[i], v.val_len[i]);
            out[i].Kv.Revision = v.mod_rev[i];
        }
        kb_result_free(scanner_.engine().ctx(), res);
        return out;
    }

    RangeResponse List(const Bytes &key, const Bytes &end, uint64_t revision = 0, int64_t limit = 0)
    {  // range.go:124-174
        if (end.empty()) throw Error(KB_EINVAL, "invalid nil end field in RangeRequest");
        const uint64_t cur = rev_;
        const uint64_t req = revision ? revision : cur;
        if (key >= end) throw Error(KB_EINVAL, "invalid range end");
        const int64_t lim = limit > 0 ? limit + 1 : limit;  // one more to learn whether there is more
        RangeResponse resp;
        resp.Revision = cur;
        resp.Kvs = scanner_.Range(coder_.EncodeObjectKey(key, 0), coder_.EncodeObjectKey(end, 0), req, lim);
        if (lim > 0 && (int64_t)resp.Kvs.size() > limit) {
            resp.More = true;
            resp.Kvs.resize(limit);
        }
        return resp;
    }
    uint64_t Count(const Bytes &key, const Bytes &end)
    {  // range.go:177-205
        return (uint64_t)scanner_.Count(coder_.EncodeObjectKey(key, 0), coder_.EncodeObjectKey(end, 0), rev_);
    }
    std::vector<StreamRangeResponse> ListByStream(const Bytes &startKey, const Bytes &endKey, uint64_t rev = 0)
    {  // range.go:247-256
        return scanner_.RangeStream(startKey, endKey, rev ? rev : rev_);
    }
    // range.go:208-244: the borders clients open one ListByStream each over (partitions + 1 of them).  The inner borders are
    // revision-record keys cut at the latest revision (kb_range_partitions).
    std::vector<Bytes> GetPartitions(const Bytes &key, const Bytes &end)
    {
        Bytes start = coder_.EncodeObjectKey(key, 0), stop = coder_.EncodeObjectKey(end, 0);
        if (partition_bytes_ == 0) return {start, stop};
        kb_range_req rq{(const uint8_t *)start.data(), start.size(), (const uint8_t *)stop.data(), stop.size(), ~0ull, 0};
        kb_result *res = nullptr;
        kb_ctx *ctx = scanner_.engine().ctx();
        scanner_.engine().Check(kb_range_partitions(ctx, &rq, partition_bytes_, max_partitions_, &res));
        kb_partition_view v;
        kb_partition_view_get(res, &v);
        std::vector<Bytes> borders;
        for (uint64_t k = 0; k <= v.n_parts; k++)
            borders.emplace_back((const char *)v.bytes + v.key_off[k], v.key_off[k + 1] - v.key_off[k]);
        kb_result_free(ctx, res);
        return borders;
    }
    std::vector<Bytes> GetCompactBorders() const
    {  // compact.go:107-127
        std::vector<Bytes> borders;
        std::vector<std::string> all{prefix_};
        all.insert(all.end(), skipped_.begin(), skipped_.end());
        for (auto key : all) {
            if (key.empty() || key.back() != '/') key += "/";
            borders.push_back(coder_.EncodeObjectKey(key, 0));
            borders.push_back(coder_.EncodeObjectKey(PrefixEnd(key), 0));
        }
        std::sort(borders.begin(), borders.end());
        return borders;
    }
    std::vector<std::vector<Victim>> Compact(uint64_t revision)
    {  // compact.go:31-68
        if (revision == 0 || revision > rev_) revision = rev_;
        auto borders = GetCompactBorders();
        std::vector<std::vector<Victim>> out;
        for (size_t i = 0; i + 1 < borders.size(); i += 2) out.push_back(scanner_.Compact(borders[i], borders[i + 1], revision));
        return out;
    }

   private:
    Scanner scanner_;
    NormalCoder coder_;
    std::string prefix_;
    std::vector<std::string> skipped_;
    uint64_t partition_bytes_, max_partitions_;
    uint64_t rev_ = 0;
};

}  // namespace kb
