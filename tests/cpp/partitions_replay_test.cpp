// partitions_replay_test.cpp -- replays, call for call, what a client of the Go storage adaptor's GetPartitions does
// through the C ABI (go/pkg/storage/b200/storage.go GetPartitions -> kb.go Engine.Partitions, then one ListByStream per
// partition, backend_test.go:508-533 -> kb.go rangePages), and checks the concatenated answer against the CPU oracle
// (oracle/libkboracle.so):
//   kb_range_partitions(start, end, read_rev = 2^64-1, PartitionBytes, MaxPartitions) -> borders, kb_result_free
//   per partition: kb_range_stream_open(KB_OUT_HOST, 300), kb_range_stream_next(64 MiB) until NULL, _close
// The partitions are cut at the latest revision and streamed at the backend's read revision; a commit above the read
// revision between the cut and the streams leaves the answer whole.
// usage: partitions_replay_test   (needs a CUDA device; tests/test_gpu_partitions.py builds and runs it)
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/kb_b200.h"
#include "../../oracle/kb_oracle.h"

#define CHECK(c)                                                                                         \
    do {                                                                                                 \
        if (!(c)) {                                                                                      \
            std::printf("FAIL %s:%d: %s  [%s]\n", __FILE__, __LINE__, #c, ctx ? kb_last_error(ctx) : ""); \
            std::exit(1);                                                                                \
        }                                                                                                \
    } while (0)

typedef std::string Bytes;
static kb_ctx *ctx = nullptr;

static const uint64_t kBatch = 300;             // rangeStreamBatch
static const uint64_t kPageBytes = 64ull << 20;  // rangeStreamPageBytes

static Bytes be64(uint64_t v)
{
    Bytes b(8, '\0');
    for (int i = 0; i < 8; i++) b[i] = (char)(v >> (8 * (7 - i)));
    return b;
}
static Bytes ikey(const Bytes &uk, uint64_t rev) { return Bytes("\x57\xfb\x80\x8b", 4) + uk + "$" + be64(rev); }

struct KV {
    Bytes key, val;
    uint64_t rev;
    bool operator==(const KV &o) const { return key == o.key && val == o.val && rev == o.rev; }
};

// kb.go Engine.Partitions
static std::vector<Bytes> partitions(const Bytes &s, const Bytes &t, uint64_t part_bytes, uint64_t max_parts)
{
    kb_range_req rq{(const uint8_t *)s.data(), s.size(), (const uint8_t *)t.data(), t.size(), ~0ull, 0};
    kb_result *res = nullptr;
    CHECK(kb_range_partitions(ctx, &rq, part_bytes, max_parts, &res) == KB_OK);
    kb_partition_view v;
    CHECK(kb_partition_view_get(res, &v) == KB_OK);
    kb_range_view rv;
    CHECK(kb_range_view_get(res, &rv) == KB_EINVAL);
    CHECK(kb_result_wait(ctx, res, nullptr) == KB_OK);
    std::vector<Bytes> borders;
    for (uint64_t k = 0; k <= v.n_parts; k++) borders.emplace_back((const char *)v.bytes + v.key_off[k], v.key_off[k + 1] - v.key_off[k]);
    kb_result_free(ctx, res);
    return borders;
}

// kb.go rangePages: the kvs of one ListByStream
static std::vector<KV> stream(const Bytes &s, const Bytes &t, uint64_t revision)
{
    kb_range_req rq{(const uint8_t *)s.data(), s.size(), (const uint8_t *)t.data(), t.size(), revision, 0};
    kb_range_stream *rs = nullptr;
    CHECK(kb_range_stream_open(ctx, &rq, KB_OUT_HOST, kBatch, &rs) == KB_OK);
    std::vector<KV> kvs;
    for (;;) {
        kb_result *page = nullptr;
        CHECK(kb_range_stream_next(ctx, rs, kPageBytes, &page) == KB_OK);
        if (!page) break;
        kb_range_view v;
        CHECK(kb_range_view_get(page, &v) == KB_OK);
        kb_partition_view pv;
        CHECK(kb_partition_view_get(page, &pv) == KB_EINVAL);
        for (uint64_t k = 0; k < v.n_kvs; k++)
            kvs.push_back(KV{Bytes((const char *)v.bytes + v.key_off[k], v.key_len[k]),
                             Bytes((const char *)v.bytes + v.val_off[k], v.val_len[k]), v.rev[k]});
        kb_result_free(ctx, page);
    }
    kb_range_stream_close(ctx, rs);
    return kvs;
}

static std::map<Bytes, Bytes> kv;

struct Packed {
    std::vector<uint8_t> keys, vals;
    std::vector<uint64_t> koff{0}, voff{0};
    ko_store view() const { return ko_store{keys.data(), koff.data(), vals.data(), voff.data(), koff.size() - 1}; }
};

static Packed pack()
{
    Packed p;
    for (auto &it : kv) {
        p.keys.insert(p.keys.end(), it.first.begin(), it.first.end());
        p.vals.insert(p.vals.end(), it.second.begin(), it.second.end());
        p.koff.push_back(p.keys.size());
        p.voff.push_back(p.vals.size());
    }
    return p;
}

static std::vector<KV> want(const Bytes &s, const Bytes &t, uint64_t revision)
{
    const Packed p = pack();
    const ko_store st = p.view();
    ko_result r;
    ko_result_init(&r);
    CHECK(ko_range(&st, (const uint8_t *)s.data(), s.size(), (const uint8_t *)t.data(), t.size(), revision, 0, 0, 0, &r) == 0);
    std::vector<KV> kvs;
    for (uint64_t i = 0; i < r.n_emit; i++) {
        const uint64_t rec = r.emit[i];
        const Bytes k((const char *)p.keys.data() + p.koff[rec], p.koff[rec + 1] - p.koff[rec]);
        uint64_t rev = 0;
        for (int b = 0; b < 8; b++) rev = (rev << 8) | (uint8_t)k[k.size() - 8 + b];
        kvs.push_back(KV{k.substr(4, k.size() - 13), Bytes((const char *)p.vals.data() + p.voff[rec], p.voff[rec + 1] - p.voff[rec]),
                         rev});
    }
    ko_result_free(&r);
    return kvs;
}

static void load()
{
    const Packed p = pack();
    CHECK(kb_load_sorted(ctx, p.keys.data(), p.koff.data(), p.vals.data(), p.voff.data(), p.koff.size() - 1) == KB_OK);
}

int main()
{
    CHECK(kb_open(0, nullptr, &ctx) == KB_OK);
    // 12 000 objects with ~2 KiB values in two versions and a revision record (~25 MB of answer)
    const uint64_t read_rev = 5000;
    for (int j = 0; j < 12000; j++) {
        char uk[64];
        std::snprintf(uk, sizeof uk, "/registry/pods/ns-%03d/pod-%06d", j % 97, j);
        const uint64_t r1 = 100 + j % 1000, r2 = 2000 + j % 2000;
        kv[ikey(uk, 0)] = be64(r2);
        kv[ikey(uk, r1)] = Bytes(2000 + j % 33, (char)('a' + j % 26));
        kv[ikey(uk, r2)] = Bytes(2048 + j % 17, (char)('A' + j % 26));
    }
    load();
    const Bytes s = ikey("/registry/", 0), t = ikey("/registry0", 0);
    const std::vector<KV> exp = want(s, t, read_rev);
    CHECK(exp.size() == 12000);

    // MaxPartitions = 64, PartitionBytes = 4 MiB: ceil(25 MB / 4 MiB) partitions
    std::vector<Bytes> b = partitions(s, t, 4ull << 20, 64);
    CHECK(b.size() >= 6 && b.size() <= 9 && b.front() == s && b.back() == t);
    std::vector<KV> got;
    for (size_t i = 1; i < b.size(); i++) {
        CHECK(b[i - 1] < b[i]);
        const std::vector<KV> part = stream(b[i - 1], b[i], read_rev);
        CHECK(!part.empty());
        got.insert(got.end(), part.begin(), part.end());
    }
    CHECK(got == exp);

    // a commit above the read revision between the cut and the streams: new versions, new keys
    b = partitions(s, t, 1ull << 20, 16);
    CHECK(b.size() == 17);
    std::vector<kb_write_op> ops;
    std::vector<Bytes> keep;
    for (int j = 0; j < 12000; j += 5) {
        char uk[64];
        std::snprintf(uk, sizeof uk, "/registry/pods/ns-%03d/pod-%06d", j % 97, j);
        keep.push_back(ikey(uk, read_rev + 1 + j));
        keep.push_back(ikey(Bytes(uk) + "x", read_rev + 1 + j));
    }
    const Bytes nv(100, 'n');
    for (const Bytes &k : keep) {
        kb_write_op op;
        memset(&op, 0, sizeof op);
        op.type = KB_OP_PUT;
        op.key = (const uint8_t *)k.data();
        op.key_len = k.size();
        op.val = (const uint8_t *)nv.data();
        op.val_len = nv.size();
        ops.push_back(op);
        kv[k] = nv;
    }
    CHECK(kb_apply_batch(ctx, ops.data(), ops.size()) == KB_OK);
    got.clear();
    for (size_t i = 1; i < b.size(); i++) {
        const std::vector<KV> part = stream(b[i - 1], b[i], read_rev);
        got.insert(got.end(), part.begin(), part.end());
    }
    CHECK(got == exp && want(s, t, read_rev) == exp);

    // the default of the adaptor, and an empty interval: one partition, the interval itself
    b = partitions(s, s, 1ull << 20, 64);
    CHECK(b.size() == 2 && b[0] == s && b[1] == s);
    kb_close(ctx);
    ctx = nullptr;
    std::printf("partitions replay OK\n");
    return 0;
}
