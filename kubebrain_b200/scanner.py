"""Host-side mirror of scanner.Scanner (pkg/backend/scanner/interface.go:24-37) on top of the C ABI.

Same method names and argument meaning as the reference: Range / RangeStream / Count / Compact take INTERNAL
keys (coder.EncodeObjectKey(key, 0)); the work runs in libkbb200.so (kb_range_batch / kb_compact_sweep).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Iterator, List, Sequence, Tuple

from ._lib import KB_OUT_COUNT, KB_OUT_HOST, CompactPage, CompactResult, Engine

RANGE_STREAM_BATCH = 300  # scanner.go:43
RANGE_STREAM_PAGE_BYTES = 64 << 20  # arena bytes per page of range_stream_paged
COMPACT_PAGE_BYTES = 64 << 20  # arena bytes per page of compact_pages
COMPACT_GROUP = 1024  # victims per group of compact_pages (one engine batch each)


@dataclass
class KeyValue:  # v2rpc.KeyValue
    key: bytes
    value: bytes
    revision: int


@dataclass
class StreamRangeResponse:  # v2rpc.StreamRangeResponse (receiver.go:129-136, scanner.go:179-192)
    revision: int
    kvs: List[KeyValue]
    more: bool
    err: str = ""


class Scanner:
    def __init__(self, engine: Engine):
        self.engine = engine

    def range(self, start: bytes, end: bytes, revision: int, limit: int) -> List[KeyValue]:
        """scanner.go:83-119"""
        res = self.engine.range_batch([(start, end, revision, limit)], KB_OUT_HOST)
        try:
            return [KeyValue(k, v, r) for k, v, r in res.kvs(0)]
        finally:
            res.close()

    def range_many(self, reqs: Sequence[Tuple[bytes, bytes, int, int]]) -> List[List[KeyValue]]:
        """a batch of independent Range calls answered by one launch sequence"""
        res = self.engine.range_batch(list(reqs), KB_OUT_HOST)
        try:
            return [[KeyValue(k, v, r) for k, v, r in res.kvs(q)] for q in range(len(reqs))]
        finally:
            res.close()

    def count(self, start: bytes, end: bytes, revision: int) -> int:
        """scanner.go:121-126"""
        res = self.engine.range_batch([(start, end, revision, 0)], KB_OUT_COUNT)
        try:
            return int(res.req_count[0])
        finally:
            res.close()

    def range_stream(self, start: bytes, end: bytes, revision: int) -> Iterator[StreamRangeResponse]:
        """scanner.go:129-145: batches of 300 kvs with More=true, then the end marker (More=false).  Q7: the batches are
        sent by *forked* receivers, and fork() does not copy readRev (receiver.go:162-166), so their header revision
        is 0; only the end marker (getListStreamEnd, scanner.go:179-192) carries the read revision."""
        try:
            kvs = self.range(start, end, revision, 0)
        except Exception as e:  # getListStreamEnd carries the error text (scanner.go:179-192)
            yield StreamRangeResponse(revision, [], False, str(e))
            return
        for i in range(0, len(kvs), RANGE_STREAM_BATCH):
            yield StreamRangeResponse(0, kvs[i : i + RANGE_STREAM_BATCH], True)
        yield StreamRangeResponse(revision, [], False)

    def range_stream_paged(self, start: bytes, end: bytes, revision: int,
                           page_bytes: int = RANGE_STREAM_PAGE_BYTES) -> Iterator[StreamRangeResponse]:
        """range_stream's messages, with the answer fetched in pages of whole 300-kv batches of at most page_bytes arena
        bytes (kb_range_stream_open / _next): memory follows the page, not the answer"""
        try:
            stream = self.engine.range_stream((start, end, revision, 0), KB_OUT_HOST, RANGE_STREAM_BATCH)
        except Exception as e:
            yield StreamRangeResponse(revision, [], False, str(e))
            return
        try:
            while True:
                try:
                    page = stream.next(page_bytes)
                except Exception as e:
                    yield StreamRangeResponse(revision, [], False, str(e))
                    return
                if page is None:
                    break
                try:
                    kvs = [KeyValue(k, v, r) for k, v, r in page.kvs(0)]
                finally:
                    page.close()
                for i in range(0, len(kvs), RANGE_STREAM_BATCH):  # a page holds whole batches but for the last one
                    yield StreamRangeResponse(0, kvs[i : i + RANGE_STREAM_BATCH], True)
        finally:
            stream.close()
        yield StreamRangeResponse(revision, [], False)

    def compact(self, start: bytes, end: bytes, revision: int, timeout_revision: int = 0,
                support_ttl: bool = True) -> CompactResult:
        """scanner.go:195-199: classify the victims of [start,end) at `revision`; the caller applies the deletes in
        bulk (the reference issues one storage transaction per victim, scanner.go:538-564)"""
        return self.engine.compact_sweep(start, end, revision, timeout_revision, support_ttl, KB_OUT_HOST)

    def compact_pages(self, start: bytes, end: bytes, revision: int, timeout_revision: int = 0, support_ttl: bool = True,
                      page_bytes: int = COMPACT_PAGE_BYTES, group: int = COMPACT_GROUP) -> Iterator[CompactPage]:
        """compact()'s victims as the keys the engine deletes (kb_compact_stream_open / _next): pages of whole groups of
        `group` victims within page_bytes arena bytes, each with the internal key of every delete call and, for classes
        3 / 4, the value the sweep read.  The caller may commit a page's deletes before it asks for the next one."""
        stream = self.engine.compact_stream(start, end, revision, timeout_revision, support_ttl, group)
        try:
            while True:
                page = stream.next(page_bytes)
                if page is None:
                    return
                yield page
        finally:
            stream.close()
