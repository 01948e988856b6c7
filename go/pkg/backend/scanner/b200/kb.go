//go:build b200

// Package b200 binds libkbb200.so (include/kb_b200.h) under the reference's scanner.Scanner seam
// (pkg/backend/scanner/interface.go:24-37) and exposes the watch matcher used by the backend's hub.
//
// NOTE: written without a Go toolchain (none exists in the build image); it is the binding a maintainer
// adds to the kubebrain tree next to pkg/backend/scanner.  Every behaviour it relies on is exercised
// through the same C ABI by tests/test_gpu_parity.py.
package b200

/*
#cgo CFLAGS: -I${SRCDIR}/../../../../../include
#cgo LDFLAGS: -L${SRCDIR}/../../../../../kubebrain_b200 -lkbb200 -Wl,-rpath,${SRCDIR}/../../../../../kubebrain_b200
#include <stdlib.h>
#include "kb_b200.h"
*/
import "C"

import (
	"context"
	"errors"
	"fmt"
	"runtime"
	"sync"
	"time"
	"unsafe"

	proto "github.com/kubewharf/kubebrain-client/api/v2rpc"

	"github.com/kubewharf/kubebrain/pkg/backend/scanner"
	"github.com/kubewharf/kubebrain/pkg/storage"
)

const rangeStreamBatch = 300 // pkg/backend/scanner/scanner.go:43

// Engine owns one kb_ctx (one GPU, one HBM-resident snapshot).
type Engine struct {
	mu  sync.Mutex
	ctx *C.kb_ctx
}

func Open(device int) (*Engine, error) {
	e := &Engine{}
	if rc := C.kb_open(C.int(device), nil, &e.ctx); rc != 0 {
		return nil, fmt.Errorf("kb_open: %d (no CUDA device; there is no CPU fallback)", int(rc))
	}
	runtime.SetFinalizer(e, func(e *Engine) { C.kb_close(e.ctx) })
	return e, nil
}

func (e *Engine) err(rc C.int) error {
	if rc == 0 {
		return nil
	}
	return fmt.Errorf("kb_b200 %d: %s", int(rc), C.GoString(C.kb_last_error(e.ctx)))
}

// ptr8 / ptr64: the address of a slice's first element, or nil for an empty slice (&x[0] panics on those)
func ptr8(b []byte) *C.uint8_t {
	if len(b) == 0 {
		return nil
	}
	return (*C.uint8_t)(unsafe.Pointer(&b[0]))
}

func ptr64(b []uint64) *C.uint64_t {
	if len(b) == 0 {
		return nil
	}
	return (*C.uint64_t)(unsafe.Pointer(&b[0]))
}

// Close releases the context; the Engine must not be used afterwards.
func (e *Engine) Close() {
	e.mu.Lock()
	defer e.mu.Unlock()
	if e.ctx != nil {
		C.kb_close(e.ctx)
		e.ctx = nil
		runtime.SetFinalizer(e, nil)
	}
}

// LoadSorted ingests a snapshot pulled from storage.Iter (ascending unique internal keys).  An empty engine
// (len(keyOff) <= 1) loads an empty snapshot.
func (e *Engine) LoadSorted(keys []byte, keyOff []uint64, vals []byte, valOff []uint64) error {
	n := 0
	if len(keyOff) > 1 {
		n = len(keyOff) - 1
	}
	zero := []uint64{0}
	if n == 0 {
		keyOff, valOff = zero, zero
	}
	e.mu.Lock()
	defer e.mu.Unlock()
	return e.err(C.kb_load_sorted(e.ctx, ptr8(keys), ptr64(keyOff), ptr8(vals), ptr64(valOff), C.uint64_t(n)))
}

// Expire drops every TTL'd record whose time has come from the mirror (kb_expire); returns how many.
func (e *Engine) Expire(nowUnix uint64) (uint64, error) {
	var n C.uint64_t
	e.mu.Lock()
	defer e.mu.Unlock()
	rc := C.kb_expire(e.ctx, C.uint64_t(nowUnix), &n)
	return uint64(n), e.err(rc)
}

// Dump / Restore persist the HBM snapshot (device layout, checksummed) so a restart need not re-iterate the engine.
func (e *Engine) Dump(path string) error {
	cs := C.CString(path)
	defer C.free(unsafe.Pointer(cs))
	return e.err(C.kb_dump(e.ctx, cs))
}

func (e *Engine) Restore(path string) error {
	cs := C.CString(path)
	defer C.free(unsafe.Pointer(cs))
	return e.err(C.kb_restore(e.ctx, cs))
}

// WriteOp mirrors one Put/Del of a committed storage.BatchWrite (pkg/storage/interface.go:62-84).
type WriteOp struct {
	Del        bool
	Key, Val   []byte
	ExpireUnix uint64 // puts with a ttl: wall-clock second at which the engine stops returning the key (0: never)
}

// ApplyBatch merges a committed batch into the HBM snapshot; the storage adaptor calls it after Commit succeeds.
func (e *Engine) ApplyBatch(ops []WriteOp) error {
	if len(ops) == 0 {
		return nil
	}
	raw := make([]C.kb_write_op, len(ops))
	pin := runtime.Pinner{}
	defer pin.Unpin()
	for i := range ops {
		if ops[i].Del {
			raw[i]._type = C.KB_OP_DEL
		} else {
			raw[i]._type = C.KB_OP_PUT
		}
		if len(ops[i].Key) > 0 {
			pin.Pin(&ops[i].Key[0])
			raw[i].key = (*C.uint8_t)(unsafe.Pointer(&ops[i].Key[0]))
		}
		raw[i].key_len = C.uint64_t(len(ops[i].Key))
		if len(ops[i].Val) > 0 {
			pin.Pin(&ops[i].Val[0])
			raw[i].val = (*C.uint8_t)(unsafe.Pointer(&ops[i].Val[0]))
		}
		raw[i].val_len = C.uint64_t(len(ops[i].Val))
		raw[i].expire_unix = C.uint64_t(ops[i].ExpireUnix)
	}
	e.mu.Lock()
	defer e.mu.Unlock()
	return e.err(C.kb_apply_batch(e.ctx, &raw[0], C.uint64_t(len(raw))))
}

// Metrics is the subset of pkg/metrics.Metrics the hot path emits (scanner.go:512-514, watcherhub.go:87).
type Metrics interface {
	EmitHistogram(name string, value interface{}, tags ...string) error
	EmitCounter(name string, value interface{}, tags ...string) error
}

type b200Scanner struct {
	e          *Engine
	SupportTTL bool          // storage.KvStorage.SupportTTL() of the wrapped engine
	TTL        time.Duration // scanner.Config.TTL (scanner.go:78-79)
	metricCli  Metrics

	histMu           sync.Mutex
	compactHistories []compactRecord
}

// NewScanner replaces scanner.NewScanner at pkg/backend/backend.go:155.
func NewScanner(e *Engine, supportTTL bool, ttl time.Duration, m Metrics) scanner.Scanner {
	return &b200Scanner{e: e, SupportTTL: supportTTL, TTL: ttl, metricCli: m}
}

// emitScanMetrics: the three histograms worker.run emits when it finishes (scanner.go:512-514)
func (s *b200Scanner) emitScanMetrics(latency time.Duration, valSize int, count int) {
	if s.metricCli == nil {
		return
	}
	_ = s.metricCli.EmitHistogram("storage.scan_worker.latency", latency.Seconds())
	_ = s.metricCli.EmitHistogram("storage.scan_worker.size", valSize)
	_ = s.metricCli.EmitHistogram("storage.scan_worker.count", count)
}

func (s *b200Scanner) rangeOnce(start, end []byte, revision uint64, limit int64, mode C.int) (*C.kb_result, C.kb_range_view, error) {
	var req C.kb_range_req
	pin := runtime.Pinner{}
	defer pin.Unpin()
	if len(start) > 0 {
		pin.Pin(&start[0])
		req.start = (*C.uint8_t)(unsafe.Pointer(&start[0]))
	}
	if len(end) > 0 {
		pin.Pin(&end[0])
		req.end = (*C.uint8_t)(unsafe.Pointer(&end[0]))
	}
	req.start_len, req.end_len = C.uint64_t(len(start)), C.uint64_t(len(end))
	req.read_rev, req.limit = C.uint64_t(revision), C.int64_t(limit)
	var res *C.kb_result
	var view C.kb_range_view
	// Two critical sections instead of one kb_range_batch: between them another goroutine's Range can submit, so two
	// scans are in flight on the device (the second one's bound search and layout overlap the first one's kernels; a
	// third submission first reads back the first one's rows).  The bound keys are only read by the submission.
	var pend *C.kb_pending
	s.e.mu.Lock()
	rc := C.kb_range_submit(s.e.ctx, &req, 1, mode, &pend)
	err := s.e.err(rc) // KB_ECOMPACTED carries the reference's message (scanner.go:620-623)
	s.e.mu.Unlock()
	if err != nil {
		return nil, view, err
	}
	s.e.mu.Lock()
	rc = C.kb_range_collect(s.e.ctx, pend, &res) // ends the pending on success and on failure
	err = s.e.err(rc)
	s.e.mu.Unlock()
	if err != nil {
		return nil, view, err
	}
	C.kb_range_view_get(res, &view)
	return res, view, nil
}

// copyKvs moves the pinned result arena into Go-owned memory: the reference keeps Key/Val slices alive after
// Iter.Close (scanner.go:493-495), so the arena cannot be handed out directly unless it is ref-counted.
func copyKvs(view C.kb_range_view) []*proto.KeyValue {
	n := int(view.n_kvs)
	if n == 0 {
		return nil
	}
	arena := C.GoBytes(unsafe.Pointer(view.bytes), C.int(view.n_bytes)) // one copy for the whole answer
	keyOff := unsafe.Slice((*uint64)(unsafe.Pointer(view.key_off)), n)
	keyLen := unsafe.Slice((*uint32)(unsafe.Pointer(view.key_len)), n)
	valOff := unsafe.Slice((*uint64)(unsafe.Pointer(view.val_off)), n)
	valLen := unsafe.Slice((*uint32)(unsafe.Pointer(view.val_len)), n)
	rev := unsafe.Slice((*uint64)(unsafe.Pointer(view.rev)), n)
	kvs := make([]*proto.KeyValue, n)
	backing := make([]proto.KeyValue, n)
	for i := 0; i < n; i++ {
		backing[i] = proto.KeyValue{
			Key:      arena[keyOff[i] : keyOff[i]+uint64(keyLen[i])],
			Value:    arena[valOff[i] : valOff[i]+uint64(valLen[i])],
			Revision: rev[i],
		}
		kvs[i] = &backing[i]
	}
	return kvs
}

func (s *b200Scanner) Range(ctx context.Context, start, end []byte, revision uint64, limit int64) ([]*proto.KeyValue, error) {
	t0 := time.Now()
	res, view, err := s.rangeOnce(start, end, revision, limit, C.KB_OUT_HOST)
	if err != nil {
		return nil, err
	}
	defer C.kb_result_free(s.e.ctx, res)
	kvs := copyKvs(view)
	valSize := 0
	for _, kv := range kvs {
		valSize += len(kv.Value)
	}
	s.emitScanMetrics(time.Since(t0), valSize, int(*view.req_count))
	return kvs, nil
}

// RangeResponseWire returns the serialised etcdserverpb.RangeResponse of a List with the USER's limit (what
// backendShim.List builds per kv on the CPU, pkg/server/etcd/backendshim.go:269-282).  Like backend.List it scans
// limit+1 (pkg/backend/range.go:150-170), keeps the first `limit` kvs -- the arena is cut at elem_off[limit] -- and derives
// More and Count from what it saw (count = len(kvs) + 1 when there is more, backendshim.go:269-277).  The kv elements are
// written by the device, head and tail are added here.  The etcd gRPC handler sends it through a pass-through codec.
func (s *b200Scanner) RangeResponseWire(start, end []byte, revision uint64, limit int64, headerRev uint64) ([]byte, error) {
	ask := limit
	if limit > 0 {
		ask = limit + 1
	}
	res, view, err := s.rangeOnce(start, end, revision, ask, C.KB_OUT_HOST|C.KB_WIRE_ETCD_KVS)
	if err != nil {
		return nil, err
	}
	defer C.kb_result_free(s.e.ctx, res)
	n, nbytes := int64(view.n_kvs), uint64(view.n_bytes)
	more := limit > 0 && n > limit
	if more {
		n = limit
		nbytes = unsafe.Slice((*uint64)(unsafe.Pointer(view.elem_off)), int(view.n_kvs)+1)[limit]
	}
	var head, tail [32]C.uint8_t
	nh := C.kb_wire_range_head(C.uint64_t(headerRev), &head[0])
	m, count := C.int(0), C.int64_t(n)
	if more {
		m, count = 1, count+1
	}
	nt := C.kb_wire_range_tail(m, count, &tail[0])
	out := make([]byte, 0, int(nh)+int(nbytes)+int(nt))
	out = append(out, C.GoBytes(unsafe.Pointer(&head[0]), C.int(nh))...)
	if nbytes > 0 {
		out = append(out, unsafe.Slice((*byte)(unsafe.Pointer(view.bytes)), int(nbytes))...)
	}
	out = append(out, C.GoBytes(unsafe.Pointer(&tail[0]), C.int(nt))...)
	return out, nil
}

func (s *b200Scanner) Count(ctx context.Context, start, end []byte, revision uint64) (int, error) {
	res, view, err := s.rangeOnce(start, end, revision, 0, C.KB_OUT_COUNT)
	if err != nil {
		return 0, err
	}
	defer C.kb_result_free(s.e.ctx, res)
	return int(*view.req_count), nil
}

// rangeStreamPageBytes bounds the arena bytes of one page of a RangeStream: the answer is scanned once and copied out
// page by page, so memory follows the page instead of the answer.
const rangeStreamPageBytes = 64 << 20

func (s *b200Scanner) RangeStream(ctx context.Context, start, end []byte, revision uint64) chan *proto.StreamRangeResponse {
	stream := make(chan *proto.StreamRangeResponse, 1000)
	go func() {
		defer close(stream)
		t0, count, valSize := time.Now(), 0, 0
		err := s.rangePages(start, end, revision, func(kvs []*proto.KeyValue) {
			count += len(kvs)
			for _, kv := range kvs {
				valSize += len(kv.Value)
			}
			// a page holds whole 300-kv batches but for the last one (receiver.go:119-138)
			for i := 0; i < len(kvs); i += rangeStreamBatch {
				j := i + rangeStreamBatch
				if j > len(kvs) {
					j = len(kvs)
				}
				stream <- &proto.StreamRangeResponse{RangeResponse: &proto.RangeResponse{
					Header: &proto.ResponseHeader{Revision: 0}, Kvs: kvs[i:j], More: true}} // forked receiver: readRev unset (receiver.go:162-166)
			}
		})
		end := &proto.StreamRangeResponse{RangeResponse: &proto.RangeResponse{
			Header: &proto.ResponseHeader{Revision: revision}}} // getListStreamEnd scanner.go:179-192
		if err != nil {
			end.Err = err.Error()
		} else {
			s.emitScanMetrics(time.Since(t0), valSize, count)
		}
		stream <- end
	}()
	return stream
}

// rangePages runs one unlimited range as a kb_range_stream and hands every page's kvs (Go-owned copies) to f.  The
// context lock is held per call only, so other goroutines' ranges and writes run between two pages; a write between
// pages is seen in the part of the range not handed out yet (kb_b200.h).
func (s *b200Scanner) rangePages(start, end []byte, revision uint64, f func([]*proto.KeyValue)) error {
	var req C.kb_range_req
	pin := runtime.Pinner{}
	defer pin.Unpin()
	if len(start) > 0 {
		pin.Pin(&start[0])
		req.start = (*C.uint8_t)(unsafe.Pointer(&start[0]))
	}
	if len(end) > 0 {
		pin.Pin(&end[0])
		req.end = (*C.uint8_t)(unsafe.Pointer(&end[0]))
	}
	req.start_len, req.end_len = C.uint64_t(len(start)), C.uint64_t(len(end))
	req.read_rev = C.uint64_t(revision)
	var rs *C.kb_range_stream
	s.e.mu.Lock()
	rc := C.kb_range_stream_open(s.e.ctx, &req, C.KB_OUT_HOST, rangeStreamBatch, &rs)
	err := s.e.err(rc) // KB_ECOMPACTED carries the reference's message (scanner.go:620-623)
	s.e.mu.Unlock()
	if err != nil {
		return err
	}
	defer func() {
		s.e.mu.Lock()
		C.kb_range_stream_close(s.e.ctx, rs)
		s.e.mu.Unlock()
	}()
	for {
		var page *C.kb_result
		s.e.mu.Lock()
		rc = C.kb_range_stream_next(s.e.ctx, rs, rangeStreamPageBytes, &page)
		err = s.e.err(rc)
		s.e.mu.Unlock()
		if err != nil {
			return err
		}
		if page == nil {
			return nil
		}
		var view C.kb_range_view
		C.kb_range_view_get(page, &view)
		kvs := copyKvs(view)
		C.kb_result_free(s.e.ctx, page)
		f(kvs)
	}
}

// Victim is one delete call of the reference's compaction loop, in order.
type Victim struct {
	Record uint32
	Class  uint8 // KB_V_*: 1 superseded, 2 tombstone (store.Del); 3 revision record, 4 ttl revision record (DelCurrent); 5 ttl object
}

// Sweep classifies only: record indices into the snapshot, valid until it changes.  Compact (below) hands the victims to
// Apply as keys instead.
func (s *b200Scanner) Sweep(start, end []byte, revision, timeoutRevision uint64, supportTTL bool) ([]Victim, int, error) {
	var res *C.kb_result
	ttl := C.int(0)
	if supportTTL {
		ttl = 1
	}
	s.e.mu.Lock()
	rc := C.kb_compact_sweep(s.e.ctx, ptr8(start), C.uint64_t(len(start)), ptr8(end), C.uint64_t(len(end)),
		C.uint64_t(revision), C.uint64_t(timeoutRevision), ttl, C.KB_OUT_HOST, &res)
	s.e.mu.Unlock()
	if rc != 0 {
		return nil, 0, s.e.err(rc)
	}
	defer C.kb_result_free(s.e.ctx, res)
	var v C.kb_compact_view
	C.kb_compact_view_get(res, &v)
	n := int(v.n_victims)
	out := make([]Victim, n)
	if n > 0 {
		idx := unsafe.Slice((*uint32)(unsafe.Pointer(v.victim_idx)), n)
		cls := unsafe.Slice((*uint8)(unsafe.Pointer(v.victim_class)), n)
		for i := range out {
			out[i] = Victim{idx[i], cls[i]}
		}
	}
	return out, int(v.count), nil
}

// CompactPage is one page of a compaction stream: victims [First, First+len(Keys)) of the sweep's ordered delete-call
// list, as the keys the engine deletes.  Keys are INTERNAL keys; Guards[i] is the value the sweep read for classes 3 / 4
// (DelCurrent: delete only if the engine still holds it), empty otherwise.  Everything is a Go-owned copy.
type CompactPage struct {
	First   uint64
	Keys    [][]byte
	Guards  [][]byte
	Classes []uint8
	Records []uint32 // record indices in the snapshot the sweep ran on (diagnostics only: stale once deletes are applied)
}

const (
	compactPageBytes = 64 << 20 // arena bytes per compaction page
	compactGroup     = 1024     // victims per group: one engine batch each (storage.go ApplyVictimPage)
)

// Apply is supplied by the storage adaptor (storage.go ApplyVictimPage): it deletes one page's victims in the engine,
// and every successful commit reaches the mirror through the commit hook.
var Apply func(ctx context.Context, page CompactPage) error

// compactPages runs one sweep as a kb_compact_stream and hands every page to f.  The engine mutex is held per C call
// only, so commits -- f's own deletes among them -- and other reads run between two pages.
func (s *b200Scanner) compactPages(start, end []byte, revision, timeoutRevision uint64, supportTTL bool,
	f func(CompactPage) error) (count int, err error) {
	ttl := C.int(0)
	if supportTTL {
		ttl = 1
	}
	pin := runtime.Pinner{}
	defer pin.Unpin()
	if len(start) > 0 {
		pin.Pin(&start[0])
	}
	if len(end) > 0 {
		pin.Pin(&end[0])
	}
	var cs *C.kb_compact_stream
	s.e.mu.Lock()
	rc := C.kb_compact_stream_open(s.e.ctx, ptr8(start), C.uint64_t(len(start)), ptr8(end), C.uint64_t(len(end)),
		C.uint64_t(revision), C.uint64_t(timeoutRevision), ttl, compactGroup, &cs)
	err = s.e.err(rc)
	var cnt C.uint64_t
	if err == nil {
		C.kb_compact_stream_info(cs, nil, &cnt, nil)
	}
	s.e.mu.Unlock()
	if err != nil {
		return 0, err
	}
	defer func() {
		s.e.mu.Lock()
		C.kb_compact_stream_close(s.e.ctx, cs)
		s.e.mu.Unlock()
	}()
	for {
		var res *C.kb_result
		s.e.mu.Lock()
		rc = C.kb_compact_stream_next(s.e.ctx, cs, compactPageBytes, &res)
		err = s.e.err(rc)
		s.e.mu.Unlock()
		if err != nil || res == nil {
			return int(cnt), err
		}
		var v C.kb_compact_page_view
		C.kb_compact_page_view_get(res, &v)
		n := int(v.n)
		page := CompactPage{First: uint64(v.first), Keys: make([][]byte, n), Guards: make([][]byte, n),
			Classes: make([]uint8, n), Records: make([]uint32, n)}
		if n > 0 {
			arena := unsafe.Slice((*byte)(unsafe.Pointer(v.bytes)), int(v.n_bytes))
			koff := unsafe.Slice((*uint64)(unsafe.Pointer(v.key_off)), n)
			klen := unsafe.Slice((*uint32)(unsafe.Pointer(v.key_len)), n)
			goff := unsafe.Slice((*uint64)(unsafe.Pointer(v.guard_off)), n)
			glen := unsafe.Slice((*uint32)(unsafe.Pointer(v.guard_len)), n)
			copy(page.Classes, unsafe.Slice((*uint8)(unsafe.Pointer(v.victim_class)), n))
			copy(page.Records, unsafe.Slice((*uint32)(unsafe.Pointer(v.rec_idx)), n))
			for i := 0; i < n; i++ {
				page.Keys[i] = append([]byte(nil), arena[koff[i]:koff[i]+uint64(klen[i])]...)
				page.Guards[i] = append([]byte(nil), arena[goff[i]:goff[i]+uint64(glen[i])]...)
			}
		}
		C.kb_result_free(s.e.ctx, res)
		if err = f(page); err != nil {
			return int(cnt), err
		}
	}
}

// compactRecord / logCompactHistory / getTimeoutRevision: pkg/backend/scanner/compact.go:22-52, scanner.go:147-177.
// Engines without TTL support (TiKV) expire /events/ keys through the compaction sweep: a key written before the compact
// revision that is now older than cfg.TTL goes (scanner.go:566-591); engines with TTL never see a timeout revision.
type compactRecord struct {
	revision uint64
	time     time.Time
}

func (s *b200Scanner) logCompactHistory(revision uint64) {
	s.histMu.Lock()
	s.compactHistories = append(s.compactHistories, compactRecord{revision, time.Now()})
	s.histMu.Unlock()
}

func (s *b200Scanner) getTimeoutRevision() uint64 {
	if s.SupportTTL {
		return 0
	}
	s.histMu.Lock()
	defer s.histMu.Unlock()
	prev := uint64(0)
	for len(s.compactHistories) > 0 && time.Since(s.compactHistories[0].time) >= s.TTL {
		prev = s.compactHistories[0].revision
		s.compactHistories = s.compactHistories[1:]
	}
	return prev
}

func (s *b200Scanner) Compact(ctx context.Context, start, end []byte, revision uint64) {
	s.logCompactHistory(revision)
	if s.SupportTTL {
		_, _ = s.e.Expire(uint64(time.Now().Unix())) // what the engine no longer returns must not be classified
	}
	t0 := time.Now()
	if Apply == nil { // no adaptor to delete the victims: the sweep still records the compact revision
		_, count, _ := s.Sweep(start, end, revision, s.getTimeoutRevision(), s.SupportTTL)
		s.emitScanMetrics(time.Since(t0), 0, count)
		return
	}
	count, _ := s.compactPages(start, end, revision, s.getTimeoutRevision(), s.SupportTTL, func(page CompactPage) error {
		return Apply(ctx, page)
	})
	s.emitScanMetrics(time.Since(t0), 0, count)
}

var errNoWatchers = errors.New("no watchers")

// Match replaces WatcherHub.Stream + processEvents for one collector batch run: it returns, per watcher id, the
// indices of the events to deliver, in order (pkg/backend/watcherhub.go:78-92, watch.go:119-159).
// getOnce submits one point read and collects it, in two critical sections like rangeOnce: the read is a lane batch, so
// it runs beside the range batches other goroutines have in flight instead of waiting for their copies.
func (e *Engine) getOnce(key []byte, rev uint64, mode C.int) (*C.kb_result, C.kb_get_view, error) {
	var req C.kb_get_req
	var view C.kb_get_view
	pin := runtime.Pinner{}
	defer pin.Unpin()
	if len(key) > 0 {
		pin.Pin(&key[0])
		req.key = (*C.uint8_t)(unsafe.Pointer(&key[0]))
	}
	req.key_len, req.revision = C.uint64_t(len(key)), C.uint64_t(rev)
	var pend *C.kb_pending
	e.mu.Lock()
	err := e.err(C.kb_get_submit(e.ctx, &req, 1, mode, &pend))
	e.mu.Unlock()
	if err != nil {
		return nil, view, err
	}
	var res *C.kb_result
	e.mu.Lock()
	err = e.err(C.kb_get_collect(e.ctx, pend, &res)) // ends the pending on success and on failure
	e.mu.Unlock()
	if err != nil {
		return nil, view, err
	}
	C.kb_get_view_get(res, &view)
	return res, view, nil
}

// Get is backend.get (pkg/backend/range.go:81-121) on the mirror: the value of the newest version of the user key at or
// below rev (0: latest) and its revision.  A missing key and a deleted one answer storage.ErrKeyNotFound; for a deleted
// key modRev is the revision of the delete, as backend.get returns it.
func (e *Engine) Get(key []byte, rev uint64) (val []byte, modRev uint64, err error) {
	res, view, err := e.getOnce(key, rev, C.KB_OUT_HOST)
	if err != nil {
		return nil, 0, err
	}
	defer C.kb_result_free(e.ctx, res)
	modRev = uint64(*view.mod_rev)
	if *view.status != C.KB_GET_FOUND {
		return nil, modRev, storage.ErrKeyNotFound
	}
	return C.GoBytes(unsafe.Pointer(uintptr(unsafe.Pointer(view.bytes))+uintptr(*view.val_off)), C.int(*view.val_len)),
		modRev, nil
}

// GetResponseWire returns the serialised etcdserverpb.RangeResponse of backendShim.Get (pkg/server/etcd/backendshim.go:
// 235-254): the read's kv element, written by the device, or none for a missing or deleted key; header revision =
// max(curRev, mod_revision) when found, else curRev (range.go:45-72); count 1 or 0.
func (e *Engine) GetResponseWire(key []byte, rev, curRev uint64) ([]byte, error) {
	res, view, err := e.getOnce(key, rev, C.KB_OUT_HOST|C.KB_WIRE_ETCD_KVS)
	if err != nil {
		return nil, err
	}
	defer C.kb_result_free(e.ctx, res)
	found := *view.status == C.KB_GET_FOUND
	h, count := curRev, C.int64_t(0)
	var elem []byte
	if found {
		if m := uint64(*view.mod_rev); m > h {
			h = m
		}
		var eo *C.uint64_t
		C.kb_get_elem_off(res, &eo)
		off := unsafe.Slice((*uint64)(unsafe.Pointer(eo)), 2)
		elem = unsafe.Slice((*byte)(unsafe.Pointer(view.bytes)), int(off[1]))[off[0]:off[1]]
		count = 1
	}
	var head, tail [32]C.uint8_t
	nh := C.kb_wire_range_head(C.uint64_t(h), &head[0])
	nt := C.kb_wire_range_tail(0, count, &tail[0])
	out := make([]byte, 0, int(nh)+len(elem)+int(nt))
	out = append(out, C.GoBytes(unsafe.Pointer(&head[0]), C.int(nh))...)
	out = append(out, elem...)
	out = append(out, C.GoBytes(unsafe.Pointer(&tail[0]), C.int(nt))...)
	return out, nil
}

func (e *Engine) Match(keys []byte, keyOff, rev, batchOff []uint64) (start []uint64, eventIdx []uint32, err error) {
	if len(rev) == 0 {
		return nil, nil, nil // nothing to deliver
	}
	nb := 0
	if len(batchOff) > 1 {
		nb = len(batchOff) - 1
	}
	ev := C.kb_events{
		keys: ptr8(keys), key_off: ptr64(keyOff), rev: ptr64(rev), n: C.uint64_t(len(rev)),
		batch_off: ptr64(batchOff), n_batches: C.uint64_t(nb),
	}
	var res *C.kb_result
	e.mu.Lock()
	rc := C.kb_watch_match(e.ctx, &ev, C.KB_OUT_HOST, &res)
	e.mu.Unlock()
	if rc != 0 {
		return nil, nil, e.err(rc)
	}
	defer C.kb_result_free(e.ctx, res)
	var v C.kb_match_view
	C.kb_match_view_get(res, &v)
	start = append([]uint64(nil), unsafe.Slice((*uint64)(unsafe.Pointer(v.start)), int(v.n_watchers)+1)...)
	if v.n_deliveries > 0 {
		eventIdx = append([]uint32(nil), unsafe.Slice((*uint32)(unsafe.Pointer(v.event_idx)), int(v.n_deliveries))...)
	}
	return start, eventIdx, nil
}

func (e *Engine) WatchAdd(prefix []byte, minRev uint64) (uint32, error) {
	var id C.uint32_t
	var p *C.uint8_t
	if len(prefix) > 0 {
		p = (*C.uint8_t)(unsafe.Pointer(&prefix[0]))
	}
	e.mu.Lock()
	defer e.mu.Unlock()
	rc := C.kb_watch_add(e.ctx, p, C.uint64_t(len(prefix)), C.uint64_t(minRev), &id) // call first: `id` is written by it
	return uint32(id), e.err(rc)
}

func (e *Engine) WatchDel(id uint32) error {
	e.mu.Lock()
	defer e.mu.Unlock()
	return e.err(C.kb_watch_del(e.ctx, C.uint32_t(id)))
}
