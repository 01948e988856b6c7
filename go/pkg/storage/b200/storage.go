//go:build b200

// Package b200 implements storage.KvStorage (pkg/storage/interface.go:34-138) by WRAPPING the durable engine
// (badger or TiKV): every write still commits to the engine first; what has been committed is mirrored into the
// HBM-resident snapshot of libkbb200.so, which then answers the backend's scans, point reads, compaction
// classification and watch fan-out (pkg/backend/scanner, pkg/backend/watch.go).  Durability, CAS semantics and
// conflict reporting stay the engine's.
//
// NOTE: written without a Go toolchain (none exists in the build image).  tests/cpp/shim_replay_test.cpp replays the
// exact C call sequence of every method below (load, commit hook, expiry ticker, delete paths) against the oracle.
package b200

import (
	"bytes"
	"context"
	"errors"
	"io"
	"math"
	"sync"
	"time"

	"github.com/kubewharf/kubebrain/pkg/storage"

	kb "github.com/kubewharf/kubebrain/pkg/backend/scanner/b200"
)

// Config selects the GPU and the snapshot file used to skip the start-up iteration of the engine.
type Config struct {
	Device       int           // CUDA device ordinal
	SnapshotPath string        // optional: kb_dump / kb_restore file (validated; falls back to a full Iter pass)
	ExpireTick   time.Duration // how often TTL'd keys are dropped from the mirror (default 1 s)
	TTL          time.Duration // scanner.Config.TTL: the ttl every /events/ key is written with (scanner.go:78-79)
	// GetPartitions: 0 returns the interval whole; > 0 cuts it on the device into partitions of about PartitionBytes
	// answer bytes each, at most MaxPartitions of them (kb_range_partitions)
	PartitionBytes uint64
	MaxPartitions  uint64
	// HostValues keeps the snapshot's value heap in mapped pinned host memory instead of HBM (kb.CfgHostValues): for
	// stores whose values do not fit the GPU's memory, or a GPU whose memory is shared with other work
	HostValues bool
	// Reconciliation of the mirror with the engine (kb_reconcile).  RepairDelay: how long a key of a commit that ended in
	// ErrUncertainResult waits before it is reconciled (default 10 s, twice the retry queue's interval, so the queue's
	// rewrite has come through first).  VerifyInterval > 0 walks [magic, magic+1) with repair that often, VerifyChunk
	// engine records per call (default 4096); 0 (the default) never walks.
	RepairDelay    time.Duration
	VerifyInterval time.Duration
	VerifyChunk    int
}

type store struct {
	inner  storage.KvStorage // the durable engine
	eng    *kb.Engine
	cfg    Config
	stopCh chan struct{}
	once   sync.Once
	// gate orders the engine commit + mirror apply of every write (RLock) against a Verify chunk's Iter + Reconcile
	// (Lock): a chunk never compares an engine read with a mirror that has not seen a commit the read includes
	gate sync.RWMutex

	mu         sync.Mutex
	suspects   map[string]time.Time // keys of uncertain commits, by when they were queued
	lastVerify VerifyReport
}

// VerifyReport sums the chunks of one Verify walk.
type VerifyReport struct {
	Start, End                      []byte
	Chunks                          int
	Engine, Missing, Extra, Changed uint64
	Repaired                        bool
	Finished                        time.Time
}

// NewKvStorage opens the GPU engine, loads the engine's current content into HBM and returns the wrapping storage.
// It is what cmd/option/option_b200.go's buildStorage returns.
func NewKvStorage(inner storage.KvStorage, cfg Config) (storage.KvStorage, error) {
	var flags uint32
	if cfg.HostValues {
		flags |= kb.CfgHostValues
	}
	eng, err := kb.OpenConfig(cfg.Device, flags)
	if err != nil {
		return nil, err
	}
	s := &store{inner: inner, eng: eng, cfg: cfg, stopCh: make(chan struct{}), suspects: map[string]time.Time{}}
	if cfg.SnapshotPath == "" || eng.Restore(cfg.SnapshotPath) != nil {
		if err := s.loadSnapshot(context.Background()); err != nil {
			return nil, err
		}
	}
	tick := cfg.ExpireTick
	if tick <= 0 {
		tick = time.Second
	}
	if inner.SupportTTL() {
		go s.expireLoop(tick)
	}
	go s.repairLoop()
	if cfg.VerifyInterval > 0 {
		go s.verifyLoop(cfg.VerifyInterval)
	}
	return s, nil
}

var magic, magicEnd = []byte{0x57, 0xfb, 0x80, 0x8b}, []byte{0x57, 0xfb, 0x80, 0x8c}

// Engine hands the GPU engine to the backend, which builds its scanner from it (kb.NewScanner) instead of
// scanner.NewScanner(store, ...) at pkg/backend/backend.go:155.
func (s *store) Engine() *kb.Engine { return s.eng }

// loadSnapshot pulls the whole key space through ONE storage.Iter pass (ascending unique internal keys, the
// iterator contract kb_load_sorted checks) and bulk-loads it: kb_load_sorted(keys, key_off, vals, val_off, n).
func (s *store) loadSnapshot(ctx context.Context) error {
	ts, err := s.inner.GetTimestampOracle(ctx)
	if err != nil {
		return err
	}
	// every internal key starts with the coder's magic 0x57fb808b (coder/normal.go:26): [magic, magic+1) is all of them
	it, err := s.inner.Iter(ctx, magic, magicEnd, ts, 0)
	if err != nil {
		return err
	}
	defer it.Close()
	var keys, vals []byte
	var ttlKeys []kb.WriteOp
	keyOff, valOff := []uint64{0}, []uint64{0}
	for {
		if err := it.Next(ctx); err != nil {
			if err == io.EOF {
				break
			}
			return err
		}
		k, v := it.Key(), it.Val()
		keys = append(keys, k...)
		vals = append(vals, v...)
		keyOff = append(keyOff, uint64(len(keys)))
		valOff = append(valOff, uint64(len(vals)))
		if s.isTTLKey(k) {
			ttlKeys = append(ttlKeys, kb.WriteOp{Key: k, Val: v})
		}
	}
	if err := s.eng.LoadSorted(keys, keyOff, vals, valOff); err != nil {
		return err
	}
	return s.registerTTL(ttlKeys)
}

func (s *store) isTTLKey(k []byte) bool {
	return s.inner.SupportTTL() && s.cfg.TTL > 0 && bytes.Contains(k, []byte("/events/"))
}

// registerTTL puts `ops` again with the full cfg.TTL from now.  storage.Iter does not expose an entry's remaining
// lifetime.  The keys that were written with a ttl are the /events/ keys (scanner.go:566-570), all with cfg.TTL:
// re-registering them with the FULL ttl from now bounds how long the mirror can keep an event object the engine has
// already dropped.
func (s *store) registerTTL(ops []kb.WriteOp) error {
	exp := uint64(time.Now().Add(s.cfg.TTL).Unix())
	for i := range ops {
		ops[i].ExpireUnix = exp
	}
	return s.eng.ApplyBatch(ops)
}

// Verify walks the engine's records of [start, end) in chunks of `chunk` and reconciles each with the mirror (repair:
// the differences are committed to the mirror; else a dry run).  A chunk is read and compared under the write gate, so
// no commit lands between the engine read and the compare.  A chunk ends at the interval's end when the engine has no
// more records, else right behind its last key (lastKey + 0x00).  After a repair the repaired /events/ keys get the full
// TTL again, as at load.
func (s *store) Verify(ctx context.Context, start, end []byte, chunk int, repair bool) (VerifyReport, error) {
	if chunk <= 0 {
		chunk = 4096
	}
	rep := VerifyReport{Start: start, End: end, Repaired: repair}
	cur := append([]byte(nil), start...)
	for {
		next, done, err := s.verifyChunk(ctx, cur, end, chunk, repair, &rep)
		if err != nil {
			return rep, err
		}
		rep.Chunks++
		if done {
			rep.Finished = time.Now()
			return rep, nil
		}
		cur = next
	}
}

func (s *store) verifyChunk(ctx context.Context, cur, end []byte, chunk int, repair bool, rep *VerifyReport) ([]byte, bool, error) {
	s.gate.Lock()
	defer s.gate.Unlock()
	ts, err := s.inner.GetTimestampOracle(ctx)
	if err != nil {
		return nil, false, err
	}
	it, err := s.inner.Iter(ctx, cur, end, ts, uint64(chunk))
	if err != nil {
		return nil, false, err
	}
	var keys, vals []byte
	keyOff, valOff := []uint64{0}, []uint64{0}
	n := 0
	for {
		if err := it.Next(ctx); err != nil {
			if err == io.EOF {
				break
			}
			it.Close()
			return nil, false, err
		}
		k, v := it.Key(), it.Val()
		keys = append(keys, k...)
		vals = append(vals, v...)
		keyOff = append(keyOff, uint64(len(keys)))
		valOff = append(valOff, uint64(len(vals)))
		n++
	}
	done := n < chunk
	to := end
	if !done { // right behind the last key (copied: an iterator may reuse Key()'s slice)
		to = append(append([]byte(nil), keys[keyOff[n-1]:keyOff[n]]...), 0)
	}
	it.Close()
	d, err := s.eng.Reconcile(cur, to, keys, keyOff, vals, valOff, !repair)
	if err != nil {
		return nil, false, err
	}
	rep.Engine += d.Engine
	rep.Missing += d.Missing
	rep.Extra += d.Extra
	rep.Changed += d.Changed
	if repair {
		var ttlKeys []kb.WriteOp
		for k, key := range d.Keys {
			if d.Kinds[k] != kb.DiffExtra && s.isTTLKey(key) {
				i := d.SrcIdx[k]
				ttlKeys = append(ttlKeys, kb.WriteOp{Key: key, Val: vals[valOff[i]:valOff[i+1]]})
			}
		}
		if err := s.registerTTL(ttlKeys); err != nil {
			return nil, false, err
		}
	}
	return to, done, nil
}

// LastVerify is the report of the last background walk (Config.VerifyInterval).
func (s *store) LastVerify() VerifyReport {
	s.mu.Lock()
	defer s.mu.Unlock()
	return s.lastVerify
}

func (s *store) verifyLoop(every time.Duration) {
	t := time.NewTicker(every)
	defer t.Stop()
	for {
		select {
		case <-s.stopCh:
			return
		case <-t.C:
			rep, err := s.Verify(context.Background(), magic, magicEnd, s.cfg.VerifyChunk, true)
			if err == nil {
				s.mu.Lock()
				s.lastVerify = rep
				s.mu.Unlock()
			}
		}
	}
}

// suspect queues the keys of a batch whose commit ended in ErrUncertainResult: the engine may hold it or not
func (s *store) suspect(ops []kb.WriteOp) {
	now := time.Now()
	s.mu.Lock()
	defer s.mu.Unlock()
	for _, op := range ops {
		s.suspects[string(op.Key)] = now
	}
}

// repairLoop reconciles every suspect key older than RepairDelay over [key, key+0x00): the record the uncertain commit
// may have left in the engine reaches the mirror, one it never wrote leaves it
func (s *store) repairLoop() {
	delay := s.cfg.RepairDelay
	if delay <= 0 {
		delay = 10 * time.Second
	}
	t := time.NewTicker(delay / 4)
	defer t.Stop()
	for {
		select {
		case <-s.stopCh:
			return
		case now := <-t.C:
			var due []string
			s.mu.Lock()
			for k, at := range s.suspects {
				if now.Sub(at) >= delay {
					due = append(due, k)
					delete(s.suspects, k)
				}
			}
			s.mu.Unlock()
			for _, k := range due {
				key := []byte(k)
				if _, err := s.Verify(context.Background(), key, append(append([]byte(nil), key...), 0), 1, true); err != nil {
					s.suspect([]kb.WriteOp{{Key: key}}) // try again on a later tick
				}
			}
		}
	}
}

func (s *store) expireLoop(tick time.Duration) {
	t := time.NewTicker(tick)
	defer t.Stop()
	for {
		select {
		case <-s.stopCh:
			return
		case now := <-t.C:
			_, _ = s.eng.Expire(uint64(now.Unix())) // kb_expire: the mirror lags the engine's TTL by at most one tick
		}
	}
}

// ---- reads that stay with the engine (not on the hot path) ---------------------------------------------------
func (s *store) GetTimestampOracle(ctx context.Context) (uint64, error) {
	return s.inner.GetTimestampOracle(ctx)
}

// GetPartitions: with PartitionBytes == 0 one HBM snapshot per GPU is one partition; with several GPUs the routing layer
// asks every shard (kubebrain_b200/sharded.py: owner_of_prefix / merge_list_runs), so the interval is returned whole.
// With PartitionBytes > 0 the interval's answer at the latest revision is cut on the device into byte-balanced
// partitions whose inner borders are revision-record keys (what adjustPartitionsBorders, scanner.go:202-225, would make
// of them), the way tikv.go:123-153 returns one partition per region.
func (s *store) GetPartitions(ctx context.Context, start, end []byte) ([]storage.Partition, error) {
	if s.cfg.PartitionBytes == 0 {
		return []storage.Partition{{Start: start, End: end}}, nil
	}
	borders, err := s.eng.Partitions(start, end, math.MaxUint64, s.cfg.PartitionBytes, s.cfg.MaxPartitions)
	if err != nil {
		return nil, err
	}
	ps := make([]storage.Partition, 0, len(borders)-1)
	for k := 1; k < len(borders); k++ {
		ps = append(ps, storage.Partition{Start: borders[k-1], End: borders[k]})
	}
	return ps, nil
}

func (s *store) Get(ctx context.Context, key []byte) ([]byte, error) { return s.inner.Get(ctx, key) }

// Iter is delegated: the scanner built from Engine() never calls it; other callers (creator, revision bootstrap)
// keep the engine's exact iterator semantics, including reverse iteration and limit.
func (s *store) Iter(ctx context.Context, start, end []byte, timestamp, limit uint64) (storage.Iter, error) {
	return s.inner.Iter(ctx, start, end, timestamp, limit)
}

func (s *store) SupportTTL() bool { return s.inner.SupportTTL() }

func (s *store) Close() error {
	s.once.Do(func() { close(s.stopCh) })
	if s.cfg.SnapshotPath != "" {
		_ = s.eng.Dump(s.cfg.SnapshotPath)
	}
	s.eng.Close()
	return s.inner.Close()
}

// ---- writes: engine first, mirror second -----------------------------------------------------------------------
type batch struct {
	s     *store
	inner storage.BatchWrite
	ops   []kb.WriteOp // what Commit will have made durable, in call order
}

func (s *store) BeginBatchWrite() storage.BatchWrite {
	return &batch{s: s, inner: s.inner.BeginBatchWrite()}
}

func expireAt(ttl int64) uint64 {
	if ttl <= 0 {
		return 0
	}
	return uint64(time.Now().Unix() + ttl)
}

func (b *batch) put(key, val []byte, ttl int64) {
	b.ops = append(b.ops, kb.WriteOp{Key: append([]byte(nil), key...), Val: append([]byte(nil), val...), ExpireUnix: expireAt(ttl)})
}

func (b *batch) PutIfNotExist(key, val []byte, ttl int64) {
	b.inner.PutIfNotExist(key, val, ttl)
	b.put(key, val, ttl)
}

func (b *batch) CAS(key, newVal, oldVal []byte, ttl int64) {
	b.inner.CAS(key, newVal, oldVal, ttl)
	b.put(key, newVal, ttl)
}

func (b *batch) Put(key, val []byte, ttl int64) {
	b.inner.Put(key, val, ttl)
	b.put(key, val, ttl)
}

func (b *batch) Del(key []byte) {
	b.inner.Del(key)
	b.ops = append(b.ops, kb.WriteOp{Del: true, Key: append([]byte(nil), key...)})
}

func (b *batch) DelCurrent(it storage.Iter) {
	b.inner.DelCurrent(it)
	b.ops = append(b.ops, kb.WriteOp{Del: true, Key: append([]byte(nil), it.Key()...)})
}

// Commit: the batch is atomic in the engine; only a batch the engine has accepted reaches the mirror (a CAS failure
// or an uncertain result leaves the mirror untouched -- for ErrUncertainResult the backend's retry queue re-reads the
// engine and issues the compensating write, which arrives here like any other batch).
// The uncertain batch's keys are queued as suspects: repairLoop reconciles them once the retry queue is done.
func (b *batch) Commit(ctx context.Context) error {
	b.s.gate.RLock()
	defer b.s.gate.RUnlock()
	if err := b.inner.Commit(ctx); err != nil {
		if errors.Is(err, storage.ErrUncertainResult) {
			b.s.suspect(b.ops)
		}
		return err
	}
	return b.s.eng.ApplyBatch(b.ops)
}

func (s *store) Del(ctx context.Context, key []byte) error {
	s.gate.RLock()
	defer s.gate.RUnlock()
	if err := s.inner.Del(ctx, key); err != nil {
		return err
	}
	return s.eng.ApplyBatch([]kb.WriteOp{{Del: true, Key: key}})
}

func (s *store) DelCurrent(ctx context.Context, it storage.Iter) error {
	key := append([]byte(nil), it.Key()...)
	s.gate.RLock()
	defer s.gate.RUnlock()
	if err := s.inner.DelCurrent(ctx, it); err != nil {
		return err
	}
	return s.eng.ApplyBatch([]kb.WriteOp{{Del: true, Key: key}})
}

// ApplyVictims deletes plain keys in bulk: ONE engine batch per `chunk` keys, then the same keys leave the mirror.  It
// has no guard, so it is only right for store.Del victims (classes 1, 2, 5); a compaction page goes through
// ApplyVictimPage, which keeps DelCurrent's compare for classes 3 / 4.
func (s *store) ApplyVictims(ctx context.Context, keys [][]byte, chunk int) error {
	if chunk <= 0 {
		chunk = 1024
	}
	for i := 0; i < len(keys); i += chunk {
		j := i + chunk
		if j > len(keys) {
			j = len(keys)
		}
		bw := s.BeginBatchWrite()
		for _, k := range keys[i:j] {
			bw.Del(k)
		}
		if err := bw.Commit(ctx); err != nil {
			return err
		}
	}
	return nil
}

// ApplyVictimPage is kb.Apply: it deletes one page of a compaction stream in the engine, group by group (the page holds
// whole groups of 1024 victims but for the last one).  Per group, classes 1 / 2 / 5 (store.Del, scanner.go:465-475,
// 582-585) go in ONE engine batch instead of the reference's one transaction per victim.  Classes 3 / 4 (store.DelCurrent,
// scanner.go:477-491, 576-581) go one at a time with DelCurrent's semantics: an Iter positioned on the key, no delete
// if its value is no longer the guard the sweep read (the backend rewrote the revision record since), otherwise
// inner.DelCurrent.  A failed CAS is a skip, not an error.  Every successful commit reaches the mirror through the
// commit hook (engine first, mirror second).  The reference's "skip the rest of a raw key after a failed delete"
// (scanner.go:530-536) is not reproduced (DESIGN.md section 7).
func (s *store) ApplyVictimPage(ctx context.Context, page kb.CompactPage) error {
	const group = 1024
	for g := 0; g < len(page.Keys); g += group {
		h := g + group
		if h > len(page.Keys) {
			h = len(page.Keys)
		}
		bw := s.BeginBatchWrite()
		n := 0
		for i := g; i < h; i++ {
			if c := page.Classes[i]; c != 3 && c != 4 {
				bw.Del(page.Keys[i])
				n++
			}
		}
		if n > 0 {
			if err := bw.Commit(ctx); err != nil {
				return err
			}
		}
		for i := g; i < h; i++ {
			if c := page.Classes[i]; c != 3 && c != 4 {
				continue
			}
			if err := s.delCurrentIf(ctx, page.Keys[i], page.Guards[i]); err != nil {
				return err
			}
		}
	}
	return nil
}

// delCurrentIf: DelCurrent of `key` iff the engine still holds `guard` there; a changed or vanished value is skipped
func (s *store) delCurrentIf(ctx context.Context, key, guard []byte) error {
	ts, err := s.inner.GetTimestampOracle(ctx)
	if err != nil {
		return err
	}
	end := append(append([]byte(nil), key...), 0) // [key, key+0x00): exactly the key
	it, err := s.inner.Iter(ctx, key, end, ts, 1)
	if err != nil {
		return err
	}
	defer it.Close()
	if err := it.Next(ctx); err != nil {
		if err == io.EOF {
			return nil // deleted meanwhile
		}
		return err
	}
	if !bytes.Equal(it.Key(), key) || !bytes.Equal(it.Val(), guard) {
		return nil // rewritten since the sweep: the reference's CAS would fail
	}
	err = s.DelCurrent(ctx, it) // engine, then the mirror
	if errors.Is(err, storage.ErrCASFailed) {
		return nil // changed between the read and the delete (a conflict is an ErrCASFailed too)
	}
	return err
}
