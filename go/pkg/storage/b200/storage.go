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
}

type store struct {
	inner  storage.KvStorage // the durable engine
	eng    *kb.Engine
	cfg    Config
	stopCh chan struct{}
	once   sync.Once
}

// NewKvStorage opens the GPU engine, loads the engine's current content into HBM and returns the wrapping storage.
// It is what cmd/option/option_b200.go's buildStorage returns.
func NewKvStorage(inner storage.KvStorage, cfg Config) (storage.KvStorage, error) {
	eng, err := kb.Open(cfg.Device)
	if err != nil {
		return nil, err
	}
	s := &store{inner: inner, eng: eng, cfg: cfg, stopCh: make(chan struct{})}
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
	return s, nil
}

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
	it, err := s.inner.Iter(ctx, []byte{0x57, 0xfb, 0x80, 0x8b}, []byte{0x57, 0xfb, 0x80, 0x8c}, ts, 0)
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
		if s.inner.SupportTTL() && s.cfg.TTL > 0 && bytes.Contains(k, []byte("/events/")) {
			ttlKeys = append(ttlKeys, kb.WriteOp{Key: k, Val: v})
		}
	}
	if err := s.eng.LoadSorted(keys, keyOff, vals, valOff); err != nil {
		return err
	}
	// storage.Iter does not expose an entry's remaining lifetime.  The keys that were written with a ttl are the /events/
	// keys (scanner.go:566-570), all with cfg.TTL: re-registering them with the FULL ttl from now bounds how long the
	// mirror can keep a pre-restart event object the engine has already dropped.
	exp := uint64(time.Now().Add(s.cfg.TTL).Unix())
	for i := range ttlKeys {
		ttlKeys[i].ExpireUnix = exp
	}
	return s.eng.ApplyBatch(ttlKeys)
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

// GetPartitions: one HBM snapshot per GPU is one partition; with several GPUs the routing layer asks every shard
// (kubebrain_b200/sharded.py: owner_of_prefix / merge_list_runs), so the interval is returned whole.
func (s *store) GetPartitions(ctx context.Context, start, end []byte) ([]storage.Partition, error) {
	return []storage.Partition{{Start: start, End: end}}, nil
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
func (b *batch) Commit(ctx context.Context) error {
	if err := b.inner.Commit(ctx); err != nil {
		return err
	}
	return b.s.eng.ApplyBatch(b.ops)
}

func (s *store) Del(ctx context.Context, key []byte) error {
	if err := s.inner.Del(ctx, key); err != nil {
		return err
	}
	return s.eng.ApplyBatch([]kb.WriteOp{{Del: true, Key: key}})
}

func (s *store) DelCurrent(ctx context.Context, it storage.Iter) error {
	key := append([]byte(nil), it.Key()...)
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
