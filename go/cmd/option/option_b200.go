//go:build b200 && (badger || tikv)

// Compile-time storage selection (cf. cmd/option/option_badger.go:15-50, option_tikv.go):
//
//	go build --tags "badger b200"
//
// storageConfig below REPLACES the one of option_badger.go / option_tikv.go, whose build constraints a maintainer
// narrows to `badger && !b200` / `tikv && !b200` (one line each, INTEGRATION.md).  The durable engine is still built by
// the engine's own package; buildStorage wraps it in the HBM mirror (pkg/storage/b200).
package option

import (
	"fmt"
	"time"

	"github.com/spf13/pflag"

	"github.com/kubewharf/kubebrain/pkg/storage"
	"github.com/kubewharf/kubebrain/pkg/storage/b200"
)

type storageConfig struct {
	engine engineConfig // option_b200_badger.go / option_b200_tikv.go: the wrapped engine's own config
	b200.Config
}

func newStorageConfig() *storageConfig {
	s := &storageConfig{engine: newEngineConfig()}
	s.Device = 0
	s.ExpireTick = time.Second
	s.PartitionBytes = 0
	s.MaxPartitions = 64
	s.RepairDelay = 10 * time.Second
	s.VerifyInterval = 0
	s.VerifyChunk = 4096
	return s
}

func (s *storageConfig) addFlag(fs *pflag.FlagSet) {
	s.engine.addFlag(fs)
	fs.IntVar(&s.Device, "b200-device", s.Device, "CUDA device ordinal holding the HBM-resident snapshot")
	fs.StringVar(&s.SnapshotPath, "b200-snapshot", s.SnapshotPath,
		"file the HBM snapshot is dumped to on shutdown and restored from at start-up (empty: iterate the engine)")
	fs.DurationVar(&s.ExpireTick, "b200-expire-tick", s.ExpireTick, "period of the TTL sweep of the HBM mirror")
	fs.Uint64Var(&s.PartitionBytes, "b200-partition-bytes", s.PartitionBytes,
		"answer bytes per partition GetPartitions cuts a range into on the GPU (0: the range is one partition)")
	fs.Uint64Var(&s.MaxPartitions, "b200-max-partitions", s.MaxPartitions,
		"most partitions GetPartitions cuts a range into (1 .. 4096)")
	fs.BoolVar(&s.HostValues, "b200-host-values", s.HostValues,
		"keep the snapshot's values in pinned host memory mapped to the GPU instead of its memory (keys and directory stay on the GPU)")
	fs.DurationVar(&s.VerifyInterval, "b200-verify-interval", s.VerifyInterval,
		"period of a background walk that compares the HBM mirror with the engine and repairs it (0: never)")
	fs.IntVar(&s.VerifyChunk, "b200-verify-chunk", s.VerifyChunk, "engine records per compare of that walk")
	fs.DurationVar(&s.RepairDelay, "b200-repair-delay", s.RepairDelay,
		"how long the keys of a commit with an uncertain result wait before they are compared with the engine and repaired")
}

func (s *storageConfig) validate() error {
	if err := s.engine.validate(); err != nil {
		return err
	}
	if s.Device < 0 {
		return fmt.Errorf("b200-device must be >= 0, got %d", s.Device)
	}
	if s.ExpireTick <= 0 {
		return fmt.Errorf("b200-expire-tick must be positive, got %s", s.ExpireTick)
	}
	if s.MaxPartitions < 1 || s.MaxPartitions > 4096 {
		return fmt.Errorf("b200-max-partitions must be in [1, 4096], got %d", s.MaxPartitions)
	}
	if s.VerifyInterval < 0 || s.VerifyChunk < 1 || s.RepairDelay <= 0 {
		return fmt.Errorf("b200-verify-interval must be >= 0, b200-verify-chunk >= 1 and b200-repair-delay positive")
	}
	if s.PartitionBytes > 0 && s.PartitionBytes < 1<<20 {
		return fmt.Errorf("b200-partition-bytes must be 0 or at least 1 MiB, got %d", s.PartitionBytes)
	}
	return nil
}

func (s *storageConfig) buildStorage() (storage.KvStorage, error) {
	inner, err := s.engine.build()
	if err != nil {
		return nil, err
	}
	return b200.NewKvStorage(inner, s.Config)
}
