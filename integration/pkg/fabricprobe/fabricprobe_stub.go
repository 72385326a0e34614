//go:build !cgo

// Stub so that `go build ./...` keeps working with CGO_ENABLED=0 (the reference's Makefile
// builds with CGO_ENABLED=1, Makefile:56-59, but tooling such as golangci-lint may not).
package fabricprobe

import (
	"context"
	"errors"
)

var (
	ErrUnsupported = errors.New("fabricprobe: not supported on this node")
	ErrTimeout     = errors.New("fabricprobe: probe timed out")
	ErrState       = errors.New("fabricprobe: handle is unusable")
	ErrCUDA        = errors.New("fabricprobe: CUDA call failed")
)

const (
	ModeReachOnly, ModeSliced, ModeFull             = 0, 1, 2
	OpRead, OpWrite                                 = 1, 2
	FlagFabricHandles, FlagMigAware, FlagLocalDiag = 0x01, 0x02, 0x04
)

type Config struct {
	LibraryPath string
	Ordinals    []int
	Bytes       uint64
	Mode        uint32
	Ops         uint32
	TimeoutMs   uint32
	Flags       uint32
	MinFraction  float32
	LinkPeakGBps float32
}

type Result struct {
	N                     int
	ReachRead, ReachWrite []bool
	GBpsRead, GBpsWrite   []float32
	Status                []int32
	ProbeMs               float64
	Verdict, Aborted      bool
	BytesPerPair          uint64
	MinGBpsRead, MinGBpsWrite   float32
	GateGBpsRead, GateGBpsWrite float32
	UnreachablePairs, SlowPairs int
}

type Probe struct{}

var DiagKinds = [5]string{"flip", "zero", "displaced", "stale", "foreign"}

type DiagSample struct {
	Offset, Expected, Observed, Word, RunSeq uint64
	Kind                                     string
	Rank                                     int
}

type Diagnosis struct {
	Op                     string
	Issuer, Target, Reader int
	RunSeq                 uint64
	Words                  uint64
	BadWords, BadGranules  uint64
	ZeroWords              uint64
	FirstBad, LastBad      uint64
	KindCount              [5]uint64
	BitFlips               [64]uint64
	Ms                     float64
	Samples                []DiagSample
}

type Latency struct {
	N                      int
	RowMask                uint32
	Hops, Reps             int
	RegionBytes            uint64
	Measured               []bool
	Status                 []int32
	NsMin, NsMedian, NsMax []float32
	Digest                 []uint64
	Ms                     float64
}

type PingPong struct {
	N                      int
	RowMask                uint32
	Trips, Reps            int
	Fenced                 bool
	CallSeq                uint64
	Measured               []bool
	Status                 []int32
	NsMin, NsMedian, NsMax []float32
	Digest                 []uint64
	Ms                     float64
}

const AtomicFetchAdd, AtomicCAS, AtomicContended = 0, 1, 2

type Atomics struct {
	N                      int
	RowMask                uint32
	Kind                   int
	Ops, Reps, Lanes       int
	CallSeq                uint64
	Native                 []uint8
	Measured               []bool
	Status                 []int32
	NsMin, NsMedian, NsMax []float32
	Digest                 []uint64
	Ms                     float64
}

type BwCurve struct {
	N                      int
	RowMask                uint32
	Reps                   int
	Path                   int
	CallSeq                uint64
	Sizes                  []uint64
	Measured               []bool
	Status                 []int32
	BadSizes               []uint32
	T0Ns, PeakGBps         []float32
	HalfBytes              []uint64
	NsMin, NsMedian, NsMax [][]float32
	Sum, Xr                [][]uint64
	Ms                     float64
}

type AllReduce struct {
	N                      int
	RowMask                uint32
	Reps                   int
	Path                   int
	CallSeq                uint64
	Sizes                  []uint64
	Measured               []bool
	Status                 []int32
	BadSizes               []uint32
	T0Ns, PeakGBps         []float32
	HalfBytes              []uint64
	NsMin, NsMedian, NsMax [][]float32
	Sum, Xr                [][]uint64
	BadWords, FirstBad     [][]uint64
	Ms                     float64
}

func Open(Config) (*Probe, error)                  { return nil, ErrUnsupported }
func (*Probe) Run(context.Context) (Result, error) { return Result{}, ErrUnsupported }
func (*Probe) Diagnose(uint32, int, int, int) (Diagnosis, error) {
	return Diagnosis{}, ErrUnsupported
}
func (*Probe) Latency(int, int) (Latency, error) { return Latency{}, ErrUnsupported }
func (*Probe) PingPong(int, int, bool) (PingPong, error) {
	return PingPong{}, ErrUnsupported
}
func (*Probe) Atomics(int, int, int) (Atomics, error) { return Atomics{}, ErrUnsupported }
func (*Probe) BwCurve(int) (BwCurve, error) { return BwCurve{}, ErrUnsupported }
func (*Probe) AllReduce(int) (AllReduce, error) { return AllReduce{}, ErrUnsupported }
func (*Probe) Close() {}
