// engine_gpubaseline_test.go -- CPU baseline harness for the H100 CheckResources evaluator (cerbos_b200).
//
// Drop this file into internal/engine/ of a cerbos/cerbos checkout (it needs the module's own internal packages and its
// module cache; `go test` of the package then builds it).  It times the reference's own engine -- engine.Check, the code
// path svc.CerbosService.CheckResources calls (internal/svc/cerbos_svc.go:156, 205, 265) -- on the SAME synthetic
// policies and requests the GPU bench uses, exported by `python tools/export_workload.py --workload C3 --out DIR`:
//
//   DIR/policies/*.yaml     the workload's policy documents (disk store)
//   DIR/inputs.jsonl        one protojson enginev1.CheckInput per line (a prefix of the workload's request stream)
//   DIR/want.jsonl          optional: the effects the GPU path produced, for a parity spot-check
//
//   CERBOS_B200_WORKLOAD_DIR=DIR CERBOS_B200_SECONDS=10 go test ./internal/engine -run TestGPUBaseline -v
//
// Shape of the measurement (BASELINE.md 2.2, SURVEY.md 8(d)): the engine is built like mkEngine
// (internal/engine/engine_test.go:347-403) over a disk store like mkRuleTable (engine_bench_test.go:92-124), with
// NumWorkers = runtime.NumCPU() + 4; GOMAXPROCS client goroutines call eng.Check on slices of at most 1024 inputs for
// the requested wall time; the result line is JSON: decisions/s (one decision = one (input, action) effect) and the
// core count.  bench.py --impl reference runs it when `go version` succeeds and prints its number; otherwise the C port
// of the algorithm (oracle/c/check_ref.c) is timed and labelled "port".
package engine

import (
	"bufio"
	"context"
	"encoding/json"
	"fmt"
	"os"
	"path/filepath"
	"runtime"
	"strconv"
	"sync"
	"sync/atomic"
	"testing"
	"time"

	"github.com/stretchr/testify/require"
	"google.golang.org/protobuf/encoding/protojson"

	effectv1 "github.com/cerbos/cerbos/api/genpb/cerbos/effect/v1"
	enginev1 "github.com/cerbos/cerbos/api/genpb/cerbos/engine/v1"
	"github.com/cerbos/cerbos/internal/audit"
	"github.com/cerbos/cerbos/internal/compile"
	"github.com/cerbos/cerbos/internal/evaluator"
	"github.com/cerbos/cerbos/internal/ruletable"
	"github.com/cerbos/cerbos/internal/schema"
	"github.com/cerbos/cerbos/internal/storage/disk"
)

const gpuBaselineBatch = 1024

func gpuBaselineEngine(tb testing.TB, policyDir string) evaluator.Evaluator {
	tb.Helper()
	ctx, cancel := context.WithCancel(context.Background())
	tb.Cleanup(cancel)

	store, err := disk.NewStore(ctx, &disk.Conf{Directory: policyDir})
	require.NoError(tb, err)
	compiler, err := compile.NewManager(ctx, store)
	require.NoError(tb, err)
	schemaConf := schema.NewConf(schema.EnforcementNone)
	schemaMgr := schema.NewFromConf(ctx, store, schemaConf)
	ruleTable, err := ruletable.NewRuleTableFromLoader(ctx, compiler)
	require.NoError(tb, err)
	rtMgr, err := ruletable.NewRuleTableManager(ruleTable, compiler, schemaMgr)
	require.NoError(tb, err)

	evalConf := &evaluator.Conf{}
	evalConf.SetDefaults()
	evalConf.NumWorkers = uint(runtime.NumCPU() + 4)
	return NewFromConf(ctx, evalConf, Components{
		PolicyLoader:      compiler,
		RuleTableManager:  rtMgr,
		SchemaMgr:         schemaMgr,
		AuditLog:          audit.NewNopLog(),
		MetadataExtractor: audit.NewMetadataExtractorFromConf(&audit.Conf{}),
	})
}

func gpuBaselineInputs(tb testing.TB, path string) []*enginev1.CheckInput {
	tb.Helper()
	f, err := os.Open(path)
	require.NoError(tb, err)
	defer f.Close()
	var out []*enginev1.CheckInput
	sc := bufio.NewScanner(f)
	sc.Buffer(make([]byte, 1<<20), 1<<26)
	for sc.Scan() {
		if len(sc.Bytes()) == 0 {
			continue
		}
		in := &enginev1.CheckInput{}
		require.NoError(tb, protojson.Unmarshal(sc.Bytes(), in))
		out = append(out, in)
	}
	require.NoError(tb, sc.Err())
	return out
}

func TestGPUBaseline(t *testing.T) {
	dir := os.Getenv("CERBOS_B200_WORKLOAD_DIR")
	if dir == "" {
		t.Skip("CERBOS_B200_WORKLOAD_DIR not set (see the header of this file)")
	}
	seconds := 10.0
	if s := os.Getenv("CERBOS_B200_SECONDS"); s != "" {
		v, err := strconv.ParseFloat(s, 64)
		require.NoError(t, err)
		seconds = v
	}
	eng := gpuBaselineEngine(t, filepath.Join(dir, "policies"))
	inputs := gpuBaselineInputs(t, filepath.Join(dir, "inputs.jsonl"))
	require.NotEmpty(t, inputs)

	// parity spot-check against the effects the GPU path produced for the same requests
	if wf, err := os.Open(filepath.Join(dir, "want.jsonl")); err == nil {
		sc := bufio.NewScanner(wf)
		sc.Buffer(make([]byte, 1<<20), 1<<26)
		i, checked := 0, 0
		for sc.Scan() && i < len(inputs) && i < 4096 {
			want := map[string]string{}
			require.NoError(t, json.Unmarshal(sc.Bytes(), &want))
			outs, err := eng.Check(context.Background(), inputs[i:i+1])
			require.NoError(t, err)
			for action, eff := range want {
				got := outs[0].Actions[action].GetEffect()
				require.Equal(t, eff, effectv1.Effect_name[int32(got)], "input %d action %s", i, action)
				checked++
			}
			i++
		}
		wf.Close()
		t.Logf("parity: %d decisions equal to the GPU path's", checked)
	}

	clients := runtime.GOMAXPROCS(0)
	var decisions atomic.Int64
	deadline := time.Now().Add(time.Duration(seconds * float64(time.Second)))
	start := time.Now()
	var wg sync.WaitGroup
	for c := 0; c < clients; c++ {
		wg.Add(1)
		go func(c int) {
			defer wg.Done()
			ctx := context.Background()
			pos := (c * gpuBaselineBatch) % len(inputs)
			for time.Now().Before(deadline) {
				end := pos + gpuBaselineBatch
				if end > len(inputs) {
					end = len(inputs)
				}
				batch := inputs[pos:end]
				outs, err := eng.Check(ctx, batch)
				if err != nil {
					t.Errorf("Check: %v", err)
					return
				}
				n := 0
				for _, in := range batch {
					n += len(in.Actions)
				}
				if len(outs) != len(batch) {
					t.Errorf("short output")
					return
				}
				decisions.Add(int64(n))
				pos = end % len(inputs)
			}
		}(c)
	}
	wg.Wait()
	elapsed := time.Since(start).Seconds()
	res := map[string]any{
		"impl": "reference", "kind": "reference", "metric": "checkresources_decisions_per_sec", "unit": "decisions/s",
		"value": float64(decisions.Load()) / elapsed, "cores": runtime.NumCPU(), "gomaxprocs": clients,
		"seconds": elapsed, "inputs": len(inputs), "batch": gpuBaselineBatch, "go": runtime.Version(),
	}
	js, _ := json.Marshal(res)
	fmt.Println("GPU_BASELINE_RESULT " + string(js))
}
