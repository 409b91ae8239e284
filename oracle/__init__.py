"""CPU oracle for the CheckResources hot path -- TEST INFRASTRUCTURE ONLY.

This package restates, on the CPU, the reference algorithm for the path
svc.CerbosService.CheckResources -> engine.Check -> ruletable.check ->
conditions (CEL).  It exists to *check* the CUDA product path, never to serve
it: only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline
legs may import or execute anything under ``oracle/``.  Nothing under
``cerbos_b200/`` imports it.

Layers
  oracle/celeval.py   tree-walking CEL evaluator with cel-go v0.27.0 semantics
                      (third-party dependency of the reference, go.mod:45 --
                      its source is NOT in the reference tree; semantics are
                      restated from the CEL spec and pinned by the reference's
                      own goldens: internal/test/testdata/cel_eval/*.yaml,
                      internal/conditions/cerbos_lib_test.go:26-134).
  oracle/check.py     structural restatement of the decision algorithm
                      (internal/ruletable/ruletable.go:785-1155 and
                      internal/ruletable/index/index.go:564-881) over
                      string-keyed rule rows.
  oracle/c/           scalar C interpreter of the flattened device table
                      (same blob + same bytecode as the CUDA kernels); used as
                      oracle #2 and as the timed CPU baseline ("port").

Parity pinning: tests/test_oracle_goldens.py runs the oracle against the
reference's engine goldens (internal/test/testdata/engine*/ , 166 decisions),
the CEL goldens (cel_eval, 15 files) and the TestCerbosLib table, all
extracted into tests/golden/*.json by tests/golden/make_golden.py.
"""
