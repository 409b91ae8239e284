"""cerbos_b200 -- H100-native batched CheckResources evaluator (the hot path of cerbos/cerbos:
engine.Check -> ruletable.check -> CEL conditions), behind a C ABI (include/cerbos_b200.h).

Layout
  csrc/      CUDA kernels (sm_90a) + C ABI             -> _lib/libcerbos_b200.so
  capi.py    ctypes binding of the C ABI
  engine.py  Engine.Check mirror (host buffers in, effects out)
  device.py  device-resident batches (torch tensors) for benchmarks / multi-GPU sharding
  table/     flattened rule table: layout, CEL->bytecode compiler, flattener
  encode.py  CheckInput batch -> SoA request columns
  policy/    policy documents -> rule rows (stand-in for the reference's Go compile + AddPolicy)
  cel/       CEL parser (stand-in for cel-go's parser: produces what CheckedExpr carries)
  narrow.py  the narrow wire format of cgpu_check_narrow;  meta.py  decoding of the metadata plane;  wire.py  CheckInput protobuf bytes
(the synthetic configurations C1..C5 of BASELINE.json are bench / test infrastructure: /workloads.py at the repository root)
"""
__all__ = ["capi", "engine", "encode"]
