"""What rule outputs cost: cgpu_check_outputs against cgpu_check_meta on the same batch -- workload C3's policies with an output
added to every rule (built in memory; workloads.py is unchanged) -- over pinned host buffers, alternated in one process.

    python tools/outputs_bench.py [--requests N] [--rounds 3] [--stride 1024] [--out outputs_bench.json]

Prints one JSON line with decisions/s of both calls and the card's name, power limit and maximum SM clock read in the same
run.  The effect bytes of both calls are compared once, and the output records are checked for overflow."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import workloads as W  # noqa: E402
from cerbos_b200 import capi  # noqa: E402
from cerbos_b200.meta import REQUEST_META_DTYPE  # noqa: E402
from cerbos_b200.policy.compile import build_rule_table, compile_expr  # noqa: E402
from cerbos_b200.table.flatten import flatten  # noqa: E402

NOW_NS = 1_704_067_200_000_000_000   # 2024-01-01T00:00:00Z
OUTPUT = 'P.id'   # one short string per entry: what is measured is the walk and the records, not a large value


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def pinned(nbytes):
    return torch.empty(max(nbytes, 1), dtype=torch.uint8).pin_memory()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=1 << 24)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--stride", type=int, default=1024)
    ap.add_argument("--out", default="outputs_bench.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("outputs_bench: no GPU")
    w = W.C3()
    rt = build_rule_table(w.policies())
    for r in rt.rows:
        if not r.from_role_policy:
            r.emit_activated = compile_expr(OUTPUT)
    ft = flatten(rt)
    enc = W.Encoder(ft.manifest)
    b = W.columns_parallel(w, a.requests, 0, enc)
    n, km = b.n, max(b.max_actions, 1)
    cols = []
    for c in b.columns:   # pinned copies of the columns: pageable memory makes every copy synchronous
        c = np.ascontiguousarray(c)
        p = pinned(c.nbytes)
        p.numpy()[: c.nbytes] = c.view(np.uint8).reshape(-1)
        cols.append(p.numpy()[: c.nbytes].view(c.dtype).reshape(c.shape))
    eff, am = pinned(n * km).numpy().reshape(n, km), pinned(n * km * 4).numpy().view(np.uint32).reshape(n, km)
    rm = pinned(n * REQUEST_META_DTYPE.itemsize).numpy().view(REQUEST_META_DTYPE)
    rec = pinned(n * a.stride).numpy().reshape(n, a.stride)
    eff2 = pinned(n * km).numpy().reshape(n, km)
    ctx = capi.Context(0)
    t = ctx.load_table(ft.blob)
    import ctypes
    from cerbos_b200.capi import _Batch, _check, lib
    ptrs = (ctypes.c_void_p * len(cols))(*[c.ctypes.data for c in cols])
    sizes = (ctypes.c_size_t * len(cols))(*[c.nbytes for c in cols])
    bt = _Batch(n, b.max_actions, NOW_NS, 0, ptrs, sizes, len(cols))
    need = ctypes.c_uint32(0)

    def run_meta():
        _check(lib().cgpu_check_meta(ctx._h, t._h, ctypes.byref(bt), eff2.ctypes.data_as(ctypes.c_void_p),
                                     am.ctypes.data_as(ctypes.c_void_p), rm.ctypes.data_as(ctypes.c_void_p)))

    def run_outputs():
        _check(lib().cgpu_check_outputs(ctx._h, t._h, ctypes.byref(bt), eff.ctypes.data_as(ctypes.c_void_p),
                                        am.ctypes.data_as(ctypes.c_void_p), rm.ctypes.data_as(ctypes.c_void_p),
                                        rec.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint32(a.stride), ctypes.byref(need)))

    run_meta()
    run_outputs()   # warm-up of both shapes
    assert (eff == eff2).all(), "effects differ between the two calls"
    n_entries = rec[:, 4:8].copy().view(np.uint32).astype(np.int64).sum()
    times = {"meta": [], "outputs": []}
    for _ in range(a.rounds):
        for name, fn in (("meta", run_meta), ("outputs", run_outputs)):
            t0 = time.perf_counter()
            fn()
            times[name].append(time.perf_counter() - t0)
    res = {"workload": "C3 + an output on every rule", "requests": n, "actions_per_request": b.max_actions, "stride": a.stride,
           "entries": int(n_entries), "card": card(),
           "meta_decisions_per_s": n * b.max_actions / min(times["meta"]),
           "outputs_decisions_per_s": n * b.max_actions / min(times["outputs"]),
           "meta_s": times["meta"], "outputs_s": times["outputs"]}
    res["outputs_over_meta_time"] = min(times["outputs"]) / min(times["meta"])
    print(json.dumps(res))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    t.release()
    ctx.close()


if __name__ == "__main__":
    main()
