"""What the decision-metadata plane costs on the serving path: cgpu_check_narrow against cgpu_check_narrow_meta over pinned
host buffers, on the C3 and C5 narrow batches at their bench sizes, alternated in one process.  A separate torch.profiler
run of one call of each gives the device time of the kernels by name (the metadata kernels against the effect kernels) and
of the copies, which says whether the metadata path is bound by its kernel or by the link.

    python tools/meta_e2e.py [--workloads C3,C5] [--requests N] [--rounds 5] [--out meta_e2e.json]

Prints one JSON line per workload (and writes them all to --out); the effect bytes of both calls are compared once."""
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
from cerbos_b200 import capi, narrow as NW  # noqa: E402
from cerbos_b200.meta import REQUEST_META_DTYPE  # noqa: E402

NOW_NS = 1_704_067_200_000_000_000   # 2024-01-01T00:00:00Z
BENCH_N = {"C3": 1 << 24, "C5": 1 << 23}   # bench.py's requests per batch per GPU


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def pin(a):
    a = np.ascontiguousarray(a)
    p = torch.empty(max(a.nbytes, 1), dtype=torch.uint8).pin_memory()
    p.numpy()[: a.nbytes] = a.view(np.uint8).reshape(-1)
    return p.data_ptr(), p


def pinned(nbytes):
    return torch.empty(max(nbytes, 1), dtype=torch.uint8).pin_memory()


def profile(fn):
    """device time (ms) of each kernel name and of the copies in one call of fn"""
    from torch.profiler import ProfilerActivity, profile as tprofile
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us:
            out[e.key] = out.get(e.key, 0.0) + us / 1e3
    return out


def run(ctx, name, n, rounds):
    w = W.WORKLOADS[name]()
    _, ft, enc = W.build(w)
    b = W.columns_parallel(w, n, 0, enc)
    K = b.max_actions
    t = ctx.load_table(ft.blob)
    t.wait_ready()
    nb = NW.narrow_batch(b, len(enc.slots))
    assert nb is not None, name
    bb, nr, keep = t.prepare_narrow(nb, NOW_NS, 0, pin=pin)
    eff, eff_m = pinned(n * K), pinned(n * K)
    am, rm = pinned(n * K * 4), pinned(n * REQUEST_META_DTYPE.itemsize)

    def plain():
        t.check_narrow_into(bb, nr, eff.data_ptr())

    def meta():
        t.check_narrow_meta_into(bb, nr, eff_m.data_ptr(), am.data_ptr(), rm.data_ptr())

    for _ in range(2):
        plain()
        meta()
    assert torch.equal(eff, eff_m), f"{name}: effect bytes of cgpu_check_narrow_meta differ from cgpu_check_narrow"
    times = {"cgpu_check_narrow": [], "cgpu_check_narrow_meta": []}
    for _ in range(rounds):           # alternated, so that both see the same host and link conditions
        for key, fn in (("cgpu_check_narrow", plain), ("cgpu_check_narrow_meta", meta)):
            t0 = time.perf_counter()
            fn()                      # returns once every result is in host memory
            times[key].append(time.perf_counter() - t0)
    res = {"workload": name, "requests": n, "actions": K, "wire_bytes_per_request": nb.wire_bytes() / n,
           "d2h_bytes_per_request": {"cgpu_check_narrow": K, "cgpu_check_narrow_meta": K * 5 + REQUEST_META_DTYPE.itemsize}}
    for key, ts in times.items():
        med = float(np.median(ts))
        res[key] = {"ms_median": med * 1e3, "ms_min": min(ts) * 1e3, "ms_max": max(ts) * 1e3, "decisions_per_s": n * K / med}
    res["meta_over_plain_time"] = res["cgpu_check_narrow_meta"]["ms_median"] / res["cgpu_check_narrow"]["ms_median"]
    # kernel and copy time, each call in a profiler run of its own (tracing slows the host: not used for the rates above)
    kp, km = profile(plain), profile(meta)
    copies = lambda d: sum(v for k, v in d.items() if k.startswith("Memcpy"))  # noqa: E731
    effect_kernels = {k: v for k, v in kp.items() if not k.startswith("Memcpy") and "widen" not in k}
    # the metadata call's kernels: the metadata form of the unique-condition kernel and the drain of its deferrals
    # (check_meta_kernel), or check_meta_kernel alone for tables the unique-condition kernels do not take
    meta_ms = sum(v for k, v in km.items() if not k.startswith("Memcpy") and "widen" not in k)
    res["profile"] = {"cgpu_check_narrow": kp, "cgpu_check_narrow_meta": km,
                      "effect_kernels_ms": sum(effect_kernels.values()), "meta_kernels_ms": meta_ms,
                      "meta_kernels_over_effect_kernels": meta_ms / max(sum(effect_kernels.values()), 1e-9),
                      "copies_ms": {"cgpu_check_narrow": copies(kp), "cgpu_check_narrow_meta": copies(km)}}
    del keep
    t.release()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="C3,C5")
    ap.add_argument("--requests", type=int, default=0, help="requests per batch (default: the bench size of each workload)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    torch.cuda.init()
    ctx = capi.Context(0)
    dev = card()
    results = []
    for name in args.workloads.split(","):
        r = run(ctx, name, args.requests or BENCH_N[name], args.rounds)
        r["card"] = dev
        print(json.dumps(r), flush=True)
        results.append(r)
    ctx.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
