#!/usr/bin/env python3
"""Row steps per 32-request warp of the unique-condition walk (cb::uc_walk), counted on the host.

Builds a workload's unique-condition image and the first requests of its first batch (the host build of the kernel
core, tools/uc_walk_steps.cpp), takes the rows each request visits per scope level of its chain from the chain descriptors, and
counts per warp of 32 consecutive requests, level by level:
  two loops   max over lanes of the DENY rows + max over lanes of the ALLOW rows (a DENY loop, then an ALLOW loop)
  one pass    max over lanes of DENY + ALLOW rows
  unrolled    the slots of the image's DENY + ALLOW segments (segment form; else the table's longest scope) at every level
              some lane reaches (the specialised walk's straight-line rows)
The walk also stops once every pair of a request is decided; that needs the condition values and is not modelled, so
the counts are upper bounds.  No device needed.

    python tools/uc_walk_steps.py C3
    python tools/uc_walk_steps.py C5 --requests 65536
"""
import argparse
import atexit
import ctypes
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LEVELS = 16
_lib = None


def _helper():
    """the host helper (uc_walk_steps.cpp: the library's own image builder and chain start), built once per process"""
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="uc_walk_steps_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libuc_walk_steps.so")
        subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", f"-I{ROOT}/include", f"-I{ROOT}/cerbos_b200/csrc", "-o", so,
                        os.path.join(ROOT, "tools", "uc_walk_steps.cpp")], check=True)
        _lib = ctypes.CDLL(so)
        _lib.uc_walk_rows.restype = ctypes.c_int64
    return _lib


def walk_rows(blob, b, flags=0):
    """-> (uint16[n, LEVELS, 2] DENY / counting ALLOW rows per request and level, the rows the walk visits per scope:
    the segment slots, or the table's longest scope)"""
    cols = [np.ascontiguousarray(c) for c in b.columns]
    out = np.zeros((b.n, LEVELS, 2), dtype=np.uint16)
    rc = _helper().uc_walk_rows(ctypes.create_string_buffer(blob, len(blob)), ctypes.c_uint64(len(blob)), ctypes.c_uint64(b.n),
                                ctypes.c_uint32(b.max_actions), ctypes.c_uint32(flags),
                                (ctypes.c_void_p * len(cols))(*[c.ctypes.data for c in cols]),
                                (ctypes.c_uint64 * len(cols))(*[c.nbytes for c in cols]),
                                ctypes.c_uint32(LEVELS), out.ctypes.data_as(ctypes.c_void_p))
    if rc < 0:
        raise RuntimeError(f"uc_walk_rows failed: {rc}")
    return out, int(rc)


def warp_steps(rows, scope_rows):
    """-> dict of per-warp row steps (float64[n_warps]) and per-level means, for full warps"""
    n = rows.shape[0] // 32 * 32
    w = rows[:n].reshape(-1, 32, LEVELS, 2).astype(np.int64)
    deny, allow = w[..., 0], w[..., 1]
    two = deny.max(axis=1) + allow.max(axis=1)           # [warps, levels]
    one = (deny + allow).max(axis=1)
    unrolled = np.where(one > 0, scope_rows, 0)
    return {"two loops": two, "one pass": one, "unrolled": unrolled}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("workload", nargs="?", default="C3")
    ap.add_argument("--requests", type=int, default=1 << 20, help="the first N requests of the batch")
    a = ap.parse_args()
    import workloads as W
    w = W.WORKLOADS[a.workload]()
    _, ft, enc = W.build(w)
    b = W.columns_parallel(w, min(a.requests, w.default_n), 0, enc)
    rows, scope_rows = walk_rows(ft.blob, b)
    steps = warp_steps(rows, scope_rows)
    reached = (rows.sum(axis=2) > 0).any(axis=0)
    n_lv = int(np.nonzero(reached)[0].max()) + 1 if reached.any() else 0
    print(f"{a.workload}: {b.n} requests, {b.n // 32} full warps; {scope_rows} unrolled rows per scope; chains up to {n_lv} levels")
    print("row steps per warp     " + "".join(f"  level {j}" for j in range(n_lv)) + "     total")
    for name, s in steps.items():
        print(f"  {name:<20}" + "".join(f"{s[:, j].mean():9.2f}" for j in range(n_lv)) + f"{s.sum(axis=1).mean():10.2f}")
    two, one = steps["two loops"].sum(axis=1).mean(), steps["one pass"].sum(axis=1).mean()
    print(f"one pass / two loops = {one / two:.3f}")


if __name__ == "__main__":
    main()
