"""ctypes driver for the host build of the unique-condition metadata body (debug aid; see meta_uc.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

from hostsim import driver

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
_SRC = os.path.join(_ROOT, "tests", "hostsim", "meta_uc.cpp")
_SO = os.path.join(_ROOT, "oracle", "_build", "libhostsim_meta_uc.so")
_lib = None


def _compile(out, defs=(), incs=()):
    subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", *defs, *[f"-I{d}" for d in incs], f"-I{_ROOT}/include",
                    f"-I{_ROOT}/cerbos_b200/csrc", "-o", out, _SRC], check=True)


def _plain():
    """The plain build (generic conditions), built when older than its sources and loaded on first use."""
    global _lib
    if _lib is None:
        deps = [_SRC] + [os.path.join(_ROOT, "cerbos_b200", "csrc", h) for h in ("cb_core.h", "cb_specialize.h", "cb_uc.h", "cb_host.h")] + \
               [os.path.join(_ROOT, "include", "cerbos_b200_format.h")]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(d) for d in deps):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = f"{_SO}.{os.getpid()}.tmp"     # parallel test workers may build at once: write aside, then rename
            _compile(tmp)
            os.replace(tmp, _SO)
        _lib = ctypes.CDLL(_SO)
    return _lib


def build_spec(blob: bytes, workdir: str):
    """The build with the unique-condition conditions generated for `blob` (cb::SpecConds); None if the table has none."""
    src = driver.generate_uc(blob)[0]
    if not src:
        return None
    with open(os.path.join(workdir, "spec_gen.inc"), "w") as f:
        f.write(src)
    so = os.path.join(workdir, "libhostsim_meta_uc_spec.so")
    _compile(so, ["-DHOSTSIM_SPEC_UC"], [workdir])
    return ctypes.CDLL(so)


def check_meta_uc(blob: bytes, columns, n, max_actions, now_ns=0, flags=0, lib=None):
    """driver.check_meta's three planes from the metadata form of the unique-condition body (cb::eval_request_uc_meta), its
    deferred requests through the reference-order body.  lib: a build_spec() library, else the plain build."""
    from cerbos_b200.meta import REQUEST_META_DTYPE
    *args, _keep = driver._batch_args(blob, columns, n, max_actions, now_ns, flags)
    km = max(max_actions, 1)
    eff = np.zeros((n, km), dtype=np.uint8)
    am = np.zeros((n, km), dtype=np.uint32)
    rm = np.zeros(n, dtype=REQUEST_META_DTYPE)
    fn = (lib if lib is not None else _plain()).hostsim_check_meta_uc
    fn.restype = ctypes.c_int
    rc = fn(*args, eff.ctypes.data_as(ctypes.c_void_p), am.ctypes.data_as(ctypes.c_void_p), rm.ctypes.data_as(ctypes.c_void_p))
    if rc != 0:
        raise RuntimeError(f"hostsim_check_meta_uc failed: {rc}")
    return eff, am, rm


def deferred(lib=None) -> int:
    """Requests the last check_meta_uc call through `lib` left to the reference-order body."""
    return int(ctypes.c_uint64.in_dll(lib if lib is not None else _plain(), "meta_uc_deferred").value)


def took(lib=None) -> bool:
    """Whether the last check_meta_uc call through `lib` ran the unique-condition metadata body (table and batch qualified)."""
    return bool(ctypes.c_int.in_dll(lib if lib is not None else _plain(), "meta_uc_took").value)
