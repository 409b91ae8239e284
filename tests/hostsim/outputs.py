"""ctypes driver for the host build of the rule-output walk (debug aid; see outputs.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

from hostsim import driver

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
_SRC = os.path.join(_ROOT, "tests", "hostsim", "outputs.cpp")
_SO = os.path.join(_ROOT, "oracle", "_build", "libhostsim_outputs.so")
_lib = None

STATUS_UNSUPPORTED, STATUS_OVERFLOW, STATUS_UNLOWERED = 1, 2, 4


def _plain():
    """Built when older than its sources and loaded on first use."""
    global _lib
    if _lib is None:
        deps = [_SRC] + [os.path.join(_ROOT, "cerbos_b200", "csrc", h) for h in ("cb_core.h", "cb_uc.h", "cb_host.h")] + \
               [os.path.join(_ROOT, "include", "cerbos_b200_format.h"), os.path.join(_ROOT, "include", "cerbos_b200.h")]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(d) for d in deps):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = f"{_SO}.{os.getpid()}.tmp"     # parallel test workers may build at once: write aside, then rename
            subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", f"-I{_ROOT}/include", f"-I{_ROOT}/cerbos_b200/csrc",
                            "-o", tmp, _SRC], check=True)
            os.replace(tmp, _SO)
        _lib = ctypes.CDLL(_SO)
        _lib.hostsim_check_outputs.restype = ctypes.c_int
    return _lib


def check_outputs(blob: bytes, columns, n, max_actions, stride=4096, now_ns=0, flags=0):
    """cb::eval_request_outputs over the batch -> (effects, action words, request records, output records uint8[n, stride],
    status bits: 0 or STATUS_*)."""
    from cerbos_b200.meta import REQUEST_META_DTYPE
    *args, _keep = driver._batch_args(blob, columns, n, max_actions, now_ns, flags)
    km = max(max_actions, 1)
    eff = np.zeros((n, km), dtype=np.uint8)
    am = np.zeros((n, km), dtype=np.uint32)
    rm = np.zeros(n, dtype=REQUEST_META_DTYPE)
    rec = np.zeros((n, stride), dtype=np.uint8)
    rc = _plain().hostsim_check_outputs(*args, eff.ctypes.data_as(ctypes.c_void_p), am.ctypes.data_as(ctypes.c_void_p),
                                        rm.ctypes.data_as(ctypes.c_void_p), rec.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint32(stride))
    if rc == -1:
        raise RuntimeError("hostsim_check_outputs: bad table or batch")
    return eff, am, rm, rec, (-rc) >> 1
