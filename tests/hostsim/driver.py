"""ctypes driver for the host build of the kernel core (debug aid; see hostsim.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
_SO = os.path.join(_ROOT, "oracle", "_build", "libhostsim.so")
_lib = None


def build():
    src = os.path.join(_ROOT, "tests", "hostsim", "hostsim.cpp")
    deps = [src] + [os.path.join(_ROOT, "cerbos_b200", "csrc", h) for h in ("cb_core.h", "cb_specialize.h", "cb_uc.h", "cb_encode.h", "cb_host.h")] + \
           [os.path.join(_ROOT, "include", "cerbos_b200_format.h")]
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(d) for d in deps):
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        tmp = f"{_SO}.{os.getpid()}.tmp"     # parallel test workers may build at once: write aside, then rename
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", f"-I{_ROOT}/include",
                        f"-I{_ROOT}/cerbos_b200/csrc", "-o", tmp, src], check=True)
        os.replace(tmp, _SO)
    return _SO


def _plain():
    """The plain build (no generated evaluators), loaded on first use."""
    global _lib
    if _lib is None:
        lib = ctypes.CDLL(build())
        lib.hostsim_check.restype = lib.hostsim_check_meta.restype = ctypes.c_int
        lib.hostsim_generate.restype = lib.hostsim_generate_uc.restype = ctypes.c_int64
        lib.hostsim_encode.restype = lib.hostsim_encoded_column.restype = ctypes.c_void_p
        _lib = lib
    return _lib


def _batch_args(blob, columns, n, max_actions, now_ns, flags):
    """The leading arguments of hostsim_check / hostsim_check_spec / hostsim_check_meta (the arrays stay alive with the tuple)."""
    cols = [np.ascontiguousarray(c) for c in columns]
    return (ctypes.create_string_buffer(blob, len(blob)), ctypes.c_uint64(len(blob)), ctypes.c_uint64(n), ctypes.c_uint32(max_actions),
            ctypes.c_int64(now_ns), ctypes.c_uint32(flags), (ctypes.c_void_p * len(cols))(*[c.ctypes.data for c in cols]),
            (ctypes.c_uint64 * len(cols))(*[c.nbytes for c in cols]), cols)


def _run_check(fn, blob, columns, n, max_actions, now_ns, flags, mode):
    *args, _keep = _batch_args(blob, columns, n, max_actions, now_ns, flags)
    km = max(max_actions, 1)
    bitmap = np.zeros((n, (km + 7) // 8), dtype=np.uint8)
    rc = fn(*args, bitmap.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(mode))
    if rc != 0:
        raise RuntimeError(f"{fn.__name__} failed: {rc}")
    bits = np.unpackbits(bitmap, axis=1, bitorder="little")[:, :km]
    return np.where(bits == 1, 1, 2).astype(np.uint8)


def check(blob: bytes, columns, n, max_actions, now_ns=0, flags=0, mode=0):
    """Returns uint8[n, max_actions] effects decoded from the packed bitmap (padding slots = DENY-coded 2)."""
    return _run_check(_plain().hostsim_check, blob, columns, n, max_actions, now_ns, flags, mode)


def generate(blob: bytes) -> str:
    """Source of the table-specialised block evaluators (cb_specialize.h); "" when the table does not qualify."""
    cap = 1 << 22
    out = ctypes.create_string_buffer(cap)
    n = _plain().hostsim_generate(ctypes.create_string_buffer(blob, len(blob)), ctypes.c_uint64(len(blob)), out, ctypes.c_uint64(cap))
    if n < 0:
        raise RuntimeError(f"hostsim_generate failed: {n}")
    return out.value.decode()


def generate_uc(blob: bytes):
    """(source of the unique-condition specialised evaluator (cb_specialize.h: generate_uc; "" = does not qualify),
    number of distinct conditions of the table (0 = no unique-condition image))."""
    cap = 1 << 22
    out = ctypes.create_string_buffer(cap)
    nu = ctypes.c_uint32(0)
    n = _plain().hostsim_generate_uc(ctypes.create_string_buffer(blob, len(blob)), ctypes.c_uint64(len(blob)), out, ctypes.c_uint64(cap), ctypes.byref(nu))
    if n < 0:
        raise RuntimeError(f"hostsim_generate_uc failed: {n}")
    return out.value.decode(), nu.value


def deferred(lib=None) -> int:
    """Requests the lean / unique-condition body left to the general body in the last call through `lib` (default: the plain build)."""
    return int(ctypes.c_uint64.in_dll(lib if lib is not None else _plain(), "hostsim_deferred").value)


def body(lib=None) -> int:
    """The body the last check call through `lib` (default: the plain build) ran, by the mode that selects it: 0 / 3 lean,
    1 general 64-bit, 2 general 32-bit, 4 / 5 unique-condition.  A mode the table or batch cannot take runs body 1."""
    return int(ctypes.c_int.in_dll(lib if lib is not None else _plain(), "hostsim_body").value)


def build_spec(blob: bytes, workdir: str, uc: bool = False):
    """Host build of the kernel core with the evaluators generated for `blob` -> ctypes library exposing hostsim_check_spec.
    uc: the unique-condition form (cb::SpecConds, used by modes 4 / 5) instead of the block-shape form (cb::SpecBlocks)."""
    src_text = generate_uc(blob)[0] if uc else generate(blob)
    if not src_text:
        return None
    with open(os.path.join(workdir, "spec_gen.inc"), "w") as f:
        f.write(src_text)
    so = os.path.join(workdir, "libhostsim_spec_uc.so" if uc else "libhostsim_spec.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-DHOSTSIM_SPEC_UC" if uc else "-DHOSTSIM_SPEC", f"-I{workdir}", f"-I{_ROOT}/include",
                    f"-I{_ROOT}/cerbos_b200/csrc", "-o", so, os.path.join(_ROOT, "tests", "hostsim", "hostsim.cpp")], check=True)
    lib = ctypes.CDLL(so)
    lib.hostsim_check_spec.restype = ctypes.c_int
    return lib


def check_spec(lib, blob: bytes, columns, n, max_actions, now_ns=0, flags=0, mode=0):
    return _run_check(lib.hostsim_check_spec, blob, columns, n, max_actions, now_ns, flags, mode)


def check_meta(blob: bytes, columns, n, max_actions, now_ns=0, flags=0):
    """The decision-metadata body: -> (effects uint8[n, K], action words uint32[n, K], request records (cerbos_b200.meta dtype))."""
    from cerbos_b200.meta import REQUEST_META_DTYPE
    *args, _keep = _batch_args(blob, columns, n, max_actions, now_ns, flags)
    km = max(max_actions, 1)
    eff = np.zeros((n, km), dtype=np.uint8)
    am = np.zeros((n, km), dtype=np.uint32)
    rm = np.zeros(n, dtype=REQUEST_META_DTYPE)
    rc = _plain().hostsim_check_meta(*args, eff.ctypes.data_as(ctypes.c_void_p), am.ctypes.data_as(ctypes.c_void_p), rm.ctypes.data_as(ctypes.c_void_p))
    if rc != 0:
        raise RuntimeError(f"hostsim_check_meta failed: {rc}")
    return eff, am, rm


def native_encode(blob: bytes, messages, default_version="default", default_scope="", lenient=False, threads=1):
    """The native batch encoder (cb_encode.h) on serialized CheckInput messages -> (list of 12 uint8 arrays, dims)."""
    lib = _plain()
    n = len(messages)
    bufs = [ctypes.create_string_buffer(m, len(m)) for m in messages]
    ptrs = (ctypes.c_void_p * n)(*[ctypes.addressof(b) for b in bufs])
    lens = (ctypes.c_uint64 * n)(*[len(m) for m in messages])
    dims = (ctypes.c_uint32 * 4)()
    h = lib.hostsim_encode(ctypes.create_string_buffer(blob, len(blob)), ctypes.c_uint64(len(blob)), default_version.encode(), default_scope.encode(),
                           ctypes.c_int(1 if lenient else 0), ptrs, lens, ctypes.c_uint64(n), dims, ctypes.c_uint32(threads))
    if not h:
        raise RuntimeError("native encoder failed")
    cols = []
    for i in range(12):
        nb = ctypes.c_uint64()
        p = lib.hostsim_encoded_column(ctypes.c_void_p(h), ctypes.c_int(i), ctypes.byref(nb))
        cols.append(np.frombuffer(ctypes.string_at(p, nb.value), dtype=np.uint8).copy())
    lib.hostsim_encoded_free(ctypes.c_void_p(h))
    return cols, list(dims)
