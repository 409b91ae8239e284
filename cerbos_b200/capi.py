"""ctypes binding of the C ABI (include/cerbos_b200.h) -- the same entry points the Go side binds via cgo
(INTEGRATION.md).  There is no fallback: if the CUDA library is missing or no GPU is present the calls fail.
"""
from __future__ import annotations

import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("CERBOS_B200_LIB") or os.path.join(_HERE, "_lib", "libcerbos_b200.so")   # override: experimental builds

N_COLUMNS = 12
OK, ERR_INVALID, ERR_CUDA, ERR_UNSUPPORTED, ERR_NO_DEVICE = 0, -1, -2, -3, -4

EXPORTS = [
    "cgpu_init", "cgpu_shutdown", "cgpu_table_load", "cgpu_table_retain", "cgpu_table_release", "cgpu_check", "cgpu_check_meta", "cgpu_check_narrow",
    "cgpu_check_narrow_meta", "cgpu_check_outputs",
    "cgpu_check_device", "cgpu_sync", "cgpu_launch_count", "cgpu_deferred_count", "cgpu_table_info", "cgpu_last_kernel_config",
    "cgpu_last_cluster_config", "cgpu_profile", "cgpu_table_wait_ready", "cgpu_table_compile_check", "cgpu_peer_alloc", "cgpu_peer_open", "cgpu_peer_close",
    "cgpu_peer_free", "cgpu_peer_read", "cgpu_check_device_gather", "cgpu_gather_wait", "cgpu_last_error",
    "cgpu_device_count", "cgpu_encoder_create", "cgpu_encoder_destroy", "cgpu_encode", "cgpu_encoded_batch", "cgpu_encoded_free",
    "cgpu_narrow_build", "cgpu_narrowed_view", "cgpu_narrowed_free",
]


class CgpuError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"cerbos_b200 error {code}: {msg}")
        self.code = code


class _Gather(ctypes.Structure):
    _fields_ = [("n_ranks", ctypes.c_uint32), ("my_rank", ctypes.c_uint32), ("gather_bufs", ctypes.POINTER(ctypes.c_void_p)),
                ("slice_bytes", ctypes.c_uint64), ("flags", ctypes.POINTER(ctypes.c_void_p)), ("step", ctypes.c_uint32), ("wait_step", ctypes.c_uint32), ("wait_flags", ctypes.c_void_p)]


class _Narrow(ctypes.Structure):
    _fields_ = [("principal_id", ctypes.c_void_p), ("hdr16", ctypes.c_void_p), ("versions", ctypes.c_void_p), ("roles", ctypes.c_void_p),
                ("role_cols", ctypes.c_uint32), ("slot_class", ctypes.c_void_p), ("slot_cols", ctypes.POINTER(ctypes.c_void_p)), ("heap_u32", ctypes.c_uint32),
                ("slot_base", ctypes.c_void_p), ("slot_base2", ctypes.c_void_p), ("principal_id16", ctypes.c_void_p), ("principal_base", ctypes.c_uint32), ("hdr_const_mask", ctypes.c_uint32),
                ("hdr_const", ctypes.c_uint16 * 4), ("versions_const", ctypes.c_uint32), ("versions_value", ctypes.c_uint8 * 2),
                ("heap_bits", ctypes.c_uint32), ("heap_base", ctypes.c_uint32), ("heap_base2", ctypes.c_uint32)]


class _Batch(ctypes.Structure):
    _fields_ = [("n_requests", ctypes.c_uint64), ("max_actions", ctypes.c_uint32),
                ("now_unix_nanos", ctypes.c_int64), ("flags", ctypes.c_uint32),
                ("columns", ctypes.POINTER(ctypes.c_void_p)), ("column_bytes", ctypes.POINTER(ctypes.c_size_t)),
                ("n_columns", ctypes.c_uint32)]


_lib = None


def lib():
    """Loads the in-tree CUDA library. Raises if it has not been built (python -m cerbos_b200.csrc.build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: build it with `python -m cerbos_b200.csrc.build` "
                              "(cerbos_b200 has no CPU fallback)")
        L = ctypes.CDLL(LIB_PATH)
        L.cgpu_init.restype = ctypes.c_int
        L.cgpu_init.argtypes = [ctypes.POINTER(ctypes.c_int), ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)]
        L.cgpu_shutdown.restype = None
        L.cgpu_shutdown.argtypes = [ctypes.c_void_p]
        L.cgpu_table_load.restype = ctypes.c_int
        L.cgpu_table_load.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_void_p)]
        L.cgpu_table_retain.restype = None
        L.cgpu_table_retain.argtypes = [ctypes.c_void_p]
        L.cgpu_table_release.restype = None
        L.cgpu_table_release.argtypes = [ctypes.c_void_p]
        L.cgpu_check.restype = ctypes.c_int
        L.cgpu_check.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(_Batch), ctypes.c_void_p]
        L.cgpu_check_narrow.restype = ctypes.c_int
        L.cgpu_check_narrow.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(_Batch), ctypes.POINTER(_Narrow), ctypes.c_void_p]
        L.cgpu_check_meta.restype = ctypes.c_int
        L.cgpu_check_meta.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(_Batch), ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        L.cgpu_check_outputs.restype = ctypes.c_int
        L.cgpu_check_outputs.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(_Batch), ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                         ctypes.c_void_p, ctypes.c_uint32, ctypes.POINTER(ctypes.c_uint32)]
        L.cgpu_check_narrow_meta.restype = ctypes.c_int
        L.cgpu_check_narrow_meta.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(_Batch), ctypes.POINTER(_Narrow), ctypes.c_void_p,
                                             ctypes.c_void_p, ctypes.c_void_p]
        L.cgpu_check_device.restype = ctypes.c_int
        L.cgpu_check_device.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(_Batch), ctypes.c_void_p,
                                        ctypes.c_void_p]
        L.cgpu_sync.restype = ctypes.c_int
        L.cgpu_sync.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.cgpu_launch_count.restype = ctypes.c_uint64
        L.cgpu_launch_count.argtypes = [ctypes.c_void_p]
        L.cgpu_deferred_count.restype = ctypes.c_int
        L.cgpu_deferred_count.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64)]
        L.cgpu_table_info.restype = ctypes.c_int
        L.cgpu_table_info.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint32), ctypes.c_uint32]
        L.cgpu_last_kernel_config.restype = ctypes.c_int
        L.cgpu_last_kernel_config.argtypes = [ctypes.c_void_p] + [ctypes.POINTER(ctypes.c_uint32)] * 3
        L.cgpu_last_cluster_config.restype = ctypes.c_int
        L.cgpu_last_cluster_config.argtypes = [ctypes.c_void_p] + [ctypes.POINTER(ctypes.c_uint32)] * 3
        L.cgpu_profile.restype = ctypes.c_int
        L.cgpu_profile.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_uint64)]
        L.cgpu_table_compile_check.restype = ctypes.c_int
        L.cgpu_table_compile_check.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)]
        L.cgpu_table_wait_ready.restype = ctypes.c_int
        L.cgpu_table_wait_ready.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int)]
        for name, args in (("cgpu_peer_alloc", [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_void_p), ctypes.c_void_p]),
                           ("cgpu_peer_open", [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p)]),
                           ("cgpu_peer_close", [ctypes.c_void_p, ctypes.c_void_p]), ("cgpu_peer_free", [ctypes.c_void_p, ctypes.c_void_p]),
                           ("cgpu_peer_read", [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t]),
                           ("cgpu_check_device_gather", [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(_Batch), ctypes.POINTER(_Gather), ctypes.c_void_p]),
                           ("cgpu_gather_wait", [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p])):
            getattr(L, name).restype = ctypes.c_int
            getattr(L, name).argtypes = args
        L.cgpu_encoder_create.restype = ctypes.c_int
        L.cgpu_encoder_create.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)]
        L.cgpu_encoder_destroy.restype = None
        L.cgpu_encoder_destroy.argtypes = [ctypes.c_void_p]
        L.cgpu_encode.restype = ctypes.c_int
        L.cgpu_encode.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_size_t), ctypes.c_uint64, ctypes.POINTER(ctypes.c_void_p)]
        L.cgpu_encoded_batch.restype = ctypes.c_int
        L.cgpu_encoded_batch.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.POINTER(_Batch)]
        L.cgpu_encoded_free.restype = None
        L.cgpu_encoded_free.argtypes = [ctypes.c_void_p]
        L.cgpu_narrow_build.restype = ctypes.c_int
        L.cgpu_narrow_build.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)]
        L.cgpu_narrowed_view.restype = ctypes.c_int
        L.cgpu_narrowed_view.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.POINTER(_Batch), ctypes.POINTER(_Narrow)]
        L.cgpu_narrowed_free.restype = None
        L.cgpu_narrowed_free.argtypes = [ctypes.c_void_p]
        L.cgpu_last_error.restype = ctypes.c_char_p
        L.cgpu_last_error.argtypes = []
        _lib = L
    return _lib


def _check(rc):
    if rc != OK:
        raise CgpuError(rc, lib().cgpu_last_error().decode("utf-8", "replace"))


def compile_check(blob: bytes):
    """Generates and NVRTC-compiles the table-specialised kernels for `blob` without touching a device.
    -> (cubin bytes, note): 0 bytes when the table does not qualify."""
    n = ctypes.c_size_t()
    buf = (ctypes.c_char * len(blob)).from_buffer_copy(blob)
    _check(lib().cgpu_table_compile_check(buf, len(blob), ctypes.byref(n)))
    return n.value, (lib().cgpu_last_error().decode("utf-8", "replace") if n.value == 0 else "ok")


class NativeEncoder:
    """cgpu_encoder: serialized enginev1.CheckInput messages -> column batch, in C++ (cb_encode.h)."""

    def __init__(self, blob: bytes, default_version="default", default_scope="", lenient_scope_search=False):
        self._h = ctypes.c_void_p()
        buf = (ctypes.c_char * len(blob)).from_buffer_copy(blob)
        _check(lib().cgpu_encoder_create(buf, len(blob), default_version.encode(), default_scope.encode(), 1 if lenient_scope_search else 0,
                                         ctypes.byref(self._h)))

    def encode(self, messages) -> "EncodedBatch":
        n = len(messages)
        keep = [ctypes.create_string_buffer(m, len(m)) for m in messages]
        ptrs = (ctypes.c_void_p * n)(*[ctypes.addressof(b) for b in keep])
        lens = (ctypes.c_size_t * n)(*[len(m) for m in messages])
        return self.encode_raw(ptrs, lens, n)

    def encode_raw(self, ptrs, lens, n) -> "EncodedBatch":
        out = ctypes.c_void_p()
        _check(lib().cgpu_encode(self._h, ptrs, lens, n, ctypes.byref(out)))
        return EncodedBatch(out)

    def close(self):
        if self._h:
            lib().cgpu_encoder_destroy(self._h)
            self._h = ctypes.c_void_p()


class EncodedBatch:
    """cgpu_encoded: the columns of one batch in page-locked memory, owned by the library."""

    def __init__(self, h):
        self._h = h

    def batch(self, now_ns: int = 0) -> _Batch:
        b = _Batch()
        _check(lib().cgpu_encoded_batch(self._h, now_ns, ctypes.byref(b)))
        return b

    def columns(self):
        """copies of the twelve columns as uint8 arrays (tests)"""
        b = self.batch()
        return [np.frombuffer(ctypes.string_at(b.columns[i], b.column_bytes[i]), dtype=np.uint8).copy() for i in range(N_COLUMNS)]

    def narrow(self, form: int = 2):
        """cgpu_narrow_build: this batch in the narrow wire form (None when an id does not fit its narrow header field).
        Free the result before this batch."""
        out = ctypes.c_void_p()
        rc = lib().cgpu_narrow_build(self._h, form, ctypes.byref(out))
        if rc == ERR_UNSUPPORTED:
            return None
        _check(rc)
        return NarrowedBatch(out)

    def free(self):
        if self._h:
            lib().cgpu_encoded_free(self._h)
            self._h = None


class NarrowedBatch:
    """cgpu_narrowed: an encoded batch in the narrow wire form, built by the library (cb_narrow.h)."""

    def __init__(self, h):
        self._h = h

    def view(self, now_ns: int = 0):
        """-> (cgpu_batch, cgpu_narrow) argument blocks for Table.check_narrow_into; valid until free()"""
        b, nr = _Batch(), _Narrow()
        _check(lib().cgpu_narrowed_view(self._h, now_ns, ctypes.byref(b), ctypes.byref(nr)))
        return b, nr

    def free(self):
        if self._h:
            lib().cgpu_narrowed_free(self._h)
            self._h = None


class Context:
    """cgpu_ctx: one CUDA device (one process per GPU)."""

    def __init__(self, device=0):
        """device: an index, or a list of indices for one context over several GPUs (cgpu_check then shards every batch)."""
        self._h = ctypes.c_void_p()
        devs = list(device) if isinstance(device, (list, tuple)) else [device]
        ids = (ctypes.c_int * len(devs))(*devs)
        _check(lib().cgpu_init(ids, len(devs), ctypes.byref(self._h)))
        self.device = devs[0]
        self.devices = devs

    def close(self):
        if self._h:
            lib().cgpu_shutdown(self._h)
            self._h = ctypes.c_void_p()

    def launch_count(self) -> int:
        return int(lib().cgpu_launch_count(self._h))

    def deferred_count(self) -> int:
        """requests the lean / unique-condition kernels left to the general kernel so far (synchronises)"""
        n = ctypes.c_uint64()
        _check(lib().cgpu_deferred_count(self._h, ctypes.byref(n)))
        return n.value

    def last_kernel_config(self):
        g, b, s = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
        _check(lib().cgpu_last_kernel_config(self._h, ctypes.byref(g), ctypes.byref(b), ctypes.byref(s)))
        cfg = {"grid": g.value, "block": b.value, "smem_bytes": s.value & 0x7FFFFFFF, "lean_body": bool(s.value >> 31)}
        c, w, nb = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
        _check(lib().cgpu_last_cluster_config(self._h, ctypes.byref(c), ctypes.byref(w), ctypes.byref(nb)))
        cfg["clustered"] = bool(c.value & 1)
        cfg["tma_column_tiles"] = bool(c.value & 2)
        cfg["table_specialised"] = bool(c.value & 4)
        cfg["unique_conditions"] = bool(c.value & 8)
        if c.value & 1:
            cfg["cluster_window"] = w.value
            cfg["cluster_buckets"] = nb.value
        return cfg

    def profile(self, enable: bool):
        """-> (check-kernel ms summed, launches) since the last call; then turns per-launch events on/off."""
        ms, n = ctypes.c_double(), ctypes.c_uint64()
        _check(lib().cgpu_profile(self._h, 1 if enable else 0, ctypes.byref(ms), ctypes.byref(n)))
        return ms.value, n.value

    # ---- peer memory for the fused all-gather (cerbos_b200/dist.py: PeerGather)
    def peer_alloc(self, nbytes: int):
        """-> (device pointer, 64-byte IPC handle)"""
        ptr, h = ctypes.c_void_p(), ctypes.create_string_buffer(64)
        _check(lib().cgpu_peer_alloc(self._h, nbytes, ctypes.byref(ptr), h))
        return ptr.value, h.raw

    def peer_open(self, handle: bytes) -> int:
        ptr = ctypes.c_void_p()
        _check(lib().cgpu_peer_open(self._h, ctypes.create_string_buffer(handle, 64), ctypes.byref(ptr)))
        return ptr.value

    def peer_close(self, ptr: int):
        _check(lib().cgpu_peer_close(self._h, ctypes.c_void_p(ptr)))

    def peer_free(self, ptr: int):
        _check(lib().cgpu_peer_free(self._h, ctypes.c_void_p(ptr)))

    def peer_read(self, ptr: int, nbytes: int) -> np.ndarray:
        out = np.empty(nbytes, dtype=np.uint8)
        _check(lib().cgpu_peer_read(self._h, ctypes.c_void_p(ptr), out.ctypes.data_as(ctypes.c_void_p), nbytes))
        return out

    def gather_wait(self, local_flags_ptr: int, n_ranks: int, step: int, stream: int = 0):
        _check(lib().cgpu_gather_wait(self._h, ctypes.c_void_p(local_flags_ptr), n_ranks, step, ctypes.c_void_p(stream)))

    def load_table(self, blob: bytes) -> "Table":
        return Table(self, blob)

    def sync(self, stream: int = 0):
        _check(lib().cgpu_sync(self._h, ctypes.c_void_p(stream)))


class Table:
    """cgpu_table: flattened rule table resident in HBM (reference counted)."""

    def __init__(self, ctx: Context, blob: bytes):
        self.ctx = ctx
        self._h = ctypes.c_void_p()
        buf = (ctypes.c_char * len(blob)).from_buffer_copy(blob)
        _check(lib().cgpu_table_load(ctx._h, buf, len(blob), ctypes.byref(self._h)))

    def release(self):
        if self._h:
            lib().cgpu_table_release(self._h)
            self._h = ctypes.c_void_p()

    def wait_ready(self):
        """Blocks until the background compilation of the table-specialised kernels has finished.
        -> (specialised: bool, note: str)"""
        sp = ctypes.c_int()
        _check(lib().cgpu_table_wait_ready(self._h, ctypes.byref(sp)))
        return bool(sp.value), lib().cgpu_last_error().decode("utf-8", "replace")

    def meta(self):
        out = (ctypes.c_uint32 * 32)()
        _check(lib().cgpu_table_info(self._h, out, 32))
        return list(out)

    # ---- host-buffer path (engine.Check)
    def check(self, columns, n: int, max_actions: int, now_ns: int = 0, flags: int = 0) -> np.ndarray:
        """columns: numpy arrays in host memory (ideally pinned), encode.py order.
        Returns uint8[n, max_actions]: 1 ALLOW, 2 DENY, 0 padding."""
        cols = [c if (isinstance(c, np.ndarray) and c.flags["C_CONTIGUOUS"]) else np.ascontiguousarray(c) for c in columns]
        ptrs = (ctypes.c_void_p * len(cols))(*[c.ctypes.data for c in cols])
        sizes = (ctypes.c_size_t * len(cols))(*[c.nbytes for c in cols])
        b = _Batch(n, max_actions, now_ns, flags, ptrs, sizes, len(cols))
        out = np.empty((n, max(max_actions, 1)), dtype=np.uint8)
        _check(lib().cgpu_check(self.ctx._h, self._h, ctypes.byref(b), out.ctypes.data_as(ctypes.c_void_p)))
        return out

    def check_encoded(self, enc: "EncodedBatch", now_ns: int = 0) -> np.ndarray:
        """cgpu_check on a batch produced by the native encoder -> uint8[n, K] effects."""
        b = enc.batch(now_ns)
        out = np.empty((b.n_requests, max(b.max_actions, 1)), dtype=np.uint8)
        _check(lib().cgpu_check(self.ctx._h, self._h, ctypes.byref(b), out.ctypes.data_as(ctypes.c_void_p)))
        return out

    def prepare_narrow(self, nb, now_ns: int = 0, flags: int = 0, pin=None):
        """Argument block for cgpu_check_narrow from a cerbos_b200.narrow.NarrowBatch.  pin(array) -> (pointer, keepalive)
        lets the caller place the columns in page-locked memory; default: the numpy buffers themselves."""
        keep = []

        def ptr(a):
            a = np.ascontiguousarray(a)
            if pin is not None:
                p, k = pin(a)
                keep.append(k)
                return p
            keep.append(a)
            return a.ctypes.data

        tabs = [ptr(t) for t in nb.tables]
        sizes = [0, 0, 0, 0] + [int(np.asarray(t).nbytes) for t in nb.tables]
        cols = (ctypes.c_void_p * N_COLUMNS)(*([None] * 4 + tabs))
        csz = (ctypes.c_size_t * N_COLUMNS)(*sizes)
        b = _Batch(nb.n, nb.max_actions, now_ns, flags, cols, csz, N_COLUMNS)
        scols = (ctypes.c_void_p * max(len(nb.slot_cols), 1))(*[ptr(c) for c in nb.slot_cols])
        p16 = nb.principal_base is not None
        nr = _Narrow(None if p16 else ptr(nb.principal_id), ptr(nb.hdr16) if nb.hdr16.size else None, ptr(nb.versions) if nb.versions is not None else None,
                     ptr(nb.roles), nb.role_cols, ptr(nb.slot_class), scols, 1 if nb.heap_u32 else 0,
                     ptr(nb.slot_base), ptr(nb.slot_base2), ptr(nb.principal_id) if p16 else None, int(nb.principal_base or 0), int(nb.hdr_const_mask),
                     (ctypes.c_uint16 * 4)(*nb.hdr_const), 1 if nb.versions_value is not None else 0,
                     (ctypes.c_uint8 * 2)(*(nb.versions_value or (0, 0))), int(nb.heap_bits), int(nb.heap_base), int(nb.heap_base2))
        keep += [cols, csz, scols]
        return b, nr, keep

    def check_narrow_into(self, b, nr, out_ptr):
        _check(lib().cgpu_check_narrow(self.ctx._h, self._h, ctypes.byref(b), ctypes.byref(nr), ctypes.c_void_p(out_ptr)))

    def check_narrow(self, nb, now_ns: int = 0, flags: int = 0) -> np.ndarray:
        b, nr, keep = self.prepare_narrow(nb, now_ns, flags)
        out = np.empty((nb.n, max(nb.max_actions, 1)), dtype=np.uint8)
        self.check_narrow_into(b, nr, out.ctypes.data)
        return out

    def check_meta(self, columns, n: int, max_actions: int, now_ns: int = 0, flags: int = 0):
        """cgpu_check_meta: -> (effects uint8[n, K], action metadata words uint32[n, K], request metadata records
        (cerbos_b200.meta.REQUEST_META_DTYPE)); decode with cerbos_b200.meta."""
        from .meta import REQUEST_META_DTYPE
        cols = [c if (isinstance(c, np.ndarray) and c.flags["C_CONTIGUOUS"]) else np.ascontiguousarray(c) for c in columns]
        ptrs = (ctypes.c_void_p * len(cols))(*[c.ctypes.data for c in cols])
        sizes = (ctypes.c_size_t * len(cols))(*[c.nbytes for c in cols])
        b = _Batch(n, max_actions, now_ns, flags, ptrs, sizes, len(cols))
        km = max(max_actions, 1)
        eff = np.empty((n, km), dtype=np.uint8)
        am = np.empty((n, km), dtype=np.uint32)
        rm = np.empty(n, dtype=REQUEST_META_DTYPE)
        _check(lib().cgpu_check_meta(self.ctx._h, self._h, ctypes.byref(b), eff.ctypes.data_as(ctypes.c_void_p),
                                     am.ctypes.data_as(ctypes.c_void_p), rm.ctypes.data_as(ctypes.c_void_p)))
        return eff, am, rm

    def check_outputs(self, columns, n: int, max_actions: int, stride: int, now_ns: int = 0, flags: int = 0):
        """cgpu_check_outputs: check_meta's three outputs + the output records uint8[n, stride] (decode with
        cerbos_b200.outputs) + the size a record that did not fit needed (0 when all fit).  A failure raises CgpuError;
        after a record overflow its `bytes_needed` is that size."""
        from .meta import REQUEST_META_DTYPE
        cols = [c if (isinstance(c, np.ndarray) and c.flags["C_CONTIGUOUS"]) else np.ascontiguousarray(c) for c in columns]
        ptrs = (ctypes.c_void_p * len(cols))(*[c.ctypes.data for c in cols])
        sizes = (ctypes.c_size_t * len(cols))(*[c.nbytes for c in cols])
        b = _Batch(n, max_actions, now_ns, flags, ptrs, sizes, len(cols))
        km = max(max_actions, 1)
        eff = np.empty((n, km), dtype=np.uint8)
        am = np.empty((n, km), dtype=np.uint32)
        rm = np.empty(n, dtype=REQUEST_META_DTYPE)
        rec = np.empty((n, stride), dtype=np.uint8)
        need = ctypes.c_uint32(0)
        rc = lib().cgpu_check_outputs(self.ctx._h, self._h, ctypes.byref(b), eff.ctypes.data_as(ctypes.c_void_p), am.ctypes.data_as(ctypes.c_void_p),
                                      rm.ctypes.data_as(ctypes.c_void_p), rec.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint32(stride), ctypes.byref(need))
        if rc != OK:
            err = CgpuError(rc, lib().cgpu_last_error().decode("utf-8", "replace"))
            err.bytes_needed = need.value
            raise err
        return eff, am, rm, rec, need.value

    def check_narrow_meta(self, nb, now_ns: int = 0, flags: int = 0):
        """cgpu_check_narrow_meta: check_meta's three outputs from a batch in the narrow wire form -- a
        cerbos_b200.narrow.NarrowBatch, or a NarrowedBatch from the native encoder (EncodedBatch.narrow(form), whose own batch
        flags apply; `flags` is then ignored)."""
        from .meta import REQUEST_META_DTYPE
        if isinstance(nb, NarrowedBatch):
            b, nr = nb.view(now_ns)
        else:
            b, nr, _keep = self.prepare_narrow(nb, now_ns, flags)
        n, km = b.n_requests, max(b.max_actions, 1)
        eff = np.empty((n, km), dtype=np.uint8)
        am = np.empty((n, km), dtype=np.uint32)
        rm = np.empty(n, dtype=REQUEST_META_DTYPE)
        self.check_narrow_meta_into(b, nr, eff.ctypes.data, am.ctypes.data, rm.ctypes.data)
        return eff, am, rm

    def check_narrow_meta_into(self, b, nr, eff_ptr, action_meta_ptr, request_meta_ptr):
        """Zero-overhead variant for timing loops: argument blocks from prepare_narrow / NarrowedBatch.view, raw output pointers."""
        _check(lib().cgpu_check_narrow_meta(self.ctx._h, self._h, ctypes.byref(b), ctypes.byref(nr), ctypes.c_void_p(eff_ptr),
                                            ctypes.c_void_p(action_meta_ptr), ctypes.c_void_p(request_meta_ptr)))

    def check_into(self, ptrs, sizes, n, max_actions, out_ptr, now_ns=0, flags=0):
        """Zero-overhead variant for timing loops: raw host pointers in, effects written to out_ptr."""
        p = (ctypes.c_void_p * len(ptrs))(*ptrs)
        s = (ctypes.c_size_t * len(sizes))(*sizes)
        b = _Batch(n, max_actions, now_ns, flags, p, s, len(ptrs))
        _check(lib().cgpu_check(self.ctx._h, self._h, ctypes.byref(b), ctypes.c_void_p(out_ptr)))

    def prepared_device_call(self, ptrs, sizes, n, max_actions, bitmap_ptr, now_ns=0, flags=0):
        """Pre-builds the argument block once; returns f(stream) that only issues cgpu_check_device
        (keeps per-launch host overhead to the ctypes call itself)."""
        p = (ctypes.c_void_p * len(ptrs))(*ptrs)
        s = (ctypes.c_size_t * len(sizes))(*sizes)
        b = _Batch(n, max_actions, now_ns, flags, p, s, len(ptrs))
        fn, ctx_h, tab_h, bref, bm = lib().cgpu_check_device, self.ctx._h, self._h, ctypes.byref(b), ctypes.c_void_p(bitmap_ptr)
        keep = (p, s, b)

        def call(stream=0, _keep=keep):
            rc = fn(ctx_h, tab_h, bref, bm, ctypes.c_void_p(stream))
            if rc != OK:
                _check(rc)
        return call

    def prepared_gather_call(self, ptrs, sizes, n, max_actions, gather_bufs, flags, my_rank, slice_bytes, now_ns=0, batch_flags=0):
        """f(step, stream): cgpu_check_device_gather with pre-built arguments (results go straight into every rank's buffer)."""
        p = (ctypes.c_void_p * len(ptrs))(*ptrs)
        s = (ctypes.c_size_t * len(sizes))(*sizes)
        b = _Batch(n, max_actions, now_ns, batch_flags, p, s, len(ptrs))
        gb = (ctypes.c_void_p * len(gather_bufs))(*gather_bufs)
        fl = (ctypes.c_void_p * len(flags))(*flags)
        g = _Gather(len(gather_bufs), my_rank, gb, slice_bytes, fl, 0, 0, None)
        fn, ctx_h, tab_h, bref, gref = lib().cgpu_check_device_gather, self.ctx._h, self._h, ctypes.byref(b), ctypes.byref(g)
        keep = (p, s, b, gb, fl, g)

        def call(step, stream=0, wait_step=0, wait_flags=None, _keep=keep):
            g.step = step
            g.wait_step = wait_step
            g.wait_flags = wait_flags
            rc = fn(ctx_h, tab_h, bref, gref, ctypes.c_void_p(stream))
            if rc != OK:
                _check(rc)
        return call

    # ---- device-resident path
    def check_device(self, ptrs, sizes, n, max_actions, bitmap_ptr, now_ns=0, flags=0, stream=0):
        """ptrs: device pointers (e.g. torch tensor .data_ptr()); asynchronous on `stream` (cudaStream_t value)."""
        p = (ctypes.c_void_p * len(ptrs))(*ptrs)
        s = (ctypes.c_size_t * len(sizes))(*sizes)
        b = _Batch(n, max_actions, now_ns, flags, p, s, len(ptrs))
        _check(lib().cgpu_check_device(self.ctx._h, self._h, ctypes.byref(b), ctypes.c_void_p(bitmap_ptr),
                                       ctypes.c_void_p(stream)))
