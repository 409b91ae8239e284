/*
 * cerbos_b200.h -- C ABI of the H100-native batched CheckResources evaluator.
 *
 * This is the drop-in boundary for the reference's hot path.  What it replaces (cerbos/cerbos):
 *
 *   cgpu_table_load     the in-memory rule index built by ruletable.NewRuleTable / RuleTable.init /
 *                       indexRules (internal/ruletable/ruletable.go:517-601) and
 *                       index.Impl.IndexRules (internal/ruletable/index/index.go:353-437); called again
 *                       from the reload hooks Manager.reload / addPolicy / deletePolicy
 *                       (internal/ruletable/manager.go:88, 183, 198).
 *   cgpu_table_release  the RWMutex-guarded table swap of Manager (manager.go:28-35, 52-57): tables are
 *                       reference counted, release is safe while checks are in flight.
 *   cgpu_check          the body of Engine.Check -- checkSerial / checkParallel
 *                       (internal/engine/engine.go:229-235, 295-344) -> Manager.Check (manager.go:52-57)
 *                       -> RuleTable.check (ruletable.go:785-1155) -> SatisfiesCondition / cel-go
 *                       (ruletable.go:1346-1486).  Host buffers in, one effect byte per (input, action) out.
 *   cgpu_check_device   same evaluation for batches already resident in HBM (benchmarks, multi-GPU
 *                       sharding): no PCIe traffic, packed 1 bit / decision result.
 *
 * Conventions kept from the reference: results are index-aligned with the inputs (engine.go:308, 338); any
 * failure fails the whole call (engine.go:304-306) -- here a negative status plus cgpu_last_error();
 * `now` is fixed once per call (evaluator_trace_common.go:22-24); unsupported CEL is a *load-time* error
 * (the host flattener refuses to build the blob), unsupported run-time values (e.g. a timestamp outside
 * 1678..2262) fail the call with CGPU_ERR_UNSUPPORTED -- never a silent divergence, never a CPU fallback.
 *
 * Go owns all Go memory: nothing passed in is retained after a call returns, there are no callbacks.
 * The reference-side cgo binding is shown in INTEGRATION.md.
 */
#ifndef CERBOS_B200_H
#define CERBOS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct cgpu_ctx cgpu_ctx;     /* devices + stream pools; create once per process.  n_devices = 1: one GPU (one process
                                       * per GPU under torchrun / MPI); n_devices > 1: one process drives several GPUs --
                                       * cgpu_table_load places the table on every device, cgpu_check cuts a batch into one
                                       * index range per device (each over its own PCIe link), results stay index-aligned */
typedef struct cgpu_table cgpu_table; /* immutable flattened rule table resident in HBM */

enum cgpu_status {
    CGPU_OK = 0,
    CGPU_ERR_INVALID = -1,      /* bad argument / malformed blob or batch */
    CGPU_ERR_CUDA = -2,         /* CUDA runtime failure (message in cgpu_last_error) */
    CGPU_ERR_UNSUPPORTED = -3,  /* a request hit a run-time value the device cannot represent exactly */
    CGPU_ERR_NO_DEVICE = -4     /* no usable CUDA device: the product never falls back to a CPU path */
};

/* Effects as in api/public/cerbos/effect/v1/effect.proto */
#define CGPU_EFFECT_ALLOW 1
#define CGPU_EFFECT_DENY 2

/* Number of SoA columns in a batch and their order (layout documented in cerbos_b200/encode.py and
 * include/cerbos_b200_format.h; SURVEY.md 8(d) gives the per-request byte accounting). */
enum cgpu_column {
    CGPU_COL_HDR0 = 0,    /* cb_hdr0[N]            16 B / request */
    CGPU_COL_HDR1,        /* cb_hdr1[N]             8 B / request */
    CGPU_COL_ROLES,       /* u32[role_cols][N]                    */
    CGPU_COL_SLOTS,       /* u64[n_slots][N]  NaN-boxed attribute values */
    CGPU_COL_HEAP,        /* u64[]   lists / maps referenced from slots */
    CGPU_COL_BSTR_OFF,    /* u32[n_batch_strings + 1] */
    CGPU_COL_BSTR_BYTES,  /* u8[] */
    CGPU_COL_CLASS_OFF,   /* u32[n_classes + 1]  resource-kind class -> resource pattern ids */
    CGPU_COL_CLASS_PATS,  /* u32[] */
    CGPU_COL_ASET_K,      /* u32[n_asets]  number of actions of each distinct action list */
    CGPU_COL_ASET_SPREAD, /* u64[n_pass][n_asets][n_apats] */
    CGPU_COL_ROW_AM,      /* u64[n_pass][n_asets][n_rows]  action mask of every (merged) table row */
    CGPU_N_COLUMNS
};

typedef struct {
    uint64_t n_requests;
    uint32_t max_actions;      /* K: effects_out / bitmap row width */
    int64_t now_unix_nanos;    /* batch-constant now() */
    uint32_t flags;            /* bit0: lenient scope search (evaluator.Conf.LenientScopeSearch) */
    const void *const *columns;   /* CGPU_N_COLUMNS pointers (host memory for cgpu_check, device for *_device) */
    const size_t *column_bytes;
    uint32_t n_columns;
} cgpu_batch;

int cgpu_init(const int *device_ids, int n_devices, cgpu_ctx **out);
int cgpu_device_count(const cgpu_ctx *ctx);
void cgpu_shutdown(cgpu_ctx *ctx);

/* blob = host-built flattened table (cerbos_b200/table/flatten.py; Go: the same writer over runtimev1.RuleTable).
 * The blob is copied to HBM; the caller may free it when the call returns. */
int cgpu_table_load(cgpu_ctx *ctx, const void *blob, size_t len, cgpu_table **out);
void cgpu_table_retain(cgpu_table *t);
void cgpu_table_release(cgpu_table *t);

/* Host-buffer path (what engine.Check calls).  effects_out: n_requests * max_actions bytes, 1 = ALLOW, 2 = DENY,
 * 0 for slots beyond an input's own action count.  Re-entrant; blocks until the result is in effects_out. */
int cgpu_check(cgpu_ctx *ctx, const cgpu_table *t, const cgpu_batch *batch, uint8_t *effects_out);

/* ---- Narrow wire format: the same batch with its per-request columns in their narrowest exact form ---------------------
 * cgpu_check is bound by the PCIe link (the kernels take a few percent of a call), so what crosses it is what counts.
 * A host encoder that knows its dictionaries are small can send
 *   principal_id  u32[N]
 *   hdr16         u16[N][4]  kind class, resource scope, principal scope, action set: 0xFFFF = none, bit 15 = the CSR /
 *                            inexact flag of the 32-bit form (needs < 32767 patterns / scopes, < 65536 action sets)
 *   versions      u8[N][2]   resource, principal policy version id; 0xFF = none
 *   roles         u8[role_cols][N]   0xFF pad, 0xFE unknown role
 *   slot columns  per attribute slot one of CGPU_SLOT_*: u64 as is; u32 string id (0xFFFFFFFF absent, ..FE error, ..FD null,
 *                 ..FC false, ..FB true); u32 heap reference (bit 31 = map; specials as before); float32 when every number of
 *                 the column is exactly a float32 (specials = quiet NaNs with payload 1 absent, 2 error, 3 null); u8 (0 false,
 *                 1 true, 2 null, 3 absent, 4 error)
 *   heap          optionally u32 words: bit 31 clear = the word (element counts), set = string id (lists / maps of strings)
 * and a widening kernel rebuilds the canonical columns in HBM (1/100 of the PCIe cost).  `batch` carries the batch-level
 * tables (columns 4..11; column 4 = the u32 heap when heap_u32) and the scalars; its columns 0..3 are ignored. */
enum cgpu_slot_class { CGPU_SLOT_U64 = 0, CGPU_SLOT_U32_ID = 1, CGPU_SLOT_U32_HEAP = 2, CGPU_SLOT_F32 = 3, CGPU_SLOT_U8 = 4,
                       CGPU_SLOT_U16_ID = 5, CGPU_SLOT_U8_NUM = 6 };
typedef struct {
    const uint32_t *principal_id;
    const uint16_t *hdr16;
    const uint8_t *versions;
    const uint8_t *roles;
    uint32_t role_cols;
    const uint8_t *slot_class;        /* [table n_slots] */
    const void *const *slot_cols;     /* [table n_slots] */
    uint32_t heap_u32;
    /* Narrower still -- every field below is optional (zero / NULL = not used; a caller of the first form zero-fills them):
     *   CGPU_SLOT_U16_ID   u16 per request: w < 0x8000 = string id slot_base[v] + w, 0x8000 <= w < 0xFFF0 = string id slot_base2[v] +
     *                      (w - 0x8000); 0xFFFF absent, ..FE error, ..FD null, ..FC false, ..FB true.  Two windows because an
     *                      attribute's strings come from two dictionaries: the table's (constants the policies name, low ids)
     *                      and the batch's (numbered from n_table_strings in order of first appearance)
     *   CGPU_SLOT_U8_NUM   u8 per request = a number that is an integer in 0 .. 0xEF (0xFF absent, 0xFE error, 0xFD null)
     *   principal_id16     u16 = principal string id - principal_base, instead of principal_id
     *   hdr_const_mask     bit f set: header field f (0 kind class, 1 resource scope, 2 principal scope, 3 action set) has the same
     *                      16-bit value hdr_const[f] in every request; hdr16 then holds only the other fields, in order:
     *                      u16[N][4 - popcount(mask)] (NULL when all four are constant)
     *   versions_const     1: both policy version ids are the same in every request (versions_value); `versions` is ignored
     *   heap_bits          16: the heap as u16 words -- bit 15 clear = the word (element counts < 32768); set = a string id, bit 14
     *                      choosing the window: heap_base + (w & 0x3FFF) or heap_base2 + (w & 0x3FFF)
     *                      (overrides heap_u32; column 4 of `batch` is the u16 heap) */
    const uint32_t *slot_base;        /* [table n_slots] */
    const uint32_t *slot_base2;       /* [table n_slots] */
    const uint16_t *principal_id16;
    uint32_t principal_base;
    uint32_t hdr_const_mask;
    uint16_t hdr_const[4];
    uint32_t versions_const;
    uint8_t versions_value[2];
    uint32_t heap_bits;
    uint32_t heap_base, heap_base2;
} cgpu_narrow;
int cgpu_check_narrow(cgpu_ctx *ctx, const cgpu_table *t, const cgpu_batch *batch, const cgpu_narrow *narrow, uint8_t *effects_out);

/* ---- Native batch encoder: serialized enginev1.CheckInput messages -> the column batch cgpu_check takes ----------------
 * Replaces, on the host, the per-input string / map work of RuleTable.check (internal/ruletable/ruletable.go:785-884) and
 * the glob lookups over actions and resource kinds (internal/util/globs_common.go; glob_map.go:138-186).  The Go side
 * passes proto.Marshal of every enginev1.CheckInput it assembled (internal/svc/cerbos_svc.go:249-265); nothing is retained
 * after cgpu_encode returns.  An encoder belongs to one table blob (its dictionaries) and is immutable: share it freely
 * between goroutines, rebuild it when the table is reloaded.  The columns come back in page-locked memory. */
typedef struct cgpu_encoder cgpu_encoder;
typedef struct cgpu_encoded cgpu_encoded;
int cgpu_encoder_create(const void *blob, size_t len, const char *default_policy_version /* evaluator.Conf, NULL = "default" */,
                        const char *default_scope /* NULL = "" */, int lenient_scope_search, cgpu_encoder **out);
void cgpu_encoder_destroy(cgpu_encoder *e);
int cgpu_encode(const cgpu_encoder *e, const void *const *inputs, const size_t *input_bytes, uint64_t n, cgpu_encoded **out);
/* fills `out` so that it can be handed to cgpu_check / cgpu_check_meta; valid until cgpu_encoded_free */
int cgpu_encoded_batch(const cgpu_encoded *r, int64_t now_unix_nanos, cgpu_batch *out);
void cgpu_encoded_free(cgpu_encoded *r);

/* The encoded batch in the narrow wire form (above), built on the host from the canonical columns: protobuf -> cgpu_encode ->
 * cgpu_narrow_build -> cgpu_check_narrow needs no other host code.  form: 2 = everything the second half of cgpu_narrow
 * describes, 1 = the first form only.  Returns CGPU_ERR_UNSUPPORTED when an id of the batch does not fit its 16- / 8-bit
 * header field (the batch is then checked with cgpu_check).  The result borrows the batch-level tables of `enc`: free it first. */
typedef struct cgpu_narrowed cgpu_narrowed;
int cgpu_narrow_build(const cgpu_encoded *enc, int form, cgpu_narrowed **out);
int cgpu_narrowed_view(const cgpu_narrowed *nb, int64_t now_unix_nanos, cgpu_batch *batch_out, cgpu_narrow *narrow_out);
void cgpu_narrowed_free(cgpu_narrowed *nb);

/* Decision metadata (the reference's IncludeMeta responses and audit entries: ActionEffect.Policy / Scope and
 * CheckOutput.EffectiveDerivedRoles -- internal/ruletable/ruletable.go:753-782, 913-922, 936-979, 1082-1148;
 * internal/svc/cerbos_svc.go:291-311).  Same inputs as cgpu_check; besides the effect bytes it returns
 *   action_meta_out   n_requests * max_actions words: scope id of the deciding scope (0xFFFF none) | source << 16
 *                     (CB_META_SRC_*, cerbos_b200_format.h) | role id << 24 (role policies)
 *   request_meta_out  n_requests records: first scope of the principal / resource chain (the policy key's scope) and
 *                     the effective derived roles as a bit set over the table's derived-role names
 * ids index the dictionaries the host encoder already holds (table MANIFEST); the host assembles the strings
 * (cerbos_b200/meta.py; Go: namer.PolicyKeyFromFQN over the same ids).  An optional plane: cgpu_check moves no extra byte. */
int cgpu_check_meta(cgpu_ctx *ctx, const cgpu_table *t, const cgpu_batch *batch, uint8_t *effects_out,
                    uint32_t *action_meta_out, void *request_meta_out /* cb_request_meta[n_requests] */);

/* Device-resident path: columns are device pointers on ctx's device.  dev_bitmap_out receives
 * n_requests * ceil(max_actions / 8) bytes, bit (k % 8) of byte n * ceil(K/8) + k / 8 set <=> ALLOW.
 * Asynchronous on `cuda_stream` (a cudaStream_t, used exactly as given; NULL = the legacy default stream).
 * Unsupported run-time values are reported by the next cgpu_sync() on the same stream. */
int cgpu_check_device(cgpu_ctx *ctx, const cgpu_table *t, const cgpu_batch *dev_batch, void *dev_bitmap_out,
                      void *cuda_stream);
/* Waits for work queued by cgpu_check_device on `cuda_stream` and returns CGPU_ERR_UNSUPPORTED / CGPU_ERR_CUDA
 * if any of it failed. */
int cgpu_sync(cgpu_ctx *ctx, void *cuda_stream);

/* cgpu_table_load also starts, on a background thread, the generation + NVRTC compilation of kernels specialised for
 * this table (small tables whose conditions all have a flat form; seconds). Checks never wait for it: they use the
 * ahead-of-time generic kernels until it is done. This call does wait; *specialised = 1 if such kernels are in use
 * (otherwise cgpu_last_error() says why not). */
int cgpu_table_wait_ready(cgpu_table *t, int *specialised);
/* Generation + NVRTC compilation only, no device needed (build / CI check of the run-time path): *cubin_bytes = size of
 * the compiled module, 0 if the table does not qualify (cgpu_last_error() says why). */
int cgpu_table_compile_check(const void *blob, size_t len, size_t *cubin_bytes);

/* ---- Fused all-gather of the decision bitmaps over NVLink peer memory (one process per GPU on one node) --------
 * Every rank allocates a gather buffer of n_ranks * slice_bytes and a flag array with cgpu_peer_alloc, publishes the
 * 64-byte handles (any host channel: torch.distributed, MPI ...) and maps the others' with cgpu_peer_open.
 * cgpu_check_device_gather then makes the check kernels store each result byte straight into this rank's slice of
 * EVERY rank's buffer (own + peers), followed by a release of `step` into flags[my_rank] of every rank; no separate
 * collective runs. cgpu_gather_wait enqueues a wait on `stream` until every rank's slice of `step` has landed here. */
#define CGPU_IPC_HANDLE_BYTES 64
#define CGPU_MAX_GATHER_RANKS 8
typedef struct {
    uint32_t n_ranks, my_rank;
    void *const *gather_bufs;      /* [n_ranks] device pointers valid in THIS process (own buffer + mapped peers) */
    uint64_t slice_bytes;          /* bytes per rank slice: n_requests * ceil(max_actions / 8) */
    uint32_t *const *flags;        /* [n_ranks] each rank's flag array (uint32[n_ranks]), same convention */
    uint32_t step;                 /* monotonically increasing, > 0 */
    uint32_t wait_step;            /* 0, or: also hold the stream until every rank's slice of this (earlier) step has landed here */
    const uint32_t *wait_flags;    /* local flag array watched for wait_step (NULL: flags[my_rank]); callers that issue steps on
                                      several streams keep one flag array per stream so that each array only ever counts up */
} cgpu_gather;
int cgpu_peer_alloc(cgpu_ctx *ctx, size_t bytes, void **dev_ptr, void *ipc_handle_out);
int cgpu_peer_open(cgpu_ctx *ctx, const void *ipc_handle, void **dev_ptr);
int cgpu_peer_close(cgpu_ctx *ctx, void *dev_ptr);
int cgpu_peer_free(cgpu_ctx *ctx, void *dev_ptr);
int cgpu_peer_read(cgpu_ctx *ctx, const void *dev_ptr, void *host_out, size_t bytes);   /* tests: synchronous D2H */
int cgpu_check_device_gather(cgpu_ctx *ctx, const cgpu_table *t, const cgpu_batch *dev_batch, const cgpu_gather *g, void *cuda_stream);
int cgpu_gather_wait(cgpu_ctx *ctx, const uint32_t *local_flags, uint32_t n_ranks, uint32_t step, void *cuda_stream);

/* Introspection used by bench.py / tests (not part of the Go surface). */
uint64_t cgpu_launch_count(const cgpu_ctx *ctx);        /* kernels launched by this library so far */
int cgpu_table_info(const cgpu_table *t, uint32_t *meta_out, uint32_t n_words);  /* copies META words */
int cgpu_last_kernel_config(const cgpu_ctx *ctx, uint32_t *grid, uint32_t *block, uint32_t *smem_bytes);
/* Whether the last launch evaluated in clustered order (requests grouped by policy block inside L2-sized windows by
 * three small kernels ahead of the check kernel; env CERBOS_B200_CLUSTER=0/1 overrides the batch-size rule).
 * *clustered bit 0: clustered order; bit 1: the request columns were staged tile by tile through TMA; bit 2: the
 * kernel was the one compiled for this table at run time (NVRTC; env CERBOS_B200_NO_JIT=1 disables). */
int cgpu_last_cluster_config(const cgpu_ctx *ctx, uint32_t *clustered, uint32_t *window, uint32_t *buckets);
/* Returns and resets the CUDA-event time (ms) spent in the check kernel itself over the launches since the last
 * call, then switches the per-launch events on or off. Measurement aid for bench.py; off by default. */
int cgpu_profile(cgpu_ctx *ctx, int enable, double *kernel_ms_sum, uint64_t *n_launches);

const char *cgpu_last_error(void);   /* thread-local; valid until the next call on this thread */

#ifdef __cplusplus
}
#endif
#endif
