// cerbos_b200.cu -- sm_90a kernels + C ABI (include/cerbos_b200.h) of the batched CheckResources evaluator.
//
// Device bodies: cb_kernels.h (+ cb_core.h); this file holds the __global__ wrappers, the clustering kernels and the host side.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include "cb_core.h"
#include "cb_kernels.h"
#include "cb_specialize.h"
#include "cb_uc.h"
#include "cb_encode.h"
#include "cb_narrow.h"
#include "cb_host.h"
#include "cb_embed.inc"
#include "cerbos_b200.h"

namespace {

constexpr int kThreads = cbk::kThreads;
#ifndef CB_MIN_BLOCKS
#define CB_MIN_BLOCKS 4   // resident CTAs / SM the check kernel is register-budgeted for (64 registers per thread)
#endif
constexpr uint32_t kMaxStageBytes = 96 * 1024;   // table images up to this size are TMA-staged into shared memory
constexpr uint32_t kMaxTilesSmem = 56 * 1024;    // image + two column-tile stages: keeps CB_MIN_BLOCKS CTAs resident per SM

using cbk::TableDesc;
using cbk::smem_u32;

// Thin __global__ wrappers around the bodies in cb_kernels.h (generic block walker).
template <bool kFast, int kStageMode>
__global__ void __launch_bounds__(kThreads, CB_MIN_BLOCKS) check_kernel(const __grid_constant__ TableDesc td, const __grid_constant__ cb::BatchView bv, uint8_t *bitmap,
                                                                      uint8_t *effects, uint32_t *status, const uint32_t stage_rt) {
    extern __shared__ __align__(128) uint8_t smem_image[];
    __shared__ __align__(8) uint64_t mbar;
    cbk::check_body<kFast, kStageMode, cb::GenericBlocks>(td, bv, bitmap, effects, status, stage_rt, smem_image, &mbar);
}
__global__ void __launch_bounds__(kThreads, CB_MIN_BLOCKS) check_kernel_tiles(const __grid_constant__ TableDesc td, const __grid_constant__ cb::BatchView bv,
                                                                            uint8_t *bitmap, uint8_t *effects, uint32_t *status, const uint32_t n_slots) {
    extern __shared__ __align__(128) uint8_t smem_image[];
    __shared__ __align__(8) uint64_t mbar_tab, mbar_col[4];
    cbk::check_tiles_body<cb::GenericBlocks>(td, bv, bitmap, effects, status, n_slots, smem_image, &mbar_tab, mbar_col);
}

// decision-metadata kernel (cgpu_check_meta): one thread per request, the reference's own loop order (cb::eval_request_meta)
// Two resident CTAs (up to 128 registers), stated: left to ptxas, this kernel's register budget moves with the size of the
// interpreter's call graph, and it fell to 32 registers with heavy spills once the format printers joined it
// Also the drain of a unique-condition metadata launch (bv.count_dev: the deferral cell, bv.perm: its list), launched in
// stream order behind it: the last CTA hands the cell back zeroed, as check_body's drain does.
__global__ void __launch_bounds__(kThreads, 2) check_meta_kernel(const __grid_constant__ TableDesc td, const __grid_constant__ cb::BatchView bv, uint8_t *effects,
                                                             uint32_t *action_meta, cb_request_meta *req_meta, uint32_t *status) {
    const uint64_t count = bv.count_dev ? (uint64_t)*bv.count_dev : bv.count;
    for (uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x; i < count; i += (uint64_t)gridDim.x * kThreads)
        cb::eval_request_meta(td.base, &td.lay, &bv, bv.first + (bv.perm ? bv.perm[i] : i), effects, action_meta, req_meta, status);
    if (bv.count_dev) {
        __shared__ uint32_t last;
        __syncthreads();   // every thread of the CTA has read the count
        if (threadIdx.x == 0) {
            __threadfence();
            last = atomicAdd(bv.count_dev + 1, 1u) == gridDim.x - 1;
            if (blockIdx.x == 0) bv.count_dev[3] += (uint32_t)count;   // the running total of cgpu_deferred_count
        }
        __syncthreads();
        if (last && threadIdx.x == 0) { bv.count_dev[0] = 0; bv.count_dev[1] = 0; }
    }
}

// rule-output kernel (cgpu_check_outputs): check_meta_kernel's planes from the same reference-order walk, plus each request's
// output record, written to the chunk's output slab (record i of the slab: request bv.first + i)
__global__ void __launch_bounds__(kThreads, 2) check_outputs_kernel(const __grid_constant__ TableDesc td, const __grid_constant__ cb::BatchView bv, uint8_t *effects,
                                                                uint32_t *action_meta, cb_request_meta *req_meta, uint32_t *status, uint8_t *out_slab,
                                                                uint32_t stride, uint32_t *needed) {
    for (uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x; i < bv.count; i += (uint64_t)gridDim.x * kThreads) {
        uint8_t *rec = out_slab + i * stride;
        cb::eval_request_outputs(td.base, &td.lay, &bv, bv.first + i, effects, action_meta, req_meta, status, rec, stride);
        const uint32_t need = reinterpret_cast<const cb_out_record *>(rec)->bytes_needed;
        if (need > stride) atomicMax(needed, need);
    }
}

// ---- narrow wire format (cgpu_check_narrow): the per-request columns travel over PCIe in their narrowest exact form and are
// widened to the canonical columns here, in HBM, right before the check kernels read them
constexpr uint32_t kMaxNarrowSlots = 64;
struct WidenParams {
    const uint32_t *pid; const uint16_t *hdr16; const uint8_t *versions; const uint8_t *roles;
    const void *slot_src[kMaxNarrowSlots];
    uint8_t slot_class[kMaxNarrowSlots];
    cb_hdr0 *hdr0; cb_hdr1 *hdr1; uint32_t *roles_out; uint64_t *slots_out;
    uint64_t first, count, stride;
    uint32_t role_cols, n_slots;
    // the narrower forms (cgpu_narrow, second half): per-slot base of the 16-bit string ids, 16-bit principal ids, header
    // fields / versions that are constant over the batch
    uint32_t slot_base[kMaxNarrowSlots], slot_base2[kMaxNarrowSlots];
    const uint16_t *pid16; uint32_t pid_base;
    uint32_t hdr_const_mask, hdr_w; uint16_t hdr_const[4];
    uint32_t versions_const; uint8_t versions_value[2];
};
__device__ __forceinline__ uint64_t widen_special(uint32_t code) {   // 0 absent, 1 error, 2 null
    return (uint64_t)(CB_V64_BOX_BASE | (code == 0 ? CB_V64_ABSENT : code == 1 ? CB_V64_ERROR : CB_V64_NULL)) << 48;
}
__global__ void __launch_bounds__(kThreads) widen_kernel(const __grid_constant__ WidenParams p) {
    for (uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x; i < p.count; i += (uint64_t)gridDim.x * kThreads) {
        const uint64_t n = p.first + i;
        uint32_t f16[4];   // kind, resource scope, principal scope, action set
        if (p.hdr_const_mask == 0) {
            const uint2 h = reinterpret_cast<const uint2 *>(p.hdr16)[n];
            f16[0] = h.x & 0xFFFF; f16[1] = h.x >> 16; f16[2] = h.y & 0xFFFF; f16[3] = h.y >> 16;
        } else {
            const uint16_t *hp = p.hdr16 + n * p.hdr_w;
            uint32_t q = 0;
            for (uint32_t f = 0; f < 4; f++) f16[f] = (p.hdr_const_mask >> f) & 1u ? p.hdr_const[f] : hp[q++];
        }
        const uint32_t k16 = f16[0], rs16 = f16[1], ps16 = f16[2], aset = f16[3];
        cb_hdr0 h0;
        h0.principal_id = p.pid16 ? p.pid_base + p.pid16[n] : p.pid[n];
        h0.kind_class = k16 == 0xFFFF ? CB_KIND_NONE : (k16 & 0x8000) ? ((k16 & 0x7FFF) | CB_KIND_CLASS_CSR_BIT) : k16;
        h0.resource_scope = rs16 == 0xFFFF ? CB_SCOPE_NONE : (rs16 & 0x8000) ? ((rs16 & 0x7FFF) | CB_SCOPE_INEXACT_BIT) : rs16;
        h0.principal_scope = ps16 == 0xFFFF ? CB_SCOPE_NONE : (ps16 & 0x8000) ? ((ps16 & 0x7FFF) | CB_SCOPE_INEXACT_BIT) : ps16;
        p.hdr0[n] = h0;
        const uint32_t rv = p.versions_const ? p.versions_value[0] : p.versions[2 * n], pv = p.versions_const ? p.versions_value[1] : p.versions[2 * n + 1];
        cb_hdr1 h1;
        h1.resource_version = (uint16_t)(rv == 0xFF ? CB_NONE16 : rv); h1.principal_version = (uint16_t)(pv == 0xFF ? CB_NONE16 : pv); h1.action_set_id = aset;
        p.hdr1[n] = h1;
        for (uint32_t c = 0; c < p.role_cols; c++) {
            const uint32_t r = p.roles[(uint64_t)c * p.stride + n];
            p.roles_out[(uint64_t)c * p.stride + n] = r == 0xFF ? CB_ROLE_PAD : r == 0xFE ? CB_ROLE_UNKNOWN : r;
        }
        for (uint32_t v = 0; v < p.n_slots; v++) {
            uint64_t out;
            switch (p.slot_class[v]) {
            case CGPU_SLOT_U32_ID: {      // string id | specials | bool
                const uint32_t w = static_cast<const uint32_t *>(p.slot_src[v])[n];
                if (w < 0xFFFFFFF0u) out = ((uint64_t)(CB_V64_BOX_BASE | CB_V64_STRING) << 48) | w;
                else if (w >= 0xFFFFFFFDu) out = widen_special(0xFFFFFFFFu - w);
                else out = ((uint64_t)(CB_V64_BOX_BASE | CB_V64_BOOL) << 48) | (w == 0xFFFFFFFBu ? 1u : 0u);
                break;
            }
            case CGPU_SLOT_U32_HEAP: {    // list / map in the batch heap | specials
                const uint32_t w = static_cast<const uint32_t *>(p.slot_src[v])[n];
                if (w >= 0xFFFFFFFDu) out = widen_special(0xFFFFFFFFu - w);
                else out = ((uint64_t)(CB_V64_BOX_BASE | ((w & 0x80000000u) ? CB_V64_MAP : CB_V64_LIST)) << 48) | CB_V64_HEAP_BATCH_BIT | (w & 0x7FFFFFFFu);
                break;
            }
            case CGPU_SLOT_F32: {         // a double that float32 holds exactly | specials as NaN payloads
                const uint32_t w = static_cast<const uint32_t *>(p.slot_src[v])[n];
                if ((w & 0x7FC00000u) == 0x7FC00000u && (w & 0x3FFFFFu)) out = widen_special((w & 3u) - 1u);
                else if (w == 0x7FC00000u) out = CB_V64_CANON_NAN;
                else out = (uint64_t)__double_as_longlong((double)__uint_as_float(w));
                break;
            }
            case CGPU_SLOT_U8: {          // 0 false, 1 true, 2 null, 3 absent, 4 error
                const uint32_t w = static_cast<const uint8_t *>(p.slot_src[v])[n];
                out = w <= 1 ? (((uint64_t)(CB_V64_BOX_BASE | CB_V64_BOOL) << 48) | w) : widen_special(w == 3 ? 0u : w == 4 ? 1u : 2u);
                break;
            }
            case CGPU_SLOT_U16_ID: {      // string id - base | specials | bool
                const uint32_t w = static_cast<const uint16_t *>(p.slot_src[v])[n];
                if (w < 0xFFF0u) out = ((uint64_t)(CB_V64_BOX_BASE | CB_V64_STRING) << 48) | (uint64_t)(w < 0x8000u ? p.slot_base[v] + w : p.slot_base2[v] + (w - 0x8000u));
                else if (w >= 0xFFFDu) out = widen_special(0xFFFFu - w);
                else out = ((uint64_t)(CB_V64_BOX_BASE | CB_V64_BOOL) << 48) | (w == 0xFFFBu ? 1u : 0u);
                break;
            }
            case CGPU_SLOT_U8_NUM: {      // a small non-negative integer (as the double it is) | specials
                const uint32_t w = static_cast<const uint8_t *>(p.slot_src[v])[n];
                out = w >= 0xFDu ? widen_special(0xFFu - w) : (uint64_t)__double_as_longlong((double)w);
                break;
            }
            default: out = static_cast<const uint64_t *>(p.slot_src[v])[n]; break;
            }
            p.slots_out[(uint64_t)v * p.stride + n] = out;
        }
    }
}
// heap words in 32 bits: bit 31 clear = the word itself (counts, zero-extended), set = a string id (boxed STRING)
__global__ void __launch_bounds__(kThreads) widen_heap_kernel(const uint32_t *src, uint64_t *dst, uint64_t n) {
    for (uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) {
        const uint32_t w = src[i];
        dst[i] = (w & 0x80000000u) ? (((uint64_t)(CB_V64_BOX_BASE | CB_V64_STRING) << 48) | (w & 0x7FFFFFFFu)) : (uint64_t)w;
    }
}

// heap words in 16 bits: bit 15 clear = the word itself, set = a string id in one of two windows (bit 14)
__global__ void __launch_bounds__(kThreads) widen_heap16_kernel(const uint16_t *src, uint64_t *dst, uint64_t n, uint32_t base, uint32_t base2) {
    for (uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) {
        const uint32_t w = src[i];
        dst[i] = (w & 0x8000u) ? (((uint64_t)(CB_V64_BOX_BASE | CB_V64_STRING) << 48) | (uint64_t)(((w & 0x4000u) ? base2 : base) + (w & 0x3FFFu))) : (uint64_t)w;
    }
}

// ------------------------------------------------------------------------------------------- host side: errors, narrow wire
thread_local std::string g_err;

int fail(int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}
#define CUDA_TRY(expr)                                                                                   \
    do {                                                                                                 \
        cudaError_t e__ = (expr);                                                                        \
        if (e__ != cudaSuccess) return fail(CGPU_ERR_CUDA, "%s failed: %s", #expr, cudaGetErrorString(e__)); \
    } while (0)

// The narrow wire on the host (a descriptor narrow_args accepted): the columns are staged in the slot's device buffer
constexpr uint8_t kNarrowElemBytes[] = {8, 4, 4, 4, 1, 2, 1};   // bytes per request of a slot column, by CGPU_SLOT_* class
inline uint32_t narrow_hdr_w(const cgpu_narrow &nb) { return 4u - (uint32_t)__builtin_popcount(nb.hdr_const_mask & 15u); }   // header fields that travel

// Byte offsets of one call's data in its slot's device buffer (slot_layout), in this order, each region rounded up to 256
// bytes; a region the call does not use is empty (offset 0 behind the effect bytes)
struct SlotLayout {
    size_t col[CGPU_N_COLUMNS], effects;                                           // the canonical columns, the effect bytes
    struct { size_t pid, hdr16, versions, roles, slot[kMaxNarrowSlots], heap; } narrow;   // a narrow batch's columns as they travel
    size_t action_meta, request_meta;                                             // the metadata planes
    size_t needed, out; uint64_t out_chunk;   // rule outputs: the needed-size word, two slabs of out_chunk records
    size_t total;
};

// The widening parameters of one call but its chunk (first / count), over the slot's device buffer `dev`, columns of stride N
WidenParams widen_params(const cgpu_narrow &nb, uint64_t N, uint32_t n_slots, uint8_t *dev, const SlotLayout &L) {
    WidenParams wp{};
    wp.pid = reinterpret_cast<const uint32_t *>(dev + L.narrow.pid); wp.pid16 = nb.principal_id16 ? reinterpret_cast<const uint16_t *>(dev + L.narrow.pid) : nullptr;
    wp.pid_base = nb.principal_base; wp.hdr16 = reinterpret_cast<const uint16_t *>(dev + L.narrow.hdr16);
    wp.hdr_const_mask = nb.hdr_const_mask; wp.hdr_w = narrow_hdr_w(nb);
    for (int f = 0; f < 4; f++) wp.hdr_const[f] = nb.hdr_const[f];
    wp.versions = dev + L.narrow.versions; wp.versions_const = nb.versions_const; wp.versions_value[0] = nb.versions_value[0]; wp.versions_value[1] = nb.versions_value[1];
    wp.roles = dev + L.narrow.roles; wp.role_cols = nb.role_cols;
    for (uint32_t v = 0; v < n_slots; v++) {
        wp.slot_src[v] = dev + L.narrow.slot[v]; wp.slot_class[v] = nb.slot_class[v];
        wp.slot_base[v] = nb.slot_base ? nb.slot_base[v] : 0u; wp.slot_base2[v] = nb.slot_base2 ? nb.slot_base2[v] : 0u;
    }
    wp.hdr0 = reinterpret_cast<cb_hdr0 *>(dev + L.col[CGPU_COL_HDR0]); wp.hdr1 = reinterpret_cast<cb_hdr1 *>(dev + L.col[CGPU_COL_HDR1]);
    wp.roles_out = reinterpret_cast<uint32_t *>(dev + L.col[CGPU_COL_ROLES]); wp.slots_out = reinterpret_cast<uint64_t *>(dev + L.col[CGPU_COL_SLOTS]);
    wp.stride = N; wp.n_slots = n_slots;
    return wp;
}

// Requests [first, first + count): their narrow columns go H2D into the staging; once they have landed, widened on `stream`
int upload_narrow_chunk(const cgpu_narrow &nb, WidenParams &wp, uint64_t first, uint64_t count, cudaStream_t h2d, cudaEvent_t landed, cudaStream_t stream,
                        std::atomic<uint64_t> &launches) {
    auto copy = [&](const void *staged, const void *src, size_t bytes) { return cudaMemcpyAsync(const_cast<void *>(staged), src, bytes, cudaMemcpyHostToDevice, h2d); };
    if (nb.principal_id16) CUDA_TRY(copy(wp.pid16 + first, nb.principal_id16 + first, count * 2));
    else CUDA_TRY(copy(wp.pid + first, nb.principal_id + first, count * 4));
    if (wp.hdr_w) CUDA_TRY(copy(wp.hdr16 + first * wp.hdr_w, nb.hdr16 + first * wp.hdr_w, count * 2 * wp.hdr_w));
    if (!nb.versions_const) CUDA_TRY(copy(wp.versions + first * 2, nb.versions + first * 2, count * 2));
    for (uint32_t i = 0; i < nb.role_cols; i++) CUDA_TRY(copy(wp.roles + i * wp.stride + first, nb.roles + i * wp.stride + first, count));
    for (uint32_t v = 0; v < wp.n_slots; v++) {
        const uint32_t es = kNarrowElemBytes[wp.slot_class[v]];
        CUDA_TRY(copy(static_cast<const uint8_t *>(wp.slot_src[v]) + first * es, static_cast<const uint8_t *>(nb.slot_cols[v]) + first * es, count * es));
    }
    CUDA_TRY(cudaEventRecord(landed, h2d));
    CUDA_TRY(cudaStreamWaitEvent(stream, landed, 0));
    wp.first = first; wp.count = count;
    const uint64_t tiles = (count + kThreads - 1) / kThreads;
    widen_kernel<<<(unsigned)(tiles < 1184 ? tiles : 1184), kThreads, 0, stream>>>(wp);
    CUDA_TRY(cudaGetLastError());
    launches.fetch_add(1, std::memory_order_relaxed);
    return CGPU_OK;
}

// unique-condition kernels (cb_uc.h image; generic condition evaluator; deferrals go to the launch's list)
template <bool kStaged>
__global__ void __launch_bounds__(kThreads, CB_MIN_BLOCKS) check_uc(const __grid_constant__ TableDesc td, const __grid_constant__ cb::BatchView bv, uint8_t *bitmap,
                                                                  uint8_t *effects, uint32_t *status, const uint32_t) {
    extern __shared__ __align__(128) uint8_t smem_image[];
    __shared__ __align__(8) uint64_t mbar;
    (void)status;
    cbk::check_uc_body<cb::GenericConds, cb::CachedCols, kStaged>(td, bv, bitmap, effects, smem_image, &mbar);
}
// ... their metadata form (cgpu_check_meta): effects, action words and request records; side: cbuc::build_meta's table
template <bool kStaged>
__global__ void __launch_bounds__(kThreads, CB_MIN_BLOCKS) check_uc_meta(const __grid_constant__ TableDesc td, const __grid_constant__ cb::BatchView bv, uint8_t *effects,
                                                                       uint32_t *action_meta, cb_request_meta *req_meta, const cb::U4 *side) {
    extern __shared__ __align__(128) uint8_t smem_image[];
    __shared__ __align__(8) uint64_t mbar;
    cbk::check_uc_body<cb::GenericConds, cb::CachedCols, kStaged>(td, bv, nullptr, effects, smem_image, &mbar, cbk::UcMeta{action_meta, req_meta, side});
}

// ------------------------------------------------------------------------------------------------ fused all-gather
struct SignalParams { uint32_t *flags[cb::CB_MAX_GATHER]; const uint32_t *wait_flags; uint32_t n_ranks, my_rank, step, wait_step; };
// After the check kernels of a gather launch: publish `step` into this rank's cell of every rank's flag array.
// Programmatically serialised behind them; their peer stores are complete (and visible system-wide) once they have.
// Pre-pass of a unique-condition launch that reads its table image from global memory: the image's rows merged with the
// batch's row x action-set masks into one 16-byte record per (action set, row) -- what the staged kernels build in
// shared memory per CTA.  One load per row in the walk instead of two dependent ones.
__global__ void __launch_bounds__(kThreads) uc_merge_rows(const __grid_constant__ TableDesc td, const __grid_constant__ cb::BatchView bv, cb::U4 *out, const uint32_t n_pk) {
    const uint32_t j = blockIdx.x * kThreads + threadIdx.x;
    if (j >= n_pk) return;
    cb::TableView tv;
    tv.base = td.base; tv.L = &td.lay;
    const uint32_t n_u = td.lay.uc_n_rows;
    cb::UcRowsGlobal g; g.urows = tv.urows(); g.row_am = bv.row_am; g.RCP = bv.rcp; g.nR = td.lay.nR;
    out[j] = g.aset(tv, bv, j / n_u).merged(tv, j % n_u);
}

__global__ void gather_signal(const __grid_constant__ SignalParams p) {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    __threadfence_system();
    if (threadIdx.x < p.n_ranks) asm volatile("red.release.sys.global.max.u32 [%0], %1;" ::"l"(p.flags[threadIdx.x] + p.my_rank), "r"(p.step) : "memory");
    if (p.wait_step) cbk::gather_wait_flags(p.wait_flags, p.n_ranks, p.wait_step);
}
// Stream-side wait: until the slice of every rank for `step` has landed in this rank's gather buffer.
__global__ void gather_wait(const uint32_t *flags, uint32_t n_ranks, uint32_t step) {
    if (threadIdx.x < n_ranks) {
        uint32_t v;
        do {
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + threadIdx.x) : "memory");
        } while ((int32_t)(v - step) < 0);
    }
}

// ------------------------------------------------------------------------------------------------ clustering
// Requests of one batch hit different policy blocks (resource kind x scope x version); evaluated in index order the
// 32 lanes of a warp would each walk another block and another set of conditions.  Three small kernels build a
// permutation that groups requests by that key inside windows of `window` requests (a window's columns fit in L2,
// so the gathers of the check kernel are served from L2 and DRAM traffic stays at the algorithmic bytes):
//   cluster_count   keys (u16) + per-(window, bucket) histogram      reads hdr0 / hdr1 once, coalesced
//   cluster_scan    exclusive scan of every window's histogram
//   cluster_scatter perm[window base + bucket offset + rank] = request offset
constexpr uint32_t kClusterChunk = 2048;   // requests per CTA (8 per thread)
constexpr uint32_t kMaxBuckets = 4096;

struct ClusterParams {
    const cb_hdr0 *hdr0;
    const cb_hdr1 *hdr1;
    uint64_t first;
    uint32_t count, window, nb;   // nb: buckets (power of two <= kMaxBuckets)
    uint32_t nV, nRP, nS;
    uint16_t *keys;
    uint32_t *hist;               // [n_windows][nb]
    uint32_t *perm;
};

__device__ __forceinline__ uint32_t cluster_key(const ClusterParams &p, uint64_t n) {
    const cb::U4 h0 = cb::ldcol128(p.hdr0 + n);
    const uint64_t h1 = cb::ldcol64(reinterpret_cast<const uint64_t *>(p.hdr1 + n));
    uint32_t kc = h0.y & ~CB_KIND_CLASS_CSR_BIT, rs = h0.z & ~CB_SCOPE_INEXACT_BIT, rv = (uint32_t)(h1 & 0xFFFF);
    kc = kc < p.nRP ? kc : p.nRP;
    rs = rs < p.nS ? rs : p.nS;
    rv = rv < p.nV ? rv : p.nV;
    return ((rv * (p.nRP + 1) + kc) * (p.nS + 1) + rs) & (p.nb - 1);
}

__global__ void __launch_bounds__(kThreads) cluster_count(const __grid_constant__ ClusterParams p) {
    __shared__ uint32_t hist[kMaxBuckets];
    for (uint32_t j = threadIdx.x; j < p.nb; j += kThreads) hist[j] = 0;
    __syncthreads();
    const uint32_t c0 = blockIdx.x * kClusterChunk;
    for (uint32_t q = 0; q < kClusterChunk / kThreads; q++) {
        const uint32_t i = c0 + q * kThreads + threadIdx.x;
        if (i < p.count) {
            const uint32_t k = cluster_key(p, p.first + i);
            p.keys[i] = (uint16_t)k;
            atomicAdd(&hist[k], 1u);
        }
    }
    __syncthreads();
    uint32_t *g = p.hist + (uint64_t)(c0 / p.window) * p.nb;
    for (uint32_t j = threadIdx.x; j < p.nb; j += kThreads)
        if (hist[j]) atomicAdd(g + j, hist[j]);
}

__global__ void __launch_bounds__(kThreads) cluster_scan(const __grid_constant__ ClusterParams p) {
    __shared__ uint32_t part[kThreads];
    uint32_t *g = p.hist + (uint64_t)blockIdx.x * p.nb;
    const uint32_t per = (p.nb + kThreads - 1) / kThreads;   // consecutive buckets per thread
    const uint32_t j0 = threadIdx.x * per;
    uint32_t sum = 0;
    for (uint32_t j = j0; j < j0 + per && j < p.nb; j++) sum += g[j];
    part[threadIdx.x] = sum;
    __syncthreads();
    for (uint32_t d = 1; d < kThreads; d <<= 1) {   // Hillis-Steele inclusive scan over the 256 partial sums
        uint32_t v = threadIdx.x >= d ? part[threadIdx.x - d] : 0;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    uint32_t run = part[threadIdx.x] - sum;
    for (uint32_t j = j0; j < j0 + per && j < p.nb; j++) { uint32_t c = g[j]; g[j] = run; run += c; }
}

__global__ void __launch_bounds__(kThreads) cluster_scatter(const __grid_constant__ ClusterParams p) {
    __shared__ uint32_t hist[kMaxBuckets];
    for (uint32_t j = threadIdx.x; j < p.nb; j += kThreads) hist[j] = 0;
    __syncthreads();
    const uint32_t c0 = blockIdx.x * kClusterChunk;
    uint32_t key[kClusterChunk / kThreads], rank[kClusterChunk / kThreads];
#pragma unroll
    for (uint32_t q = 0; q < kClusterChunk / kThreads; q++) {
        const uint32_t i = c0 + q * kThreads + threadIdx.x;
        key[q] = 0; rank[q] = 0;
        if (i < p.count) { key[q] = p.keys[i]; rank[q] = atomicAdd(&hist[key[q]], 1u); }
    }
    __syncthreads();
    uint32_t *g = p.hist + (uint64_t)(c0 / p.window) * p.nb;
    for (uint32_t j = threadIdx.x; j < p.nb; j += kThreads)
        if (hist[j]) hist[j] = atomicAdd(g + j, hist[j]);   // this CTA's range inside the bucket
    __syncthreads();
    const uint32_t wbase = (c0 / p.window) * p.window;
#pragma unroll
    for (uint32_t q = 0; q < kClusterChunk / kThreads; q++) {
        const uint32_t i = c0 + q * kThreads + threadIdx.x;
        if (i < p.count) p.perm[wbase + hist[key[q]] + rank[q]] = i;
    }
}

// ------------------------------------------------------------------------------------------- host side: check launches
struct Slot {   // per in-flight cgpu_check call
    cudaStream_t stream = nullptr;                 // kernels
    cudaStream_t h2d = nullptr, d2h = nullptr;     // column chunks in, effect bytes out (PCIe is full duplex)
    std::vector<cudaEvent_t> ev;                   // two per chunk: columns landed, results ready
    void *dev = nullptr;
    size_t dev_cap = 0;
    uint32_t *h_status = nullptr;   // pinned
    uint32_t *d_status = nullptr;
    bool busy = false;
};

// The main kernel of a check launch (plan_launch picks it, kernel_fn maps it to its entry point).  The kernels from
// SpecTiles on are compiled for the table at run time (NVRTC, cb_specialize.h).
enum class Kernel : uint8_t {
    General, GeneralGlobal,         // check_kernel<false, 2>: general body, table image staged / read from global memory
    Lean, LeanGlobal, LeanTiles,    // check_kernel<true, 1> / <true, 0>, check_kernel_tiles (request columns through TMA)
    Uc, UcGlobal,                   // check_uc<true> / <false>
    SpecTiles, SpecDirect,          // cb_spec_tiles / cb_spec_direct (block-shape form)
    SpecUc, SpecUcGlobal,           // cb_spec_uc / cb_spec_uc_global (unique-condition form)
    // metadata forms of the four unique-condition kernels (cgpu_check_meta): check_uc_meta<true> / <false>,
    // cb_spec_uc_meta / cb_spec_uc_meta_global
    UcMeta, UcMetaGlobal, SpecUcMeta, SpecUcMetaGlobal,
};
constexpr int kKernels = (int)Kernel::SpecUcMetaGlobal + 1;

// What one check launch runs: plan_launch decides it, launch_check executes it.
struct LaunchPlan {
    Kernel kernel = Kernel::General;
    uint32_t smem = 0;          // dynamic shared memory of the main kernel
    uint32_t last_arg = 0;      // its last argument: stage_rt (check_kernel, cb_spec_direct) or n_slots (column tiles)
    bool stage = false;         // the table image is staged in shared memory (general and lean bodies)
    bool lean = false;          // lean body: the requests it defers go to a list the general kernel drains right behind it
    bool uc = false;            // unique-condition kernel
    bool uc_staged = false;     // ... with its compact image and merged rows in shared memory
    bool col_tiles = false;     // request columns staged tile by tile through TMA
    bool cluster = false;       // clustered evaluation order
    bool spec = false;          // the kernel compiled for this table at run time
    bool strpred = false;       // the kernel reads per-string predicate words (filled by cb_spec_strpred)
    bool merge_rows = false;    // uc_merge_rows pre-pass
    bool serialise = false;     // programmatically serialised behind the previous launch's drain kernel
};

// A device buffer of a deferral lane.  fit() grows it to a power of two of at least min_cap elements, stream-ordered: the
// old buffer is released only after everything queued on this stream so far -- the only launches that can still read
// it -- has completed.
template <class T> struct LaneBuf {
    T *ptr = nullptr;
    size_t cap = 0;
    cudaError_t fit(size_t n, size_t min_cap, cudaStream_t stream) {
        if (cap >= n) return cudaSuccess;
        size_t c = min_cap;
        while (c < n) c <<= 1;
        T *fresh = nullptr;
        const cudaError_t e = cudaMallocAsync(reinterpret_cast<void **>(&fresh), c * sizeof(T), stream);
        if (e != cudaSuccess) return e;
        T *old = ptr;
        ptr = fresh;
        cap = c;
        return old ? cudaFreeAsync(old, stream) : cudaSuccess;
    }
};

}  // namespace

struct cgpu_ctx {
    int device = 0;
    int sm_count = 0;
    uint32_t *d_status = nullptr;       // for cgpu_check_device / cgpu_sync
    std::atomic<uint64_t> launches{0};
    std::mutex mu;
    std::vector<Slot> slots;
    // the last check launch (cgpu_last_kernel_config / cgpu_last_cluster_config); window / buckets: the last clustered one
    LaunchPlan last_plan;
    uint32_t last_grid = 0, last_window = 0, last_buckets = 0;
    int force_no_stage = 0;
    int force_general = 0;   // CERBOS_B200_FORCE_GENERAL=1: never pick the lean kernel body (tests)
    int cluster_mode = -1;   // CERBOS_B200_CLUSTER: 0 never, 1 always, unset = batches of >= kClusterMinRequests
    int force_no_tiles = 0;  // CERBOS_B200_NO_TILES=1: never stage request columns through TMA (tests)
    int force_no_jit = 0;    // CERBOS_B200_NO_JIT=1: never compile table-specialised kernels (tests)
    // Deferral state is owned by the STREAM a launch is issued on (a cgpu_check slot has its own stream): launches on one
    // stream complete in order, and with programmatic launch chaining at most three consecutive ones are in flight
    // together (k draining, k+1 running, k+2 starting), so every stream rotates over four lists / counter cells of its own.
    struct DeferLane {
        uint32_t seq = 0;
        uint32_t *cells = nullptr;   // 4 x {count, done, tile counter, drained total}, count / done zero between uses (the drain kernel re-zeroes)
        struct Bufs {
            LaneBuf<uint32_t> list;
            LaneBuf<uint32_t> strpred;   // per-string predicate words of the specialised unique-condition kernels
            LaneBuf<cb::U4> pk;          // merged row records of unique-condition launches on a global image
        } q[4];
    };
    std::map<cudaStream_t, DeferLane> defer_lanes;
    std::mutex defer_mu;
    // copy-engine result exchange (cgpu_check_device_gather, large slices): a side stream + a ring of events
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t copy_ev[16] = {};
    uint32_t copy_seq = 0;
    struct SliceUse { const void *ptr; cudaEvent_t done; uint8_t *stage; size_t stage_bytes; };   // stage: where the kernels write (plain device memory)
    std::vector<SliceUse> slice_uses;   // own slices whose last push to the peers may still be in flight
    std::mutex copy_mu;
    std::vector<cgpu_ctx *> peers;   // cgpu_init with n_devices > 1: the contexts of devices 1..n-1 (owned)
    int uc_mode = -1;        // CERBOS_B200_UC: 0 never use the unique-condition kernels, 1 whenever the table allows, unset = tables with > 1 block shape
    bool profiling = false;  // cgpu_profile(): CUDA events around the check kernel of every launch
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    double prof_ms = 0;
    uint64_t prof_n = 0;
    bool prof_pending = false;
};

struct cgpu_encoder { cbenc::Encoder enc; };
struct cgpu_encoded {
    cbenc::Columns cols;
    void *pinned = nullptr;              // one page-locked block holding all twelve columns (null: no CUDA device, columns stay in `cols`)
    size_t pinned_cap = 0;               // (the block comes from / returns to the staging pool)
    const void *ptrs[CGPU_N_COLUMNS] = {};
    size_t bytes[CGPU_N_COLUMNS] = {};
    uint32_t flags = 0;
    uint32_t n_slots = 0, role_cols = 1;   // of the table / of this batch (cgpu_narrow_build)
};
struct cgpu_narrowed {
    cbnarrow::Narrowed nb;
    const cgpu_encoded *enc = nullptr;
    void *pinned = nullptr;                // one page-locked block holding every narrow column (null: no CUDA device, they stay in `nb`)
    bool pinned_is_malloc = false;         // tests without a device: the same single-block layout in plain memory (CERBOS_B200_NARROW_BLOCK=1)
    size_t pinned_cap = 0;
    const void *pid = nullptr, *hdr16 = nullptr, *versions = nullptr, *roles = nullptr, *heap = nullptr;
    std::vector<const void *> slot_ptrs;
    size_t heap_bytes = 0;
    const void *cols[CGPU_N_COLUMNS] = {};
    size_t col_bytes[CGPU_N_COLUMNS] = {};
};

struct cgpu_table {
    cgpu_ctx *ctx = nullptr;
    std::atomic<int> refs{1};
    uint8_t *d_image = nullptr;
    TableDesc desc{};
    uint32_t meta[CB_META_WORDS]{};
    // resident CTAs / SM per kernel (resident_ctas): footprint << 32 | CTAs in one word, 0 = not queried yet
    mutable std::atomic<uint64_t> occ[kKernels]{};
    // table-specialised lean kernels (cb_specialize.h), compiled with NVRTC on first use
    std::vector<uint8_t> host_image;
    std::mutex spec_mu;
    std::atomic<int> spec_state{0};   // 0 not tried, 1 ready, -1 unavailable
    cudaLibrary_t spec_lib = nullptr;
    cudaKernel_t spec_tiles = nullptr, spec_direct = nullptr, spec_uc = nullptr, spec_uc_global = nullptr, spec_strpred = nullptr;
    cudaKernel_t spec_uc_meta = nullptr, spec_uc_meta_global = nullptr;
    uint32_t spec_n_strpred = 0;   // string predicates the specialised unique-condition kernel reads from the per-string pre-pass
    std::string spec_note;
    // unique-condition image (cb_uc.h): compact copy of the table for tables whose blocks differ in shape
    uint64_t sec_len[cbhost::kMaxSec]{};
    std::vector<cgpu_table *> peer_tables;   // the same table on the other devices of a multi-device context (owned)
    cbuc::Image uc;
    uint8_t *d_uc_image = nullptr;
    TableDesc uc_desc{};
    cbuc::MetaSide uc_meta;            // side table of the metadata forms of the unique-condition kernels (cb_uc.h: build_meta)
    cb::U4 *d_uc_meta = nullptr;       // (own allocation: the image the effect kernels read stays as it is)
    std::thread spec_thread;          // compiles the specialised kernels in the background from cgpu_table_load on
    std::mutex join_mu;
};

namespace {

// A shared host check (cb_host.h) that failed: its message becomes the error of the call.
int invalid(const std::string &why) { return why.empty() ? CGPU_OK : fail(CGPU_ERR_INVALID, "%s", why.c_str()); }

// ---------------------------------------------------------------------------------------------- run-time specialisation
// NVRTC is loaded lazily with dlopen: a host without it simply keeps the ahead-of-time (generic) kernels.
struct Nvrtc {
    void *h = nullptr;
    int (*create)(void **, const char *, const char *, int, const char *const *, const char *const *) = nullptr;
    int (*compile)(void *, int, const char *const *) = nullptr;
    int (*log_size)(void *, size_t *) = nullptr;
    int (*log)(void *, char *) = nullptr;
    int (*cubin_size)(void *, size_t *) = nullptr;
    int (*cubin)(void *, char *) = nullptr;
    int (*destroy)(void **) = nullptr;
    bool ok = false;
};
Nvrtc &nvrtc() {
    static Nvrtc n;
    static std::once_flag once;
    std::call_once(once, [] {
        for (const char *name : {"libnvrtc.so.12", "libnvrtc.so"}) {
            n.h = dlopen(name, RTLD_NOW | RTLD_LOCAL);
            if (n.h) break;
        }
        if (!n.h) return;
        n.create = reinterpret_cast<decltype(n.create)>(dlsym(n.h, "nvrtcCreateProgram"));
        n.compile = reinterpret_cast<decltype(n.compile)>(dlsym(n.h, "nvrtcCompileProgram"));
        n.log_size = reinterpret_cast<decltype(n.log_size)>(dlsym(n.h, "nvrtcGetProgramLogSize"));
        n.log = reinterpret_cast<decltype(n.log)>(dlsym(n.h, "nvrtcGetProgramLog"));
        n.cubin_size = reinterpret_cast<decltype(n.cubin_size)>(dlsym(n.h, "nvrtcGetCUBINSize"));
        n.cubin = reinterpret_cast<decltype(n.cubin)>(dlsym(n.h, "nvrtcGetCUBIN"));
        n.destroy = reinterpret_cast<decltype(n.destroy)>(dlsym(n.h, "nvrtcDestroyProgram"));
        n.ok = n.create && n.compile && n.log_size && n.log && n.cubin_size && n.cubin && n.destroy;
    });
    return n;
}

const char kSpecPrelude[] =
    "#define CB_LEAN_ONLY 1\n"
    "#ifndef CB_SPEC_MIN_BLOCKS\n#define CB_SPEC_MIN_BLOCKS 5\n#endif\n"
    "typedef unsigned char uint8_t; typedef unsigned short uint16_t; typedef unsigned int uint32_t; typedef unsigned long long uint64_t;\n"
    "typedef signed char int8_t; typedef short int16_t; typedef int int32_t; typedef long long int64_t; typedef unsigned long long uintptr_t;\n";
const char kSpecKernels[] =
    "\nextern \"C\" __global__ void __launch_bounds__(256, CB_SPEC_MIN_BLOCKS) cb_spec_tiles(const __grid_constant__ cbk::TableDesc td, const __grid_constant__ cb::BatchView bv,\n"
    "        uint8_t *bitmap, uint8_t *effects, uint32_t *status, const uint32_t n_slots) {\n"
    "    extern __shared__ __align__(128) uint8_t smem_image[];\n"
    "    __shared__ __align__(8) uint64_t mbar_tab, mbar_col[4];\n"
    "    cbk::check_tiles_body<cb::SpecBlocks>(td, bv, bitmap, effects, status, n_slots, smem_image, &mbar_tab, mbar_col);\n"
    "}\n"
    "extern \"C\" __global__ void __launch_bounds__(256, CB_SPEC_MIN_BLOCKS) cb_spec_direct(const __grid_constant__ cbk::TableDesc td, const __grid_constant__ cb::BatchView bv,\n"
    "        uint8_t *bitmap, uint8_t *effects, uint32_t *status, const uint32_t stage_rt) {\n"
    "    extern __shared__ __align__(128) uint8_t smem_image[];\n"
    "    __shared__ __align__(8) uint64_t mbar;\n"
    "    cbk::check_body<true, 1, cb::SpecBlocks>(td, bv, bitmap, effects, status, stage_rt, smem_image, &mbar);\n"
    "}\n";
// unique-condition form: the compact image staged in shared memory, every distinct condition as straight-line code
const char kSpecUcStaged[] =
    "\nextern \"C\" __global__ void __launch_bounds__(256, CB_SPEC_UC_MIN_BLOCKS) cb_spec_uc(const __grid_constant__ cbk::TableDesc td, const __grid_constant__ cb::BatchView bv,\n"
    "        uint8_t *bitmap, uint8_t *effects, uint32_t *status, const uint32_t) {\n"
    "    extern __shared__ __align__(128) uint8_t smem_image[];\n"
    "    __shared__ __align__(8) uint64_t mbar;\n"
    "    cbk::check_uc_body<cb::SpecConds, cb::GlobalCols, true>(td, bv, bitmap, effects, smem_image, &mbar);\n"
    "}\n";
// the same body with the image and the rows read from global memory (L2 / L1): images too large for shared memory
const char kSpecUcGlobal[] =
    "\nextern \"C\" __global__ void __launch_bounds__(256, CB_SPEC_UC_MIN_BLOCKS) cb_spec_uc_global(const __grid_constant__ cbk::TableDesc td, const __grid_constant__ cb::BatchView bv,\n"
    "        uint8_t *bitmap, uint8_t *effects, uint32_t *status, const uint32_t) {\n"
    "    cbk::check_uc_body<cb::SpecConds, cb::GlobalCols, false>(td, bv, bitmap, effects, nullptr, nullptr);\n"
    "}\n";
// metadata forms of the two (cgpu_check_meta; side: cbuc::build_meta's table)
const char kSpecUcMetaStaged[] =
    "\nextern \"C\" __global__ void __launch_bounds__(256, CB_SPEC_UC_MIN_BLOCKS) cb_spec_uc_meta(const __grid_constant__ cbk::TableDesc td, const __grid_constant__ cb::BatchView bv,\n"
    "        uint8_t *effects, uint32_t *action_meta, cb_request_meta *req_meta, const cb::U4 *side) {\n"
    "    extern __shared__ __align__(128) uint8_t smem_image[];\n"
    "    __shared__ __align__(8) uint64_t mbar;\n"
    "    cbk::check_uc_body<cb::SpecConds, cb::GlobalCols, true>(td, bv, nullptr, effects, smem_image, &mbar, cbk::UcMeta{action_meta, req_meta, side});\n"
    "}\n";
const char kSpecUcMetaGlobal[] =
    "\nextern \"C\" __global__ void __launch_bounds__(256, CB_SPEC_UC_MIN_BLOCKS) cb_spec_uc_meta_global(const __grid_constant__ cbk::TableDesc td, const __grid_constant__ cb::BatchView bv,\n"
    "        uint8_t *effects, uint32_t *action_meta, cb_request_meta *req_meta, const cb::U4 *side) {\n"
    "    cbk::check_uc_body<cb::SpecConds, cb::GlobalCols, false>(td, bv, nullptr, effects, nullptr, nullptr, cbk::UcMeta{action_meta, req_meta, side});\n"
    "}\n";
// pre-pass over the string dictionary (table strings, then the batch's): one predicate word per string
const char kSpecUcStrpred[] =
    "\nextern \"C\" __global__ void __launch_bounds__(256) cb_spec_strpred(const __grid_constant__ cbk::TableDesc td, const __grid_constant__ cb::BatchView bv, uint32_t *out, const uint32_t n) {\n"
    "    const uint32_t id = blockIdx.x * 256u + threadIdx.x;\n"
    "    cb::TableView tv; tv.base = td.base; tv.L = &td.lay;\n"
    "    if (id < n) out[id] = cb::SpecConds().strpred(tv, bv, id);\n"
    "}\n";

uint64_t fnv1a(const void *p, size_t n, uint64_t h = 1469598103934665603ull) {
    const uint8_t *b = static_cast<const uint8_t *>(p);
    for (size_t i = 0; i < n; i++) { h ^= b[i]; h *= 1099511628211ull; }
    return h;
}
// Compiled modules are cached on disk under their source hash (CERBOS_B200_CACHE_DIR, default ~/.cache/cerbos_b200;
// CERBOS_B200_CACHE_DIR="" disables): a PDP restarting with the same policy set skips the NVRTC compile.
std::string cache_path(uint64_t key) {
    const char *d = getenv("CERBOS_B200_CACHE_DIR");
    std::string dir;
    if (d) { if (!d[0]) return ""; dir = d; }
    else { const char *home = getenv("HOME"); if (!home || !home[0]) return ""; dir = std::string(home) + "/.cache/cerbos_b200"; }
    char name[64];
    snprintf(name, sizeof name, "/spec_%016llx.cubin", (unsigned long long)key);
    return dir + name;
}
bool cache_read(const std::string &path, std::vector<char> *out) {
    if (path.empty()) return false;
    FILE *f = fopen(path.c_str(), "rb");
    if (!f) return false;
    fseek(f, 0, SEEK_END);
    const long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    bool ok = n > 0;
    if (ok) { out->resize((size_t)n); ok = fread(out->data(), 1, (size_t)n, f) == (size_t)n; }
    fclose(f);
    return ok;
}
void cache_write(const std::string &path, const std::vector<char> &data) {
    if (path.empty()) return;
    const std::string dir = path.substr(0, path.rfind('/'));
    for (size_t i = 1; i <= dir.size(); i++)
        if (i == dir.size() || dir[i] == '/') mkdir(dir.substr(0, i).c_str(), 0755);
    const std::string tmp = path + ".tmp" + std::to_string((unsigned long long)getpid());
    FILE *f = fopen(tmp.c_str(), "wb");
    if (!f) return;
    const bool ok = fwrite(data.data(), 1, data.size(), f) == data.size();
    fclose(f);
    if (ok) rename(tmp.c_str(), path.c_str()); else remove(tmp.c_str());
}

// Which specialised form a table gets: per-shape block evaluators when its blocks share (nearly) one shape, else the
// unique-condition form when every distinct condition has a flat form.  `gen` receives the generated source.
enum SpecForm { SPEC_NONE = 0, SPEC_SHAPES = 1, SPEC_UC = 2 };
constexpr uint32_t kUcMaxSmem = 72 * 1024;   // compact image + merged rows: three CTAs / SM at least

// Shared memory of a staged unique-condition launch: the compact image, then one 16-byte merged row per (action set, slot or image row).
uint64_t uc_smem_bytes(const cbuc::Image &uc, uint64_t n_pk) { return (((uint64_t)uc.lay.image_bytes + 127) & ~127ull) + 16 * n_pk; }
// Whether the staged unique-condition kernel fits with n_pk merged rows.  With one (the default) it is the question whether
// the image leaves room at all, which decides whether the specialised translation unit carries the staged kernel.
bool uc_stageable(const cbuc::Image &uc, uint64_t n_pk = 1) { return uc_smem_bytes(uc, n_pk) <= kUcMaxSmem; }

SpecForm spec_generate(const uint8_t *image, const cb::TableLayout &lay, const uint32_t *meta, const cbuc::Image &uc, std::string *gen, std::string *why, uint32_t *n_strpred,
                       uint32_t *n_atoms = nullptr) {
    *n_strpred = 0;
    if (n_atoms) *n_atoms = 0;
    // the specialised kernels are lean bodies: a table that can never take a lean kernel needs none
    if (!cbhost::lean_table(lay, meta)) {
        *why = "table is not lean-eligible (principal / role policies, parent roles or resource globs): general kernel only";
        return SPEC_NONE;
    }
    if (lay.image_bytes <= kMaxStageBytes) {
        *gen = cbspec::generate(image, lay.off, meta);
        if (!gen->empty()) return SPEC_SHAPES;
    }
    if (uc.ok) {   // any image size: cb_spec_uc stages the image in shared memory, cb_spec_uc_global reads it through L2 / L1
        cbspec::UcSource us = cbspec::generate_uc(uc.bytes.data(), uc.lay.off, uc.lay.uc_conds_off, uc.n_uconds, lay.n_slots, meta[CB_META_N_CONSTS]);
        *gen = us.src;
        *n_strpred = us.n_strpred;
        if (n_atoms) *n_atoms = us.n_atoms;
        if (!gen->empty()) return SPEC_UC;
    }
    *why = "table does not qualify (too many block shapes and: more than 127 distinct conditions, or a condition program the translator does not take -- "
           "list / map literals, collecting comprehensions, runtime.effectiveDerivedRoles)";
    return SPEC_NONE;
}

// Generates the table's specialised translation unit and compiles it with NVRTC (no CUDA runtime call: also works on
// a host without a GPU).  SPEC_NONE + *why when the table does not qualify or something is unavailable.
SpecForm spec_compile(const uint8_t *image, const cb::TableLayout &lay, const uint32_t *meta, const cbuc::Image &uc, std::vector<char> *cubin, std::string *why, uint32_t *n_strpred) {
    std::string gen;
    uint32_t n_atoms = 0;
    const SpecForm form = spec_generate(image, lay, meta, uc, &gen, why, n_strpred, &n_atoms);
    if (form == SPEC_NONE) return SPEC_NONE;
    std::string src = kSpecPrelude;
    if (n_atoms) src += "#define CB_SPEC_PROGRAMS 1\n";   // leaf programs call the value helpers of cb_core.h
    for (const char *const *p = kEmbedFormat; *p; p++) src += *p;
    for (const char *const *p = kEmbedCore; *p; p++) src += *p;
    src += gen;
    for (const char *const *p = kEmbedKernels; *p; p++) src += *p;
    if (form == SPEC_UC) {
        // an image that can never be staged (larger than the shared-memory budget of the staged kernel) gets the global
        // variant only, a small one both: which of the two a launch takes also depends on the batch's action sets
        if (uc_stageable(uc)) { src += kSpecUcStaged; src += kSpecUcMetaStaged; }
        src += kSpecUcGlobal;
        src += kSpecUcMetaGlobal;
        src += kSpecUcStrpred;
    } else src += kSpecKernels;
    const char *mb = getenv("CERBOS_B200_SPEC_BLOCKS");   // experiments: resident CTAs / SM the specialised kernels are budgeted for
    const std::string mbopt = std::string("-DCB_SPEC_MIN_BLOCKS=") + (mb && mb[0] >= '1' && mb[0] <= '8' && !mb[1] ? mb : "5");
    const char *ub = getenv("CERBOS_B200_SPEC_UC_BLOCKS");
    // leaf programs keep whole values (tag + payload) in registers: budget 128 registers / thread for them, 80 otherwise
    // (at 64, C3's register-resident slots and lists spill to local memory; on an H100, 3 CTAs / SM at 80 registers run
    // C3 in 2.28 ms per 2^24 batch against 3.03 ms at 4 CTAs / SM)
    const std::string ubopt = std::string("-DCB_SPEC_UC_MIN_BLOCKS=") + (ub && ub[0] >= '1' && ub[0] <= '8' && !ub[1] ? ub : n_atoms ? "2" : "3");
    if (const char *dump = getenv("CERBOS_B200_SPEC_DUMP")) {   // profiling aid: the translation unit handed to NVRTC
        if (FILE *f = fopen(dump, "w")) { fwrite(src.data(), 1, src.size(), f); fclose(f); }
    }
    std::vector<std::string> defs;   // experiments: extra -D options for the generated translation unit, space separated
    if (const char *xd = getenv("CERBOS_B200_SPEC_DEFS")) {
        std::string cur;
        for (const char *c = xd;; c++) {
            if (*c == ' ' || *c == 0) { if (!cur.empty()) defs.push_back(cur); cur.clear(); if (!*c) break; }
            else cur += *c;
        }
    }
    uint64_t key = fnv1a(ubopt.data(), ubopt.size(), fnv1a(mbopt.data(), mbopt.size(), fnv1a(src.data(), src.size())));
    for (const std::string &d : defs) key = fnv1a(d.data(), d.size(), key);
    const std::string cpath = cache_path(key);
    if (cache_read(cpath, cubin)) return form;
    Nvrtc &n = nvrtc();
    if (!n.ok) { *why = "libnvrtc not available"; return SPEC_NONE; }
    void *prog = nullptr;
    if (n.create(&prog, src.c_str(), "cerbos_b200_spec.cu", 0, nullptr, nullptr) != 0) { *why = "nvrtcCreateProgram failed"; return SPEC_NONE; }
    std::vector<const char *> opts = {"--gpu-architecture=sm_90a", "-std=c++17", "-lineinfo", mbopt.c_str(), ubopt.c_str()};
    for (const std::string &d : defs) opts.push_back(d.c_str());
    if (n_atoms) opts.push_back("--device-int128");   // parse_duration_text (cb_core.h) scales fractions in 128 bits
    const int rc = n.compile(prog, (int)opts.size(), opts.data());
    if (rc != 0) {
        size_t ls = 0;
        n.log_size(prog, &ls);
        std::string log(ls, '\0');
        if (ls) n.log(prog, &log[0]);
        n.destroy(&prog);
        *why = "NVRTC compile failed: " + log.substr(0, 600);
        return SPEC_NONE;
    }
    size_t cs = 0;
    n.cubin_size(prog, &cs);
    cubin->resize(cs);
    n.cubin(prog, cubin->data());
    n.destroy(&prog);
    cache_write(cpath, *cubin);
    return form;
}

// Compiles and loads the table's specialised kernels (once; thread-safe). Returns whether they are usable.
bool ensure_spec(cgpu_ctx *ctx, cgpu_table *t) {
    int st = t->spec_state.load(std::memory_order_acquire);
    if (st != 0) return st > 0;
    std::lock_guard<std::mutex> g(t->spec_mu);
    st = t->spec_state.load(std::memory_order_acquire);
    if (st != 0) return st > 0;
    auto give_up = [&](const std::string &why) { t->spec_note = why; t->spec_state.store(-1, std::memory_order_release); return false; };
    if (ctx->force_no_jit) return give_up("disabled (CERBOS_B200_NO_JIT)");
    std::vector<char> cubin;
    std::string why;
    const SpecForm form = spec_compile(t->host_image.data(), t->desc.lay, t->meta, t->uc, &cubin, &why, &t->spec_n_strpred);
    if (form == SPEC_NONE) return give_up(why);
    if (cudaLibraryLoadData(&t->spec_lib, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0) != cudaSuccess) { cudaGetLastError(); return give_up("cudaLibraryLoadData failed"); }
    bool got = form == SPEC_UC ? (!uc_stageable(t->uc) || (cudaLibraryGetKernel(&t->spec_uc, t->spec_lib, "cb_spec_uc") == cudaSuccess &&
                                                            cudaLibraryGetKernel(&t->spec_uc_meta, t->spec_lib, "cb_spec_uc_meta") == cudaSuccess)) &&
                                     cudaLibraryGetKernel(&t->spec_uc_global, t->spec_lib, "cb_spec_uc_global") == cudaSuccess &&
                                     cudaLibraryGetKernel(&t->spec_uc_meta_global, t->spec_lib, "cb_spec_uc_meta_global") == cudaSuccess &&
                                     cudaLibraryGetKernel(&t->spec_strpred, t->spec_lib, "cb_spec_strpred") == cudaSuccess
                               : cudaLibraryGetKernel(&t->spec_tiles, t->spec_lib, "cb_spec_tiles") == cudaSuccess &&
                                     cudaLibraryGetKernel(&t->spec_direct, t->spec_lib, "cb_spec_direct") == cudaSuccess;
    if (!got) {
        cudaGetLastError();
        cudaLibraryUnload(t->spec_lib);
        t->spec_lib = nullptr;
        t->spec_tiles = t->spec_direct = t->spec_uc = t->spec_uc_global = t->spec_strpred = nullptr;
        t->spec_uc_meta = t->spec_uc_meta_global = nullptr;
        return give_up("cudaLibraryGetKernel failed");
    }
    t->spec_note = "ok";
    t->spec_state.store(1, std::memory_order_release);
    return true;
}

constexpr uint64_t kClusterMinRequests = 32768;
constexpr uint64_t kClusterWindowBytes = 12u << 20;   // columns of one window: comfortably inside the 50 MB L2 of an H100

// Builds the clustered evaluation order of `bv` on `stream` (stream-ordered scratch); *perm_out is freed by the caller.
int launch_cluster(cgpu_ctx *ctx, const cgpu_table *t, const cb::BatchView &bv, uint32_t **perm_out, cudaStream_t stream) {
    const cb::TableLayout &lay = t->desc.lay;
    ClusterParams p{};
    p.hdr0 = bv.hdr0; p.hdr1 = bv.hdr1; p.first = bv.first; p.count = (uint32_t)bv.count;
    p.nV = lay.nV; p.nRP = lay.nRP; p.nS = lay.nS;
    const uint64_t nkeys = (uint64_t)(lay.nV + 1) * (lay.nRP + 1) * (lay.nS + 1);
    p.nb = 32;
    while (p.nb < nkeys && p.nb < kMaxBuckets) p.nb <<= 1;
    // window: a power of two number of requests whose header + role + slot columns take about kClusterWindowBytes,
    // at least 64 requests per bucket
    const uint64_t per_req = 24 + 4ull * bv.role_cols + 8ull * lay.n_slots + 16;
    uint64_t w = kClusterChunk;
    while (w * 2 * per_req <= kClusterWindowBytes) w <<= 1;
    while (w < 64ull * p.nb && w < (1ull << 22)) w <<= 1;
    p.window = (uint32_t)w;
    const uint32_t n_win = (uint32_t)((bv.count + w - 1) / w);
    const uint32_t n_chunks = (uint32_t)((bv.count + kClusterChunk - 1) / kClusterChunk);
    const size_t perm_bytes = ((size_t)bv.count * 4 + 255) & ~(size_t)255, keys_bytes = ((size_t)bv.count * 2 + 255) & ~(size_t)255;
    const size_t hist_bytes = (size_t)n_win * p.nb * 4;
    uint8_t *scratch = nullptr;
    CUDA_TRY(cudaMallocAsync(reinterpret_cast<void **>(&scratch), perm_bytes + keys_bytes + hist_bytes, stream));
    p.perm = reinterpret_cast<uint32_t *>(scratch);
    p.keys = reinterpret_cast<uint16_t *>(scratch + perm_bytes);
    p.hist = reinterpret_cast<uint32_t *>(scratch + perm_bytes + keys_bytes);
    CUDA_TRY(cudaMemsetAsync(p.hist, 0, hist_bytes, stream));
    cluster_count<<<n_chunks, kThreads, 0, stream>>>(p);
    cluster_scan<<<n_win, kThreads, 0, stream>>>(p);
    cluster_scatter<<<n_chunks, kThreads, 0, stream>>>(p);
    CUDA_TRY(cudaGetLastError());
    ctx->launches.fetch_add(3, std::memory_order_relaxed);
    ctx->last_window = p.window; ctx->last_buckets = p.nb;
    *perm_out = p.perm;
    return CGPU_OK;
}

// The launch's deferral list + counter cell, and the pre-pass buffers it asks for (n_strpred / n_pk elements; 0: none,
// the pointer is then null), owned by the stream it is issued on (see cgpu_ctx::DeferLane).
int acquire_defer(cgpu_ctx *ctx, cudaStream_t stream, uint64_t count, uint32_t **list, uint32_t **cell, size_t n_strpred, uint32_t **strpred,
                  size_t n_pk, cb::U4 **pk) {
    std::lock_guard<std::mutex> g(ctx->defer_mu);
    cgpu_ctx::DeferLane &ln = ctx->defer_lanes[stream];
    if (!ln.cells) {
        CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(&ln.cells), 4 * 16));
        CUDA_TRY(cudaMemset(ln.cells, 0, 4 * 16));
    }
    const uint32_t q = ln.seq++ & 3;
    cgpu_ctx::DeferLane::Bufs &b = ln.q[q];
    CUDA_TRY(b.list.fit(count, 1024, stream));
    if (n_strpred) CUDA_TRY(b.strpred.fit(n_strpred, 4096, stream));
    if (n_pk) CUDA_TRY(b.pk.fit(n_pk, 4096, stream));
    *list = b.list.ptr;
    *cell = ln.cells + 4 * q;   // {count, done, tile counter, drained total}
    *strpred = n_strpred ? b.strpred.ptr : nullptr;
    *pk = n_pk ? b.pk.ptr : nullptr;
    return CGPU_OK;
}

// Which kernels one check launch runs, and how: from the table, the batch and the context's switches alone (no CUDA call).
LaunchPlan plan_launch(const cgpu_ctx &ctx, const cgpu_table &t, const cb::BatchView &bv) {
    const cb::TableLayout &lay = t.desc.lay;
    LaunchPlan p;
    p.stage = !ctx.force_no_stage && lay.image_bytes <= kMaxStageBytes;
    // the kernels compiled for the table are used once they are loaded: a launch never waits for the compile
    const bool spec_ready = t.spec_state.load(std::memory_order_acquire) == 1;
    const bool uc_spec_ready = spec_ready && t.spec_uc_global != nullptr;
    // A table most of whose conditions have no flat form gains nothing from a lean kernel until its specialised kernel
    // (leaf programs as straight-line code) is loaded: the lean body would defer nearly every request to the one-CTA-per-SM
    // drain launch.  Such launches go to the general kernel at full occupancy instead.
    const bool mostly_programs = t.uc.ok && !uc_spec_ready && 2 * (uint64_t)t.uc.n_gids_flat < t.uc.n_gids;
    p.lean = !ctx.force_general && !mostly_programs && cbhost::lean_eligible(lay, t.meta, bv);
    // Unique-condition kernels: lean-eligible tables with <= 63 distinct conditions whose blocks differ in shape
    // (with one shape the per-shape specialised tile kernel is the better fit).  Index order, no clustering.
    // (an image with condition programs or index-form rows is only good for the specialised kernel: cbuc::Image::needs_spec)
    const uint64_t n_pk = (uint64_t)bv.n_asets * t.uc.lay.uc_n_rows;   // merged rows: one per (action set, slot or image row)
    p.uc = p.lean && cbhost::uc_eligible(lay, t.uc, bv) && (uc_spec_ready || !t.uc.needs_spec()) && t.d_uc_image &&
           (ctx.uc_mode == 1 || (ctx.uc_mode != 0 && ctx.cluster_mode != 1 && t.meta[CB_META_BLOCK_SHAPES] > 1));   // CERBOS_B200_CLUSTER=1 keeps the clustered path reachable
    // Clustering pays when the policy blocks differ in shape (rows / conditions): with a single shape every lane runs
    // the same control flow in index order already and the coalesced column loads are worth more.
    p.cluster = !p.uc && bv.count < (1ull << 32) &&
                (ctx.cluster_mode == 1 || (ctx.cluster_mode != 0 && bv.count >= kClusterMinRequests && t.meta[CB_META_BLOCK_SHAPES] > 1));
    // Index-order lean launches stage the request columns through TMA too, when every tile's column runs are
    // 16-byte aligned and image + two tile stages fit the shared-memory budget of CB_MIN_BLOCKS resident CTAs.
    const uint32_t tile_bytes = cb::tile_cols_bytes(bv.role_cols, lay.n_slots);
    // [image][tile stage 0][tile stage 1][row_am copy][aset_k copy]
    const uint64_t small_tabs = (uint64_t)bv.n_asets * lay.n_rows * 8 + (((uint64_t)bv.n_asets + 1) & ~1ull) * 4 + 16 + 2 * kThreads;   // + tile_s[2] + res_s[2][256]
    const uint32_t tiles_smem = ((lay.image_bytes + 127u) & ~127u) + 2 * tile_bytes + (uint32_t)(small_tabs < 65536 ? small_tabs : 65536);
    auto al16 = [](const void *ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
    p.col_tiles = !p.uc && p.lean && p.stage && !p.cluster && !ctx.force_no_tiles && tiles_smem <= kMaxTilesSmem && bv.stride % 4 == 0 &&
                  bv.first % 4 == 0 && al16(bv.hdr0) && al16(bv.hdr1) && al16(bv.roles) && al16(bv.slots);
    // unique-condition launch: staged (compact image + merged rows in shared memory) when that fits
    p.uc_staged = p.uc && !ctx.force_no_stage && uc_stageable(t.uc, n_pk) && (!uc_spec_ready || t.spec_uc != nullptr);
    // lean launches with a staged table use the kernels specialised for this table when they exist (NVRTC, first use)
    p.spec = p.uc ? uc_spec_ready : p.lean && p.stage && bv.count < (1ull << 32) && spec_ready && t.spec_tiles != nullptr;
    p.kernel = p.uc        ? (p.spec ? (p.uc_staged ? Kernel::SpecUc : Kernel::SpecUcGlobal) : p.uc_staged ? Kernel::Uc : Kernel::UcGlobal)
             : p.spec      ? (p.col_tiles ? Kernel::SpecTiles : Kernel::SpecDirect)
             : p.col_tiles ? Kernel::LeanTiles
             : p.lean      ? (p.stage ? Kernel::Lean : Kernel::LeanGlobal)
                           : (p.stage ? Kernel::General : Kernel::GeneralGlobal);
    p.smem = p.uc ? (p.uc_staged ? (uint32_t)uc_smem_bytes(t.uc, n_pk) : 0) : p.col_tiles ? tiles_smem : p.stage ? lay.image_bytes : 0;
    p.last_arg = p.col_tiles ? lay.n_slots : p.stage ? 1u : 0u;
    p.serialise = p.spec && !p.uc && !ctx.profiling;
    p.strpred = p.uc && p.spec && t.spec_n_strpred;
    // on a global image the rows are merged with the batch's action-set masks once, up front
    p.merge_rows = p.uc && !p.uc_staged && n_pk <= (1u << 19);
    return p;
}

const void *kernel_fn(const cgpu_table &t, Kernel k) {
    switch (k) {
    case Kernel::General:
    case Kernel::GeneralGlobal: return (const void *)check_kernel<false, 2>;
    case Kernel::Lean: return (const void *)check_kernel<true, 1>;
    case Kernel::LeanGlobal: return (const void *)check_kernel<true, 0>;
    case Kernel::LeanTiles: return (const void *)check_kernel_tiles;
    case Kernel::Uc: return (const void *)check_uc<true>;
    case Kernel::UcGlobal: return (const void *)check_uc<false>;
    case Kernel::SpecTiles: return (const void *)t.spec_tiles;
    case Kernel::SpecDirect: return (const void *)t.spec_direct;
    case Kernel::SpecUc: return (const void *)t.spec_uc;
    case Kernel::SpecUcGlobal: return (const void *)t.spec_uc_global;
    case Kernel::UcMeta: return (const void *)check_uc_meta<true>;
    case Kernel::UcMetaGlobal: return (const void *)check_uc_meta<false>;
    case Kernel::SpecUcMeta: return (const void *)t.spec_uc_meta;
    case Kernel::SpecUcMetaGlobal: return (const void *)t.spec_uc_meta_global;
    }
    return nullptr;
}
// the metadata form of a unique-condition kernel
Kernel meta_kernel(Kernel k) {
    return k == Kernel::Uc ? Kernel::UcMeta : k == Kernel::UcGlobal ? Kernel::UcMetaGlobal : k == Kernel::SpecUc ? Kernel::SpecUcMeta : Kernel::SpecUcMetaGlobal;
}

// The device outputs of a metadata launch (cgpu_check_meta) beyond the effect bytes.
struct MetaDev {
    uint32_t *action_meta;
    cb_request_meta *req_meta;
};

// Resident CTAs per SM of kernel k with `smem` bytes of dynamic shared memory, queried once per (table, kernel, footprint);
// also lifts the kernel's dynamic shared-memory limit to kMaxStageBytes.  A CGPU_ERR_* code (< 0) when the query fails.
int resident_ctas(const cgpu_table &t, Kernel k, uint32_t smem) {
    std::atomic<uint64_t> &entry = t.occ[(int)k];
    const uint64_t e = entry.load(std::memory_order_relaxed);
    if ((uint32_t)e != 0 && (uint32_t)(e >> 32) == smem) return (int)(uint32_t)e;
    const void *fn = kernel_fn(t, k);
    int occ = 0;
    if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxStageBytes) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, kThreads, smem) != cudaSuccess) {
        if (k < Kernel::SpecTiles || k == Kernel::UcMeta || k == Kernel::UcMetaGlobal) return fail(CGPU_ERR_CUDA, "kernel attribute / occupancy query failed: %s", cudaGetErrorString(cudaGetLastError()));
        cudaGetLastError();
        occ = CB_MIN_BLOCKS;   // run-time loaded kernel on a runtime that cannot query it: the launch-bounds minimum
    }
    if (occ < 1) occ = 1;
    entry.store((uint64_t)smem << 32 | (uint32_t)occ, std::memory_order_relaxed);
    return occ;
}

// Launches fn programmatically serialised behind the kernel before it on `stream`: its CTAs may start while that kernel's
// last ones still run, and wait for it (griddepcontrol.wait) before they read what it wrote.
cudaError_t launch_serialised(const void *fn, uint32_t grid, uint32_t block, uint32_t smem, cudaStream_t stream, void **args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(block); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute pdl[1];
    pdl[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    pdl[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = pdl; cfg.numAttrs = 1;
    return cudaLaunchKernelExC(&cfg, fn, args);
}

// A reference-order kernel (a thread per request, grid-stride) over `count` requests: -> its grid, or a CGPU_ERR_* code (< 0)
template <class... Params, class... Args>
int launch_reference(cgpu_ctx *ctx, void (*kernel)(Params...), uint64_t count, cudaStream_t stream, Args... args) {
    const uint64_t tiles = (count + kThreads - 1) / kThreads, gmax = (uint64_t)ctx->sm_count * 4;
    const uint32_t grid = (uint32_t)(tiles < gmax ? tiles : gmax);
    kernel<<<grid, kThreads, 0, stream>>>(args...);
    CUDA_TRY(cudaGetLastError());
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    return (int)grid;
}

// Issues the launches of `plan` (plan_launch for this table and batch) on `stream`.  md: the metadata form of the plan's
// unique-condition kernel (cbuc::build_meta's table must exist), its deferrals drained by check_meta_kernel.
int launch_check(cgpu_ctx *ctx, const cgpu_table *t, const LaunchPlan &plan_in, const cb::BatchView &bv, uint8_t *d_bitmap, uint8_t *d_effects,
                 uint32_t *d_status, cudaStream_t stream, const MetaDev *md = nullptr) {
    LaunchPlan plan = plan_in;
    if (md) plan.kernel = meta_kernel(plan.kernel);
    const cb::TableLayout &lay = t->desc.lay;
    const uint64_t tiles = (bv.count + kThreads - 1) / kThreads;
    const int occ = resident_ctas(*t, plan.kernel, plan.smem);
    if (occ < 0) return occ;
    const uint64_t max_ctas = (uint64_t)ctx->sm_count * (uint64_t)occ;
    uint32_t grid = (uint32_t)(tiles < max_ctas ? tiles : max_ctas);
    if (grid == 0) grid = 1;
    TableDesc td = plan.uc ? t->uc_desc : t->desc;
    cb::BatchView bvv = bv;
    bvv.perm = nullptr;
    // few slot columns: every tile prefetches all of them one tile ahead (all loads of the tile then hit L1);
    // otherwise each policy block prefetches the slots its own conditions read
    bvv.prefetch_slots = lay.n_slots <= 8 ? lay.n_slots : 0;
    uint32_t *perm = nullptr;
    if (plan.cluster) {
        int rc = launch_cluster(ctx, t, bv, &perm, stream);
        if (rc != CGPU_OK) return rc;
        bvv.perm = perm;
    }
    uint32_t last_arg = plan.last_arg;
    uint32_t *defer = nullptr;
    if (plan.lean) {   // requests a lean kernel leaves to the general kernel go to a list drained right behind it
        uint32_t *cell = nullptr, *strpred = nullptr;
        cb::U4 *pk = nullptr;
        const uint32_t n_str = lay.nT + bv.n_bstr;
        const uint64_t n_pk = (uint64_t)bv.n_asets * t->uc.lay.uc_n_rows;
        int rc = acquire_defer(ctx, stream, bv.count, &defer, &cell, plan.strpred ? (size_t)n_str + 1 : 0, &strpred, plan.merge_rows ? (size_t)n_pk : 0, &pk);
        if (rc != CGPU_OK) return rc;
        if (plan.merge_rows) {
            uc_merge_rows<<<(unsigned)((n_pk + kThreads - 1) / kThreads), kThreads, 0, stream>>>(t->uc_desc, bvv, pk, (uint32_t)n_pk);
            CUDA_TRY(cudaGetLastError());
            ctx->launches.fetch_add(1, std::memory_order_relaxed);
            bvv.uc_rows_pk = pk;
        }
        bvv.defer_count = cell;
        bvv.tile_counter = plan.col_tiles ? cell + 2 : nullptr;
        bvv.defer_list = defer;
        if (plan.strpred && n_str) {
            // string predicates against constants: evaluated once per distinct string of the dictionary, not once per request
            TableDesc ptd = t->uc_desc;
            uint32_t n_arg = n_str;
            void *pargs[] = {&ptd, &bvv, &strpred, &n_arg};
            CUDA_TRY(cudaLaunchKernel((const void *)t->spec_strpred, dim3((n_str + 255) / 256), dim3(256), pargs, 0, stream));
            ctx->launches.fetch_add(1, std::memory_order_relaxed);
        }
        bvv.strpred = strpred;
    }
    const void *fn = kernel_fn(*t, plan.kernel);
    void *args[] = {&td, &bvv, &d_bitmap, &d_effects, &d_status, &last_arg};
    uint32_t *d_am = md ? md->action_meta : nullptr;
    cb_request_meta *d_rm = md ? md->req_meta : nullptr;
    const cb::U4 *d_side = t->d_uc_meta;
    void *margs[] = {&td, &bvv, &d_effects, &d_am, &d_rm, &d_side};
    if (ctx->profiling) {
        if (ctx->prof_pending && cudaEventSynchronize(ctx->ev1) == cudaSuccess) {
            float ms = 0;
            if (cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1) == cudaSuccess) { ctx->prof_ms += ms; ctx->prof_n++; }
            ctx->prof_pending = false;
        }
        CUDA_TRY(cudaEventRecord(ctx->ev0, stream));
    }
    if (plan.serialise) {
        // behind the previous launch's drain kernel (which releases its dependents at once): this kernel's CTAs start as the
        // previous specialised kernel's last tiles retire -- back-to-back launches on one stream overlap at their tails.
        // It reads nothing the previous launch writes.
        CUDA_TRY(launch_serialised(fn, grid, kThreads, plan.smem, stream, args));
    } else {
        CUDA_TRY(cudaLaunchKernel(fn, dim3(grid), dim3(kThreads), md ? margs : args, plan.smem, stream));
    }
    CUDA_TRY(cudaGetLastError());
    if (ctx->profiling) { CUDA_TRY(cudaEventRecord(ctx->ev1, stream)); ctx->prof_pending = true; }
    if (md) {
        // drain the deferral list with the reference-order metadata body, in stream order (it has no programmatic wait)
        cb::BatchView dv = bv;
        dv.perm = defer;
        dv.count_dev = bvv.defer_count;
        const int rc = launch_reference(ctx, check_meta_kernel, bv.count, stream, t->desc, dv, d_effects, d_am, d_rm, d_status);
        if (rc < 0) return rc;
    } else if (plan.lean) {
        // drain the deferral list with the general body (usually empty: the kernel then exits at once); it also does the
        // fused-gather signalling (BatchView::sig_*)
        cb::BatchView dv = bv;
        dv.perm = defer;
        dv.count_dev = bvv.defer_count;
        dv.prefetch_slots = 0;
        const Kernel gk = plan.stage ? Kernel::General : Kernel::GeneralGlobal;
        const uint32_t gsmem = plan.stage ? lay.image_bytes : 0;
        const int gocc = resident_ctas(*t, gk, gsmem);   // (for the shared-memory limit it sets: the grid does not depend on it)
        if (gocc < 0) return gocc;
        // one CTA per SM: the list is normally empty (every CTA then exits at once), and grid-stride loops otherwise
        const uint64_t gmax = (uint64_t)ctx->sm_count;
        const uint32_t ggrid = (uint32_t)(tiles < gmax ? tiles : gmax);
        uint32_t stage_arg = plan.stage ? 1u : 0u;
        TableDesc gtd = t->desc;
        void *gargs[] = {&gtd, &dv, &d_bitmap, &d_effects, &d_status, &stage_arg};
        CUDA_TRY(launch_serialised(kernel_fn(*t, gk), ggrid ? ggrid : 1, kThreads, gsmem, stream, gargs));
        CUDA_TRY(cudaGetLastError());
        ctx->launches.fetch_add(1, std::memory_order_relaxed);
    }
    if (perm) CUDA_TRY(cudaFreeAsync(perm, stream));
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    ctx->last_plan = plan;
    ctx->last_grid = grid;
    return CGPU_OK;
}

}  // namespace

extern "C" {

const char *cgpu_last_error(void) { return g_err.c_str(); }

int cgpu_init(const int *device_ids, int n_devices, cgpu_ctx **out) {
    if (!out) return fail(CGPU_ERR_INVALID, "cgpu_init: out is null");
    *out = nullptr;
    if (n_devices < 1 || !device_ids) return fail(CGPU_ERR_INVALID, "cgpu_init: at least one device; got %d", n_devices);
    if (n_devices > 1) {
        // one context per device; the first one is the handle, the others hang off it (SURVEY.md 8(b): a Go PDP is one process)
        for (int i = 0; i < n_devices; i++)
            for (int j = 0; j < i; j++)
                if (device_ids[i] == device_ids[j]) return fail(CGPU_ERR_INVALID, "cgpu_init: device %d listed twice", device_ids[i]);
        cgpu_ctx *head = nullptr;
        int rc = cgpu_init(device_ids, 1, &head);
        if (rc != CGPU_OK) return rc;
        for (int i = 1; i < n_devices; i++) {
            cgpu_ctx *c = nullptr;
            rc = cgpu_init(device_ids + i, 1, &c);
            if (rc != CGPU_OK) { const std::string why = g_err; cgpu_shutdown(head); return fail(rc, "%s", why.c_str()); }
            head->peers.push_back(c);
        }
        *out = head;
        return CGPU_OK;
    }
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) return fail(CGPU_ERR_NO_DEVICE, "no CUDA device available (%s); cerbos_b200 has no CPU fallback", e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    if (device_ids[0] < 0 || device_ids[0] >= count) return fail(CGPU_ERR_INVALID, "cgpu_init: device %d out of range (0..%d)", device_ids[0], count - 1);
    cgpu_ctx *ctx = new (std::nothrow) cgpu_ctx();
    if (!ctx) return fail(CGPU_ERR_INVALID, "out of memory");
    ctx->device = device_ids[0];
    {
        cudaDeviceProp prop;
        cudaError_t ie = cudaSetDevice(ctx->device);
        if (ie == cudaSuccess) ie = cudaGetDeviceProperties(&prop, ctx->device);
        if (ie == cudaSuccess) { ctx->sm_count = prop.multiProcessorCount; ie = cudaMalloc(&ctx->d_status, sizeof(uint32_t)); }
        if (ie == cudaSuccess) ie = cudaMemset(ctx->d_status, 0, sizeof(uint32_t));
        if (ie != cudaSuccess) {   // nothing leaks on a failed init
            if (ctx->d_status) cudaFree(ctx->d_status);
            delete ctx;
            return fail(CGPU_ERR_CUDA, "cgpu_init: %s", cudaGetErrorString(ie));
        }
    }
    const char *ns = getenv("CERBOS_B200_NO_STAGE");
    ctx->force_no_stage = ns && ns[0] == '1';
    const char *fg = getenv("CERBOS_B200_FORCE_GENERAL");
    ctx->force_general = fg && fg[0] == '1';
    const char *nj = getenv("CERBOS_B200_NO_JIT");
    ctx->force_no_jit = nj && nj[0] == '1';
    const char *nt = getenv("CERBOS_B200_NO_TILES");
    ctx->force_no_tiles = nt && nt[0] == '1';
    const char *um = getenv("CERBOS_B200_UC");
    ctx->uc_mode = um && (um[0] == '0' || um[0] == '1') ? um[0] - '0' : -1;
    const char *cm = getenv("CERBOS_B200_CLUSTER");
    ctx->cluster_mode = cm && (cm[0] == '0' || cm[0] == '1') ? cm[0] - '0' : -1;
    // stream-ordered scratch (clustering): keep freed blocks in the pool instead of returning them to the driver
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, ctx->device) == cudaSuccess) {
        uint64_t keep = ~0ull;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    ctx->slots.resize(4);
    *out = ctx;
    return CGPU_OK;
}

void cgpu_shutdown(cgpu_ctx *ctx) {
    if (!ctx) return;
    for (cgpu_ctx *p : ctx->peers) cgpu_shutdown(p);
    ctx->peers.clear();
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    for (auto &s : ctx->slots) {
        if (s.stream) cudaStreamDestroy(s.stream);
        if (s.h2d) cudaStreamDestroy(s.h2d);
        if (s.d2h) cudaStreamDestroy(s.d2h);
        for (auto e : s.ev) cudaEventDestroy(e);
        if (s.dev) cudaFree(s.dev);
        if (s.h_status) cudaFreeHost(s.h_status);
        if (s.d_status) cudaFree(s.d_status);
    }
    if (ctx->d_status) cudaFree(ctx->d_status);
    for (auto &kv : ctx->defer_lanes) {
        for (auto &b : kv.second.q) { cudaFree(b.list.ptr); cudaFree(b.strpred.ptr); cudaFree(b.pk.ptr); }
        if (kv.second.cells) cudaFree(kv.second.cells);
    }
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    for (auto e : ctx->copy_ev) if (e) cudaEventDestroy(e);
    for (auto &u : ctx->slice_uses) { if (u.done) cudaEventDestroy(u.done); if (u.stage) cudaFree(u.stage); }
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    delete ctx;
}

int cgpu_table_load(cgpu_ctx *ctx, const void *blob, size_t len, cgpu_table **out) {
    if (!ctx || !out) return fail(CGPU_ERR_INVALID, "cgpu_table_load: null argument");
    *out = nullptr;
    cgpu_table *t = new (std::nothrow) cgpu_table();
    if (!t) return fail(CGPU_ERR_INVALID, "out of memory");
    t->ctx = ctx;
    int rc = invalid(cbhost::parse_blob(blob, len, &t->desc.lay, t->meta, t->sec_len));
    if (rc != CGPU_OK) { delete t; return rc; }
    t->uc = cbuc::build(static_cast<const uint8_t *>(blob), t->desc.lay.off, t->sec_len, t->meta, t->desc.lay);
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void **>(&t->d_image), t->desc.lay.image_bytes);
    if (e == cudaSuccess) e = cudaMemcpy(t->d_image, blob, t->desc.lay.image_bytes, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && t->uc.ok) {
        e = cudaMalloc(reinterpret_cast<void **>(&t->d_uc_image), t->uc.bytes.size());
        if (e == cudaSuccess) e = cudaMemcpy(t->d_uc_image, t->uc.bytes.data(), t->uc.bytes.size(), cudaMemcpyHostToDevice);
        t->uc_meta = cbuc::build_meta(static_cast<const uint8_t *>(blob), t->desc.lay.off, t->sec_len, t->meta, t->desc.lay, t->uc);
        if (e == cudaSuccess && t->uc_meta.ok) {
            e = cudaMalloc(reinterpret_cast<void **>(&t->d_uc_meta), t->uc_meta.words.size() * 4);
            if (e == cudaSuccess) e = cudaMemcpy(t->d_uc_meta, t->uc_meta.words.data(), t->uc_meta.words.size() * 4, cudaMemcpyHostToDevice);
        }
    }
    if (e != cudaSuccess) {
        if (t->d_image) cudaFree(t->d_image);
        if (t->d_uc_image) cudaFree(t->d_uc_image);
        if (t->d_uc_meta) cudaFree(t->d_uc_meta);
        delete t;
        return fail(CGPU_ERR_CUDA, "table upload failed: %s", cudaGetErrorString(e));
    }
    t->desc.base = t->d_image;
    t->uc_desc.base = t->d_uc_image;
    t->uc_desc.lay = t->uc.lay;
    t->host_image.assign(static_cast<const uint8_t *>(blob), static_cast<const uint8_t *>(blob) + t->desc.lay.image_bytes);
    // table-specialised kernels are generated + compiled off the caller's thread; launches use the generic kernels
    // until they are ready (cgpu_table_wait_ready blocks for them)
    t->spec_thread = std::thread([ctx, t] {
        cudaSetDevice(ctx->device);
        ensure_spec(ctx, t);
    });
    // a multi-device context holds the table on every device ("broadcast" of the blob: one process, so a copy per device)
    for (cgpu_ctx *p : ctx->peers) {
        cgpu_table *pt = nullptr;
        rc = cgpu_table_load(p, blob, len, &pt);
        if (rc != CGPU_OK) { const std::string why = g_err; cgpu_table_release(t); return fail(rc, "%s", why.c_str()); }
        t->peer_tables.push_back(pt);
    }
    *out = t;
    return CGPU_OK;
}

void cgpu_table_retain(cgpu_table *t) { if (t) t->refs.fetch_add(1); }
int cgpu_device_count(const cgpu_ctx *ctx) { return ctx ? 1 + (int)ctx->peers.size() : 0; }

void cgpu_table_release(cgpu_table *t) {
    if (!t) return;
    if (t->refs.fetch_sub(1) == 1) {
        for (cgpu_table *pt : t->peer_tables) cgpu_table_release(pt);
        t->peer_tables.clear();
        { std::lock_guard<std::mutex> g(t->join_mu); if (t->spec_thread.joinable()) t->spec_thread.join(); }
        cudaSetDevice(t->ctx->device);
        cudaDeviceSynchronize();   // no kernel may still read the image
        cudaFree(t->d_image);
        if (t->d_uc_image) cudaFree(t->d_uc_image);
        if (t->d_uc_meta) cudaFree(t->d_uc_meta);
        if (t->spec_lib) cudaLibraryUnload(t->spec_lib);
        delete t;
    }
}

int cgpu_table_compile_check(const void *blob, size_t len, size_t *cubin_bytes) {
    if (!blob || !cubin_bytes) return fail(CGPU_ERR_INVALID, "cgpu_table_compile_check: null argument");
    *cubin_bytes = 0;
    cb::TableLayout lay;
    uint32_t meta[CB_META_WORDS];
    uint64_t sec_len[cbhost::kMaxSec] = {0};
    int rc = invalid(cbhost::parse_blob(blob, len, &lay, meta, sec_len));
    if (rc != CGPU_OK) return rc;
    const cbuc::Image uc = cbuc::build(static_cast<const uint8_t *>(blob), lay.off, sec_len, meta, lay);
    std::vector<char> cubin;
    std::string why;
    uint32_t n_strpred = 0;
    const SpecForm form = spec_compile(static_cast<const uint8_t *>(blob), lay, meta, uc, &cubin, &why, &n_strpred);
    if (form == SPEC_NONE) {
        g_err = why;
        return why.rfind("NVRTC compile failed", 0) == 0 ? CGPU_ERR_CUDA : CGPU_OK;   // not qualifying is not an error
    }
    g_err = form == SPEC_UC ? "unique-condition form" : "block-shape form";
    *cubin_bytes = cubin.size();
    return CGPU_OK;
}

int cgpu_table_wait_ready(cgpu_table *t, int *specialised) {
    if (!t) return fail(CGPU_ERR_INVALID, "cgpu_table_wait_ready: null table");
    for (cgpu_table *pt : t->peer_tables) cgpu_table_wait_ready(pt, nullptr);
    { std::lock_guard<std::mutex> g(t->join_mu); if (t->spec_thread.joinable()) t->spec_thread.join(); }
    if (specialised) *specialised = t->spec_state.load(std::memory_order_acquire) == 1 ? 1 : 0;
    g_err = t->spec_note;   // why not, if not (readable through cgpu_last_error)
    return CGPU_OK;
}

int cgpu_table_info(const cgpu_table *t, uint32_t *meta_out, uint32_t n_words) {
    if (!t || !meta_out) return fail(CGPU_ERR_INVALID, "cgpu_table_info: null argument");
    if (n_words > CB_META_WORDS) n_words = CB_META_WORDS;
    memcpy(meta_out, t->meta, n_words * 4);
    return CGPU_OK;
}

uint64_t cgpu_launch_count(const cgpu_ctx *ctx) { return ctx ? ctx->launches.load() : 0; }

int cgpu_deferred_count(cgpu_ctx *ctx, uint64_t *total) {
    if (!ctx || !total) return fail(CGPU_ERR_INVALID, "cgpu_deferred_count: null argument");
    *total = 0;
    struct RestoreDevice {   // the caller's current device, whichever way this returns
        int dev = -1;
        RestoreDevice() { if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); dev = -1; } }
        ~RestoreDevice() { if (dev >= 0) cudaSetDevice(dev); }
    } restore;
    std::vector<cgpu_ctx *> all{ctx};
    all.insert(all.end(), ctx->peers.begin(), ctx->peers.end());
    for (cgpu_ctx *c : all) {
        CUDA_TRY(cudaSetDevice(c->device));
        CUDA_TRY(cudaDeviceSynchronize());
        std::lock_guard<std::mutex> g(c->defer_mu);
        for (auto &kv : c->defer_lanes) {
            if (!kv.second.cells) continue;
            uint32_t w[16];
            CUDA_TRY(cudaMemcpy(w, kv.second.cells, sizeof(w), cudaMemcpyDeviceToHost));
            for (int q = 0; q < 4; q++) *total += w[4 * q + 3];
        }
    }
    return CGPU_OK;
}

int cgpu_last_kernel_config(const cgpu_ctx *ctx, uint32_t *grid, uint32_t *block, uint32_t *smem_bytes) {
    if (!ctx) return fail(CGPU_ERR_INVALID, "null ctx");
    if (grid) *grid = ctx->last_grid;
    if (block) *block = ctx->last_grid ? kThreads : 0;   // 0 before the first launch
    if (smem_bytes) *smem_bytes = ctx->last_plan.smem | (uint32_t)ctx->last_plan.lean << 31;   // bit 31: lean kernel body was used
    return CGPU_OK;
}

int cgpu_last_cluster_config(const cgpu_ctx *ctx, uint32_t *clustered, uint32_t *window, uint32_t *buckets) {
    if (!ctx) return fail(CGPU_ERR_INVALID, "null ctx");
    const LaunchPlan &p = ctx->last_plan;
    if (clustered) *clustered = (uint32_t)p.cluster | (uint32_t)p.col_tiles << 1 | (uint32_t)p.spec << 2 | (uint32_t)p.uc << 3;   // include/cerbos_b200.h
    if (window) *window = ctx->last_window;
    if (buckets) *buckets = ctx->last_buckets;
    return CGPU_OK;
}

int cgpu_profile(cgpu_ctx *ctx, int enable, double *kernel_ms_sum, uint64_t *n_launches) {
    if (!ctx) return fail(CGPU_ERR_INVALID, "null ctx");
    CUDA_TRY(cudaSetDevice(ctx->device));
    if (ctx->prof_pending) {
        CUDA_TRY(cudaEventSynchronize(ctx->ev1));
        float ms = 0;
        CUDA_TRY(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
        ctx->prof_ms += ms; ctx->prof_n++;
        ctx->prof_pending = false;
    }
    if (kernel_ms_sum) *kernel_ms_sum = ctx->prof_ms;
    if (n_launches) *n_launches = ctx->prof_n;
    ctx->prof_ms = 0; ctx->prof_n = 0;
    if (enable && !ctx->ev0) { CUDA_TRY(cudaEventCreate(&ctx->ev0)); CUDA_TRY(cudaEventCreate(&ctx->ev1)); }
    ctx->profiling = enable != 0;
    return CGPU_OK;
}

int cgpu_check_device(cgpu_ctx *ctx, const cgpu_table *t, const cgpu_batch *dev_batch, void *dev_bitmap_out, void *cuda_stream) {
    if (!ctx || !t || !dev_batch || !dev_bitmap_out) return fail(CGPU_ERR_INVALID, "cgpu_check_device: null argument");
    if (t->ctx != ctx) return fail(CGPU_ERR_INVALID, "table belongs to another context");
    cb::BatchView bv;
    int rc = invalid(cbhost::make_batch_view(t->desc.lay, dev_batch, 0, dev_batch->n_requests, &bv));
    if (rc != CGPU_OK) return rc;
    CUDA_TRY(cudaSetDevice(ctx->device));
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);   // NULL = the legacy default stream
    return launch_check(ctx, t, plan_launch(*ctx, *t, bv), bv, static_cast<uint8_t *>(dev_bitmap_out), nullptr, ctx->d_status, s);
}

int cgpu_peer_alloc(cgpu_ctx *ctx, size_t bytes, void **dev_ptr, void *ipc_handle_out) {
    if (!ctx || !dev_ptr || !ipc_handle_out || bytes == 0) return fail(CGPU_ERR_INVALID, "cgpu_peer_alloc: bad argument");
    CUDA_TRY(cudaSetDevice(ctx->device));
    void *p = nullptr;
    CUDA_TRY(cudaMalloc(&p, bytes));
    CUDA_TRY(cudaMemset(p, 0, bytes));
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) { cudaFree(p); return fail(CGPU_ERR_CUDA, "cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e)); }
    static_assert(sizeof(h) == CGPU_IPC_HANDLE_BYTES, "IPC handle size");
    memcpy(ipc_handle_out, &h, sizeof(h));
    *dev_ptr = p;
    return CGPU_OK;
}

int cgpu_peer_open(cgpu_ctx *ctx, const void *ipc_handle, void **dev_ptr) {
    if (!ctx || !ipc_handle || !dev_ptr) return fail(CGPU_ERR_INVALID, "cgpu_peer_open: null argument");
    CUDA_TRY(cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, ipc_handle, sizeof(h));
    CUDA_TRY(cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return CGPU_OK;
}

int cgpu_peer_close(cgpu_ctx *ctx, void *dev_ptr) {
    if (!ctx || !dev_ptr) return fail(CGPU_ERR_INVALID, "cgpu_peer_close: null argument");
    CUDA_TRY(cudaSetDevice(ctx->device));
    CUDA_TRY(cudaIpcCloseMemHandle(dev_ptr));
    return CGPU_OK;
}

int cgpu_peer_free(cgpu_ctx *ctx, void *dev_ptr) {
    if (!ctx || !dev_ptr) return fail(CGPU_ERR_INVALID, "cgpu_peer_free: null argument");
    CUDA_TRY(cudaSetDevice(ctx->device));
    CUDA_TRY(cudaFree(dev_ptr));
    return CGPU_OK;
}

int cgpu_peer_read(cgpu_ctx *ctx, const void *dev_ptr, void *host_out, size_t bytes) {
    if (!ctx || !dev_ptr || !host_out) return fail(CGPU_ERR_INVALID, "cgpu_peer_read: null argument");
    CUDA_TRY(cudaSetDevice(ctx->device));
    CUDA_TRY(cudaMemcpy(host_out, dev_ptr, bytes, cudaMemcpyDeviceToHost));
    return CGPU_OK;
}

int cgpu_check_device_gather(cgpu_ctx *ctx, const cgpu_table *t, const cgpu_batch *dev_batch, const cgpu_gather *g, void *cuda_stream) {
    if (!ctx || !t || !dev_batch || !g || !g->gather_bufs || !g->flags) return fail(CGPU_ERR_INVALID, "cgpu_check_device_gather: null argument");
    if (t->ctx != ctx) return fail(CGPU_ERR_INVALID, "table belongs to another context");
    if (g->n_ranks == 0 || g->n_ranks > cb::CB_MAX_GATHER || g->my_rank >= g->n_ranks || g->step == 0)
        return fail(CGPU_ERR_INVALID, "cgpu_check_device_gather: 1..%d ranks, my_rank < n_ranks, step > 0", cb::CB_MAX_GATHER);
    cb::BatchView bv;
    int rc = invalid(cbhost::make_batch_view(t->desc.lay, dev_batch, 0, dev_batch->n_requests, &bv));
    if (rc != CGPU_OK) return rc;
    if (bv.kbytes > 8) return fail(CGPU_ERR_UNSUPPORTED, "fused gather supports up to 64 actions per request");
    if ((uint64_t)bv.count * bv.kbytes > g->slice_bytes) return fail(CGPU_ERR_INVALID, "gather slice too small");
    SignalParams sp{};
    for (uint32_t r = 0; r < g->n_ranks; r++) {
        if (!g->gather_bufs[r] || !g->flags[r]) return fail(CGPU_ERR_INVALID, "gather buffer / flags of rank %u missing", r);
        bv.outs[r] = static_cast<uint8_t *>(g->gather_bufs[r]) + (uint64_t)g->my_rank * g->slice_bytes;
        sp.flags[r] = g->flags[r];
    }
    sp.n_ranks = g->n_ranks; sp.my_rank = g->my_rank; sp.step = g->step;
    sp.wait_flags = g->wait_flags ? g->wait_flags : g->flags[g->my_rank]; sp.wait_step = g->wait_step;
    CUDA_TRY(cudaSetDevice(ctx->device));
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    const uint64_t slice_used = (uint64_t)bv.count * bv.kbytes;
    const char *ce = getenv("CERBOS_B200_CE_GATHER");
    const bool ce_gather = g->n_ranks > 1 && (ce ? ce[0] == '1' : slice_used >= (1u << 20));
    if (ce_gather) {
        // Large slices: the kernels store this rank's results into its own slice only; the copy engines then push that
        // slice to every peer over NVLink on a side stream (no SM is involved and the next batch's kernel runs meanwhile),
        // and a one-warp kernel behind the copies releases the step into every rank's flag array.
        std::lock_guard<std::mutex> lk(ctx->copy_mu);
        if (!ctx->copy_stream) CUDA_TRY(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
        uint8_t *own = bv.outs[g->my_rank];
        // the previous push out of this very slice must have drained before the kernel overwrites it
        cgpu_ctx::SliceUse *use = nullptr;
        for (auto &u : ctx->slice_uses) if (u.ptr == own) use = &u;
        if (use) CUDA_TRY(cudaStreamWaitEvent(s, use->done, 0));
        else {
            cgpu_ctx::SliceUse nu{own, nullptr, nullptr, 0};
            CUDA_TRY(cudaEventCreateWithFlags(&nu.done, cudaEventDisableTiming));
            ctx->slice_uses.push_back(nu);
            use = &ctx->slice_uses.back();
        }
        // The kernels write into plain device memory; the copy engines move the slice from there into every rank's gather
        // buffer, this rank's own included, so that the check kernels never store across NVLink themselves.
        if (use->stage_bytes < slice_used) {
            if (use->stage) { CUDA_TRY(cudaStreamSynchronize(ctx->copy_stream)); CUDA_TRY(cudaFree(use->stage)); use->stage = nullptr; use->stage_bytes = 0; }
            CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(&use->stage), slice_used));
            use->stage_bytes = slice_used;
        }
        rc = launch_check(ctx, t, plan_launch(*ctx, *t, bv), bv, use->stage, nullptr, ctx->d_status, s);
        if (rc != CGPU_OK) return rc;
        cudaEvent_t &ev = ctx->copy_ev[ctx->copy_seq++ & 15];
        if (!ev) CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        CUDA_TRY(cudaEventRecord(ev, s));
        CUDA_TRY(cudaStreamWaitEvent(ctx->copy_stream, ev, 0));
        for (uint32_t q = 0; q < g->n_ranks; q++) {   // peers first (NVLink), starting with the next rank so that the pushes of all ranks spread over the links
            const uint32_t r = (g->my_rank + 1 + q) % g->n_ranks;
            CUDA_TRY(cudaMemcpyAsync(bv.outs[r], use->stage, slice_used, cudaMemcpyDeviceToDevice, ctx->copy_stream));
        }
        SignalParams sp2 = sp;
        sp2.wait_step = 0;
        void *args[] = {&sp2};
        CUDA_TRY(cudaLaunchKernel((const void *)gather_signal, dim3(1), dim3(32), args, 0, ctx->copy_stream));
        CUDA_TRY(cudaEventRecord(use->done, ctx->copy_stream));
        ctx->launches.fetch_add(1, std::memory_order_relaxed);
        if (g->wait_step) {   // hold the issuing stream until every rank's slice of the older step has landed here
            gather_wait<<<1, 32, 0, s>>>(sp.wait_flags, g->n_ranks, g->wait_step);
            CUDA_TRY(cudaGetLastError());
            ctx->launches.fetch_add(1, std::memory_order_relaxed);
        }
        return CGPU_OK;
    }
    bv.n_out = g->n_ranks;
    for (uint32_t r = 0; r < g->n_ranks; r++) bv.sig_flags[r] = g->flags[r];
    bv.sig_rank = g->my_rank; bv.sig_step = g->step;
    bv.wait_flags = sp.wait_flags; bv.wait_step = g->wait_step;
    const LaunchPlan plan = plan_launch(*ctx, *t, bv);
    rc = launch_check(ctx, t, plan, bv, bv.outs[g->my_rank], nullptr, ctx->d_status, s);
    if (rc != CGPU_OK) return rc;
    if (!plan.lean) {   // no drain kernel to do the signalling: a one-warp kernel behind the check publishes the step (and does the lagged wait)
        void *args[] = {&sp};
        CUDA_TRY(launch_serialised((const void *)gather_signal, 1, 32, 0, s, args));
        ctx->launches.fetch_add(1, std::memory_order_relaxed);
    }
    return CGPU_OK;
}

int cgpu_gather_wait(cgpu_ctx *ctx, const uint32_t *local_flags, uint32_t n_ranks, uint32_t step, void *cuda_stream) {
    if (!ctx || !local_flags || n_ranks == 0 || n_ranks > cb::CB_MAX_GATHER) return fail(CGPU_ERR_INVALID, "cgpu_gather_wait: bad argument");
    CUDA_TRY(cudaSetDevice(ctx->device));
    gather_wait<<<1, 32, 0, static_cast<cudaStream_t>(cuda_stream)>>>(local_flags, n_ranks, step);
    CUDA_TRY(cudaGetLastError());
    ctx->launches.fetch_add(1, std::memory_order_relaxed);
    return CGPU_OK;
}

int cgpu_sync(cgpu_ctx *ctx, void *cuda_stream) {
    if (!ctx) return fail(CGPU_ERR_INVALID, "null ctx");
    CUDA_TRY(cudaSetDevice(ctx->device));
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    uint32_t st = 0;
    CUDA_TRY(cudaMemcpyAsync(&st, ctx->d_status, 4, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    if (st) {
        CUDA_TRY(cudaMemsetAsync(ctx->d_status, 0, 4, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        return fail(CGPU_ERR_UNSUPPORTED, "a request produced a run-time value the device cannot represent exactly (e.g. timestamp outside 1678..2262, string->double, concatenation)");
    }
    return CGPU_OK;
}

// ---- native batch encoder (cb_encode.h) ----------------------------------------------------------------------------
// Page-locked staging blocks of cgpu_encode / cgpu_narrow_build are recycled: cudaHostAlloc costs milliseconds for the tens of
// megabytes a batch takes, every call.  A block goes back to a small free list (eight blocks) when its batch is freed; blocks
// are sized in steps so that batches of similar size reuse each other's.  (Without a CUDA device there is nothing to pin: the
// columns stay in their vectors, or -- CERBOS_B200_NARROW_BLOCK=1, tests -- in plain memory laid out the same way.)
struct HostBlock { void *p = nullptr; size_t cap = 0; bool is_malloc = false; };
struct HostBlockPool {
    std::mutex mu;
    std::vector<HostBlock> free_list;
    HostBlock take(size_t bytes, bool allow_malloc) {
        size_t cap = 1u << 20;                    // powers of two up to 64 MB, then multiples of 64 MB
        while (cap < bytes && cap < (64u << 20)) cap <<= 1;
        if (cap < bytes) cap = (bytes + (64u << 20) - 1) / (64u << 20) * (64u << 20);
        {
            std::lock_guard<std::mutex> g(mu);
            size_t best = free_list.size();
            for (size_t i = 0; i < free_list.size(); i++)
                if (free_list[i].cap >= bytes && (allow_malloc || !free_list[i].is_malloc) && (best == free_list.size() || free_list[i].cap < free_list[best].cap)) best = i;
            if (best != free_list.size()) { HostBlock b = free_list[best]; free_list.erase(free_list.begin() + (long)best); return b; }
        }
        HostBlock b;
        if (cudaHostAlloc(&b.p, cap, cudaHostAllocDefault) == cudaSuccess) { b.cap = cap; return b; }
        cudaGetLastError();
        b.p = nullptr;
        if (allow_malloc) { b.p = malloc(cap); b.cap = b.p ? cap : 0; b.is_malloc = b.p != nullptr; }
        return b;
    }
    void give(HostBlock b) {
        if (!b.p) return;
        {
            std::lock_guard<std::mutex> g(mu);
            if (free_list.size() < 8) { free_list.push_back(b); return; }
        }
        if (b.is_malloc) free(b.p); else cudaFreeHost(b.p);
    }
};
static HostBlockPool &host_pool() { static HostBlockPool *p = new HostBlockPool(); return *p; }   // (never destroyed: blocks may outlive static teardown order)

int cgpu_encoder_create(const void *blob, size_t len, const char *default_version, const char *default_scope, int lenient_scope_search, cgpu_encoder **out) {
    if (!blob || !out) return fail(CGPU_ERR_INVALID, "cgpu_encoder_create: null argument");
    *out = nullptr;
    cgpu_encoder *e = new (std::nothrow) cgpu_encoder();
    if (!e) return fail(CGPU_ERR_INVALID, "out of memory");
    cbenc::Conf conf;
    if (default_version && default_version[0]) conf.default_version = default_version;
    if (default_scope) conf.default_scope = default_scope;
    conf.lenient = lenient_scope_search != 0;
    if (!e->enc.init(blob, len, conf)) { const std::string why = e->enc.error; delete e; return fail(CGPU_ERR_INVALID, "%s", why.c_str()); }
    *out = e;
    return CGPU_OK;
}
void cgpu_encoder_destroy(cgpu_encoder *e) { delete e; }

int cgpu_encode(const cgpu_encoder *e, const void *const *inputs, const size_t *input_bytes, uint64_t n, cgpu_encoded **out) {
    if (!e || !inputs || !input_bytes || !out || n == 0) return fail(CGPU_ERR_INVALID, "cgpu_encode: null argument or empty batch");
    *out = nullptr;
    cgpu_encoded *r = new (std::nothrow) cgpu_encoded();
    if (!r) return fail(CGPU_ERR_INVALID, "out of memory");
    std::string enc_err;               // (the encoder itself is read-only here: concurrent cgpu_encode calls share it)
    // shards of the batch are encoded on host threads and merged in order (CERBOS_B200_ENCODE_THREADS, default: the cores, at most 32)
    unsigned threads = std::thread::hardware_concurrency();
    if (threads > 32) threads = 32;
    if (const char *et = getenv("CERBOS_B200_ENCODE_THREADS")) { const long v = strtol(et, nullptr, 10); if (v >= 1 && v <= 256) threads = (unsigned)v; }
    if (!e->enc.encode(inputs, input_bytes, n, &r->cols, threads ? threads : 1, &enc_err)) { delete r; return fail(CGPU_ERR_INVALID, "cgpu_encode: %s", enc_err.c_str()); }
    r->flags = e->enc.conf.lenient ? CB_BATCH_FLAG_LENIENT : 0;
    r->n_slots = (uint32_t)e->enc.slots.size();
    r->role_cols = r->cols.role_cols;
    size_t total = 0, offs[CGPU_N_COLUMNS];
    for (int i = 0; i < CGPU_N_COLUMNS; i++) { offs[i] = total; r->bytes[i] = r->cols.bytes(i); total += (r->bytes[i] + 255) & ~(size_t)255; }
    // page-locked staging so that cgpu_check's chunked H2D copies run asynchronously; without a CUDA device the columns
    // simply stay where they were built (host memory either way: this is data marshalling, not evaluation)
    const HostBlock hb = host_pool().take(total ? total : 256, false);
    r->pinned = hb.p; r->pinned_cap = hb.cap;
    if (r->pinned) {
        for (int i = 0; i < CGPU_N_COLUMNS; i++) {
            if (r->bytes[i]) memcpy(static_cast<uint8_t *>(r->pinned) + offs[i], r->cols.ptr(i), r->bytes[i]);
            r->ptrs[i] = static_cast<uint8_t *>(r->pinned) + offs[i];
        }
        const uint64_t nreq = r->cols.n;
        const uint32_t ma = r->cols.max_actions;
        r->cols = cbenc::Columns();
        r->cols.n = nreq; r->cols.max_actions = ma;
    } else {
        for (int i = 0; i < CGPU_N_COLUMNS; i++) r->ptrs[i] = r->cols.ptr(i);
    }
    *out = r;
    return CGPU_OK;
}

int cgpu_encoded_batch(const cgpu_encoded *r, int64_t now_unix_nanos, cgpu_batch *out) {
    if (!r || !out) return fail(CGPU_ERR_INVALID, "cgpu_encoded_batch: null argument");
    out->n_requests = r->cols.n;
    out->max_actions = r->cols.max_actions;
    out->now_unix_nanos = now_unix_nanos;
    out->flags = r->flags;
    out->columns = r->ptrs;
    out->column_bytes = r->bytes;
    out->n_columns = CGPU_N_COLUMNS;
    return CGPU_OK;
}

void cgpu_encoded_free(cgpu_encoded *r) {
    if (!r) return;
    if (r->pinned) { HostBlock hb; hb.p = r->pinned; hb.cap = r->pinned_cap; host_pool().give(hb); }
    delete r;
}

int cgpu_narrow_build(const cgpu_encoded *enc, int form, cgpu_narrowed **out) {
    if (!enc || !out || (form != 1 && form != 2)) return fail(CGPU_ERR_INVALID, "cgpu_narrow_build: null argument, or form not 1 / 2");
    *out = nullptr;
    cgpu_narrowed *r = new (std::nothrow) cgpu_narrowed();
    if (!r) return fail(CGPU_ERR_INVALID, "out of memory");
    const uint64_t n = enc->cols.n;
    r->nb = cbnarrow::build(static_cast<const uint32_t *>(enc->ptrs[CGPU_COL_HDR0]), static_cast<const uint8_t *>(enc->ptrs[CGPU_COL_HDR1]),
                            static_cast<const uint32_t *>(enc->ptrs[CGPU_COL_ROLES]), static_cast<const uint64_t *>(enc->ptrs[CGPU_COL_SLOTS]),
                            static_cast<const uint64_t *>(enc->ptrs[CGPU_COL_HEAP]), enc->bytes[CGPU_COL_HEAP] / 8, n, enc->role_cols, enc->n_slots, form == 2);
    if (!r->nb.ok) { delete r; return fail(CGPU_ERR_UNSUPPORTED, "cgpu_narrow_build: an id of this batch does not fit its narrow header field"); }
    r->enc = enc;
    cbnarrow::Narrowed &nb = r->nb;
    // page-locked staging, like cgpu_encode (without a CUDA device the columns stay where they were built)
    std::vector<std::pair<const void **, std::vector<uint8_t> *>> parts;
    std::vector<uint8_t> hdr_bytes(reinterpret_cast<const uint8_t *>(nb.hdr16.data()), reinterpret_cast<const uint8_t *>(nb.hdr16.data()) + nb.hdr16.size() * 2);
    r->slot_ptrs.assign(nb.slot_cols.size() ? nb.slot_cols.size() : 1, nullptr);
    size_t total = 0;
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    total += al(nb.pid.size()) + al(hdr_bytes.size()) + al(nb.versions.size()) + al(nb.roles.size()) + al(nb.heap.size());
    for (const auto &c : nb.slot_cols) total += al(c.size());
    uint8_t *base = nullptr;
    {
        const char *tb = getenv("CERBOS_B200_NARROW_BLOCK");
        const HostBlock hb = host_pool().take(total ? total : 256, tb && tb[0] == '1');
        base = static_cast<uint8_t *>(hb.p);
        r->pinned = hb.p; r->pinned_cap = hb.cap; r->pinned_is_malloc = hb.is_malloc;
    }
    size_t at = 0;
    auto place = [&](const uint8_t *src, size_t bytes) -> const void * {
        if (!bytes) return nullptr;
        if (!base) return src;
        memcpy(base + at, src, bytes);
        const void *p = base + at;
        at += al(bytes);
        return p;
    };
    r->pid = place(nb.pid.data(), nb.pid.size());
    r->hdr16 = place(hdr_bytes.data(), hdr_bytes.size());
    if (!base && !hdr_bytes.empty()) r->hdr16 = nb.hdr16.data();     // (hdr_bytes is a temporary)
    r->versions = place(nb.versions.data(), nb.versions.size());
    r->roles = place(nb.roles.data(), nb.roles.size());
    r->heap = place(nb.heap.data(), nb.heap.size());
    r->heap_bytes = nb.heap.size();
    for (size_t v = 0; v < nb.slot_cols.size(); v++) r->slot_ptrs[v] = place(nb.slot_cols[v].data(), nb.slot_cols[v].size());
    for (int i = 0; i < CGPU_N_COLUMNS; i++) { r->cols[i] = i < CGPU_COL_HEAP ? nullptr : enc->ptrs[i]; r->col_bytes[i] = i < CGPU_COL_HEAP ? 0 : enc->bytes[i]; }
    r->cols[CGPU_COL_HEAP] = r->heap; r->col_bytes[CGPU_COL_HEAP] = r->heap_bytes;
    *out = r;
    return CGPU_OK;
}

int cgpu_narrowed_view(const cgpu_narrowed *r, int64_t now_unix_nanos, cgpu_batch *batch_out, cgpu_narrow *narrow_out) {
    if (!r || !batch_out || !narrow_out) return fail(CGPU_ERR_INVALID, "cgpu_narrowed_view: null argument");
    const cbnarrow::Narrowed &nb = r->nb;
    batch_out->n_requests = nb.n;
    batch_out->max_actions = r->enc->cols.max_actions;
    batch_out->now_unix_nanos = now_unix_nanos;
    batch_out->flags = r->enc->flags;
    batch_out->columns = r->cols;
    batch_out->column_bytes = r->col_bytes;
    batch_out->n_columns = CGPU_N_COLUMNS;
    memset(narrow_out, 0, sizeof(*narrow_out));
    if (nb.pid16) { narrow_out->principal_id16 = static_cast<const uint16_t *>(r->pid); narrow_out->principal_base = nb.principal_base; }
    else narrow_out->principal_id = static_cast<const uint32_t *>(r->pid);
    narrow_out->hdr16 = static_cast<const uint16_t *>(r->hdr16);
    narrow_out->versions = static_cast<const uint8_t *>(r->versions);
    narrow_out->roles = static_cast<const uint8_t *>(r->roles);
    narrow_out->role_cols = nb.role_cols;
    narrow_out->slot_class = nb.slot_class.data();
    narrow_out->slot_cols = r->slot_ptrs.data();
    narrow_out->heap_u32 = nb.heap_u32 ? 1 : 0;
    narrow_out->slot_base = nb.slot_base.data();
    narrow_out->slot_base2 = nb.slot_base2.data();
    narrow_out->hdr_const_mask = nb.hdr_const_mask;
    for (int f = 0; f < 4; f++) narrow_out->hdr_const[f] = nb.hdr_const[f];
    narrow_out->versions_const = nb.versions_const ? 1 : 0;
    narrow_out->versions_value[0] = nb.versions_value[0]; narrow_out->versions_value[1] = nb.versions_value[1];
    narrow_out->heap_bits = nb.heap_bits;
    narrow_out->heap_base = nb.heap_base; narrow_out->heap_base2 = nb.heap_base2;
    return CGPU_OK;
}

void cgpu_narrowed_free(cgpu_narrowed *r) {
    if (!r) return;
    if (r->pinned) { HostBlock hb; hb.p = r->pinned; hb.cap = r->pinned_cap; hb.is_malloc = r->pinned_is_malloc; host_pool().give(hb); }
    delete r;
}

// The decision-metadata outputs of a check (cgpu_check_meta / cgpu_check_narrow_meta), host buffers covering the whole batch.
struct MetaOut {
    uint32_t *action_meta;          // n_requests * max_actions words
    cb_request_meta *request_meta;  // n_requests records
    // rule outputs (cgpu_check_outputs; null for the metadata calls): n_requests records of `stride` bytes, and the largest
    // size a record that did not fit needed (over every device's range)
    uint8_t *outputs;
    uint32_t stride;
    std::atomic<uint32_t> *needed;
};
// Device memory of the output records: each stream slot holds two chunk slabs (one filled while the other drains) within
// this budget, so a call's chunk shrinks as the stride grows instead of device memory growing with stride x chunk.
static constexpr size_t kOutputSlabBytes = 256ull << 20;
static constexpr uint32_t kMaxOutputStride = (uint32_t)(kOutputSlabBytes / 2 / 256);   // a chunk keeps at least 256 requests

static inline size_t round256(size_t n) { return (n + 255) & ~(size_t)255; }

// The batch a narrow batch stands for on the device: its per-request columns and heap at their canonical (widened) sizes,
// in cols / bytes; a null column gets a placeholder
static cgpu_batch canonical_batch(const cgpu_batch &b, const cgpu_narrow &nb, uint32_t n_slots, const void **cols, size_t *bytes) {
    const uint64_t N = b.n_requests;
    for (int i = 0; i < CGPU_N_COLUMNS; i++) { bytes[i] = b.column_bytes[i]; cols[i] = b.columns[i] ? b.columns[i] : static_cast<const void *>(""); }
    bytes[CGPU_COL_HDR0] = N * sizeof(cb_hdr0); bytes[CGPU_COL_HDR1] = N * sizeof(cb_hdr1);
    bytes[CGPU_COL_ROLES] = (size_t)nb.role_cols * N * 4;
    bytes[CGPU_COL_SLOTS] = (size_t)(n_slots ? n_slots : 1) * N * 8;
    bytes[CGPU_COL_HEAP] *= nb.heap_bits == 16 ? 4 : nb.heap_u32 ? 2 : 1;   // 16- / 32-bit heap words widen to 64 bits
    cgpu_batch c = b;
    c.columns = cols; c.column_bytes = bytes;
    return c;
}

static SlotLayout slot_layout(const cgpu_batch &b, const cgpu_narrow *nb, size_t narrow_heap_bytes, uint32_t n_slots, const MetaOut *meta) {
    SlotLayout L{};
    auto take = [&](size_t bytes) { const size_t at = L.total; L.total += round256(bytes); return at; };
    const uint64_t N = b.n_requests;
    const uint32_t km = b.max_actions ? b.max_actions : 1;
    for (int i = 0; i < CGPU_N_COLUMNS; i++) L.col[i] = take(b.column_bytes[i]);
    L.effects = take(N * km);
    if (nb) {
        L.narrow.pid = take(N * (nb->principal_id16 ? 2 : 4));
        L.narrow.hdr16 = take(N * 2 * narrow_hdr_w(*nb));
        L.narrow.versions = take(nb->versions_const ? 0 : N * 2);
        L.narrow.roles = take((size_t)nb->role_cols * N);
        for (uint32_t v = 0; v < n_slots; v++) L.narrow.slot[v] = take(N * kNarrowElemBytes[nb->slot_class[v]]);
        if (nb->heap_u32 || nb->heap_bits) L.narrow.heap = take(narrow_heap_bytes);
    }
    if (meta) { L.action_meta = take(N * km * 4); L.request_meta = take(N * sizeof(cb_request_meta)); }
    if (meta && meta->outputs) {
        L.out_chunk = (kOutputSlabBytes / 2 / meta->stride) & ~(uint64_t)255;
        L.needed = take(4);
        L.out = take(2 * L.out_chunk * meta->stride);
    }
    return L;
}

// Requests [first, first + count) of a wide batch: their columns go H2D from host view to device view; the kernels wait for them
static int upload_chunk(const cb::BatchView &hv, const cb::BatchView &dv, uint32_t n_slots, uint64_t first, uint64_t count, const Slot &slot, cudaEvent_t landed) {
    auto copy = [&](const void *dst, const void *src, size_t bytes) { return cudaMemcpyAsync(const_cast<void *>(dst), src, bytes, cudaMemcpyHostToDevice, slot.h2d); };
    CUDA_TRY(copy(dv.hdr0 + first, hv.hdr0 + first, count * sizeof(cb_hdr0)));
    CUDA_TRY(copy(dv.hdr1 + first, hv.hdr1 + first, count * sizeof(cb_hdr1)));
    for (uint32_t i = 0; i < dv.role_cols; i++) CUDA_TRY(copy(dv.roles + i * dv.stride + first, hv.roles + i * hv.stride + first, count * 4));
    for (uint32_t v = 0; v < n_slots; v++) CUDA_TRY(copy(dv.slots + v * dv.stride + first, hv.slots + v * hv.stride + first, count * 8));
    CUDA_TRY(cudaEventRecord(landed, slot.h2d));
    CUDA_TRY(cudaStreamWaitEvent(slot.stream, landed, 0));
    return CGPU_OK;
}

// Evaluates chunk cv on `stream`, effect bytes written directly.  Rule outputs (into `slab`): the reference-order body, whose
// row order they follow.  Metadata: the effect plan's unique-condition kernel in metadata form where the table has the side
// table it reads, else the reference-order body.  Effects alone: the effect launch.
static int launch_chunk(cgpu_ctx *ctx, const cgpu_table *t, const cb::BatchView &cv, const MetaOut *meta, uint8_t *dev, const SlotLayout &L, uint8_t *slab,
                        uint32_t *d_status, cudaStream_t stream) {
    uint8_t *d_effects = dev + L.effects;
    if (!meta) return launch_check(ctx, t, plan_launch(*ctx, *t, cv), cv, nullptr, d_effects, d_status, stream);
    uint32_t *d_am = reinterpret_cast<uint32_t *>(dev + L.action_meta);
    cb_request_meta *d_rm = reinterpret_cast<cb_request_meta *>(dev + L.request_meta);
    const LaunchPlan plan = meta->outputs ? LaunchPlan() : plan_launch(*ctx, *t, cv);
    const MetaDev md{d_am, d_rm};
    if (plan.uc && t->d_uc_meta) return launch_check(ctx, t, plan, cv, nullptr, d_effects, d_status, stream, &md);
    const int grid = meta->outputs ? launch_reference(ctx, check_outputs_kernel, cv.count, stream, t->desc, cv, d_effects, d_am, d_rm, d_status, slab,
                                                      meta->stride, reinterpret_cast<uint32_t *>(dev + L.needed))
                                   : launch_reference(ctx, check_meta_kernel, cv.count, stream, t->desc, cv, d_effects, d_am, d_rm, d_status);
    if (grid < 0) return grid;
    ctx->last_plan = LaunchPlan();   // (general body, no unique-condition kernel)
    ctx->last_grid = (uint32_t)grid;
    return CGPU_OK;
}

// requests [lo, hi) of `batch` on ctx's device: pipelined H2D / kernels / D2H (see below); effects_out covers the whole batch.
// meta: also the metadata planes (and rule outputs), nullptr: effects only.  nb: the batch is in the narrow form (valid).
static int check_range(cgpu_ctx *ctx, const cgpu_table *t, const cgpu_batch *batch_in, uint64_t lo, uint64_t hi, uint8_t *effects_out, const cgpu_narrow *nb,
                       const MetaOut *meta) {
    const uint32_t n_slots = t->desc.lay.n_slots;
    const void *ccols[CGPU_N_COLUMNS];
    size_t cbytes[CGPU_N_COLUMNS];
    const cgpu_batch batch = nb ? canonical_batch(*batch_in, *nb, n_slots, ccols, cbytes) : *batch_in;
    const uint64_t N = batch.n_requests;
    const uint32_t km = batch.max_actions ? batch.max_actions : 1;
    cb::BatchView hv;
    int rc = invalid(cbhost::make_batch_view(t->desc.lay, &batch, 0, N, &hv));   // validates sizes (pointers here are host pointers)
    if (rc != CGPU_OK) return rc;
    CUDA_TRY(cudaSetDevice(ctx->device));

    // acquire a slot (stream + scratch); more concurrent callers than slots simply wait
    Slot *slot = nullptr;
    for (;;) {
        {
            std::lock_guard<std::mutex> g(ctx->mu);
            for (auto &s : ctx->slots)
                if (!s.busy) { s.busy = true; slot = &s; break; }
        }
        if (slot) break;
        std::this_thread::yield();
    }
    struct Release { cgpu_ctx *c; Slot *s; ~Release() { std::lock_guard<std::mutex> g(c->mu); s->busy = false; } } rel{ctx, slot};

    if (!slot->stream) CUDA_TRY(cudaStreamCreateWithFlags(&slot->stream, cudaStreamNonBlocking));
    if (!slot->h2d) CUDA_TRY(cudaStreamCreateWithFlags(&slot->h2d, cudaStreamNonBlocking));
    if (!slot->d2h) CUDA_TRY(cudaStreamCreateWithFlags(&slot->d2h, cudaStreamNonBlocking));
    if (!slot->d_status) { CUDA_TRY(cudaMalloc(&slot->d_status, 4)); CUDA_TRY(cudaMemset(slot->d_status, 0, 4)); }
    if (!slot->h_status) CUDA_TRY(cudaMallocHost(reinterpret_cast<void **>(&slot->h_status), 4));
    // a failed call must not leave work queued on the slot's streams when the slot goes back to the pool
    struct Quiesce { Slot *s; bool armed = true; ~Quiesce() { if (armed) { cudaStreamSynchronize(s->h2d); cudaStreamSynchronize(s->stream); cudaStreamSynchronize(s->d2h); } } } quiesce{slot};

    const SlotLayout L = slot_layout(batch, nb, batch_in->column_bytes[CGPU_COL_HEAP], n_slots, meta);
    if (slot->dev_cap < L.total) {
        if (slot->dev) cudaFree(slot->dev);
        slot->dev = nullptr; slot->dev_cap = 0;
        CUDA_TRY(cudaMalloc(&slot->dev, L.total));
        slot->dev_cap = L.total;
    }
    uint8_t *dev = static_cast<uint8_t *>(slot->dev);
    const void *dcols[CGPU_N_COLUMNS];
    for (int i = 0; i < CGPU_N_COLUMNS; i++) dcols[i] = dev + L.col[i];
    cgpu_batch db = batch;
    db.columns = dcols;
    cb::BatchView bv;
    rc = invalid(cbhost::make_batch_view(t->desc.lay, &db, 0, N, &bv));
    if (rc != CGPU_OK) return rc;

    // Pipeline: the batch-level tables and the heap go first, then the per-request columns travel in chunks of
    // `chunk` requests -- while chunk k is evaluated, chunk k+1 is on its way in and the effect bytes of chunk k-1 on
    // their way out (three streams, PCIe in both directions at once).  The kernels take a sub-range of the batch
    // (BatchView::first / count over columns of stride N), so nothing is re-packed.  Host buffers should be pinned
    // (cudaHostAlloc / cudaHostRegister): pageable memory makes every copy synchronous.
    // Chunk size: every column of a chunk is one copy, so chunks must be large for the link to run near its rate -- measured
    // on C3's narrow form (52 B / request): 2^18 requests 38 GB/s, 2^19 42.5, 2^20 44.8, 2^21 46.3, 2^22 44.6
    // (tools/e2e_chunk_sweep.py) -- but a call should still be cut in two so that copy-in, kernels and copy-out overlap.
    const bool outs = meta && meta->outputs;
    const char *ce = getenv("CERBOS_B200_CHECK_CHUNK");
    uint64_t chunk = ce ? strtoull(ce, nullptr, 10) : (1ull << 21);
    if (!ce && hi - lo < 2 * chunk) {
        chunk = (hi - lo + 1) / 2;
        if (chunk < (1ull << 18)) chunk = 1ull << 18;
        chunk = round256(chunk);
    }
    if (chunk < 4096) chunk = 4096;
    chunk &= ~(uint64_t)255;
    if (outs && chunk > L.out_chunk) chunk = L.out_chunk;
    const uint64_t n_chunks = (hi - lo + chunk - 1) / chunk;
    const uint64_t n_ev = (outs ? 3 : 2) * n_chunks;   // per chunk: columns in, kernel done, (outputs) output slab drained
    if (outs) CUDA_TRY(cudaMemsetAsync(dev + L.needed, 0, 4, slot->stream));
    while (slot->ev.size() < n_ev) {
        cudaEvent_t e;
        CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        slot->ev.push_back(e);
    }
    // the batch-level tables and the heap, once per call; a 16- or 32-bit heap is widened into the canonical one on the copy stream
    const bool narrow_heap = nb && (nb->heap_u32 || nb->heap_bits);
    if (const size_t hb = narrow_heap ? batch_in->column_bytes[CGPU_COL_HEAP] : 0) {
        CUDA_TRY(cudaMemcpyAsync(dev + L.narrow.heap, batch.columns[CGPU_COL_HEAP], hb, cudaMemcpyHostToDevice, slot->h2d));
        const uint64_t words = hb / (nb->heap_bits == 16 ? 2 : 4), tiles = (words + kThreads - 1) / kThreads;
        const unsigned hgrid = (unsigned)(tiles < 1184 ? tiles : 1184);
        uint64_t *heap = reinterpret_cast<uint64_t *>(dev + L.col[CGPU_COL_HEAP]);
        if (nb->heap_bits == 16) widen_heap16_kernel<<<hgrid, kThreads, 0, slot->h2d>>>(reinterpret_cast<const uint16_t *>(dev + L.narrow.heap), heap, words, nb->heap_base, nb->heap_base2);
        else widen_heap_kernel<<<hgrid, kThreads, 0, slot->h2d>>>(reinterpret_cast<const uint32_t *>(dev + L.narrow.heap), heap, words);
        CUDA_TRY(cudaGetLastError());
        ctx->launches.fetch_add(1, std::memory_order_relaxed);
    }
    for (int i = narrow_heap ? CGPU_COL_HEAP + 1 : CGPU_COL_HEAP; i < CGPU_N_COLUMNS; i++)
        if (batch.column_bytes[i]) CUDA_TRY(cudaMemcpyAsync(dev + L.col[i], batch.columns[i], batch.column_bytes[i], cudaMemcpyHostToDevice, slot->h2d));
    WidenParams wp{};
    if (nb) wp = widen_params(*nb, N, n_slots, dev, L);
    for (uint64_t k = 0; k < n_chunks; k++) {
        const uint64_t c0 = lo + k * chunk, cnt = hi - c0 < chunk ? hi - c0 : chunk;
        rc = nb ? upload_narrow_chunk(*nb, wp, c0, cnt, slot->h2d, slot->ev[2 * k], slot->stream, ctx->launches)
                : upload_chunk(hv, bv, n_slots, c0, cnt, *slot, slot->ev[2 * k]);
        if (rc != CGPU_OK) return rc;
        cb::BatchView cv = bv;
        cv.first = c0; cv.count = cnt;
        uint8_t *slab = outs ? dev + L.out + (k & 1) * L.out_chunk * meta->stride : nullptr;
        if (outs && k >= 2) CUDA_TRY(cudaStreamWaitEvent(slot->stream, slot->ev[2 * n_chunks + k - 2], 0));   // that slab's last copy-out
        rc = launch_chunk(ctx, t, cv, meta, dev, L, slab, slot->d_status, slot->stream);
        if (rc != CGPU_OK) return rc;
        CUDA_TRY(cudaEventRecord(slot->ev[2 * k + 1], slot->stream));
        CUDA_TRY(cudaStreamWaitEvent(slot->d2h, slot->ev[2 * k + 1], 0));
        CUDA_TRY(cudaMemcpyAsync(effects_out + c0 * km, dev + L.effects + c0 * km, cnt * km, cudaMemcpyDeviceToHost, slot->d2h));
        if (meta) {
            CUDA_TRY(cudaMemcpyAsync(meta->action_meta + c0 * km, dev + L.action_meta + c0 * km * 4, cnt * km * 4, cudaMemcpyDeviceToHost, slot->d2h));
            CUDA_TRY(cudaMemcpyAsync(meta->request_meta + c0, dev + L.request_meta + c0 * sizeof(cb_request_meta), cnt * sizeof(cb_request_meta), cudaMemcpyDeviceToHost, slot->d2h));
        }
        if (outs) {
            CUDA_TRY(cudaMemcpyAsync(meta->outputs + c0 * meta->stride, slab, cnt * meta->stride, cudaMemcpyDeviceToHost, slot->d2h));
            CUDA_TRY(cudaEventRecord(slot->ev[2 * n_chunks + k], slot->d2h));
        }
    }
    uint32_t h_need = 0;
    if (outs) CUDA_TRY(cudaMemcpyAsync(&h_need, dev + L.needed, 4, cudaMemcpyDeviceToHost, slot->d2h));
    CUDA_TRY(cudaMemcpyAsync(slot->h_status, slot->d_status, 4, cudaMemcpyDeviceToHost, slot->d2h));   // behind the last chunk's results
    CUDA_TRY(cudaStreamSynchronize(slot->d2h));
    quiesce.armed = false;   // d2h waited for every kernel, every kernel for its columns: all three streams are idle
    if (const uint32_t st = *slot->h_status) {
        CUDA_TRY(cudaMemset(slot->d_status, 0, 4));
        if (st & 1u)
            return fail(CGPU_ERR_UNSUPPORTED, "a request produced a run-time value the device cannot represent exactly (e.g. timestamp outside 1678..2262, string->double, concatenation)");
        if (outs && (st & cb::CB_OUT_STATUS_UNLOWERED))
            return fail(CGPU_ERR_UNSUPPORTED, "a request reached a rule output the device cannot evaluate (the table's MANIFEST lists them as unlowered_outputs)");
        if (outs && (st & cb::CB_OUT_STATUS_OVERFLOW)) {
            uint32_t cur = meta->needed->load();
            while (h_need > cur && !meta->needed->compare_exchange_weak(cur, h_need)) {}
            return fail(CGPU_ERR_UNSUPPORTED, "rule outputs: a request's output record needs %u bytes, more than the stride of %u", h_need, meta->stride);
        }
    }
    return CGPU_OK;
}

// Every host-buffer check (cgpu_check, cgpu_check_narrow, cgpu_check_meta, cgpu_check_narrow_meta) on the devices of ctx.
// A context over several devices (cgpu_init with n_devices > 1): the requests are independent (engine.go:302-310), so the
// batch is cut into one contiguous index range per device, each range travels over that device's own PCIe link and is
// evaluated there; results land index-aligned in the outputs.  The narrow columns are addressed by absolute request index
// with stride N like the wide ones, so a range of a narrow batch is cut the same way.  One host thread per device.
static int check_sharded(cgpu_ctx *ctx, const cgpu_table *t, const cgpu_batch *batch, uint8_t *effects_out, const cgpu_narrow *nb, const MetaOut *meta) {
    const uint64_t N = batch->n_requests;
    if (N == 0) return CGPU_OK;
    const size_t n_dev = 1 + ctx->peers.size();
    if (n_dev == 1 || N < 2 * 4096) return check_range(ctx, t, batch, 0, N, effects_out, nb, meta);
    if (t->peer_tables.size() != ctx->peers.size()) return fail(CGPU_ERR_INVALID, "table was not loaded on every device of the context");
    std::vector<int> rcs(n_dev, CGPU_OK);
    std::vector<std::string> errs(n_dev);
    const uint64_t per = (((N + n_dev - 1) / n_dev) + 255) & ~(uint64_t)255;
    std::vector<std::thread> th;
    auto work = [&](size_t d) {
        const uint64_t lo = d * per < N ? d * per : N, hi = lo + per < N ? lo + per : N;
        if (lo >= hi) return;
        rcs[d] = d == 0 ? check_range(ctx, t, batch, lo, hi, effects_out, nb, meta)
                        : check_range(ctx->peers[d - 1], t->peer_tables[d - 1], batch, lo, hi, effects_out, nb, meta);
        if (rcs[d] != CGPU_OK) errs[d] = g_err;
    };
    for (size_t d = 1; d < n_dev; d++) th.emplace_back(work, d);
    work(0);
    for (auto &x : th) x.join();
    for (size_t d = 0; d < n_dev; d++)
        if (rcs[d] != CGPU_OK) return fail(rcs[d], "device %zu: %s", d, errs[d].c_str());
    return CGPU_OK;
}

// the argument checks of the narrow entry points, the whole descriptor included, before any device work and at any batch size
static int narrow_args(const char *fn, cgpu_ctx *ctx, const cgpu_table *t, const cgpu_batch *batch, const cgpu_narrow *nb, const uint8_t *effects_out) {
    if (!ctx || !t || !batch || !nb || !effects_out) return fail(CGPU_ERR_INVALID, "%s: null argument", fn);
    if (t->ctx != ctx) return fail(CGPU_ERR_INVALID, "table belongs to another context");
    if (!nb->roles || !nb->slot_class || !nb->slot_cols || nb->role_cols == 0 || (nb->hdr_const_mask & ~15u) || (narrow_hdr_w(*nb) && !nb->hdr16) ||
        (!nb->versions_const && !nb->versions) || (!nb->principal_id16 && !nb->principal_id))
        return fail(CGPU_ERR_INVALID, "%s: missing narrow column", fn);
    if (nb->heap_bits != 0 && nb->heap_bits != 16) return fail(CGPU_ERR_INVALID, "%s: heap_bits %u (0 or 16)", fn, nb->heap_bits);
    const uint32_t n_slots = t->desc.lay.n_slots;
    if (n_slots > kMaxNarrowSlots) return fail(CGPU_ERR_INVALID, "%s: more than %u attribute slots", fn, kMaxNarrowSlots);
    for (uint32_t v = 0; v < n_slots; v++) {
        const uint32_t cl = nb->slot_class[v];
        if (cl > CGPU_SLOT_U8_NUM) return fail(CGPU_ERR_INVALID, "%s: slot class %u", fn, cl);
        if (cl == CGPU_SLOT_U16_ID && !nb->slot_base) return fail(CGPU_ERR_INVALID, "%s: CGPU_SLOT_U16_ID needs slot_base", fn);
    }
    return CGPU_OK;
}

int cgpu_check_narrow(cgpu_ctx *ctx, const cgpu_table *t, const cgpu_batch *batch, const cgpu_narrow *narrow, uint8_t *effects_out) {
    const int rc = narrow_args("cgpu_check_narrow", ctx, t, batch, narrow, effects_out);
    if (rc != CGPU_OK) return rc;
    return check_sharded(ctx, t, batch, effects_out, narrow, nullptr);
}

int cgpu_check(cgpu_ctx *ctx, const cgpu_table *t, const cgpu_batch *batch, uint8_t *effects_out) {
    if (!ctx || !t || !batch || !effects_out) return fail(CGPU_ERR_INVALID, "cgpu_check: null argument");
    if (t->ctx != ctx) return fail(CGPU_ERR_INVALID, "table belongs to another context");
    return check_sharded(ctx, t, batch, effects_out, nullptr, nullptr);
}

int cgpu_check_meta(cgpu_ctx *ctx, const cgpu_table *t, const cgpu_batch *batch, uint8_t *effects_out, uint32_t *action_meta_out, void *request_meta_out) {
    if (!ctx || !t || !batch || !effects_out || !action_meta_out || !request_meta_out) return fail(CGPU_ERR_INVALID, "cgpu_check_meta: null argument");
    if (t->ctx != ctx) return fail(CGPU_ERR_INVALID, "table belongs to another context");
    const MetaOut meta{action_meta_out, static_cast<cb_request_meta *>(request_meta_out)};
    return check_sharded(ctx, t, batch, effects_out, nullptr, &meta);
}

int cgpu_check_outputs(cgpu_ctx *ctx, const cgpu_table *t, const cgpu_batch *batch, uint8_t *effects_out, uint32_t *action_meta_out,
                       void *request_meta_out, uint8_t *outputs_out, uint32_t outputs_stride, uint32_t *outputs_bytes_needed) {
    if (!ctx || !t || !batch || !effects_out || !action_meta_out || !request_meta_out || !outputs_out || !outputs_bytes_needed)
        return fail(CGPU_ERR_INVALID, "cgpu_check_outputs: null argument");
    if (t->ctx != ctx) return fail(CGPU_ERR_INVALID, "table belongs to another context");
    *outputs_bytes_needed = 0;
    if (outputs_stride < CB_OUT_RECORD_HEADER || outputs_stride % 8 || outputs_stride > kMaxOutputStride)
        return fail(CGPU_ERR_INVALID, "cgpu_check_outputs: outputs_stride %u (a multiple of 8 in [%d, %u])", outputs_stride, CB_OUT_RECORD_HEADER, kMaxOutputStride);
    std::atomic<uint32_t> needed{0};
    const MetaOut meta{action_meta_out, static_cast<cb_request_meta *>(request_meta_out), outputs_out, outputs_stride, &needed};
    const int rc = check_sharded(ctx, t, batch, effects_out, nullptr, &meta);
    *outputs_bytes_needed = needed.load();
    return rc;
}

int cgpu_check_narrow_meta(cgpu_ctx *ctx, const cgpu_table *t, const cgpu_batch *batch, const cgpu_narrow *narrow, uint8_t *effects_out,
                           uint32_t *action_meta_out, void *request_meta_out) {
    if (!action_meta_out || !request_meta_out) return fail(CGPU_ERR_INVALID, "cgpu_check_narrow_meta: null argument");
    const int rc = narrow_args("cgpu_check_narrow_meta", ctx, t, batch, narrow, effects_out);
    if (rc != CGPU_OK) return rc;
    const MetaOut meta{action_meta_out, static_cast<cb_request_meta *>(request_meta_out)};
    return check_sharded(ctx, t, batch, effects_out, narrow, &meta);
}

}  // extern "C"
