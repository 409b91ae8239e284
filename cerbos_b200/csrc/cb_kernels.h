// cb_kernels.h -- device bodies of the CheckResources kernels (sm_90a).
//
// Included twice: by cerbos_b200.cu (ahead-of-time build: every body, generic block walker) and, as embedded text,
// by the translation unit the library compiles with NVRTC when a table is loaded (CB_LEAN_ONLY: lean bodies only,
// with the straight-line block evaluators cb_specialize.h generates from that table).
//
// Kernel design (H100):
//   * persistent grid: (SM count x resident CTAs) CTAs of 256 threads loop over 256-request tiles;
//   * the flattened rule table image (row blocks, scope tables, bytecode, constants; KBs) is staged ONCE per CTA
//     into shared memory by the TMA unit: 1-D `cp.async.bulk.shared::cluster.global` copies completing on an
//     mbarrier, overlapped with the first tile's loads; tables too large for shared memory are read through L1/L2;
//   * index-order lean launches stage the REQUEST COLUMNS the same way, tile by tile, double-buffered;
//   * one thread per request, bit-parallel (action x role) walk + condition evaluation (cb_core.h);
//   * result: 1 bit per decision (or 1 byte for the host-buffer ABI), coalesced stores.
// Integer / branchy work bounded by HBM bandwidth: no tensor cores are involved.
#pragma once
#include "cb_core.h"

namespace cbk {

constexpr int kThreads = 256;

struct TableDesc {
    const uint8_t *base;       // device blob image
    cb::TableLayout lay;       // section offsets + dims (image_bytes: bytes [0, image_bytes) hold every device section)
};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok = 0;
    while (!ok) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok)
                     : "r"(smem_u32(bar)), "r"(parity)
                     : "memory");
    }
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// 1-D bulk copy global -> shared by the TMA unit, completing `bytes` on the mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_load_1d(void *dst_smem, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)), "l"(src),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void tma_load_image(uint8_t *dst_smem, const TableDesc &td, uint64_t *bar) {   // one thread
    mbar_expect_tx(bar, td.lay.image_bytes);
    for (uint32_t o = 0; o < td.lay.image_bytes; o += 32768) {   // <= 32 KB per copy, all completing on the same mbarrier
        uint32_t nb = td.lay.image_bytes - o < 32768 ? td.lay.image_bytes - o : 32768;
        tma_load_1d(dst_smem + o, td.base + o, nb, bar);
    }
}

// A request the lean body cannot decide (differing policy versions, an operand outside the 8-byte fast forms ...) is
// appended to the launch's deferral list, which the general kernel drains right behind this one.  (Only the general
// and the metadata kernels carry the generic interpreter: it is compiled once per kernel that can reach it.)
__device__ __forceinline__ void defer_request(const cb::TableView tv, const cb::BatchView &bv, uint64_t n, uint8_t *bitmap, uint8_t *effects, uint32_t *status) {
    (void)tv; (void)bitmap; (void)effects; (void)status;
    const uint32_t k = atomicAdd(bv.defer_count, 1u);
    bv.defer_list[k] = (uint32_t)(n - bv.first);
}

// fused all-gather bookkeeping (see BatchView): executed by one warp
__device__ __forceinline__ void gather_signal_flags(const cb::BatchView &bv) {
    __threadfence_system();
    // max, not a plain store: consecutive launches overlap at their tails, the cell must never step backwards
    if (threadIdx.x < bv.n_out) asm volatile("red.release.sys.global.max.u32 [%0], %1;" ::"l"(bv.sig_flags[threadIdx.x] + bv.sig_rank), "r"(bv.sig_step) : "memory");
}
__device__ __forceinline__ void gather_wait_flags(const uint32_t *flags, uint32_t n_ranks, uint32_t step) {
    if (threadIdx.x < n_ranks) {
        uint32_t v;
        do {
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + threadIdx.x) : "memory");
        } while ((int)(v - step) < 0);
    }
}

// Persistent body, columns read straight from global memory (any evaluation order: bv.perm).
// kFast: the lean resource-policy-only body (cb::eval_request_fast), else the general body with 64-bit pair masks.
// kStageMode 0: table read from global memory, 1: from the staged shared-memory image (compile-time, so that every
// table access of the lean body is an LDS with 32-bit address arithmetic instead of a generic load), 2: decided by
// the `stage_rt` argument (general body: one instantiation keeps the build time down).
template <bool kFast, int kStageMode, typename Blocks>
__device__ __forceinline__ void check_body(const TableDesc &td, const cb::BatchView &bv, uint8_t *bitmap, uint8_t *effects, uint32_t *status, const uint32_t stage_rt,
                                           uint8_t *smem_image, uint64_t *mbar) {
    const bool kStage = kStageMode == 2 ? stage_rt != 0 : kStageMode == 1;
    // deferred mode (drains the list a specialised lean kernel left): the request count lives in device memory.  The
    // launch is programmatically serialised behind that kernel (its CTAs become resident while the last tiles of the
    // producer are still running): wait here until the producer has completed and its writes are visible.
    if (bv.count_dev) {
        // let the NEXT launch's specialised kernel (programmatically serialised behind this one) take SM slots as the
        // producer's last tiles retire: it does not depend on anything this launch writes
        asm volatile("griddepcontrol.launch_dependents;");
        asm volatile("griddepcontrol.wait;" ::: "memory");
        if (blockIdx.x == 0 && threadIdx.x == 0) bv.count_dev[2] = 0;   // the producer's tile counter: back to zero for the cell's next user
        if (blockIdx.x == 0 && threadIdx.x < 32 && bv.wait_step) gather_wait_flags(bv.wait_flags, bv.n_out, bv.wait_step);
    }
    const uint64_t count = bv.count_dev ? (uint64_t)*bv.count_dev : bv.count;
    if (count == 0) {   // the usual case in deferred mode: nothing was deferred
        if (bv.count_dev && bv.sig_step && blockIdx.x == 0 && threadIdx.x < 32) gather_signal_flags(bv);
        return;
    }
    // the cell's last word keeps a running total of the requests drained through it (cgpu_deferred_count)
    if (bv.count_dev && blockIdx.x == 0 && threadIdx.x == 0) bv.count_dev[3] += (uint32_t)count;
    const uint8_t *base = td.base;
    if (kStage) {
        if (threadIdx.x == 0) {
            mbar_init(mbar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();
        if (threadIdx.x == 0) tma_load_image(smem_image, td, mbar);
        base = smem_image;
    }
#ifdef CB_LEAN_ONLY
    asm volatile("griddepcontrol.launch_dependents;");
#endif
    cb::TableView tv;
    tv.base = kStageMode == 1 ? smem_image : kStageMode == 0 ? td.base : base;
    tv.L = &td.lay;
    const uint64_t n_tiles = (count + kThreads - 1) / kThreads;
    {   // columns of this thread's first request: in flight while the table image is still being staged
        const uint64_t i0 = (uint64_t)blockIdx.x * kThreads + threadIdx.x;
        if (i0 < count) cb::prefetch_request(bv, bv.first + (bv.perm ? bv.perm[i0] : i0));
    }
    bool staged = !kStage;
    for (uint64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        uint64_t i = tile * kThreads + threadIdx.x;
        // clustered order: thread i evaluates request perm[i] (cluster kernels), so that the lanes of a warp walk the
        // same policy blocks
        uint64_t req = i, req_next = i + (uint64_t)gridDim.x * kThreads;
        if (bv.perm) {
            if (i < count) req = bv.perm[i];
            if (req_next < count) req_next = bv.perm[req_next]; else req_next = count;
        }
        if (!staged) {   // every thread waits for the table image (phase 0) before its first table access
            mbar_wait(mbar, 0);
            staged = true;
        }
        // the next tile of this thread: start pulling its columns towards L1 now
        if (req_next < count) cb::prefetch_request(bv, bv.first + req_next);
        if (i < count) {
            if (kFast) {
                cb::GlobalCols gc;
                gc.b = &bv; gc.n = bv.first + req;
                if (cb::eval_request_fast(tv, bv, gc, bv.first + req, bitmap, effects, Blocks())) defer_request(tv, bv, bv.first + req, bitmap, effects, status);
            } else {
#ifndef CB_LEAN_ONLY
                cb::eval_request<uint64_t>(tv, bv, bv.first + req, bitmap, effects, status);
#endif
            }
        }
    }
    if (!staged) mbar_wait(mbar, 0);   // CTA had no tile: drain the bulk copy before shared memory is released
#ifdef CB_LEAN_ONLY
    asm volatile("griddepcontrol.wait;" ::: "memory");   // see check_tiles_body: complete only after the previous launch has
#endif
    if (bv.count_dev) {
        // deferred mode: the last CTA to finish hands the {count, done} cell back zeroed (it comes from a small pool of
        // pre-zeroed cells, so that a launch needs no memset)
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence();
            if (atomicAdd(bv.count_dev + 1, 1u) == gridDim.x - 1) { bv.count_dev[0] = 0; bv.count_dev[1] = 0; mbar[0] = 1; } else mbar[0] = 0;
        }
        __syncthreads();
        if (bv.sig_step && mbar[0] == 1 && threadIdx.x < 32) gather_signal_flags(bv);   // the last CTA: every result of this launch is stored
    }
}

// Lean body with BOTH the table image and the request columns staged by the TMA unit.  Index-order batches only
// (the columns of a tile of 256 requests are contiguous runs: 2 + role_cols + n_slots bulk copies per tile, issued by
// one thread, double-buffered: tile k+1 streams into shared memory while tile k is evaluated, so no thread ever
// waits on DRAM and every column read is an LDS).  Shared memory: [image][tile stage 0][tile stage 1].
template <typename Blocks>
__device__ __forceinline__ void check_tiles_body(const TableDesc &td, const cb::BatchView &bv, uint8_t *bitmap, uint8_t *effects, uint32_t *status, const uint32_t n_slots,
                                                 uint8_t *smem_image, uint64_t *mbar_tab, uint64_t *mbar_col /* [4]: full[2], empty[2] */) {
    const uint32_t image_pad = (td.lay.image_bytes + 127u) & ~127u;
    const uint32_t tile_bytes = cb::tile_cols_bytes(bv.role_cols, n_slots);
    const uint32_t slots_off = cb::CB_TILE * (24u + 4u * bv.role_cols);
    uint8_t *stage0 = smem_image + image_pad;
    const uint64_t n_tiles = (bv.count + kThreads - 1) / kThreads, n_full = bv.count / kThreads;
    uint64_t *full = mbar_col, *empty = mbar_col + 2;
    // small per-batch tables behind the two tile stages: row x action-set masks and actions per action set
    uint64_t *row_am_s = reinterpret_cast<uint64_t *>(stage0 + 2 * tile_bytes);
    const uint32_t n_am = bv.n_asets * bv.n_rows;
    uint32_t *aset_k_s = reinterpret_cast<uint32_t *>(row_am_s + n_am);

    auto issue_tile = [&](uint64_t tile, uint32_t st) {   // one thread: bulk copies of every column run of `tile`
        uint8_t *dst = stage0 + st * tile_bytes;
        const uint64_t r0 = bv.first + tile * kThreads;
        mbar_expect_tx(&full[st], tile_bytes);
        tma_load_1d(dst, bv.hdr0 + r0, kThreads * 16, &full[st]);
        tma_load_1d(dst + kThreads * 16, bv.hdr1 + r0, kThreads * 8, &full[st]);
        for (uint32_t i = 0; i < bv.role_cols; i++) tma_load_1d(dst + kThreads * 24 + i * (kThreads * 4), bv.roles + i * bv.stride + r0, kThreads * 4, &full[st]);
        for (uint32_t v = 0; v < n_slots; v++) tma_load_1d(dst + slots_off + v * (kThreads * 8), bv.slots + v * bv.stride + r0, kThreads * 8, &full[st]);
    };

    if (threadIdx.x == 0) {
        mbar_init(mbar_tab, 1);
        mbar_init(&full[0], 1);
        mbar_init(&full[1], 1);
        mbar_init(&empty[0], kThreads / 32);   // one arrival per warp
        mbar_init(&empty[1], kThreads / 32);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        tma_load_image(smem_image, td, mbar_tab);
        if (blockIdx.x < n_full) issue_tile(blockIdx.x, 0);
    }
#ifdef CB_LEAN_ONLY
    asm volatile("griddepcontrol.launch_dependents;");   // the drain kernel's CTAs may take the slots this grid frees at its tail
#endif
    for (uint32_t j = threadIdx.x; j < n_am; j += kThreads) row_am_s[j] = bv.row_am[j];
    for (uint32_t j = threadIdx.x; j < bv.n_asets; j += kThreads) aset_k_s[j] = bv.aset_k[j];
    __syncthreads();
    cb::TableView tv;
    tv.base = smem_image;
    tv.L = &td.lay;
    // Tile order: the first tile of a CTA is its block index; the following ones come from a global counter when the
    // launch provides one (claimed by thread 0 one tile ahead, published through `tile_s` under the stage's full
    // barrier), so the tail of the grid stays balanced; else the static grid stride.
    uint64_t *tile_s = reinterpret_cast<uint64_t *>(aset_k_s + ((bv.n_asets + 1u) & ~1u));   // [2]
    // fused all-gather: result bytes of a tile, per stage; warp 0 forwards them to the peers once the tile is complete
    uint8_t *res_s = reinterpret_cast<uint8_t *>(tile_s + 2);                                // [2][kThreads]
    bool remote = bv.n_out > 1 && bv.kbytes == 1 && (bv.first & 7) == 0;
    for (uint32_t r = 0; r < bv.n_out; r++) remote = remote && (reinterpret_cast<uintptr_t>(bv.outs[r]) & 7) == 0;   // 8-byte stores per lane
    auto flush_remote = [&](uint32_t st, uint64_t t) {   // warp 0, all lanes: 256 bytes of tile t to every peer, 8 bytes per lane
        const uint64_t v = *reinterpret_cast<const uint64_t *>(res_s + st * kThreads + threadIdx.x * 8);
        for (uint32_t r = 0; r < bv.n_out; r++)
            if (r != bv.sig_rank) *reinterpret_cast<uint64_t *>(bv.outs[r] + bv.first + t * kThreads + threadIdx.x * 8) = v;
    };
    uint32_t k = 0;
    uint64_t tile = blockIdx.x, prev_tile = 0;
    while (tile < n_tiles) {
        if (threadIdx.x < 32) {
            const uint32_t st = (k + 1) & 1;
            // stage st was read in iteration k-1: reuse it once all eight warps have released it.  No CTA-wide barrier:
            // only this warp waits, and it is normally released long before
            if (k >= 1) {
                if (threadIdx.x == 0) mbar_wait(&empty[st], ((k - 1) >> 1) & 1);
                __syncwarp();
                if (remote && prev_tile < n_full) flush_remote(st, prev_tile);   // before the refill lets anyone overwrite res_s[st]
                __syncwarp();
            }
            if (threadIdx.x == 0) {
                const uint64_t next = bv.tile_counter ? (uint64_t)atomicAdd(bv.tile_counter, 1u) + gridDim.x : tile + gridDim.x;
                tile_s[st] = next;
                if (next < n_full) issue_tile(next, st);
                else asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&full[st])) : "memory");   // nothing to copy: complete the phase
            }
            __syncwarp();
        }
        if (k == 0) mbar_wait(mbar_tab, 0);
        const uint64_t n = bv.first + tile * kThreads + threadIdx.x;
        if (tile < n_full) {
            if (k == 0) mbar_wait(&full[0], 0);
            cb::TileCols tc;
            tc.base = stage0 + (k & 1) * tile_bytes; tc.tid = threadIdx.x; tc.slots_off = slots_off;
            tc.aset_k_s = aset_k_s; tc.row_am_s = row_am_s;
            tc.res_s = remote ? res_s + (k & 1) * kThreads : nullptr;
            if (cb::eval_request_fast(tv, bv, tc, n, bitmap, effects, Blocks())) defer_request(tv, bv, n, bitmap, effects, status);
        } else if (tile * kThreads + threadIdx.x < bv.count) {   // the ragged last tile: straight from global memory
            cb::GlobalCols gc;
            gc.b = &bv; gc.n = n;
            if (cb::eval_request_fast(tv, bv, gc, n, bitmap, effects, Blocks())) defer_request(tv, bv, n, bitmap, effects, status);
        }
        __syncwarp();
        if ((threadIdx.x & 31) == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&empty[k & 1])) : "memory");
        // next tile: its index (and, for a full tile, its columns) are published when stage (k+1)&1 completes
        prev_tile = tile;
        k++;
        mbar_wait(&full[k & 1], (k >> 1) & 1);
        tile = tile_s[k & 1];
    }
    if (remote && k >= 1 && threadIdx.x < 32 && prev_tile < n_full) {   // results of the last tile
        if (threadIdx.x == 0) mbar_wait(&empty[(k - 1) & 1], ((k - 1) >> 1) & 1);
        __syncwarp();
        flush_remote((k - 1) & 1, prev_tile);
    }
    if (k == 0) mbar_wait(mbar_tab, 0);   // no tile: drain the table copy before shared memory is released
#ifdef CB_LEAN_ONLY
    // launched programmatically serialised behind the previous launch's drain kernel and never synchronised with it so
    // far: do not COMPLETE before it has (keeps "this kernel done => everything before it in the stream done")
    asm volatile("griddepcontrol.wait;" ::: "memory");
#endif
}

// Unique-condition body (cb::eval_request_uc): index order, columns read straight from global memory with coalesced
// loads (a warp covers 32 consecutive requests: 256 B per slot column), every lane running the same instruction stream
// whatever policy block its request hits.  No column staging: the specialised build pulls all the slots of a request
// into registers up front, so each warp keeps ~(3 + role_cols + n_slots) independent loads in flight and the SM's
// occupancy is bounded by registers only.  kStaged: the compact table image (cb_uc.h; a few KB) is staged once per
// persistent CTA by the TMA unit and the rows are merged with the batch's row x action-set masks into one 8-byte record
// per row in shared memory; otherwise both are read from global memory (images too large for shared memory).
// Work distribution is warp-granular: warp w of the grid takes the 32-request chunks w, w + n_warps, ... -- no
// CTA-wide barrier in the loop.  Deferred requests (an operand the 8-byte forms cannot decide, differing policy
// versions) go to the launch's deferral list, drained by the general kernel right behind; they are first written as
// DENY so that a lost deferral could only fail closed.
// smem layout (kStaged): [image, 128-byte padded][merged rows: n_asets x uc_n_rows (slots or rows) x 16 B]
// Meta: UcMeta -- the metadata form (cb::eval_request_uc_meta: effect bytes, action words and request records; the
// deferred requests go to the reference-order body, check_meta_kernel), else the effect form.
struct UcEffects { static constexpr bool kMeta = false; };
struct UcMeta {
    static constexpr bool kMeta = true;
    uint32_t *action_meta;
    cb_request_meta *req_meta;
    const cb::U4 *side;   // cbuc::build_meta
};
template <typename Conds, typename Cols, bool kStaged, typename Meta = UcEffects>
__device__ __forceinline__ void check_uc_body(const TableDesc &td, const cb::BatchView &bv, uint8_t *bitmap, uint8_t *effects, uint8_t *smem_image, uint64_t *mbar,
                                              const Meta meta = Meta()) {
    cb::TableView tv;
    tv.L = &td.lay;
    tv.base = kStaged ? smem_image : td.base;
    const cb::U4 *pk = kStaged ? nullptr : bv.uc_rows_pk;   // global image: the rows merged by the launch's pre-pass, if any
    // prefetch table: the 128-byte lines the columns of 32 consecutive requests span (hdr0 4, hdr1 2, a role column 1, a slot
    // column 2), as column base + offset of the line and the shift that turns a request index into a byte offset
    __shared__ unsigned long long pf_base[64];
    __shared__ uint32_t pf_shift[64];
    const uint32_t n_pf = min(64u, 6u + bv.role_cols + 2u * td.lay.n_slots);
    for (uint32_t q = threadIdx.x; q < n_pf; q += kThreads) {
        unsigned long long p;
        uint32_t sh;
        if (q < 4) { p = (unsigned long long)bv.hdr0 + q * 128u; sh = 4; }
        else if (q < 6) { p = (unsigned long long)bv.hdr1 + (q - 4) * 128u; sh = 3; }
        else if (q < 6 + bv.role_cols) { p = (unsigned long long)(bv.roles + (uint64_t)(q - 6) * bv.stride); sh = 2; }
        else { const uint32_t v = q - 6 - bv.role_cols; p = (unsigned long long)(bv.slots + (uint64_t)(v >> 1) * bv.stride) + (v & 1u) * 128u; sh = 3; }
        pf_base[q] = p;
        pf_shift[q] = sh;
    }
    if (!kStaged) __syncthreads();
    if (kStaged) {
        if (threadIdx.x == 0) {
            mbar_init(mbar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();
        if (threadIdx.x == 0) tma_load_image(smem_image, td, mbar);
        mbar_wait(mbar, 0);
        cb::U4 *pks = reinterpret_cast<cb::U4 *>(smem_image + ((td.lay.image_bytes + 127u) & ~127u));
        const uint32_t n_u = td.lay.uc_n_rows, n_pk = bv.n_asets * n_u;
        cb::UcRowsGlobal g; g.urows = tv.urows(); g.row_am = bv.row_am; g.RCP = bv.rcp; g.nR = td.lay.nR;
        for (uint32_t j = threadIdx.x; j < n_pk; j += kThreads) pks[j] = g.aset(tv, bv, j / n_u).merged(tv, j % n_u);
        __syncthreads();
        pk = pks;
    }
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t n_chunks = (bv.count + 31) / 32;
    const uint64_t n_warps = (uint64_t)gridDim.x * (kThreads / 32);
    for (uint64_t chunk = (uint64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5); chunk < n_chunks; chunk += n_warps) {
        const uint64_t i = chunk * 32 + lane;
        {   // this warp's next chunk: pull its columns towards L2 now, one lane per 128-byte line (table built above)
            const uint64_t c2 = chunk + n_warps;
            if (c2 * 32 + 32 <= bv.count) {
                const uint64_t n2 = bv.first + c2 * 32;
                for (uint32_t q = lane; q < n_pf; q += 32) asm volatile("prefetch.global.L2 [%0];" ::"l"(pf_base[q] + (n2 << pf_shift[q])));
            }
        }
        if (i < bv.count) {
            const uint64_t n = bv.first + i;
            Cols gc;
            gc.b = &bv; gc.n = n;
            bool d;
            if constexpr (Meta::kMeta) {
                if (kStaged || pk) { cb::UcRowsPacked rows; rows.pk = pk; rows.by_slot = true; d = cb::eval_request_uc_meta(tv, bv, gc, rows, meta.side, n, effects, meta.action_meta, meta.req_meta, Conds()); }
                else { cb::UcRowsGlobal rows; rows.urows = tv.urows(); rows.row_am = bv.row_am; rows.RCP = bv.rcp; rows.nR = td.lay.nR; d = cb::eval_request_uc_meta(tv, bv, gc, rows, meta.side, n, effects, meta.action_meta, meta.req_meta, Conds()); }
            } else {
                if (kStaged || pk) { cb::UcRowsPacked rows; rows.pk = pk; rows.by_slot = true; d = cb::eval_request_uc(tv, bv, gc, rows, n, bitmap, effects, Conds()); }
                else { cb::UcRowsGlobal rows; rows.urows = tv.urows(); rows.row_am = bv.row_am; rows.RCP = bv.rcp; rows.nR = td.lay.nR; d = cb::eval_request_uc(tv, bv, gc, rows, n, bitmap, effects, Conds()); }
            }
            if (d) {
                cb::store_result(bv, gc, n, bitmap, effects, bv.max_actions, 0u);
                const uint32_t k = atomicAdd(bv.defer_count, 1u);
                bv.defer_list[k] = (uint32_t)i;
            }
        }
#ifndef CB_UC_NO_LIST_PF   // tools/uc_variants.sh: without the list-header prefetch
        if constexpr (Conds::kListSlots > 0) {
            // this warp's next chunk: pull the headers of its register-resident lists towards L2 (cb::list_header_pf).
            // Here, after the walk, the next chunk's slot words are L2 hits (prefetched above, one chunk ago) and hold
            // no register during the term evaluation.  Prefetches never fault and change no value.
            const uint64_t i2 = (chunk + n_warps) * 32 + lane;
            if (i2 < bv.count) {
#pragma unroll
                for (uint32_t s = 0; s < Conds::kListSlots; s++)
                    if (const uint64_t *p = cb::list_header_pf(bv, cb::ldcol64(bv.slots + (uint64_t)Conds::kListSlot[s] * bv.stride + bv.first + i2)))
                        asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
            }
        }
#endif
    }
}

}  // namespace cbk
