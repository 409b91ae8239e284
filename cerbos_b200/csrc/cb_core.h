// cb_core.h -- per-request evaluation core of the H100 CheckResources kernels.
//
// One thread evaluates one request (principal, resource, K actions) against the flattened rule table:
//   * scope chains + existence checks      (reference: ruletable.go:611-645, 804-863; index.go:1089-1172)
//   * ONE pass over the rows of every policy block on the chain; every satisfied row contributes a
//     bit pattern (action x role-column) so the reference's per-action / per-role walk
//     (ruletable.go:885-1152) becomes a handful of 64-bit mask operations ("bit-parallel walk"):
//         within a scope   DENY beats ALLOW                         (:1083-1091)
//         OVERRIDE_PARENT  satisfied ALLOW finishes the (action, role) pair     (:1115-1118)
//         REQUIRE_PARENTAL_CONSENT  ALLOW is dropped, walk continues   (:1113-1114)
//         an action is ALLOWed iff the principal-policy walk allows it, or it is undecided there
//         and some role's resource-policy walk allows it            (:1124-1148)
//   * role-policy DENY synthesis             (index.go:688-776)
//   * CEL conditions by a stack bytecode interpreter with cel-go error semantics
//     (bytecode produced by cerbos_b200/table/bytecode.py; leaf rule ruletable.go:1425-1441)
//
// The file is plain C++ guarded by CB_HD so that tests/hostsim can compile the very same code for the
// host and step through it without a GPU (debug aid only -- the product never runs it on the CPU).
#pragma once
#include <stdint.h>
#if !defined(__CUDACC_RTC__)
#include <math.h>      // (ceil / floor / round / trunc / fabs / sqrt of ext.Math; built in under NVRTC)
#endif

#include "cerbos_b200_format.h"

#if defined(__CUDACC__)
#define CB_HD __host__ __device__ __forceinline__
#define CB_HD_NOINLINE __host__ __device__ __noinline__
#else
#define CB_HD inline
#define CB_HD_NOINLINE
#endif

namespace cb {

struct alignas(16) U4 { uint32_t x, y, z, w; };

// ---------------------------------------------------------------------------------------------- views
// Section offsets + dimensions of the table image.  In the kernels this lives in the (grid-constant) kernel
// parameters, so reading a field is a constant-bank operand and costs no register.
struct TableLayout {
    uint32_t off[32];   // by section id (CB_SEC_*)
    uint32_t nV, nRP, nS, nP, nR, nAP, nT, n_slots, n_rows;
    uint32_t has_role_policies, has_parent_roles, has_principal_policies;
    uint32_t image_bytes;
    // "unique condition" image (cb_uc.h): offsets of the three derived sections, number of distinct conditions (0 = none)
    uint32_t uc_conds_off, uc_rows_off, uc_chain_off, n_uconds;
    uint32_t theap_words;   // 8-byte words in THEAP
    uint32_t uses_runtime;  // a condition reads runtime.effectiveDerivedRoles
};

// base = start of the table image: shared memory (TMA-staged) or global memory.
struct TableView {
    const uint8_t *base;
    const TableLayout *L;
    template <typename T>
    CB_HD const T *sec(int id) const { return reinterpret_cast<const T *>(base + L->off[id]); }
    CB_HD const uint32_t *scope_parent() const { return sec<uint32_t>(CB_SEC_SCOPE_PARENT); }
    CB_HD const uint32_t *scope_flags() const { return sec<uint32_t>(CB_SEC_SCOPE_FLAGS); }
    CB_HD const uint32_t *res_block_map() const { return sec<uint32_t>(CB_SEC_RES_BLOCK_MAP); }
    CB_HD const uint8_t *res_exists() const { return sec<uint8_t>(CB_SEC_RES_EXISTS); }
    CB_HD const uint32_t *prin_block_map() const { return sec<uint32_t>(CB_SEC_PRIN_BLOCK_MAP); }
    CB_HD const uint8_t *prin_exists() const { return sec<uint8_t>(CB_SEC_PRIN_EXISTS); }
    CB_HD const uint32_t *prin_of_string() const { return sec<uint32_t>(CB_SEC_PRIN_OF_STRING); }
    CB_HD const cb_block *blocks() const { return sec<cb_block>(CB_SEC_BLOCKS); }
    CB_HD const cb_row *rows() const { return sec<cb_row>(CB_SEC_ROWS); }
    CB_HD const cb_cond *conds() const { return sec<cb_cond>(CB_SEC_CONDS); }
    CB_HD const cb_instr *code() const { return sec<cb_instr>(CB_SEC_CODE); }
    CB_HD const cb_const *consts() const { return sec<cb_const>(CB_SEC_CONSTS); }
    CB_HD const uint64_t *consts_v64() const { return sec<uint64_t>(CB_SEC_CONSTS_V64); }
    CB_HD const uint64_t *theap() const { return sec<uint64_t>(CB_SEC_THEAP); }
    CB_HD const uint32_t *str_off() const { return sec<uint32_t>(CB_SEC_STR_OFF); }
    CB_HD const uint8_t *str_bytes() const { return sec<uint8_t>(CB_SEC_STR_BYTES); }
    CB_HD const uint32_t *par_off() const { return sec<uint32_t>(CB_SEC_ROLE_PARENTS_OFF); }
    CB_HD const uint32_t *par_list() const { return sec<uint32_t>(CB_SEC_ROLE_PARENTS); }
    CB_HD const uint32_t *rp_off() const { return sec<uint32_t>(CB_SEC_ROLEPOL_OFF); }
    CB_HD const cb_rolepol_entry *rp_entries() const { return sec<cb_rolepol_entry>(CB_SEC_ROLEPOL_ENTRIES); }
    CB_HD const cb_rolepol_rule *rp_rules() const { return sec<cb_rolepol_rule>(CB_SEC_ROLEPOL_RULES); }
    CB_HD const uint32_t *rp_apats() const { return sec<uint32_t>(CB_SEC_ROLEPOL_APATS); }
    CB_HD const uint32_t *block_slots_off() const { return sec<uint32_t>(CB_SEC_BLOCK_SLOTS_OFF); }
    CB_HD const uint32_t *block_slots() const { return sec<uint32_t>(CB_SEC_BLOCK_SLOTS); }
    CB_HD const uint32_t *dr_off() const { return sec<uint32_t>(CB_SEC_DR_OFF); }
    CB_HD const uint32_t *dr_entries() const { return sec<uint32_t>(CB_SEC_DR_ENTRIES); }   // 4 words each
    CB_HD const uint32_t *dr_parents() const { return sec<uint32_t>(CB_SEC_DR_PARENTS); }
    CB_HD const uint32_t *dr_name_str() const { return sec<uint32_t>(CB_SEC_DR_NAME_STR); }
    CB_HD const cb_cond *uconds() const { return reinterpret_cast<const cb_cond *>(base + L->uc_conds_off); }     // [n_uconds + 1], entry 0 unused
    CB_HD const U4 *urows() const { return reinterpret_cast<const U4 *>(base + L->uc_rows_off); }                 // [n_rows] 16-byte rows, DENY first per block
    CB_HD const U4 *uc_chain() const { return reinterpret_cast<const U4 *>(base + L->uc_chain_off); }             // like RES_BLOCK_MAP: one scope-walk step each
};

enum { CB_MAX_GATHER = 8 };
struct BatchView {
    const cb_hdr0 *hdr0;
    const cb_hdr1 *hdr1;
    const uint32_t *roles;      // [role_cols][stride]
    const uint64_t *slots;      // [n_slots][stride]
    const uint64_t *heap;
    const uint32_t *bstr_off;
    const uint8_t *bstr_bytes;
    const uint32_t *class_off, *class_pats, *aset_k;
    const uint64_t *aset_spread;  // [n_pass][n_asets][nAP]
    const uint64_t *row_am;       // [n_pass][n_asets][n_rows]
    uint32_t n_rows;
    uint64_t stride;            // requests per column (N of the whole batch)
    uint64_t first, count;      // sub-range evaluated by this launch
    uint32_t role_cols, n_asets, kc, n_pass, max_actions, kbytes, flags;
    uint32_t rcp, stride_pattern;   // set by finish_batch_view(): pow2 >= role_cols; bit j*role_cols for every j (32-bit)
    int64_t now;
    const uint32_t *perm;       // clustered evaluation order (request offsets from `first`), or null = index order
    uint32_t prefetch_slots;    // > 0: the table reads this many slot columns in all (few): prefetch every one per tile
    uint32_t *defer_list, *defer_count;   // run-time specialised lean kernels: requests left to the general kernel
    uint32_t *count_dev;                  // general kernel draining such a list: {length, CTAs done, tile counter} in device memory, else null
    uint32_t *tile_counter;               // tile kernel: tiles beyond each CTA's first are claimed from this counter (null: static stride)
    // fused all-gather: n_out > 0 = write every result to this rank's slice of n_out gather buffers (own + peers over
    // NVLink, peer-mapped pointers already offset to the slice) instead of `bitmap`
    uint8_t *outs[CB_MAX_GATHER];
    uint32_t n_out;
    // ... and, in the general kernel draining a specialised kernel's deferral list (always the last kernel of such a
    // launch): release `sig_step` into cell sig_rank of every rank's flag array once all results are stored, and
    // first wait until every rank's `wait_step` has arrived in the local flags (0 = no wait)
    uint32_t *sig_flags[CB_MAX_GATHER];
    const uint32_t *wait_flags;
    uint32_t sig_rank, sig_step, wait_step;
    // run-time specialised unique-condition kernels: one word per string id (table strings, then batch strings) holding
    // the outcome of every `attribute.startsWith / endsWith / contains(constant)` predicate of the table, computed once
    // per distinct string by a pre-pass over the batch's string dictionary (null: none)
    const uint32_t *strpred;
    // ... launched with the table image in global memory: the image's rows merged with this batch's row x action-set
    // masks (cb::uc_row_record), one 16-byte record per (action set, row), built by a pre-pass (null: merge on the fly)
    const U4 *uc_rows_pk;
    uint32_t n_bstr;            // strings in the batch dictionary
    uint64_t heap_words;        // 8-byte words in `heap`
};

// Table data may live in shared memory (TMA-staged image) or in global memory, heap references may point
// into either the table or the batch: those loads are plain (generic) loads.  Only the big streaming request
// columns -- read exactly once -- use the read-only, no-L1-allocate path so they do not evict the table.
// derived BatchView fields (host side, once per launch)
#ifndef __CUDACC_RTC__
inline void finish_batch_view(BatchView &b) {
    b.perm = nullptr;
    b.prefetch_slots = 0;
    b.defer_list = nullptr; b.defer_count = nullptr; b.count_dev = nullptr; b.tile_counter = nullptr;
    b.n_out = 0;
    for (int i = 0; i < CB_MAX_GATHER; i++) { b.outs[i] = nullptr; b.sig_flags[i] = nullptr; }
    b.wait_flags = nullptr; b.sig_rank = 0; b.sig_step = 0; b.wait_step = 0;
    b.strpred = nullptr;
    b.uc_rows_pk = nullptr;
    b.rcp = 1;
    while (b.rcp < b.role_cols) b.rcp <<= 1;
    b.stride_pattern = 0;
    for (uint32_t j = 0; j * b.role_cols < 32; j++) b.stride_pattern |= 1u << (j * b.role_cols);
}
#endif

template <typename T>
CB_HD T ldg(const T *p) { return *p; }

CB_HD uint64_t ldcol64(const uint64_t *p) {
#if defined(__CUDA_ARCH__)
    uint64_t v;
    asm("ld.global.nc.L1::no_allocate.u64 %0, [%1];" : "=l"(v) : "l"(p));
    return v;
#else
    return *p;
#endif
}
CB_HD uint32_t ldcol32(const uint32_t *p) {
#if defined(__CUDA_ARCH__)
    uint32_t v;
    asm("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
#else
    return *p;
#endif
}

// 128-bit loads of the 16-byte records (their C structs are only 4-byte aligned, the buffers are 16-byte aligned)
CB_HD U4 ld16(const void *p) { return *reinterpret_cast<const U4 *>(p); }
CB_HD U4 ldcol128(const void *p) {
#if defined(__CUDA_ARCH__)
    U4 r;
    asm("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
#else
    return *reinterpret_cast<const U4 *>(p);
#endif
}
CB_HD cb_hdr0 load_hdr0(const cb_hdr0 *p) { U4 v = ldcol128(p); cb_hdr0 h; h.principal_id = v.x; h.kind_class = v.y; h.resource_scope = v.z; h.principal_scope = v.w; return h; }
CB_HD cb_hdr1 load_hdr1(const cb_hdr1 *p) {
    uint64_t v = ldcol64(reinterpret_cast<const uint64_t *>(p));
    cb_hdr1 h; h.resource_version = (uint16_t)(v & 0xFFFF); h.principal_version = (uint16_t)((v >> 16) & 0xFFFF); h.action_set_id = (uint32_t)(v >> 32); return h;
}
CB_HD cb_block load_block(const cb_block *p) { U4 v = ld16(p); cb_block b; b.row_start = v.x; b.n_rows = v.y; b.cond_base = v.z; b.n_conds = v.w; return b; }
CB_HD cb_row load_row(const cb_row *p) {
    U4 v = ld16(p);
    cb_row r; r.role = (uint16_t)(v.x & 0xFFFF); r.cond = (uint16_t)(v.x >> 16); r.drcond = (uint16_t)(v.y & 0xFFFF); r.respat = (uint16_t)(v.y >> 16);
    r.effect = (uint8_t)(v.z & 0xFF); r.flags = (uint8_t)((v.z >> 8) & 0xFF); r.n_pats = (uint16_t)(v.z >> 16); r.pat_start = v.w; return r;
}
CB_HD cb_rolepol_entry load_rp_entry(const cb_rolepol_entry *p) { U4 v = ld16(p); cb_rolepol_entry e; e.role = v.x; e.rule_start = v.y; e.n_rules = v.z; e.pad = v.w; return e; }
CB_HD cb_rolepol_rule load_rp_rule(const cb_rolepol_rule *p) { U4 v = ld16(p); cb_rolepol_rule e; e.respat = v.x; e.cond = v.y; e.apat_start = v.z; e.n_apats = v.w; return e; }

CB_HD double u2d(uint64_t u) {
#if defined(__CUDA_ARCH__)
    return __longlong_as_double((long long)u);
#else
    double d; __builtin_memcpy(&d, &u, 8); return d;
#endif
}
CB_HD uint64_t d2u(double d) {
#if defined(__CUDA_ARCH__)
    return (uint64_t)__double_as_longlong(d);
#else
    uint64_t u; __builtin_memcpy(&u, &d, 8); return u;
#endif
}

// generic values + the helpers behind every bytecode instruction: not part of the lean-only (run-time specialised) build
// unless the table's specialised code contains leaf programs (cb_specialize.h: CB_SPEC_PROGRAMS)
#if !defined(CB_LEAN_ONLY) || defined(CB_SPEC_PROGRAMS)
// ---------------------------------------------------------------------------------------------- values
struct Val {
    uint32_t tag;
    uint64_t u;
};
static constexpr uint64_t kHeapBatch = 1ull << 63;
// Values made at run time (list / string producing functions, comprehensions that build lists or maps, concatenation)
// live in a small per-thread scratch arena inside Ctx: lists / maps as [n, elements...] words exactly like the heaps,
// strings as raw bytes.  A program that outgrows it raises the sticky `unsupported` flag (the call fails loudly).
static constexpr uint64_t kHeapScratch = 1ull << 62;          // Val.u of a LIST / MAP: word offset into Ctx::scratch
static constexpr uint64_t kStrDyn = 1ull << 47;               // Val.u / V64 payload of a STRING: byte offset << 16 | byte length
static constexpr uint64_t kV64ScratchBit = 1ull << 46;        // V64 payload of a LIST / MAP element living in the arena
enum { CB_SCRATCH_WORDS = 192, CB_T_SKIP = 15 };              // CB_T_SKIP: comprehension iteration filtered out (internal)

CB_HD Val mk(uint32_t tag, uint64_t u) { Val v; v.tag = tag; v.u = u; return v; }
CB_HD Val mk_err() { return mk(CB_T_ERR, 0); }
CB_HD Val mk_bool(bool b) { return mk(CB_T_BOOL, b ? 1u : 0u); }
CB_HD Val mk_int(int64_t i) { return mk(CB_T_INT, (uint64_t)i); }
CB_HD Val mk_double(double d) { return mk(CB_T_DOUBLE, d != d ? (uint64_t)CB_V64_CANON_NAN : d2u(d)); }

enum { SLOT_VALUE = 0, SLOT_ABSENT = 1, SLOT_ERROR = 2 };

CB_HD Val decode_v64(uint64_t bits, int *state) {
    // branch-free: lanes of a warp hold values of different classes (a switch here was an indirect branch per decode)
    const uint32_t top = (uint32_t)(bits >> 48);
    const bool boxed = (top & 0xFFF0u) == 0xFFF0u && (top & 0xFu) != 0;
    const uint32_t vt = top & 0xFu;
    const uint64_t pay = bits & 0xFFFFFFFFFFFFull;
    // value class by box tag: NULL 1 -> NULL, BOOL 2 -> BOOL, STRING 3 -> STRING, LIST 4 -> LIST, MAP 5 -> MAP, INT 8 -> INT, the rest -> ERR
    const uint64_t kTagOf = (uint64_t)CB_T_NULL << 4 | (uint64_t)CB_T_BOOL << 8 | (uint64_t)CB_T_STRING << 12 | (uint64_t)CB_T_LIST << 16 |
                            (uint64_t)CB_T_MAP << 20 | (uint64_t)CB_T_INT << 32;
    const uint32_t tag = boxed ? (uint32_t)(kTagOf >> (4 * vt)) & 0xFu : (uint32_t)CB_T_DOUBLE;
    uint64_t off = pay & (CB_V64_HEAP_BATCH_BIT - 1);
    off = (pay & CB_V64_HEAP_BATCH_BIT) ? off | kHeapBatch : (off & kV64ScratchBit) ? (off & ~kV64ScratchBit) | kHeapScratch : off;
    const uint64_t u = !boxed                                  ? bits
                       : vt == CB_V64_BOOL                     ? (uint64_t)(pay != 0)
                       : vt == CB_V64_STRING                   ? pay
                       : (vt == CB_V64_LIST || vt == CB_V64_MAP) ? off
                       : vt == CB_V64_INT                      ? (uint64_t)((int64_t)(pay << 16) >> 16)
                                                               : 0ull;
    *state = !boxed || tag != CB_T_ERR ? SLOT_VALUE : vt == CB_V64_ABSENT ? SLOT_ABSENT : SLOT_ERROR;
    return mk(tag, u);
}
CB_HD Val decode_elem(uint64_t bits) { int s; return decode_v64(bits, &s); }

struct Ctx {
    const TableView *t;
    const BatchView *b;
    uint64_t req;          // absolute request index (column index)
    uint32_t pid;          // hdr0.principal_id
    uint32_t unsupported;  // sticky
    Val vars[CB_MAX_VARS];
    uint64_t edr;          // runtime.effectiveDerivedRoles of the policy being evaluated: bit set over MANIFEST.derived_roles
    uint32_t scr_used;     // words of `scratch` in use
    uint64_t scratch[CB_SCRATCH_WORDS];
};

CB_HD const uint64_t *heap_ptr(const Ctx &c, uint64_t ref) {
    return (ref & kHeapBatch) ? c.b->heap + (ref & ~kHeapBatch) : (ref & kHeapScratch) ? c.scratch + (ref & 0xFFFFu) : c.t->theap() + ref;
}
CB_HD void str_get(const Ctx &c, uint64_t id, const uint8_t *&p, uint32_t &len) {
    if (id & kStrDyn) {
        p = reinterpret_cast<const uint8_t *>(c.scratch) + ((id >> 16) & 0xFFFFu);
        len = (uint32_t)(id & 0xFFFFu);
    } else if (id < c.t->L->nT) {
        uint32_t o = ldg(c.t->str_off() + id);
        p = c.t->str_bytes() + o;
        len = ldg(c.t->str_off() + id + 1) - o;
    } else {
        uint64_t j = id - c.t->L->nT;
        uint32_t o = ldg(c.b->bstr_off + j);
        p = c.b->bstr_bytes + o;
        len = ldg(c.b->bstr_off + j + 1) - o;
    }
}

CB_HD bool is_num(const Val &v) { return v.tag == CB_T_INT || v.tag == CB_T_UINT || v.tag == CB_T_DOUBLE; }

// cel-go cross-type numeric comparison (types/compare.go): -1/0/1, 2 = unordered (NaN)
CB_HD int num_cmp(const Val &a, const Val &b) {
    if (a.tag == CB_T_DOUBLE || b.tag == CB_T_DOUBLE) {
        if (a.tag == CB_T_DOUBLE && b.tag == CB_T_DOUBLE) {
            double x = u2d(a.u), y = u2d(b.u);
            if (x != x || y != y) return 2;
            return x < y ? -1 : (x > y ? 1 : 0);
        }
        int sign = 1;
        Val dv = a, iv = b;
        if (a.tag != CB_T_DOUBLE) { dv = b; iv = a; sign = -1; }
        double d = u2d(dv.u);
        if (d != d) return 2;
        int r;
        if (iv.tag == CB_T_UINT) {
            if (d < 0) r = -1;
            else if (d > 18446744073709551615.0) r = 1;
            else { double y = (double)iv.u; r = d < y ? -1 : (d > y ? 1 : 0); }
        } else {
            if (d < -9223372036854775808.0) r = -1;
            else if (d > 9223372036854775807.0) r = 1;
            else { double y = (double)(int64_t)iv.u; r = d < y ? -1 : (d > y ? 1 : 0); }
        }
        return r * sign;
    }
    if (a.tag == b.tag) {
        if (a.tag == CB_T_INT) { int64_t x = (int64_t)a.u, y = (int64_t)b.u; return x < y ? -1 : (x > y ? 1 : 0); }
        return a.u < b.u ? -1 : (a.u > b.u ? 1 : 0);
    }
    if (a.tag == CB_T_INT) {
        int64_t x = (int64_t)a.u;
        if (x < 0) return -1;
        return (uint64_t)x < b.u ? -1 : ((uint64_t)x > b.u ? 1 : 0);
    }
    int64_t y = (int64_t)b.u;
    if (y < 0) return 1;
    return a.u < (uint64_t)y ? -1 : (a.u > (uint64_t)y ? 1 : 0);
}

// strings: interned ids are unique per string; one made at run time is compared by its bytes
CB_HD bool str_equal(const Ctx &c, uint64_t a, uint64_t b) {
    if (a == b) return true;
    if (!((a | b) & kStrDyn)) return false;
    const uint8_t *pa, *pb;
    uint32_t la, lb;
    str_get(c, a, pa, la);
    str_get(c, b, pb, lb);
    if (la != lb) return false;
    for (uint32_t i = 0; i < la; i++)
        if (ldg(pa + i) != ldg(pb + i)) return false;
    return true;
}
// scalar (non-container) equality; containers handled by the callers below
CB_HD bool scalar_equal(const Ctx &c, const Val &a, const Val &b) {
    if (is_num(a) && is_num(b)) return num_cmp(a, b) == 0;
    if (a.tag != b.tag) return false;
    if (a.tag == CB_T_NULL) return true;
    if (a.tag == CB_T_STRING || a.tag == CB_T_BYTES) return str_equal(c, a.u, b.u);
    return a.u == b.u;  // BOOL / TS / DUR / TYPE
}
CB_HD bool is_container(const Val &v) { return v.tag == CB_T_LIST || v.tag == CB_T_MAP; }

CB_HD bool map_find(const Ctx &c, const Val &m, const Val &key, Val *out) {
    if (is_container(key) || key.tag == CB_T_ERR) return false;   // keys are scalars: string (JSON), int / uint / bool (literals, comprehensions)
    const uint64_t *p = heap_ptr(c, m.u);
    uint64_t n = ldg(p);
    for (uint64_t i = 0; i < n; i++) {
        Val k = decode_elem(ldg(p + 1 + i));
        if (scalar_equal(c, k, key)) {
            if (out) *out = decode_elem(ldg(p + 1 + n + i));
            return true;
        }
    }
    return false;
}

// Heterogeneous equality (cel-go types.Equal).  Containers are compared to a nesting depth of 3;
// deeper structures raise the sticky `unsupported` flag (the call then fails loudly).
template <int DEPTH>
struct Eq {
    static CB_HD bool eq(Ctx &c, const Val &a, const Val &b) {
        if (!is_container(a) || !is_container(b)) {
            if (is_container(a) != is_container(b)) return false;
            return scalar_equal(c, a, b);
        }
        if (a.tag != b.tag) return false;
        const uint64_t *pa = heap_ptr(c, a.u), *pb = heap_ptr(c, b.u);
        uint64_t n = ldg(pa);
        if (n != ldg(pb)) return false;
        if (a.tag == CB_T_LIST) {
            for (uint64_t i = 0; i < n; i++)
                if (!Eq<DEPTH - 1>::eq(c, decode_elem(ldg(pa + 1 + i)), decode_elem(ldg(pb + 1 + i)))) return false;
            return true;
        }
        for (uint64_t i = 0; i < n; i++) {
            Val ov;
            if (!map_find(c, b, decode_elem(ldg(pa + 1 + i)), &ov)) return false;
            if (!Eq<DEPTH - 1>::eq(c, decode_elem(ldg(pa + 1 + n + i)), ov)) return false;
        }
        return true;
    }
};
template <>
struct Eq<0> {
    static CB_HD bool eq(Ctx &c, const Val &a, const Val &b) {
        if (is_container(a) && is_container(b)) { c.unsupported = 1; return false; }
        if (is_container(a) != is_container(b)) return false;
        return scalar_equal(c, a, b);
    }
};
// Container equality stays out of line: inlined into every compare of a generated leaf program (cb_specialize.h) the
// nested loops made NVRTC spend ~2 s per call site; scalars -- nearly every compare -- take the short inline path.
CB_HD_NOINLINE bool container_equal(Ctx &c, const Val &a, const Val &b) { return Eq<3>::eq(c, a, b); }
CB_HD bool val_equal(Ctx &c, const Val &a, const Val &b) {
    if (!is_container(a) || !is_container(b)) { if (is_container(a) != is_container(b)) return false; return scalar_equal(c, a, b); }
    return container_equal(c, a, b);
}

CB_HD int str_cmp(const Ctx &c, uint64_t ia, uint64_t ib) {
    const uint8_t *pa, *pb;
    uint32_t la, lb;
    str_get(c, ia, pa, la);
    str_get(c, ib, pb, lb);
    uint32_t m = la < lb ? la : lb;
    for (uint32_t i = 0; i < m; i++) {
        uint8_t x = ldg(pa + i), y = ldg(pb + i);
        if (x != y) return x < y ? -1 : 1;
    }
    return la < lb ? -1 : (la > lb ? 1 : 0);
}

// -1/0/1, 3 = error (no such overload / NaN)
CB_HD int val_order(const Ctx &c, const Val &a, const Val &b) {
    if (is_num(a) && is_num(b)) { int r = num_cmp(a, b); return r == 2 ? 3 : r; }
    if (a.tag != b.tag) return 3;
    switch (a.tag) {
    case CB_T_BOOL: return a.u < b.u ? -1 : (a.u > b.u ? 1 : 0);
    case CB_T_STRING: return a.u == b.u ? 0 : str_cmp(c, a.u, b.u);
    case CB_T_TS:
    case CB_T_DUR: { int64_t x = (int64_t)a.u, y = (int64_t)b.u; return x < y ? -1 : (x > y ? 1 : 0); }
    default: return 3;
    }
}

CB_HD_NOINLINE int spiffe_equal(Ctx &c, const Val &a, const Val &b);   // with the SPIFFE functions below
CB_HD Val do_cmp(Ctx &c, int ci, const Val &a, const Val &b) {
    if (a.tag == CB_T_ERR || b.tag == CB_T_ERR) return mk_err();
    if (ci <= 1 && (a.tag == CB_T_SPIFFE_ID || a.tag == CB_T_SPIFFE_TD)) {   // the left operand's Equal decides (spiffe.go)
        const int r = spiffe_equal(c, a, b);
        return r == 2 ? mk_err() : mk_bool((r == 1) == (ci == 0));
    }
    if (ci == 0) return mk_bool(val_equal(c, a, b));
    if (ci == 1) return mk_bool(!val_equal(c, a, b));
    int r = val_order(c, a, b);
    if (r == 3) return mk_err();
    switch (ci) {
    case 2: return mk_bool(r < 0);
    case 3: return mk_bool(r <= 0);
    case 4: return mk_bool(r > 0);
    default: return mk_bool(r >= 0);
    }
}

CB_HD Val do_in(Ctx &c, const Val &x, const Val &cont) {
    if (x.tag == CB_T_ERR || cont.tag == CB_T_ERR) return mk_err();
    if (cont.tag == CB_T_LIST) {
        const uint64_t *p = heap_ptr(c, cont.u);
        uint64_t n = ldg(p);
        for (uint64_t i = 0; i < n; i++)
            if (val_equal(c, x, decode_elem(ldg(p + 1 + i)))) return mk_bool(true);
        return mk_bool(false);
    }
    if (cont.tag == CB_T_MAP) return mk_bool(map_find(c, cont, x, nullptr));
    return mk_err();
}

CB_HD Val do_index(Ctx &c, const Val &cont, const Val &key) {
    if (cont.tag == CB_T_ERR || key.tag == CB_T_ERR) return mk_err();
    if (cont.tag == CB_T_LIST) {
        int64_t idx;
        if (key.tag == CB_T_INT) idx = (int64_t)key.u;
        else if (key.tag == CB_T_UINT) { if (key.u > 0x7FFFFFFFFFFFFFFFull) return mk_err(); idx = (int64_t)key.u; }
        else if (key.tag == CB_T_DOUBLE) {
            double d = u2d(key.u);
            if (!(d == (double)(int64_t)d) || !(d > -9.2e18 && d < 9.2e18)) return mk_err();
            idx = (int64_t)d;
        } else return mk_err();
        const uint64_t *p = heap_ptr(c, cont.u);
        if (idx < 0 || (uint64_t)idx >= ldg(p)) return mk_err();
        return decode_elem(ldg(p + 1 + idx));
    }
    if (cont.tag == CB_T_MAP) { Val out; return map_find(c, cont, key, &out) ? out : mk_err(); }
    return mk_err();
}

// ---- Cerbos set functions (cerbos_lib.go:323-431).  When the larger list has > 3 elements that are all
// hashable the reference probes a Go map keyed by ref.Val: identity is (dynamic type, value), i.e. no
// cross-type numeric equality; otherwise it scans with Equal. ----
CB_HD bool hashable(const Val &v) {
    return v.tag == CB_T_STRING || v.tag == CB_T_INT || v.tag == CB_T_UINT || v.tag == CB_T_DOUBLE || v.tag == CB_T_DUR || v.tag == CB_T_TS;
}
CB_HD bool uses_go_map(const Ctx &c, const Val &b) {
    const uint64_t *p = heap_ptr(c, b.u);
    uint64_t n = ldg(p);
    if (n <= 3) return false;
    for (uint64_t i = 0; i < n; i++)
        if (!hashable(decode_elem(ldg(p + 1 + i)))) return false;
    return true;
}
CB_HD bool key_identical(const Ctx &c, const Val &a, const Val &b) {
    if (a.tag != b.tag) return false;
    if (a.tag == CB_T_DOUBLE) return u2d(a.u) == u2d(b.u);
    if (a.tag == CB_T_STRING) return str_equal(c, a.u, b.u);
    return a.u == b.u;
}
CB_HD bool list_member(Ctx &c, bool go_map, const Val &b, const Val &x) {
    const uint64_t *p = heap_ptr(c, b.u);
    uint64_t n = ldg(p);
    for (uint64_t i = 0; i < n; i++) {
        Val e = decode_elem(ldg(p + 1 + i));
        if (go_map ? key_identical(c, x, e) : val_equal(c, x, e)) return true;
    }
    return false;
}
CB_HD Val do_set_pred(Ctx &c, bool subset, Val a, Val b) {
    if (a.tag != CB_T_LIST || b.tag != CB_T_LIST) return mk_err();
    if (!subset && ldg(heap_ptr(c, a.u)) > ldg(heap_ptr(c, b.u))) { Val t = a; a = b; b = t; }
    bool gm = uses_go_map(c, b);
    const uint64_t *p = heap_ptr(c, a.u);
    uint64_t n = ldg(p);
    for (uint64_t i = 0; i < n; i++) {
        bool m = list_member(c, gm, b, decode_elem(ldg(p + 1 + i)));
        if (subset && !m) return mk_bool(false);
        if (!subset && m) return mk_bool(true);
    }
    return mk_bool(subset);
}

// ---- arithmetic with cel-go overflow rules ----
#if defined(__CUDA_ARCH__)
CB_HD bool add_ovf(int64_t x, int64_t y, int64_t *r) { int64_t s = (int64_t)((uint64_t)x + (uint64_t)y); *r = s; return ((x ^ s) & (y ^ s)) < 0; }
CB_HD bool sub_ovf(int64_t x, int64_t y, int64_t *r) { int64_t s = (int64_t)((uint64_t)x - (uint64_t)y); *r = s; return ((x ^ y) & (x ^ s)) < 0; }
CB_HD bool mul_ovf(int64_t x, int64_t y, int64_t *r) {
    int64_t lo = (int64_t)((uint64_t)x * (uint64_t)y);
    int64_t hi = __mul64hi(x, y);
    *r = lo;
    return hi != (lo >> 63);
}
CB_HD bool umul_ovf(uint64_t x, uint64_t y, uint64_t *r) { *r = x * y; return __umul64hi(x, y) != 0; }
#else
CB_HD bool add_ovf(int64_t x, int64_t y, int64_t *r) { return __builtin_add_overflow(x, y, r); }
CB_HD bool sub_ovf(int64_t x, int64_t y, int64_t *r) { return __builtin_sub_overflow(x, y, r); }
CB_HD bool mul_ovf(int64_t x, int64_t y, int64_t *r) { return __builtin_mul_overflow(x, y, r); }
CB_HD bool umul_ovf(uint64_t x, uint64_t y, uint64_t *r) { return __builtin_mul_overflow(x, y, r); }
#endif

CB_HD_NOINLINE Val dyn_concat(Ctx &c, const Val &a, const Val &b);   // defined with the run-time values below
CB_HD Val do_arith(Ctx &c, int op, const Val &a, const Val &b) {
    if (a.tag == CB_T_ERR || b.tag == CB_T_ERR) return mk_err();
    const int64_t kMin = (int64_t)0x8000000000000000ull;
    if (a.tag == CB_T_INT && b.tag == CB_T_INT) {
        int64_t x = (int64_t)a.u, y = (int64_t)b.u, r;
        switch (op) {
        case CB_OP_ADD: return add_ovf(x, y, &r) ? mk_err() : mk_int(r);
        case CB_OP_SUB: return sub_ovf(x, y, &r) ? mk_err() : mk_int(r);
        case CB_OP_MUL: return mul_ovf(x, y, &r) ? mk_err() : mk_int(r);
        case CB_OP_DIV: return (y == 0 || (x == kMin && y == -1)) ? mk_err() : mk_int(x / y);
        default: return (y == 0 || (x == kMin && y == -1)) ? mk_err() : mk_int(x % y);
        }
    }
    if (a.tag == CB_T_UINT && b.tag == CB_T_UINT) {
        uint64_t x = a.u, y = b.u, r;
        switch (op) {
        case CB_OP_ADD: r = x + y; return r < x ? mk_err() : mk(CB_T_UINT, r);
        case CB_OP_SUB: return y > x ? mk_err() : mk(CB_T_UINT, x - y);
        case CB_OP_MUL: return umul_ovf(x, y, &r) ? mk_err() : mk(CB_T_UINT, r);
        case CB_OP_DIV: return y == 0 ? mk_err() : mk(CB_T_UINT, x / y);
        default: return y == 0 ? mk_err() : mk(CB_T_UINT, x % y);
        }
    }
    if (a.tag == CB_T_DOUBLE && b.tag == CB_T_DOUBLE) {
        double x = u2d(a.u), y = u2d(b.u);
        switch (op) {
        case CB_OP_ADD: return mk_double(x + y);
        case CB_OP_SUB: return mk_double(x - y);
        case CB_OP_MUL: return mk_double(x * y);
        case CB_OP_DIV: return mk_double(x / y);
        default: return mk_err();
        }
    }
    int64_t x = (int64_t)a.u, y = (int64_t)b.u, r;
    if (op == CB_OP_ADD) {
        if ((a.tag == CB_T_TS && b.tag == CB_T_DUR) || (a.tag == CB_T_DUR && b.tag == CB_T_TS)) {
            if (add_ovf(x, y, &r)) { c.unsupported = 1; return mk_err(); }
            return mk(CB_T_TS, (uint64_t)r);
        }
        if (a.tag == CB_T_DUR && b.tag == CB_T_DUR) return add_ovf(x, y, &r) ? mk_err() : mk(CB_T_DUR, (uint64_t)r);
        if ((a.tag == CB_T_STRING && b.tag == CB_T_STRING) || (a.tag == CB_T_LIST && b.tag == CB_T_LIST)) return dyn_concat(c, a, b);
    }
    if (op == CB_OP_SUB) {
        if (a.tag == CB_T_TS && b.tag == CB_T_TS) return sub_ovf(x, y, &r) ? mk_err() : mk(CB_T_DUR, (uint64_t)r);
        if (a.tag == CB_T_TS && b.tag == CB_T_DUR) {
            if (sub_ovf(x, y, &r)) { c.unsupported = 1; return mk_err(); }
            return mk(CB_T_TS, (uint64_t)r);
        }
        if (a.tag == CB_T_DUR && b.tag == CB_T_DUR) return sub_ovf(x, y, &r) ? mk_err() : mk(CB_T_DUR, (uint64_t)r);
    }
    return mk_err();
}

// ---- string predicates (byte-wise; UTF-8 makes prefix/suffix/substring tests byte-exact) ----
CB_HD bool bytes_eq(const uint8_t *a, const uint8_t *b, uint32_t n) {
    for (uint32_t i = 0; i < n; i++)
        if (ldg(a + i) != ldg(b + i)) return false;
    return true;
}
CB_HD Val do_str2(const Ctx &c, int op, const Val &s, const Val &t) {
    if (s.tag != CB_T_STRING || t.tag != CB_T_STRING) return mk_err();
    const uint8_t *ps, *pt;
    uint32_t ls, lt;
    str_get(c, s.u, ps, ls);
    str_get(c, t.u, pt, lt);
    if (lt > ls) return mk_bool(false);
    if (op == CB_OP_STARTS_WITH) return mk_bool(bytes_eq(ps, pt, lt));
    if (op == CB_OP_ENDS_WITH) return mk_bool(bytes_eq(ps + (ls - lt), pt, lt));
    for (uint32_t i = 0; i + lt <= ls; i++)
        if (bytes_eq(ps + i, pt, lt)) return mk_bool(true);
    return mk_bool(false);
}
CB_HD uint32_t utf8_len(const uint8_t *p, uint32_t n) {
    uint32_t k = 0;
    for (uint32_t i = 0; i < n; i++) k += (ldg(p + i) & 0xC0) != 0x80;
    return k;
}

// ---- Go time.ParseDuration (cel-go duration(string)): [+-] then one or more <digits>[.<digits>]<unit>, or "0" ----
// -> 0 ok, 1 invalid / out of range (CEL error), 2 more than 25 fraction digits (not representable here)
CB_HD int parse_duration_text(const uint8_t *p, uint32_t n, int64_t *out) {
    uint32_t i = 0;
    bool neg = false;
    if (n == 0) return 1;
    if (ldg(p) == '+' || ldg(p) == '-') { neg = ldg(p) == '-'; i = 1; }
    if (n - i == 1 && ldg(p + i) == '0') { *out = 0; return 0; }
    if (i == n) return 1;
    const uint64_t kLimit = 1ull << 63;
    uint64_t total = 0;
    bool over = false;
    while (i < n) {
        uint64_t whole = 0;
        bool any = false;
        while (i < n && ldg(p + i) >= '0' && ldg(p + i) <= '9') {
            const uint64_t d = ldg(p + i) - '0';
            if (whole > (kLimit - d) / 10) over = true; else whole = whole * 10 + d;
            any = true; i++;
        }
        unsigned __int128 frac = 0, scale = 1;
        uint32_t nfrac = 0;
        if (i < n && ldg(p + i) == '.') {
            i++;
            while (i < n && ldg(p + i) >= '0' && ldg(p + i) <= '9') {
                if (nfrac >= 25) return 2;
                frac = frac * 10 + (ldg(p + i) - '0'); scale *= 10; nfrac++; i++;
            }
        }
        if (!any && nfrac == 0) return 1;
        uint64_t unit = 0;
        const uint32_t rem = n - i;
        const uint8_t c0 = rem > 0 ? ldg(p + i) : 0, c1 = rem > 1 ? ldg(p + i + 1) : 0, c2 = rem > 2 ? ldg(p + i + 2) : 0;
        if (c0 == 'n' && c1 == 's') { unit = 1; i += 2; }
        else if (c0 == 'u' && c1 == 's') { unit = 1000; i += 2; }
        else if ((c0 == 0xC2 && c1 == 0xB5 && c2 == 's') || (c0 == 0xCE && c1 == 0xBC && c2 == 's')) { unit = 1000; i += 3; }   // U+00B5 / U+03BC
        else if (c0 == 'm' && c1 == 's') { unit = 1000000; i += 2; }
        else if (c0 == 's') { unit = 1000000000ull; i += 1; }
        else if (c0 == 'm') { unit = 60000000000ull; i += 1; }
        else if (c0 == 'h') { unit = 3600000000000ull; i += 1; }
        else return 1;
        if (whole > kLimit / unit) over = true;
        uint64_t v = over ? 0 : whole * unit;
        const unsigned __int128 fv = frac * unit / scale;   // < unit
        if (!over) { v += (uint64_t)fv; if (v > kLimit || total + v > kLimit || total + v < total) over = true; else total += v; }
    }
    if (over) return 1;
    if (neg) { *out = total == kLimit ? (int64_t)0x8000000000000000ull : -(int64_t)total; return 0; }
    if (total > kLimit - 1) return 1;
    *out = (int64_t)total;
    return 0;
}

// ---- timestamp / duration accessors in UTC (cel-go getFullYear ... getMilliseconds) ----
CB_HD int64_t days_from_civil(int64_t y, int m, int d);
CB_HD int64_t floor_div(int64_t a, int64_t b) { int64_t q = a / b; return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q; }
CB_HD void civil_from_days(int64_t z, int64_t *y, int *m, int *d) {   // days since 1970-01-01 -> proleptic Gregorian date
    z += 719468;
    const int64_t era = floor_div(z, 146097);
    const int64_t doe = z - era * 146097;
    const int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    const int64_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
    const int64_t mp = (5 * doy + 2) / 153;
    *d = (int)(doy - (153 * mp + 2) / 5 + 1);
    *m = (int)(mp < 10 ? mp + 3 : mp - 9);
    *y = yoe + era * 400 + (*m <= 2);
}
CB_HD Val do_ts_get(uint32_t field, const Val &v, uint32_t tzform, int32_t offset_s) {
    const int64_t ns = (int64_t)v.u;
    if (field == 0xFF) return mk_err();
    if (v.tag == CB_T_DUR) {
        if (tzform) return mk_err();   // total hours / minutes / seconds / milliseconds, truncated toward zero (Go integer division)
        switch (field) {
        case CB_TS_GETHOURS: return mk_int(ns / 3600000000000ll);
        case CB_TS_GETMINUTES: return mk_int(ns / 60000000000ll);
        case CB_TS_GETSECONDS: return mk_int(ns / 1000000000ll);
        case CB_TS_GETMILLISECONDS: return mk_int(ns / 1000000ll);
        default: return mk_err();
        }
    }
    if (v.tag != CB_T_TS) return mk_err();
    const int64_t s0 = floor_div(ns, 1000000000ll), sub = ns - s0 * 1000000000ll;
    const int64_t s = s0 + offset_s;
    const int64_t days = floor_div(s, 86400), rem = s - days * 86400;
    int64_t y; int m, d;
    civil_from_days(days, &y, &m, &d);
    switch (field) {
    case CB_TS_GETFULLYEAR: return mk_int(y);
    case CB_TS_GETMONTH: return mk_int(m - 1);
    case CB_TS_GETDAYOFYEAR: return mk_int(days - days_from_civil(y, 1, 1));
    case CB_TS_GETDAYOFMONTH: return mk_int(d - 1);
    case CB_TS_GETDATE: return mk_int(d);
    case CB_TS_GETDAYOFWEEK: return mk_int(((days + 4) % 7 + 7) % 7);
    case CB_TS_GETHOURS: return mk_int(rem / 3600);
    case CB_TS_GETMINUTES: return mk_int(rem % 3600 / 60);
    case CB_TS_GETSECONDS: return mk_int(rem % 60);
    default: return mk_int(sub / 1000000);
    }
}

// ---- hierarchy(s, delim) (conditions/types/hierarchy.go:146-410): segments = strings.Split(s, delim), never
// materialised -- the relations walk both strings segment by segment
struct HierIt { const uint8_t *p; uint32_t n; const uint8_t *d; uint32_t dn; uint32_t pos; bool more; };
CB_HD HierIt hier_it(const Ctx &c, uint64_t sid, uint32_t delim_id) {
    HierIt h;
    str_get(c, sid, h.p, h.n);
    str_get(c, delim_id, h.d, h.dn);
    h.pos = 0; h.more = true;
    return h;
}
// next segment -> [*s, *s + *l); false when there is none left
CB_HD bool hier_next(HierIt &h, uint32_t *s, uint32_t *l) {
    if (!h.more) return false;
    *s = h.pos;
    for (uint32_t i = h.pos; i + h.dn <= h.n; i++) {
        if (bytes_eq(h.p + i, h.d, h.dn)) { *l = i - h.pos; h.pos = i + h.dn; return true; }
    }
    *l = h.n - h.pos;
    h.more = false;
    return true;
}
CB_HD uint32_t hier_count(HierIt h) {
    uint32_t k = 0, s, l;
    while (hier_next(h, &s, &l)) k++;
    return k;
}
// number of equal leading segments of a and b, at most `limit`
CB_HD uint32_t hier_common(HierIt a, HierIt b, uint32_t limit) {
    uint32_t k = 0, sa, la, sb, lb;
    while (k < limit && hier_next(a, &sa, &la) && hier_next(b, &sb, &lb)) {
        if (la != lb || !bytes_eq(a.p + sa, b.p + sb, la)) break;
        k++;
    }
    return k;
}
CB_HD bool hier_rel(uint32_t rel, const HierIt &a, const HierIt &b) {
    const uint32_t na = hier_count(a), nb = hier_count(b);
    switch (rel) {
    case CB_HIER_ANCESTOROF: return nb > na && hier_common(a, b, na) == na;
    case CB_HIER_DESCENDENTOF: return na > nb && hier_common(a, b, nb) == nb;
    case CB_HIER_IMMEDIATEPARENTOF: return nb == na + 1 && hier_common(a, b, na) == na;
    case CB_HIER_IMMEDIATECHILDOF: return na == nb + 1 && hier_common(a, b, nb) == nb;
    case CB_HIER_SIBLINGOF: return na == nb && hier_common(a, b, na - 1) == na - 1;
    case CB_HIER_OVERLAPS: { const uint32_t m = na < nb ? na : nb; return hier_common(a, b, m) == m; }
    default: return na == nb && hier_common(a, b, na) == na;   // CB_HIER_EQUALS
    }
}
CB_HD uint32_t hier_ca_size(const HierIt &a, const HierIt &b) {   // size of a.commonAncestors(b)
    const uint32_t na = hier_count(a), nb = hier_count(b);
    uint32_t m = na < nb ? na : nb;
    if (na == nb) m = na - 1;
    return hier_common(a, b, m);
}
// operand of a hierarchy op: a string, else error (list operands -- hierarchy(list) -- are not representable here)
CB_HD bool hier_operand(Ctx &c, const Val &v) {
    if (v.tag == CB_T_LIST) c.unsupported = 1;
    return v.tag == CB_T_STRING;
}

// ---- RFC 3339 text -> int64 nanoseconds ----
CB_HD int64_t days_from_civil(int64_t y, int m, int d) {
    y -= m <= 2;
    int64_t era = (y >= 0 ? y : y - 399) / 400;
    int64_t yoe = y - era * 400;
    int64_t doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
    int64_t doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    return era * 146097 + doe - 719468;
}
CB_HD bool digits(const uint8_t *p, int n, int *out) {
    int v = 0;
    for (int i = 0; i < n; i++) {
        uint8_t ch = ldg(p + i);
        if (ch < '0' || ch > '9') return false;
        v = v * 10 + (ch - '0');
    }
    *out = v;
    return true;
}
// timestamp(string): Go's time.Parse(time.RFC3339, s) as cel-go calls it -- 'T' and 'Z' in upper case only, a fraction after '.' or
// ',' of any length (nine digits kept), offsets up to 24:60 -- then cel-go's range check on the instant.
CB_HD_NOINLINE Val parse_ts(Ctx &c, const Val &s) {
    const uint8_t *p;
    uint32_t n;
    str_get(c, s.u, p, n);
    int y, mo, d, h, mi, se;
    if (n < 20) return mk_err();
    uint8_t tch = ldg(p + 10);
    if (!digits(p, 4, &y) || ldg(p + 4) != '-' || !digits(p + 5, 2, &mo) || ldg(p + 7) != '-' || !digits(p + 8, 2, &d) ||
        tch != 'T' || !digits(p + 11, 2, &h) || ldg(p + 13) != ':' || !digits(p + 14, 2, &mi) ||
        ldg(p + 16) != ':' || !digits(p + 17, 2, &se))
        return mk_err();
    uint32_t i = 19;
    int64_t ns = 0;
    uint8_t ch = ldg(p + i);
    if (ch == '.' || ch == ',') {
        i++;
        int k = 0;
        uint32_t st = i;
        while (i < n) {
            uint8_t dch = ldg(p + i);
            if (dch < '0' || dch > '9') break;
            if (k < 9) { ns = ns * 10 + (dch - '0'); k++; }
            i++;
        }
        if (i == st) return mk_err();
        while (k < 9) { ns *= 10; k++; }
    }
    if (i >= n) return mk_err();
    int64_t off = 0;
    ch = ldg(p + i);
    if (ch == 'Z') {
        if (i + 1 != n) return mk_err();
    } else if (ch == '+' || ch == '-') {
        int oh, om;     // (Go's range test is `>`: "some people do write offsets of 24 hours or 60 minutes")
        if (i + 6 != n || !digits(p + i + 1, 2, &oh) || ldg(p + i + 3) != ':' || !digits(p + i + 4, 2, &om) || oh > 24 || om > 60)
            return mk_err();
        off = (int64_t)(oh * 3600 + om * 60) * (ch == '+' ? 1 : -1);
    } else return mk_err();
    bool leap = (y % 4 == 0 && (y % 100 != 0 || y % 400 == 0));
    int dim = (mo == 2) ? (leap ? 29 : 28) : ((mo == 4 || mo == 6 || mo == 9 || mo == 11) ? 30 : 31);
    if (mo < 1 || mo > 12 || d < 1 || d > dim || h > 23 || mi > 59 || se > 59) return mk_err();
    int64_t secs = days_from_civil(y, mo, d) * 86400 + h * 3600 + mi * 60 + se - off;
    // cel-go: the INSTANT must lie in 0001-01-01T00:00:00Z .. 9999-12-31T23:59:59Z (year 0000 with a negative offset can)
    if (secs < -62135596800ll || secs > 253402300799ll) return mk_err();
    int64_t total;
    if (mul_ovf(secs, 1000000000ll, &total) || add_ovf(total, ns, &total)) {
        c.unsupported = 1;  // valid CEL timestamp outside the int64-nanosecond device range
        return mk_err();
    }
    return mk(CB_T_TS, (uint64_t)total);
}

// ---- IP addresses (Go net.ParseIP / IPNet.Contains) ----
CB_HD bool parse_ipv4(const uint8_t *p, uint32_t n, uint32_t *out) {
    uint32_t v = 0, i = 0;
    for (int part = 0; part < 4; part++) {
        uint32_t st = i;
        int x = 0;
        while (i < n) {
            uint8_t ch = ldg(p + i);
            if (ch < '0' || ch > '9') break;
            x = x * 10 + (ch - '0');
            i++;
            if (i - st > 3) return false;
        }
        if (i == st || x > 255 || (i - st > 1 && ldg(p + st) == '0')) return false;
        v = (v << 8) | (uint32_t)x;
        if (part < 3) {
            if (i >= n || ldg(p + i) != '.') return false;
            i++;
        }
    }
    if (i != n) return false;
    *out = v;
    return true;
}
CB_HD int hexv(uint8_t ch) {
    if (ch >= '0' && ch <= '9') return ch - '0';
    if (ch >= 'a' && ch <= 'f') return ch - 'a' + 10;
    if (ch >= 'A' && ch <= 'F') return ch - 'A' + 10;
    return -1;
}
// groups are accumulated into two 64-bit halves to avoid a dynamically indexed local array
CB_HD void ip6_set(uint64_t &hi, uint64_t &lo, int idx, uint32_t v) {
    if (idx < 4) hi |= (uint64_t)v << (48 - 16 * idx);
    else lo |= (uint64_t)v << (48 - 16 * (idx - 4));
}
CB_HD_NOINLINE bool parse_ipv6(const uint8_t *p, uint32_t n, uint64_t *ohi, uint64_t *olo) {
    // pass 1: count groups before/after "::" ; pass 2: place them
    uint64_t hi = 0, lo = 0;
    int ng = 0, ell = -1;
    uint32_t i = 0;
    uint32_t gv[8];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int q = 0; q < 8; q++) gv[q] = 0;
    if (n >= 2 && ldg(p) == ':' && ldg(p + 1) == ':') {
        ell = 0;
        i = 2;
    } else if (n >= 1 && ldg(p) == ':') return false;
    while (i < n) {
        uint32_t j = i;
        bool isv4 = false;
        while (j < n && ldg(p + j) != ':') { if (ldg(p + j) == '.') isv4 = true; j++; }
        if (isv4) {
            uint32_t v4;
            if (j != n || ng > 6 || !parse_ipv4(p + i, n - i, &v4)) return false;
            gv[ng++] = v4 >> 16;
            gv[ng++] = v4 & 0xFFFF;
            i = n;
            break;
        }
        if (j == i || j - i > 4 || ng >= 8) return false;
        uint32_t v = 0;
        for (uint32_t k = i; k < j; k++) {
            int h = hexv(ldg(p + k));
            if (h < 0) return false;
            v = v * 16 + (uint32_t)h;
        }
        gv[ng++] = v;
        i = j;
        if (i < n) {
            i++;
            if (i < n && ldg(p + i) == ':') {
                if (ell >= 0) return false;
                ell = ng;
                i++;
            } else if (i == n) return false;
        }
    }
    if (ell >= 0) {
        if (ng >= 8) return false;
        int tail = ng - ell;
        for (int q = 0; q < ell; q++) ip6_set(hi, lo, q, gv[q]);
        for (int q = 0; q < tail; q++) ip6_set(hi, lo, 8 - tail + q, gv[ell + q]);
    } else {
        if (ng != 8) return false;
        for (int q = 0; q < 8; q++) ip6_set(hi, lo, q, gv[q]);
    }
    *ohi = hi;
    *olo = lo;
    return true;
}
CB_HD_NOINLINE Val do_in_ip_range(Ctx &c, const Val &ip, const uint64_t *cidr) {
    if (ip.tag != CB_T_STRING) return mk_err();
    const uint8_t *p;
    uint32_t n;
    str_get(c, ip.u, p, n);
    bool has_colon = false, has_dot = false;
    for (uint32_t i = 0; i < n; i++) {
        uint8_t ch = ldg(p + i);
        if (ch == ':') has_colon = true;
        if (ch == '.') has_dot = true;
        if (ch == '%') return mk_err();
    }
    uint64_t fam = ldg(cidr), bits = ldg(cidr + 1), hi = ldg(cidr + 2), lo = ldg(cidr + 3);
    bool is4 = false;
    uint32_t v4 = 0;
    uint64_t ihi = 0, ilo = 0;
    if (has_dot && !has_colon) {
        if (!parse_ipv4(p, n, &v4)) return mk_err();
        is4 = true;
    } else if (has_colon) {
        if (!parse_ipv6(p, n, &ihi, &ilo)) return mk_err();
        if (ihi == 0 && (ilo >> 32) == 0xFFFF) { is4 = true; v4 = (uint32_t)ilo; }
    } else return mk_err();
    uint64_t nfam = fam, nbits = bits, nlo = lo;
    if (fam == 6 && hi == 0 && (lo >> 32) == 0xFFFF && bits >= 96) { nfam = 4; nbits = bits - 96; nlo = lo & 0xFFFFFFFFull; }
    if (is4) {
        if (nfam != 4) return mk_bool(false);
        uint32_t mask = nbits == 0 ? 0u : (uint32_t)(0xFFFFFFFFull << (32 - nbits));
        return mk_bool((v4 & mask) == ((uint32_t)nlo & mask));
    }
    if (nfam != 6) return mk_bool(false);
    uint64_t mhi = bits >= 64 ? ~0ull : (bits == 0 ? 0ull : (~0ull << (64 - bits)));
    uint64_t mlo = bits <= 64 ? 0ull : (bits == 128 ? ~0ull : (~0ull << (128 - bits)));
    return mk_bool((ihi & mhi) == (hi & mhi) && (ilo & mlo) == (lo & mlo));
}

// ---- conversions ----
CB_HD_NOINLINE Val conv_int(Ctx &c, const Val &v) {
    switch (v.tag) {
    case CB_T_INT: return v;
    case CB_T_UINT: return v.u > 0x7FFFFFFFFFFFFFFFull ? mk_err() : mk_int((int64_t)v.u);
    case CB_T_DOUBLE: {
        double d = u2d(v.u);
        if (d != d || d <= -9223372036854775808.0 || d >= 9223372036854775808.0) return mk_err();
        return mk_int((int64_t)d);
    }
    case CB_T_STRING: {
        const uint8_t *p;
        uint32_t n;
        str_get(c, v.u, p, n);
        uint32_t i = 0;
        bool neg = false;
        if (n) { uint8_t ch = ldg(p); if (ch == '+' || ch == '-') { neg = ch == '-'; i = 1; } }
        if (i == n) return mk_err();
        uint64_t acc = 0;
        for (; i < n; i++) {
            uint8_t ch = ldg(p + i);
            if (ch < '0' || ch > '9') return mk_err();
            if (acc > (0xFFFFFFFFFFFFFFFFull - 9) / 10) return mk_err();
            acc = acc * 10 + (uint64_t)(ch - '0');
        }
        if (neg) { if (acc > 0x8000000000000000ull) return mk_err(); return mk_int((int64_t)(0 - acc)); }
        if (acc > 0x7FFFFFFFFFFFFFFFull) return mk_err();
        return mk_int((int64_t)acc);
    }
    case CB_T_TS: { int64_t ns = (int64_t)v.u; int64_t s = ns / 1000000000; if (ns % 1000000000 < 0) s--; return mk_int(s); }
    case CB_T_DUR: return mk_int((int64_t)v.u);
    default: return mk_err();
    }
}
CB_HD_NOINLINE Val conv_uint(Ctx &c, const Val &v) {
    switch (v.tag) {
    case CB_T_UINT: return v;
    case CB_T_INT: return (int64_t)v.u < 0 ? mk_err() : mk(CB_T_UINT, v.u);
    case CB_T_DOUBLE: {
        double d = u2d(v.u);
        if (d != d || d < 0 || d >= 18446744073709551616.0) return mk_err();
        return mk(CB_T_UINT, (uint64_t)d);
    }
    case CB_T_STRING: {
        const uint8_t *p;
        uint32_t n;
        str_get(c, v.u, p, n);
        uint32_t i = 0;
        if (n == 0) return mk_err();      // strconv.ParseUint(s, 10, 64): digits only, "A sign prefix is not permitted"
        uint64_t acc = 0;
        for (; i < n; i++) {
            uint8_t ch = ldg(p + i);
            if (ch < '0' || ch > '9') return mk_err();
            uint64_t dg = (uint64_t)(ch - '0');
            if (acc > (0xFFFFFFFFFFFFFFFFull - dg) / 10) return mk_err();
            acc = acc * 10 + dg;
        }
        return mk(CB_T_UINT, acc);
    }
    default: return mk_err();
    }
}

// ---------------------------------------------------------------------------------------------- run-time values
// List / string producing functions (cel-go ext.Strings / ext.Lists, conditions/cel.go:62-75; Cerbos except /
// intersect, cerbos_lib.go:287, 433; hierarchy(list), hierarchy[i], types/hierarchy.go).  Results live in Ctx::scratch.
CB_HD bool scr_alloc(Ctx &c, uint32_t words, uint32_t *off) {
    if (c.scr_used + words > CB_SCRATCH_WORDS) { c.unsupported = 1; return false; }
    *off = c.scr_used;
    c.scr_used += words;
    return true;
}
// NaN-boxed element form of a value (what lists / maps hold); false: not representable (sets `unsupported`)
CB_HD bool encode_elem(Ctx &c, const Val &v, uint64_t *out) {
    switch (v.tag) {
    case CB_T_NULL: *out = (uint64_t)(CB_V64_BOX_BASE | CB_V64_NULL) << 48; return true;
    case CB_T_BOOL: *out = ((uint64_t)(CB_V64_BOX_BASE | CB_V64_BOOL) << 48) | (v.u & 1); return true;
    case CB_T_DOUBLE: *out = v.u; return true;
    case CB_T_STRING: *out = ((uint64_t)(CB_V64_BOX_BASE | CB_V64_STRING) << 48) | (v.u & 0xFFFFFFFFFFFFull); return true;
    case CB_T_INT: {
        const int64_t i = (int64_t)v.u;
        if (i < -(1ll << 47) || i >= (1ll << 47)) { c.unsupported = 1; return false; }
        *out = ((uint64_t)(CB_V64_BOX_BASE | CB_V64_INT) << 48) | (v.u & 0xFFFFFFFFFFFFull);
        return true;
    }
    case CB_T_LIST:
    case CB_T_MAP: {
        uint64_t pay = v.u & ~(kHeapBatch | kHeapScratch);
        if (v.u & kHeapBatch) pay |= CB_V64_HEAP_BATCH_BIT;
        else if (v.u & kHeapScratch) pay |= kV64ScratchBit;
        *out = ((uint64_t)(CB_V64_BOX_BASE | (v.tag == CB_T_LIST ? CB_V64_LIST : CB_V64_MAP)) << 48) | pay;
        return true;
    }
    default: c.unsupported = 1; return false;   // uint / timestamp / duration / bytes elements have no 8-byte form
    }
}
CB_HD Val mk_scratch(uint32_t tag, uint32_t off) { return mk(tag, kHeapScratch | off); }
// a list of n elements whose words the caller fills at c.scratch[*off + 1 ...]
CB_HD bool list_new(Ctx &c, uint32_t n, uint32_t *off) {
    if (!scr_alloc(c, n + 1, off)) return false;
    c.scratch[*off] = n;
    return true;
}
// string under construction at the top of the arena
struct StrB {
    Ctx *c; uint32_t b0, len, cap; bool ok;
};
CB_HD StrB strb_begin(Ctx &c) { StrB s; s.c = &c; s.b0 = c.scr_used * 8; s.len = 0; s.cap = (CB_SCRATCH_WORDS - c.scr_used) * 8; s.ok = true; return s; }
CB_HD void strb_put(StrB &s, uint8_t ch) {
    if (s.len >= s.cap || s.len >= 0xFFFF) { s.ok = false; return; }
    reinterpret_cast<uint8_t *>(s.c->scratch)[s.b0 + s.len++] = ch;
}
CB_HD void strb_bytes(StrB &s, const uint8_t *p, uint32_t n) { for (uint32_t i = 0; i < n; i++) strb_put(s, ldg(p + i)); }
CB_HD Val strb_end(StrB &s) {
    if (!s.ok) { s.c->unsupported = 1; return mk_err(); }
    s.c->scr_used += (s.len + 7) / 8;
    return mk(CB_T_STRING, kStrDyn | ((uint64_t)s.b0 << 16) | s.len);
}
CB_HD uint32_t rune_len(uint8_t lead) { return lead < 0x80 ? 1u : lead < 0xE0 ? 2u : lead < 0xF0 ? 3u : 4u; }
// byte offset of rune index r (r <= rune count)
CB_HD uint32_t rune_off(const uint8_t *p, uint32_t n, uint32_t r) {
    uint32_t i = 0;
    while (r > 0 && i < n) { i += rune_len(ldg(p + i)); r--; }
    return i < n ? i : n;
}
CB_HD uint32_t rune_at(const uint8_t *p, uint32_t n, uint32_t i, uint32_t *adv) {
    const uint8_t b0 = ldg(p + i);
    uint32_t l = rune_len(b0);
    if (i + l > n) l = n - i;
    *adv = l;
    if (l == 1) return b0;
    uint32_t cp = b0 & (0xFFu >> (l + 1));
    for (uint32_t k = 1; k < l; k++) cp = (cp << 6) | (ldg(p + i + k) & 0x3F);
    return cp;
}
CB_HD bool go_space(uint32_t r) {   // unicode.IsSpace (strings.TrimSpace)
    return r == 0x20 || (r >= 0x09 && r <= 0x0D) || r == 0x85 || r == 0xA0 || r == 0x1680 || (r >= 0x2000 && r <= 0x200A) || r == 0x2028 || r == 0x2029 ||
           r == 0x202F || r == 0x205F || r == 0x3000;
}
// first byte offset >= from where [q, q + m) occurs in [p, p + n), or n + 1
CB_HD uint32_t bytes_find(const uint8_t *p, uint32_t n, const uint8_t *q, uint32_t m, uint32_t from) {
    for (uint32_t i = from; i + m <= n; i++)
        if (bytes_eq(p + i, q, m)) return i;
    return n + 1;
}
struct LView { const uint64_t *p; uint32_t n; };
CB_HD LView lview(const Ctx &c, const Val &v) { LView l; l.p = heap_ptr(c, v.u); l.n = (uint32_t)ldg(l.p); l.p += 1; return l; }
CB_HD bool arg_int(const Val &v, int64_t *out) { if (v.tag != CB_T_INT) return false; *out = (int64_t)v.u; return true; }

CB_HD_NOINLINE Val dyn_concat(Ctx &c, const Val &a, const Val &b) {
    if (a.tag == CB_T_STRING && b.tag == CB_T_STRING) {
        const uint8_t *pa, *pb; uint32_t la, lb;
        str_get(c, a.u, pa, la); str_get(c, b.u, pb, lb);
        StrB s = strb_begin(c);
        strb_bytes(s, pa, la); strb_bytes(s, pb, lb);
        return strb_end(s);
    }
    if (a.tag == CB_T_LIST && b.tag == CB_T_LIST) {
        const LView x = lview(c, a), y = lview(c, b);
        uint32_t off;
        if (!list_new(c, x.n + y.n, &off)) return mk_err();
        for (uint32_t i = 0; i < x.n; i++) c.scratch[off + 1 + i] = ldg(x.p + i);
        for (uint32_t i = 0; i < y.n; i++) c.scratch[off + 1 + x.n + i] = ldg(y.p + i);
        // elements copied from another heap keep their own references (table / batch / arena bits travel in the word)
        return mk_scratch(CB_T_LIST, off);
    }
    return mk_err();
}

// ---------------------------------------------------------------------------------------------- printing
// ext.Strings format / strings.quote (oracle/celeval.py: _str_format, _fmt_verb, _fmt_s, format_double, format_timestamp,
// _f_quote).  Doubles print exactly: the shortest digits that round-trip by Schubfach (PAPERS.md), %f / %e from the exact
// decimal expansion of the binary value.  All text goes to the arena string under construction (StrB).
CB_HD uint64_t mulhi64(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}
// Schubfach's g(k) = floor(10^-k * 2^-r) + 1 with 2^125 < g(k) <= 2^126 and r = flog2pow10(-k) - 125, for -k = -292 .. 324,
// as g / 2^63 and g mod 2^63.  Computed with exact integer arithmetic; tests/test_format.py recomputes every entry.
#define CB_SCHUBFACH_G \
    0x7fbbd8fe5f5e6e27ull, 0x497a3a2704eec3dfull, \
    0x4fd5679efb9b04d8ull, 0x5dec645863153a6cull, \
    0x63cac186ba81c60eull, 0x75677d6e7bda8906ull, \
    0x7cbd71e869223792ull, 0x52c15cca1ad12b48ull, \
    0x4df6673141b562bbull, 0x53b8d9fe50c2bb0dull, \
    0x617400fd9222bb6aull, 0x48a7107de4f369d0ull, \
    0x79d1013cf6ab6a45ull, 0x1ad0d49d5e304444ull, \
    0x4c22a0c61a2b226bull, 0x20c284e25ade2aabull, \
    0x5f2b48f7a0b5eb06ull, 0x08f3261af195b555ull, \
    0x76f61b3588e365c7ull, 0x4b2fefa1adfb22abull, \
    0x4a59d101758e1f9cull, 0x5efdf5c50cbcf5abull, \
    0x5cf04541d2f1a783ull, 0x76bd73364fec3315ull, \
    0x742c569247ae1164ull, 0x746cd003e3e73fdbull, \
    0x489bb61b6ccccadfull, 0x08c402026e7087e9ull, \
    0x5ac2a3a247fffd96ull, 0x6af502830a0ca9e3ull, \
    0x71734c8ad9fffcfcull, 0x45b24323cc8fd45cull, \
    0x46e80fd6c83ffe1dull, 0x6b8f69f65fd9e4b9ull, \
    0x58a213cc7a4ffda5ull, 0x26734473f7d05de8ull, \
    0x6eca98bf98e3fd0eull, 0x50101590f5c47561ull, \
    0x453e9f77bf8e7e29ull, 0x120a0d7a999ac95dull, \
    0x568e4755af721db3ull, 0x368c90d940017bb4ull, \
    0x6c31d92b1b4ea520ull, 0x242fb50f9001daa1ull, \
    0x439f27baf1112734ull, 0x169dd129ba0128a5ull, \
    0x5486f1a9ad557101ull, 0x1c454574288172ceull, \
    0x69a8ae1418aacd41ull, 0x435696d132a1cf81ull, \
    0x42096ccc8f6ac048ull, 0x7a161e42bfa521b1ull, \
    0x528bc7ffb345705bull, 0x189ba5d36f8e6a1dull, \
    0x672eb9ffa016cc71ull, 0x7ec28f484b7204a4ull, \
    0x407d343fc40e3fc7ull, 0x1f39998d2f2742e7ull, \
    0x509c814fb511cfb9ull, 0x0707fff07af113a1ull, \
    0x64c3a1a3a25643a7ull, 0x28c9ffec99ad5889ull, \
    0x7df48a0c8aebd491ull, 0x12fc7fe7c018aeabull, \
    0x4eb8d647d6d364daull, 0x5bddcff0d80f6d2bull, \
    0x62670bd9cc883e11ull, 0x32d543ed0e134875ull, \
    0x7b00ced03faa4d95ull, 0x5f8a94e851981a93ull, \
    0x4ce0814227ca707dull, 0x4bb69d1132ff109cull, \
    0x6018a192b1bd0c9cull, 0x7ea444557fbed4c3ull, \
    0x781ec9f75e2c4fc4ull, 0x1e4d556adfae89f3ull, \
    0x4b133e3a9adbb1daull, 0x52f05562cbcd1638ull, \
    0x5dd80dc941929e51ull, 0x27ac6abb7ec05bc6ull, \
    0x754e113b91f745e5ull, 0x5197856a5e7072b8ull, \
    0x4950cac53b3a8bafull, 0x42feb3627b0647b3ull, \
    0x5ba4fd768a092e9bull, 0x33be603b19c7d99full, \
    0x728e3cd42c8b7a42ull, 0x20adf849e039d007ull, \
    0x4798e6049bd72c69ull, 0x346cbb2e2c242205ull, \
    0x597f1f85c2ccf783ull, 0x6187e9f9b72d2a86ull, \
    0x6fdee76733803564ull, 0x59e9e47824f87527ull, \
    0x45eb50a08030215eull, 0x78322ecb171b4939ull, \
    0x576624c8a03c29b6ull, 0x563eba7ddce21b87ull, \
    0x6d3fadfac84b3424ull, 0x2bce691d541aa268ull, \
    0x4447ccbcbd2f0096ull, 0x5b6101b25490a581ull, \
    0x5559bfebec7ac0bcull, 0x3239421ee9b4cee1ull, \
    0x6ab02fe6e79970ebull, 0x3ec792a6a422029aull, \
    0x42ae1df050bfe693ull, 0x173cbba8269541a0ull, \
    0x5359a56c64efe037ull, 0x7d0bea92303a9208ull, \
    0x68300ec77e2bd845ull, 0x7c4ee536bc49368aull, \
    0x411e093caedb672bull, 0x5db14f4235adc217ull, \
    0x51658b8bda9240f6ull, 0x551da312c319329cull, \
    0x65beee6ed136d134ull, 0x2a650bd773df7f43ull, \
    0x7f2eaa0a85848581ull, 0x34fe4ecd50d75f14ull, \
    0x4f7d2a469372d370ull, 0x711ef14052869b6cull, \
    0x635c74d8384f884dull, 0x0d66ad9067284247ull, \
    0x7c33920e46636a60ull, 0x30c058f480f252d9ull, \
    0x4da03b48ebfe227cull, 0x1e783798d09773c8ull, \
    0x61084a1b26fdab1bull, 0x2616457f04bd50baull, \
    0x794a5ca1f0bd15e2ull, 0x0f9bd6dec5eca4e8ull, \
    0x4bce79e536762dadull, 0x29c1664b3bb3e711ull, \
    0x5ec2185e8413b918ull, 0x5431bfde0aa0e0d5ull, \
    0x76729e762518a75eull, 0x693e2fd58d49190bull, \
    0x4a07a309d72f689bull, 0x21c6dde5784dafa7ull, \
    0x5c898bcc4cfb42c2ull, 0x0a38955ed6611b90ull, \
    0x73abeebf603a1372ull, 0x4cc6bab68bf96274ull, \
    0x484b75379c244c27ull, 0x4ffc34b2177bdd89ull, \
    0x5a5e5285832d5f31ull, 0x43fb41de9d5ad4ebull, \
    0x70f5e726e3f8b6fdull, 0x74fa125644b18a26ull, \
    0x4699b0784e7b725eull, 0x591c4b75eaeef658ull, \
    0x58401c96621a4ef6ull, 0x2f635e5365aab3edull, \
    0x6e5023bbfaa0e2b3ull, 0x7b3c35e83f1560e9ull, \
    0x44f216557ca48db0ull, 0x3d05a1b1276d5c92ull, \
    0x562e9beadbcdb11cull, 0x4c470a1d7148b3b6ull, \
    0x6bba42e592c11d63ull, 0x5f58cca4cd9ae0a3ull, \
    0x435469cf7bb8b25eull, 0x2b977fe70080cc66ull, \
    0x542984435aa6def5ull, 0x767d5fe0c0a0ff80ull, \
    0x6933e554315096b3ull, 0x341cb7d8f0c93f5full, \
    0x41c06f549ed25e30ull, 0x1091f2e7967dc79cull, \
    0x52308b29c686f5bcull, 0x14b66fa17c1d3983ull, \
    0x66bcadf43828b32bull, 0x19e40b89db2487e3ull, \
    0x4035ecb8a3196ffbull, 0x002e873628f6d4eeull, \
    0x504367e6cbdfcbf9ull, 0x603a2903b3348a2aull, \
    0x645441e07ed7bef8ull, 0x1848b344a001acb4ull, \
    0x7d6952589e8daeb6ull, 0x1e5ae015c80217e1ull, \
    0x4e61d37763188d31ull, 0x72f8cc0d9d014eedull, \
    0x61fa48553bdeb07eull, 0x2fb6ff110441a2a8ull, \
    0x7a78da6a8ad65c9dull, 0x7ba4bed545520b52ull, \
    0x4c8b888296c5f9e2ull, 0x5d46f7454b534713ull, \
    0x5fae6aa33c77785bull, 0x3498b5169e2818d8ull, \
    0x779a054c0b955672ull, 0x21bee25c45b21f0eull, \
    0x4ac0434f873d5607ull, 0x35174d79ab8f5369ull, \
    0x5d705423690cab89ull, 0x225d20d816732843ull, \
    0x74cc692c434fd66bull, 0x4af4690e1c0ff253ull, \
    0x48ffc1bbaa11e603ull, 0x1ed8c1a8d189f774ull, \
    0x5b3fb22a94965f84ull, 0x068ef21305ec7551ull, \
    0x720f9eb539bbf765ull, 0x0832ae97c76792a5ull, \
    0x4749c33144157a9full, 0x151fad1edca0bba8ull, \
    0x591c33fd951ad946ull, 0x7a67986693c8ea91ull, \
    0x6f6340fcfa618f98ull, 0x59017e8038bb2536ull, \
    0x459e089e1c7cf9bfull, 0x37a0ef102374f742ull, \
    0x57058ac5a39c382full, 0x25892ad42c523512ull, \
    0x6cc6ed770c83463bull, 0x0eeb75893766c256ull, \
    0x43fc546a67d20be4ull, 0x79532975c2a03976ull, \
    0x54fb698501c68edeull, 0x17a7f3d3334847d4ull, \
    0x6a3a43e642383295ull, 0x5d91f0c8001a59c8ull, \
    0x42646a6fe9631f9dull, 0x4a7b367d0010781dull, \
    0x52fd850be3bbe784ull, 0x7d1a041c40149625ull, \
    0x67bce64edcaae166ull, 0x1c6085235019bbaeull, \
    0x40d60ff149eaccdfull, 0x71bc53361210154dull, \
    0x510b93ed9c658017ull, 0x6e2b680396941aa0ull, \
    0x654e78e9037ee01dull, 0x69b642047c392148ull, \
    0x7ea21723445e9825ull, 0x2423d2859b476999ull, \
    0x4f254e760abb1f17ull, 0x26966393810ca200ull, \
    0x62eea2138d69e6ddull, 0x103bfc78614fca80ull, \
    0x7baa4a9870c46094ull, 0x344afb9679a3bd20ull, \
    0x4d4a6e9f467abc5cull, 0x60aedd3e0c065634ull, \
    0x609d0a4718196b73ull, 0x78da948d8f07ebc1ull, \
    0x78c44cd8de1fc650ull, 0x771139b0f2c9e6b1ull, \
    0x4b7ab0078ad3dbf2ull, 0x4a6ac40e97be302full, \
    0x5e595c096d88d2efull, 0x1d0575123dadbc3aull, \
    0x75efb30bc8eb07abull, 0x0446d256cd192b49ull, \
    0x49b5cfe75d92e4caull, 0x72ac4376402fbb0eull, \
    0x5c2343e134f79dfdull, 0x4f575453d03ba9d1ull, \
    0x732c14d98235857dull, 0x032d2968c44a9445ull, \
    0x47fb8d07f161736eull, 0x11fc39e17aae9cabull, \
    0x59fa7049edb9d049ull, 0x567b4859d95a43d6ull, \
    0x70790c5c6928445cull, 0x0c1a1a704fb0d4ccull, \
    0x464ba7b9c1b92ab9ull, 0x4790508631ce84ffull, \
    0x57de91a832277567ull, 0x797464a7be42263full, \
    0x6dd636123eb152c1ull, 0x77d17dd1add2afcfull, \
    0x44a5e1cb672ed3b9ull, 0x1ae2eea30ca3ade1ull, \
    0x55cf5a3e40fa88a7ull, 0x419baa4bcfcc995aull, \
    0x6b4330cdd1392ad1ull, 0x320294dec3bfbfb0ull, \
    0x4309fe80a2c3bac2ull, 0x6f419d0b3a57d7ceull, \
    0x53cc7e20cb74a973ull, 0x4b12044e08edcdc2ull, \
    0x68bf9da8fe51d3d0ull, 0x3dd685618b294132ull, \
    0x4177c2899ef32462ull, 0x26a6135cf6f9c8bfull, \
    0x51d5b32c06afed7aull, 0x704f983434b83aefull, \
    0x664b1ff7085be8d9ull, 0x4c637e4141e649abull, \
    0x7fdde7f4ca72e30full, 0x7f7c5dd1925fdc15ull, \
    0x4feab0f8fe87cde9ull, 0x7fadbaa2fb7be98dull, \
    0x63e55d373e29c164ull, 0x3f99294bba5ae3f1ull, \
    0x7cdeb4850db431bdull, 0x4f7f739ea8f19cedull, \
    0x4e0b30d328909f16ull, 0x41afa84329970214ull, \
    0x618dfd07f2b4c6dcull, 0x121b9253f3fcc299ull, \
    0x79f17c49ef61f893ull, 0x16a276e8f0fbf33full, \
    0x4c36edae359d3b5bull, 0x7e258a51969d7808ull, \
    0x5f44a919c3048a32ull, 0x7daeece5fc44d609ull, \
    0x7715d36033c5acbfull, 0x5d1aa81f7b560b8cull, \
    0x4a6da41c205b8bf7ull, 0x6a30a913ad15c738ull, \
    0x5d090d2328726ef5ull, 0x64bcd358985b3905ull, \
    0x744b506bf28f0ab3ull, 0x1dec082ebe720746ull, \
    0x48af1243779966b0ull, 0x02b3851d3707448cull, \
    0x5adad6d4557fc05cull, 0x0360666484c915afull, \
    0x71918c896adfb073ull, 0x04387ffda5fb5b1bull, \
    0x46faf7d5e2cbce47ull, 0x72a34ffe87bd18f1ull, \
    0x58b9b5cb5b7ec1d9ull, 0x6f4c23fe29ac5f2dull, \
    0x6ee8233e325e7250ull, 0x2b1f2cfdb41776f8ull, \
    0x45511606df7b0772ull, 0x1af37c1e908eaa5bull, \
    0x56a55b889759c94eull, 0x61b05b2634b254f2ull, \
    0x6c4eb26abd303ba2ull, 0x3a1c71efc1deea2eull, \
    0x43b12f82b63e2545ull, 0x4451c735d92b525dull, \
    0x549d7b6363cdae96ull, 0x756639034f7626f4ull, \
    0x69c4da3c3cc11a3cull, 0x52bfc7442353b0b1ull, \
    0x421b0865a5f8b065ull, 0x73b7dc8a96144e6full, \
    0x52a1ca7f0f76dc7full, 0x30a5d3ad3b99620bull, \
    0x674a3d1ed354939full, 0x1ccf48988a7fba8dull, \
    0x408e66334414dc43ull, 0x42018d5f568fd498ull, \
    0x50b1ffc0151a1354ull, 0x3281f0b72c33c9beull, \
    0x64de7fb01a609829ull, 0x3f226ce4f740bc2eull, \
    0x7e161f9c20f8be33ull, 0x6eeb081e3510eb39ull, \
    0x4ecdd3c1949b76e0ull, 0x3552e512e12a9304ull, \
    0x628148b1f9c25498ull, 0x42a79e57997537c5ull, \
    0x7b219ade7832e9beull, 0x535185ed7fd285b6ull, \
    0x4cf500cb0b1fd217ull, 0x1412f3b46fe39392ull, \
    0x603240fdcde7c69cull, 0x7917b0a18bdc7876ull, \
    0x783ed13d4161b844ull, 0x175d9cc9eed39694ull, \
    0x4b2742c648dd132aull, 0x4e9a81fe35443e1cull, \
    0x5df11377db1457f5ull, 0x2241227dc2954da3ull, \
    0x756d5855d1d96df2ull, 0x4ad16b1d333aa10cull, \
    0x49645735a327e4b7ull, 0x4ec2e2f24004a4a8ull, \
    0x5bbd6d030bf1dde5ull, 0x42739baed005cdd2ull, \
    0x72acc843ceee555eull, 0x7310829a84074146ull, \
    0x47abfd2a6154f55bull, 0x27ea51a0928488ccull, \
    0x5996fc74f9aa32b2ull, 0x11e4e608b725aaffull, \
    0x6ffcbb923814bf5eull, 0x565e1f8ae4ef15beull, \
    0x45fdf53b630cf79bull, 0x15fad3b6cf156d97ull, \
    0x577d728a3bd03581ull, 0x7b7988a482dac8fdull, \
    0x6d5ccf2ccac442e2ull, 0x3a57eacda3917b3cull, \
    0x445a017bfebaa9cdull, 0x4476f2c0863aed06ull, \
    0x557081dafe695440ull, 0x7594af70a7c9a847ull, \
    0x6acca251be03a951ull, 0x12f9db4cd1bc1258ull, \
    0x42bfe57316c249d2ull, 0x5bdc291003158b77ull, \
    0x536fdecfdc72dc47ull, 0x32d3335403daee55ull, \
    0x684bd683d38f9359ull, 0x1f88002904d1a9eaull, \
    0x412f66126439bc17ull, 0x63b50019a3030a33ull, \
    0x517b3f96fd482b1dull, 0x5ca240200bc3ccbfull, \
    0x65da0f7cbc9a35e5ull, 0x13cad0280eb4bfefull, \
    0x7f50935bebc0c35eull, 0x38bd84321261efebull, \
    0x4f925c1973587a1bull, 0x0376729f4b7d35f3ull, \
    0x6376f31fd02e98a1ull, 0x64540f471e5c836full, \
    0x7c54afe7c43a3ecaull, 0x1d691318e5f3a44bull, \
    0x4db4edf0daa4673eull, 0x3261abef8fb846afull, \
    0x6122296d114d810dull, 0x7efa16eb73a6585bull, \
    0x796ab3c855a0e151ull, 0x3eb89ca6508fee71ull, \
    0x4be2b05d35848cd2ull, 0x773361e7f259f507ull, \
    0x5edb5c7482e5b007ull, 0x55003a61eef07249ull, \
    0x76923391a39f1c09ull, 0x4a4048fa6aac8edbull, \
    0x4a1b603b06437185ull, 0x7e682d9c82abd949ull, \
    0x5ca23849c7d44de7ull, 0x3e023903a356cf9bull, \
    0x73cac65c39c96161ull, 0x2d82c7448c2c8382ull, \
    0x485ebbf9a41ddcdcull, 0x6c71bc8ad79bd231ull, \
    0x5a766af80d255414ull, 0x078e2bad8d82c6bdull, \
    0x711405b6106ea919ull, 0x0971b698f0e3786dull, \
    0x46ac8391ca4529afull, 0x55e7121f968e2b44ull, \
    0x5857a4763cd6741bull, 0x4b60d6a77c31b615ull, \
    0x6e6d8d93cc0c1122ull, 0x3e390c515b3e239aull, \
    0x4504787c5f878ab5ull, 0x46e3a7b2d906d640ull, \
    0x5645969b77696d62ull, 0x789c919f8f488bd0ull, \
    0x6bd6fc425543c8bbull, 0x56c3b607731aaec4ull, \
    0x43665da9754a5d75ull, 0x263a51c4a7f0ad3bull, \
    0x543ff513d29cf4d2ull, 0x4fc8e635d1ecd88aull, \
    0x694ff258c7443207ull, 0x23bb1fc346680eacull, \
    0x41d1f7777c8a9f44ull, 0x4654f3da0c01092cull, \
    0x524675555bad4715ull, 0x57ea30d08f014b76ull, \
    0x66d812aab29898dbull, 0x0de4bd04b2c19e54ull, \
    0x40470baaaf9f5f88ull, 0x78aef622efb902f5ull, \
    0x5058ce955b87376bull, 0x16dab3ababa743b2ull, \
    0x646f023ab2690545ull, 0x7c9160969691149eull, \
    0x7d8ac2c95f034697ull, 0x3bb5b8bc3c3559c5ull, \
    0x4e76b9bddb620c1eull, 0x55519375a5a1581bull, \
    0x6214682d523a8f26ull, 0x2aa5f8530f09ae22ull, \
    0x7a998238a6c932efull, 0x754f7667d2cc19abull, \
    0x4c9ff163683dbfd5ull, 0x7951aa00e3bf900bull, \
    0x5fc7edbc424d2fcbull, 0x37a614811caf740dull, \
    0x77b9e92b52e07bbeull, 0x258f99a163db5111ull, \
    0x4ad431bb13cc4d56ull, 0x7779c004de6912abull, \
    0x5d893e29d8bf60acull, 0x5558300616035755ull, \
    0x74eb8db44eef38d7ull, 0x6aae3c079b842d2aull, \
    0x49133890b1558386ull, 0x72ace584c1329c3bull, \
    0x5b5806b4ddaae468ull, 0x4f581ee5f17f4349ull, \
    0x722e086215159d82ull, 0x632e269f6ddf141bull, \
    0x475cc53d4d2d8271ull, 0x5dfcd823a4ab6c91ull, \
    0x5933f68ca078e30eull, 0x157c0e2c8dd647b5ull, \
    0x6f80f42fc8971bd1ull, 0x5adb11b7b14bd9a3ull, \
    0x45b0989ddd5e7163ull, 0x08c8eb12cecf6806ull, \
    0x571cbec554b60dbbull, 0x6afb25d782834207ull, \
    0x6ce3ee76a9e3912aull, 0x65b9ef4d63241289ull, \
    0x440e750a2a2e3abaull, 0x5f9435905df68b96ull, \
    0x5512124cb4b9c969ull, 0x377942f475742e7bull, \
    0x6a5696dfe1e83bc3ull, 0x655793b192d13a1aull, \
    0x42761e4bed31255aull, 0x2f56bc4efbc2c450ull, \
    0x5313a5dee87d6eb0ull, 0x7b2c6b62bab37564ull, \
    0x67d88f56a29cca5dull, 0x19f7863b696052bdull, \
    0x40e7599625a1fe7aull, 0x203ab3e521dc33b6ull, \
    0x51212ffbaf0a7e18ull, 0x684960de6a5340a4ull, \
    0x65697bfa9acd1d9full, 0x025bb91604e810cdull, \
    0x7ec3daf941806506ull, 0x62f2a75b86221500ull, \
    0x4f3a68dbc8f03f24ull, 0x1dd7a89933d54d20ull, \
    0x63090312bb2c4eedull, 0x254d92bf80caa068ull, \
    0x7bcb43d769f762a8ull, 0x4ea0f76f60fd4882ull, \
    0x4d5f0a66a23a9da9ull, 0x31249aa59c9e4d51ull, \
    0x60b6cd004ac94513ull, 0x5d6dc14f03c5e0a5ull, \
    0x78e480405d7b9658ull, 0x54c931a2c4b758cfull, \
    0x4b8ed0283a6d3df7ull, 0x34fdbf05baf29781ull, \
    0x5e72843249088d75ull, 0x223d2ec729af3d62ull, \
    0x760f253edb4ab0d2ull, 0x4acc7a78f41b0cbaull, \
    0x49c97747490eae83ull, 0x4ebfcc8b9890e7f4ull, \
    0x5c3bd5191b525a24ull, 0x426fbfae7eb521f1ull, \
    0x734aca5f6226f0adull, 0x530baf9a1e626a6dull, \
    0x480ebe7b9d58566cull, 0x43e74dc052fd8285ull, \
    0x5a126e1a84ae6c07ull, 0x54e1213067bce326ull, \
    0x709709a125da0709ull, 0x4a19697c81ac1befull, \
    0x465e6604b7a84465ull, 0x7e4fe1edd10b9175ull, \
    0x57f5ff85e592557full, 0x3de3da69454e75d3ull, \
    0x6df37f675ef6eadfull, 0x2d5cd10396a21347ull, \
    0x44b82fa09b5a52cbull, 0x4c5a02a23e254c0dull, \
    0x55e63b88c230e77eull, 0x3f70834acdae9f10ull, \
    0x6b5fca6af2bd215eull, 0x0f4ca41d811a46d4ull, \
    0x431bde82d7b634daull, 0x698fe69270b06c44ull, \
    0x53e2d6238da3c211ull, 0x43f3e0370cdc8755ull, \
    0x68db8bac710cb295ull, 0x74f0d844d013a92bull, \
    0x4189374bc6a7ef9dull, 0x5916872b020c49bbull, \
    0x51eb851eb851eb85ull, 0x0f5c28f5c28f5c29ull, \
    0x6666666666666666ull, 0x3333333333333334ull, \
    0x4000000000000000ull, 0x0000000000000001ull, \
    0x5000000000000000ull, 0x0000000000000001ull, \
    0x6400000000000000ull, 0x0000000000000001ull, \
    0x7d00000000000000ull, 0x0000000000000001ull, \
    0x4e20000000000000ull, 0x0000000000000001ull, \
    0x61a8000000000000ull, 0x0000000000000001ull, \
    0x7a12000000000000ull, 0x0000000000000001ull, \
    0x4c4b400000000000ull, 0x0000000000000001ull, \
    0x5f5e100000000000ull, 0x0000000000000001ull, \
    0x7735940000000000ull, 0x0000000000000001ull, \
    0x4a817c8000000000ull, 0x0000000000000001ull, \
    0x5d21dba000000000ull, 0x0000000000000001ull, \
    0x746a528800000000ull, 0x0000000000000001ull, \
    0x48c2739500000000ull, 0x0000000000000001ull, \
    0x5af3107a40000000ull, 0x0000000000000001ull, \
    0x71afd498d0000000ull, 0x0000000000000001ull, \
    0x470de4df82000000ull, 0x0000000000000001ull, \
    0x58d15e1762800000ull, 0x0000000000000001ull, \
    0x6f05b59d3b200000ull, 0x0000000000000001ull, \
    0x4563918244f40000ull, 0x0000000000000001ull, \
    0x56bc75e2d6310000ull, 0x0000000000000001ull, \
    0x6c6b935b8bbd4000ull, 0x0000000000000001ull, \
    0x43c33c1937564800ull, 0x0000000000000001ull, \
    0x54b40b1f852bda00ull, 0x0000000000000001ull, \
    0x69e10de76676d080ull, 0x0000000000000001ull, \
    0x422ca8b0a00a4250ull, 0x0000000000000001ull, \
    0x52b7d2dcc80cd2e4ull, 0x0000000000000001ull, \
    0x6765c793fa10079dull, 0x0000000000000001ull, \
    0x409f9cbc7c4a04c2ull, 0x1000000000000001ull, \
    0x50c783eb9b5c85f2ull, 0x5400000000000001ull, \
    0x64f964e68233a76full, 0x2900000000000001ull, \
    0x7e37be2022c0914bull, 0x1340000000000001ull, \
    0x4ee2d6d415b85aceull, 0x7c08000000000001ull, \
    0x629b8c891b267182ull, 0x5b0a000000000001ull, \
    0x7b426fab61f00de3ull, 0x31cc800000000001ull, \
    0x4d0985cb1d3608aeull, 0x0f1fd00000000001ull, \
    0x604be73de4838ad9ull, 0x52e7c40000000001ull, \
    0x785ee10d5da46d90ull, 0x07a1b50000000001ull, \
    0x4b3b4ca85a86c47aull, 0x04c5112000000001ull, \
    0x5e0a1fd271287598ull, 0x45f6556800000001ull, \
    0x758ca7c70d7292feull, 0x5773eac200000001ull, \
    0x4977e8dc68679bdfull, 0x16a872b940000001ull, \
    0x5bd5e313828182d6ull, 0x7c528f6790000001ull, \
    0x72cb5bd86321e38cull, 0x5b67334174000001ull, \
    0x47bf19673df52e37ull, 0x79208008e8800001ull, \
    0x59aedfc10d7279c5ull, 0x7768a00b22a00001ull, \
    0x701a97b150cf1837ull, 0x3542c80deb480001ull, \
    0x46109eced2816f22ull, 0x5149bd08b30d0001ull, \
    0x5794c6828721caebull, 0x259c2c4adfd04001ull, \
    0x6d79f82328ea3da6ull, 0x0f03375d97c45001ull, \
    0x446c3b15f9926687ull, 0x6962029a7edab201ull, \
    0x558749db77f70029ull, 0x63ba83411e915e81ull, \
    0x6ae91c5255f4c034ull, 0x1ca924116635b621ull, \
    0x42d1b1b375b8f820ull, 0x51e9b68adfe191d5ull, \
    0x53861e2053273628ull, 0x6664242d97d9f64aull, \
    0x6867a5a867f103b2ull, 0x7ffd2d38fdd073dcull, \
    0x4140c78940f6a24full, 0x6ffe3c439ea2486aull, \
    0x5190f96b91344ae3ull, 0x6bfdcb54864ada84ull, \
    0x65f537c675815d9cull, 0x66fd3e29a7dd9125ull, \
    0x7f7285b812e1b504ull, 0x00bc8db411d4f56eull, \
    0x4fa793930bcd1122ull, 0x4075d8908b251965ull, \
    0x63917877cec0556bull, 0x10934eb4adee5fbeull, \
    0x7c75d695c2706ac5ull, 0x74b82261d969f7adull, \
    0x4dc9a61d998642bbull, 0x58f3157d27e23accull, \
    0x613c0fa4ffe7d36aull, 0x4f2fdadc71dac97full, \
    0x798b138e3fe1c845ull, 0x22fbd1938e517bdfull, \
    0x4bf6ec38e7ed1d2bull, 0x25dd62fc38f2ed6cull, \
    0x5ef4a74721e86476ull, 0x0f54bbbb472fa8c6ull, \
    0x76b1d118ea627d93ull, 0x5329eaaa18fb92f8ull, \
    0x4a2f22af927d8e7cull, 0x23fa32aa4f9d3bdbull, \
    0x5cbaeb5b771cf21bull, 0x2cf8bf54e3848ad2ull, \
    0x73e9a63254e42ea2ull, 0x1836ef2a1c65ad86ull, \
    0x487207df750e9d25ull, 0x2f22557a51bf8c74ull, \
    0x5a8e89d75252446eull, 0x5aeaead8e62f6f91ull, \
    0x71322c4d26e6d58aull, 0x31a5a58f1fbb4b75ull, \
    0x46bf5bb038504576ull, 0x3f07877973d50f29ull, \
    0x586f329c466456d4ull, 0x0ec96957d0ca52f3ull, \
    0x6e8aff4357fd6c89ull, 0x127bc3adc4fce7b0ull, \
    0x4516df8a16fe63d5ull, 0x5b8d5a4c9b1e10ceull, \
    0x565c976c9cbdfccbull, 0x1270b0dfc1e59502ull, \
    0x6bf3bd47c3ed7bfdull, 0x770cdd17b25efa42ull, \
    0x4378564cda746d7eull, 0x5a680a2ecf7b5c69ull, \
    0x54566be0111188deull, 0x31020cba835a3384ull, \
    0x696c06d81555eb15ull, 0x7d428fe92430c065ull, \
    0x41e384470d55b2edull, 0x5e4999f1b69e783full, \
    0x525c6558d0ab1fa9ull, 0x15dc006e2446164full, \
    0x66f37eaf04d5e793ull, 0x3b530089ad579be2ull, \
    0x40582f2d6305b0bcull, 0x1513e0560c56c16eull, \
    0x506e3af8bbc71cebull, 0x1a58d86b8f6c71c9ull, \
    0x6489c9b6eab8e426ull, 0x00ef0e8673478e3bull, \
    0x7dac3c24a5671d2full, 0x412ad228101971c9ull, \
    0x4e8ba596e760723dull, 0x58bac3590a0fe71eull, \
    0x622e8efca1388ecdull, 0x0ee9742f4c93e0e6ull, \
    0x7aba32bbc986b280ull, 0x32a3d13b1fb8d91full, \
    0x4cb45fb55df42f90ull, 0x1fa662c4f3d387b3ull, \
    0x5fe177a2b5713b74ull, 0x278ffb7630c869a0ull, \
    0x77d9d58b62cd8a51ull, 0x3173fa53bcfa8408ull, \
    0x4ae825771dc07672ull, 0x6ee87c74561c9285ull, \
    0x5da22ed4e530940full, 0x4aa29b916ba3b726ull, \
    0x750aba8a1e7cb913ull, 0x3d4b4275c68ca4f0ull, \
    0x4926b496530df3acull, 0x164f09899c17e716ull, \
    0x5b7061bbe7d17097ull, 0x1be2cbec031de0dcull, \
    0x724c7a2ae1c5ccbdull, 0x02db7ee703e55912ull, \
    0x476fcc5acd1b9ff6ull, 0x11c92f50626f57acull, \
    0x594bbf71806287f3ull, 0x563b7b247b0b2d96ull, \
    0x6f9eaf4de07b29f0ull, 0x4bca59ed99cdf8fcull, \
    0x45c32d90ac4cfa36ull, 0x2f5e78348020bb9eull, \
    0x5733f8f4d76038c3ull, 0x7b361641a028ea85ull, \
    0x6d00f7320d3846f4ull, 0x7a039bd208332526ull, \
    0x44209a7f48432c59ull, 0x0c424163451ff738ull, \
    0x5528c11f1a53f76full, 0x2f52d1bc1667f506ull, \
    0x6a72f166e0e8f54bull, 0x1b27862b1c01f247ull, \
    0x4287d6e04c91994full, 0x00f8b3daf181376dull, \
    0x5329cc985fb5ffa2ull, 0x6136e0d1ade18548ull, \
    0x67f43fbe77a37f8bull, 0x398499061959e699ull, \
    0x40f8a7d70ac62fb7ull, 0x13f2dfa3cfd83020ull, \
    0x5136d1cccd77bba4ull, 0x78ef978cc3ce3c28ull, \
    0x6584864000d5aa8eull, 0x172b7d6ff4c1cb32ull, \
    0x7ee5a7d0010b1531ull, 0x5cf65ccbf1f23dfeull, \
    0x4f4f88e200a6ed3full, 0x0a19f9ff773766bfull, \
    0x63236b1a80d0a88eull, 0x6ca0787f5505406full, \
    0x7bec45e12104d2b2ull, 0x47c8969f2a46908aull, \
    0x4d73abacb4a303afull, 0x4cdd5e237a6c1a57ull, \
    0x60d09697e1cbc49bull, 0x4014b5ac590720ecull, \
    0x7904bc3dda3eb5c2ull, 0x3019e3176f48e927ull, \
    0x4ba2f5a6a8673199ull, 0x3e102deea58d91b9ull, \
    0x5e8bb3105280fdffull, 0x6d94396a4ef0f627ull, \
    0x762e9fd467213d7full, 0x68f947c4e2ad33b0ull, \
    0x49dd23e4c074c66full, 0x719bccdb0dac404eull, \
    0x5c546cddf091f80bull, 0x6e02c011d1175062ull, \
    0x736988156cb6760eull, 0x69837016455d247aull, \
    0x4821f50d63f209c9ull, 0x21f2260deb5a36ccull, \
    0x5a2a7250bcee8c3bull, 0x4a6eaf916630c47full, \
    0x70b50ee4ec2a2f4aull, 0x3d0a5b75bfbcf59full, \
    0x4671294f139a5d8eull, 0x4626792997d61984ull, \
    0x580d73a2d880f4f2ull, 0x17b01773fdcb9fe4ull, \
    0x6e10d08b8ea1322eull, 0x5d9c1d50fd3e87ddull, \
    0x44ca82573924bf5dull, 0x1a8192529e4714ebull, \
    0x55fd22ed076def34ull, 0x4121f6e745d8da25ull, \
    0x6b7c6ba849496b01ull, 0x516a74a1174f10aeull, \
    0x432dc3492dcde2e1ull, 0x02e288e4ae916a6dull, \
    0x53f9341b79415b99ull, 0x239b2b1dda35c508ull, \
    0x68f781225791b27full, 0x4c81f5e550c3364aull, \
    0x419ab0b576bb0f8full, 0x5fd139af527a01efull, \
    0x52015ce2d469d373ull, 0x57c5881b2718826aull, \
    0x6681b41b89844850ull, 0x4db6ea21f0dea304ull, \
    0x4011109135f2ad32ull, 0x30925255368b25e3ull, \
    0x501554b5836f587eull, 0x7cb6e6ea842def5cull, \
    0x641aa9e2e44b2e9eull, 0x5be4a0a525396b32ull, \
    0x7d21545b9d5dfa46ull, 0x32ddc8ce6e87c5ffull, \
    0x4e34d4b9425abc6bull, 0x7fca9d810514dbbfull, \
    0x61c209e792f16b86ull, 0x7fbd44e1465a12afull, \
    0x7a328c6177adc668ull, 0x5fac961997f0975bull, \
    0x4c5f97bceacc9c01ull, 0x3bcbddcffef65e99ull, \
    0x5f777dac257fc301ull, 0x6abed543feb3f63full, \
    0x77555d172edfb3c2ull, 0x256e8a94fe60f3cfull, \
    0x4a955a2e7d4bd059ull, 0x3765169d1efc9861ull, \
    0x5d3ab0ba1c9ec46full, 0x653e5c4466bbbe7aull, \
    0x74895ce8a3c6758bull, 0x5e8df355806aae18ull, \
    0x48d5da11665c0977ull, 0x2b18b8157042accfull, \
    0x5b0b5095bff30bd5ull, 0x15dee61acc535803ull, \
    0x71ce24bb2fefcecaull, 0x3b569fa17f682e03ull, \
    0x4720d6f4fdf5e13eull, 0x451623c4efa11cc2ull, \
    0x58e90cb23d73598eull, 0x165bacb62b8963f3ull, \
    0x6f234fdeccd02ff1ull, 0x5bf297e3b66bbcefull, \
    0x457611eb40021df7ull, 0x09779eee52035616ull, \
    0x56d396661002a574ull, 0x6bd586a9e6842b9bull, \
    0x6c887bff94034ed2ull, 0x06cae85460253682ull, \
    0x43d54d7fbc821143ull, 0x243ed134bc174211ull, \
    0x54caa0dfaba29594ull, 0x0d4e8581eb1d1295ull, \
    0x69fd4917968b3af9ull, 0x10a226e265e4573bull, \
    0x423e4daebe1704dbull, 0x5a65584d7faeb685ull, \
    0x52cde11a6d9cc612ull, 0x50feae60df9a6426ull, \
    0x678159610903f797ull, 0x253e59f91780fd2full, \
    0x40b0d7dca5a27abeull, 0x4746f83baeb09e3eull, \
    0x50dd0dd3cf0b196eull, 0x1918b64a9a5cc5cdull, \
    0x65145148c2cddfc9ull, 0x5f5ee3dd40f3f740ull, \
    0x7e59659af38157bcull, 0x17369cd49130f510ull, \
    0x4ef7df80d830d6d5ull, 0x4e822204dabe992aull, \
    0x62b5d7610e3d0c8bull, 0x0222aa86116e3f75ull, \
    0x7b634d3951cc4fadull, 0x62ab552795c9cf52ull, \
    0x4d1e1043d31fb1ccull, 0x4dab1538bd9e2193ull, \
    0x60659454c7e79e3full, 0x6115da86ed05a9f8ull, \
    0x787ef969f9e185cfull, 0x595b5128a8471476ull, \
    0x4b4f5be23c2cf3a1ull, 0x67d912b9692c6ccaull, \
    0x5e2332dacb38308aull, 0x21cf5767c37787fcull, \
    0x75abff917e063cacull, 0x6a432d41b45569fbull, \
    0x498b7fbaeec3e5ecull, 0x0269fc4910b5623dull, \
    0x5bee5fa9aa74df67ull, 0x03047b5b54e2baccull, \
    0x72e9f79415121740ull, 0x63c59a322a1b697full, \
    0x47d23abc8d2b4e88ull, 0x3e5b805f5a5121f0ull, \
    0x59c6c96bb076222aull, 0x4df2607730e56a6cull, \
    0x70387bc69c93aab5ull, 0x216ef894fd1ec506ull, \
    0x46234d5c21dc4ab1ull, 0x24e55b5d1e333b24ull, \
    0x57ac20b32a535d5dull, 0x4e1eb23465c009edull, \
    0x6d9728dff4e834b5ull, 0x01a65ec17f300c68ull, \
    0x447e798bf91120f1ull, 0x1107fb38ef7e07c1ull, \
    0x559e17eef755692dull, 0x3549fa072b5d89b1ull, \
    0x6b059deab52ac378ull, 0x629c7888f634ec1eull, \
    0x42e382b2b13aba2bull, 0x3da1cb5599e11393ull, \
    0x539c635f5d8968b6ull, 0x2d0a3e2b00595877ull, \
    0x68837c3734ebc2e3ull, 0x784ccdb5c06fae95ull, \
    0x41522da2811359ceull, 0x3b3000919845cd1dull, \
    0x51a6b90b21583042ull, 0x09fc00b5fe574065ull, \
    0x6610674de9ae3c52ull, 0x4c7b00e37ded107eull, \
    0x7f9481216419cb67ull, 0x1f99c11c5d68549dull, \
    0x4fbcd0b4de901f20ull, 0x43c018b1ba6134e2ull, \
    0x63ac04e2163426e8ull, 0x54b01ede28f9821bull, \
    0x7c97061a9bc130a2ull, 0x69dc2695b337e2a1ull, \
    0x4dde63d0a158be65ull, 0x6229981d9002eda5ull, \
    0x6155fcc4c9aeedffull, 0x1ab3fe24f403a90eull, \
    0x79ab7bf5fc1aa97full, 0x0160fdae31049351ull, \
    0x4c0b2d79bd90a9efull, 0x30dc9e8cdea2dc13ull, \
    0x5f0df8d82cf4d46bull, 0x1d13c630164b9318ull, \
    0x76d1770e38320986ull, 0x0458b7bc1bde77ddull, \
    0x4a42ea68e31f45f3ull, 0x62b772d5916b0aebull, \
    0x5cd3a5031be71770ull, 0x5b654f8af5c5cda5ull, \
    0x74088e43e2e0dd4cull, 0x723ea36db337410eull, \
    0x488558ea6dcc8a50ull, 0x07672624900288a9ull, \
    0x5aa6af25093face4ull, 0x0940efadb4032ad3ull, \
    0x71505aee4b8f981dull, 0x0b912b992103f588ull, \
    0x46d238d4ef39bf12ull, 0x173abb3fb4a27975ull, \
    0x5886c70a2b082ed6ull, 0x5d096a0fa1cb17d2ull, \
    0x6ea878ccb5ca3a8cull, 0x344bc4938a3dddc7ull, \
    0x45294b7ff19e6497ull, 0x60af5adc3666aa9cull, \
    0x56739e5fee05fdbdull, 0x58db319344005543ull, \
    0x6c1085f7e9877d2dull, 0x0f11fdf815006a94ull, \
    0x438a53baf1f4ae3cull, 0x196b3ebb0d20429dull, \
    0x546ce8a9ae71d9cbull, 0x1fc60e69d0685344ull, \
    0x698822d41a0e503eull, 0x07b7920444826815ull, \
    0x41f515c49048f226ull, 0x64d2bb42aad1810dull, \
    0x52725b35b45b2eb0ull, 0x3e076a135585e150ull, \
    0x670ef2032171fa5cull, 0x4d8944982ae759a4ull, \
    0x40695741f4e73c79ull, 0x7075cadf1ad09807ull, \
    0x5083ad1272210b98ull, 0x2c933d96e184be08ull, \
    0x64a498570ea94e7eull, 0x37b80cfc99e5ed8aull, \
    0x7dcdbe6cd253a21eull, 0x05a6103bc05f68edull, \
    0x4ea0970403744552ull, 0x6387ca25583ba194ull, \
    0x6248bcc5045156a7ull, 0x3c69bcaeae4a89f9ull, \
    0x7adaebf64565ac51ull, 0x2b842bda59dd2c77ull, \
    0x4cc8d379eb5f8bb2ull, 0x6b329b68782a3bcbull, \
    0x5ffb085866376e9full, 0x45ff42429634cabdull, \
    0x77f9ca6e7fc54a47ull, 0x377f12d33bc1fd6dull, \
    0x4afc1e850fdb4e6cull, 0x52af6bc405593e64ull, \
    0x5dbb262653d22207ull, 0x675b46b506af8dfdull, \
    0x7529efafe8c6aa89ull, 0x61321862485b717cull, \
    0x493a35cdf17c2a96ull, 0x0cbf4f3d6d3926eeull, \
    0x5b88c3416ddb353bull, 0x4fef230cc88770a9ull, \
    0x726af411c952028aull, 0x43eaebcffaa94cd3ull, \
    0x4782d88b1dd34196ull, 0x4a72d361fca9d004ull, \
    0x59638eade54811fcull, 0x1d0f883a7bd44405ull, \
    0x6fbc72595e9a167bull, 0x24536a491ac95506ull, \
    0x45d5c777db204e0dull, 0x06b4226db0bdd524ull, \
    0x574b3955d1e86190ull, 0x28612b091ced4a6dull, \
    0x6d1e07ab466279f4ull, 0x327975cb64289d08ull, \
    0x4432c4cb0bfd8c38ull, 0x5f8be99f1e996225ull, \
    0x553f75fdcefcef46ull, 0x776ee406e63fbaaeull, \
    0x6a8f537d42bc2b18ull, 0x554a9d089fcfa95aull, \
    0x4299942e49b59aefull, 0x354ea22563e1c9d8ull, \
    0x533ff939dc2301abull, 0x22a24aaebcda3c4eull, \
    0x680ff788532bc216ull, 0x0b4add5a6c10cb62ull, \
    0x4109fab533fb594dull, 0x670eca58838a7f1dull, \
    0x514c796280fa2fa1ull, 0x20d27ceea46d1ee4ull, \
    0x659f97bb2138bb89ull, 0x49071c2a4d88669dull, \
    0x7f077da9e986ea6bull, 0x7b48e334e0ea8045ull, \
    0x4f64ae8a31f45283ull, 0x3d0d8e010c92902bull, \
    0x633dda2cbe716724ull, 0x2c50f1814fb73436ull, \
    0x7c0d50b7ee0dc0edull, 0x37652de1a3a50143ull, \
    0x4d885272f4c89894ull, 0x329f3cad064720caull, \
    0x60ea670fb1fabeb9ull, 0x3f470bd847d8e8fdull, \
    0x792500d39e796e67ull, 0x6f18cece59cf233cull, \
    0x4bb72084430be500ull, 0x756f8140f8217605ull, \
    0x5ea4e8a553cede41ull, 0x12cb61913629d387ull, \
    0x764e22cea8c295d1ull, 0x377e39f583b44868ull, \
    0x49f0d5c129799da2ull, 0x72aee4397250ad41ull, \
    0x5c6d0b3173d8050bull, 0x4f5a9d47cee4d891ull, \
    0x73884dfdd0ce064eull, 0x43314499c29e0eb6ull, \
    0x483530bea280c3f1ull, 0x09fecae019a2c932ull, \
    0x5a427cee4b20f4edull, 0x2c7e7d98200b7b7eull, \
    0x70d31c29dde93228ull, 0x579e1cfe280e5a5dull, \
    0x4683f19a2ab1bf59ull, 0x36c2d21ed908f87bull, \
    0x5824ee00b55e2f2full, 0x647386a68f4b3699ull, \
    0x6e2e2980e2b5bafbull, 0x5d906850331e043full, \
    0x44dcd9f08db194ddull, 0x2a7a41321ff2c2a8ull, \
    0x5614106cb11dfa14ull, 0x5518d17ea7ef7352ull, \
    0x6b991487dd657899ull, 0x6a5f05de51eb5026ull, \
    0x433facd4ea5f6b60ull, 0x127b63aaf3331218ull, \
    0x540f980a24f74638ull, 0x171a3c95afffd69eull, \
    0x69137e0cae3517c6ull, 0x1ce0cbbb1bffcc45ull, \
    0x41ac2ec7ece12edbull, 0x720c7f54f17fdfabull, \
    0x52173a79e8197a92ull, 0x6e8f9f2a2ddfd796ull, \
    0x669d0918621fd937ull, 0x4a3386f4b957cd7bull, \
    0x402225af3d53e7c2ull, 0x5e603458f3d6e06dull, \
    0x502aaf1b0ca8e1b3ull, 0x35f8416f30cc9888ull, \
    0x64355ae1cfd31a20ull, 0x237651cafcffbeaaull, \
    0x7d42b19a43c7e0a8ull, 0x2c53e63dbc3fae55ull, \
    0x4e49af006a5cec69ull, 0x1bb46fe695a7ccf5ull, \
    0x61dc1ac084f42783ull, 0x42a18be03b11c033ull, \
    0x7a532170a6313164ull, 0x3349eed849d6303full, \
    0x4c73f4e667debedeull, 0x600e35472e25de28ull, \
    0x5f90f22001d66e96ull, 0x3811c298f9af55b1ull, \
    0x77752ea8024c0a3cull, 0x0616333f381b2b1eull, \
    0x4aa93d29016f8665ull, 0x43cde0078310faf3ull, \
    0x5d538c7341cb67feull, 0x74c1580963d539afull, \
    0x74a86f90123e41feull, 0x51f1ae0bbcca881bull, \
    0x48e945ba0b66e93full, 0x13370cc755fe9511ull, \
    0x5b2397288e40a38eull, 0x7804cff92b7e3a55ull, \
    0x71ec7cf2b1d0cc72ull, 0x560603f7765dc8eaull, \
    0x4733ce17af227fc7ull, 0x55c3c27aa9fa9d93ull, \
    0x5900c19d9aeb1fb9ull, 0x4b34b319547944f7ull, \
    0x6f40f20501a5e7a7ull, 0x7e01dfdfa9979635ull, \
    0x458897432107b0c8ull, 0x7ec12bebc9febde1ull, \
    0x56eabd13e9499cfbull, 0x1e7176e6bc7e6d59ull, \
    0x6ca56c58e39c043aull, 0x060dd4a06b9e08b0ull, \
    0x43e763b78e4182a4ull, 0x23c8a4e44342c56eull, \
    0x54e13ca571d1e34dull, 0x2cbace1d541376c9ull, \
    0x6a198bcece465c20ull, 0x57e981a4a918547bull, \
    0x424ff76140ebf994ull, 0x36f1f106e9af34cdull, \
    0x52e3f5399126f7f9ull, 0x44ae6d48a41b0201ull, \
    0x679cf287f570b5f7ull, 0x75da089acd21c281ull, \
    0x40c21794f96671baull, 0x79a84560c0351991ull, \
    0x50f29d7a37c00e29ull, 0x581256b8f0425ff5ull, \
    0x652f44d8c5b011b4ull, 0x0e16ec672c52f7f2ull, \
    0x7e7b160ef71c1621ull, 0x119ca780f767b5eeull, \
    0x4f0cedc95a718dd4ull, 0x5b01e8b09aa0d1b5ull
#if defined(__CUDACC__)
static __device__ const uint64_t kSchubfachG[] = {CB_SCHUBFACH_G};
#endif
#if !defined(__CUDACC_RTC__)
static const uint64_t kSchubfachGHost[] = {CB_SCHUBFACH_G};
#endif
CB_HD uint64_t schubfach_g(uint32_t i) {
#if defined(__CUDA_ARCH__)
    return kSchubfachG[i];
#else
    return kSchubfachGHost[i];
#endif
}
CB_HD int flog10pow2(int q) { return (int)(((int64_t)q * 661971961083ll) >> 41); }                       // floor(q log10 2)
CB_HD int flog10_3q_pow2(int q) { return (int)(((int64_t)q * 661971961083ll - 274743187321ll) >> 41); }  // floor(log10(3/4 2^q))
CB_HD int flog2pow10(int e) { return (int)(((int64_t)e * 913124641741ll) >> 38); }                       // floor(e log2 10)
// g * cp / 2^127 rounded to odd, over the bits the paper's rop keeps (g = g1 2^63 + g0)
CB_HD uint64_t schubfach_rop(uint64_t g1, uint64_t g0, uint64_t cp) {
    const uint64_t z = ((g1 * cp) >> 1) + mulhi64(g0, cp);
    return (mulhi64(g1, cp) + (z >> 63)) | (((z & 0x7FFFFFFFFFFFFFFFull) + 0x7FFFFFFFFFFFFFFFull) >> 63);
}
// The shortest decimal f * 10^e that rounds to the finite double `bits` (> 0); of several, the closest (a tie: even f).
CB_HD_NOINLINE void shortest_digits(uint64_t bits, uint64_t *f, int *e) {
    const int bq = (int)((bits >> 52) & 0x7FF);
    const uint64_t c = bq ? (bits & 0xFFFFFFFFFFFFFull) | (1ull << 52) : bits & 0xFFFFFFFFFFFFFull;
    const int q = bq ? bq - 1075 : -1074;
    const uint64_t out = c & 1, cb = c << 2, cbr = cb + 2;
    uint64_t cbl;
    int k;
    if (c != (1ull << 52) || q == -1074) { cbl = cb - 2; k = flog10pow2(q); }
    else { cbl = cb - 1; k = flog10_3q_pow2(q); }   // a power of two: the lower neighbour is half as far
    const int h = q + flog2pow10(-k) + 2;
    const uint32_t gi = 2u * (uint32_t)(292 - k);
    const uint64_t g1 = schubfach_g(gi), g0 = schubfach_g(gi + 1);
    const uint64_t vb = schubfach_rop(g1, g0, cb << h), vbl = schubfach_rop(g1, g0, cbl << h), vbr = schubfach_rop(g1, g0, cbr << h);
    const uint64_t s = vb >> 2;
    // one digit fewer, when that still rounds to the double.  The paper tries it from s >= 100 only (Java prints at least two
    // digits); Go prints the shortest, so the subnormals with s in 10..99 (c = 3..20) try it too: 8e-323, not 7.9e-323.
    if (s >= 10) {
        const uint64_t sp10 = s / 10 * 10, tp10 = sp10 + 10;
        const bool upin = vbl + out <= sp10 << 2, wpin = (tp10 << 2) + out <= vbr;
        if (upin != wpin) { *f = upin ? sp10 : tp10; *e = k; return; }
    }
    const uint64_t t = s + 1;
    const bool uin = vbl + out <= s << 2, win = (t << 2) + out <= vbr;
    *e = k;
    if (uin != win) { *f = uin ? s : t; return; }
    const int64_t cmp = (int64_t)(vb - ((s + t) << 1));
    *f = cmp < 0 || (cmp == 0 && (s & 1) == 0) ? s : t;
}
CB_HD void put_cstr(StrB &s, const char *t) { for (; *t; t++) strb_put(s, (uint8_t)*t); }
// reverses the bytes written since `from`
CB_HD void strb_reverse(StrB &s, uint32_t from) {
    uint8_t *b = reinterpret_cast<uint8_t *>(s.c->scratch) + s.b0;
    for (uint32_t i = from, j = s.len; i + 1 < j; i++, j--) { const uint8_t t = b[i]; b[i] = b[j - 1]; b[j - 1] = t; }
}
// Working memory of the printers: `bytes` (a multiple of 8) taken from the top of the arena, above what the string under
// construction may use; null when there is no room (the string is then marked overflowed).  Released in reverse order.  Keeping
// it out of the thread's stack keeps the interpreter kernels' stack frames as they are.
CB_HD void *strb_reserve(StrB &s, uint32_t bytes) {
    if (s.cap < s.len + bytes) { s.ok = false; return nullptr; }
    s.cap -= bytes;
    return reinterpret_cast<uint8_t *>(s.c->scratch) + s.b0 + s.cap;
}
CB_HD void strb_release(StrB &s, uint32_t bytes) { s.cap += bytes; }
CB_HD void put_u64(StrB &s, uint64_t v, uint32_t base, bool upper) {
    const uint32_t from = s.len;
    do { const uint32_t r = (uint32_t)(v % base); strb_put(s, (uint8_t)(r < 10 ? '0' + r : (upper ? 'A' : 'a') + r - 10)); v /= base; } while (v);
    strb_reverse(s, from);
}
CB_HD void put_int(StrB &s, const Val &x, uint32_t base, bool upper) {   // INT (sign, then magnitude) or UINT
    const bool neg = x.tag == CB_T_INT && (int64_t)x.u < 0;
    if (neg) strb_put(s, '-');
    put_u64(s, neg ? 0ull - x.u : x.u, base, upper);
}
CB_HD void put_exp10(StrB &s, int x) {   // e+XX: sign, at least two digits
    strb_put(s, 'e');
    strb_put(s, x < 0 ? '-' : '+');
    const uint32_t a = (uint32_t)(x < 0 ? -x : x);
    if (a < 10) strb_put(s, '0');
    put_u64(s, a, 10, false);
}
// Go strconv.FormatFloat(d, 'g', -1, 64) of a finite double: the shortest digits, in exponent form when the decimal exponent
// is below -4 or at least 6
CB_HD_NOINLINE void put_double_g(StrB &s, uint64_t bits) {
    if (bits >> 63) strb_put(s, '-');
    bits &= ~(1ull << 63);
    if (bits == 0) { strb_put(s, '0'); return; }
    uint64_t f;
    int e;
    shortest_digits(bits, &f, &e);
    while (f % 10 == 0) { f /= 10; e++; }
    uint64_t p10 = 1;
    int nd = 1;
    while (f / p10 >= 10) { p10 *= 10; nd++; }
    const int dp = nd + e, x = dp - 1;   // digits before the decimal point; decimal exponent
    const bool sci = x < -4 || x >= 6;
    const int point = sci ? 1 : dp;      // the decimal point goes before digit `point` (none when that is not inside the digits)
    if (point <= 0) {
        strb_put(s, '0'); strb_put(s, '.');
        for (int i = 0; i < -dp; i++) strb_put(s, '0');
    }
    for (int i = 0; i < nd || i < point; i++) {   // the digits, most significant first; zeros up to the point
        if (i == point && point > 0 && i < nd) strb_put(s, '.');
        strb_put(s, i < nd ? (uint8_t)('0' + f / p10 % 10) : (uint8_t)'0');
        p10 /= 10;
    }
    if (sci) put_exp10(s, x);
}
// Exact decimal expansion of a finite double's magnitude c * 2^q: the integer part in base-10^9 chunks (read most significant
// digit first), the fraction as a numerator over 2^fbits whose digits come out one at a time (times ten).
struct ExactDec {
    uint32_t ich[36], nich;   // integer part, least significant chunk first
    uint32_t fr[34], nfr;     // fraction numerator, 32-bit limbs, least significant first (the integer part's limbs while it is converted)
    uint32_t fbits, nid, j;   // fraction bits; integer digits; integer digits read so far
};
enum { CB_EXACT_BYTES = (sizeof(ExactDec) + 7) / 8 * 8 };
CB_HD_NOINLINE void exact_init(ExactDec &x, uint64_t bits) {
    const int bq = (int)((bits >> 52) & 0x7FF);
    uint64_t c = bits & 0xFFFFFFFFFFFFFull;
    if (bq) c |= 1ull << 52;
    const int q = bq ? bq - 1075 : -1074;
    x.nich = 0; x.nfr = 0; x.fbits = 0; x.j = 0;
    if (q >= 0) {             // c * 2^q as 32-bit limbs, converted to base 10^9 by repeated division
        uint32_t *L = x.fr;
        const uint32_t w = (uint32_t)q / 32, b = (uint32_t)q % 32;
        const uint64_t lo = c << b, hi = b ? c >> (64 - b) : 0;
        for (uint32_t i = 0; i < w; i++) L[i] = 0;
        L[w] = (uint32_t)lo; L[w + 1] = (uint32_t)(lo >> 32); L[w + 2] = (uint32_t)hi;
        uint32_t nl = w + 3;
        while (nl && L[nl - 1] == 0) nl--;
        while (nl) {
            uint64_t r = 0;
            for (uint32_t i = nl; i-- > 0;) {
                const uint64_t cur = (r << 32) | L[i];
                L[i] = (uint32_t)(cur / 1000000000u);
                r = cur % 1000000000u;
            }
            x.ich[x.nich++] = (uint32_t)r;
            while (nl && L[nl - 1] == 0) nl--;
        }
    } else {
        const uint32_t sh = (uint32_t)-q;
        for (uint64_t ip = sh >= 64 ? 0 : c >> sh; ip; ip /= 1000000000u) x.ich[x.nich++] = (uint32_t)(ip % 1000000000u);
        const uint64_t fp = sh >= 64 ? c : c & ((1ull << sh) - 1);
        x.fbits = sh;
        x.nfr = (sh + 31) / 32;
        for (uint32_t i = 0; i < x.nfr; i++) x.fr[i] = i == 0 ? (uint32_t)fp : i == 1 ? (uint32_t)(fp >> 32) : 0u;
    }
    x.nid = 0;
    if (x.nich) {
        x.nid = 9 * (x.nich - 1);
        for (uint32_t v = x.ich[x.nich - 1]; v; v /= 10) x.nid++;
    }
}
CB_HD uint32_t exact_int_digit(const ExactDec &x, uint32_t j) {   // j-th integer digit, most significant first
    const uint32_t r = x.nid - 1 - j;
    uint32_t v = x.ich[r / 9];
    for (uint32_t i = 0; i < r % 9; i++) v /= 10;
    return v % 10;
}
CB_HD uint32_t exact_frac_digit(ExactDec &x) {
    if (!x.nfr) return 0;
    uint64_t carry = 0;
    for (uint32_t i = 0; i < x.nfr; i++) {
        const uint64_t v = (uint64_t)x.fr[i] * 10u + carry;
        x.fr[i] = (uint32_t)v;
        carry = v >> 32;
    }
    const uint32_t tb = x.fbits - 32 * (x.nfr - 1);   // fraction bits in the top limb (1 .. 32)
    if (tb == 32) return (uint32_t)carry;
    const uint32_t d = (x.fr[x.nfr - 1] >> tb) | (uint32_t)(carry << (32 - tb));
    x.fr[x.nfr - 1] &= (1u << tb) - 1;
    return d;
}
CB_HD uint32_t exact_next(ExactDec &x) { return x.j < x.nid ? exact_int_digit(x, x.j++) : exact_frac_digit(x); }
CB_HD bool exact_rest_nonzero(const ExactDec &x) {   // any digit not read yet is non-zero
    for (uint32_t j = x.j; j < x.nid; j++) if (exact_int_digit(x, j)) return true;
    for (uint32_t i = 0; i < x.nfr; i++) if (x.fr[i]) return true;
    return false;
}
// Adds one unit in the last place to the digits written since byte `from` (a '.' is skipped); true: they were all nines
// (now zeros) and a leading one is missing.
CB_HD bool round_up_digits(StrB &s, uint32_t from) {
    uint8_t *b = reinterpret_cast<uint8_t *>(s.c->scratch) + s.b0;
    for (uint32_t i = s.len; i-- > from;) {
        if (b[i] == '.') continue;
        if (b[i] == '9') { b[i] = '0'; continue; }
        b[i]++;
        return false;
    }
    return true;
}
CB_HD bool round_half_even(uint32_t next, bool sticky, uint8_t last) { return next > 5 || (next == 5 && (sticky || (last & 1))); }
CB_HD uint8_t strb_last(const StrB &s) { return reinterpret_cast<const uint8_t *>(s.c->scratch)[s.b0 + s.len - 1]; }
// %.{prec}f (sci = false) or %.{prec}e of a finite double, exactly rounded (ties to even on the binary value)
CB_HD_NOINLINE void put_fixed_sci(StrB &s, uint64_t bits, uint32_t prec, bool sci) {
    ExactDec *xp = static_cast<ExactDec *>(strb_reserve(s, CB_EXACT_BYTES));
    if (!xp) return;
    ExactDec &x = *xp;
    exact_init(x, bits);
    if (bits >> 63) strb_put(s, '-');
    const uint32_t from = s.len;
    int x10 = 0;
    if (!sci) {
        if (x.nid == 0) strb_put(s, '0');
        while (x.j < x.nid) strb_put(s, (uint8_t)('0' + exact_next(x)));
    } else {
        uint32_t d0 = 0;
        if ((bits << 1) == 0) d0 = 0;
        else if (x.nid) { x10 = (int)x.nid - 1; d0 = exact_next(x); }
        else { x10 = -1; d0 = exact_frac_digit(x); while (d0 == 0) { x10--; d0 = exact_frac_digit(x); } }
        strb_put(s, (uint8_t)('0' + d0));
    }
    if (prec) strb_put(s, '.');
    for (uint32_t i = 0; i < prec && s.ok; i++) strb_put(s, (uint8_t)('0' + exact_next(x)));
    const uint32_t next = s.ok ? exact_next(x) : 0;   // the first digit dropped, then whether any later one is non-zero
    if (s.ok && round_half_even(next, exact_rest_nonzero(x), strb_last(s)) && round_up_digits(s, from)) {
        uint8_t *b = reinterpret_cast<uint8_t *>(s.c->scratch) + s.b0;
        if (sci) { b[from] = '1'; x10++; }           // 9.99e+00 -> 1.00e+01
        else {                                         // 9.99 -> 10.00
            strb_put(s, '0');
            if (s.ok) { for (uint32_t i = s.len - 1; i > from; i--) b[i] = b[i - 1]; b[from] = '1'; }
        }
    }
    strb_release(s, CB_EXACT_BYTES);
    if (sci) put_exp10(s, x10);
}
CB_HD void put_fixed(StrB &s, uint64_t bits, uint32_t prec) { put_fixed_sci(s, bits, prec, false); }
CB_HD void put_sci(StrB &s, uint64_t bits, uint32_t prec) { put_fixed_sci(s, bits, prec, true); }
// bytes that are valid UTF-8 (Go utf8.Valid: no overlong forms, no surrogates, nothing above U+10FFFF; the check
// string(bytes) makes)
CB_HD bool utf8_valid(const uint8_t *q, uint32_t m) {
    for (uint32_t i = 0; i < m;) {
        const uint32_t b0 = ldg(q + i);
        uint32_t need = 0, lo = 0x80, hi = 0xBF;
        if (b0 < 0x80) { i++; continue; }
        if (b0 >= 0xC2 && b0 <= 0xDF) need = 1;
        else if (b0 >= 0xE0 && b0 <= 0xEF) { need = 2; if (b0 == 0xE0) lo = 0xA0; if (b0 == 0xED) hi = 0x9F; }
        else if (b0 >= 0xF0 && b0 <= 0xF4) { need = 3; if (b0 == 0xF0) lo = 0x90; if (b0 == 0xF4) hi = 0x8F; }
        else return false;
        if (i + need >= m) return false;
        for (uint32_t k = 1; k <= need; k++) {
            const uint32_t bk = ldg(q + i + k);
            if (bk < (k == 1 ? lo : 0x80u) || bk > (k == 1 ? hi : 0xBFu)) return false;
        }
        i += need + 1;
    }
    return true;
}
CB_HD void put_2d(StrB &s, uint32_t v) { strb_put(s, (uint8_t)('0' + v / 10)); strb_put(s, (uint8_t)('0' + v % 10)); }
CB_HD void put_frac9(StrB &s, uint32_t ns) {   // .ddddddddd without trailing zeros (nothing for 0)
    if (!ns) return;
    strb_put(s, '.');
    uint32_t div = 100000000u;
    while (ns) { strb_put(s, (uint8_t)('0' + ns / div)); ns %= div; div /= 10; }
}
// RFC 3339 in UTC with the fraction's trailing zeros dropped (oracle #1 format_timestamp)
CB_HD void put_timestamp(StrB &s, int64_t ns) {
    const int64_t sec = floor_div(ns, 1000000000ll), sub = ns - sec * 1000000000ll;
    const int64_t days = floor_div(sec, 86400), rem = sec - days * 86400;
    int64_t y;
    int m, d;
    civil_from_days(days, &y, &m, &d);
    put_2d(s, (uint32_t)(y / 100)); put_2d(s, (uint32_t)(y % 100));   // (device timestamps lie in 1677 .. 2262)
    strb_put(s, '-'); put_2d(s, (uint32_t)m); strb_put(s, '-'); put_2d(s, (uint32_t)d);
    strb_put(s, 'T'); put_2d(s, (uint32_t)(rem / 3600)); strb_put(s, ':'); put_2d(s, (uint32_t)(rem % 3600 / 60));
    strb_put(s, ':'); put_2d(s, (uint32_t)(rem % 60));
    put_frac9(s, (uint32_t)sub);
    strb_put(s, 'Z');
}
CB_HD void put_duration(StrB &s, int64_t ns) {   // seconds with the fraction's trailing zeros dropped, then "s"
    const uint64_t a = ns < 0 ? 0ull - (uint64_t)ns : (uint64_t)ns;
    if (ns < 0) strb_put(s, '-');
    put_u64(s, a / 1000000000u, 10, false);
    put_frac9(s, (uint32_t)(a % 1000000000u));
    strb_put(s, 's');
}
CB_HD void put_nonfinite(StrB &s, double d) { put_cstr(s, d != d ? "NaN" : d > 0 ? "Infinity" : "-Infinity"); }
CB_HD const char *type_name_of(uint64_t code) {   // the name `%s` prints for a TYPE value (layout.TYPE_CODES)
    switch (code) {
    case CB_TYPE_BOOL: return "bool";
    case CB_TYPE_INT: return "int";
    case CB_TYPE_UINT: return "uint";
    case CB_TYPE_DOUBLE: return "double";
    case CB_TYPE_STRING: return "string";
    case CB_TYPE_BYTES: return "bytes";
    case CB_TYPE_LIST: return "list";
    case CB_TYPE_MAP: return "map";
    case CB_TYPE_NULL_TYPE: return "null_type";
    case CB_TYPE_TIMESTAMP: return "google.protobuf.Timestamp";
    case CB_TYPE_DURATION: return "google.protobuf.Duration";
    case CB_TYPE_TYPE: return "type";
    default: return nullptr;
    }
}
CB_HD int text_cmp(const uint8_t *b, uint32_t a0, uint32_t a1, uint32_t b0, uint32_t b1) {   // bytes [a0, a1) vs [b0, b1)
    for (; a0 < a1 && b0 < b1; a0++, b0++)
        if (b[a0] != b[b0]) return b[a0] < b[b0] ? -1 : 1;
    return a0 < a1 ? 1 : b0 < b1 ? -1 : 0;
}
// %s of a scalar; false: a CEL error (the format call's value is an error)
CB_HD_NOINLINE bool fmt_scalar(Ctx &c, StrB &s, const Val &x) {
    switch (x.tag) {
    case CB_T_NULL: put_cstr(s, "null"); return true;
    case CB_T_BOOL: put_cstr(s, x.u ? "true" : "false"); return true;
    case CB_T_INT: case CB_T_UINT: put_int(s, x, 10, false); return true;
    case CB_T_DOUBLE: {
        const double d = u2d(x.u);
        if (d != d || d - d != d - d) put_nonfinite(s, d);
        else put_double_g(s, x.u);
        return true;
    }
    case CB_T_STRING: case CB_T_BYTES: {
        const uint8_t *p;
        uint32_t n;
        str_get(c, x.u, p, n);
        if (x.tag == CB_T_BYTES && !utf8_valid(p, n)) return false;
        strb_bytes(s, p, n);
        return true;
    }
    case CB_T_TS: put_timestamp(s, (int64_t)x.u); return true;
    case CB_T_DUR: put_duration(s, (int64_t)x.u); return true;
    case CB_T_TYPE: {
        const char *name = type_name_of(x.u);
        if (!name) { c.unsupported = 1; return false; }
        put_cstr(s, name);
        return true;
    }
    case CB_T_ERR: return false;
    default: c.unsupported = 1; return false;   // SPIFFE ids / trust domains: custom types, not modelled
    }
}
enum { CB_FMT_MAX_DEPTH = 4, CB_FMT_MAX_ENTRIES = 16 };
// One open list or map of `%s`, kept at the top of the arena (strb_reserve) while its items print; a nested container's frame
// lies right below its parent's.  A map's entries are printed in arrival order first, then copied in sorted order and moved
// down over the unsorted text.
struct FmtFrame {
    uint64_t ref;                   // Val.u of the container
    uint32_t n, i;                  // elements (map: entries); items started (map: keys and values alternately)
    uint32_t start, is_map;         // where its text starts
    uint16_t k0[CB_FMT_MAX_ENTRIES], k1[CB_FMT_MAX_ENTRIES], v1[CB_FMT_MAX_ENTRIES];   // key text [k0, k1), value text [k1, v1)
    uint8_t ord[CB_FMT_MAX_ENTRIES];                                                  // entries by (key text, value text)
};
enum { CB_FMT_FRAME_BYTES = (sizeof(FmtFrame) + 7) / 8 * 8 };
// closes a map: its entries again, in order, behind the unsorted text, then moved down to its start
CB_HD void fmt_close_map(StrB &s, FmtFrame &f) {
    uint8_t *b = reinterpret_cast<uint8_t *>(s.c->scratch) + s.b0;
    for (uint32_t i = 0; i < f.n; i++) {          // insertion sort of the entry numbers
        uint32_t j = i;
        for (; j > 0; j--) {
            const uint32_t p = f.ord[j - 1];
            int r = text_cmp(b, f.k0[p], f.k1[p], f.k0[i], f.k1[i]);
            if (r == 0) r = text_cmp(b, f.k1[p], f.v1[p], f.k1[i], f.v1[i]);
            if (r <= 0) break;
            f.ord[j] = f.ord[j - 1];
        }
        f.ord[j] = (uint8_t)i;
    }
    const uint32_t body = s.len;
    strb_put(s, '{');
    for (uint32_t i = 0; i < f.n; i++) {
        const uint32_t p = f.ord[i];
        if (i) { strb_put(s, ','); strb_put(s, ' '); }
        for (uint32_t q = f.k0[p]; q < f.k1[p]; q++) strb_put(s, b[q]);
        strb_put(s, ':'); strb_put(s, ' ');
        for (uint32_t q = f.k1[p]; q < f.v1[p]; q++) strb_put(s, b[q]);
    }
    strb_put(s, '}');
    if (!s.ok) return;
    for (uint32_t q = body; q < s.len; q++) b[f.start + q - body] = b[q];
    s.len = f.start + (s.len - body);
}
// %s of any value, lists and maps included (without recursion: the open containers are frames in the arena).  Nesting deeper
// than CB_FMT_MAX_DEPTH containers or a map of more than CB_FMT_MAX_ENTRIES entries raises `unsupported`.
CB_HD_NOINLINE bool fmt_value(Ctx &c, StrB &s, const Val &x) {
    if (x.tag != CB_T_LIST && x.tag != CB_T_MAP) return fmt_scalar(c, s, x);
    FmtFrame *f = nullptr;   // the innermost open container
    uint32_t depth = 0;
    bool ok = true;
    Val v = x;
    for (;;) {
        if (v.tag == CB_T_LIST || v.tag == CB_T_MAP) {
            const uint32_t n = (uint32_t)ldg(heap_ptr(c, v.u));
            if (depth == CB_FMT_MAX_DEPTH || (v.tag == CB_T_MAP && n > CB_FMT_MAX_ENTRIES)) { c.unsupported = 1; ok = false; break; }
            FmtFrame *g = static_cast<FmtFrame *>(strb_reserve(s, CB_FMT_FRAME_BYTES));
            if (!g) break;                        // no room: the string is overflowed (flagged by strb_end)
            g->ref = v.u; g->n = n; g->i = 0; g->start = s.len; g->is_map = v.tag == CB_T_MAP;
            if (!g->is_map) strb_put(s, '[');
            f = g;
            depth++;
        } else {
            if (!fmt_scalar(c, s, v)) { ok = false; break; }
            if (f->is_map && (f->i & 1) == 0) f->v1[(f->i - 1) / 2] = (uint16_t)s.len;   // a value ended
        }
        // the next item to print, closing the containers that are complete
        bool next = false;
        while (depth && s.ok) {
            const uint64_t *p = heap_ptr(c, f->ref) + 1;
            if (f->i < (f->is_map ? 2 * f->n : f->n)) {
                const uint32_t j = f->i++;
                if (!f->is_map) {
                    if (j) { strb_put(s, ','); strb_put(s, ' '); }
                    v = decode_elem(ldg(p + j));
                } else if ((j & 1) == 0) {
                    f->k0[j / 2] = (uint16_t)s.len;
                    v = decode_elem(ldg(p + j / 2));
                } else {
                    f->k1[j / 2] = (uint16_t)s.len;
                    v = decode_elem(ldg(p + f->n + j / 2));
                }
                next = true;
                break;
            }
            if (f->is_map) fmt_close_map(s, *f);
            else strb_put(s, ']');
            strb_release(s, CB_FMT_FRAME_BYTES);
            depth--;
            f = f + 1;                            // the parent's frame (unused once depth is 0)
            if (depth && f->is_map && (f->i & 1) == 0) f->v1[(f->i - 1) / 2] = (uint16_t)s.len;
        }
        if (!next) break;
    }
    strb_release(s, depth * CB_FMT_FRAME_BYTES);
    return ok;
}
// one clause; false: a CEL error
CB_HD_NOINLINE bool fmt_verb(Ctx &c, StrB &s, uint32_t verb, uint32_t prec, const Val &x) {
    const bool is_int = x.tag == CB_T_INT || x.tag == CB_T_UINT;
    switch (verb) {
    case 's': return fmt_value(c, s, x);
    case 'd': {
        if (is_int) { put_int(s, x, 10, false); return true; }
        const double d = u2d(x.u);
        if (x.tag == CB_T_DOUBLE && (d != d || d - d != d - d)) { put_nonfinite(s, d); return true; }
        return false;
    }
    case 'f': case 'e': {
        if (!is_num(x)) return false;
        const double d = x.tag == CB_T_DOUBLE ? u2d(x.u) : x.tag == CB_T_INT ? (double)(int64_t)x.u : (double)x.u;
        if (d != d || d - d != d - d) put_nonfinite(s, d);
        else put_fixed_sci(s, d2u(d), prec, verb == 'e');
        return true;
    }
    case 'b':
        if (x.tag == CB_T_BOOL) { strb_put(s, x.u ? '1' : '0'); return true; }
        if (is_int) { put_int(s, x, 2, false); return true; }
        return false;
    case 'o':
        if (is_int) { put_int(s, x, 8, false); return true; }
        return false;
    case 'x': case 'X':
        if (is_int) { put_int(s, x, 16, verb == 'X'); return true; }
        if (x.tag == CB_T_STRING || x.tag == CB_T_BYTES) {
            const uint8_t *p;
            uint32_t n;
            str_get(c, x.u, p, n);
            const char *hx = verb == 'X' ? "0123456789ABCDEF" : "0123456789abcdef";
            for (uint32_t i = 0; i < n && s.ok; i++) { const uint8_t ch = ldg(p + i); strb_put(s, (uint8_t)hx[ch >> 4]); strb_put(s, (uint8_t)hx[ch & 15]); }
            return true;
        }
        return false;
    default: return false;
    }
}
// fmt.format(args) by the clause record at theap[rec] (layout.py FN FORMAT).  mode CB_FORMAT_ARGS_STACK: a[0 .. n) are the
// elements of the list literal; CB_FORMAT_ARGS_LIST: a[0] is the list.
CB_HD Val op_format(Ctx &c, const Val *a, uint32_t n, uint32_t mode, uint32_t rec) {
    LView l;
    l.p = nullptr; l.n = 0;
    if (mode == CB_FORMAT_ARGS_LIST) {
        if (n != 1 || a[0].tag != CB_T_LIST) return mk_err();
        l = lview(c, a[0]);
        n = l.n;
    } else {
        for (uint32_t i = 0; i < n; i++) if (a[i].tag == CB_T_ERR) return mk_err();
    }
    const uint64_t *r = c.t->theap() + rec;
    const uint64_t items = ldg(r);
    StrB s = strb_begin(c);
    uint32_t ai = 0;
    for (uint64_t i = 0; i < items && s.ok; i++) {
        const uint64_t w = ldg(r + 1 + i);
        const uint32_t verb = (uint32_t)(w & 0xFF);
        if (verb == 0) {      // a literal run
            const uint8_t *p;
            uint32_t len;
            str_get(c, w >> 32, p, len);
            strb_bytes(s, p, len);
            continue;
        }
        if (ai >= n) return mk_err();   // fewer arguments than clauses
        const Val x = mode == CB_FORMAT_ARGS_LIST ? decode_elem(ldg(l.p + ai)) : a[ai];
        ai++;
        const uint32_t prec = (uint32_t)((w >> 16) & 0xFFFF);
        if (!fmt_verb(c, s, verb, prec == CB_FMT_PREC_DEFAULT ? 6u : prec, x)) return mk_err();
    }
    return strb_end(s);
}
// strings.quote: s between double quotes with \a \b \f \n \r \t \v \\ \" escaped, every other byte as it is (device strings
// are valid UTF-8: a bytes value becomes a string only through that check)
CB_HD Val str_quote(Ctx &c, const Val &x) {
    if (x.tag != CB_T_STRING) return mk_err();
    const uint8_t *p;
    uint32_t n;
    str_get(c, x.u, p, n);
    StrB s = strb_begin(c);
    strb_put(s, '"');
    for (uint32_t i = 0; i < n && s.ok; i++) {
        const uint8_t ch = ldg(p + i);
        const char *esc = ch == 7 ? "\\a" : ch == 8 ? "\\b" : ch == 12 ? "\\f" : ch == 10 ? "\\n" : ch == 13 ? "\\r" : ch == 9 ? "\\t" :
                          ch == 11 ? "\\v" : ch == '\\' ? "\\\\" : ch == '"' ? "\\\"" : nullptr;
        if (esc) put_cstr(s, esc);
        else strb_put(s, ch);
    }
    strb_put(s, '"');
    return strb_end(s);
}
// The functions after the ext.Math block, reached through math_fn (op_fn sends every id from CB_FN_MATH_GREATEST on there):
// strings.quote, and format with its clause record first (an INT: THEAP offset | mode << 32).  Inlined into math_fn: a call
// edge of its own there changes how ptxas allocates registers across the interpreter's call graph (check_meta_kernel).
CB_HD Val fmt_fn(Ctx &c, uint32_t fn, const Val *a, uint32_t argc) {
    if (fn == CB_FN_QUOTE) return str_quote(c, a[0]);
    if (fn != CB_FN_FORMAT || argc < 1 || a[0].tag != CB_T_INT) { c.unsupported = 1; return mk_err(); }
    return op_format(c, a + 1, argc - 1, (uint32_t)(a[0].u >> 32), (uint32_t)a[0].u);
}

// string functions of cel-go ext.Strings (indices count code points)
CB_HD_NOINLINE Val dyn_strfn(Ctx &c, uint32_t fn, const Val *a, uint32_t argc) {
    for (uint32_t i = 0; i < argc; i++) if (a[i].tag == CB_T_ERR) return mk_err();
    if (fn == CB_FN_JOIN) {
        if (a[0].tag != CB_T_LIST || (argc == 2 && a[1].tag != CB_T_STRING)) return mk_err();
        const LView l = lview(c, a[0]);
        const uint8_t *ps = nullptr; uint32_t ls = 0;
        if (argc == 2) str_get(c, a[1].u, ps, ls);
        for (uint32_t i = 0; i < l.n; i++) if (decode_elem(ldg(l.p + i)).tag != CB_T_STRING) return mk_err();
        StrB s = strb_begin(c);
        for (uint32_t i = 0; i < l.n; i++) {
            const uint8_t *pe; uint32_t le;
            str_get(c, decode_elem(ldg(l.p + i)).u, pe, le);
            if (i) strb_bytes(s, ps, ls);
            strb_bytes(s, pe, le);
        }
        return strb_end(s);
    }
    if (fn == CB_FN_HIER_JOIN) {   // hierarchy(list of strings): the parts joined by U+001F, which no part may contain
        if (a[0].tag != CB_T_LIST) return mk_err();
        const LView l = lview(c, a[0]);
        for (uint32_t i = 0; i < l.n; i++) if (decode_elem(ldg(l.p + i)).tag != CB_T_STRING) return mk_err();
        StrB s = strb_begin(c);
        for (uint32_t i = 0; i < l.n; i++) {
            const uint8_t *pe; uint32_t le;
            str_get(c, decode_elem(ldg(l.p + i)).u, pe, le);
            for (uint32_t j = 0; j < le; j++) if (ldg(pe + j) == 0x1F) c.unsupported = 1;
            if (i) strb_put(s, 0x1F);
            strb_bytes(s, pe, le);
        }
        return strb_end(s);
    }
    if (fn == CB_FN_TO_BYTES) return (a[0].tag == CB_T_STRING || a[0].tag == CB_T_BYTES) ? mk(CB_T_BYTES, a[0].u) : mk_err();
    if (fn == CB_FN_TYPE_OF) {      // type(x): the run-time type as a TYPE value
        uint32_t code;
        switch (a[0].tag) {
        case CB_T_BOOL: code = CB_TYPE_BOOL; break;
        case CB_T_INT: code = CB_TYPE_INT; break;
        case CB_T_UINT: code = CB_TYPE_UINT; break;
        case CB_T_DOUBLE: code = CB_TYPE_DOUBLE; break;
        case CB_T_STRING: code = CB_TYPE_STRING; break;
        case CB_T_BYTES: code = CB_TYPE_BYTES; break;
        case CB_T_LIST: code = CB_TYPE_LIST; break;
        case CB_T_MAP: code = CB_TYPE_MAP; break;
        case CB_T_NULL: code = CB_TYPE_NULL_TYPE; break;
        case CB_T_TS: code = CB_TYPE_TIMESTAMP; break;
        case CB_T_DUR: code = CB_TYPE_DURATION; break;
        case CB_T_TYPE: code = CB_TYPE_TYPE; break;
        case CB_T_ERR: return mk_err();
        default: c.unsupported = 1; return mk_err();      // SPIFFE ids / trust domains: custom types, not modelled
        }
        return mk(CB_T_TYPE, code);
    }
    if (fn == CB_FN_TO_BOOL) {      // cel-go ConvertToType(BoolType): strconv.ParseBool on a string
        if (a[0].tag == CB_T_BOOL) return a[0];
        if (a[0].tag != CB_T_STRING) return mk_err();
        const uint8_t *q; uint32_t m;
        str_get(c, a[0].u, q, m);
        if (m == 0 || m > 5) return mk_err();
        uint8_t w[5] = {0, 0, 0, 0, 0};
        for (uint32_t i = 0; i < m; i++) w[i] = ldg(q + i);
        const bool rest_t = (w[1] == 'r' && w[2] == 'u' && w[3] == 'e') || (w[0] == 'T' && w[1] == 'R' && w[2] == 'U' && w[3] == 'E');
        const bool rest_f = (w[1] == 'a' && w[2] == 'l' && w[3] == 's' && w[4] == 'e') || (w[0] == 'F' && w[1] == 'A' && w[2] == 'L' && w[3] == 'S' && w[4] == 'E');
        if (m == 1 && (w[0] == '1' || w[0] == 't' || w[0] == 'T')) return mk_bool(true);
        if (m == 1 && (w[0] == '0' || w[0] == 'f' || w[0] == 'F')) return mk_bool(false);
        if (m == 4 && (w[0] == 't' || w[0] == 'T') && rest_t) return mk_bool(true);
        if (m == 5 && (w[0] == 'f' || w[0] == 'F') && rest_f) return mk_bool(false);
        return mk_err();
    }
    if (fn == CB_FN_TO_STRING) {
        // cel-go ConvertToType(StringType): string, int, uint, bool, bytes holding valid UTF-8, double.  A double prints by
        // strconv.FormatFloat(d, 'f', -1, 64): exact here for NaN, the infinities and integral values below 2^53 (JSON
        // numbers used as ids); shortest-digit printing of the rest, timestamps and durations is flagged, never approximated.
        const Val &x = a[0];
        if (x.tag == CB_T_STRING) return x;
        if (x.tag == CB_T_BYTES) {
            const uint8_t *q; uint32_t m;
            str_get(c, x.u, q, m);
            for (uint32_t i = 0; i < m;) {
                const uint32_t b0 = ldg(q + i);
                uint32_t need = 0, lo = 0x80, hi = 0xBF;
                if (b0 < 0x80) { i++; continue; }
                if (b0 >= 0xC2 && b0 <= 0xDF) need = 1;
                else if (b0 >= 0xE0 && b0 <= 0xEF) { need = 2; if (b0 == 0xE0) lo = 0xA0; if (b0 == 0xED) hi = 0x9F; }
                else if (b0 >= 0xF0 && b0 <= 0xF4) { need = 3; if (b0 == 0xF0) lo = 0x90; if (b0 == 0xF4) hi = 0x8F; }
                else return mk_err();
                if (i + need >= m) return mk_err();
                for (uint32_t k = 1; k <= need; k++) {
                    const uint32_t bk = ldg(q + i + k);
                    if (bk < (k == 1 ? lo : 0x80u) || bk > (k == 1 ? hi : 0xBFu)) return mk_err();
                }
                i += need + 1;
            }
            return mk(CB_T_STRING, x.u);
        }
        StrB s = strb_begin(c);
        if (x.tag == CB_T_BOOL) {
            const char *t = x.u ? "true" : "false";
            for (uint32_t i = 0; t[i]; i++) strb_put(s, (uint8_t)t[i]);
            return strb_end(s);
        }
        uint64_t mag;
        bool neg = false;
        if (x.tag == CB_T_INT) { neg = (int64_t)x.u < 0; mag = neg ? 0ull - x.u : x.u; }
        else if (x.tag == CB_T_UINT) mag = x.u;
        else if (x.tag == CB_T_DOUBLE) {
            const double d = u2d(x.u);
            if (d != d) { strb_put(s, 'N'); strb_put(s, 'a'); strb_put(s, 'N'); return strb_end(s); }
            if (d - d != d - d) { strb_put(s, d > 0 ? '+' : '-'); strb_put(s, 'I'); strb_put(s, 'n'); strb_put(s, 'f'); return strb_end(s); }
            const double ad = fabs(d);
            if (ad >= 9007199254740992.0 || floor(ad) != ad) { c.unsupported = 1; return mk_err(); }
            neg = (x.u >> 63) != 0;       // (-0 prints "-0")
            mag = (uint64_t)ad;
        } else {
            if (x.tag == CB_T_TS || x.tag == CB_T_DUR) c.unsupported = 1;
            return mk_err();
        }
        uint8_t dig[20];
        uint32_t nd = 0;
        do { dig[nd++] = (uint8_t)('0' + mag % 10); mag /= 10; } while (mag);
        if (neg) strb_put(s, '-');
        while (nd) strb_put(s, dig[--nd]);
        return strb_end(s);
    }
    if (fn == CB_FN_B64ENC) {
        if (a[0].tag != CB_T_BYTES) return mk_err();
        const uint8_t *q; uint32_t m;
        str_get(c, a[0].u, q, m);
        const char *abc = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
        StrB s = strb_begin(c);
        for (uint32_t i = 0; i < m; i += 3) {
            const uint32_t b0 = ldg(q + i), b1 = i + 1 < m ? ldg(q + i + 1) : 0, b2 = i + 2 < m ? ldg(q + i + 2) : 0;
            strb_put(s, (uint8_t)abc[b0 >> 2]);
            strb_put(s, (uint8_t)abc[((b0 & 3) << 4) | (b1 >> 4)]);
            strb_put(s, i + 1 < m ? (uint8_t)abc[((b1 & 15) << 2) | (b2 >> 6)] : (uint8_t)'=');
            strb_put(s, i + 2 < m ? (uint8_t)abc[b2 & 63] : (uint8_t)'=');
        }
        return strb_end(s);
    }
    if (fn == CB_FN_B64DEC) {
        // cel-go ext.Encoders: base64.StdEncoding.DecodeString, then RawStdEncoding (padding missing).  Go's decoder skips
        // '\r' and '\n' anywhere in the text and is not strict: non-zero trailing bits of the last quantum are dropped.
        if (a[0].tag != CB_T_STRING) return mk_err();
        const uint8_t *q; uint32_t m;
        str_get(c, a[0].u, q, m);
        uint32_t eff = 0, pad = 0;          // characters that count (no CR / LF), '=' at their end (at most two looked at)
        for (uint32_t i = 0; i < m; i++) {
            const uint8_t ch = ldg(q + i);
            if (ch == '\r' || ch == '\n') continue;
            eff++;
            pad = ch == '=' ? (pad < 2 ? pad + 1 : 3) : 0;
        }
        if (pad > 2) return mk_err();
        const uint32_t body = eff - pad;
        if (pad && (eff & 3) != 0) return mk_err();
        if ((body & 3) == 1) return mk_err();
        if (pad && (body & 3) + pad != 4) return mk_err();
        StrB s = strb_begin(c);
        uint32_t acc = 0, bits = 0, seen = 0;
        for (uint32_t i = 0; i < m && seen < body; i++) {
            const uint8_t ch = ldg(q + i);
            if (ch == '\r' || ch == '\n') continue;
            seen++;
            uint32_t v;
            if (ch >= 'A' && ch <= 'Z') v = ch - 'A'; else if (ch >= 'a' && ch <= 'z') v = ch - 'a' + 26;
            else if (ch >= '0' && ch <= '9') v = ch - '0' + 52; else if (ch == '+') v = 62; else if (ch == '/') v = 63; else return mk_err();
            acc = (acc << 6) | v; bits += 6;
            if (bits >= 8) { bits -= 8; strb_put(s, (uint8_t)(acc >> bits)); acc &= (1u << bits) - 1; }
        }
        Val r = strb_end(s);
        if (r.tag == CB_T_STRING) r.tag = CB_T_BYTES;
        return r;
    }
    if (a[0].tag != CB_T_STRING) return mk_err();
    const uint8_t *p; uint32_t n;
    str_get(c, a[0].u, p, n);
    const uint32_t nr = utf8_len(p, n);
    switch (fn) {
    case CB_FN_LOWER: case CB_FN_UPPER: {
        StrB s = strb_begin(c);
        for (uint32_t i = 0; i < n; i++) {
            uint8_t ch = ldg(p + i);
            if (fn == CB_FN_LOWER && ch >= 'A' && ch <= 'Z') ch += 32;
            if (fn == CB_FN_UPPER && ch >= 'a' && ch <= 'z') ch -= 32;
            strb_put(s, ch);
        }
        return strb_end(s);
    }
    case CB_FN_TRIM: {
        uint32_t lo = 0, hi = n, adv;
        while (lo < hi && go_space(rune_at(p, n, lo, &adv))) lo += adv;
        while (hi > lo) {   // step back one rune
            uint32_t q = hi - 1;
            while (q > lo && (ldg(p + q) & 0xC0) == 0x80) q--;
            if (!go_space(rune_at(p, n, q, &adv))) break;
            hi = q;
        }
        StrB s = strb_begin(c);
        strb_bytes(s, p + lo, hi - lo);
        return strb_end(s);
    }
    case CB_FN_STR_REVERSE: {
        StrB s = strb_begin(c);
        uint32_t hi = n;
        while (hi > 0) {
            uint32_t q = hi - 1;
            while (q > 0 && (ldg(p + q) & 0xC0) == 0x80) q--;
            strb_bytes(s, p + q, hi - q);
            hi = q;
        }
        return strb_end(s);
    }
    case CB_FN_CHARAT: {
        int64_t i;
        if (argc != 2 || !arg_int(a[1], &i)) return mk_err();
        if (i < 0 || i > (int64_t)nr) return mk_err();
        StrB s = strb_begin(c);
        if (i < (int64_t)nr) { const uint32_t o = rune_off(p, n, (uint32_t)i); strb_bytes(s, p + o, rune_len(ldg(p + o))); }
        return strb_end(s);
    }
    case CB_FN_INDEXOF: case CB_FN_LASTINDEXOF: {
        if (argc < 2 || a[1].tag != CB_T_STRING) return mk_err();
        const uint8_t *q; uint32_t m;
        str_get(c, a[1].u, q, m);
        int64_t off = fn == CB_FN_INDEXOF ? 0 : (int64_t)nr;
        if (argc == 3) { if (!arg_int(a[2], &off) || off < 0 || off > (int64_t)nr) return mk_err(); }
        if (m == 0) return mk_int(off);
        if (fn == CB_FN_INDEXOF) {
            const uint32_t at = bytes_find(p, n, q, m, rune_off(p, n, (uint32_t)off));
            return mk_int(at > n ? -1 : (int64_t)utf8_len(p, at));
        }
        // the last occurrence that starts at or before rune `off`
        const uint32_t lim = rune_off(p, n, (uint32_t)off);
        int64_t best = -1;
        for (uint32_t i = 0; i + m <= n && i <= lim; i++)
            if ((ldg(p + i) & 0xC0) != 0x80 && bytes_eq(p + i, q, m)) best = (int64_t)utf8_len(p, i);
        return mk_int(best);
    }
    case CB_FN_SUBSTRING: {
        int64_t st, en = (int64_t)nr;
        if (argc < 2 || !arg_int(a[1], &st) || (argc == 3 && !arg_int(a[2], &en))) return mk_err();
        if (st < 0 || st > (int64_t)nr || en < 0 || en > (int64_t)nr || st > en) return mk_err();
        const uint32_t o0 = rune_off(p, n, (uint32_t)st), o1 = rune_off(p, n, (uint32_t)en);
        StrB s = strb_begin(c);
        strb_bytes(s, p + o0, o1 - o0);
        return strb_end(s);
    }
    case CB_FN_REPLACE: {
        if (argc < 3 || a[1].tag != CB_T_STRING || a[2].tag != CB_T_STRING) return mk_err();
        int64_t lim = -1;
        if (argc == 4 && !arg_int(a[3], &lim)) return mk_err();
        const uint8_t *po, *pn; uint32_t lo, ln;
        str_get(c, a[1].u, po, lo); str_get(c, a[2].u, pn, ln);
        StrB s = strb_begin(c);
        int64_t done = 0;
        if (lo == 0) {   // Go strings.Replace with an empty `old`: `new` before every rune (and at the end) up to lim times
            uint32_t i = 0;
            while (i < n) {
                if (lim < 0 || done < lim) { strb_bytes(s, pn, ln); done++; }
                const uint32_t l = rune_len(ldg(p + i));
                strb_bytes(s, p + i, i + l <= n ? l : n - i);
                i += l;
            }
            if (lim < 0 || done < lim) strb_bytes(s, pn, ln);
            return strb_end(s);
        }
        uint32_t i = 0;
        while (i < n) {
            if ((lim < 0 || done < lim) && i + lo <= n && bytes_eq(p + i, po, lo)) { strb_bytes(s, pn, ln); i += lo; done++; }
            else strb_put(s, ldg(p + i++));
        }
        return strb_end(s);
    }
    case CB_FN_SPLIT: {
        if (argc < 2 || a[1].tag != CB_T_STRING) return mk_err();
        int64_t lim = -1;
        if (argc == 3 && !arg_int(a[2], &lim)) return mk_err();
        const uint8_t *q; uint32_t m;
        str_get(c, a[1].u, q, m);
        // count the pieces first (Go strings.SplitN)
        uint32_t pieces = 0;
        if (lim != 0) {
            if (m == 0) pieces = nr;
            else { pieces = 1; for (uint32_t i = 0; i + m <= n;) { if (bytes_eq(p + i, q, m)) { pieces++; i += m; } else i++; } }
            if (lim > 0 && (int64_t)pieces > lim) pieces = (uint32_t)lim;
        }
        uint32_t off;
        if (!list_new(c, pieces, &off)) return mk_err();
        uint32_t i = 0;
        for (uint32_t k = 0; k < pieces; k++) {
            uint32_t end;
            if (k + 1 == pieces) end = n;
            else if (m == 0) end = i + rune_len(ldg(p + i));
            else end = bytes_find(p, n, q, m, i);
            StrB s = strb_begin(c);
            strb_bytes(s, p + i, end - i);
            const Val piece = strb_end(s);
            if (piece.tag == CB_T_ERR) return mk_err();
            encode_elem(c, piece, &c.scratch[off + 1 + k]);
            i = end + (m == 0 ? 0 : m);
        }
        return mk_scratch(CB_T_LIST, off);
    }
    case CB_FN_HIER_AT: {   // hierarchy(s, delim a[2])[a[1]]
        int64_t i;
        if (argc != 3 || !arg_int(a[1], &i) || a[2].tag != CB_T_STRING) return mk_err();
        HierIt it = hier_it(c, a[0].u, (uint32_t)a[2].u);
        uint32_t s0, l0;
        int64_t k = 0;
        while (hier_next(it, &s0, &l0)) {
            if (k++ == i) { StrB s = strb_begin(c); strb_bytes(s, it.p + s0, l0); return strb_end(s); }
        }
        return mk_err();   // index out of range
    }
    default: c.unsupported = 1; return mk_err();
    }
}

// list functions: cel-go ext.Lists (sort, slice, flatten, reverse, distinct, lists.range) and Cerbos except / intersect
CB_HD_NOINLINE Val dyn_listfn(Ctx &c, uint32_t fn, const Val *a, uint32_t argc) {
    for (uint32_t i = 0; i < argc; i++) if (a[i].tag == CB_T_ERR) return mk_err();
    uint32_t off;
    if (fn == CB_FN_RANGE) {
        int64_t n;
        if (!arg_int(a[0], &n)) return mk_err();
        if (n < 0) n = 0;
        if (n > CB_SCRATCH_WORDS) { c.unsupported = 1; return mk_err(); }
        if (!list_new(c, (uint32_t)n, &off)) return mk_err();
        for (int64_t i = 0; i < n; i++) encode_elem(c, mk_int(i), &c.scratch[off + 1 + i]);
        return mk_scratch(CB_T_LIST, off);
    }
    if (a[0].tag != CB_T_LIST) return mk_err();
    const LView x = lview(c, a[0]);
    switch (fn) {
    case CB_FN_EXCEPT: case CB_FN_INTERSECT: {
        if (argc != 2 || a[1].tag != CB_T_LIST) return mk_err();
        Val la = a[0], lb = a[1];
        if (fn == CB_FN_INTERSECT && x.n > lview(c, lb).n) { la = a[1]; lb = a[0]; }   // cerbos_lib.go:433-470: probe the larger list
        const LView xa = lview(c, la);
        const bool gm = uses_go_map(c, lb);
        if (!list_new(c, xa.n, &off)) return mk_err();
        uint32_t k = 0;
        for (uint32_t i = 0; i < xa.n; i++) {
            const uint64_t w = ldg(xa.p + i);
            if (list_member(c, gm, lb, decode_elem(w)) == (fn == CB_FN_INTERSECT)) c.scratch[off + 1 + k++] = w;
        }
        c.scratch[off] = k;
        return mk_scratch(CB_T_LIST, off);
    }
    case CB_FN_REVERSE: {
        if (!list_new(c, x.n, &off)) return mk_err();
        for (uint32_t i = 0; i < x.n; i++) c.scratch[off + 1 + i] = ldg(x.p + (x.n - 1 - i));
        return mk_scratch(CB_T_LIST, off);
    }
    case CB_FN_SLICE: {
        int64_t s0, e0;
        if (argc != 3 || !arg_int(a[1], &s0) || !arg_int(a[2], &e0)) return mk_err();
        if (s0 < 0 || e0 < 0 || s0 > e0 || e0 > (int64_t)x.n) return mk_err();
        if (!list_new(c, (uint32_t)(e0 - s0), &off)) return mk_err();
        for (int64_t i = s0; i < e0; i++) c.scratch[off + 1 + (i - s0)] = ldg(x.p + i);
        return mk_scratch(CB_T_LIST, off);
    }
    case CB_FN_FLATTEN: {
        int64_t depth = 1;
        if (argc == 2 && !arg_int(a[1], &depth)) return mk_err();
        if (depth < 0) return mk_err();
        if (depth > 1) { c.unsupported = 1; return mk_err(); }
        uint32_t total = 0;
        for (uint32_t i = 0; i < x.n; i++) { const Val e = decode_elem(ldg(x.p + i)); total += (depth && e.tag == CB_T_LIST) ? lview(c, e).n : 1; }
        if (!list_new(c, total, &off)) return mk_err();
        uint32_t k = 0;
        for (uint32_t i = 0; i < x.n; i++) {
            const uint64_t w = ldg(x.p + i);
            const Val e = decode_elem(w);
            if (depth && e.tag == CB_T_LIST) { const LView y = lview(c, e); for (uint32_t j = 0; j < y.n; j++) c.scratch[off + 1 + k++] = ldg(y.p + j); }
            else c.scratch[off + 1 + k++] = w;
        }
        return mk_scratch(CB_T_LIST, off);
    }
    case CB_FN_DISTINCT: {
        if (!list_new(c, x.n, &off)) return mk_err();
        uint32_t k = 0;
        for (uint32_t i = 0; i < x.n; i++) {
            const Val e = decode_elem(ldg(x.p + i));
            bool seen = false;
            for (uint32_t j = 0; j < k && !seen; j++) seen = val_equal(c, e, decode_elem(c.scratch[off + 1 + j]));
            if (!seen) c.scratch[off + 1 + k++] = ldg(x.p + i);
        }
        c.scratch[off] = k;
        return mk_scratch(CB_T_LIST, off);
    }
    case CB_FN_SORT: {
        if (!list_new(c, x.n, &off)) return mk_err();
        if (x.n == 0) return mk_scratch(CB_T_LIST, off);
        const uint32_t t0 = decode_elem(ldg(x.p)).tag;
        if (!(t0 == CB_T_INT || t0 == CB_T_UINT || t0 == CB_T_DOUBLE || t0 == CB_T_BOOL || t0 == CB_T_STRING || t0 == CB_T_TS || t0 == CB_T_DUR)) return mk_err();
        for (uint32_t i = 0; i < x.n; i++) {   // stable insertion sort
            const uint64_t w = ldg(x.p + i);
            const Val e = decode_elem(w);
            if (e.tag != t0) return mk_err();   // "list elements must have the same type"
            uint32_t j = i;
            while (j > 0) {
                const int r = val_order(c, decode_elem(c.scratch[off + j]), e);
                if (r == 3) return mk_err();
                if (r <= 0) break;
                c.scratch[off + 1 + j] = c.scratch[off + j];
                j--;
            }
            c.scratch[off + 1 + j] = w;
        }
        return mk_scratch(CB_T_LIST, off);
    }
    default: c.unsupported = 1; return mk_err();
    }
}

// ---- 3-valued && / || with cel-go error absorption ----
CB_HD Val and_or(bool is_or, const Val &a, const Val &b) {
    bool ab = a.tag == CB_T_BOOL, bb = b.tag == CB_T_BOOL;
    uint64_t dom = is_or ? 1 : 0;
    if (ab && a.u == dom) return a;
    if (bb && b.u == dom) return b;
    if (ab && bb) return mk_bool(!is_or);
    return mk_err();
}

CB_HD Val load_slot(const Ctx &c, uint32_t s, int *state) {
    return decode_v64(ldcol64(c.b->slots + (uint64_t)s * c.b->stride + c.req), state);
}
CB_HD Val load_const(const Ctx &c, uint32_t k) {
    const cb_const *p = c.t->consts() + k;
    return mk(ldg(&p->tag), ldg(&p->bits));
}

struct Loop {
    Val range;
    uint64_t i, n;
    uint32_t any_err;
    int64_t count;
    uint32_t out;      // collecting comprehensions (map / filter / transform*): result under construction in the arena
};

CB_HD void loop_bind(Ctx &c, const Loop &L, int var, bool two) {
    const uint64_t *p = heap_ptr(c, L.range.u);
    if (L.range.tag == CB_T_LIST) {
        Val e = decode_elem(ldg(p + 1 + L.i));
        if (two) { c.vars[var] = mk_int((int64_t)L.i); c.vars[var + 1] = e; } else c.vars[var] = e;
    } else {
        Val k = decode_elem(ldg(p + 1 + L.i));
        if (two) { c.vars[var] = k; c.vars[var + 1] = decode_elem(ldg(p + 1 + L.n + L.i)); } else c.vars[var] = k;
    }
}

// ---- SPIFFE ids and trust domains (conditions/types/spiffe.go over go-spiffe's spiffeid package) ------------------------
// A SPIFFE id is its validated string (tag CB_T_SPIFFE_ID, payload = the string reference), a trust domain its name (tag
// CB_T_SPIFFE_TD); a matcher never exists as a value: spiffeMatchX(arg).matchesID(x) is one fused function.
CB_HD bool spiffe_td_char(uint8_t ch) { return (ch >= 'a' && ch <= 'z') || (ch >= '0' && ch <= '9') || ch == '-' || ch == '.' || ch == '_'; }
CB_HD bool spiffe_seg_char(uint8_t ch) { return spiffe_td_char(ch) || (ch >= 'A' && ch <= 'Z'); }
// spiffeid.FromString: "spiffe://" + trust domain (lower case, digits, - . _; not empty) + path of non-empty segments
// (letters, digits, - . _; no "." / ".." segment, no trailing slash).  *pathidx = where the path starts.
CB_HD_NOINLINE bool spiffe_parse_id(const uint8_t *p, uint32_t n, uint32_t *pathidx) {
    const uint8_t pre[9] = {'s', 'p', 'i', 'f', 'f', 'e', ':', '/', '/'};
    if (n < 9) return false;
    for (uint32_t i = 0; i < 9; i++) if (ldg(p + i) != pre[i]) return false;
    uint32_t i = 9;
    while (i < n && ldg(p + i) != '/') { if (!spiffe_td_char(ldg(p + i))) return false; i++; }
    if (i == 9) return false;
    *pathidx = i;
    uint32_t seg = i + 1;
    for (uint32_t k = i + 1; k <= n && i < n; k++) {
        if (k == n || ldg(p + k) == '/') {
            const uint32_t len = k - seg;
            if (len == 0) return false;
            if (len == 1 && ldg(p + seg) == '.') return false;
            if (len == 2 && ldg(p + seg) == '.' && ldg(p + seg + 1) == '.') return false;
            seg = k + 1;
        } else if (!spiffe_seg_char(ldg(p + k))) return false;
    }
    return true;
}
// bytes [from, to) of string `ref` as a string of its own (the whole string: the reference itself)
CB_HD Val spiffe_substr(Ctx &c, uint64_t ref, const uint8_t *p, uint32_t n, uint32_t from, uint32_t to) {
    if (from == 0 && to == n) return mk(CB_T_STRING, ref);
    StrB s = strb_begin(c);
    strb_bytes(s, p + from, to - from);
    return strb_end(s);
}
// spiffeid.TrustDomainFromString: an id (anything containing ":/") gives its trust domain, else the text must be a name
CB_HD_NOINLINE Val spiffe_td_from_string(Ctx &c, uint64_t ref) {
    const uint8_t *p; uint32_t n;
    str_get(c, ref, p, n);
    if (n == 0) return mk_err();
    bool looks_like_id = false;
    for (uint32_t i = 0; i + 1 < n; i++) looks_like_id |= ldg(p + i) == ':' && ldg(p + i + 1) == '/';
    if (looks_like_id) {
        uint32_t px;
        if (!spiffe_parse_id(p, n, &px)) return mk_err();
        Val v = spiffe_substr(c, ref, p, n, 9, px);
        if (v.tag == CB_T_STRING) v.tag = CB_T_SPIFFE_TD;
        return v;
    }
    for (uint32_t i = 0; i < n; i++) if (!spiffe_td_char(ldg(p + i))) return mk_err();
    return mk(CB_T_SPIFFE_TD, ref);
}
CB_HD Val spiffe_id_of(Ctx &c, const Val &v) {   // spiffeID(string | id); also how matchesID takes its argument
    if (v.tag == CB_T_SPIFFE_ID) return v;
    if (v.tag != CB_T_STRING) return mk_err();
    const uint8_t *p; uint32_t n, px;
    str_get(c, v.u, p, n);
    return spiffe_parse_id(p, n, &px) ? mk(CB_T_SPIFFE_ID, v.u) : mk_err();
}
CB_HD Val spiffe_td_of_id(Ctx &c, const Val &id) {
    const uint8_t *p; uint32_t n, px = 9;
    str_get(c, id.u, p, n);
    spiffe_parse_id(p, n, &px);
    Val v = spiffe_substr(c, id.u, p, n, 9, px);
    if (v.tag == CB_T_STRING) v.tag = CB_T_SPIFFE_TD;
    return v;
}
CB_HD Val spiffe_td_of(Ctx &c, const Val &v) {   // spiffeTrustDomain(string | id | trust domain); spiffeMatchTrustDomain's argument
    if (v.tag == CB_T_SPIFFE_TD) return v;
    if (v.tag == CB_T_SPIFFE_ID) return spiffe_td_of_id(c, v);
    if (v.tag == CB_T_STRING) return spiffe_td_from_string(c, v.u);
    return mk_err();
}
CB_HD_NOINLINE Val spiffe_fn(Ctx &c, uint32_t fn, const Val *a, uint32_t argc) {
    for (uint32_t i = 0; i < argc; i++) if (a[i].tag == CB_T_ERR) return mk_err();
    switch (fn) {
    case CB_FN_SPIFFE_ID: return spiffe_id_of(c, a[0]);
    case CB_FN_SPIFFE_IDSTR: { Val v = spiffe_id_of(c, a[0]); if (v.tag == CB_T_SPIFFE_ID) v.tag = CB_T_STRING; return v; }
    case CB_FN_SPIFFE_TD: return spiffe_td_of(c, a[0]);
    case CB_FN_SPIFFE_TD_OF: return a[0].tag == CB_T_SPIFFE_ID ? spiffe_td_of_id(c, a[0]) : mk_err();
    case CB_FN_SPIFFE_PATH: {
        if (a[0].tag != CB_T_SPIFFE_ID) return mk_err();
        const uint8_t *p; uint32_t n, px = 0;
        str_get(c, a[0].u, p, n);
        spiffe_parse_id(p, n, &px);
        if (px == n) { StrB s = strb_begin(c); return strb_end(s); }   // no path: the empty string
        return spiffe_substr(c, a[0].u, p, n, px, n);
    }
    case CB_FN_SPIFFE_MEMBER: {
        if (a[0].tag != CB_T_SPIFFE_ID || a[1].tag != CB_T_SPIFFE_TD) return mk_err();
        const Val td = spiffe_td_of_id(c, a[0]);
        return td.tag == CB_T_SPIFFE_TD ? mk_bool(str_equal(c, td.u, a[1].u)) : mk_err();
    }
    case CB_FN_SPIFFE_TD_NAME: return a[0].tag == CB_T_SPIFFE_TD ? mk(CB_T_STRING, a[0].u) : mk_err();
    case CB_FN_SPIFFE_TD_ID: {      // "spiffe://" + name; id(x) of any other value is x (cerbos_lib.go)
        if (a[0].tag != CB_T_SPIFFE_TD) return a[0];
        const uint8_t pre[9] = {'s', 'p', 'i', 'f', 'f', 'e', ':', '/', '/'};
        const uint8_t *p; uint32_t n;
        str_get(c, a[0].u, p, n);
        StrB s = strb_begin(c);
        for (uint32_t i = 0; i < 9; i++) strb_put(s, pre[i]);
        strb_bytes(s, p, n);
        return strb_end(s);
    }
    case CB_FN_SPIFFE_MATCH_ANY: return spiffe_id_of(c, a[0]).tag == CB_T_SPIFFE_ID ? mk_bool(true) : mk_err();
    case CB_FN_SPIFFE_MATCH_EXACT: {
        const Val want = spiffe_id_of(c, a[0]), got = spiffe_id_of(c, a[1]);
        if (want.tag != CB_T_SPIFFE_ID || got.tag != CB_T_SPIFFE_ID) return mk_err();
        return mk_bool(str_equal(c, want.u, got.u));
    }
    case CB_FN_SPIFFE_MATCH_ONEOF: {   // every element must be (the string of) a valid id, else no such overload
        if (a[0].tag != CB_T_LIST) return mk_err();
        const LView l = lview(c, a[0]);
        for (uint32_t i = 0; i < l.n; i++) if (spiffe_id_of(c, decode_elem(ldg(l.p + i))).tag != CB_T_SPIFFE_ID) return mk_err();
        const Val got = spiffe_id_of(c, a[1]);
        if (got.tag != CB_T_SPIFFE_ID) return mk_err();
        bool found = false;
        for (uint32_t i = 0; i < l.n; i++) found |= str_equal(c, decode_elem(ldg(l.p + i)).u, got.u);
        return mk_bool(found);
    }
    case CB_FN_SPIFFE_MATCH_TD: {
        const Val td = spiffe_td_of(c, a[0]);
        if (td.tag != CB_T_SPIFFE_TD || a[0].tag == CB_T_SPIFFE_ID) return mk_err();   // (an id is no argument of spiffeMatchTrustDomain)
        const Val got = spiffe_id_of(c, a[1]);
        if (got.tag != CB_T_SPIFFE_ID) return mk_err();
        const Val gtd = spiffe_td_of_id(c, got);
        return gtd.tag == CB_T_SPIFFE_TD ? mk_bool(str_equal(c, gtd.u, td.u)) : mk_err();
    }
    default: c.unsupported = 1; return mk_err();
    }
}
// `==` with a SPIFFE value on the left (spiffe.go:346-360, 443-461); 0 false, 1 true, 2 no such overload
CB_HD_NOINLINE int spiffe_equal(Ctx &c, const Val &a, const Val &b) {
    if (a.tag == CB_T_SPIFFE_ID) {
        if (b.tag == CB_T_SPIFFE_ID || b.tag == CB_T_STRING) return str_equal(c, a.u, b.u) ? 1 : 0;
        return 2;
    }
    if (b.tag == CB_T_SPIFFE_TD) return str_equal(c, a.u, b.u) ? 1 : 0;
    if (b.tag == CB_T_STRING) {   // a string that is no trust domain is simply unequal
        const Val t = spiffe_td_from_string(c, b.u);
        return t.tag == CB_T_SPIFFE_TD && str_equal(c, a.u, t.u) ? 1 : 0;
    }
    return 2;
}

// ---- single-instruction bodies: shared by the interpreter below and by the straight-line code that
// cb_specialize.h (generate_uc) emits from a condition's program for the run-time specialised kernels
CB_HD Val op_select(Ctx &c, const Val &m, uint32_t key) { Val o; return (m.tag == CB_T_MAP && map_find(c, m, mk(CB_T_STRING, key), &o)) ? o : mk_err(); }
CB_HD Val op_has(Ctx &c, const Val &m, uint32_t key) { return m.tag == CB_T_MAP ? mk_bool(map_find(c, m, mk(CB_T_STRING, key), nullptr)) : mk_err(); }
CB_HD Val op_has_slot(int s) { return s == SLOT_ERROR ? mk_err() : mk_bool(s == SLOT_VALUE); }
CB_HD Val op_neg(const Val &v) {
    const int64_t kMin = (int64_t)0x8000000000000000ull;
    if (v.tag == CB_T_INT) return (int64_t)v.u == kMin ? mk_err() : mk_int(-(int64_t)v.u);
    if (v.tag == CB_T_DOUBLE) return mk_double(-u2d(v.u));
    if (v.tag == CB_T_DUR) return (int64_t)v.u == kMin ? mk_err() : mk(CB_T_DUR, (uint64_t)(-(int64_t)v.u));
    return mk_err();
}
CB_HD Val op_not(const Val &v) { return v.tag == CB_T_BOOL ? mk_bool(!v.u) : mk_err(); }
CB_HD Val op_size(Ctx &c, const Val &v) {
    if (v.tag == CB_T_STRING) { const uint8_t *p; uint32_t n; str_get(c, v.u, p, n); return mk_int(utf8_len(p, n)); }
    if (v.tag == CB_T_BYTES) { const uint8_t *p; uint32_t n; str_get(c, v.u, p, n); return mk_int(n); }
    if (is_container(v)) return mk_int((int64_t)ldg(heap_ptr(c, v.u)));
    return mk_err();
}
CB_HD Val op_double(Ctx &c, const Val &v) {
    if (v.tag == CB_T_INT) return mk_double((double)(int64_t)v.u);
    if (v.tag == CB_T_UINT) return mk_double((double)v.u);
    if (v.tag == CB_T_STRING) { c.unsupported = 1; return mk_err(); }  // strconv.ParseFloat at run time
    if (v.tag != CB_T_DOUBLE) return mk_err();
    return v;
}
CB_HD Val op_timestamp(Ctx &c, const Val &v) {
    if (v.tag == CB_T_TS) return v;
    if (v.tag == CB_T_STRING) return parse_ts(c, v);
    if (v.tag == CB_T_INT) {
        int64_t s = (int64_t)v.u, ns;
        if (s < -62135596800ll || s > 253402300799ll) return mk_err();
        if (mul_ovf(s, 1000000000ll, &ns)) { c.unsupported = 1; return mk_err(); }
        return mk(CB_T_TS, (uint64_t)ns);
    }
    return mk_err();
}
CB_HD Val op_duration(Ctx &c, const Val &v) {
    if (v.tag == CB_T_DUR) return v;
    if (v.tag == CB_T_INT) return mk(CB_T_DUR, v.u);
    if (v.tag == CB_T_STRING) {
        const uint8_t *p; uint32_t n; int64_t ns = 0;
        str_get(c, v.u, p, n);
        const int rc = parse_duration_text(p, n, &ns);
        if (rc == 2) c.unsupported = 1;
        return rc == 0 ? mk(CB_T_DUR, (uint64_t)ns) : mk_err();
    }
    return mk_err();
}
CB_HD Val op_hier_rel(Ctx &c, uint32_t rel, uint32_t da, uint32_t db, const Val &a, const Val &b) {
    const bool ok = hier_operand(c, a) & hier_operand(c, b);
    return ok ? mk_bool(hier_rel(rel, hier_it(c, a.u, da), hier_it(c, b.u, db))) : mk_err();
}
CB_HD Val op_ts_get(Ctx &c, const Val &v, uint32_t ia, uint32_t ib, uint32_t ic) {
    int32_t off_s = (int32_t)ic;
    if (ib == 2 && v.tag == CB_T_TS) {
        // IANA zone: the offset in force at this instant, from the zone's transition table (bytecode.iana_zone_words)
        const uint64_t *z = c.t->theap() + ic;
        const int64_t sec = floor_div((int64_t)v.u, 1000000000ll);
        const uint64_t nz = ldg(z);
        if (sec < (int64_t)ldg(z + 1) || sec >= (int64_t)ldg(z + 2)) { c.unsupported = 1; return mk_err(); }
        uint64_t lo = 0, hi = nz;          // last entry whose start <= sec
        while (hi - lo > 1) { const uint64_t mid = (lo + hi) / 2; if ((int64_t)ldg(z + 3 + 2 * mid) <= sec) lo = mid; else hi = mid; }
        off_s = (int32_t)(int64_t)ldg(z + 3 + 2 * lo + 1);
    }
    return do_ts_get(ia, v, ib, off_s);
}
CB_HD Val op_in_split(Ctx &c, const Val &x, const Val &sv, uint32_t delim) {   // x in s.split(delim)
    if (x.tag == CB_T_ERR || sv.tag != CB_T_STRING) return mk_err();
    bool found = false;
    if (x.tag == CB_T_STRING) {
        const uint8_t *px; uint32_t lx, s0, l0;
        str_get(c, x.u, px, lx);
        HierIt it = hier_it(c, sv.u, delim);
        while (hier_next(it, &s0, &l0)) found |= l0 == lx && bytes_eq(it.p + s0, px, lx);
    }
    return mk_bool(found);
}
CB_HD Val op_hier_size(Ctx &c, const Val &v, uint32_t delim) { return hier_operand(c, v) ? mk_int((int64_t)hier_count(hier_it(c, v.u, delim))) : mk_err(); }
CB_HD Val op_hier_ca2(Ctx &c, const Val &a, const Val &b, uint32_t ib, uint32_t ic) {
    const bool ok = hier_operand(c, a) & hier_operand(c, b);
    return ok ? mk_int((int64_t)hier_ca_size(hier_it(c, a.u, ib), hier_it(c, b.u, ic & 0xFFFF))) : mk_err();
}
CB_HD Val op_hier_ca3(Ctx &c, const Val &a0, const Val &b0, const Val &z0, uint32_t ib, uint32_t ic) {
    const bool ok = hier_operand(c, a0) & hier_operand(c, b0) & hier_operand(c, z0);
    if (!ok) return mk_err();
    const HierIt a = hier_it(c, a0.u, ib), b2 = hier_it(c, b0.u, ic & 0xFFFF), z = hier_it(c, z0.u, ic >> 16);
    const uint32_t k = hier_ca_size(a, b2);
    return mk_bool(hier_count(z) == k && hier_common(a, z, k) == k);
}
// cel-go ext.Math (ext/math.go).  greatest / least: one number is itself, one list gives its extreme, several arguments theirs;
// numbers of different types compare by value (num_cmp), the winner keeps its type, ties keep the earlier one, a NaN cannot
// be ordered (error).  ceil / floor / round / trunc / isNaN / isInf / isFinite take doubles only; the bit operations take
// (int, int) or (uint, uint); shifts by 64 or more give 0, a negative count is an error, >> on an int is a logical shift.
CB_HD bool math_pick(Val &best, bool &have, const Val &v, bool greater) {
    if (!is_num(v)) return false;
    if (!have) { best = v; have = true; return true; }
    const int r = num_cmp(v, best);
    if (r == 2) return false;
    if (greater ? r > 0 : r < 0) best = v;
    return true;
}
CB_HD_NOINLINE Val math_fn(Ctx &c, uint32_t fn, const Val *a, uint32_t argc) {
    if (fn >= CB_FN_QUOTE) return fmt_fn(c, fn, a, argc);   // the ids after the ext.Math block that op_fn does not take itself
    const int64_t kMin = (int64_t)0x8000000000000000ull;
    if (fn == CB_FN_MATH_GREATEST || fn == CB_FN_MATH_LEAST) {
        const bool greater = fn == CB_FN_MATH_GREATEST;
        Val best = mk_err();
        bool have = false;
        if (argc == 1) {
            if (is_num(a[0])) return a[0];
            if (a[0].tag != CB_T_LIST) return mk_err();
            const uint64_t *h = heap_ptr(c, a[0].u);
            const uint32_t n = (uint32_t)ldg(h);
            for (uint32_t i = 0; i < n; i++)
                if (!math_pick(best, have, decode_elem(ldg(h + 1 + i)), greater)) return mk_err();
            return best;          // (an empty list: error)
        }
        for (uint32_t i = 0; i < argc; i++)
            if (!math_pick(best, have, a[i], greater)) return mk_err();
        return best;
    }
    const Val &x = a[0];
    switch (fn) {
    case CB_FN_MATH_CEIL: case CB_FN_MATH_FLOOR: case CB_FN_MATH_ROUND: case CB_FN_MATH_TRUNC: {
        if (argc != 1 || x.tag != CB_T_DOUBLE) return mk_err();
        const double d = u2d(x.u);
        return mk_double(fn == CB_FN_MATH_CEIL ? ceil(d) : fn == CB_FN_MATH_FLOOR ? floor(d) : fn == CB_FN_MATH_ROUND ? round(d) : trunc(d));
    }
    case CB_FN_MATH_ABS:
        if (argc != 1) return mk_err();
        if (x.tag == CB_T_INT) return (int64_t)x.u == kMin ? mk_err() : mk_int((int64_t)x.u < 0 ? -(int64_t)x.u : (int64_t)x.u);
        if (x.tag == CB_T_UINT) return x;
        if (x.tag == CB_T_DOUBLE) return mk_double(fabs(u2d(x.u)));
        return mk_err();
    case CB_FN_MATH_SIGN:
        if (argc != 1) return mk_err();
        if (x.tag == CB_T_INT) return mk_int(((int64_t)x.u > 0) - ((int64_t)x.u < 0));
        if (x.tag == CB_T_UINT) return mk(CB_T_UINT, x.u ? 1u : 0u);
        if (x.tag == CB_T_DOUBLE) { const double d = u2d(x.u); return mk_double(d != d ? d : d > 0 ? 1.0 : d < 0 ? -1.0 : 0.0); }
        return mk_err();
    case CB_FN_MATH_ISNAN: case CB_FN_MATH_ISINF: case CB_FN_MATH_ISFINITE: {
        if (argc != 1 || x.tag != CB_T_DOUBLE) return mk_err();
        const double d = u2d(x.u);
        const bool nan = d != d, inf = !nan && (d - d) != (d - d);      // (inf - inf is NaN)
        return mk_bool(fn == CB_FN_MATH_ISNAN ? nan : fn == CB_FN_MATH_ISINF ? inf : !nan && !inf);
    }
    case CB_FN_MATH_BITAND: case CB_FN_MATH_BITOR: case CB_FN_MATH_BITXOR: {
        if (argc != 2 || a[0].tag != a[1].tag || (x.tag != CB_T_INT && x.tag != CB_T_UINT)) return mk_err();
        const uint64_t y = a[1].u;
        return mk(x.tag, fn == CB_FN_MATH_BITAND ? x.u & y : fn == CB_FN_MATH_BITOR ? x.u | y : x.u ^ y);
    }
    case CB_FN_MATH_BITNOT:
        if (argc != 1 || (x.tag != CB_T_INT && x.tag != CB_T_UINT)) return mk_err();
        return mk(x.tag, ~x.u);
    case CB_FN_MATH_SHL: case CB_FN_MATH_SHR: {
        if (argc != 2 || a[1].tag != CB_T_INT || (x.tag != CB_T_INT && x.tag != CB_T_UINT)) return mk_err();
        const int64_t k = (int64_t)a[1].u;
        if (k < 0) return mk_err();
        if (k > 63) return mk(x.tag, 0);
        return mk(x.tag, fn == CB_FN_MATH_SHL ? x.u << k : x.u >> k);
    }
    case CB_FN_MATH_SQRT: {
        if (argc != 1 || !is_num(x)) return mk_err();
        const double d = x.tag == CB_T_DOUBLE ? u2d(x.u) : x.tag == CB_T_INT ? (double)(int64_t)x.u : (double)x.u;
        return mk_double(sqrt(d));      // (a negative number: NaN)
    }
    }
    return mk_err();
}
CB_HD Val op_fn(Ctx &c, uint32_t fn, uint32_t argc, Val *a) {   // a[0..argc): arguments (target first)
    if (fn == CB_FN_TO_STRING || fn == CB_FN_TO_BOOL || fn == CB_FN_TYPE_OF) return dyn_strfn(c, fn, a, argc);
    if (fn >= CB_FN_MATH_GREATEST) return math_fn(c, fn, a, argc);
    if (fn >= CB_FN_SPIFFE_ID) return spiffe_fn(c, fn, a, argc);
    if (fn == CB_FN_REVERSE && a[0].tag == CB_T_STRING) return dyn_strfn(c, CB_FN_STR_REVERSE, a, argc);
    return fn >= CB_FN_EXCEPT ? dyn_listfn(c, fn, a, argc) : dyn_strfn(c, fn, a, argc);
}
CB_HD Val op_matches(Ctx &c, const Val &v, uint32_t ic) {   // RE2 search by the DFA table at theap[ic]: text = BOT, bytes, EOT (cel/regex_dfa.py)
    if (v.tag != CB_T_STRING) return mk_err();
    const uint64_t *d = c.t->theap() + ic;
    const uint64_t h = ldg(d);
    const uint32_t ns = (uint32_t)(h & 0xFFFF), nc = (uint32_t)((h >> 16) & 0xFFFF);
    uint32_t state = (uint32_t)(h >> 32) & 0xFFFF;
    const uint8_t *cm = reinterpret_cast<const uint8_t *>(d + 1);
    const uint64_t *acc = d + 1 + 33, *tr = acc + (ns + 63) / 64;
    const uint8_t *p; uint32_t n;
    str_get(c, v.u, p, n);
    for (uint32_t i = 0; i < n + 2; i++) {
        const uint32_t sym = i == 0 ? 256u : i == n + 1 ? 257u : (uint32_t)ldg(p + i - 1);
        const uint32_t q = state * nc + ldg(cm + sym);
        state = (uint32_t)(ldg(tr + (q >> 2)) >> (16 * (q & 3))) & 0xFFFFu;
    }
    return mk_bool((ldg(acc + (state >> 6)) >> (state & 63)) & 1);
}
// Quantifier comprehensions (all / exists / exists_one).  qloop_init: true = entered, the first element is bound;
// false = *res is the comprehension's value.  qloop_next (r = the body's value): true = finished with *res,
// false = the next element is bound.
CB_HD bool qloop_init(Ctx &c, Loop &L, const Val &r, int kind, bool two, int var, Val *res) {
    if (!is_container(r)) { *res = mk_err(); return false; }
    L.range = r; L.i = 0; L.n = ldg(heap_ptr(c, r.u)); L.any_err = 0; L.count = 0; L.out = 0;
    if (L.n == 0) { *res = mk_bool(kind == CB_LOOP_ALL); return false; }
    loop_bind(c, L, var, two);
    return true;
}
CB_HD bool qloop_next(Ctx &c, Loop &L, const Val &r, int kind, bool two, int var, Val *res) {
    bool done = false;
    *res = mk_err();
    if (kind == CB_LOOP_EXISTS_ONE) {
        if (r.tag != CB_T_BOOL) L.any_err = 1; else if (r.u) L.count++;
    } else {
        uint64_t dom = kind == CB_LOOP_EXISTS ? 1 : 0;
        if (r.tag == CB_T_BOOL) { if (r.u == dom) { done = true; *res = mk_bool(dom != 0); } }
        else L.any_err = 1;
    }
    L.i++;
    if (!done && L.i >= L.n) {
        done = true;
        if (L.any_err) *res = mk_err();
        else if (kind == CB_LOOP_EXISTS_ONE) *res = mk_bool(L.count == 1);
        else *res = mk_bool(kind == CB_LOOP_ALL);
    }
    if (!done) loop_bind(c, L, var, two);
    return done;
}
CB_HD bool cond_true(const Val &v) { return v.tag == CB_T_BOOL && v.u == 1; }

#endif  // !CB_LEAN_ONLY || CB_SPEC_PROGRAMS

#ifndef CB_LEAN_ONLY   // the stack interpreter
// Runs one condition program; returns true iff it yields BOOL true (ruletable.go:1425-1441).
CB_HD_NOINLINE bool run_program(Ctx &c, const cb_instr *code) {
    Val st[CB_MAX_STACK + 1];
    Loop loops[CB_MAX_LOOP_DEPTH];
    int sp = 0, ld = 0;
    uint32_t pc = 0;
    for (;;) {
        // one 8-byte instruction fetch
        uint64_t raw = ldg(reinterpret_cast<const uint64_t *>(code + pc));
        pc++;
        uint32_t op = (uint32_t)(raw & 0xFF), ia = (uint32_t)((raw >> 8) & 0xFF), ib = (uint32_t)((raw >> 16) & 0xFFFF);
        uint32_t ic = (uint32_t)(raw >> 32);
        switch (op) {
        case CB_OP_RET: return cond_true(st[sp - 1]);
        case CB_OP_CONST: st[sp++] = load_const(c, ic); break;
        case CB_OP_SLOT: { int s; st[sp++] = load_slot(c, ic, &s); break; }
        case CB_OP_HAS_SLOT: { int s; load_slot(c, ic, &s); st[sp++] = op_has_slot(s); break; }
        case CB_OP_PID: st[sp++] = mk(CB_T_STRING, c.pid); break;
        case CB_OP_NOW: st[sp++] = mk(CB_T_TS, (uint64_t)c.b->now); break;
        case CB_OP_VAR: st[sp++] = c.vars[ia]; break;
        case CB_OP_SELECT: st[sp - 1] = op_select(c, st[sp - 1], ic); break;
        case CB_OP_HAS: st[sp - 1] = op_has(c, st[sp - 1], ic); break;
        case CB_OP_INDEX: sp--; st[sp - 1] = do_index(c, st[sp - 1], st[sp]); break;
        case CB_OP_EQ: case CB_OP_NE: case CB_OP_LT: case CB_OP_LE: case CB_OP_GT: case CB_OP_GE:
            sp--; st[sp - 1] = do_cmp(c, (int)op - CB_OP_EQ, st[sp - 1], st[sp]); break;
        case CB_OP_ADD: case CB_OP_SUB: case CB_OP_MUL: case CB_OP_DIV: case CB_OP_MOD:
            sp--; st[sp - 1] = do_arith(c, (int)op, st[sp - 1], st[sp]); break;
        case CB_OP_NEG: st[sp - 1] = op_neg(st[sp - 1]); break;
        case CB_OP_NOT: st[sp - 1] = op_not(st[sp - 1]); break;
        case CB_OP_IN: sp--; st[sp - 1] = do_in(c, st[sp - 1], st[sp]); break;
        case CB_OP_SIZE: st[sp - 1] = op_size(c, st[sp - 1]); break;
        case CB_OP_STARTS_WITH: case CB_OP_ENDS_WITH: case CB_OP_CONTAINS:
            sp--; st[sp - 1] = do_str2(c, (int)op, st[sp - 1], st[sp]); break;
        case CB_OP_JF_KEEP: if (st[sp - 1].tag == CB_T_BOOL && st[sp - 1].u == 0) pc = ic; break;
        case CB_OP_JT_KEEP: if (st[sp - 1].tag == CB_T_BOOL && st[sp - 1].u == 1) pc = ic; break;
        case CB_OP_AND: sp--; st[sp - 1] = and_or(false, st[sp - 1], st[sp]); break;
        case CB_OP_OR: sp--; st[sp - 1] = and_or(true, st[sp - 1], st[sp]); break;
        case CB_OP_JMP: pc = ic; break;
        case CB_OP_TERN: {
            Val v = st[--sp];
            if (v.tag == CB_T_BOOL) { if (!v.u) pc = ic; }
            else { st[sp++] = mk_err(); pc = ib; }
            break;
        }
        case CB_OP_HAS_INTERSECTION: sp--; st[sp - 1] = do_set_pred(c, false, st[sp - 1], st[sp]); break;
        case CB_OP_IS_SUBSET: sp--; st[sp - 1] = do_set_pred(c, true, st[sp - 1], st[sp]); break;
        case CB_OP_LOOP_INIT: {
            Val r = st[--sp];
            int kind = (int)(ib & 0xFF);
            bool two = (ib >> 8) & 1;
            if (!is_container(r)) { st[sp++] = mk_err(); pc = ic; break; }
            Loop &L = loops[ld];
            L.range = r; L.i = 0; L.n = ldg(heap_ptr(c, r.u)); L.any_err = 0; L.count = 0; L.out = 0;
            if (kind >= CB_LOOP_MAP) {
                // result capacity: one element (map entry) per iteration; a list is [n, e...], a map [n, keys..., values...]
                if (L.n > CB_SCRATCH_WORDS) { c.unsupported = 1; st[sp++] = mk_err(); pc = ic; break; }
                const bool is_map = kind == CB_LOOP_TMAP || kind == CB_LOOP_TENTRY || kind == CB_LOOP_SORTBY;   // sortBy: elements + their keys
                if (kind == CB_LOOP_SORTBY && r.tag != CB_T_LIST) { st[sp++] = mk_err(); pc = ic; break; }
                if (!scr_alloc(c, 1 + (uint32_t)L.n * (is_map ? 2u : 1u), &L.out)) { st[sp++] = mk_err(); pc = ic; break; }
                c.scratch[L.out] = 0;
                if (L.n == 0) { st[sp++] = mk_scratch(is_map && kind != CB_LOOP_SORTBY ? CB_T_MAP : CB_T_LIST, L.out); pc = ic; break; }
            } else if (L.n == 0) { st[sp++] = mk_bool(kind == CB_LOOP_ALL); pc = ic; break; }
            ld++;
            loop_bind(c, L, (int)ia, two);
            break;
        }
        case CB_OP_LOOP_NEXT: {
            Val r = st[--sp];
            int kind = (int)(ib & 0xFF);
            bool two = (ib >> 8) & 1;
            Loop &L = loops[ld - 1];
            bool done = false;
            Val res = mk_err();
            if (kind >= CB_LOOP_MAP) {
                // an erroring body (or predicate) makes the whole comprehension an error; CB_T_SKIP = filtered out
                const uint32_t cap = (uint32_t)L.n;
                if (r.tag == CB_T_ERR) { done = true; }
                else if (r.tag != CB_T_SKIP) {
                    uint64_t w = 0;
                    if (kind == CB_LOOP_MAP) {
                        if (!encode_elem(c, r, &w)) done = true; else c.scratch[L.out + 1 + L.count++] = w;
                    } else if (kind == CB_LOOP_FILTER) {
                        if (r.tag != CB_T_BOOL) done = true;
                        else if (r.u) { if (!encode_elem(c, c.vars[ia], &w)) done = true; else c.scratch[L.out + 1 + L.count++] = w; }
                    } else if (kind == CB_LOOP_SORTBY) {    // insert the element where its key belongs (stable): elements at [1..], keys `cap` behind
                        uint64_t ew = 0;
                        const uint32_t t0 = L.count ? decode_elem(c.scratch[L.out + 1 + cap]).tag : r.tag;
                        const bool cmpable = r.tag == CB_T_INT || r.tag == CB_T_UINT || r.tag == CB_T_DOUBLE || r.tag == CB_T_BOOL || r.tag == CB_T_STRING;
                        if (!cmpable || r.tag != t0 || !encode_elem(c, c.vars[ia], &ew) || !encode_elem(c, r, &w)) done = true;
                        else {
                            int64_t j = L.count;
                            while (j > 0 && val_order(c, decode_elem(c.scratch[L.out + cap + j]), r) > 0 && val_order(c, decode_elem(c.scratch[L.out + cap + j]), r) != 3) {
                                c.scratch[L.out + 1 + j] = c.scratch[L.out + j];
                                c.scratch[L.out + 1 + cap + j] = c.scratch[L.out + cap + j];
                                j--;
                            }
                            c.scratch[L.out + 1 + j] = ew;
                            c.scratch[L.out + 1 + cap + j] = w;
                            L.count++;
                        }
                    } else if (kind == CB_LOOP_TMAP) {      // key of this iteration -> body value
                        uint64_t kw = 0;
                        if (!encode_elem(c, c.vars[ia], &kw) || !encode_elem(c, r, &w)) done = true;
                        else { c.scratch[L.out + 1 + L.count] = kw; c.scratch[L.out + 1 + cap + L.count] = w; L.count++; }
                    } else {                                // transformMapEntry: the body yields a map whose entries are merged
                        if (r.tag != CB_T_MAP) done = true;
                        else {
                            const uint64_t *mp = heap_ptr(c, r.u);
                            const uint64_t mn = ldg(mp);
                            for (uint64_t q = 0; q < mn && !done; q++) {
                                const uint64_t kw = ldg(mp + 1 + q), vw = ldg(mp + 1 + mn + q);
                                Val mv = mk_scratch(CB_T_MAP, L.out);
                                // look the key up among the entries merged so far (values sit `cap` words behind the keys)
                                bool dup = false;
                                for (int64_t z = 0; z < L.count && !dup; z++) dup = scalar_equal(c, decode_elem(c.scratch[L.out + 1 + z]), decode_elem(kw));
                                (void)mv;
                                if (dup) done = true;                                   // "insert failed: key already exists"
                                else if ((uint64_t)L.count >= cap) { c.unsupported = 1; done = true; }
                                else { c.scratch[L.out + 1 + L.count] = kw; c.scratch[L.out + 1 + cap + L.count] = vw; L.count++; }
                            }
                        }
                    }
                }
                const bool failed = done;
                L.i++;
                if (!failed && L.i >= L.n) {
                    done = true;
                    const bool is_map = kind == CB_LOOP_TMAP || kind == CB_LOOP_TENTRY;   // (sortBy: the keys behind the elements are simply dropped)
                    if (is_map) for (int64_t z = 0; z < L.count; z++) c.scratch[L.out + 1 + L.count + z] = c.scratch[L.out + 1 + cap + z];   // values right behind the keys
                    c.scratch[L.out] = (uint64_t)L.count;
                    res = mk_scratch(is_map ? CB_T_MAP : CB_T_LIST, L.out);
                }
                if (done) { ld--; st[sp++] = res; }
                else { loop_bind(c, L, (int)ia, two); pc = ic; }
                break;
            }
            if (qloop_next(c, L, r, kind, two, (int)ia, &res)) { ld--; st[sp++] = res; }
            else pc = ic;
            break;
        }
        case CB_OP_TO_COND: { Val v = st[sp - 1]; st[sp - 1] = mk_bool(v.tag == CB_T_BOOL && v.u == 1); break; }
        case CB_OP_COND_NOT: st[sp - 1] = mk_bool(!st[sp - 1].u); break;
        case CB_OP_NOERR: st[sp - 1] = mk_bool(st[sp - 1].tag != CB_T_ERR); break;
        case CB_OP_INT: st[sp - 1] = conv_int(c, st[sp - 1]); break;
        case CB_OP_UINT: st[sp - 1] = conv_uint(c, st[sp - 1]); break;
        case CB_OP_DOUBLE: st[sp - 1] = op_double(c, st[sp - 1]); break;
        case CB_OP_TIMESTAMP: st[sp - 1] = op_timestamp(c, st[sp - 1]); break;
        case CB_OP_DURATION: st[sp - 1] = op_duration(c, st[sp - 1]); break;
        case CB_OP_DYN: break;
        case CB_OP_CMP_SLOT_CONST: { int s; Val a = load_slot(c, ib, &s); st[sp++] = do_cmp(c, (int)ia, a, load_const(c, ic)); break; }
        case CB_OP_CMP_SLOT_SLOT: { int s; Val a = load_slot(c, ib, &s); Val b = load_slot(c, ic, &s); st[sp++] = do_cmp(c, (int)ia, a, b); break; }
        case CB_OP_CMP_SLOT_PID: { int s; Val a = load_slot(c, ib, &s); st[sp++] = do_cmp(c, (int)ia, a, mk(CB_T_STRING, c.pid)); break; }
        case CB_OP_IN_SLOT_CONST: { int s; Val a = load_slot(c, ib, &s); st[sp++] = do_in(c, a, load_const(c, ic)); break; }
        case CB_OP_IN_CONST_SLOT: { int s; Val a = load_slot(c, ib, &s); st[sp++] = do_in(c, load_const(c, ic), a); break; }
        case CB_OP_IN_IP_RANGE: st[sp - 1] = st[sp - 1].tag == CB_T_ERR ? mk_err() : do_in_ip_range(c, st[sp - 1], c.t->theap() + ic); break;
        case CB_OP_HIER_REL: sp--; st[sp - 1] = op_hier_rel(c, ia, ib, ic, st[sp - 1], st[sp]); break;
        case CB_OP_TS_GET: st[sp - 1] = op_ts_get(c, st[sp - 1], ia, ib, ic); break;
        case CB_OP_IN_SPLIT: sp--; st[sp - 1] = op_in_split(c, st[sp - 1], st[sp], ib); break;   // [x, s]: x in s.split(delim ib)
        case CB_OP_HIER_SIZE: st[sp - 1] = op_hier_size(c, st[sp - 1], ib); break;
        case CB_OP_HIER_CA:
            if (ia == 0) { sp--; st[sp - 1] = op_hier_ca2(c, st[sp - 1], st[sp], ib, ic); }
            else { sp -= 2; st[sp - 1] = op_hier_ca3(c, st[sp - 1], st[sp], st[sp + 1], ib, ic); }
            break;
        case CB_OP_FN: sp -= (int)ib - 1; st[sp - 1] = op_fn(c, ia, ib, &st[sp - 1]); break;   // ia = function, ib = argument count
        case CB_OP_MKLIST: {   // ic elements on the stack -> list
            sp -= (int)ic;
            uint32_t off;
            bool ok = list_new(c, ic, &off);
            for (uint32_t q = 0; q < ic && ok; q++) ok = st[sp + q].tag != CB_T_ERR && encode_elem(c, st[sp + q], &c.scratch[off + 1 + q]);
            st[sp++] = ok ? mk_scratch(CB_T_LIST, off) : mk_err();
            break;
        }
        case CB_OP_MKMAP: {    // ic (key, value) pairs on the stack -> map; keys: string / int / double / bool
            sp -= 2 * (int)ic;
            uint32_t off;
            bool ok = scr_alloc(c, 1 + 2 * ic, &off);
            if (ok) c.scratch[off] = ic;
            for (uint32_t q = 0; q < ic && ok; q++) {
                const Val k = st[sp + 2 * q], v = st[sp + 2 * q + 1];
                ok = k.tag != CB_T_ERR && v.tag != CB_T_ERR && !is_container(k) && k.tag != CB_T_NULL &&
                     encode_elem(c, k, &c.scratch[off + 1 + q]) && encode_elem(c, v, &c.scratch[off + 1 + ic + q]);
                for (uint32_t z = 0; z < q && ok; z++) ok = !scalar_equal(c, decode_elem(c.scratch[off + 1 + z]), k);   // repeated key: error
            }
            st[sp++] = ok ? mk_scratch(CB_T_MAP, off) : mk_err();
            break;
        }
        case CB_OP_RUNTIME_EDR: {   // runtime.effectiveDerivedRoles: the names of the set bits, already in sorted order
            uint32_t cnt = 0, off;
            for (uint64_t m = c.edr; m; m &= m - 1) cnt++;
            if (!list_new(c, cnt, &off)) { st[sp++] = mk_err(); break; }
            uint32_t k = 0;
            for (uint32_t bit = 0; bit < 64; bit++)
                if ((c.edr >> bit) & 1) c.scratch[off + 1 + k++] = ((uint64_t)(CB_V64_BOX_BASE | CB_V64_STRING) << 48) | ldg(c.t->dr_name_str() + bit);
            st[sp++] = mk_scratch(CB_T_LIST, off);
            break;
        }
        case CB_OP_MATCHES: st[sp - 1] = op_matches(c, st[sp - 1], ic); break;
        case CB_OP_LOOP_PRED: {   // predicate of a filtering map / transform*: false -> this iteration is skipped
            const Val v = st[sp - 1];
            if (v.tag != CB_T_BOOL) { st[sp - 1] = mk_err(); pc = ic; }
            else if (!v.u) { st[sp - 1] = mk(CB_T_SKIP, 0); pc = ic; }
            else sp--;
            break;
        }
        default: c.unsupported = 1; return false;
        }
    }
}

#endif  // !CB_LEAN_ONLY

// Packed decision bits of request n (kbytes <= 8): to `bitmap`, or -- fused all-gather -- to this rank's slice of every
// rank's gather buffer (plain stores; peer buffers are NVLink-mapped).
CB_HD void store_bits(const BatchView &b, uint8_t *bitmap, uint64_t n, uint64_t acc) {
    if (b.n_out == 0 && b.kbytes == 1) { bitmap[n] = (uint8_t)acc; return; }
    uint32_t r = 0;
    do {
        uint8_t *base = b.n_out ? b.outs[r] : bitmap;
        if (b.kbytes == 1) base[n] = (uint8_t)acc;
        else {
            uint8_t *out = base + n * b.kbytes;
            for (uint32_t q = 0; q < b.kbytes; q++) out[q] = (uint8_t)(acc >> (8 * q));
        }
    } while (++r < b.n_out);
}

// ---------------------------------------------------------------------------------------------- column access
// The lean body reads the per-request columns through one of two accessors: straight from global memory (any
// evaluation order), or from a tile of the columns that the TMA unit staged in shared memory one tile ahead
// (index order only).  Layout of a staged tile of CB_TILE requests:
//   [hdr0 CB_TILE x 16 B][hdr1 CB_TILE x 8 B][roles role_cols x CB_TILE x 4 B][slots n_slots x CB_TILE x 8 B]
enum { CB_TILE = 256 };
struct GlobalCols {
    const BatchView *b;
    uint64_t n;
    CB_HD U4 hdr0() const { return ldcol128(b->hdr0 + n); }
    CB_HD uint64_t hdr1() const { return ldcol64(reinterpret_cast<const uint64_t *>(b->hdr1 + n)); }
    CB_HD uint32_t role(uint32_t i) const { return ldcol32(b->roles + (uint64_t)i * b->stride + n); }
    CB_HD uint64_t slot(uint32_t v) const { return ldcol64(b->slots + (uint64_t)v * b->stride + n); }
    CB_HD void prefetch_slot(uint32_t v) const {
#if defined(__CUDA_ARCH__)
        asm volatile("prefetch.global.L1 [%0];" ::"l"(b->slots + (uint64_t)v * b->stride + n));
#endif
    }
    CB_HD bool staged() const { return b->prefetch_slots != 0; }   // every slot column was prefetched with the tile
    CB_HD uint32_t aset_k(uint32_t aset) const { return ldg(b->aset_k + aset); }
    CB_HD const uint64_t *row_am() const { return b->row_am; }
    CB_HD bool stage_result(uint32_t) const { return false; }
};
struct TileCols {
    const uint8_t *base;   // staged tile (shared memory on the device)
    uint32_t tid, slots_off;
    CB_HD U4 hdr0() const { return *reinterpret_cast<const U4 *>(base + tid * 16u); }
    CB_HD uint64_t hdr1() const { return *reinterpret_cast<const uint64_t *>(base + CB_TILE * 16u + tid * 8u); }
    CB_HD uint32_t role(uint32_t i) const { return *reinterpret_cast<const uint32_t *>(base + CB_TILE * 24u + i * (CB_TILE * 4u) + tid * 4u); }
    CB_HD uint64_t slot(uint32_t v) const { return *reinterpret_cast<const uint64_t *>(base + slots_off + v * (CB_TILE * 8u) + tid * 8u); }
    CB_HD void prefetch_slot(uint32_t) const {}
    CB_HD bool staged() const { return true; }
    // small per-batch tables (actions per action set, row x action-set masks): copies in shared memory when they fit
    const uint32_t *aset_k_s;
    const uint64_t *row_am_s;
    CB_HD uint32_t aset_k(uint32_t aset) const { return ldg(aset_k_s + aset); }
    CB_HD const uint64_t *row_am() const { return row_am_s; }
    // fused all-gather: the tile's result bytes are collected in shared memory and leave for the peers as one 256-byte
    // store per tile and peer (NVLink moves 32-byte writes poorly); the thread then stores its byte locally only
    uint8_t *res_s;
    CB_HD bool stage_result(uint32_t acc) const { if (!res_s) return false; res_s[tid] = (uint8_t)acc; return true; }
};
CB_HD uint32_t tile_cols_bytes(uint32_t role_cols, uint32_t n_slots) { return CB_TILE * (24u + 4u * role_cols + 8u * n_slots); }

// ---------------------------------------------------------------------------------------------- flat fast path
enum { TRI_F = 0, TRI_T = 1, TRI_E = 2, TRI_SLOW = 3 };

CB_HD uint32_t v64_tag(uint64_t b) {   // 0 = double
    uint32_t top = (uint32_t)(b >> 48);
    return ((top & 0xFFF0u) == 0xFFF0u) ? (top & 0xFu) : 0u;
}

// ---------------------------------------------------------------------------------------------- decision walk
#ifndef CB_LEAN_ONLY
CB_HD bool in_class(const BatchView &b, uint32_t c0, uint32_t c1, uint32_t pat) {
    for (uint32_t j = c0; j < c1; j++)
        if (ldg(b.class_pats + j) == pat) return true;
    return false;
}

// NOTE on structure: everything the hot path keeps per request lives in plain scalars.  Objects whose address
// is handed to a non-inlined function are forced into local memory (the first version of this kernel spent most
// of its time there), so the cold helpers below take their arguments BY VALUE and rebuild what they need.

// is table role `role` in {req_role} U parents(exact resource scope, req_role)   (index.go:805-836)
CB_HD bool role_in_pr(const TableView t, uint32_t role, uint32_t req_role, uint32_t rscope) {
    if (req_role == role) return true;
    if (!t.L->has_parent_roles || req_role >= t.L->nR) return false;
    if (rscope == CB_SCOPE_NONE || (rscope & CB_SCOPE_INEXACT_BIT) || rscope >= t.L->nS) return false;
    uint64_t idx = (uint64_t)rscope * t.L->nR + req_role;
    for (uint32_t j = ldg(t.par_off() + idx), e = ldg(t.par_off() + idx + 1); j < e; j++)
        if (ldg(t.par_list() + j) == role) return true;
    return false;
}

// Evaluates condition `gid` (global id) with the generic stack interpreter.  bit0: it yields BOOL true
// (ruletable.go:1425-1441); bit1: a run-time value the device cannot represent exactly was met.
// Scalar arguments only: aggregates would travel through local memory under the device ABI.
CB_HD_NOINLINE uint32_t cond_sat(const uint8_t *base, const TableLayout *L, const BatchView *b, uint64_t req, uint32_t pid, uint32_t gid, uint64_t edr = 0) {
    TableView t; t.base = base; t.L = L;
    Ctx c;
    c.t = &t; c.b = b; c.req = req; c.pid = pid; c.unsupported = 0; c.scr_used = 0; c.edr = edr;
    bool s = run_program(c, t.code() + ldg(&t.conds()[gid].code_off));
    return (s ? 1u : 0u) | (c.unsupported ? 2u : 0u);
}

// same, for a program given by its offset in CODE (the unique-condition image has no CONDS section)
CB_HD_NOINLINE uint32_t cond_sat_code(const uint8_t *base, const TableLayout *L, const BatchView *b, uint64_t req, uint32_t pid, uint32_t code_off) {
    TableView t; t.base = base; t.L = L;
    Ctx c;
    c.t = &t; c.b = b; c.req = req; c.pid = pid; c.unsupported = 0; c.scr_used = 0; c.edr = 0;
    bool s = run_program(c, t.code() + code_off);
    return (s ? 1u : 0u) | (c.unsupported ? 2u : 0u);
}

#endif  // !CB_LEAN_ONLY

// ---- inline DNF evaluator of the lean body (layout FLAT_DNF, compiled by bytecode.FlatCompiler) --------------
// Works directly on the 8-byte NaN-boxed values.  No calls and no early exits: every lane walks every term with
// predicates, so lanes evaluating the same condition shape stay converged.  Anything it cannot decide exactly
// (container equality, int list elements, string ordering ...) sets `slow`: the request is then re-evaluated by
// the general body with the generic interpreter.
struct StrRef { const uint8_t *p; uint32_t len; };
CB_HD StrRef str_ref(const TableView t, const BatchView &b, uint64_t v) {   // v: boxed STRING
    uint32_t id = (uint32_t)(v & 0xFFFFFFFFu);
    StrRef r;
    if (id < t.L->nT) { uint32_t o = ldg(t.str_off() + id); r.p = t.str_bytes() + o; r.len = ldg(t.str_off() + id + 1) - o; }
    else { uint32_t j = id - t.L->nT; uint32_t o = ldg(b.bstr_off + j); r.p = b.bstr_bytes + o; r.len = ldg(b.bstr_off + j + 1) - o; }
    return r;
}
CB_HD const uint64_t *list_ptr(const TableView t, const BatchView &b, uint64_t v) {   // v: boxed LIST / MAP
    uint64_t pay = v & 0xFFFFFFFFFFFFull;
    return (pay & CB_V64_HEAP_BATCH_BIT) ? b.heap + (pay & (CB_V64_HEAP_BATCH_BIT - 1)) : t.theap() + pay;
}
// scalar equality of two NaN-boxed values whose tags are <= STRING (double / null / bool / string)
CB_HD bool scalar_eq64(uint64_t x, uint64_t y) {
    return (v64_tag(x) == 0 && v64_tag(y) == 0) ? u2d(x) == u2d(y) : x == y;
}
template <typename Cols>
CB_HD uint64_t term_operand(const TableView t, const BatchView &b, const Cols &cols, uint32_t pid, uint32_t kind, uint32_t v, uint32_t aux) {
    const uint64_t kErr = (uint64_t)(CB_V64_BOX_BASE | CB_V64_ERROR) << 48;
    if (kind == CB_OPK_CONST) return ldg(t.consts_v64() + v);
    if (kind == CB_OPK_PID) return ((uint64_t)(CB_V64_BOX_BASE | CB_V64_STRING) << 48) | pid;
    uint64_t x = cols.slot(v);
    if (kind == CB_OPK_SLOT) return x;
    uint32_t tx = v64_tag(x);
    if (kind == CB_OPK_SLOT_ELEM) {
        if (tx != CB_V64_LIST) return kErr;                       // map[int] / scalar[int]: no such key / overload
        const uint64_t *p = list_ptr(t, b, x);
        return aux < (uint32_t)ldg(p) ? ldg(p + 1 + aux) : kErr;   // index out of bounds is an error
    }
    // SLOT_SIZE -> double (the compare against an int constant is exact for these magnitudes)
    if (tx == CB_V64_LIST || tx == CB_V64_MAP) return d2u((double)(uint32_t)ldg(list_ptr(t, b, x)));
    if (tx == CB_V64_STRING) {
        StrRef s = str_ref(t, b, x);
        uint32_t k = 0;
        for (uint32_t i = 0; i < s.len; i++) k += (ldg(s.p + i) & 0xC0) != 0x80;
        return d2u((double)k);
    }
    return kErr;
}
// shape-specialised term kernels (bytecode._specialize_term): straight-line code, same results as the generic term
CB_HD bool v64_bad(uint64_t x) { return ((uint32_t)(x >> 48) & 0xFFFEu) == (CB_V64_BOX_BASE | CB_V64_ABSENT); }   // ABSENT or ERROR
CB_HD int eq_tri(uint64_t x, uint64_t y, bool &slow) {
    const uint32_t tx = v64_tag(x), ty = v64_tag(y);
    if (v64_bad(x) || v64_bad(y)) return TRI_E;
    if (tx == 0 && ty == 0) return u2d(x) == u2d(y);
    if (tx <= CB_V64_STRING && ty <= CB_V64_STRING) return x == y;   // null / bool / interned string / mixed
    slow = true;                                                       // containers
    return TRI_E;
}
CB_HD int ord_tri(uint32_t ci, uint64_t x, uint64_t y, bool &slow) {
    const uint32_t tx = v64_tag(x), ty = v64_tag(y);
    if (v64_bad(x) || v64_bad(y)) return TRI_E;
    if (tx == 0 && ty == 0) {
        const double dx = u2d(x), dy = u2d(y);
        if (dx != dx || dy != dy) return TRI_E;
        return ci == 2 ? dx < dy : ci == 3 ? dx <= dy : ci == 4 ? dx > dy : dx >= dy;
    }
    if (tx != ty) return TRI_E;   // no ordering across types
    slow = true;                  // strings, bools ...: out of line
    return TRI_E;
}
// x in list(y); elems_scalar: the list is a table constant whose elements are known to be scalars
CB_HD int in_tri(const TableView t, const BatchView &b, uint64_t x, uint64_t y, bool elems_scalar, bool &slow) {
    if (v64_bad(x) || v64_bad(y)) return TRI_E;
    if (v64_tag(y) != CB_V64_LIST || v64_tag(x) > CB_V64_STRING) { slow = true; return TRI_E; }
    const uint64_t *p = list_ptr(t, b, y);
    const uint32_t ln = (uint32_t)ldg(p);
    bool found = false;
    for (uint32_t j = 0; j < ln; j++) {
        const uint64_t e = ldg(p + 1 + j);
        if (!elems_scalar) slow |= v64_tag(e) > CB_V64_STRING;
        found |= scalar_eq64(x, e);
    }
    return found;
}
// x in (constant list of scalars) with the elements inlined as arguments (run-time specialised kernels): same outcome
// as in_tri() with elems_scalar
template <typename... E>
CB_HD int in_const_tri(uint64_t x, bool &slow, E... elems) {
    if (v64_bad(x)) return TRI_E;
    if (v64_tag(x) > CB_V64_STRING) { slow = true; return TRI_E; }
    bool found = false;
    ((found |= scalar_eq64(x, (uint64_t)elems)), ...);
    return found ? TRI_T : TRI_F;
}
// One term {op | flags<<8 | xk<<16 | yk<<24, x, y, xa | ya<<16} -> TRI_T / TRI_F / TRI_E; `slow` is raised for operands
// this path cannot decide exactly.  Force-inlined: called with a compile-time constant `w` (run-time specialised
// kernels, cb_specialize.h) the switch, the operand kinds and the slot indices all fold away.
template <typename Cols>
CB_HD int term_tri(const TableView t, const BatchView &b, const Cols &cols, uint32_t pid, const U4 w, bool &slow) {
    const uint32_t op = w.x & 0xFF, flags = (w.x >> 8) & 0xFF, xk = (w.x >> 16) & 0xFF, yk = w.x >> 24;
    int tri = TRI_E;
    switch (w.x & 0xFF) {
    case CB_TERM_EQ_SS: tri = eq_tri(cols.slot(w.y), cols.slot(w.z), slow); break;
    case CB_TERM_EQ_SC: tri = eq_tri(cols.slot(w.y), ldg(t.consts_v64() + w.z), slow); break;
    case CB_TERM_EQ_SP: tri = eq_tri(cols.slot(w.y), ((uint64_t)(CB_V64_BOX_BASE | CB_V64_STRING) << 48) | pid, slow); break;
    case CB_TERM_ORD_SS: tri = ord_tri(flags & CB_TERM_CI_MASK, cols.slot(w.y), cols.slot(w.z), slow); break;
    case CB_TERM_ORD_SC: tri = ord_tri(flags & CB_TERM_CI_MASK, cols.slot(w.y), ldg(t.consts_v64() + w.z), slow); break;
    case CB_TERM_IN_SC: tri = in_tri(t, b, cols.slot(w.y), ldg(t.consts_v64() + w.z), true, slow); break;
    case CB_TERM_IN_CS: tri = in_tri(t, b, ldg(t.consts_v64() + w.y), cols.slot(w.z), false, slow); break;
    case CB_TERM_IN_SS: tri = in_tri(t, b, cols.slot(w.y), cols.slot(w.z), false, slow); break;
    default: {
        const uint64_t x = term_operand(t, b, cols, pid, xk, w.y, w.w & 0xFFFF);
        const uint64_t y = op == CB_TERM_HAS ? 0 : term_operand(t, b, cols, pid, yk, w.z, w.w >> 16);
        const uint32_t tx = v64_tag(x), ty = v64_tag(y);
        const bool xerr = tx == CB_V64_ABSENT || tx == CB_V64_ERROR, yerr = ty == CB_V64_ABSENT || ty == CB_V64_ERROR;
        if (op == CB_TERM_HAS) {
            tri = tx == CB_V64_ERROR ? TRI_E : (tx != CB_V64_ABSENT);
        } else if (xerr || yerr) {
            tri = TRI_E;
        } else if (op == CB_TERM_CMP) {
            const uint32_t ci = flags & CB_TERM_CI_MASK;
            if (tx == 0 && ty == 0) {
                const double dx = u2d(x), dy = u2d(y);
                if (ci == 0) tri = dx == dy;
                else if (dx != dx || dy != dy) tri = TRI_E;
                else tri = ci == 2 ? dx < dy : ci == 3 ? dx <= dy : ci == 4 ? dx > dy : dx >= dy;
            } else if (ci == 0 && tx <= CB_V64_STRING && ty <= CB_V64_STRING) tri = x == y;   // null / bool / interned string / mixed
            else if (ci != 0 && tx != ty) tri = TRI_E;                                         // no ordering across types
            else slow = true;                                                                  // containers, string ordering, ints
        } else if (op == CB_TERM_IN) {
            if (ty != CB_V64_LIST || tx > CB_V64_STRING) slow = true;   // maps, container members: out of line
            else {
                const uint64_t *p = list_ptr(t, b, y);
                const uint32_t ln = (uint32_t)ldg(p);
                bool found = false;
                for (uint32_t j = 0; j < ln; j++) {
                    const uint64_t e = ldg(p + 1 + j);
                    slow |= v64_tag(e) > CB_V64_STRING;               // int / container elements
                    found |= scalar_eq64(x, e);
                }
                tri = found;
            }
        } else if (op == CB_TERM_STARTS || op == CB_TERM_ENDS || op == CB_TERM_CONTAINS) {
            if (tx != CB_V64_STRING || ty != CB_V64_STRING) tri = TRI_E;
            else {
                const StrRef a = str_ref(t, b, x), c = str_ref(t, b, y);
                if (c.len > a.len) tri = TRI_F;
                else if (op == CB_TERM_CONTAINS) {
                    bool hit = false;
                    for (uint32_t o = 0; o + c.len <= a.len; o++) {
                        bool eq = true;
                        for (uint32_t j = 0; j < c.len; j++) eq &= ldg(a.p + o + j) == ldg(c.p + j);
                        hit |= eq;
                    }
                    tri = hit;
                } else {
                    const uint8_t *ap = op == CB_TERM_STARTS ? a.p : a.p + (a.len - c.len);
                    bool eq = true;
                    for (uint32_t j = 0; j < c.len; j++) eq &= ldg(ap + j) == ldg(c.p + j);
                    tri = eq;
                }
            }
        } else {   // INTERSECTS / SUBSET on two lists (cerbos_lib.go:323-431)
            if (tx != CB_V64_LIST || ty != CB_V64_LIST) tri = TRI_E;
            else {
                const uint64_t *pa = list_ptr(t, b, x), *pb = list_ptr(t, b, y);
                const uint32_t na = (uint32_t)ldg(pa), nb = (uint32_t)ldg(pb);
                bool any_hit = false, all_hit = true;
                for (uint32_t i2 = 0; i2 < na; i2++) {
                    const uint64_t ea = ldg(pa + 1 + i2);
                    slow |= v64_tag(ea) > CB_V64_STRING;
                    bool hit = false;
                    for (uint32_t j = 0; j < nb; j++) {
                        const uint64_t eb = ldg(pb + 1 + j);
                        slow |= v64_tag(eb) > CB_V64_STRING;       // ints would need the Go-map identity rule
                        hit |= scalar_eq64(ea, eb);
                    }
                    any_hit |= hit;
                    all_hit &= hit;
                }
                tri = op == CB_TERM_INTERSECTS ? any_hit : all_hit;
            }
        }
    }
    }
    return tri;
}
// ---- register-resident lists (run-time specialised unique-condition kernels) ----------------------------------------
// Several conditions of a table usually read the same list attribute (principal groups, allowed groups ...).  The
// specialised build loads such a list ONCE per request into registers -- length + up to CB_LC elements, normalised so
// that scalar equality is plain 64-bit equality (-0.0 -> +0.0; padding = a sentinel that equals nothing) -- and every
// membership / set predicate over it is a fully unrolled run of compares.  Lists the cache cannot hold exactly (longer,
// container / int / NaN elements) raise `slow`: the request goes to the general body.
// The element loops stop at `bound`: the longest list among the lanes of the warp (the device build; the host build
// uses the list's own length), clamped to CB_LC.  It is warp-uniform, so every `if (j < bound)` below is a uniform
// branch over a constant index (the arrays stay in registers), and positions at or above every lane's length hold only
// padding: skipping them changes no result.
enum { CB_LC = 8 };
CB_HD uint32_t list_bound(uint32_t own) {
#if defined(__CUDA_ARCH__)
    return __reduce_max_sync(__activemask(), own);
#else
    return own;
#endif
}
#ifndef CB_LIST_KEYS64
// Lists of interned strings (what set / membership conditions over attributes hold in practice) are cached as their
// 32-bit string ids: half the registers and compares of the boxed words.  Any other element (number, bool, null,
// container) makes the list one "this cache cannot hold": the general body decides.
struct ListRegs {
    uint32_t st, len;        // st 0: cached list; 1: slot ABSENT / ERROR; 2: a list this cache cannot hold exactly; 3: another type
    uint32_t bound;          // element positions the loops visit (see above)
    uint32_t e[CB_LC];
};
static constexpr uint32_t kListPad = 0xFFFFFFFEu;      // never a string id
static constexpr uint32_t kListNoKey = 0xFFFFFFFFu;    // a scalar that is not a string: equal to no element of a cached list
static constexpr uint32_t kStringTop = CB_V64_BOX_BASE | CB_V64_STRING;
CB_HD uint32_t list_key(uint64_t w) { return (uint32_t)w; }
CB_HD bool list_elem_odd(uint64_t w) { return (uint32_t)(w >> 48) != kStringTop; }
static constexpr uint64_t kListBeyondHeap = 0ull;      // a word past the end of the heap: not a string, so the list defers
#else
struct ListRegs {
    uint32_t st, len;        // st 0: cached list; 1: slot ABSENT / ERROR; 2: a list this cache cannot hold exactly; 3: another type
    uint32_t bound;          // element positions the loops visit (see above)
    uint64_t e[CB_LC];
};
static constexpr uint64_t kListPad = 0xFFFE000000000001ull;    // box tag 14: never produced by an encoder
CB_HD uint64_t norm_scalar(uint64_t v) { return v == 0x8000000000000000ull ? 0ull : v; }
CB_HD uint64_t list_key(uint64_t w) { return norm_scalar(w); }
CB_HD bool list_elem_odd(uint64_t w) { return v64_tag(w) > CB_V64_STRING || w == CB_V64_CANON_NAN; }
static constexpr uint64_t kListBeyondHeap = kListPad;          // tag 14: the list defers
#endif
CB_HD ListRegs list_load(const TableView t, const BatchView &b, uint64_t x) {
    ListRegs L;
    L.st = v64_bad(x) ? 1u : v64_tag(x) == CB_V64_LIST ? 0u : 3u;
    L.len = 0;
#ifdef CB_UC_STUB_LISTS   // tools/uc_variants.sh: no heap loads, no compares (wrong results)
    L.len = (uint32_t)x & 7u;
    L.bound = CB_LC;
    for (int j = 0; j < CB_LC; j++) L.e[j] = (uint32_t)x + j;
    return L;
#endif
    const uint64_t *p = nullptr;
    uint64_t room = 0;   // words from p to the end of its heap
    if (L.st == 0) {
        const uint64_t pay = x & 0xFFFFFFFFFFFFull;
        const bool in_batch = (pay & CB_V64_HEAP_BATCH_BIT) != 0;
        const uint64_t off = in_batch ? pay & (CB_V64_HEAP_BATCH_BIT - 1) : pay;
        p = (in_batch ? b.heap : t.theap()) + off;
        room = (in_batch ? b.heap_words : (uint64_t)t.L->theap_words) - off;
        L.len = (uint32_t)ldg(p);
    }
    // every element word below the bound is requested at once (bounded by the end of the heap, not by this lane's
    // length); words beyond the length are discarded below
    L.bound = list_bound(L.len < CB_LC ? L.len : CB_LC);
    uint64_t w[CB_LC];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int j = 0; j < CB_LC; j++) {
        w[j] = kListBeyondHeap;
        if ((uint32_t)j < L.bound && (uint64_t)(j + 1) < room) w[j] = ldg(p + 1 + j);
    }
    bool odd = L.len > CB_LC;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int j = 0; j < CB_LC; j++) {
        const bool in = (uint32_t)j < L.len;
        odd |= in && list_elem_odd(w[j]);
        L.e[j] = in ? list_key(w[j]) : kListPad;
    }
    if (L.st == 0) L.st = odd ? 2u : 0u;
    return L;
}
// x in L: the outcome of in_tri() / the IN branch of term_tri() for every input this form decides, `slow` otherwise
CB_HD int list_in_tri(uint64_t x, const ListRegs &L, bool &slow) {
#ifdef CB_UC_STUB_LISTS
    return (uint32_t)x == L.e[0] ? TRI_T : TRI_F;
#endif
    if (v64_bad(x) || L.st == 1) return TRI_E;
    if (L.st != 0 || v64_tag(x) > CB_V64_STRING || x == CB_V64_CANON_NAN) { slow = true; return TRI_E; }
#ifndef CB_LIST_KEYS64
    const uint32_t nx = (uint32_t)(x >> 48) == kStringTop ? (uint32_t)x : kListNoKey;   // number / bool / null: in no list of strings
#else
    const uint64_t nx = norm_scalar(x);
#endif
    bool found = false;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int j = 0; j < CB_LC; j++)
        if ((uint32_t)j < L.bound) found |= nx == L.e[j];
    return found ? TRI_T : TRI_F;
}
// Which elements of A occur in B: bit i for element i (i < A.len).  Every set predicate over the same two list slots
// reads this one mask (cb_specialize.h: generate_uc): one compare grid per pair instead of one per predicate.
CB_HD uint32_t list_mask(const ListRegs &A, const ListRegs &B) {
    uint32_t m = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int i = 0; i < CB_LC; i++) {
        if ((uint32_t)i >= A.bound) continue;
        bool hit = false;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int j = 0; j < CB_LC; j++)
            if ((uint32_t)j < B.bound) hit |= A.e[i] == B.e[j];
        m |= (uint32_t)(hit && (uint32_t)i < A.len) << i;   // padding of A would "hit" the padding of B
    }
    return m;
}
// the INTERSECTS / SUBSET branch of term_tri() from m = list_mask(A, B): isSubset(A, B) is "every element of A hit",
// hasIntersection(A, B) -- and hasIntersection(B, A), the status tests being symmetric -- is "some element hit"
CB_HD int list_set_tri(bool subset, const ListRegs &A, const ListRegs &B, uint32_t m, bool &slow) {
#ifdef CB_UC_STUB_LISTS
    return (A.e[0] == B.e[subset] + m) ? TRI_T : TRI_F;
#endif
    if (A.st == 1 || B.st == 1) return TRI_E;
    if (A.st == 3 || B.st == 3) return TRI_E;
    if (A.st == 2 || B.st == 2) { slow = true; return TRI_E; }
    return (subset ? m == (1u << A.len) - 1u : m != 0u) ? TRI_T : TRI_F;   // st 0: len <= CB_LC
}
// attribute.startsWith / endsWith / contains(constant string) through the per-string predicate word (BatchView::strpred)
CB_HD int strpred_tri(const BatchView &b, uint64_t x, uint32_t p) {
#ifdef CB_UC_STUB_STRPRED   // tools/uc_variants.sh: attribution of kernel time (wrong results)
    return (int)((x >> p) & 1u);
#endif
    if (v64_bad(x)) return TRI_E;
    if (v64_tag(x) != CB_V64_STRING) return TRI_E;
    return (int)((ldg(b.strpred + (uint32_t)(x & 0xFFFFFFFFu)) >> p) & 1u);
}
// a one-value column accessor: evaluates a term for a given string (the predicate pre-pass)
struct OneCols {
    uint64_t x;
    CB_HD uint64_t slot(uint32_t) const { return x; }
};
CB_HD bool term_lit(int tri, uint32_t flags) { return (flags & CB_TERM_LIT_F) ? tri == TRI_F : tri == TRI_T; }
// -> bit0 satisfied, bit2: needs the out-of-line general path
template <typename Cols>
CB_HD uint32_t flat_dnf_inline(const TableView t, const BatchView &b, const Cols &cols, uint32_t pid, uint32_t flat_off, uint32_t info) {
    const uint32_t nt = info & 0xFFFF;
    const cb_instr *terms = t.code() + flat_off;
    bool any = false, group = true, slow = false;
    for (uint32_t i = 0; i < nt; i++) {
        const U4 w = ld16(terms + 2 * i);
        const uint32_t flags = (w.x >> 8) & 0xFF;
        group &= term_lit(term_tri(t, b, cols, pid, w, slow), flags);
        if (flags & CB_TERM_GROUP_END) { any |= group; group = true; }
    }
    if (slow) return 4u;
    return (uint32_t)(any != (bool)((info >> 24) & 1));
}
// condition `gid` on the call-free fast path: bit0 satisfied, bit2 = cannot decide here (no flat form or an
// unusual operand): the request is then re-evaluated by the general body
template <typename Cols>
CB_HD uint32_t cond_eval(const TableView t, const BatchView &b, const Cols &cols, uint32_t pid, uint32_t gid) {
    U4 cd = ld16(t.conds() + gid);   // {code_off, code_len, flat_off, flat_info}
    if (cd.w) return flat_dnf_inline(t, b, cols, pid, cd.z, cd.w);
    return 4u;
}

// first scope of the chain for `kind_flag`, honouring strict / lenient search (ruletable.go:626-632)
CB_HD uint32_t chain_start(const TableView t, uint32_t scope, uint32_t kind_flag, bool lenient) {
    if (scope == CB_SCOPE_NONE) return CB_NONE32;
    uint32_t s = scope & ~CB_SCOPE_INEXACT_BIT;
    if (s >= t.L->nS) return CB_NONE32;
    if (!(ldg(t.scope_flags() + s) & kind_flag)) {
        if (!lenient) return CB_NONE32;
        do { s = ldg(t.scope_parent() + s); } while (s != CB_NONE32 && !(ldg(t.scope_flags() + s) & kind_flag));
    }
    return s;
}
CB_HD uint32_t chain_next(const TableView t, uint32_t s, uint32_t kind_flag) {
    do { s = ldg(t.scope_parent() + s); } while (s != CB_NONE32 && !(ldg(t.scope_flags() + s) & kind_flag));
    return s;
}

CB_HD void prefetch_l1(const void *p) {
#if defined(__CUDA_ARCH__)
    asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
#else
    (void)p;
#endif
}

// Issues L1 prefetches for the header / role columns of request `n` (the next tile of this thread).
CB_HD void prefetch_request(const BatchView &b, uint64_t n) {
    prefetch_l1(b.hdr0 + n);
    prefetch_l1(b.hdr1 + n);
    const uint32_t *pr = b.roles + n;
    for (uint32_t i = 0; i < b.role_cols; i++, pr += b.stride) prefetch_l1(pr);
    const uint64_t *ps = b.slots + n;
    for (uint32_t q = 0; q < b.prefetch_slots; q++, ps += b.stride) prefetch_l1(ps);
}

#ifndef CB_LEAN_ONLY
// The resource patterns a request kind matches; kc is hdr0.kind_class: the pattern id itself when there is exactly
// one (CB_KIND_NONE: none), else an index into the class CSR.
CB_HD uint32_t kind_count(const BatchView &b, uint32_t kc) {
    if (kc == CB_KIND_NONE) return 0;
    if (!(kc & CB_KIND_CLASS_CSR_BIT)) return 1;
    uint32_t c = kc & ~CB_KIND_CLASS_CSR_BIT;
    return ldg(b.class_off + c + 1) - ldg(b.class_off + c);
}
CB_HD uint32_t kind_pat_at(const BatchView &b, uint32_t kc, uint32_t j) {
    if (!(kc & CB_KIND_CLASS_CSR_BIT)) return kc;
    return ldg(b.class_pats + ldg(b.class_off + (kc & ~CB_KIND_CLASS_CSR_BIT)) + j);
}
CB_HD bool kind_has(const BatchView &b, uint32_t kc, uint32_t pat) {
    if (!(kc & CB_KIND_CLASS_CSR_BIT)) return kc == pat;   // KIND_NONE never equals a pattern id
    for (uint32_t j = 0, n = kind_count(b, kc); j < n; j++)
        if (kind_pat_at(b, kc, j) == pat) return true;
    return false;
}

// ---- per-request role table: for every table role r, the principal role columns i with r in {role_i} U
// parents(role_i) (index.go:805-836), RCP bits per role, so a row's role test is one shift (rp0/rp1, 128 bits).
// Tables with more roles than fit use the slow helper, which re-reads the request's role columns. ----
template <typename M>
CB_HD_NOINLINE M role_cols_slow(const uint8_t *base, const TableLayout *L, const BatchView *b, uint64_t n, uint32_t n_roles, uint32_t rscope, uint32_t role) {
    TableView t; t.base = base; t.L = L;
    M m = 0;
    for (uint32_t i = 0; i < n_roles; i++) m |= (M)role_in_pr(t, role, ldcol32(b->roles + (uint64_t)i * b->stride + n), rscope) << i;
    return m;
}
struct U2x64 { uint64_t a, b; };
CB_HD_NOINLINE U2x64 role_tab_parents(const uint8_t *base, const TableLayout *L, const BatchView *b, uint64_t n, uint32_t n_roles, uint32_t rscope, uint32_t RCP,
                                     uint64_t rp0, uint64_t rp1) {
    TableView t; t.base = base; t.L = L;
    for (uint32_t i = 0; i < n_roles; i++) {
        uint32_t r = ldcol32(b->roles + (uint64_t)i * b->stride + n);
        if (r >= t.L->nR) continue;
        uint64_t idx = (uint64_t)rscope * t.L->nR + r;
        for (uint32_t j = ldg(t.par_off() + idx), e = ldg(t.par_off() + idx + 1); j < e; j++) {
            uint32_t pq = ldg(t.par_list() + j) * RCP + i;
            if (pq < 64) rp0 |= 1ull << pq; else if (pq < 128) rp1 |= 1ull << (pq - 64);
        }
    }
    U2x64 r; r.a = rp0; r.b = rp1; return r;
}

#endif  // !CB_LEAN_ONLY
// row record accessors on the raw 16-byte load (cb_row: role u16, cond u16 | drcond u16, respat u16 | effect u8,
// flags u8, n_pats u16 | pat_start u32)
CB_HD uint32_t row_role(const U4 &r) { return r.x & 0xFFFF; }
CB_HD uint32_t row_cond(const U4 &r) { return r.x >> 16; }
CB_HD uint32_t row_drcond(const U4 &r) { return r.y & 0xFFFF; }
CB_HD uint32_t row_respat(const U4 &r) { return r.y >> 16; }
CB_HD uint32_t row_effect(const U4 &r) { return r.z & 0xFF; }
#ifndef CB_LEAN_ONLY

// Existence checks (ruletable.go:852-863): false => every action is DENY.  Only reachable when the principal
// and resource policy versions differ (see eval_request).
CB_HD_NOINLINE bool exists_check(const uint8_t *base, const TableLayout *L, const BatchView *b, uint32_t kc, uint32_t pscope, uint32_t r0,
                                 uint32_t pv, uint32_t rv, bool lenient) {
    TableView t; t.base = base; t.L = L;
    bool p_exists = false, r_exists = false;
    if (pv != CB_NONE16)
        for (uint32_t s = chain_start(t, pscope, CB_SCOPE_FLAG_PRINCIPAL, lenient); s != CB_NONE32; s = chain_next(t, s, CB_SCOPE_FLAG_PRINCIPAL))
            p_exists |= ldg(t.prin_exists() + (uint64_t)pv * t.L->nS + s) != 0;
    for (uint32_t s = r0; s != CB_NONE32; s = chain_next(t, s, CB_SCOPE_FLAG_RESOURCE))
        for (uint32_t j = 0, nk = kind_count(*b, kc); j < nk; j++)
            r_exists |= (ldg(t.res_exists() + ((uint64_t)rv * t.L->nRP + kind_pat_at(*b, kc, j)) * t.L->nS + s) & CB_EXISTS_RESOURCE_KIND) != 0;
    return p_exists || r_exists;
}

CB_HD void prefetch_block_slots(const TableView t, const BatchView &b, uint32_t bid, uint64_t n) {
    for (uint32_t q = ldg(t.block_slots_off() + bid), e = ldg(t.block_slots_off() + bid + 1); q < e; q++)
        prefetch_l1(b.slots + (uint64_t)ldg(t.block_slots() + q) * b.stride + n);
}

// ---- effectiveDerivedRoles (ruletable.go:936-979) ------------------------------------------------------------------
// The derived roles of resource policy block `bid` whose parent roles intersect the principal's roles (+ parents in the
// request's resource scope) and whose condition holds: bit set over MANIFEST.derived_roles.  Feeds
// runtime.effectiveDerivedRoles while that policy's conditions are evaluated and the decision metadata.
CB_HD_NOINLINE uint64_t compute_edr(const uint8_t *base, const TableLayout *L, const BatchView *b, uint64_t n, uint32_t pid, uint32_t bid, uint32_t n_roles,
                                    uint32_t rscope, uint32_t *unsupported) {
    TableView t; t.base = base; t.L = L;
    uint64_t mask = 0;
    for (uint32_t e = ldg(t.dr_off() + bid), ee = ldg(t.dr_off() + bid + 1); e < ee; e++) {
        const U4 en = ld16(t.dr_entries() + 4 * (uint64_t)e);   // {name index, cond + 1, parents start, n parents}
        bool hit = false;
        for (uint32_t q = 0; q < en.w && !hit; q++) {
            const uint32_t pr = ldg(t.dr_parents() + en.z + q);
            if (pr == CB_ROLE_ANY) { hit = true; break; }
            for (uint32_t i = 0; i < n_roles && !hit; i++) hit = role_in_pr(t, pr, ldcol32(b->roles + (uint64_t)i * b->stride + n), rscope);
        }
        if (!hit) continue;
        bool sat = true;
        if (en.y) { const uint32_t r = cond_sat(base, L, b, n, pid, en.y - 1); *unsupported |= r & 2; sat = r & 1; }
        if (sat) mask |= 1ull << (en.x & 63);
    }
    return mask;
}

template <typename M>
struct PairMasks { M deny, allow; uint32_t unsupported; };

// Principal policies: role agnostic, decided per action (state lives on role column 0)  (ruletable.go:905-910).
// Cold path (few tables have principal policies for the calling principal): self-contained, arguments by value.
template <typename M>
CB_HD_NOINLINE PairMasks<M> principal_walk(const uint8_t *base, const TableLayout *L, const BatchView *b, uint64_t n, uint32_t pid, uint32_t kc, uint32_t pidx,
                                           uint32_t p0, uint32_t rv, M amask, const uint64_t *row_am) {
    TableView t; t.base = base; t.L = L;
    PairMasks<M> out; out.deny = 0; out.allow = 0; out.unsupported = 0;
    M alive = amask;
    for (uint32_t s = p0; s != CB_NONE32 && alive; s = chain_next(t, s, CB_SCOPE_FLAG_PRINCIPAL)) {
        uint32_t bid = ldg(t.prin_block_map() + ((uint64_t)rv * t.L->nP + pidx) * t.L->nS + s);
        if (bid == CB_NONE32) continue;
        U4 bl = ld16(t.blocks() + bid);   // {row_start, n_rows, cond_base, n_conds}
        M D = 0, A = 0;
        for (uint32_t ri = bl.x, re = bl.x + bl.y; ri < re; ri++) {
            M m = (M)ldg(reinterpret_cast<const M *>(row_am + ri)) & alive;
            if (!m) continue;
            U4 row = ld16(t.rows() + ri);
            if (!kind_has(*b, kc, row_respat(row))) continue;
            if (row_effect(row) == CB_EFFECT_DENY ? (m & ~D) == 0 : (m & ~A) == 0) continue;   // nothing new to learn
            bool sat = true;
            if (row_drcond(row)) { uint32_t r = cond_sat(t.base, t.L, b, n, pid, bl.z + row_drcond(row) - 1); out.unsupported |= r & 2; sat = r & 1; }
            if (sat && row_cond(row)) { uint32_t r = cond_sat(t.base, t.L, b, n, pid, bl.z + row_cond(row) - 1); out.unsupported |= r & 2; sat = r & 1; }
            if (!sat) continue;
            if (row_effect(row) == CB_EFFECT_DENY) D |= m; else A |= m;
        }
        out.deny |= D;
        alive &= ~D;
        uint32_t perm = (ldg(t.scope_flags() + s) >> CB_SCOPE_PERM_SHIFT) & 3;
        if (perm == 1) { M a = A & alive; out.allow |= a; alive &= ~a; }
    }
    return out;
}

// Synthesized role-policy DENY rows of one scope (index.go:688-776): returns the pair mask D extended by them.
template <typename M>
CB_HD_NOINLINE PairMasks<M> rolepol_denies(const uint8_t *base, const TableLayout *L, const BatchView *b, uint64_t n, uint32_t pid, uint32_t kc, uint32_t n_roles,
                                           uint32_t rscope, uint32_t RCP, uint64_t rp0, uint64_t rp1, bool packed, uint32_t rv, uint32_t s,
                                           uint32_t ps, uint32_t aset, M amask, M alive, M D) {
    TableView t; t.base = base; t.L = L;
    PairMasks<M> out; out.allow = 0; out.unsupported = 0;
    const M role_all = (M)(((M)1 << n_roles) - 1);
    const uint32_t nAP = t.L->nAP ? t.L->nAP : 1;
    const uint64_t *spread = b->aset_spread + ((uint64_t)ps * b->n_asets + aset) * nAP;
    uint64_t ro = (uint64_t)rv * t.L->nS + s;
    for (uint32_t e = ldg(t.rp_off() + ro), ee = ldg(t.rp_off() + ro + 1); e < ee; e++) {
        U4 en = ld16(t.rp_entries() + e);   // {role, rule_start, n_rules, pad}
        M rmask;
        if (packed) { uint32_t pos = en.x * RCP; rmask = (M)(pos < 64 ? rp0 >> pos : rp1 >> (pos - 64)) & role_all; }
        else rmask = role_cols_slow<M>(t.base, t.L, b, n, n_roles, rscope, en.x);
        if (!rmask) continue;
        M matched = 0;   // action bits (role column 0) with at least one matching allow rule
        for (uint32_t q = 0; q < en.z; q++) {
            U4 ru = ld16(t.rp_rules() + en.y + q);   // {respat, cond, apat_start, n_apats}
            if (!kind_has(*b, kc, ru.x)) continue;
            M am = 0;
            for (uint32_t a = 0; a < ru.w; a++) am |= (M)ldg(spread + ldg(t.rp_apats() + ru.z + a));
            if (!am) continue;
            matched |= am;
            if (ru.y && ((am * rmask) & alive & ~D)) {
                uint32_t r = cond_sat(t.base, t.L, b, n, pid, ru.y - 1);
                out.unsupported |= r & 2;
                if (!(r & 1)) D |= (am * rmask) & alive;   // DENY none(cond)
            }
        }
        D |= ((amask & ~matched) * rmask) & alive;   // blanket DENY for actions no allow rule matches
    }
    out.deny = D;
    return out;
}

// Evaluates request `n` (absolute column index).  Output: the packed ALLOW bitmap (kbytes bytes per request), or,
// if `effects` is non-null, max_actions effect bytes per request (1 ALLOW / 2 DENY / 0 beyond the request's own
// action count).
// M is the (action x role-column) pair-mask type: uint32_t when max_actions * role_cols <= 32 (the common
// CheckResources shape: halves the register and instruction cost of the mask algebra), else uint64_t.
template <typename M>
CB_HD void eval_request(const TableView t, const BatchView &b, uint64_t n, uint8_t *bitmap, uint8_t *effects, uint32_t *status) {
    constexpr M kOne = 1;
    const U4 h0 = ldcol128(b.hdr0 + n);                                         // principal_id, kind_class, resource_scope, principal_scope
    const uint64_t h1 = ldcol64(reinterpret_cast<const uint64_t *>(b.hdr1 + n));  // rv u16 | pv u16 | action_set_id u32
    const uint32_t pid = h0.x, kc = h0.y, rscope = h0.z, pscope = h0.w;
    const uint32_t rv = (uint32_t)(h1 & 0xFFFF), pv = (uint32_t)((h1 >> 16) & 0xFFFF), aset = (uint32_t)(h1 >> 32);
    const uint32_t RC = b.role_cols;
    const uint32_t K = aset < b.n_asets ? ldg(b.aset_k + aset) : 0;
    uint32_t unsupported = 0;

    // role table (see above)
    uint32_t RCP = 1;
    while (RCP < RC) RCP <<= 1;
    const bool packed = (uint64_t)t.L->nR * RCP <= 128;
    uint64_t rp0 = 0, rp1 = 0;
    uint32_t n_roles = 0;
    for (uint32_t i = 0; i < RC; i++) {
        uint32_t rr = ldcol32(b.roles + (uint64_t)i * b.stride + n);
        if (rr != CB_ROLE_PAD) n_roles = i + 1;   // the encoder packs roles to the front
        if (rr < t.L->nR) {
            uint32_t pos = rr * RCP + i;
            if (pos < 64) rp0 |= 1ull << pos; else if (pos < 128) rp1 |= 1ull << (pos - 64);
        }
    }

    // result: actions 0..63 accumulate in `acc`; wider action lists (rare) write their bytes directly
    uint64_t acc = 0;
    const bool wide = b.kbytes > 8;
    uint8_t *out = effects ? nullptr : bitmap + n * b.kbytes;
    uint8_t *eff = effects ? effects + n * (uint64_t)b.max_actions : nullptr;
    if (wide) {
        if (eff) for (uint32_t q = 0; q < b.max_actions; q++) eff[q] = (uint8_t)(q < K ? CB_EFFECT_DENY : 0);
        else for (uint32_t q = 0; q < b.kbytes; q++) out[q] = 0;
    }

    const bool lenient = (b.flags & CB_BATCH_FLAG_LENIENT) != 0;
    uint32_t p0 = CB_NONE32, r0 = CB_NONE32;
    bool live = n_roles != 0 && K != 0 && rv != CB_NONE16;
    if (live) {
        if (t.L->has_principal_policies) p0 = chain_start(t, pscope, CB_SCOPE_FLAG_PRINCIPAL, lenient);
        r0 = chain_start(t, rscope, CB_SCOPE_FLAG_RESOURCE, lenient);
        // The existence checks can only change a decision when the principal and resource policy versions
        // differ: with equal versions "no principal row / no resource row" already means the walks find nothing.
        if (pv != rv && !exists_check(t.base, t.L, &b, kc, pscope, r0, pv, rv, lenient)) live = false;
        if (p0 == CB_NONE32 && r0 == CB_NONE32) live = false;
    }

    if (live) {
        const uint32_t pidx = (t.L->has_principal_policies && pid < t.L->nT) ? ldg(t.prin_of_string() + pid) : CB_NONE32;
        const M role_all = (M)((kOne << n_roles) - 1);   // n_roles <= 16
        if (t.L->has_parent_roles && packed && rscope != CB_SCOPE_NONE && !(rscope & CB_SCOPE_INEXACT_BIT) && rscope < t.L->nS) {
            U2x64 r = role_tab_parents(t.base, t.L, &b, n, n_roles, rscope, RCP, rp0, rp1);
            rp0 = r.a; rp1 = r.b;
        }
        const uint32_t nk = kind_count(b, kc);

        for (uint32_t ps = 0; ps < b.n_pass; ps++) {
            const uint32_t kbase = ps * b.kc;
            if (kbase >= K) break;
            const uint32_t kn = K - kbase < b.kc ? K - kbase : b.kc;            // actions in this pass
            const uint64_t *row_am = b.row_am + ((uint64_t)ps * b.n_asets + aset) * b.n_rows;
            M amask = 0;                                                         // bit kk*RC for every action of this pass
            for (uint32_t kk = 0; kk < kn; kk++) amask |= kOne << (kk * RC);

            M p_allow = 0, p_deny = 0;
            if (pidx != CB_NONE32 && p0 != CB_NONE32) {
                PairMasks<M> pm = principal_walk<M>(t.base, t.L, &b, n, pid, kc, pidx, p0, rv, amask, row_am);
                p_allow = pm.allow; p_deny = pm.deny; unsupported |= pm.unsupported;
            }

            // ---- resource policies: (action x role) pairs walk the chain together ----
            const M undecided = amask & ~(p_allow | p_deny);
            M r_allow_pairs = 0;
            if (undecided && r0 != CB_NONE32) {
                M alive = undecided * role_all;              // every role column of every undecided action
                for (uint32_t s = r0; s != CB_NONE32 && alive; s = chain_next(t, s, CB_SCOPE_FLAG_RESOURCE)) {
                    M D = 0, A = 0;
                    bool any_row = false;
                    for (uint32_t j = 0; j < nk; j++) {
                        uint64_t mi = ((uint64_t)rv * t.L->nRP + kind_pat_at(b, kc, j)) * t.L->nS + s;
                        if (t.L->has_role_policies) any_row |= (ldg(t.res_exists() + mi) & CB_EXISTS_ANY_ROW) != 0;
                        uint32_t bid = ldg(t.res_block_map() + mi);
                        if (bid == CB_NONE32) continue;
                        prefetch_block_slots(t, b, bid, n);
                        const U4 bl = ld16(t.blocks() + bid);   // {row_start, n_rows, cond_base, n_conds}
                        const uint32_t re = bl.x + bl.y;
                        // One policy block in three tight phases: (1) which conditions can matter for the pairs
                        // still alive, (2) evaluate exactly those (the only calls), (3) accumulate DENY / ALLOW.
                        uint64_t need = 0;
                        for (uint32_t ri = bl.x; ri < re; ri++) {
                            M am = (M)ldg(reinterpret_cast<const M *>(row_am + ri));   // little endian: the low half when M is 32-bit
                            if (!am) continue;
                            U4 row = ld16(t.rows() + ri);
                            uint32_t role = row_role(row);
                            M rc;
                            if (role == CB_ROLE_ANY) rc = role_all;
                            else if (packed) { uint32_t pos = role * RCP; rc = (M)(pos < 64 ? rp0 >> pos : rp1 >> (pos - 64)) & role_all; }
                            else rc = role_cols_slow<M>(t.base, t.L, &b, n, n_roles, rscope, role);
                            if (!((am * rc) & alive)) continue;
                            uint32_t c1 = row_cond(row), c2 = row_drcond(row);
                            if (c1 && c1 <= 64) need |= 1ull << (c1 - 1);
                            if (c2 && c2 <= 64) need |= 1ull << (c2 - 1);
                        }
                        const uint64_t edr = t.L->uses_runtime ? compute_edr(t.base, t.L, &b, n, pid, bid, n_roles, rscope, &unsupported) : 0ull;
                        uint64_t val = 0;
                        for (uint64_t w = need; w;) {
#if defined(__CUDA_ARCH__)
                            int li = __ffsll((long long)w) - 1;
#else
                            int li = __builtin_ctzll(w);
#endif
                            w &= w - 1;
                            uint32_t r = cond_sat(t.base, t.L, &b, n, pid, bl.z + (uint32_t)li, edr);
                            unsupported |= r & 2;
                            val |= (uint64_t)(r & 1) << li;
                        }
                        for (uint32_t ri = bl.x; ri < re; ri++) {
                            M am = (M)ldg(reinterpret_cast<const M *>(row_am + ri));
                            if (!am) continue;
                            U4 row = ld16(t.rows() + ri);
                            uint32_t role = row_role(row);
                            M rc;
                            if (role == CB_ROLE_ANY) rc = role_all;
                            else if (packed) { uint32_t pos = role * RCP; rc = (M)(pos < 64 ? rp0 >> pos : rp1 >> (pos - 64)) & role_all; }
                            else rc = role_cols_slow<M>(t.base, t.L, &b, n, n_roles, rscope, role);
                            M m = (am * rc) & alive;
                            if (!m) continue;
                            uint32_t c1 = row_cond(row), c2 = row_drcond(row);
                            bool sat = true;   // blocks with more than 64 distinct conditions evaluate the overflow ones unmemoised
                            if (c2) { if (c2 <= 64) sat = (val >> (c2 - 1)) & 1; else { uint32_t r = cond_sat(t.base, t.L, &b, n, pid, bl.z + c2 - 1, edr); unsupported |= r & 2; sat = r & 1; } }
                            if (sat && c1) { if (c1 <= 64) sat = (val >> (c1 - 1)) & 1; else { uint32_t r = cond_sat(t.base, t.L, &b, n, pid, bl.z + c1 - 1, edr); unsupported |= r & 2; sat = r & 1; } }
                            if (!sat) continue;
                            if (row_effect(row) == CB_EFFECT_DENY) D |= m; else A |= m;
                        }
                    }
                    if (t.L->has_role_policies && any_row) {
                        PairMasks<M> pm = rolepol_denies<M>(t.base, t.L, &b, n, pid, kc, n_roles, rscope, RCP, rp0, rp1, packed, rv, s, ps, aset, amask, alive, D);
                        D = pm.deny; unsupported |= pm.unsupported;
                    }
                    alive &= ~D;
                    uint32_t perm = (ldg(t.scope_flags() + s) >> CB_SCOPE_PERM_SHIFT) & 3;
                    if (perm == 1) { M a = A & alive; r_allow_pairs |= a; alive &= ~a; }
                }
            }

            // ---- fold: ALLOW iff the principal walk allowed, or undecided there and any role column allowed ----
            M any_role = r_allow_pairs;
            for (uint32_t j = 1; j < RC; j++) any_role |= r_allow_pairs >> j;      // OR the role columns down to column 0
            const M allow_bits = p_allow | (undecided & any_role);                // bits at kk * RC
            for (uint32_t kk = 0; kk < kn; kk++) {
                if (!((allow_bits >> (kk * RC)) & 1)) continue;
                uint32_t k = kbase + kk;
                if (!wide) acc |= 1ull << k; else if (eff) eff[k] = CB_EFFECT_ALLOW; else out[k >> 3] |= (uint8_t)(1u << (k & 7));
            }
        }
    }

    // ---- store ----
    if (!wide) {
        if (eff) {
            if (b.max_actions == 8) {   // one 8-byte store: the common CheckResources shape
                uint64_t v = 0;
                for (uint32_t k = 0; k < 8; k++) v |= (uint64_t)(k < K ? (((acc >> k) & 1) ? CB_EFFECT_ALLOW : CB_EFFECT_DENY) : 0) << (8 * k);
                *reinterpret_cast<uint64_t *>(eff) = v;
            } else {
                for (uint32_t k = 0; k < b.max_actions; k++) eff[k] = (uint8_t)(k < K ? (((acc >> k) & 1) ? CB_EFFECT_ALLOW : CB_EFFECT_DENY) : 0);
            }
        } else {
            store_bits(b, bitmap, n, acc);
        }
    }
    if (unsupported && status) {
#if defined(__CUDA_ARCH__)
        atomicOr(status, 1u);
#else
        *status |= 1u;
#endif
    }
}

// ---------------------------------------------------------------------------------------------- decision metadata
// ActionEffect.Policy / Scope and CheckOutput.EffectiveDerivedRoles (ruletable.go:753-782, 913-922, 936-979, 1082-1148)
// depend on WHICH row decided -- which role column, which scope, whether it came from a role policy -- so this body
// keeps the reference's own loop order (action -> policy kind -> role -> scope -> candidate rows in index order)
// instead of the bit-parallel walk.  It is the optional metadata plane (cgpu_check_meta): one thread per request, every
// condition through the generic interpreter.  The effect it derives is the same decision; tests hold it against both
// the bit-parallel kernels and the oracle.
struct MetaInfo { uint32_t effect, src, scope, role; };   // effect 0 = NO_MATCH
CB_HD uint32_t pack_meta(const MetaInfo &m) { return (m.scope == CB_NONE32 ? 0xFFFFu : (m.scope & 0xFFFFu)) | (m.src & 0xFFu) << 16 | (m.role & 0xFFu) << 24; }

CB_HD bool meta_row_action(const BatchView &b, uint32_t aset, uint32_t n_rows, uint32_t ps, uint32_t kk, uint32_t ri) {
    return ((ldg(b.row_am + ((uint64_t)ps * b.n_asets + aset) * n_rows + ri) >> (kk * b.role_cols)) & 1) != 0;
}

CB_HD_NOINLINE void eval_request_meta(const uint8_t *base, const TableLayout *L, const BatchView *bp, uint64_t n, uint8_t *effects, uint32_t *action_meta,
                                      cb_request_meta *req_meta, uint32_t *status) {
    TableView t; t.base = base; t.L = L;
    const BatchView &b = *bp;
    const U4 h0 = ldcol128(b.hdr0 + n);
    const uint64_t h1 = ldcol64(reinterpret_cast<const uint64_t *>(b.hdr1 + n));
    const uint32_t pid = h0.x, kc = h0.y, rscope = h0.z, pscope = h0.w;
    const uint32_t rv = (uint32_t)(h1 & 0xFFFF), pv = (uint32_t)((h1 >> 16) & 0xFFFF), aset = (uint32_t)(h1 >> 32);
    const uint32_t K = aset < b.n_asets ? ldg(b.aset_k + aset) : 0;
    const uint32_t KM = b.max_actions;
    uint32_t unsupported = 0;
    uint8_t *eff = effects + n * (uint64_t)KM;
    uint32_t *am = action_meta + n * (uint64_t)KM;
    for (uint32_t k = 0; k < KM; k++) { eff[k] = (uint8_t)(k < K ? CB_EFFECT_DENY : 0); am[k] = 0xFFFFu; }
    cb_request_meta rm; rm.principal_first_scope = 0xFFFF; rm.resource_first_scope = 0xFFFF; rm.flags = 0; rm.effective_derived_roles = 0;

    uint32_t roles[CB_MAX_ROLE_COLS], n_roles = 0;
    for (uint32_t i = 0; i < b.role_cols; i++) { const uint32_t rr = ldcol32(b.roles + (uint64_t)i * b.stride + n); if (rr != CB_ROLE_PAD) roles[n_roles++] = rr; }
    const bool lenient = (b.flags & CB_BATCH_FLAG_LENIENT) != 0;
    uint32_t pchain[CB_MAX_CHAIN], rchain[CB_MAX_CHAIN], np = 0, nr = 0;
    for (uint32_t s = chain_start(t, pscope, CB_SCOPE_FLAG_PRINCIPAL, lenient); s != CB_NONE32 && np < CB_MAX_CHAIN; s = chain_next(t, s, CB_SCOPE_FLAG_PRINCIPAL)) pchain[np++] = s;
    for (uint32_t s = chain_start(t, rscope, CB_SCOPE_FLAG_RESOURCE, lenient); s != CB_NONE32 && nr < CB_MAX_CHAIN; s = chain_next(t, s, CB_SCOPE_FLAG_RESOURCE)) rchain[nr++] = s;
    if (np) rm.principal_first_scope = (uint16_t)pchain[0];
    if (nr) rm.resource_first_scope = (uint16_t)rchain[0];
    req_meta[n] = rm;
    if ((np == 0 && nr == 0) || K == 0) return;

    const uint32_t nk = kind_count(b, kc);
    bool p_exists = false, r_exists = false;
    if (pv != CB_NONE16) for (uint32_t i = 0; i < np; i++) p_exists |= ldg(t.prin_exists() + (uint64_t)pv * L->nS + pchain[i]) != 0;
    if (rv != CB_NONE16)
        for (uint32_t i = 0; i < nr; i++)
            for (uint32_t j = 0; j < nk; j++)
                r_exists |= (ldg(t.res_exists() + ((uint64_t)rv * L->nRP + kind_pat_at(b, kc, j)) * L->nS + rchain[i]) & CB_EXISTS_RESOURCE_KIND) != 0;
    if (!p_exists && !r_exists) return;
    const uint32_t pidx = (L->has_principal_policies && pid < L->nT) ? ldg(t.prin_of_string() + pid) : CB_NONE32;
    const bool rows_ok = rv != CB_NONE16;   // candidate rows are those of the resource policy version (ruletable.go:874)
    // allRoles = the principal's roles, then their parents in the resource scope (index.go:805-836): the order candidate
    // rows come in (index.go:564-801); duplicates add nothing
    uint32_t all_roles[CB_MAX_ROLE_COLS * 3], n_all = 0;
    for (uint32_t i = 0; i < n_roles; i++) all_roles[n_all++] = roles[i];
    if (L->has_parent_roles && rscope != CB_SCOPE_NONE && !(rscope & CB_SCOPE_INEXACT_BIT) && rscope < L->nS)
        for (uint32_t i = 0; i < n_roles; i++) {
            if (roles[i] >= L->nR) continue;
            const uint64_t idx = (uint64_t)rscope * L->nR + roles[i];
            for (uint32_t j = ldg(t.par_off() + idx), e = ldg(t.par_off() + idx + 1); j < e && n_all < CB_MAX_ROLE_COLS * 3; j++) all_roles[n_all++] = ldg(t.par_list() + j);
        }
    const uint32_t nAP = L->nAP ? L->nAP : 1;
    uint32_t processed = 0;      // resource chain positions whose derived roles have been evaluated
    uint64_t cur_edr = 0, all_edr = 0;

    for (uint32_t k = 0; k < K; k++) {
        const uint32_t ps = k / b.kc, kk = k % b.kc;
        const uint64_t *spread = b.aset_spread + ((uint64_t)ps * b.n_asets + aset) * nAP;
        MetaInfo info; info.effect = 0; info.src = CB_META_SRC_NO_MATCH; info.scope = CB_NONE32; info.role = 0;
        for (uint32_t pt = 0; pt < 2; pt++) {        // principal policies, then resource policies
            const bool principal = pt == 0;
            const uint32_t *chain = principal ? pchain : rchain;
            const uint32_t nc = principal ? np : nr;
            info.effect = 0;
            for (uint32_t i = 0; i < n_roles; i++) {
                if (i > 0 && principal) break;       // principal policies are role agnostic
                MetaInfo ri; ri.effect = 0; ri.scope = CB_NONE32; ri.role = 0;
                ri.src = (principal ? p_exists : r_exists) ? (principal ? CB_META_SRC_PRINCIPAL_POLICY : CB_META_SRC_RESOURCE_POLICY) : CB_META_SRC_NO_MATCH;
                for (uint32_t si = 0; si < nc; si++) {
                    const uint32_t s = chain[si];
                    if (!principal && !((processed >> si) & 1)) {
                        uint64_t edr = 0;
                        if (rows_ok)
                            for (uint32_t j = 0; j < nk; j++) {
                                const uint32_t bid = ldg(t.res_block_map() + ((uint64_t)rv * L->nRP + kind_pat_at(b, kc, j)) * L->nS + s);
                                if (bid != CB_NONE32) edr |= compute_edr(base, L, bp, n, pid, bid, n_roles, rscope, &unsupported);
                            }
                        cur_edr = edr;
                        all_edr |= edr;
                        processed |= 1u << si;
                    }
                    if (ri.effect) break;
                    bool saw_allow = false, deny = false, deny_rp = false;
                    uint32_t deny_role = 0;
                    if (principal) {
                        const uint32_t bid = (pidx != CB_NONE32 && rows_ok) ? ldg(t.prin_block_map() + ((uint64_t)rv * L->nP + pidx) * L->nS + s) : CB_NONE32;
                        if (bid != CB_NONE32) {
                            const U4 bl = ld16(t.blocks() + bid);
                            for (uint32_t q = 0; q < bl.y && !deny; q++) {
                                const uint32_t rix = bl.x + q;
                                const U4 row = ld16(t.rows() + rix);
                                if (!kind_has(b, kc, row_respat(row)) || !meta_row_action(b, aset, L->n_rows, ps, kk, rix)) continue;
                                if (row_drcond(row)) { const uint32_t r = cond_sat(base, L, bp, n, pid, bl.z + row_drcond(row) - 1, cur_edr); unsupported |= r & 2; if (!(r & 1)) continue; }
                                if (row_cond(row)) { const uint32_t r = cond_sat(base, L, bp, n, pid, bl.z + row_cond(row) - 1, cur_edr); unsupported |= r & 2; if (!(r & 1)) continue; }
                                if (row_effect(row) == CB_EFFECT_DENY) deny = true; else saw_allow = true;
                            }
                        }
                    } else if (rows_ok) {
                        bool any_row = false;
                        for (uint32_t j = 0; j < nk; j++) any_row |= (ldg(t.res_exists() + ((uint64_t)rv * L->nRP + kind_pat_at(b, kc, j)) * L->nS + s) & CB_EXISTS_ANY_ROW) != 0;
                        // candidate rows in index order: for every role R of allRoles, the role policy of R (synthesised
                        // DENY rows) and then the resource policy rows naming R ("*" rows travel with the first role)
                        for (uint32_t a = 0; a < n_all && !deny; a++) {
                            const uint32_t R = all_roles[a];
                            bool dup = false;
                            for (uint32_t z = 0; z < a; z++) dup |= all_roles[z] == R;
                            if (dup) continue;
                            const bool in_pr = role_in_pr(t, R, roles[i], rscope);
                            if (in_pr && any_row && L->has_role_policies) {
                                const uint64_t ro = (uint64_t)rv * L->nS + s;
                                for (uint32_t e = ldg(t.rp_off() + ro), ee = ldg(t.rp_off() + ro + 1); e < ee && !deny; e++) {
                                    const U4 en = ld16(t.rp_entries() + e);   // {role, rule_start, n_rules, pad}
                                    if (en.x != R) continue;
                                    bool matched = false;
                                    for (uint32_t q = 0; q < en.z && !deny; q++) {
                                        const U4 ru = ld16(t.rp_rules() + en.y + q);   // {respat, cond, apat_start, n_apats}
                                        if (!kind_has(b, kc, ru.x)) continue;
                                        bool amatch = false;
                                        for (uint32_t x = 0; x < ru.w && !amatch; x++) amatch = ((ldg(spread + ldg(t.rp_apats() + ru.z + x)) >> (kk * b.role_cols)) & 1) != 0;
                                        if (!amatch) continue;
                                        matched = true;
                                        if (ru.y) { const uint32_t r = cond_sat(base, L, bp, n, pid, ru.y - 1, cur_edr); unsupported |= r & 2; if (!(r & 1)) deny = true; }   // DENY none(cond)
                                    }
                                    if (!matched) deny = true;   // no allow rule of the role policy covers the action
                                    if (deny) { deny_rp = true; deny_role = R; }
                                }
                            }
                            if (deny) break;
                            for (uint32_t j = 0; j < nk && !deny; j++) {
                                const uint32_t bid = ldg(t.res_block_map() + ((uint64_t)rv * L->nRP + kind_pat_at(b, kc, j)) * L->nS + s);
                                if (bid == CB_NONE32) continue;
                                const U4 bl = ld16(t.blocks() + bid);
                                for (uint32_t q = 0; q < bl.y && !deny; q++) {
                                    const uint32_t rix = bl.x + q;
                                    const U4 row = ld16(t.rows() + rix);
                                    const uint32_t rr = row_role(row);
                                    if (!(rr == CB_ROLE_ANY ? a == 0 : (rr == R && in_pr))) continue;
                                    if (!meta_row_action(b, aset, L->n_rows, ps, kk, rix)) continue;
                                    if (row_drcond(row)) { const uint32_t r = cond_sat(base, L, bp, n, pid, bl.z + row_drcond(row) - 1, cur_edr); unsupported |= r & 2; if (!(r & 1)) continue; }
                                    if (row_cond(row)) { const uint32_t r = cond_sat(base, L, bp, n, pid, bl.z + row_cond(row) - 1, cur_edr); unsupported |= r & 2; if (!(r & 1)) continue; }
                                    if (row_effect(row) == CB_EFFECT_DENY) deny = true; else saw_allow = true;
                                }
                            }
                        }
                    }
                    if (deny) {
                        ri.effect = CB_EFFECT_DENY; ri.scope = s;
                        if (deny_rp) { ri.src = CB_META_SRC_ROLE_POLICY; ri.role = deny_role; }
                        break;
                    }
                    if (saw_allow && ((ldg(t.scope_flags() + s) >> CB_SCOPE_PERM_SHIFT) & 3) == 1) { ri.effect = CB_EFFECT_ALLOW; ri.scope = s; break; }
                }
                if (info.effect == 0) info = ri;
                if (ri.effect == CB_EFFECT_ALLOW) { info = ri; break; }
                else if (ri.effect == CB_EFFECT_DENY && info.src == CB_META_SRC_NO_MATCH_FOR_SCOPE_PERMISSIONS && ri.src != CB_META_SRC_NO_MATCH_FOR_SCOPE_PERMISSIONS) info = ri;
            }
            if (info.effect) break;
        }
        eff[k] = (uint8_t)(info.effect == CB_EFFECT_ALLOW ? CB_EFFECT_ALLOW : CB_EFFECT_DENY);
        am[k] = pack_meta(info);
    }
    rm.effective_derived_roles = all_edr;
    req_meta[n] = rm;
    if (unsupported && status) {
#if defined(__CUDA_ARCH__)
        atomicOr(status, 1u);
#else
        *status |= 1u;
#endif
    }
}

#endif  // !CB_LEAN_ONLY

// ---------------------------------------------------------------------------------------------- fast kernel body
// The common deployment shape -- resource policies (+ derived roles, scopes) only: no principal policies, no role
// policies / parent roles, no resource globs -- with max_actions * role_cols <= 32 and n_roles * RCP <= 64.
// Same decision semantics as eval_request<M>, stripped of every cold branch so that the whole per-request state
// is a handful of 32-bit scalars (host code picks this body when table and batch qualify; tests compare both).
// Returns true if the request must be re-evaluated by the general body (nothing has been written then): a
// condition without a flat form, an operand the 8-byte fast forms cannot decide, differing policy versions, or
// a block with more than 32 conditions.  The body itself makes NO calls, so nothing is forced into local memory,
// and its loops contain no early exits (`continue` / `break` would leave lanes diverged until the loop ends).
// one row of a block: its (action x role column) pairs, if its conditions hold, join the DENY or the ALLOW mask
CB_HD void row_apply(uint32_t am, const U4 row, uint64_t rp, uint32_t RCP, uint32_t role_all, uint32_t alive, uint32_t val, uint32_t &D, uint32_t &A) {
    const uint32_t role = row_role(row);
    const uint32_t rc = role == CB_ROLE_ANY ? role_all : (uint32_t)(rp >> (role * RCP)) & role_all;
    const uint32_t sat = (val >> (row.x >> 16)) & (val >> (row.y & 0xFFFF)) & 1u;   // rule condition AND derived-role condition
    const uint32_t ms = (am * rc) & alive & (0u - sat);
    const bool deny = row_effect(row) == CB_EFFECT_DENY;
    D |= deny ? ms : 0u;
    A |= deny ? 0u : ms;
}
// How the lean body evaluates one policy block: this generic walker interprets the block's records; a run-time
// specialised build (cb_specialize.h) substitutes straight-line code generated from the table.
struct GenericBlocks {
    template <typename Cols>
    CB_HD void operator()(const TableView t, const BatchView &b, const Cols &cols, uint32_t pid, uint32_t bid, uint64_t rp, uint32_t RCP, uint32_t role_all,
                          uint32_t alive, const uint64_t *row_am, uint32_t &D, uint32_t &A, bool &defer) const {
        if (!cols.staged())
            for (uint32_t q = ldg(t.block_slots_off() + bid), e = ldg(t.block_slots_off() + bid + 1); q < e; q++)
                cols.prefetch_slot(ldg(t.block_slots() + q));
        const U4 bl = ld16(t.blocks() + bid);   // {row_start, n_rows, cond_base, n_conds}
        defer |= bl.w > 31;
        // phase 1: every condition of the block, once, into one bit each (bit 0 = "no condition" = true).  The
        // lanes of a warp evaluate the same condition list together; a row the request does not reach simply
        // ignores its bit (conditions have no side effects; an operand this path cannot decide defers).
        uint32_t val = 1;
        for (uint32_t c = 0, nc = bl.w > 31 ? 0 : bl.w; c < nc; c++) {
            const uint32_t r = cond_eval(t, b, cols, pid, bl.z + c);
            defer |= (r & 4) != 0;
            val |= (r & 1) << (c + 1);
        }
        // phase 2: rows are pure mask algebra
        for (uint32_t ri = bl.x, re = bl.x + bl.y; ri < re; ri++)
            row_apply(ldg(reinterpret_cast<const uint32_t *>(row_am + ri)), ld16(t.rows() + ri), rp, RCP, role_all, alive, val, D, A);
    }
};

// result of one request on the lean bodies: effect bytes (host-buffer ABI) or packed ALLOW bits
template <typename Cols>
CB_HD void store_result(const BatchView &b, const Cols &cols, uint64_t n, uint8_t *bitmap, uint8_t *effects, uint32_t K, uint32_t acc) {
    if (effects) {
        uint8_t *eff = effects + n * (uint64_t)b.max_actions;
        if (b.max_actions == 8) {
            uint64_t v = 0;
            for (uint32_t k = 0; k < 8; k++) v |= (uint64_t)(k < K ? (((acc >> k) & 1) ? CB_EFFECT_ALLOW : CB_EFFECT_DENY) : 0) << (8 * k);
            *reinterpret_cast<uint64_t *>(eff) = v;
        } else {
            for (uint32_t k = 0; k < b.max_actions; k++) eff[k] = (uint8_t)(k < K ? (((acc >> k) & 1) ? CB_EFFECT_ALLOW : CB_EFFECT_DENY) : 0);
        }
    } else {
        if (cols.stage_result(acc)) bitmap[n] = (uint8_t)acc;   // (kbytes == 1; `bitmap` is this rank's own gather slice)
        else store_bits(b, bitmap, n, acc);
    }
}

template <typename Cols, typename Blocks = GenericBlocks>
CB_HD bool eval_request_fast(const TableView t, const BatchView &b, const Cols &cols, uint64_t n, uint8_t *bitmap, uint8_t *effects, const Blocks blocks = Blocks()) {
    const U4 h0 = cols.hdr0();         // principal_id, kind (pattern id), resource_scope, principal_scope
    const uint64_t h1 = cols.hdr1();   // rv u16 | pv u16 | action_set_id u32
    const uint32_t pid = h0.x, kc = h0.y, rscope = h0.z;
    const uint32_t rv = (uint32_t)(h1 & 0xFFFF), pv = (uint32_t)((h1 >> 16) & 0xFFFF), aset = (uint32_t)(h1 >> 32);
    const uint32_t RC = b.role_cols, RCP = b.rcp;
    const uint32_t K = aset < b.n_asets ? cols.aset_k(aset) : 0;
    uint64_t rp = 0;          // role table: RCP bits per table role
    uint32_t n_roles = 0;
    for (uint32_t i = 0; i < RC; i++) {
        uint32_t rr = cols.role(i);
        n_roles = rr != CB_ROLE_PAD ? i + 1 : n_roles;
        rp |= rr < t.L->nR ? 1ull << (rr * RCP + i) : 0ull;
    }
    if (pv != rv) return true;   // existence checks matter only then (ruletable.go:852-863): general body
    uint32_t acc = 0;
    const bool live = n_roles != 0 && K != 0 && rv != CB_NONE16 && kc != CB_KIND_NONE;
    const uint32_t r0 = live ? chain_start(t, rscope, CB_SCOPE_FLAG_RESOURCE, (b.flags & CB_BATCH_FLAG_LENIENT) != 0) : CB_NONE32;
    if (r0 != CB_NONE32) {
        const uint32_t role_all = (1u << n_roles) - 1;
        const uint64_t *row_am = cols.row_am() + (uint64_t)aset * b.n_rows;
        const uint32_t amask = K * RC >= 32 ? b.stride_pattern : b.stride_pattern & ((1u << (K * RC)) - 1);   // bit kk*RC per action
        uint32_t alive = amask * role_all, allow_pairs = 0;
        bool defer = false;
        for (uint32_t s = r0; s != CB_NONE32 && alive; s = chain_next(t, s, CB_SCOPE_FLAG_RESOURCE)) {
            const uint32_t bid = ldg(t.res_block_map() + ((uint64_t)rv * t.L->nRP + kc) * t.L->nS + s);
            if (bid != CB_NONE32) {
                // pull the attribute slots this block's conditions read towards L1 so the lazy loads overlap
                uint32_t D = 0, A = 0;   // DENY / ALLOW pair masks of this scope
                blocks(t, b, cols, pid, bid, rp, RCP, role_all, alive, row_am, D, A, defer);
                alive &= ~D;
                if (((ldg(t.scope_flags() + s) >> CB_SCOPE_PERM_SHIFT) & 3) == 1) { uint32_t a = A & alive; allow_pairs |= a; alive &= ~a; }
            }
        }
        if (defer) return true;
        // fold: an action is ALLOWed iff some role column allowed it; then pack the stride-RC bits
        uint32_t x = allow_pairs;
        for (uint32_t j = 1; j < RC; j++) x |= allow_pairs >> j;
        x &= amask;
        if (RC == 1) acc = x;
        else if (RC == 2) { x = (x | x >> 1) & 0x33333333u; x = (x | x >> 2) & 0x0F0F0F0Fu; x = (x | x >> 4) & 0x00FF00FFu; acc = (x | x >> 8) & 0xFFFFu; }
        else for (uint32_t kk = 0; kk < K; kk++) acc |= ((x >> (kk * RC)) & 1) << kk;
    }
    store_result(b, cols, n, bitmap, effects, K, acc);
    return false;
}

// ---------------------------------------------------------------------------------------------- unique-condition body
// Tables whose policy blocks differ in shape (many kinds x scopes, each with its own rule list) make the lanes of a
// warp walk different condition lists in index order.  But real policy sets draw their conditions from a small pool:
// the same derived-role and rule conditions recur across policies (the reference memoises them per request under their
// EvaluationKey, ruletable.go:1015, 1050, 1061).  cb_uc.h therefore numbers the DISTINCT conditions of the table
// (1..U, U <= 63) and rewrites every row to {role, condition bit, derived-role condition bit, effect} (4 bytes).  This
// body evaluates ALL U conditions of a request once, up front, into one 64-bit word -- every lane runs the same
// instruction stream over coalesced column loads, whatever block each request hits -- and then walks the request's
// scope chain with rows that are pure mask algebra on that word.  Conditions have no side effects and an error is
// "not satisfied" (ruletable.go:1425-1441), so evaluating one that no row of the request needs cannot change a result.
// Same domain as eval_request_fast (resource policies only, pair masks <= 32 bits); same deferral contract.
// Rows of the unique-condition image (cb_uc.h), 16 bytes each, DENY rows first inside every block:
//   {original row index (for the batch's row x action-set masks), role8 | effect << 8, need_lo, need_hi}
// need = bit of the rule condition | bit of the derived-role condition | bit 0: the row is satisfied iff
// (condition word & need) == need.  What the walk consumes is the record merged with the batch:
//   {action mask of the request's action set, need_lo, need_hi, shift of the row's role field in the role table}
CB_HD U4 uc_row_record(const U4 ur, uint32_t am, uint32_t RCP, uint32_t nR) {
    const uint32_t role = ur.y & 0xFFu;
    U4 r; r.x = am; r.y = ur.z; r.z = ur.w; r.w = (role == 0xFFu ? nR : role) * RCP;   // field nR of the role table = "any role"
    return r;
}
struct UcRowsGlobal {   // straight from the table image and the batch's row_am column
    const U4 *urows; const uint64_t *row_am; uint32_t RCP, nR;
    CB_HD U4 get(uint32_t aset_base, uint32_t ri) const { const U4 ur = ld16(urows + ri); return uc_row_record(ur, (uint32_t)ldg(row_am + aset_base + ur.x), RCP, nR); }
};
struct UcRowsPacked {   // one merged record per (action set, row), built once per CTA in shared memory
    const U4 *pk;
    CB_HD U4 get(uint32_t aset_base, uint32_t ri) const { return ld16(pk + aset_base + ri); }
};

// column access with L1 allocation: the eager condition pass reads the same slot from several terms
struct CachedCols {
    const BatchView *b;
    uint64_t n;
    CB_HD U4 hdr0() const { return ldcol128(b->hdr0 + n); }
    CB_HD uint64_t hdr1() const { return ldcol64(reinterpret_cast<const uint64_t *>(b->hdr1 + n)); }
    CB_HD uint32_t role(uint32_t i) const { return ldcol32(b->roles + (uint64_t)i * b->stride + n); }
    CB_HD uint64_t slot(uint32_t v) const {
#if defined(__CUDA_ARCH__)
        uint64_t x;
        asm("ld.global.nc.u64 %0, [%1];" : "=l"(x) : "l"(b->slots + (uint64_t)v * b->stride + n));
        return x;
#else
        return b->slots[(uint64_t)v * b->stride + n];
#endif
    }
    CB_HD void prefetch_slot(uint32_t) const {}
    CB_HD bool staged() const { return true; }
    CB_HD uint32_t aset_k(uint32_t aset) const { return ldg(b->aset_k + aset); }
    CB_HD const uint64_t *row_am() const { return b->row_am; }
    CB_HD bool stage_result(uint32_t) const { return false; }
};

// How the unique-condition body gets a request's condition word: this generic evaluator interprets the table's DNF
// terms; a run-time
// specialised build (cb_specialize.h: generate_uc) substitutes straight-line code over register-resident slots.
// The condition word: bit u = distinct condition u holds, bit 0 = "no condition".  Form 0: at most 32 bits, rows carry a
// 32-bit need mask; form 1: 64 bits, 64-bit need masks; form 2 (64..127 distinct conditions, run-time specialised
// kernels only): rows carry the two condition NUMBERS they need instead of a mask.
struct CondWord { uint64_t lo, hi; };
enum { CB_UC_FORM_MASK32 = 0, CB_UC_FORM_MASK64 = 1, CB_UC_FORM_INDEX = 2 };
struct GenericConds {
    static constexpr int kForm = CB_UC_FORM_MASK64;   // the condition word may use all 64 bits
    template <typename Cols>
    CB_HD Cols load(const TableView, const BatchView &, const Cols &cols) const { return cols; }
    template <typename Cols>
    CB_HD CondWord operator()(const TableView t, const BatchView &b, const Cols &cols, uint32_t pid, uint64_t n, bool &slow) const {
        if (t.L->n_uconds > 63) { slow = true; CondWord w; w.lo = 1; w.hi = 0; return w; }   // index-form image: specialised kernels only
        uint64_t val = 1;
        for (uint32_t u = 1, nu = t.L->n_uconds; u <= nu; u++) {
            const U4 cd = ld16(t.uconds() + u);   // {code_off, code_len, flat_off, flat_info}
            uint32_t r;
            if (cd.w) r = flat_dnf_inline(t, b, cols, pid, cd.z, cd.w);
            else r = 4u;   // no flat form: the request goes to the general kernel (cb_uc.h only builds images whose conditions are all flat)
            slow |= (r & 4u) != 0;
            val |= (uint64_t)(r & 1u) << u;
        }
        CondWord w; w.lo = val; w.hi = 0;
        return w;
    }
};

// (action x role column) pairs of one row if its conditions hold: a needed condition bit that is clear zeroes the role columns
CB_HD uint32_t cond_bit(const CondWord v, uint32_t u) { return (uint32_t)(((u & 64u) ? v.hi : v.lo) >> (u & 63u)) & 1u; }
template <typename RP, int kForm>
CB_HD uint32_t uc_row_pairs(const U4 r, const RP rp, const CondWord v, const uint32_t role_all) {
    const uint32_t vlo = (uint32_t)v.lo, vhi = (uint32_t)(v.lo >> 32);
    const uint32_t miss = kForm == CB_UC_FORM_MASK32   ? r.y & ~vlo
                          : kForm == CB_UC_FORM_MASK64 ? (r.y & ~vlo) | (r.z & ~vhi)
                                                       : (cond_bit(v, r.y & 0xFFu) & cond_bit(v, (r.y >> 8) & 0xFFu)) ^ 1u;
    const uint32_t rc = miss ? 0u : (uint32_t)(rp >> r.w) & role_all;
    return r.x * rc;
}
// The scope-chain walk of the unique-condition body: per scope the DENY rows, then the ALLOW rows, each row three or
// four ALU operations on registers.  One 16-byte step record per scope (cb_uc.h: the chain descriptors, indexed like
// RES_BLOCK_MAP) gives the row ranges and the next scope of the chain, so a scope costs one table load ahead of its rows.
// RP: the role table word (32 bits when every role field fits, else 64); kForm: how the rows name their conditions
// (known when the kernel is generated for a table).
template <typename RP, int kForm, typename Rows>
CB_HD uint32_t uc_walk(const TableView t, const Rows rows, const RP rp, const CondWord val, const uint32_t r0, const uint32_t bm_base,
                       const uint32_t aset_base, const uint32_t role_all, uint32_t alive) {
    uint32_t allow_pairs = 0;
    const U4 *chain = t.uc_chain() + bm_base;
    for (uint32_t s = r0; s != CB_NONE32 && alive;) {
        const U4 d = ld16(chain + s);   // {first DENY row, first ALLOW row, end of the ALLOW rows, next scope}
        uint32_t D = 0, A = 0;          // DENY / ALLOW pair masks of this scope
        uint32_t ri = d.x;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
        for (; ri < d.y; ri++) D |= uc_row_pairs<RP, kForm>(rows.get(aset_base, ri), rp, val, role_all) & alive;
        alive &= ~D;
#if defined(__CUDA_ARCH__)
#pragma unroll 4
#endif
        for (; ri < d.z; ri++) A |= uc_row_pairs<RP, kForm>(rows.get(aset_base, ri), rp, val, role_all) & alive;
        allow_pairs |= A;   // ALLOW rows are listed only where they count (SCOPE_PERM)
        alive &= ~A;
        s = d.w;
    }
    return allow_pairs;
}

template <typename Cols, typename Rows, typename Conds = GenericConds>
CB_HD bool eval_request_uc(const TableView t, const BatchView &b, const Cols &cols, const Rows rows, uint64_t n, uint8_t *bitmap, uint8_t *effects,
                           const Conds conds = Conds()) {
    const U4 h0 = cols.hdr0();         // principal_id, kind (pattern id), resource_scope, principal_scope
    const uint64_t h1 = cols.hdr1();   // rv u16 | pv u16 | action_set_id u32
    const auto regs = conds.load(t, b, cols);   // specialised build: every attribute slot (and list) the table reads, in flight at once
    const uint32_t pid = h0.x, kc = h0.y, rscope = h0.z;
    const uint32_t rv = (uint32_t)(h1 & 0xFFFF), pv = (uint32_t)((h1 >> 16) & 0xFFFF), aset = (uint32_t)(h1 >> 32);
    const uint32_t RC = b.role_cols, RCP = b.rcp;
    const uint32_t K = aset < b.n_asets ? cols.aset_k(aset) : 0;
    uint64_t rp = 0;          // role table: RCP bits per table role
    uint32_t n_roles = 0;
    for (uint32_t i = 0; i < RC; i++) {
        uint32_t rr = cols.role(i);
        n_roles = rr != CB_ROLE_PAD ? i + 1 : n_roles;
        rp |= rr < t.L->nR ? 1ull << (rr * RCP + i) : 0ull;
    }
    if (pv != rv) return true;   // existence checks matter only then (ruletable.go:852-863): general body
    uint32_t acc = 0;
    const bool live = n_roles != 0 && K != 0 && rv != CB_NONE16 && kc != CB_KIND_NONE;
#ifdef CB_UC_STUB_WALK   // tools/uc_variants.sh: no scope chain, no rows (wrong results)
    const uint32_t r0 = live ? rscope & 0xFFFFu : CB_NONE32;
#else
    const uint32_t r0 = live ? chain_start(t, rscope, CB_SCOPE_FLAG_RESOURCE, (b.flags & CB_BATCH_FLAG_LENIENT) != 0) : CB_NONE32;
#endif
    if (r0 != CB_NONE32) {
        bool slow = false;
        const CondWord val = conds(t, b, regs, pid, n, slow);   // bit u: distinct condition u holds; bit 0: "no condition"
        if (slow) return true;
        const uint32_t role_all = (1u << n_roles) - 1;
        const uint32_t aset_base = aset * b.n_rows;
        const uint32_t amask = K * RC >= 32 ? b.stride_pattern : b.stride_pattern & ((1u << (K * RC)) - 1);   // bit kk*RC per action
        const uint32_t alive0 = amask * role_all;
        const uint32_t bm_base = (rv * t.L->nRP + kc) * t.L->nS;
        uint32_t allow_pairs;
#ifdef CB_UC_STUB_WALK
        allow_pairs = alive0 & ((uint32_t)val.lo ^ (uint32_t)(val.lo >> 32) ^ (uint32_t)rp ^ r0 ^ bm_base ^ aset_base);
        (void)rows;
#else
        // the role table gets one more field, "any role"; when it all fits 32 bits the per-row shift is a single SHF
        if ((t.L->nR + 1) * RCP <= 32) allow_pairs = uc_walk<uint32_t, Conds::kForm>(t, rows, (uint32_t)rp | role_all << (t.L->nR * RCP), val, r0, bm_base, aset_base, role_all, alive0);
        else allow_pairs = uc_walk<uint64_t, Conds::kForm>(t, rows, rp | (uint64_t)role_all << (t.L->nR * RCP), val, r0, bm_base, aset_base, role_all, alive0);
#endif
        // fold: an action is ALLOWed iff some role column allowed it; then pack the stride-RC bits
        uint32_t x = allow_pairs;
        x |= RC > 1 ? allow_pairs >> 1 : 0u;
        x |= RC > 2 ? allow_pairs >> 2 : 0u;
        x |= RC > 3 ? allow_pairs >> 3 : 0u;
        for (uint32_t j = 4; j < RC; j++) x |= allow_pairs >> j;
        x &= amask;
        if (RC == 1) acc = x;
        else if (RC == 2) { x = (x | x >> 1) & 0x33333333u; x = (x | x >> 2) & 0x0F0F0F0Fu; x = (x | x >> 4) & 0x00FF00FFu; acc = (x | x >> 8) & 0xFFFFu; }
        else if (RC == 3) { x = (x | x >> 2) & 0xC30C30C3u; x = (x | x >> 4) & 0x0F00F00Fu; x = (x | x >> 8) & 0xFF0000FFu; acc = (x | x >> 16) & 0x7FFu; }
        else if (RC == 4) { x = (x | x >> 3) & 0x03030303u; x = (x | x >> 6) & 0x000F000Fu; acc = (x | x >> 12) & 0xFFu; }
        else for (uint32_t kk = 0; kk < K; kk++) acc |= ((x >> (kk * RC)) & 1) << kk;
    }
    store_result(b, cols, n, bitmap, effects, K, acc);
    return false;
}

#ifndef CB_LEAN_ONLY
// out-of-line general body for the requests the fast body defers
CB_HD_NOINLINE void eval_request_general(const uint8_t *base, const TableLayout *L, const BatchView *b, uint64_t n, uint8_t *bitmap,
                                         uint8_t *effects, uint32_t *status) {
    TableView t; t.base = base; t.L = L;
    eval_request<uint64_t>(t, *b, n, bitmap, effects, status);
}

#endif  // !CB_LEAN_ONLY

}  // namespace cb
