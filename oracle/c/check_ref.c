/*
 * oracle/c/check_ref.c -- CPU oracle #2 and CPU baseline ("port").  TEST INFRASTRUCTURE ONLY:
 * nothing under cerbos_b200/ links or calls this; it checks the CUDA path and is the timed
 * cpu_baseline in bench.py.
 *
 * A scalar, plain-C interpreter of the flattened table blob (include/cerbos_b200_format.h) over the
 * same SoA request columns the GPU consumes.  It is written independently of the CUDA kernels and
 * keeps the reference's loop structure (action -> policy kind -> role -> scope -> rows) instead of the
 * kernels' bit-parallel formulation, so a flattening bug and a kernel bug cannot cancel out:
 *
 *   decision walk             internal/ruletable/ruletable.go:885-1152   (check_request)
 *   scope chains              ruletable.go:611-645                        (build_chain)
 *   existence checks          internal/ruletable/index/index.go:1089-1172 (p_exists / r_exists)
 *   role-policy DENY synthesis index.go:688-776                           (rolepol_denies)
 *   row predicate             index.go:91-116                             (row loop)
 *   parent roles              index.go:805-881                            (role_in_pr)
 *   condition leaf rule       ruletable.go:1425-1441 (error / non-bool => false)  (OP_TO_COND)
 *   CEL operator semantics    cel-go v0.27.0 (go.mod:45, not vendored): restated from the CEL spec,
 *                             pinned through oracle #1 (oracle/celeval.py) on the reference goldens.
 *   Cerbos set functions      internal/conditions/cerbos_lib.go:323-431 incl. the Go-map fast path
 *                             (convertToMap :370-389) whose key identity is (type, value).
 *
 * Build: see oracle/c/Makefile (gcc -O2 -shared -fPIC -pthread).
 */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "cerbos_b200_format.h"

typedef struct {
    uint64_t n_requests;
    uint32_t max_actions;
    int64_t now_unix_nanos;
    uint32_t flags;
    const void *const *columns;
    const size_t *column_bytes;
    uint32_t n_columns;
} cref_batch;

enum { COL_HDR0, COL_HDR1, COL_ROLES, COL_SLOTS, COL_HEAP, COL_BSTR_OFF, COL_BSTR_BYTES, COL_CLASS_OFF,
       COL_CLASS_PATS, COL_ASET_K, COL_ASET_SPREAD, COL_ROW_AM, N_COLS };

#define CREF_OK 0
#define CREF_ERR_BLOB (-1)
#define CREF_ERR_UNSUPPORTED (-2)
#define CREF_ERR_BATCH (-3)

typedef struct {
    const uint32_t *meta;
    const uint32_t *scope_parent, *scope_flags, *res_block_map, *prin_block_map, *prin_of_string;
    const uint8_t *res_exists, *prin_exists;
    const cb_block *blocks;
    const cb_row *rows;
    const cb_cond *conds;
    const cb_instr *code;
    const cb_const *consts;
    const uint64_t *theap;
    const uint32_t *str_off;
    const uint8_t *str_bytes;
    const uint32_t *par_off, *par_list, *rp_off, *rp_apats, *row_apats;
    const cb_rolepol_entry *rp_entries;
    const cb_rolepol_rule *rp_rules;
    uint32_t nV, nRP, nS, nP, nR, nAP, nT, n_slots, n_conds;
} table_t;

typedef struct {
    const table_t *t;
    const cref_batch *b;
    const cb_hdr0 *hdr0;
    const cb_hdr1 *hdr1;
    const uint32_t *roles;
    const uint64_t *slots, *heap, *aset_spread;
    const uint32_t *bstr_off, *class_off, *class_pats, *aset_k;
    const uint8_t *bstr_bytes;
    uint32_t role_cols, n_asets, kc, n_pass;
    uint64_t N;
} batch_t;

static int load_table(const void *blob, size_t len, table_t *t) {
    if (len < sizeof(cb_blob_header)) return CREF_ERR_BLOB;
    const cb_blob_header *h = (const cb_blob_header *)blob;
    if (h->magic != CB_MAGIC || h->version != CB_VERSION || h->total_bytes > len) return CREF_ERR_BLOB;
    const cb_section_desc *d = (const cb_section_desc *)((const char *)blob + sizeof(cb_blob_header));
    memset(t, 0, sizeof(*t));
    for (uint32_t i = 0; i < h->n_sections; i++) {
        const void *p = (const char *)blob + d[i].offset;
        if (d[i].offset + d[i].n_bytes > len) return CREF_ERR_BLOB;
        switch (d[i].id) {
        case CB_SEC_META: t->meta = p; break;
        case CB_SEC_SCOPE_PARENT: t->scope_parent = p; break;
        case CB_SEC_SCOPE_FLAGS: t->scope_flags = p; break;
        case CB_SEC_RES_BLOCK_MAP: t->res_block_map = p; break;
        case CB_SEC_RES_EXISTS: t->res_exists = p; break;
        case CB_SEC_PRIN_BLOCK_MAP: t->prin_block_map = p; break;
        case CB_SEC_PRIN_EXISTS: t->prin_exists = p; break;
        case CB_SEC_PRIN_OF_STRING: t->prin_of_string = p; break;
        case CB_SEC_BLOCKS: t->blocks = p; break;
        case CB_SEC_ROWS: t->rows = p; break;
        case CB_SEC_CONDS: t->conds = p; break;
        case CB_SEC_CODE: t->code = p; break;
        case CB_SEC_CONSTS: t->consts = p; break;
        case CB_SEC_THEAP: t->theap = p; break;
        case CB_SEC_STR_OFF: t->str_off = p; break;
        case CB_SEC_STR_BYTES: t->str_bytes = p; break;
        case CB_SEC_ROLE_PARENTS_OFF: t->par_off = p; break;
        case CB_SEC_ROLE_PARENTS: t->par_list = p; break;
        case CB_SEC_ROLEPOL_OFF: t->rp_off = p; break;
        case CB_SEC_ROLEPOL_ENTRIES: t->rp_entries = p; break;
        case CB_SEC_ROLEPOL_RULES: t->rp_rules = p; break;
        case CB_SEC_ROLEPOL_APATS: t->rp_apats = p; break;
        case CB_SEC_ROW_APATS: t->row_apats = p; break;
        default: break;
        }
    }
    if (!t->meta || !t->rows || !t->blocks || !t->code) return CREF_ERR_BLOB;
    t->nV = t->meta[CB_META_N_VERSIONS]; t->nRP = t->meta[CB_META_N_RESPATS]; t->nS = t->meta[CB_META_N_SCOPES];
    t->nP = t->meta[CB_META_N_PRINCIPALS]; t->nR = t->meta[CB_META_N_ROLES]; t->nAP = t->meta[CB_META_N_APATS];
    t->nT = t->meta[CB_META_N_STRINGS]; t->n_slots = t->meta[CB_META_N_SLOTS]; t->n_conds = t->meta[CB_META_N_CONDS];
    return CREF_OK;
}

/* ------------------------------------------------------------------------------------------- values */
typedef struct { uint32_t tag; uint64_t u; } val_t;
#define HEAP_BATCH (1ull << 63)   /* internal: list/map ref lives in the batch heap */

static inline val_t mk(uint32_t tag, uint64_t u) { val_t v; v.tag = tag; v.u = u; return v; }
static inline val_t mk_err(void) { return mk(CB_T_ERR, 0); }
static inline val_t mk_bool(int b) { return mk(CB_T_BOOL, b ? 1 : 0); }
static inline val_t mk_int(int64_t i) { return mk(CB_T_INT, (uint64_t)i); }
static inline val_t mk_double(double d) {
    uint64_t u;
    if (d != d) u = CB_V64_CANON_NAN; else memcpy(&u, &d, 8);
    return mk(CB_T_DOUBLE, u);
}
static inline double as_double(val_t v) { double d; memcpy(&d, &v.u, 8); return d; }

/* slot state returned next to the decoded value */
enum { SLOT_VALUE, SLOT_ABSENT, SLOT_ERROR };

static val_t decode_v64(uint64_t bits, int *state) {
    if (state) *state = SLOT_VALUE;
    if ((bits >> 52) == 0xFFF && ((bits >> 48) & 0xF) != 0) {
        uint32_t tag = (uint32_t)((bits >> 48) & 0xF);
        uint64_t pay = bits & 0xFFFFFFFFFFFFull;
        switch (tag) {
        case CB_V64_NULL: return mk(CB_T_NULL, 0);
        case CB_V64_BOOL: return mk_bool(pay != 0);
        case CB_V64_STRING: return mk(CB_T_STRING, pay);
        case CB_V64_LIST:
        case CB_V64_MAP: {
            uint64_t off = pay & (CB_V64_HEAP_BATCH_BIT - 1);
            if (pay & CB_V64_HEAP_BATCH_BIT) off |= HEAP_BATCH;
            return mk(tag == CB_V64_LIST ? CB_T_LIST : CB_T_MAP, off);
        }
        case CB_V64_INT: {
            int64_t i = (int64_t)(pay << 16) >> 16;
            return mk_int(i);
        }
        case CB_V64_ABSENT: if (state) *state = SLOT_ABSENT; return mk_err();
        default: if (state) *state = SLOT_ERROR; return mk_err();
        }
    }
    return mk(CB_T_DOUBLE, bits);
}

typedef struct {
    const table_t *t;
    const batch_t *b;
    uint64_t req;
    int unsupported;
    val_t vars[CB_MAX_VARS];
} ectx_t;

static inline const uint64_t *heap_ptr(const ectx_t *c, uint64_t ref) {
    return (ref & HEAP_BATCH) ? c->b->heap + (ref & ~HEAP_BATCH) : c->t->theap + ref;
}
static inline void str_get(const ectx_t *c, uint64_t id, const uint8_t **p, uint32_t *len) {
    if (id < c->t->nT) { *p = c->t->str_bytes + c->t->str_off[id]; *len = c->t->str_off[id + 1] - c->t->str_off[id]; }
    else { uint64_t j = id - c->t->nT; *p = c->b->bstr_bytes + c->b->bstr_off[j]; *len = c->b->bstr_off[j + 1] - c->b->bstr_off[j]; }
}

static inline int is_num(val_t v) { return v.tag == CB_T_INT || v.tag == CB_T_UINT || v.tag == CB_T_DOUBLE; }

/* cel-go cross-type numeric compare: -1/0/1, 2 = unordered (NaN) */
static int num_cmp(val_t a, val_t b) {
    if (a.tag == CB_T_DOUBLE || b.tag == CB_T_DOUBLE) {
        if (a.tag == CB_T_DOUBLE && b.tag == CB_T_DOUBLE) {
            double x = as_double(a), y = as_double(b);
            if (x != x || y != y) return 2;
            return x < y ? -1 : (x > y ? 1 : 0);
        }
        int sign = 1;
        val_t dv = a, iv = b;
        if (a.tag != CB_T_DOUBLE) { dv = b; iv = a; sign = -1; }
        double d = as_double(dv);
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
    if (a.tag == CB_T_INT && b.tag == CB_T_INT) { int64_t x = (int64_t)a.u, y = (int64_t)b.u; return x < y ? -1 : (x > y ? 1 : 0); }
    if (a.tag == CB_T_UINT && b.tag == CB_T_UINT) return a.u < b.u ? -1 : (a.u > b.u ? 1 : 0);
    if (a.tag == CB_T_INT) { /* int vs uint */
        int64_t x = (int64_t)a.u;
        if (x < 0) return -1;
        return (uint64_t)x < b.u ? -1 : ((uint64_t)x > b.u ? 1 : 0);
    }
    { int64_t y = (int64_t)b.u; if (y < 0) return 1; return a.u < (uint64_t)y ? -1 : (a.u > (uint64_t)y ? 1 : 0); }
}

static int val_equal(ectx_t *c, val_t a, val_t b, int depth);

static int list_equal(ectx_t *c, val_t a, val_t b, int depth) {
    const uint64_t *pa = heap_ptr(c, a.u), *pb = heap_ptr(c, b.u);
    if (pa[0] != pb[0]) return 0;
    for (uint64_t i = 0; i < pa[0]; i++)
        if (!val_equal(c, decode_v64(pa[1 + i], 0), decode_v64(pb[1 + i], 0), depth + 1)) return 0;
    return 1;
}

static int map_find(ectx_t *c, val_t m, val_t key, val_t *out) {
    const uint64_t *p = heap_ptr(c, m.u);
    uint64_t n = p[0];
    /* keys are scalars: strings (JSON maps), ints / uints / bools (map literals); a number finds a numerically equal key of
     * another numeric type (cel-go maps look a key up across int / uint / double) */
    if (key.tag != CB_T_STRING && key.tag != CB_T_BOOL && !is_num(key)) return 0;
    for (uint64_t i = 0; i < n; i++) {
        val_t k = decode_v64(p[1 + i], 0);
        int same = (is_num(k) && is_num(key)) ? num_cmp(k, key) == 0 : (k.tag == key.tag && k.u == key.u);
        if (same) { if (out) *out = decode_v64(p[1 + n + i], 0); return 1; }
    }
    return 0;
}

static int map_equal(ectx_t *c, val_t a, val_t b, int depth) {
    const uint64_t *pa = heap_ptr(c, a.u), *pb = heap_ptr(c, b.u);
    if (pa[0] != pb[0]) return 0;
    uint64_t n = pa[0];
    for (uint64_t i = 0; i < n; i++) {
        val_t ov;
        if (!map_find(c, b, decode_v64(pa[1 + i], 0), &ov)) return 0;
        if (!val_equal(c, decode_v64(pa[1 + n + i], 0), ov, depth + 1)) return 0;
    }
    return 1;
}

/* heterogeneous equality (cel-go types.Equal): mismatched types are simply unequal */
static int val_equal(ectx_t *c, val_t a, val_t b, int depth) {
    if (depth > 32) { c->unsupported = 1; return 0; }
    if (is_num(a) && is_num(b)) return num_cmp(a, b) == 0;
    if (a.tag != b.tag) return 0;
    switch (a.tag) {
    case CB_T_NULL: return 1;
    case CB_T_BOOL: case CB_T_STRING: case CB_T_TS: case CB_T_DUR: return a.u == b.u;
    case CB_T_LIST: return list_equal(c, a, b, depth);
    case CB_T_MAP: return map_equal(c, a, b, depth);
    default: return 0;
    }
}

static int str_cmp(ectx_t *c, uint64_t ia, uint64_t ib) {
    const uint8_t *pa, *pb; uint32_t la, lb;
    str_get(c, ia, &pa, &la); str_get(c, ib, &pb, &lb);
    uint32_t m = la < lb ? la : lb;
    int r = memcmp(pa, pb, m);
    if (r) return r < 0 ? -1 : 1;
    return la < lb ? -1 : (la > lb ? 1 : 0);
}

/* ordering: returns -1/0/1, or 3 = error (no overload / NaN) */
static int val_order(ectx_t *c, val_t a, val_t b) {
    if (is_num(a) && is_num(b)) { int r = num_cmp(a, b); return r == 2 ? 3 : r; }
    if (a.tag != b.tag) return 3;
    switch (a.tag) {
    case CB_T_BOOL: return a.u < b.u ? -1 : (a.u > b.u ? 1 : 0);
    case CB_T_STRING: return a.u == b.u ? 0 : str_cmp(c, a.u, b.u);
    case CB_T_TS: case CB_T_DUR: { int64_t x = (int64_t)a.u, y = (int64_t)b.u; return x < y ? -1 : (x > y ? 1 : 0); }
    default: return 3;
    }
}

static val_t do_cmp(ectx_t *c, int ci, val_t a, val_t b) {
    if (a.tag == CB_T_ERR || b.tag == CB_T_ERR) return mk_err();
    if (ci == 0) return mk_bool(val_equal(c, a, b, 0));
    if (ci == 1) return mk_bool(!val_equal(c, a, b, 0));
    int r = val_order(c, a, b);
    if (r == 3) return mk_err();
    switch (ci) {
    case 2: return mk_bool(r < 0);
    case 3: return mk_bool(r <= 0);
    case 4: return mk_bool(r > 0);
    default: return mk_bool(r >= 0);
    }
}

static val_t do_in(ectx_t *c, val_t x, val_t cont) {
    if (x.tag == CB_T_ERR || cont.tag == CB_T_ERR) return mk_err();
    if (cont.tag == CB_T_LIST) {
        const uint64_t *p = heap_ptr(c, cont.u);
        for (uint64_t i = 0; i < p[0]; i++)
            if (val_equal(c, x, decode_v64(p[1 + i], 0), 0)) return mk_bool(1);
        return mk_bool(0);
    }
    if (cont.tag == CB_T_MAP) return mk_bool(map_find(c, cont, x, 0));
    return mk_err();
}

static val_t do_index(ectx_t *c, val_t cont, val_t key) {
    if (cont.tag == CB_T_ERR || key.tag == CB_T_ERR) return mk_err();
    if (cont.tag == CB_T_LIST) {
        int64_t idx;
        if (key.tag == CB_T_INT) idx = (int64_t)key.u;
        else if (key.tag == CB_T_UINT) { if (key.u > (uint64_t)INT64_MAX) return mk_err(); idx = (int64_t)key.u; }
        else if (key.tag == CB_T_DOUBLE) {
            double d = as_double(key);
            if (!(d == floor(d)) || !(fabs(d) < 9.2e18)) return mk_err();
            idx = (int64_t)d;
        } else return mk_err();
        const uint64_t *p = heap_ptr(c, cont.u);
        if (idx < 0 || (uint64_t)idx >= p[0]) return mk_err();
        return decode_v64(p[1 + idx], 0);
    }
    if (cont.tag == CB_T_MAP) { val_t out; if (map_find(c, cont, key, &out)) return out; return mk_err(); }
    return mk_err();
}

static uint32_t utf8_len(const uint8_t *p, uint32_t n) {
    uint32_t k = 0;
    for (uint32_t i = 0; i < n; i++) if ((p[i] & 0xC0) != 0x80) k++;
    return k;
}

/* ---- Cerbos set helpers: Go-map fast path identity is (dynamic type, value) (cerbos_lib.go:370-389) ---- */
static int hashable(val_t v) { return v.tag == CB_T_STRING || v.tag == CB_T_INT || v.tag == CB_T_UINT || v.tag == CB_T_DOUBLE || v.tag == CB_T_DUR || v.tag == CB_T_TS; }
static int uses_map(ectx_t *c, val_t b) {
    const uint64_t *p = heap_ptr(c, b.u);
    if (p[0] <= 3) return 0;
    for (uint64_t i = 0; i < p[0]; i++) if (!hashable(decode_v64(p[1 + i], 0))) return 0;
    return 1;
}
static int key_identical(val_t a, val_t b) {
    if (a.tag != b.tag) return 0;
    if (a.tag == CB_T_DOUBLE) { double x = as_double(a), y = as_double(b); return x == y; } /* NaN never, +0 == -0 */
    return a.u == b.u;
}
static int member(ectx_t *c, int use_map, val_t b, val_t x) {
    const uint64_t *p = heap_ptr(c, b.u);
    for (uint64_t i = 0; i < p[0]; i++) {
        val_t e = decode_v64(p[1 + i], 0);
        if (use_map ? key_identical(x, e) : val_equal(c, x, e, 0)) return 1;
    }
    return 0;
}
static val_t do_has_intersection(ectx_t *c, val_t a, val_t b) {
    if (a.tag != CB_T_LIST || b.tag != CB_T_LIST) return mk_err();
    if (heap_ptr(c, a.u)[0] > heap_ptr(c, b.u)[0]) { val_t t = a; a = b; b = t; }
    int um = uses_map(c, b);
    const uint64_t *p = heap_ptr(c, a.u);
    for (uint64_t i = 0; i < p[0]; i++) if (member(c, um, b, decode_v64(p[1 + i], 0))) return mk_bool(1);
    return mk_bool(0);
}
static val_t do_is_subset(ectx_t *c, val_t a, val_t b) {
    if (a.tag != CB_T_LIST || b.tag != CB_T_LIST) return mk_err();
    int um = uses_map(c, b);
    const uint64_t *p = heap_ptr(c, a.u);
    for (uint64_t i = 0; i < p[0]; i++) if (!member(c, um, b, decode_v64(p[1 + i], 0))) return mk_bool(0);
    return mk_bool(1);
}

/* ---- arithmetic ---- */
static val_t do_arith(ectx_t *c, int op, val_t a, val_t b) {
    if (a.tag == CB_T_ERR || b.tag == CB_T_ERR) return mk_err();
    if (a.tag == CB_T_INT && b.tag == CB_T_INT) {
        int64_t x = (int64_t)a.u, y = (int64_t)b.u, r;
        switch (op) {
        case CB_OP_ADD: if (__builtin_add_overflow(x, y, &r)) return mk_err(); return mk_int(r);
        case CB_OP_SUB: if (__builtin_sub_overflow(x, y, &r)) return mk_err(); return mk_int(r);
        case CB_OP_MUL: if (__builtin_mul_overflow(x, y, &r)) return mk_err(); return mk_int(r);
        case CB_OP_DIV: if (y == 0 || (x == INT64_MIN && y == -1)) return mk_err(); return mk_int(x / y);
        default: if (y == 0 || (x == INT64_MIN && y == -1)) return mk_err(); return mk_int(x % y);
        }
    }
    if (a.tag == CB_T_UINT && b.tag == CB_T_UINT) {
        uint64_t x = a.u, y = b.u, r;
        switch (op) {
        case CB_OP_ADD: if (__builtin_add_overflow(x, y, &r)) return mk_err(); return mk(CB_T_UINT, r);
        case CB_OP_SUB: if (y > x) return mk_err(); return mk(CB_T_UINT, x - y);
        case CB_OP_MUL: if (__builtin_mul_overflow(x, y, &r)) return mk_err(); return mk(CB_T_UINT, r);
        case CB_OP_DIV: if (y == 0) return mk_err(); return mk(CB_T_UINT, x / y);
        default: if (y == 0) return mk_err(); return mk(CB_T_UINT, x % y);
        }
    }
    if (a.tag == CB_T_DOUBLE && b.tag == CB_T_DOUBLE) {
        double x = as_double(a), y = as_double(b);
        switch (op) {
        case CB_OP_ADD: return mk_double(x + y);
        case CB_OP_SUB: return mk_double(x - y);
        case CB_OP_MUL: return mk_double(x * y);
        case CB_OP_DIV: return mk_double(x / y);
        default: return mk_err();
        }
    }
    /* time arithmetic */
    int64_t x = (int64_t)a.u, y = (int64_t)b.u, r;
    if (op == CB_OP_ADD) {
        if ((a.tag == CB_T_TS && b.tag == CB_T_DUR) || (a.tag == CB_T_DUR && b.tag == CB_T_TS)) {
            if (__builtin_add_overflow(x, y, &r)) { c->unsupported = 1; return mk_err(); }
            return mk(CB_T_TS, (uint64_t)r);
        }
        if (a.tag == CB_T_DUR && b.tag == CB_T_DUR) { if (__builtin_add_overflow(x, y, &r)) return mk_err(); return mk(CB_T_DUR, (uint64_t)r); }
    }
    if (op == CB_OP_SUB) {
        if (a.tag == CB_T_TS && b.tag == CB_T_TS) { if (__builtin_sub_overflow(x, y, &r)) return mk_err(); return mk(CB_T_DUR, (uint64_t)r); }
        if (a.tag == CB_T_TS && b.tag == CB_T_DUR) { if (__builtin_sub_overflow(x, y, &r)) { c->unsupported = 1; return mk_err(); } return mk(CB_T_TS, (uint64_t)r); }
        if (a.tag == CB_T_DUR && b.tag == CB_T_DUR) { if (__builtin_sub_overflow(x, y, &r)) return mk_err(); return mk(CB_T_DUR, (uint64_t)r); }
    }
    if ((a.tag == CB_T_STRING && b.tag == CB_T_STRING && op == CB_OP_ADD) || (a.tag == CB_T_LIST && b.tag == CB_T_LIST && op == CB_OP_ADD)) {
        c->unsupported = 1;   /* string / list concatenation needs allocation: rejected by the compiler normally */
        return mk_err();
    }
    return mk_err();
}

/* ---- string predicates ---- */
static val_t do_str2(ectx_t *c, int op, val_t s, val_t t) {
    if (s.tag != CB_T_STRING || t.tag != CB_T_STRING) return mk_err();
    const uint8_t *ps, *pt; uint32_t ls, lt;
    str_get(c, s.u, &ps, &ls); str_get(c, t.u, &pt, &lt);
    if (lt > ls) return mk_bool(0);
    if (op == CB_OP_STARTS_WITH) return mk_bool(memcmp(ps, pt, lt) == 0);
    if (op == CB_OP_ENDS_WITH) return mk_bool(memcmp(ps + ls - lt, pt, lt) == 0);
    if (lt == 0) return mk_bool(1);
    for (uint32_t i = 0; i + lt <= ls; i++) if (memcmp(ps + i, pt, lt) == 0) return mk_bool(1);
    return mk_bool(0);
}

/* ---- Go time.ParseDuration, restated after the standard library's loop (leadingInt / leadingFraction / unit map) ---- */
static int parse_go_duration(const uint8_t *s, uint32_t n, int64_t *out) {   /* 0 ok, 1 error, 2 not representable here */
    uint32_t i = 0; int neg = 0;
    if (n == 0) return 1;
    if (s[0] == '-' || s[0] == '+') { neg = s[0] == '-'; i++; }
    if (n - i == 1 && s[i] == '0') { *out = 0; return 0; }
    if (i == n) return 1;
    unsigned __int128 d = 0;   /* arbitrary-precision enough: range-checked at the end like the Python oracle */
    while (i < n) {
        unsigned __int128 v = 0, f = 0, scale = 1; int pre = 0, post = 0, nd = 0;
        while (i < n && s[i] >= '0' && s[i] <= '9') { if (v < ((unsigned __int128)1 << 100)) v = v * 10 + (s[i] - '0'); pre = 1; i++; }
        if (i < n && s[i] == '.') {
            i++;
            while (i < n && s[i] >= '0' && s[i] <= '9') { if (++nd > 25) return 2; f = f * 10 + (s[i] - '0'); scale *= 10; post = 1; i++; }
        }
        if (!pre && !post) return 1;
        uint64_t unit;
        if (i + 1 < n && s[i] == 'n' && s[i + 1] == 's') { unit = 1; i += 2; }
        else if (i + 1 < n && s[i] == 'u' && s[i + 1] == 's') { unit = 1000; i += 2; }
        else if (i + 2 < n && ((s[i] == 0xC2 && s[i + 1] == 0xB5) || (s[i] == 0xCE && s[i + 1] == 0xBC)) && s[i + 2] == 's') { unit = 1000; i += 3; }
        else if (i + 1 < n && s[i] == 'm' && s[i + 1] == 's') { unit = 1000000; i += 2; }
        else if (i < n && s[i] == 's') { unit = 1000000000ull; i += 1; }
        else if (i < n && s[i] == 'm') { unit = 60000000000ull; i += 1; }
        else if (i < n && s[i] == 'h') { unit = 3600000000000ull; i += 1; }
        else return 1;
        d += v * unit + f * unit / scale;
        if (d > ((unsigned __int128)1 << 110)) return 1;
    }
    const unsigned __int128 lim = (unsigned __int128)1 << 63;
    if (neg) { if (d > lim) return 1; *out = d == lim ? INT64_MIN : -(int64_t)(uint64_t)d; return 0; }
    if (d > lim - 1) return 1;
    *out = (int64_t)(uint64_t)d;
    return 0;
}

/* ---- timestamp / duration accessors (UTC): cel-go timestamp.getFullYear() ... duration.getMilliseconds() ---- */
static int64_t fdiv(int64_t a, int64_t b) { int64_t q = a / b, r = a % b; return (r != 0 && ((r < 0) != (b < 0))) ? q - 1 : q; }
static val_t do_ts_get(uint32_t field, val_t v, uint32_t tzform, int32_t offset_s) {
    int64_t ns = (int64_t)v.u;
    if (field == 0xFF) return mk_err();   /* invalid zone text */
    if (v.tag == CB_T_DUR) {
        if (tzform) return mk_err();
        if (field == CB_TS_GETHOURS) return mk(CB_T_INT, (uint64_t)(ns / 3600000000000ll));
        if (field == CB_TS_GETMINUTES) return mk(CB_T_INT, (uint64_t)(ns / 60000000000ll));
        if (field == CB_TS_GETSECONDS) return mk(CB_T_INT, (uint64_t)(ns / 1000000000ll));
        if (field == CB_TS_GETMILLISECONDS) return mk(CB_T_INT, (uint64_t)(ns / 1000000ll));
        return mk_err();
    }
    if (v.tag != CB_T_TS) return mk_err();
    int64_t secs = fdiv(ns, 1000000000ll), sub = ns - secs * 1000000000ll;
    secs += offset_s;   /* fixed zone offset east of UTC (cel-go timeZone(): "[+-]HH:MM" forms) */
    int64_t days = fdiv(secs, 86400), rem = secs - days * 86400;
    /* walk years / months from 1970 (independent of the kernels' closed-form civil_from_days) */
    int64_t y = 1970, dd = days;
    for (;;) {
        int leap = (y % 4 == 0 && y % 100 != 0) || y % 400 == 0;
        int64_t yl = leap ? 366 : 365;
        if (dd < 0) { y--; leap = (y % 4 == 0 && y % 100 != 0) || y % 400 == 0; dd += leap ? 366 : 365; continue; }
        if (dd >= yl) { dd -= yl; y++; continue; }
        break;
    }
    int leap = (y % 4 == 0 && y % 100 != 0) || y % 400 == 0;
    static const int ml[12] = {31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
    int64_t doy = dd; int m = 0;
    while (m < 12) { int l = ml[m] + (m == 1 && leap); if (dd < l) break; dd -= l; m++; }
    switch (field) {
    case CB_TS_GETFULLYEAR: return mk(CB_T_INT, (uint64_t)y);
    case CB_TS_GETMONTH: return mk(CB_T_INT, (uint64_t)m);
    case CB_TS_GETDAYOFYEAR: return mk(CB_T_INT, (uint64_t)doy);
    case CB_TS_GETDAYOFMONTH: return mk(CB_T_INT, (uint64_t)dd);
    case CB_TS_GETDATE: return mk(CB_T_INT, (uint64_t)(dd + 1));
    case CB_TS_GETDAYOFWEEK: return mk(CB_T_INT, (uint64_t)(((days + 4) % 7 + 7) % 7));
    case CB_TS_GETHOURS: return mk(CB_T_INT, (uint64_t)(rem / 3600));
    case CB_TS_GETMINUTES: return mk(CB_T_INT, (uint64_t)(rem % 3600 / 60));
    case CB_TS_GETSECONDS: return mk(CB_T_INT, (uint64_t)(rem % 60));
    default: return mk(CB_T_INT, (uint64_t)(sub / 1000000));
    }
}

/* ---- hierarchy(s, delim): conditions/types/hierarchy.go:146-410.  Restated the way the reference does it: split into
 * segments (strings.Split), then compare the segment lists. ---- */
#define HIER_MAX_SEG 256
typedef struct { const uint8_t *p[HIER_MAX_SEG]; uint32_t l[HIER_MAX_SEG]; uint32_t n; } hier_t;
static int hier_split(ectx_t *c, val_t v, uint32_t delim_id, hier_t *h) {
    if (v.tag != CB_T_STRING) { if (v.tag == CB_T_LIST) c->unsupported = 1; return 0; }   /* hierarchy(list): not lowered */
    const uint8_t *s, *d; uint32_t ls, ld;
    str_get(c, v.u, &s, &ls); str_get(c, delim_id, &d, &ld);
    h->n = 0;
    uint32_t start = 0, i = 0;
    while (i + ld <= ls) {
        if (memcmp(s + i, d, ld) == 0) {
            if (h->n >= HIER_MAX_SEG - 1) { c->unsupported = 1; return 0; }
            h->p[h->n] = s + start; h->l[h->n] = i - start; h->n++;
            i += ld; start = i;
        } else i++;
    }
    h->p[h->n] = s + start; h->l[h->n] = ls - start; h->n++;
    return 1;
}
static int hier_seg_eq(const hier_t *a, uint32_t i, const hier_t *b, uint32_t j) { return a->l[i] == b->l[j] && memcmp(a->p[i], b->p[j], a->l[i]) == 0; }
static int hier_ancestor_of(const hier_t *h, const hier_t *child) {          /* hierarchy.go:283-299 */
    if (child->n <= h->n) return 0;
    for (uint32_t i = 0; i < h->n; i++) if (!hier_seg_eq(child, i, h, i)) return 0;
    return 1;
}
static int hier_immediate_parent_of(const hier_t *h, const hier_t *child) {  /* :343-359 */
    if (child->n != h->n + 1) return 0;
    for (uint32_t i = 0; i < h->n; i++) if (!hier_seg_eq(child, i, h, i)) return 0;
    return 1;
}
static uint32_t hier_common_ancestors(const hier_t *h, const hier_t *o) {    /* :301-326 -> number of ancestors (a prefix of either) */
    const hier_t *sh = h, *lo = o;
    if (o->n < h->n) { lo = h; sh = o; }
    uint32_t ns = sh->n, nl = lo->n;
    if (nl == ns) { nl--; ns--; }
    uint32_t k = 0;
    for (uint32_t i = 0; i < ns; i++) { if (!hier_seg_eq(lo, i, sh, i)) break; k++; }
    (void)nl;
    return k;
}
static val_t do_hier_rel(ectx_t *c, uint32_t rel, val_t x, uint32_t dx, val_t y, uint32_t dy) {
    static __thread hier_t a, b;
    int ok = hier_split(c, x, dx, &a);
    ok &= hier_split(c, y, dy, &b);
    if (!ok) return mk_err();
    switch (rel) {
    case CB_HIER_ANCESTOROF: return mk_bool(hier_ancestor_of(&a, &b));
    case CB_HIER_DESCENDENTOF: return mk_bool(hier_ancestor_of(&b, &a));                /* :328-335 */
    case CB_HIER_IMMEDIATEPARENTOF: return mk_bool(hier_immediate_parent_of(&a, &b));
    case CB_HIER_IMMEDIATECHILDOF: return mk_bool(hier_immediate_parent_of(&b, &a));     /* :337-341 */
    case CB_HIER_SIBLINGOF: {                                                             /* :361-377 */
        if (a.n != b.n) return mk_bool(0);
        for (uint32_t i = 0; i + 1 < a.n; i++) if (!hier_seg_eq(&a, i, &b, i)) return mk_bool(0);
        return mk_bool(1);
    }
    case CB_HIER_OVERLAPS: {                                                              /* :379-397 */
        const hier_t *sh = &a, *lo = &b;
        if (b.n < a.n) { lo = &a; sh = &b; }
        for (uint32_t i = 0; i < sh->n; i++) if (!hier_seg_eq(lo, i, sh, i)) return mk_bool(0);
        return mk_bool(1);
    }
    default: {                                                                            /* Equal, :231-248 */
        if (a.n != b.n) return mk_bool(0);
        for (uint32_t i = 0; i < a.n; i++) if (!hier_seg_eq(&a, i, &b, i)) return mk_bool(0);
        return mk_bool(1);
    }
    }
}

/* ---- RFC 3339 -> ns ---- */
static int64_t days_from_civil(int64_t y, int m, int d) {
    y -= m <= 2;
    int64_t era = (y >= 0 ? y : y - 399) / 400;
    int64_t yoe = y - era * 400;
    int64_t doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
    int64_t doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    return era * 146097 + doe - 719468;
}
static int dig(const uint8_t *p, int n, int *out) {
    int v = 0;
    for (int i = 0; i < n; i++) { if (p[i] < '0' || p[i] > '9') return 0; v = v * 10 + (p[i] - '0'); }
    *out = v; return 1;
}
static val_t parse_ts(ectx_t *c, val_t s) {
    const uint8_t *p; uint32_t n;
    str_get(c, s.u, &p, &n);
    int y, mo, d, h, mi, se;
    if (n < 20) return mk_err();
    if (!dig(p, 4, &y) || p[4] != '-' || !dig(p + 5, 2, &mo) || p[7] != '-' || !dig(p + 8, 2, &d) || p[10] != 'T' ||
        !dig(p + 11, 2, &h) || p[13] != ':' || !dig(p + 14, 2, &mi) || p[16] != ':' || !dig(p + 17, 2, &se)) return mk_err();
    uint32_t i = 19;
    int64_t ns = 0;
    if (p[i] == '.' || p[i] == ',') {
        i++;
        int k = 0;
        uint32_t st = i;
        while (i < n && p[i] >= '0' && p[i] <= '9') { if (k < 9) { ns = ns * 10 + (p[i] - '0'); k++; } i++; }
        if (i == st) return mk_err();
        while (k < 9) { ns *= 10; k++; }
    }
    if (i >= n) return mk_err();
    int64_t off = 0;
    if (p[i] == 'Z') { if (i + 1 != n) return mk_err(); }   /* Go's time.Parse: 'T' and 'Z' literally */
    else if (p[i] == '+' || p[i] == '-') {
        int oh, om;
        if (i + 6 != n || !dig(p + i + 1, 2, &oh) || p[i + 3] != ':' || !dig(p + i + 4, 2, &om) || oh > 24 || om > 60) return mk_err();   /* (Go's range test is `>`) */
        off = (oh * 3600 + om * 60) * (p[i] == '+' ? 1 : -1);
    } else return mk_err();
    int leap = (y % 4 == 0 && (y % 100 != 0 || y % 400 == 0));
    static const int dim[12] = {31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
    if (mo < 1 || mo > 12 || d < 1 || d > dim[mo - 1] + (mo == 2 && leap) || h > 23 || mi > 59 || se > 59) return mk_err();
    int64_t secs = days_from_civil(y, mo, d) * 86400 + h * 3600 + mi * 60 + se - off;
    if (secs < -62135596800ll || secs > 253402300799ll) return mk_err();   /* cel-go: the instant within 0001..9999 */
    int64_t total;
    if (__builtin_mul_overflow(secs, (int64_t)1000000000, &total) || __builtin_add_overflow(total, ns, &total)) {
        c->unsupported = 1;   /* valid CEL timestamp outside the int64-nanosecond device range */
        return mk_err();
    }
    return mk(CB_T_TS, (uint64_t)total);
}

/* ---- IP parsing (Go net.ParseIP) ---- */
static int parse_ipv4(const uint8_t *p, uint32_t n, uint32_t *out) {
    uint32_t v = 0; int parts = 0; uint32_t i = 0;
    while (parts < 4) {
        uint32_t st = i; int x = 0;
        while (i < n && p[i] >= '0' && p[i] <= '9') { x = x * 10 + (p[i] - '0'); i++; if (i - st > 3) return 0; }
        if (i == st || x > 255 || (i - st > 1 && p[st] == '0')) return 0;
        v = (v << 8) | (uint32_t)x; parts++;
        if (parts < 4) { if (i >= n || p[i] != '.') return 0; i++; }
    }
    if (i != n) return 0;
    *out = v; return 1;
}
static int hexv(uint8_t ch) { if (ch >= '0' && ch <= '9') return ch - '0'; if (ch >= 'a' && ch <= 'f') return ch - 'a' + 10; if (ch >= 'A' && ch <= 'F') return ch - 'A' + 10; return -1; }
static int parse_ipv6(const uint8_t *p, uint32_t n, uint16_t g[8]) {
    int ng = 0, ell = -1; uint32_t i = 0;
    if (n >= 2 && p[0] == ':' && p[1] == ':') { ell = 0; i = 2; if (i == n) { memset(g, 0, 16); return 1; } }
    else if (n >= 1 && p[0] == ':') return 0;
    while (i < n) {
        /* embedded IPv4 tail? */
        uint32_t j = i; int isv4 = 0;
        while (j < n && p[j] != ':') { if (p[j] == '.') isv4 = 1; j++; }
        if (isv4) {
            uint32_t v4;
            if (j != n || ng > 6 || !parse_ipv4(p + i, n - i, &v4)) return 0;
            g[ng++] = (uint16_t)(v4 >> 16); g[ng++] = (uint16_t)(v4 & 0xFFFF);
            i = n; break;
        }
        if (j == i || j - i > 4 || ng >= 8) return 0;
        int v = 0;
        for (uint32_t k = i; k < j; k++) { int h = hexv(p[k]); if (h < 0) return 0; v = v * 16 + h; }
        g[ng++] = (uint16_t)v;
        i = j;
        if (i < n) {            /* at ':' */
            i++;
            if (i < n && p[i] == ':') { if (ell >= 0) return 0; ell = ng; i++; if (i == n) break; }
            else if (i == n) return 0;   /* trailing single ':' */
        }
    }
    if (ell >= 0) {
        if (ng >= 8) return 0;
        int tail = ng - ell;
        memmove(g + 8 - tail, g + ell, (size_t)tail * 2);
        memset(g + ell, 0, (size_t)(8 - ng) * 2);
    } else if (ng != 8) return 0;
    return 1;
}
static val_t do_in_ip_range(ectx_t *c, val_t ip, const uint64_t *cidr) {
    if (ip.tag != CB_T_STRING) return mk_err();
    const uint8_t *p; uint32_t n;
    str_get(c, ip.u, &p, &n);
    int has_colon = 0, has_dot = 0;
    for (uint32_t i = 0; i < n; i++) { if (p[i] == ':') has_colon = 1; if (p[i] == '.') has_dot = 1; if (p[i] == '%') return mk_err(); }
    uint64_t fam = cidr[0], bits = cidr[1], hi = cidr[2], lo = cidr[3];
    int is4 = 0; uint32_t v4 = 0; uint64_t ihi = 0, ilo = 0;
    if (has_dot && !has_colon) { if (!parse_ipv4(p, n, &v4)) return mk_err(); is4 = 1; }
    else if (has_colon) {
        uint16_t g[8];
        if (!parse_ipv6(p, n, g)) return mk_err();
        ihi = ((uint64_t)g[0] << 48) | ((uint64_t)g[1] << 32) | ((uint64_t)g[2] << 16) | g[3];
        ilo = ((uint64_t)g[4] << 48) | ((uint64_t)g[5] << 32) | ((uint64_t)g[6] << 16) | g[7];
        if (ihi == 0 && (ilo >> 32) == 0xFFFF) { is4 = 1; v4 = (uint32_t)ilo; }   /* v4-mapped: ip.To4() succeeds */
    } else return mk_err();
    /* net.IPNet.Contains: compares in 4-byte form when both reduce to IPv4, else lengths must agree */
    uint64_t nfam = fam, nbits = bits, nlo = lo;
    if (fam == 6 && hi == 0 && (lo >> 32) == 0xFFFF && bits >= 96) { nfam = 4; nbits = bits - 96; nlo = lo & 0xFFFFFFFFull; }
    if (is4) {
        if (nfam != 4) return mk_bool(0);
        uint32_t mask = nbits == 0 ? 0 : (uint32_t)(0xFFFFFFFFull << (32 - nbits));
        return mk_bool((v4 & mask) == ((uint32_t)nlo & mask));
    }
    if (nfam != 6) return mk_bool(0);
    uint64_t mhi = bits >= 64 ? ~0ull : (bits == 0 ? 0 : (~0ull << (64 - bits)));
    uint64_t mlo = bits <= 64 ? 0 : (bits == 128 ? ~0ull : (~0ull << (128 - bits)));
    return mk_bool((ihi & mhi) == (hi & mhi) && (ilo & mlo) == (lo & mlo));
}

/* ---- conversions ---- */
static val_t conv_int(ectx_t *c, val_t v) {
    switch (v.tag) {
    case CB_T_INT: return v;
    case CB_T_UINT: if (v.u > (uint64_t)INT64_MAX) return mk_err(); return mk_int((int64_t)v.u);
    case CB_T_DOUBLE: { double d = as_double(v); if (d != d || d <= -9223372036854775808.0 || d >= 9223372036854775808.0) return mk_err(); return mk_int((int64_t)d); }
    case CB_T_STRING: {
        const uint8_t *p; uint32_t n; str_get(c, v.u, &p, &n);
        uint32_t i = 0; int neg = 0;
        if (n && (p[0] == '+' || p[0] == '-')) { neg = p[0] == '-'; i = 1; }
        if (i == n) return mk_err();
        uint64_t acc = 0;
        for (; i < n; i++) {
            if (p[i] < '0' || p[i] > '9') return mk_err();
            if (acc > (UINT64_MAX - 9) / 10) return mk_err();
            acc = acc * 10 + (uint64_t)(p[i] - '0');
        }
        if (neg) { if (acc > (uint64_t)INT64_MAX + 1) return mk_err(); return mk_int((int64_t)(0 - acc)); }
        if (acc > (uint64_t)INT64_MAX) return mk_err();
        return mk_int((int64_t)acc);
    }
    case CB_T_TS: { int64_t ns = (int64_t)v.u; int64_t s = ns / 1000000000; if (ns % 1000000000 < 0) s--; return mk_int(s); }
    case CB_T_DUR: return mk_int((int64_t)v.u);
    default: return mk_err();
    }
}
static val_t conv_uint(ectx_t *c, val_t v) {
    switch (v.tag) {
    case CB_T_UINT: return v;
    case CB_T_INT: if ((int64_t)v.u < 0) return mk_err(); return mk(CB_T_UINT, v.u);
    case CB_T_DOUBLE: { double d = as_double(v); if (d != d || d < 0 || d >= 18446744073709551616.0) return mk_err(); return mk(CB_T_UINT, (uint64_t)d); }
    case CB_T_STRING: {
        const uint8_t *p; uint32_t n; str_get(c, v.u, &p, &n);
        uint32_t i = 0;
        if (n == 0) return mk_err();   /* strconv.ParseUint(s, 10, 64): digits only, "A sign prefix is not permitted" */
        uint64_t acc = 0;
        for (; i < n; i++) {
            if (p[i] < '0' || p[i] > '9') return mk_err();
            uint64_t dg = (uint64_t)(p[i] - '0');
            if (acc > (UINT64_MAX - dg) / 10) return mk_err();
            acc = acc * 10 + dg;
        }
        return mk(CB_T_UINT, acc);
    }
    default: return mk_err();
    }
}
static val_t conv_double(ectx_t *c, val_t v) {
    switch (v.tag) {
    case CB_T_DOUBLE: return v;
    case CB_T_INT: return mk_double((double)(int64_t)v.u);
    case CB_T_UINT: return mk_double((double)v.u);
    case CB_T_STRING: c->unsupported = 1; return mk_err();   /* strconv.ParseFloat at run time: not on the device */
    default: return mk_err();
    }
}

/* ---- loops ---- */
typedef struct { val_t range; uint64_t i, n; int any_err; int64_t count; } loop_t;

static void loop_bind(ectx_t *c, loop_t *L, int var, int two) {
    const uint64_t *p = heap_ptr(c, L->range.u);
    if (L->range.tag == CB_T_LIST) {
        val_t e = decode_v64(p[1 + L->i], 0);
        if (two) { c->vars[var] = mk_int((int64_t)L->i); c->vars[var + 1] = e; } else c->vars[var] = e;
    } else {
        val_t k = decode_v64(p[1 + L->i], 0);
        if (two) { c->vars[var] = k; c->vars[var + 1] = decode_v64(p[1 + L->n + L->i], 0); } else c->vars[var] = k;
    }
}

static val_t and_or(int is_or, val_t a, val_t b) {
    int abool = a.tag == CB_T_BOOL, bbool = b.tag == CB_T_BOOL;
    uint64_t dom = is_or ? 1 : 0;
    if (abool && a.u == dom) return a;
    if (bbool && b.u == dom) return b;
    if (abool && bbool) return mk_bool(!dom);
    return mk_err();
}

static val_t load_slot(ectx_t *c, uint32_t s, int *state) {
    return decode_v64(c->b->slots[(uint64_t)s * c->b->N + c->req], state);
}

static val_t run_program(ectx_t *c, const cb_instr *code, int64_t now) {
    val_t st[CB_MAX_STACK + 2];
    loop_t loops[CB_MAX_LOOP_DEPTH];
    int sp = 0, ld = 0;
    uint32_t pc = 0;
    for (;;) {
        cb_instr in = code[pc++];
        switch (in.op) {
        case CB_OP_RET: return st[sp - 1];
        case CB_OP_CONST: { cb_const k = c->t->consts[in.c]; st[sp++] = mk(k.tag, k.bits); break; }
        case CB_OP_SLOT: { int s; st[sp++] = load_slot(c, in.c, &s); break; }
        case CB_OP_HAS_SLOT: { int s; load_slot(c, in.c, &s); st[sp++] = s == SLOT_ERROR ? mk_err() : mk_bool(s == SLOT_VALUE); break; }
        case CB_OP_PID: st[sp++] = mk(CB_T_STRING, c->b->hdr0[c->req].principal_id); break;
        case CB_OP_NOW: st[sp++] = mk(CB_T_TS, (uint64_t)now); break;
        case CB_OP_VAR: st[sp++] = c->vars[in.a]; break;
        case CB_OP_SELECT: { val_t m = st[sp - 1]; val_t o; if (m.tag == CB_T_MAP && map_find(c, m, mk(CB_T_STRING, in.c), &o)) st[sp - 1] = o; else st[sp - 1] = mk_err(); break; }
        case CB_OP_HAS: { val_t m = st[sp - 1]; st[sp - 1] = m.tag == CB_T_MAP ? mk_bool(map_find(c, m, mk(CB_T_STRING, in.c), 0)) : mk_err(); break; }
        case CB_OP_INDEX: sp--; st[sp - 1] = do_index(c, st[sp - 1], st[sp]); break;
        case CB_OP_EQ: case CB_OP_NE: case CB_OP_LT: case CB_OP_LE: case CB_OP_GT: case CB_OP_GE:
            sp--; st[sp - 1] = do_cmp(c, in.op - CB_OP_EQ, st[sp - 1], st[sp]); break;
        case CB_OP_ADD: case CB_OP_SUB: case CB_OP_MUL: case CB_OP_DIV: case CB_OP_MOD:
            sp--; st[sp - 1] = do_arith(c, in.op, st[sp - 1], st[sp]); break;
        case CB_OP_NEG: {
            val_t v = st[sp - 1];
            if (v.tag == CB_T_INT) st[sp - 1] = (int64_t)v.u == INT64_MIN ? mk_err() : mk_int(-(int64_t)v.u);
            else if (v.tag == CB_T_DOUBLE) st[sp - 1] = mk_double(-as_double(v));
            else if (v.tag == CB_T_DUR) st[sp - 1] = (int64_t)v.u == INT64_MIN ? mk_err() : mk(CB_T_DUR, (uint64_t)(-(int64_t)v.u));
            else st[sp - 1] = mk_err();
            break;
        }
        case CB_OP_NOT: { val_t v = st[sp - 1]; st[sp - 1] = v.tag == CB_T_BOOL ? mk_bool(!v.u) : mk_err(); break; }
        case CB_OP_IN: sp--; st[sp - 1] = do_in(c, st[sp - 1], st[sp]); break;
        case CB_OP_SIZE: {
            val_t v = st[sp - 1];
            if (v.tag == CB_T_STRING) { const uint8_t *p; uint32_t n; str_get(c, v.u, &p, &n); st[sp - 1] = mk_int(utf8_len(p, n)); }
            else if (v.tag == CB_T_LIST || v.tag == CB_T_MAP) st[sp - 1] = mk_int((int64_t)heap_ptr(c, v.u)[0]);
            else st[sp - 1] = mk_err();
            break;
        }
        case CB_OP_STARTS_WITH: case CB_OP_ENDS_WITH: case CB_OP_CONTAINS:
            sp--; st[sp - 1] = do_str2(c, in.op, st[sp - 1], st[sp]); break;
        case CB_OP_JF_KEEP: if (st[sp - 1].tag == CB_T_BOOL && st[sp - 1].u == 0) pc = in.c; break;
        case CB_OP_JT_KEEP: if (st[sp - 1].tag == CB_T_BOOL && st[sp - 1].u == 1) pc = in.c; break;
        case CB_OP_AND: sp--; st[sp - 1] = and_or(0, st[sp - 1], st[sp]); break;
        case CB_OP_OR: sp--; st[sp - 1] = and_or(1, st[sp - 1], st[sp]); break;
        case CB_OP_JMP: pc = in.c; break;
        case CB_OP_TERN: {
            val_t v = st[--sp];
            if (v.tag == CB_T_BOOL) { if (!v.u) pc = in.c; }
            else { st[sp++] = mk_err(); pc = in.b; }
            break;
        }
        case CB_OP_HAS_INTERSECTION: sp--; st[sp - 1] = do_has_intersection(c, st[sp - 1], st[sp]); break;
        case CB_OP_IS_SUBSET: sp--; st[sp - 1] = do_is_subset(c, st[sp - 1], st[sp]); break;
        case CB_OP_LOOP_INIT: {
            val_t r = st[--sp];
            int kind = in.b & 0xFF, two = (in.b >> 8) & 1;
            if (kind > CB_LOOP_EXISTS_ONE) { c->unsupported = 1; return mk_err(); }   /* collecting comprehensions (map / filter / transform*): not in this port */
            if (r.tag != CB_T_LIST && r.tag != CB_T_MAP) { st[sp++] = mk_err(); pc = in.c; break; }
            loop_t *L = &loops[ld];
            L->range = r; L->i = 0; L->n = heap_ptr(c, r.u)[0]; L->any_err = 0; L->count = 0;
            if (L->n == 0) { st[sp++] = mk_bool(kind == CB_LOOP_ALL); pc = in.c; break; }
            ld++;
            loop_bind(c, L, in.a, two);
            break;
        }
        case CB_OP_LOOP_NEXT: {
            val_t r = st[--sp];
            int kind = in.b & 0xFF, two = (in.b >> 8) & 1;
            loop_t *L = &loops[ld - 1];
            int done = 0; val_t res = mk_err();
            if (kind == CB_LOOP_EXISTS_ONE) {
                /* strict fold: any error / non-bool poisons the result */
                if (r.tag != CB_T_BOOL) L->any_err = 1; else if (r.u) L->count++;
            } else {
                uint64_t dom = kind == CB_LOOP_EXISTS ? 1 : 0;
                if (r.tag == CB_T_BOOL) { if (r.u == dom) { done = 1; res = mk_bool((int)dom); } }
                else L->any_err = 1;
            }
            L->i++;
            if (!done && L->i >= L->n) {
                done = 1;
                if (L->any_err) res = mk_err();
                else if (kind == CB_LOOP_EXISTS_ONE) res = mk_bool(L->count == 1);
                else res = mk_bool(kind == CB_LOOP_ALL);
            }
            if (done) { ld--; st[sp++] = res; }
            else { loop_bind(c, L, in.a, two); pc = in.c; }
            break;
        }
        case CB_OP_TO_COND: { val_t v = st[sp - 1]; st[sp - 1] = mk_bool(v.tag == CB_T_BOOL && v.u == 1); break; }
        case CB_OP_COND_NOT: st[sp - 1] = mk_bool(!st[sp - 1].u); break;
        case CB_OP_NOERR: st[sp - 1] = mk_bool(st[sp - 1].tag != CB_T_ERR); break;
        case CB_OP_INT: st[sp - 1] = conv_int(c, st[sp - 1]); break;
        case CB_OP_UINT: st[sp - 1] = conv_uint(c, st[sp - 1]); break;
        case CB_OP_DOUBLE: st[sp - 1] = conv_double(c, st[sp - 1]); break;
        case CB_OP_TIMESTAMP: {
            val_t v = st[sp - 1];
            if (v.tag == CB_T_TS) break;
            if (v.tag == CB_T_STRING) st[sp - 1] = parse_ts(c, v);
            else if (v.tag == CB_T_INT) {
                int64_t s = (int64_t)v.u, ns;
                if (s < -62135596800ll || s > 253402300799ll) st[sp - 1] = mk_err();
                else if (__builtin_mul_overflow(s, (int64_t)1000000000, &ns)) { c->unsupported = 1; st[sp - 1] = mk_err(); }
                else st[sp - 1] = mk(CB_T_TS, (uint64_t)ns);
            } else st[sp - 1] = mk_err();
            break;
        }
        case CB_OP_DURATION: { val_t v = st[sp - 1]; if (v.tag == CB_T_DUR) break; if (v.tag == CB_T_INT) st[sp - 1] = mk(CB_T_DUR, v.u); else if (v.tag == CB_T_STRING) { const uint8_t *p; uint32_t n; int64_t ns = 0; str_get(c, v.u, &p, &n); int rc = parse_go_duration(p, n, &ns); if (rc == 2) c->unsupported = 1; st[sp - 1] = rc == 0 ? mk(CB_T_DUR, (uint64_t)ns) : mk_err(); } else st[sp - 1] = mk_err(); break; }
        case CB_OP_DYN: break;
        case CB_OP_CMP_SLOT_CONST: { int s; val_t a = load_slot(c, in.b, &s); cb_const k = c->t->consts[in.c]; st[sp++] = do_cmp(c, in.a, a, mk(k.tag, k.bits)); break; }
        case CB_OP_CMP_SLOT_SLOT: { int s; val_t a = load_slot(c, in.b, &s); val_t b = load_slot(c, in.c, &s); st[sp++] = do_cmp(c, in.a, a, b); break; }
        case CB_OP_CMP_SLOT_PID: { int s; val_t a = load_slot(c, in.b, &s); st[sp++] = do_cmp(c, in.a, a, mk(CB_T_STRING, c->b->hdr0[c->req].principal_id)); break; }
        case CB_OP_IN_SLOT_CONST: { int s; val_t a = load_slot(c, in.b, &s); cb_const k = c->t->consts[in.c]; st[sp++] = do_in(c, a, mk(k.tag, k.bits)); break; }
        case CB_OP_IN_CONST_SLOT: { int s; val_t a = load_slot(c, in.b, &s); cb_const k = c->t->consts[in.c]; st[sp++] = do_in(c, mk(k.tag, k.bits), a); break; }
        case CB_OP_IN_IP_RANGE: st[sp - 1] = st[sp - 1].tag == CB_T_ERR ? mk_err() : do_in_ip_range(c, st[sp - 1], c->t->theap + in.c); break;
        case CB_OP_HIER_REL: sp--; st[sp - 1] = do_hier_rel(c, in.a, st[sp - 1], in.b, st[sp], in.c); break;
        case CB_OP_TS_GET: {
            int32_t off_s = (int32_t)in.c;
            if (in.b == 2 && st[sp - 1].tag == CB_T_TS) {
                /* an IANA zone name: the UTC offset in force at this instant, from the zone's transition records in THEAP
                 * (table/bytecode.py: iana_zone_words -- [n, first second, end second, n x (from second, offset)]);
                 * scanned linearly here.  Instants the records do not cover are flagged. */
                const uint64_t *z = c->t->theap + in.c;
                const int64_t sec = fdiv((int64_t)st[sp - 1].u, 1000000000ll);
                if (sec < (int64_t)z[1] || sec >= (int64_t)z[2]) { c->unsupported = 1; st[sp - 1] = mk_err(); break; }
                off_s = (int32_t)(int64_t)z[4];
                for (uint64_t k = 0; k < z[0]; k++)
                    if ((int64_t)z[3 + 2 * k] <= sec) off_s = (int32_t)(int64_t)z[3 + 2 * k + 1];
            }
            st[sp - 1] = do_ts_get(in.a, st[sp - 1], in.b, off_s);
            break;
        }
        case CB_OP_IN_SPLIT: {   /* x in s.split(sep): ext strings split + the `in` operator over the token list */
            static __thread hier_t toks;
            sp--;
            val_t x = st[sp - 1], sv = st[sp];
            if (x.tag == CB_T_ERR || sv.tag != CB_T_STRING || !hier_split(c, sv, in.b, &toks)) { st[sp - 1] = mk_err(); break; }
            int found = 0;
            if (x.tag == CB_T_STRING) {
                const uint8_t *px; uint32_t lx;
                str_get(c, x.u, &px, &lx);
                for (uint32_t i = 0; i < toks.n; i++) if (toks.l[i] == lx && memcmp(toks.p[i], px, lx) == 0) found = 1;
            }
            st[sp - 1] = mk_bool(found);
            break;
        }
        case CB_OP_HIER_SIZE: { static __thread hier_t h; st[sp - 1] = hier_split(c, st[sp - 1], in.b, &h) ? mk(CB_T_INT, h.n) : mk_err(); break; }
        case CB_OP_HIER_CA: {
            static __thread hier_t a, b, z;
            if (in.a == 0) {
                sp--;
                int ok = hier_split(c, st[sp - 1], in.b, &a); ok &= hier_split(c, st[sp], in.c & 0xFFFF, &b);
                st[sp - 1] = ok ? mk(CB_T_INT, hier_common_ancestors(&a, &b)) : mk_err();
            } else {
                sp -= 2;
                int ok = hier_split(c, st[sp - 1], in.b, &a); ok &= hier_split(c, st[sp], in.c & 0xFFFF, &b); ok &= hier_split(c, st[sp + 1], in.c >> 16, &z);
                if (!ok) { st[sp - 1] = mk_err(); break; }
                uint32_t k = hier_common_ancestors(&a, &b), eq = z.n == k;
                for (uint32_t i = 0; eq && i < k; i++) eq = hier_seg_eq(&a, i, &z, i);
                st[sp - 1] = mk_bool(eq);
            }
            break;
        }
        default: c->unsupported = 1; return mk_err();
        }
    }
}

/* ------------------------------------------------------------------------------------------- decision walk */
typedef struct {
    ectx_t ec;
    int8_t *memo;          /* per global cond: -1 unknown, 0 false, 1 true */
    uint32_t *memo_touched; uint32_t n_touched;
    int64_t now;
} rctx_t;

static int cond_sat(rctx_t *r, uint32_t gid) {
    if (r->memo[gid] >= 0) return r->memo[gid];
    const cb_cond *cd = &r->ec.t->conds[gid];
    val_t v = run_program(&r->ec, r->ec.t->code + cd->code_off, r->now);
    int s = v.tag == CB_T_BOOL && v.u == 1;
    r->memo[gid] = (int8_t)s;
    r->memo_touched[r->n_touched++] = gid;
    return s;
}

static int build_chain(const table_t *t, uint32_t scope, uint32_t kind_flag, int lenient, uint32_t *chain) {
    int n = 0;
    if (scope == CB_SCOPE_NONE) return 0;
    uint32_t s = scope & ~CB_SCOPE_INEXACT_BIT;
    if (s >= t->nS) return 0;
    if (!(t->scope_flags[s] & kind_flag) && !lenient) return 0;   /* strict: the request scope itself must exist for this kind */
    for (; s != CB_NONE32; s = t->scope_parent[s])
        if (t->scope_flags[s] & kind_flag) chain[n++] = s;
    return n;
}

static int action_matches(const batch_t *b, const table_t *t, uint32_t aset, uint32_t k, uint32_t apat) {
    uint32_t ps = k / b->kc, kk = k % b->kc;
    uint64_t m = b->aset_spread[((uint64_t)ps * b->n_asets + aset) * (t->nAP ? t->nAP : 1) + apat];
    return (int)((m >> (kk * b->role_cols)) & 1);
}

/* hdr0.kind_class: direct pattern id, CB_KIND_NONE, or CSR index (CB_KIND_CLASS_CSR_BIT) */
static uint32_t class_pats(const batch_t *b, uint32_t cls, uint32_t *out) {
    if (cls == CB_KIND_NONE) return 0;
    if (!(cls & CB_KIND_CLASS_CSR_BIT)) { out[0] = cls; return 1; }
    uint32_t c = cls & ~CB_KIND_CLASS_CSR_BIT, n = 0;
    for (uint32_t j = b->class_off[c]; j < b->class_off[c + 1] && n < CB_MAX_CLASS_PATS; j++) out[n++] = b->class_pats[j];
    return n;
}
static int in_pats(const uint32_t *pats, uint32_t n, uint32_t pat) {
    for (uint32_t j = 0; j < n; j++) if (pats[j] == pat) return 1;
    return 0;
}
static int row_action_matches(const batch_t *b, const table_t *t, uint32_t aset, uint32_t k, const cb_row *row) {
    for (uint32_t q = 0; q < row->n_pats; q++) if (action_matches(b, t, aset, k, t->row_apats[row->pat_start + q])) return 1;
    return 0;
}

/* is table role `role` in {request role} U parents(exact resource scope, request role) */
static int role_in_pr(const table_t *t, uint32_t role, uint32_t req_role, uint32_t rscope) {
    if (req_role == role) return 1;
    if (!t->meta[CB_META_HAS_PARENT_ROLES] || req_role >= t->nR) return 0;
    if (rscope == CB_SCOPE_NONE || (rscope & CB_SCOPE_INEXACT_BIT) || rscope >= t->nS) return 0;
    uint64_t idx = (uint64_t)rscope * t->nR + req_role;
    for (uint32_t j = t->par_off[idx]; j < t->par_off[idx + 1]; j++) if (t->par_list[j] == role) return 1;
    return 0;
}

static void check_request(rctx_t *r, uint64_t n, uint8_t *out) {
    const table_t *t = r->ec.t; const batch_t *b = r->ec.b;
    r->ec.req = n;
    for (uint32_t i = 0; i < r->n_touched; i++) r->memo[r->memo_touched[i]] = -1;
    r->n_touched = 0;
    cb_hdr0 h0 = b->hdr0[n]; cb_hdr1 h1 = b->hdr1[n];
    uint32_t K = h1.action_set_id < b->n_asets ? b->aset_k[h1.action_set_id] : 0;
    uint32_t KM = b->b->max_actions;
    for (uint32_t k = 0; k < KM; k++) out[k] = k < K ? CB_EFFECT_DENY : 0;
    uint32_t roles[CB_MAX_ROLE_COLS]; uint32_t n_roles = 0;
    for (uint32_t i = 0; i < b->role_cols; i++) { uint32_t rr = b->roles[(uint64_t)i * b->N + n]; if (rr != CB_ROLE_PAD) roles[n_roles++] = rr; }
    if (n_roles == 0 || K == 0) return;
    int lenient = (b->b->flags & CB_BATCH_FLAG_LENIENT) != 0;
    uint32_t pchain[CB_MAX_CHAIN], rchain[CB_MAX_CHAIN];
    int np = build_chain(t, h0.principal_scope, CB_SCOPE_FLAG_PRINCIPAL, lenient, pchain);
    int nr = build_chain(t, h0.resource_scope, CB_SCOPE_FLAG_RESOURCE, lenient, rchain);
    if (np == 0 && nr == 0) return;
    uint32_t rv = h1.resource_version, pv = h1.principal_version;
    uint32_t kpats[CB_MAX_CLASS_PATS];
    uint32_t n_kp = class_pats(b, h0.kind_class, kpats);
    int p_exists = 0, r_exists = 0;
    if (pv != CB_NONE16) for (int i = 0; i < np; i++) p_exists |= t->prin_exists[(uint64_t)pv * t->nS + pchain[i]];
    if (rv != CB_NONE16)
        for (int i = 0; i < nr; i++)
            for (uint32_t j = 0; j < n_kp; j++)
                r_exists |= t->res_exists[((uint64_t)rv * t->nRP + kpats[j]) * t->nS + rchain[i]] & CB_EXISTS_RESOURCE_KIND;
    if (!p_exists && !r_exists) return;
    if (rv == CB_NONE16) return;   /* candidate rows are filtered by the resource version (ruletable.go:874) */
    uint32_t pidx = h0.principal_id < t->nT ? t->prin_of_string[h0.principal_id] : CB_NONE32;
    uint32_t rscope_exact = h0.resource_scope;

    for (uint32_t k = 0; k < K; k++) {
        int eff = 0;   /* 0 = NO_MATCH */
        /* ---- principal policies (role agnostic; first role only, ruletable.go:905-910) ---- */
        for (int si = 0; si < np && pidx != CB_NONE32; si++) {
            uint32_t s = pchain[si];
            uint32_t bid = t->prin_block_map[((uint64_t)rv * t->nP + pidx) * t->nS + s];
            int saw_allow = 0, deny = 0;
            if (bid != CB_NONE32) {
                cb_block bl = t->blocks[bid];
                for (uint32_t ri = 0; ri < bl.n_rows && !deny; ri++) {
                    cb_row row = t->rows[bl.row_start + ri];
                    if (!in_pats(kpats, n_kp, row.respat)) continue;
                    if (!row_action_matches(b, t, h1.action_set_id, k, &row)) continue;
                    if (row.drcond && !cond_sat(r, bl.cond_base + row.drcond - 1)) continue;
                    if (row.cond && !cond_sat(r, bl.cond_base + row.cond - 1)) continue;
                    if (row.effect == CB_EFFECT_DENY) deny = 1; else saw_allow = 1;
                }
            }
            if (deny) { eff = CB_EFFECT_DENY; break; }
            if (saw_allow) {
                uint32_t perm = (t->scope_flags[s] >> CB_SCOPE_PERM_SHIFT) & 3;
                if (perm == 1) { eff = CB_EFFECT_ALLOW; break; }
            }
        }
        if (eff) { out[k] = (uint8_t)eff; continue; }
        /* ---- resource policies: per role, first ALLOW wins (ruletable.go:1124-1131) ---- */
        for (uint32_t i = 0; i < n_roles && eff != CB_EFFECT_ALLOW; i++) {
            int role_eff = 0;
            for (int si = 0; si < nr && !role_eff; si++) {
                uint32_t s = rchain[si];
                int saw_allow = 0, deny = 0;
                int any_row = 0;
                for (uint32_t j = 0; j < n_kp && !deny; j++) {
                    uint32_t pat = kpats[j];
                    uint64_t mi = ((uint64_t)rv * t->nRP + pat) * t->nS + s;
                    if (t->res_exists[mi] & CB_EXISTS_ANY_ROW) any_row = 1;
                    uint32_t bid = t->res_block_map[mi];
                    if (bid == CB_NONE32) continue;
                    cb_block bl = t->blocks[bid];
                    for (uint32_t ri = 0; ri < bl.n_rows && !deny; ri++) {
                        cb_row row = t->rows[bl.row_start + ri];
                        if (!row_action_matches(b, t, h1.action_set_id, k, &row)) continue;
                        if (row.role != CB_ROLE_ANY && !role_in_pr(t, row.role, roles[i], rscope_exact)) continue;
                        if (row.drcond && !cond_sat(r, bl.cond_base + row.drcond - 1)) continue;
                        if (row.cond && !cond_sat(r, bl.cond_base + row.cond - 1)) continue;
                        if (row.effect == CB_EFFECT_DENY) deny = 1; else saw_allow = 1;
                    }
                }
                /* synthesized role-policy DENY rows (index.go:688-776) */
                if (!deny && any_row && t->meta[CB_META_HAS_ROLE_POLICIES]) {
                    uint64_t ro = (uint64_t)rv * t->nS + s;
                    for (uint32_t e = t->rp_off[ro]; e < t->rp_off[ro + 1] && !deny; e++) {
                        cb_rolepol_entry en = t->rp_entries[e];
                        if (!role_in_pr(t, en.role, roles[i], rscope_exact)) continue;
                        int matched = 0;
                        for (uint32_t q = 0; q < en.n_rules && !deny; q++) {
                            cb_rolepol_rule ru = t->rp_rules[en.rule_start + q];
                            if (!in_pats(kpats, n_kp, ru.respat)) continue;
                            int am = 0;
                            for (uint32_t a = 0; a < ru.n_apats; a++) if (action_matches(b, t, h1.action_set_id, k, t->rp_apats[ru.apat_start + a])) { am = 1; break; }
                            if (!am) continue;
                            matched = 1;
                            if (ru.cond && !cond_sat(r, ru.cond - 1)) deny = 1;   /* DENY none(cond) */
                        }
                        if (!matched) deny = 1;   /* blanket DENY: no allow-action matches */
                    }
                }
                if (deny) { role_eff = CB_EFFECT_DENY; break; }
                if (saw_allow) {
                    uint32_t perm = (t->scope_flags[s] >> CB_SCOPE_PERM_SHIFT) & 3;
                    if (perm == 1) { role_eff = CB_EFFECT_ALLOW; break; }
                }
            }
            if (!eff) eff = role_eff;
            if (role_eff == CB_EFFECT_ALLOW) eff = CB_EFFECT_ALLOW;
        }
        out[k] = (uint8_t)(eff == CB_EFFECT_ALLOW ? CB_EFFECT_ALLOW : CB_EFFECT_DENY);
    }
}

typedef struct { const table_t *t; const batch_t *b; uint64_t lo, hi; uint8_t *out; int unsupported; } job_t;

static void *worker(void *arg) {
    job_t *j = arg;
    rctx_t r; memset(&r, 0, sizeof(r));
    r.ec.t = j->t; r.ec.b = j->b; r.now = j->b->b->now_unix_nanos;
    uint32_t nc = j->t->n_conds ? j->t->n_conds : 1;
    r.memo = malloc(nc); r.memo_touched = malloc(sizeof(uint32_t) * nc);
    memset(r.memo, -1, nc);
    uint32_t KM = j->b->b->max_actions;
    for (uint64_t n = j->lo; n < j->hi; n++) check_request(&r, n, j->out + n * KM);
    j->unsupported = r.ec.unsupported;
    free(r.memo); free(r.memo_touched);
    return 0;
}

int cref_check(const void *blob, size_t blob_len, const cref_batch *batch, uint8_t *effects_out, int n_threads) {
    table_t t; batch_t b;
    int rc = load_table(blob, blob_len, &t);
    if (rc) return rc;
    if (batch->n_columns < N_COLS) return CREF_ERR_BATCH;
    memset(&b, 0, sizeof(b));
    b.t = &t; b.b = batch; b.N = batch->n_requests;
    b.hdr0 = batch->columns[COL_HDR0]; b.hdr1 = batch->columns[COL_HDR1]; b.roles = batch->columns[COL_ROLES];
    b.slots = batch->columns[COL_SLOTS]; b.heap = batch->columns[COL_HEAP]; b.bstr_off = batch->columns[COL_BSTR_OFF];
    b.bstr_bytes = batch->columns[COL_BSTR_BYTES]; b.class_off = batch->columns[COL_CLASS_OFF];
    b.class_pats = batch->columns[COL_CLASS_PATS]; b.aset_k = batch->columns[COL_ASET_K];
    b.aset_spread = batch->columns[COL_ASET_SPREAD];
    if (b.N == 0) return CREF_OK;
    b.role_cols = (uint32_t)(batch->column_bytes[COL_ROLES] / (4 * b.N));
    b.n_asets = (uint32_t)(batch->column_bytes[COL_ASET_K] / 4);
    if (b.role_cols == 0 || b.role_cols > CB_MAX_ROLE_COLS || b.n_asets == 0) return CREF_ERR_BATCH;
    uint32_t km = batch->max_actions ? batch->max_actions : 1;
    b.kc = 64 / b.role_cols; if (b.kc > km) b.kc = km; if (b.kc == 0) b.kc = 1;
    b.n_pass = (km + b.kc - 1) / b.kc;
    if (batch->column_bytes[COL_ASET_SPREAD] < (size_t)8 * b.n_pass * b.n_asets * (t.nAP ? t.nAP : 1)) return CREF_ERR_BATCH;
    if (batch->column_bytes[COL_SLOTS] < (size_t)8 * t.n_slots * b.N) return CREF_ERR_BATCH;
    if (n_threads < 1) n_threads = 1;
    if ((uint64_t)n_threads > b.N) n_threads = (int)b.N;
    pthread_t *th = malloc(sizeof(pthread_t) * (size_t)n_threads);
    job_t *jobs = malloc(sizeof(job_t) * (size_t)n_threads);
    uint64_t per = (b.N + (uint64_t)n_threads - 1) / (uint64_t)n_threads;
    for (int i = 0; i < n_threads; i++) {
        jobs[i].t = &t; jobs[i].b = &b; jobs[i].out = effects_out; jobs[i].unsupported = 0;
        jobs[i].lo = per * (uint64_t)i; jobs[i].hi = jobs[i].lo + per > b.N ? b.N : jobs[i].lo + per;
        if (jobs[i].lo > b.N) jobs[i].lo = b.N;
        pthread_create(&th[i], 0, worker, &jobs[i]);
    }
    int unsup = 0;
    for (int i = 0; i < n_threads; i++) { pthread_join(th[i], 0); unsup |= jobs[i].unsupported; }
    free(th); free(jobs);
    return unsup ? CREF_ERR_UNSUPPORTED : CREF_OK;
}
