// cb_host.h -- how a table and a batch are set up on the host, shared by the library (cerbos_b200.cu) and its host build
// (tests/hostsim): blob parsing, batch views, and which kernel bodies a table and batch may take.  Plain C++17, no CUDA;
// not part of the device code (cb_core.h and the NVRTC translation unit do not include it).
#pragma once
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>

#include "cb_core.h"
#include "cb_uc.h"
#include "cerbos_b200.h"

namespace cbhost {

constexpr int kMaxSec = 32;   // section ids the image carries (cb::TableLayout::off); higher ids are host-only

// The checks below report failure as a message ("" = success).
inline std::string msg(const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    return buf;
}

// Validates the blob (every section against the blob length, overflow-safe; every section META sizes) and fills the
// layout, the META words and the byte length of every section.
inline std::string parse_blob(const void *blob, size_t len, cb::TableLayout *lay, uint32_t *meta, uint64_t *sec_len) {
    if (!blob || len < sizeof(cb_blob_header)) return "table blob too small";
    const cb_blob_header *h = static_cast<const cb_blob_header *>(blob);
    if (h->magic != CB_MAGIC) return "table blob: bad magic";
    if (h->version != CB_VERSION) return msg("table blob: version %u, library expects %u", h->version, CB_VERSION);
    if (h->total_bytes > len || sizeof(cb_blob_header) + (size_t)h->n_sections * sizeof(cb_section_desc) > len)
        return "table blob truncated";
    const cb_section_desc *sd = reinterpret_cast<const cb_section_desc *>(static_cast<const char *>(blob) + sizeof(cb_blob_header));
    memset(lay, 0, sizeof(*lay));
    uint64_t image_end = 0;
    bool seen[kMaxSec] = {false};
    for (uint32_t i = 0; i < h->n_sections; i++) {
        if (sd[i].offset > len || sd[i].n_bytes > len - sd[i].offset || (sd[i].offset & 15)) return msg("table blob: bad section %u", sd[i].id);
        if (sd[i].id == CB_SEC_MANIFEST) continue;   // host-only
        if (sd[i].id >= kMaxSec) continue;
        if (sd[i].offset > 0xFFFFFFF0ull) return "table blob too large";
        lay->off[sd[i].id] = (uint32_t)sd[i].offset;
        sec_len[sd[i].id] = sd[i].n_bytes;
        seen[sd[i].id] = true;
        uint64_t end = (sd[i].offset + sd[i].n_bytes + 15) & ~15ull;
        if (end > image_end) image_end = end;
        if (sd[i].id == CB_SEC_META) {
            if (sd[i].n_bytes < CB_META_WORDS * 4) return "table blob: short META";
            memcpy(meta, static_cast<const char *>(blob) + sd[i].offset, CB_META_WORDS * 4);
        }
    }
    for (int id = CB_SEC_META; id <= CB_SEC_DR_NAME_STR; id++)
        if (!seen[id]) return msg("table blob: missing section %d", id);
    if (image_end > 0xFFFFFFF0ull) return "table blob too large";
    if (image_end > len) image_end = len;   // the last device section may end unaligned at the end of the blob (sections themselves are bounds-checked above)
    lay->image_bytes = (uint32_t)image_end;
    lay->nV = meta[CB_META_N_VERSIONS]; lay->nRP = meta[CB_META_N_RESPATS]; lay->nS = meta[CB_META_N_SCOPES];
    lay->nP = meta[CB_META_N_PRINCIPALS]; lay->nR = meta[CB_META_N_ROLES]; lay->nAP = meta[CB_META_N_APATS];
    lay->nT = meta[CB_META_N_STRINGS]; lay->n_slots = meta[CB_META_N_SLOTS]; lay->n_rows = meta[CB_META_N_ROWS] ? meta[CB_META_N_ROWS] : 1;
    lay->has_role_policies = meta[CB_META_HAS_ROLE_POLICIES]; lay->has_parent_roles = meta[CB_META_HAS_PARENT_ROLES];
    lay->has_principal_policies = meta[CB_META_HAS_PRINCIPAL_POLICIES];
    lay->uses_runtime = meta[CB_META_USES_RUNTIME];
    struct { int id; uint64_t need; } chk[] = {
        {CB_SEC_SCOPE_PARENT, 4ull * lay->nS}, {CB_SEC_SCOPE_FLAGS, 4ull * lay->nS},
        {CB_SEC_RES_BLOCK_MAP, 4ull * lay->nV * lay->nRP * lay->nS}, {CB_SEC_RES_EXISTS, 1ull * lay->nV * lay->nRP * lay->nS},
        {CB_SEC_PRIN_BLOCK_MAP, 4ull * lay->nV * lay->nP * lay->nS}, {CB_SEC_PRIN_EXISTS, 1ull * lay->nV * lay->nS},
        {CB_SEC_BLOCKS, 16ull * meta[CB_META_N_BLOCKS]}, {CB_SEC_ROWS, 16ull * meta[CB_META_N_ROWS]}, {CB_SEC_CONDS, 16ull * meta[CB_META_N_CONDS]},
        {CB_SEC_CODE, 8ull * meta[CB_META_N_CODE]}, {CB_SEC_CONSTS, 16ull * meta[CB_META_N_CONSTS]}, {CB_SEC_CONSTS_V64, 8ull * meta[CB_META_N_CONSTS]},
        {CB_SEC_STR_OFF, 4ull * (lay->nT + 1)}, {CB_SEC_THEAP, 8ull * meta[CB_META_THEAP_WORDS]},
        {CB_SEC_BLOCK_SLOTS_OFF, 4ull * (meta[CB_META_N_BLOCKS] + 1)}, {CB_SEC_DR_OFF, 4ull * (meta[CB_META_N_BLOCKS] + 1)},
        {CB_SEC_DR_NAME_STR, 4ull * meta[CB_META_N_DR_NAMES]},
    };
    for (const auto &c : chk)
        if (sec_len[c.id] < c.need) return msg("table blob: section %d holds %llu bytes, META needs %llu", c.id, (unsigned long long)sec_len[c.id], (unsigned long long)c.need);
    if (meta[CB_META_MAX_STACK] > CB_MAX_STACK || meta[CB_META_MAX_LOOP_DEPTH] > CB_MAX_LOOP_DEPTH || meta[CB_META_N_VARS] > CB_MAX_VARS)
        return "table blob needs a deeper interpreter than this build provides";
    return "";
}

// Validates the batch against the table and fills the view (pointers are used as given).
inline std::string make_batch_view(const cb::TableLayout &lay, const cgpu_batch *b, uint64_t first, uint64_t count, cb::BatchView *v) {
    if (!b || b->n_columns < CGPU_N_COLUMNS || !b->columns || !b->column_bytes) return msg("batch: expected %d columns", CGPU_N_COLUMNS);
    const uint64_t N = b->n_requests;
    if (N == 0) return "batch: empty";
    const size_t *cb_ = b->column_bytes;
    if (cb_[CGPU_COL_HDR0] < N * 16 || cb_[CGPU_COL_HDR1] < N * 8) return "batch: header columns too small";
    if (cb_[CGPU_COL_ROLES] % (4 * N) != 0) return "batch: roles column is not a multiple of n_requests";
    uint32_t role_cols = (uint32_t)(cb_[CGPU_COL_ROLES] / (4 * N));
    if (role_cols == 0 || role_cols > CB_MAX_ROLE_COLS) return msg("batch: %u role columns (supported 1..%d)", role_cols, CB_MAX_ROLE_COLS);
    if (cb_[CGPU_COL_SLOTS] < (size_t)8 * lay.n_slots * N) return msg("batch: slot columns too small for the table's %u slots", lay.n_slots);
    uint32_t n_asets = (uint32_t)(cb_[CGPU_COL_ASET_K] / 4);
    if (n_asets == 0) return "batch: no action sets";
    uint32_t km = b->max_actions ? b->max_actions : 1;
    uint32_t kc = 64 / role_cols;
    if (kc > km) kc = km;
    uint32_t n_pass = (km + kc - 1) / kc;
    uint32_t nAP = lay.nAP ? lay.nAP : 1;
    if (cb_[CGPU_COL_ASET_SPREAD] < (size_t)8 * n_pass * n_asets * nAP) return "batch: aset_spread too small";
    if (cb_[CGPU_COL_ROW_AM] < (size_t)8 * n_pass * n_asets * lay.n_rows) return "batch: row_am too small";
    for (int i = 0; i < CGPU_N_COLUMNS; i++)
        if (!b->columns[i]) return msg("batch: column %d is null", i);
    v->hdr0 = static_cast<const cb_hdr0 *>(b->columns[CGPU_COL_HDR0]);
    v->hdr1 = static_cast<const cb_hdr1 *>(b->columns[CGPU_COL_HDR1]);
    v->roles = static_cast<const uint32_t *>(b->columns[CGPU_COL_ROLES]);
    v->slots = static_cast<const uint64_t *>(b->columns[CGPU_COL_SLOTS]);
    v->heap = static_cast<const uint64_t *>(b->columns[CGPU_COL_HEAP]);
    v->bstr_off = static_cast<const uint32_t *>(b->columns[CGPU_COL_BSTR_OFF]);
    v->bstr_bytes = static_cast<const uint8_t *>(b->columns[CGPU_COL_BSTR_BYTES]);
    v->class_off = static_cast<const uint32_t *>(b->columns[CGPU_COL_CLASS_OFF]);
    v->class_pats = static_cast<const uint32_t *>(b->columns[CGPU_COL_CLASS_PATS]);
    v->aset_k = static_cast<const uint32_t *>(b->columns[CGPU_COL_ASET_K]);
    v->aset_spread = static_cast<const uint64_t *>(b->columns[CGPU_COL_ASET_SPREAD]);
    v->row_am = static_cast<const uint64_t *>(b->columns[CGPU_COL_ROW_AM]);
    v->n_rows = lay.n_rows;
    v->stride = N; v->first = first; v->count = count;
    v->role_cols = role_cols; v->n_asets = n_asets; v->kc = kc; v->n_pass = n_pass; v->max_actions = km;
    v->kbytes = (km + 7) / 8; v->flags = b->flags; v->now = b->now_unix_nanos;
    cb::finish_batch_view(*v);
    v->n_bstr = cb_[CGPU_COL_BSTR_OFF] >= 4 ? (uint32_t)(cb_[CGPU_COL_BSTR_OFF] / 4 - 1) : 0;
    v->heap_words = cb_[CGPU_COL_HEAP] / 8;
    return "";
}

// Which bodies a table and batch may take.  The library's launch plan adds what depends on its context and on the
// kernels compiled for the table; the host build takes these alone.

// Resource-policy-only tables (no principal / role policies, no parent roles) whose kinds resolve without resource globs:
// the only tables a lean kernel body can evaluate.
inline bool lean_table(const cb::TableLayout &lay, const uint32_t *meta) {
    return !lay.has_principal_policies && !lay.has_role_policies && !lay.has_parent_roles && meta[CB_META_DIRECT_KINDS];
}
// The lean body: a lean table, one pass whose (action x role column) pair masks fit 32 bits, and a role table of 64 bits.
inline bool lean_eligible(const cb::TableLayout &lay, const uint32_t *meta, const cb::BatchView &bv) {
    return bv.n_pass == 1 && (uint64_t)bv.max_actions * bv.role_cols <= 32 && bv.kbytes <= 4 && lean_table(lay, meta) &&
           (uint64_t)lay.nR * bv.rcp <= 64;
}
// The unique-condition body, on top of the lean body's conditions: a built image, 32-bit request indices and merged-row
// counts, and a role word with room for the "any role" column nR.
inline bool uc_eligible(const cb::TableLayout &lay, const cbuc::Image &uc, const cb::BatchView &bv) {
    return uc.ok && (uint64_t)(lay.nR + 1) * bv.rcp <= 64 && bv.count < (1ull << 32) && (uint64_t)bv.n_asets * lay.n_rows < (1ull << 31);
}

}  // namespace cbhost
