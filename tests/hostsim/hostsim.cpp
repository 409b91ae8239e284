// tests/hostsim/hostsim.cpp -- DEBUG AID (test infrastructure, never shipped, never timed).
// Compiles the kernels' per-request core (cerbos_b200/csrc/cb_core.h) for the host so its logic can be
// checked against the oracles on a machine without a GPU.  The product
// library (libcerbos_b200.so) contains no such path: without a CUDA device cgpu_init fails.
#include <cstdint>
#include <cstring>
#include <vector>

#include "cb_core.h"
#include "cb_specialize.h"
#include "cb_uc.h"
#include "cb_encode.h"

#if defined(HOSTSIM_SPEC_UC)
#include "spec_gen.inc"   // generated for one table by hostsim_generate_uc: cb::SpecConds (unique-condition form)
typedef cb::GenericBlocks HostBlocks;
typedef cb::SpecConds HostConds;
#define HOSTSIM_ENTRY hostsim_check_spec
#elif defined(HOSTSIM_SPEC)
#include "spec_gen.inc"   // generated for one table by hostsim_generate (tests/test_specialize.py)
typedef cb::SpecBlocks HostBlocks;
typedef cb::GenericConds HostConds;
#define HOSTSIM_ENTRY hostsim_check_spec
#else
typedef cb::GenericBlocks HostBlocks;
typedef cb::GenericConds HostConds;
#define HOSTSIM_ENTRY hostsim_check
#endif

extern "C" { uint64_t hostsim_deferred = 0; }   // requests the lean / unique-condition body left to the general body in the last call
static bool parse_sections(const void *blob, uint64_t blob_len, uint32_t *off, uint64_t *len) {
    const cb_blob_header *h = static_cast<const cb_blob_header *>(blob);
    if (blob_len < sizeof(*h) || h->magic != CB_MAGIC || h->version != CB_VERSION) return false;
    const cb_section_desc *sd = reinterpret_cast<const cb_section_desc *>(static_cast<const char *>(blob) + sizeof(cb_blob_header));
    for (uint32_t i = 0; i < h->n_sections; i++) if (sd[i].id < 128) { off[sd[i].id] = (uint32_t)sd[i].offset; len[sd[i].id] = sd[i].n_bytes; }
    return true;
}

extern "C" int HOSTSIM_ENTRY(const void *blob, uint64_t blob_len, uint64_t n, uint32_t max_actions, int64_t now, uint32_t flags,
                             const void *const *cols, const uint64_t *col_bytes, uint8_t *bitmap, int mode) {
    const cb_blob_header *h = static_cast<const cb_blob_header *>(blob);
    if (blob_len < sizeof(*h) || h->magic != CB_MAGIC || h->version != CB_VERSION) return -1;
    const cb_section_desc *sd = reinterpret_cast<const cb_section_desc *>(static_cast<const char *>(blob) + sizeof(cb_blob_header));
    const uint8_t *base = static_cast<const uint8_t *>(blob);
    uint64_t off[128] = {0};
    for (uint32_t i = 0; i < h->n_sections; i++) if (sd[i].id < 128) off[sd[i].id] = sd[i].offset;
    const uint32_t *meta = reinterpret_cast<const uint32_t *>(base + off[CB_SEC_META]);
    cb::TableLayout lay;
    memset(&lay, 0, sizeof(lay));
    for (int i = 0; i < 32; i++) lay.off[i] = (uint32_t)off[i];
    lay.uses_runtime = meta[CB_META_USES_RUNTIME];
    lay.nV = meta[CB_META_N_VERSIONS]; lay.nRP = meta[CB_META_N_RESPATS]; lay.nS = meta[CB_META_N_SCOPES]; lay.nP = meta[CB_META_N_PRINCIPALS];
    lay.nR = meta[CB_META_N_ROLES]; lay.nAP = meta[CB_META_N_APATS]; lay.nT = meta[CB_META_N_STRINGS]; lay.n_slots = meta[CB_META_N_SLOTS];
    lay.n_rows = meta[CB_META_N_ROWS] ? meta[CB_META_N_ROWS] : 1;
    lay.has_role_policies = meta[CB_META_HAS_ROLE_POLICIES]; lay.has_parent_roles = meta[CB_META_HAS_PARENT_ROLES];
    lay.has_principal_policies = meta[CB_META_HAS_PRINCIPAL_POLICIES];
    cb::TableView t;
    t.base = base; t.L = &lay;

    cb::BatchView b;
    b.hdr0 = static_cast<const cb_hdr0 *>(cols[0]); b.hdr1 = static_cast<const cb_hdr1 *>(cols[1]);
    b.roles = static_cast<const uint32_t *>(cols[2]); b.slots = static_cast<const uint64_t *>(cols[3]);
    b.heap = static_cast<const uint64_t *>(cols[4]); b.bstr_off = static_cast<const uint32_t *>(cols[5]);
    b.bstr_bytes = static_cast<const uint8_t *>(cols[6]); b.class_off = static_cast<const uint32_t *>(cols[7]);
    b.class_pats = static_cast<const uint32_t *>(cols[8]); b.aset_k = static_cast<const uint32_t *>(cols[9]);
    b.aset_spread = static_cast<const uint64_t *>(cols[10]);
    b.row_am = static_cast<const uint64_t *>(cols[11]);
    b.n_rows = meta[CB_META_N_ROWS] ? meta[CB_META_N_ROWS] : 1;
    b.stride = n; b.first = 0; b.count = n;
    b.role_cols = (uint32_t)(col_bytes[2] / (4 * n)); b.n_asets = (uint32_t)(col_bytes[9] / 4);
    uint32_t km = max_actions ? max_actions : 1;
    b.kc = 64 / b.role_cols; if (b.kc > km) b.kc = km;
    b.n_pass = (km + b.kc - 1) / b.kc; b.max_actions = km; b.kbytes = (km + 7) / 8; b.flags = flags; b.now = now;
    cb::finish_batch_view(b);
    b.n_bstr = col_bytes[5] >= 4 ? (uint32_t)(col_bytes[5] / 4 - 1) : 0;
    b.heap_words = col_bytes[4] / 8;
    uint32_t status = 0;
    hostsim_deferred = 0;
    // mode 0: what the library would pick; 1: force the general 64-bit body; 2: general 32-bit body;
    // 3: the lean body reading a tile of the columns staged the way the kernel's TMA copies lay it out in shared memory
    const bool narrow = b.n_pass == 1 && (uint64_t)km * b.role_cols <= 32;
    uint32_t rcp = 1; while (rcp < b.role_cols) rcp <<= 1;
    const bool fast = narrow && !lay.has_principal_policies && !lay.has_role_policies && !lay.has_parent_roles &&
                      meta[CB_META_DIRECT_KINDS] && (uint64_t)lay.nR * rcp <= 64 && b.kbytes <= 4;
    // modes 4 / 5: the unique-condition body (cb_uc.h image) with rows read from the image / from merged 8-byte records
    if ((mode == 4 || mode == 5) && fast) {
        uint32_t off32[128] = {0};
        uint64_t len64[128] = {0};
        if (!parse_sections(blob, blob_len, off32, len64)) return -1;
        const cbuc::Image uc = cbuc::build(base, off32, len64, meta, lay);
        if (!uc.ok) return -3;
        cb::TableView ut;
        ut.base = uc.bytes.data(); ut.L = &uc.lay;
        std::vector<cb::U4> pk((size_t)b.n_asets * b.n_rows);
        for (size_t j = 0; j < pk.size(); j++) {
            const cb::U4 u = ut.urows()[j % b.n_rows];
            pk[j] = cb::uc_row_record(u, (uint32_t)b.row_am[(j / b.n_rows) * b.n_rows + u.x], b.rcp, lay.nR);
        }
#if defined(HOSTSIM_SPEC_UC)
        // the per-string predicate words the library's pre-pass kernel would compute (one per table / batch string)
        std::vector<uint32_t> strpred(lay.nT + b.n_bstr + 1, 0);
        if (HostConds::n_strpred)
            for (uint32_t id = 0; id < lay.nT + b.n_bstr; id++) strpred[id] = HostConds().strpred(ut, b, id);
        b.strpred = strpred.data();
#endif
        for (uint64_t i = 0; i < n; i++) {
            cb::CachedCols gc; gc.b = &b; gc.n = i;
            bool d;
            if (mode == 5) { cb::UcRowsPacked rows; rows.pk = pk.data(); d = cb::eval_request_uc(ut, b, gc, rows, i, bitmap, nullptr, HostConds()); }
            else { cb::UcRowsGlobal rows; rows.urows = ut.urows(); rows.row_am = b.row_am; rows.RCP = b.rcp; rows.nR = lay.nR; d = cb::eval_request_uc(ut, b, gc, rows, i, bitmap, nullptr, HostConds()); }
            if (d) { hostsim_deferred++; cb::eval_request_general(t.base, t.L, &b, i, bitmap, nullptr, &status); }
        }
        return status ? -2 : 0;
    }
    if (mode == 3 && fast) {
        std::vector<uint64_t> tile(cb::tile_cols_bytes(b.role_cols, lay.n_slots) / 8 + 2);
        uint8_t *tb = reinterpret_cast<uint8_t *>(tile.data());
        for (uint64_t t0 = 0; t0 < n; t0 += cb::CB_TILE) {
            const uint64_t cnt = n - t0 < cb::CB_TILE ? n - t0 : cb::CB_TILE;
            memcpy(tb, b.hdr0 + t0, cnt * 16);
            memcpy(tb + cb::CB_TILE * 16, b.hdr1 + t0, cnt * 8);
            for (uint32_t i = 0; i < b.role_cols; i++) memcpy(tb + cb::CB_TILE * 24 + i * cb::CB_TILE * 4, b.roles + i * b.stride + t0, cnt * 4);
            const uint32_t so = cb::CB_TILE * (24 + 4 * b.role_cols);
            for (uint32_t v = 0; v < lay.n_slots; v++) memcpy(tb + so + v * cb::CB_TILE * 8, b.slots + v * b.stride + t0, cnt * 8);
            for (uint32_t j = 0; j < cnt; j++) {
                cb::TileCols tc; tc.base = tb; tc.tid = j; tc.slots_off = so; tc.aset_k_s = b.aset_k; tc.row_am_s = b.row_am; tc.res_s = nullptr;
                if (cb::eval_request_fast(t, b, tc, t0 + j, bitmap, nullptr, HostBlocks())) cb::eval_request_general(t.base, t.L, &b, t0 + j, bitmap, nullptr, &status);
            }
        }
        return status ? -2 : 0;
    }
    for (uint64_t i = 0; i < n; i++) {
        if (mode == 0 && fast) {
            cb::GlobalCols gc; gc.b = &b; gc.n = i;
            if (cb::eval_request_fast(t, b, gc, i, bitmap, nullptr, HostBlocks())) cb::eval_request_general(t.base, t.L, &b, i, bitmap, nullptr, &status);
        }
        else if (mode == 2 && narrow) cb::eval_request<uint32_t>(t, b, i, bitmap, nullptr, &status);
        else cb::eval_request<uint64_t>(t, b, i, bitmap, nullptr, &status);
    }
    return status ? -2 : 0;
}

#if !defined(HOSTSIM_SPEC) && !defined(HOSTSIM_SPEC_UC)
// the native batch encoder (cb_encode.h): n serialized CheckInput messages -> the twelve columns; the caller reads them
// back through hostsim_encoded_column() and releases with hostsim_encoded_free()
struct HostEncoded { cbenc::Columns cols; };
extern "C" void *hostsim_encode(const void *blob, uint64_t blob_len, const char *default_version, const char *default_scope, int lenient,
                                const void *const *inputs, const uint64_t *lens, uint64_t n, uint32_t *dims /* max_actions, role_cols, kc, n_pass */, uint32_t n_threads) {
    cbenc::Encoder enc;
    cbenc::Conf conf;
    conf.default_version = default_version; conf.default_scope = default_scope; conf.lenient = lenient != 0;
    if (!enc.init(blob, blob_len, conf)) return nullptr;
    std::vector<size_t> ls(lens, lens + n);
    HostEncoded *he = new HostEncoded();
    if (!enc.encode(inputs, ls.data(), n, &he->cols, n_threads)) { delete he; return nullptr; }
    dims[0] = he->cols.max_actions; dims[1] = he->cols.role_cols; dims[2] = he->cols.kc; dims[3] = he->cols.n_pass;
    return he;
}
extern "C" const void *hostsim_encoded_column(const void *h, int i, uint64_t *bytes) {
    const HostEncoded *he = static_cast<const HostEncoded *>(h);
    *bytes = he->cols.bytes(i);
    return he->cols.ptr(i);
}
extern "C" void hostsim_encoded_free(void *h) { delete static_cast<HostEncoded *>(h); }

// the decision-metadata body (cb::eval_request_meta): effects + per-action metadata words + per-request metadata
extern "C" int hostsim_check_meta(const void *blob, uint64_t blob_len, uint64_t n, uint32_t max_actions, int64_t now, uint32_t flags,
                                  const void *const *cols, const uint64_t *col_bytes, uint8_t *effects, uint32_t *action_meta, cb_request_meta *req_meta) {
    const cb_blob_header *h = static_cast<const cb_blob_header *>(blob);
    if (blob_len < sizeof(*h) || h->magic != CB_MAGIC || h->version != CB_VERSION) return -1;
    const cb_section_desc *sd = reinterpret_cast<const cb_section_desc *>(static_cast<const char *>(blob) + sizeof(cb_blob_header));
    const uint8_t *base = static_cast<const uint8_t *>(blob);
    uint64_t off[128] = {0};
    for (uint32_t i = 0; i < h->n_sections; i++) if (sd[i].id < 128) off[sd[i].id] = sd[i].offset;
    const uint32_t *meta = reinterpret_cast<const uint32_t *>(base + off[CB_SEC_META]);
    cb::TableLayout lay;
    memset(&lay, 0, sizeof(lay));
    for (int i = 0; i < 32; i++) lay.off[i] = (uint32_t)off[i];
    lay.nV = meta[CB_META_N_VERSIONS]; lay.nRP = meta[CB_META_N_RESPATS]; lay.nS = meta[CB_META_N_SCOPES]; lay.nP = meta[CB_META_N_PRINCIPALS];
    lay.nR = meta[CB_META_N_ROLES]; lay.nAP = meta[CB_META_N_APATS]; lay.nT = meta[CB_META_N_STRINGS]; lay.n_slots = meta[CB_META_N_SLOTS];
    lay.n_rows = meta[CB_META_N_ROWS] ? meta[CB_META_N_ROWS] : 1;
    lay.has_role_policies = meta[CB_META_HAS_ROLE_POLICIES]; lay.has_parent_roles = meta[CB_META_HAS_PARENT_ROLES];
    lay.has_principal_policies = meta[CB_META_HAS_PRINCIPAL_POLICIES]; lay.uses_runtime = meta[CB_META_USES_RUNTIME];
    cb::BatchView b;
    b.hdr0 = static_cast<const cb_hdr0 *>(cols[0]); b.hdr1 = static_cast<const cb_hdr1 *>(cols[1]);
    b.roles = static_cast<const uint32_t *>(cols[2]); b.slots = static_cast<const uint64_t *>(cols[3]);
    b.heap = static_cast<const uint64_t *>(cols[4]); b.bstr_off = static_cast<const uint32_t *>(cols[5]);
    b.bstr_bytes = static_cast<const uint8_t *>(cols[6]); b.class_off = static_cast<const uint32_t *>(cols[7]);
    b.class_pats = static_cast<const uint32_t *>(cols[8]); b.aset_k = static_cast<const uint32_t *>(cols[9]);
    b.aset_spread = static_cast<const uint64_t *>(cols[10]); b.row_am = static_cast<const uint64_t *>(cols[11]);
    b.n_rows = lay.n_rows; b.stride = n; b.first = 0; b.count = n;
    b.role_cols = (uint32_t)(col_bytes[2] / (4 * n)); b.n_asets = (uint32_t)(col_bytes[9] / 4);
    uint32_t km = max_actions ? max_actions : 1;
    b.kc = 64 / b.role_cols; if (b.kc > km) b.kc = km;
    b.n_pass = (km + b.kc - 1) / b.kc; b.max_actions = km; b.kbytes = (km + 7) / 8; b.flags = flags; b.now = now;
    cb::finish_batch_view(b);
    b.n_bstr = col_bytes[5] >= 4 ? (uint32_t)(col_bytes[5] / 4 - 1) : 0;
    b.heap_words = col_bytes[4] / 8;
    uint32_t status = 0;
    for (uint64_t i = 0; i < n; i++) cb::eval_request_meta(base, &lay, &b, i, effects, action_meta, req_meta, &status);
    return status ? -2 : 0;
}
// the unique-condition form of the specialised source (cb::SpecConds); "" if the table does not qualify; *n_uconds_out = distinct conditions
extern "C" int64_t hostsim_generate_uc(const void *blob, uint64_t blob_len, char *out, uint64_t cap, uint32_t *n_uconds_out) {
    uint32_t off[128] = {0};
    uint64_t len[128] = {0};
    if (!parse_sections(blob, blob_len, off, len)) return -1;
    const uint8_t *base = static_cast<const uint8_t *>(blob);
    const uint32_t *meta = reinterpret_cast<const uint32_t *>(base + off[CB_SEC_META]);
    cb::TableLayout lay;
    memset(&lay, 0, sizeof(lay));
    for (int i = 0; i < 32; i++) lay.off[i] = off[i];
    lay.nR = meta[CB_META_N_ROLES]; lay.n_slots = meta[CB_META_N_SLOTS];
    const cbuc::Image uc = cbuc::build(base, off, len, meta, lay);
    if (n_uconds_out) *n_uconds_out = uc.ok ? uc.n_uconds : 0;
    std::string src = uc.ok ? cbspec::generate_uc(uc.bytes.data(), uc.lay.off, uc.lay.uc_conds_off, uc.n_uconds, lay.n_slots, meta[CB_META_N_CONSTS]).src : std::string();
    if (src.size() + 1 > cap) return -(int64_t)src.size() - 2;
    memcpy(out, src.c_str(), src.size() + 1);
    return (int64_t)src.size();
}
// the table-specialised block evaluators the library would hand to NVRTC (source text; "" if the table does not qualify)
extern "C" int64_t hostsim_generate(const void *blob, uint64_t blob_len, char *out, uint64_t cap) {
    const cb_blob_header *h = static_cast<const cb_blob_header *>(blob);
    if (blob_len < sizeof(*h) || h->magic != CB_MAGIC || h->version != CB_VERSION) return -1;
    const cb_section_desc *sd = reinterpret_cast<const cb_section_desc *>(static_cast<const char *>(blob) + sizeof(cb_blob_header));
    uint32_t off[128] = {0};
    for (uint32_t i = 0; i < h->n_sections; i++) if (sd[i].id < 128) off[sd[i].id] = (uint32_t)sd[i].offset;
    const uint8_t *base = static_cast<const uint8_t *>(blob);
    std::string src = cbspec::generate(base, off, reinterpret_cast<const uint32_t *>(base + off[CB_SEC_META]));
    if (src.size() + 1 > cap) return -(int64_t)src.size() - 2;
    memcpy(out, src.c_str(), src.size() + 1);
    return (int64_t)src.size();
}
#endif
